"""CPU (-m "not gpu"): the device group's C-ABI (include/vqcuda_group.h) without a device. The band plans are the single owner of
the row split for C and C++ callers, so they must return exactly what vqengine_b200/distributed.py returns for the torch path; every
argument refusal happens before a device is touched; the header is plain C and the library exports what it declares, while the two
headers whose entry points are tabled elsewhere (vqcuda.h, vqcuda_prefilter_multi.h) do not see the group's functions."""
import ctypes as C
import os
import re
import subprocess

import pytest

from vqengine_b200 import distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vqcuda_group.h")


def test_band_rows_equal_python(vq):
    for n in range(1, 9):
        for rows in range(0, 601):
            eq, ev = dist.equal_tiles(rows, n), dist.even_tiles(rows, n)
            for r in range(n):
                assert vq.band_rows(rows, n, r) == eq[r], (rows, n, r)
                assert vq.band_rows(rows, n, r, even=True) == ev[r], (rows, n, r)


def test_specular_rank_ranges_equal_python(vq):
    for res in range(1, 1025):
        for mips in range(1, vq.mip_level_count(res, res) + 1):
            for n in range(1, 9):
                plan = dist.InterleavedSpecularPlan(res, mips, n)
                for r in range(n):
                    assert vq.specular_rank_ranges(res, mips, n, r) == plan.row_ranges(r), (res, mips, n, r)


def _refused(vq, rc, words):
    assert rc == vq.VQ_ERR_INVALID_ARG, rc
    msg = vq.lib.vq_last_error().decode()
    assert words in msg, msg


def test_band_rows_refusals(vq):
    a, b = C.c_int(), C.c_int()
    for args, words in [((-1, 2, 0, 0), "n_rows"), ((10, 0, 0, 0), "n_ranks"), ((10, 9, 0, 0), "n_ranks"), ((10, 2, 2, 0), "rank"),
                        ((10, 2, -1, 0), "rank"), ((10, 2, 0, 2), "even")]:
        _refused(vq, vq.lib.vq_band_rows(*args, C.byref(a), C.byref(b)), words)
    _refused(vq, vq.lib.vq_band_rows(10, 2, 0, 0, None, C.byref(b)), "null output")


def test_specular_rank_ranges_refusals(vq):
    n = C.c_int()
    buf = (C.c_int * 32)()
    for args, words in [((0, 1, 1, 0), "res"), ((128, 0, 1, 0), "mips"), ((128, 9, 1, 0), "mips"), ((128, 4, 0, 0), "n_ranks"),
                        ((128, 4, 9, 0), "n_ranks"), ((128, 4, 2, 2), "rank")]:
        _refused(vq, vq.lib.vq_specular_rank_ranges(*args, buf, 16, C.byref(n)), words)
    _refused(vq, vq.lib.vq_specular_rank_ranges(128, 4, 2, 0, None, 4, C.byref(n)), "null ranges")
    _refused(vq, vq.lib.vq_specular_rank_ranges(128, 4, 2, 0, buf, 3, C.byref(n)), "capacity")
    assert n.value == 4, "the count is reported with a too-small capacity"
    _refused(vq, vq.lib.vq_specular_rank_ranges(128, 4, 2, 0, buf, 4, None), "n_ranges")
    assert vq.lib.vq_specular_rank_ranges(128, 4, 2, 0, None, 0, C.byref(n)) == vq.VQ_ERR_INVALID_ARG and n.value == 4


def test_group_refusals_without_device(vq):
    """every check of vq_group_create, vq_group_rank_order and vq_group_signal runs before a context is read or a device touched:
    the contexts here are addresses of host words, never dereferenced"""
    words = (C.c_uint64 * 8)()
    fake = [C.addressof(words) + 8 * i for i in range(8)]
    out = C.c_void_p()
    ctxs = lambda lst: (C.c_void_p * max(len(lst), 1))(*lst)
    _refused(vq, vq.lib.vq_group_create(ctxs(fake[:2]), 2, None, None), "out is null")
    _refused(vq, vq.lib.vq_group_create(None, 2, None, C.byref(out)), "ctxs is null")
    for n in (0, 9, -1):
        _refused(vq, vq.lib.vq_group_create(ctxs(fake + [fake[0]]), n, None, C.byref(out)), "n_ranks")
    _refused(vq, vq.lib.vq_group_create(ctxs([fake[0], None, fake[2]]), 3, None, C.byref(out)), "null context")
    _refused(vq, vq.lib.vq_group_create(ctxs([fake[0], fake[1], fake[0]]), 3, None, C.byref(out)), "appears twice")
    flags = (C.c_void_p * 2)(C.addressof(words), None)
    _refused(vq, vq.lib.vq_group_create(ctxs(fake[:2]), 2, flags, C.byref(out)), "null flag array")
    assert not out.value
    o = (C.c_int * 8)()
    _refused(vq, vq.lib.vq_group_rank_order(None, 0, o), "null group")
    _refused(vq, vq.lib.vq_group_signal(None, 0, 1, C.byref(vq.PeerSignal())), "null group")
    _refused(vq, vq.lib.vq_group_arrive(None, 0, 1, None), "null group")
    assert vq.lib.vq_group_destroy(None) == vq.VQ_OK


def test_header_is_c99_and_exported(vq, tmp_path):
    hdr = open(HEADER).read()
    declared = sorted(set(re.findall(r"VQ_API\s+[\w\s\*]+?\b(vq_\w+)\s*\(", hdr)))
    assert declared == sorted(vq.GROUP_SYMBOLS), set(declared) ^ set(vq.GROUP_SYMBOLS)
    for name in declared:
        assert hasattr(vq.lib, name), f"libvqcuda.so does not export {name}"
    src = tmp_path / "g.c"
    src.write_text('#include "vqcuda_group.h"\nint main(void) { VqGroup* g = 0; return vq_group_destroy(g); }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only",
                           "-I", os.path.join(ROOT, "include"), str(src)])


def test_tabled_headers_do_not_declare_group_calls():
    """vqcuda.h and vqcuda_prefilter_multi.h have a table row for each of their signalled and stream entry points; the group's
    declarations live in their own header so that those tables stay complete"""
    for name in ("vqcuda.h", "vqcuda_prefilter_multi.h"):
        text = open(os.path.join(ROOT, "include", name)).read()
        assert "vq_group_" not in text and "vq_band_rows" not in text and "vq_specular_rank_ranges" not in text
        assert "vqcuda_group.h" not in text
