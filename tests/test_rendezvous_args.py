"""CPU (-m "not gpu"): the rendezvous policy's C-ABI (include/vqcuda_rendezvous.h) and its group calls (vqcuda_group.h) without a
device. The header is plain C, the library exports what it declares and the package binds it; every argument refusal happens before
a device is touched; the headers whose entry points are tabled elsewhere (vqcuda.h, vqcuda_prefilter_multi.h) do not declare the
new calls. The contexts and groups here are zeroed host memory, never used as more than the fields the checks read."""
import ctypes as C
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vqcuda_rendezvous.h")
NEW_GROUP_CALLS = ["vq_group_set_rendezvous_deadline", "vq_group_cancel", "vq_group_barrier"]


def _refused(vq, rc, words):
    assert rc == vq.VQ_ERR_INVALID_ARG, rc
    msg = vq.lib.vq_last_error().decode()
    assert words in msg, msg


def _zeroed():
    """a zeroed host block standing in for a VqContext or a VqGroup that has nothing registered"""
    buf = (C.c_uint64 * 8192)()
    return buf, C.c_void_p(C.addressof(buf))


def test_header_is_c99_and_exported(vq, tmp_path):
    hdr = open(HEADER).read()
    declared = sorted(set(re.findall(r"VQ_API\s+[\w\s\*]+?\b(vq_\w+)\s*\(", hdr)))
    assert declared == sorted(vq.RENDEZVOUS_SYMBOLS), set(declared) ^ set(vq.RENDEZVOUS_SYMBOLS)
    for name in declared + NEW_GROUP_CALLS:
        assert hasattr(vq.lib, name), f"libvqcuda.so does not export {name}"
        assert getattr(vq.lib, name).argtypes, f"{name} is not bound"
    assert set(NEW_GROUP_CALLS) <= set(vq.GROUP_SYMBOLS)
    m = re.search(r"#define\s+VQ_RENDEZVOUS_MAX_DEADLINE_NS\s+(\d+)ull", hdr)
    assert m and int(m.group(1)) == vq.RENDEZVOUS_MAX_DEADLINE_NS == 20 * 10 ** 9
    src = tmp_path / "r.c"
    src.write_text('#include "vqcuda_rendezvous.h"\n'
                   'int main(void) { VqRendezvousStatus s; VqContext* c = 0; return vq_ctx_rendezvous_status(c, 0, &s); }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only",
                           "-I", os.path.join(ROOT, "include"), str(src)])


def test_status_layout(vq):
    assert C.sizeof(vq.RendezvousStatus) == 20
    assert [f for f, _ in vq.RendezvousStatus._fields_] == ["failures", "first_epoch", "last_epoch", "missing_mask", "cancelled"]
    st = vq.RendezvousStatus(1, 5, 5, 0b10100, 0)
    assert st.missing_ranks() == [2, 4]


def test_tabled_headers_do_not_declare_the_policy():
    """the stream and signal tables of vqcuda.h and vqcuda_prefilter_multi.h stay complete without rows for the new calls"""
    for name in ("vqcuda.h", "vqcuda_prefilter_multi.h"):
        text = open(os.path.join(ROOT, "include", name)).read()
        assert "#include \"vqcuda_rendezvous.h\"" not in text
        for sym in ["vq_ctx_set_rendezvous_deadline", "vq_ctx_cancel_rendezvous", "vq_ctx_rendezvous_status",
                    "vq_ctx_rendezvous_clear"] + NEW_GROUP_CALLS:
            assert sym not in text, (name, sym)


def test_context_refusals(vq):
    lib = vq.lib
    st = vq.RendezvousStatus()
    _refused(vq, lib.vq_ctx_set_rendezvous_deadline(None, 100_000_000), "null context")
    _refused(vq, lib.vq_ctx_cancel_rendezvous(None), "null context")
    _refused(vq, lib.vq_ctx_rendezvous_status(None, None, C.byref(st)), "null context")
    _refused(vq, lib.vq_ctx_rendezvous_clear(None, None), "null context")
    keep, ctx = _zeroed()
    for ns in (0, vq.RENDEZVOUS_MAX_DEADLINE_NS + 1, 2 ** 64 - 1):
        _refused(vq, lib.vq_ctx_set_rendezvous_deadline(ctx, ns), "deadline")
    _refused(vq, lib.vq_ctx_cancel_rendezvous(ctx), "no rendezvous deadline")
    _refused(vq, lib.vq_ctx_rendezvous_status(ctx, None, None), "out is null")
    # nothing registered: an all-zero record and nothing to clear, with no device work
    st.failures = 7
    assert lib.vq_ctx_rendezvous_status(ctx, None, C.byref(st)) == vq.VQ_OK and st.failures == 0
    assert lib.vq_ctx_rendezvous_clear(ctx, None) == vq.VQ_OK
    assert not any(keep), "a refused or empty call wrote into the context"


def test_group_refusals(vq):
    lib = vq.lib
    _refused(vq, lib.vq_group_set_rendezvous_deadline(None, 1000), "null group")
    _refused(vq, lib.vq_group_cancel(None), "null group")
    _refused(vq, lib.vq_group_barrier(None, 0, 1, None), "null group")
    keep, g = _zeroed()
    for ns in (0, vq.RENDEZVOUS_MAX_DEADLINE_NS + 1):
        _refused(vq, lib.vq_group_set_rendezvous_deadline(g, ns), "deadline")
    for rank in (-1, 0, 1):                 # the zeroed group has no ranks
        _refused(vq, lib.vq_group_barrier(g, rank, 1, None), "rank out of range")
    assert not any(keep)
