"""The stream contract (tests/test_stream_contract_gpu.py, part 1) for the environment prefilter's band calls and the cube blur:
each call only enqueues on its stream, leaves its outputs untouched until the work ahead of it has run, and then stores the bits of
the ungated call. The three calls are declared in include/vqcuda_prefilter_multi.h, which vqcuda.h includes; the CPU test checks that the table below
names every entry point of that header that takes a stream."""
import os
import re

import pytest
import torch

import vqengine_b200 as vq
from test_stream_contract_gpu import (ROWS, Row, _mipped_hdri, _sentinels, _snapshot, assert_bits, gate, legacy, reference,  # noqa: F401
                                      scene, sctx, sg, stream_entry_points, streams)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMPANION = os.path.join(ROOT, "include", "vqcuda_prefilter_multi.h")


def _cubes(res, n):
    return [torch.empty((vq.cubemap_texel_count(res, 1), 4), dtype=torch.float32, device="cuda") for _ in range(n)]


def r_diffuse_multi(S, seed):
    d, p = _mipped_hdri(S.ctx, seed)
    outs = _cubes(8, 2)
    cubes = [vq.cubemap_of(o, 8, 1) for o in outs]
    return Row([d], outs, lambda c, s: c.diffuse_irradiance_multi(p, cubes, n_phi=16, n_theta=4, src_mip=2, row_begin=5, row_end=40,
                                                                  stream=s), keep=(p, cubes))


def r_lut_multi(S, seed):
    outs = [torch.empty((24, 40, 2), dtype=torch.float32, device="cuda") for _ in range(3)]
    return Row([], outs, lambda c, s: c.brdf_integration_lut_multi([vq.image_of(o, 2) for o in outs], 64, row_begin=2, row_end=21,
                                                                   stream=s))


def r_blur_cube(S, seed, inplace=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    src = torch.randn((vq.cubemap_texel_count(16, 1), 4), device="cuda", generator=g)
    o = src if inplace else _cubes(16, 1)[0]
    return Row([src], [o], lambda c, s: c.gaussian_blur_cube(vq.cubemap_of(src, 16, 1), vq.cubemap_of(o, 16, 1), stream=s))


NEW_ROWS = {
    "diffuse_irradiance multi_signal": (("vq_diffuse_irradiance_multi_signal",), r_diffuse_multi),
    "brdf_integration_lut multi_signal": (("vq_brdf_integration_lut_multi_signal",), r_lut_multi),
    "gaussian_blur_cube": (("vq_gaussian_blur_cube",), r_blur_cube),
    "gaussian_blur_cube in place": (("vq_gaussian_blur_cube",), lambda S, k: r_blur_cube(S, k, inplace=True)),
}


def companion_stream_entry_points():
    """every VQ_API function of vqcuda_prefilter_multi.h with a `void* stream` parameter (the parse of stream_entry_points)"""
    text = re.sub(r"/\*.*?\*/", " ", open(COMPANION).read(), flags=re.S)
    return {m.group(1) for m in re.finditer(r"VQ_API\s+[\w\s\*]*?\b(vq_\w+)\s*\(([^;]*)\)\s*;", text)
            if re.search(r"\bvoid\s*\*\s*stream\b", m.group(2))}


def test_every_companion_stream_entry_point_has_a_row():
    """CPU: the table above names every entry point of vqcuda_prefilter_multi.h that takes a stream, and nothing else; vqcuda.h
    includes that header, and its own entry points are the stream contract's table's (tests/test_stream_contract_gpu.py)"""
    want = companion_stream_entry_points()
    assert want == {"vq_diffuse_irradiance_multi_signal", "vq_brdf_integration_lut_multi_signal", "vq_gaussian_blur_cube"}, sorted(want)
    have = set().union(*(covers for covers, _ in NEW_ROWS.values()))
    assert have == want, (sorted(have), sorted(want))
    assert not want & stream_entry_points() and not want & set().union(*(covers for covers, _ in ROWS.values()))
    assert '#include "vqcuda_prefilter_multi.h"' in open(os.path.join(ROOT, "include", "vqcuda.h")).read()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(NEW_ROWS))
def test_enqueues_behind_earlier_work(sctx, scene, gate, streams, name):
    s, s2 = streams
    row = NEW_ROWS[name][1](scene, 7)
    ref = reference(row, sctx, s)
    snaps = [torch.empty_like(o) for o in row.outs]
    _sentinels(row)
    assert all(_snapshot(snaps, row.outs, s2))
    with gate.closed(s) as go:
        row.prime(s)
        row.run(sctx, s)
        st = gate.status()
        assert st in ("armed", "waiting"), f"{name}: the call returned with the gate {st}: it waited for earlier work on its stream"
        legacy().synchronize()
        held = _snapshot(snaps, row.outs, s2)
        assert all(held), f"{name}: outputs {[k for k, h in enumerate(held) if not h]} were written before the gate opened"
        go.set()
    s.synchronize()
    assert gate.status() == "opened"
    assert_bits(name, row.outs, ref)
