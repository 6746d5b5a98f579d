"""No GPU needed: which rows each post pass of a rank's band must produce. vq_fsr_easu_source_rows against a float32 brute force of
the EASU tap rule (the rows f-1 .. f+2 of every output row's 'f' = floor(fl(y * con0.y) + con0.w), folded as the sampler folds
them), and distributed.post_chain_rows against the stencils of the passes it plans."""
import numpy as np
import pytest

import vqengine_b200 as vq
from vqengine_b200.distributed import equal_tiles, post_chain_rows

MODES = (vq.VQ_ADDRESS_WRAP, vq.VQ_ADDRESS_CLAMP)


def con0_y(con):
    c = np.frombuffer(bytes(con), np.uint32)[:4].view(np.float32)
    return c[1], c[3]


def brute_reads(con, in_h, out_h, mode):
    """[out_h, in_h] bool: the input rows each output row reads (float32 arithmetic, unfused, as the kernels' easu_pos)"""
    scale, bias = con0_y(con)
    y = np.arange(out_h, dtype=np.float32)
    f = np.floor((y * scale).astype(np.float32) + bias).astype(np.int64)
    taps = f[:, None] + np.arange(-1, 3)[None, :]
    taps = taps % in_h if mode == vq.VQ_ADDRESS_WRAP else np.clip(taps, 0, in_h - 1)
    reads = np.zeros((out_h, in_h), bool)
    reads[np.repeat(np.arange(out_h), 4), taps.ravel()] = True
    return reads


def ranges_of(mask):
    """increasing, disjoint, non-adjacent [begin, end) runs of a bool row mask"""
    d = np.diff(np.concatenate([[0], mask.astype(np.int8), [0]]))
    return list(zip(np.flatnonzero(d == 1).tolist(), np.flatnonzero(d == -1).tolist()))


def bands(out_h):
    return sorted({t for n in range(1, 9) for t in equal_tiles(out_h, n)} | {(0, 0), (out_h, out_h), (0, 1), (out_h - 1, out_h)})


def check(con, in_h, out_h, mode):
    cum = np.concatenate([np.zeros((1, in_h), np.int32), np.cumsum(brute_reads(con, in_h, out_h, mode), axis=0, dtype=np.int32)])
    for a, b in bands(out_h):
        want = ranges_of(cum[b] - cum[a] > 0)
        got = vq.fsr_easu_source_rows(con, in_h, out_h, a, b, address_mode=mode)
        assert got == want, (con0_y(con), in_h, out_h, mode, (a, b), got, want)
        assert len(got) <= 2


def viewports(in_h):
    """every viewport height up to 24 input rows; above, the edges and the middle of the range (the full sweep takes minutes)"""
    return range(1, in_h + 1) if in_h <= 24 else sorted({1, 2, in_h // 3, in_h // 2, in_h - 1, in_h})


@pytest.mark.parametrize("in_h", range(1, 65))
def test_source_rows_every_viewport_and_ratio(in_h):
    """FsrEasuCon with viewport <= input height, every output height from half to twice the input, every band of equal_tiles for
    1..8 ranks plus single rows at both edges, both address modes"""
    for vp in viewports(in_h):
        for out_h in range((in_h + 1) // 2, 2 * in_h + 1):
            con = vq.fsr_easu_con(16, vp, 16, in_h, 16, out_h)
            for mode in MODES:
                check(con, in_h, out_h, mode)


@pytest.mark.parametrize("ratio", [0.77, 0.67, 0.58, 0.50])
@pytest.mark.parametrize("out_w,out_h", [(1920, 1080), (2560, 1440), (3840, 2160)])
def test_source_rows_presets(ratio, out_w, out_h):
    """the engine's FSR presets (render scale per axis) at 1080p, 1440p and 4K"""
    in_w, in_h = int(out_w * ratio), int(out_h * ratio)
    con = vq.fsr_easu_con(in_w, in_h, in_w, in_h, out_w, out_h)
    for mode in MODES:
        check(con, in_h, out_h, mode)


def test_source_rows_2x_at_4k():
    con = vq.fsr_easu_con(3840, 2160, 3840, 2160, 7680, 4320)
    for mode in MODES:
        check(con, 2160, 4320, mode)
    # WRAP: the first and last bands also read the opposite edge; CLAMP never does
    assert vq.fsr_easu_source_rows(con, 2160, 4320, 0, 541) == [(0, 272), (2158, 2160)]
    assert vq.fsr_easu_source_rows(con, 2160, 4320, 3779, 4320) == [(0, 2), (1888, 2160)]
    assert vq.fsr_easu_source_rows(con, 2160, 4320, 0, 541, address_mode=vq.VQ_ADDRESS_CLAMP) == [(0, 272)]


@pytest.mark.parametrize("args", [(0, 1, -1, 4), (0, 1, 5, 4), (0, 1, 0, 9), (0, 0, 0, 1), (0, 1, 0, 1, 3), (0, -1, 0, 1)])
def test_source_rows_refusals(args):
    """rows outside the output or reversed, zero heights, an unknown address mode"""
    con = vq.fsr_easu_con(4, 4, 4, 4, 8, 8)
    in_h, out_h, a, b = 4, 8, 0, 8
    if len(args) == 4:
        _, _, a, b = args
    if args == (0, 0, 0, 1):
        in_h = 0
    if args == (0, -1, 0, 1):
        out_h = 0
    mode = args[4] if len(args) == 5 else vq.VQ_ADDRESS_WRAP
    with pytest.raises(vq.VqError):
        vq.fsr_easu_source_rows(con, in_h, out_h, a, b, address_mode=mode)


def test_source_rows_refuses_constants_outside_the_image():
    con = vq.fsr_easu_con(4, 4, 4, 4, 8, 8)
    con[3] = int(np.float32(40.0).view(np.uint32))
    with pytest.raises(vq.VqError, match="taps outside"):
        vq.fsr_easu_source_rows(con, 4, 8, 0, 8)
    con[3] = int(np.float32(np.nan).view(np.uint32))
    with pytest.raises(vq.VqError, match="not finite"):
        vq.fsr_easu_source_rows(con, 4, 8, 0, 8)


def _stencil_rows(rows, halo, n):
    """the rows a pass with a +-halo row stencil (zero border) reads to produce `rows`"""
    s = set()
    for a, b in rows:
        s |= set(range(max(a - halo, 0), min(b + halo, n)))
    return s


def _covered(rows):
    return {y for a, b in rows for y in range(a, b)}


CHAINS = [("fsr", 270, 540, vq.VQ_ADDRESS_WRAP), ("fsr", 270, 540, vq.VQ_ADDRESS_CLAMP), ("fsr", 37, 61, vq.VQ_ADDRESS_WRAP),
          ("fsr", 2160, 4320, vq.VQ_ADDRESS_WRAP), ("fsr_preset", 1662, 2160, vq.VQ_ADDRESS_WRAP), ("cas", 53, 53, None),
          ("tonemap", 53, 53, None)]


@pytest.mark.parametrize("kind,in_h,out_h,mode", CHAINS)
def test_post_chain_rows_feed_every_stage(kind, in_h, out_h, mode):
    """each stage produces at least the rows the next stage reads for its rows, and the last stage produces exactly the band"""
    for n in range(1, 9):
        for band in equal_tiles(out_h, n):
            if kind.startswith("fsr"):
                in_w = in_h * 16 // 9
                con = vq.fsr_easu_con(in_w, in_h, in_w, in_h, out_h * 16 // 9, out_h)
                plan = post_chain_rows(in_h, out_h, band, fsr_con=con, address_mode=mode)
                assert list(plan) == ["tonemap", "fsr_easu", "fsr_rcas"]
                assert _covered(plan["fsr_rcas"]) == set(range(*band))
                assert _stencil_rows(plan["fsr_rcas"], 1, out_h) <= _covered(plan["fsr_easu"])
                reads = brute_reads(con, in_h, out_h, mode)
                need = {int(r) for a, b in plan["fsr_easu"] for r in np.flatnonzero(reads[a:b].any(axis=0))}
                assert need <= _covered(plan["tonemap"])
                assert len(plan["tonemap"]) <= 2
            elif kind == "cas":
                plan = post_chain_rows(in_h, out_h, band, cas=True)
                assert list(plan) == ["tonemap", "cas"]
                assert _covered(plan["cas"]) == set(range(*band))
                assert _stencil_rows(plan["cas"], 1, out_h) <= _covered(plan["tonemap"])
            else:
                plan = post_chain_rows(in_h, out_h, band)
                assert list(plan) == ["tonemap"] and _covered(plan["tonemap"]) == set(range(*band))
            for rows in plan.values():
                assert all(a < b for a, b in rows)


def test_post_chain_rows_empty_band():
    con = vq.fsr_easu_con(8, 8, 8, 8, 16, 16)
    assert post_chain_rows(8, 16, (5, 5), fsr_con=con) == {"tonemap": [], "fsr_easu": [], "fsr_rcas": []}
    assert post_chain_rows(8, 8, (0, 0), cas=True) == {"tonemap": [], "cas": []}
