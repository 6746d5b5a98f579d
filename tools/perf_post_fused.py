"""GPU-box helper: RenderPostProcess in one launch (vq_post_process) against the three-call chain it replaces
(vq_tonemap -> vq_fsr_easu -> vq_fsr_rcas), at 3840x2160 -> 7680x4320 (exact 2x) and 2560x1440 -> 3840x2160 (FSR "quality",
the upscaling path).

  python tools/perf_post_fused.py [--rounds 5] [--iters 50]

Per size, after warm-up, the two are timed alternately (`rounds` times each, CUDA events, `iters` launches per timing) and the
median is reported with the spread, the fraction of the data-sheet HBM bandwidth (3.35 TB/s) the algorithmic bytes make
(16 B per input pixel + 16 B per output pixel for the fused call, plus both intermediates written and read again for the
chain), the intermediate memory the fused call does not allocate, and whether the two display frames are the same bits.
The card's name and power limit are read in the same run."""
import argparse, json, os, statistics, sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
import vqengine_b200 as vq
from vqengine_b200 import synth
import bench
from perf_multi_shading import card

DATASHEET_BPS = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    ctx = vq.Context(0)
    res = {"card": card(0), "lib": vq.LIB_PATH}
    for name, (iw, ih, ow, oh) in {"4k_to_8k_2x": (3840, 2160, 7680, 4320), "1440p_to_4k": (2560, 1440, 3840, 2160)}.items():
        src = torch.from_numpy(synth.hdr_image(iw, ih)).cuda()
        tm = synth.default_tonemapper()
        easu, rcas = vq.fsr_easu_con(iw, ih, iw, ih, ow, oh), vq.fsr_rcas_con(0.2)
        t = torch.empty((ih, iw, 4), dtype=torch.float32, device="cuda")
        e, r, f = (torch.empty((oh, ow, 4), dtype=torch.float32, device="cuda") for _ in range(3))

        def chain():
            ctx.tonemap(tm, src, t)
            ctx.fsr_easu(easu, t, e)
            ctx.fsr_rcas(rcas, e, r)

        def fused():
            ctx.post_process(tm, src, f, easu=easu, rcas=rcas)

        singles = {"vq_tonemap": lambda: ctx.tonemap(tm, src, t), "vq_fsr_easu": lambda: ctx.fsr_easu(easu, t, e),
                   "vq_fsr_rcas": lambda: ctx.fsr_rcas(rcas, e, r)}
        chain(); fused()
        torch.cuda.synchronize()
        same = bool(torch.equal(r.view(torch.int32), f.view(torch.int32)))
        times = {"chain": [], "fused": []}
        for _ in range(a.rounds):                      # alternate: both see the same clocks and neighbours
            times["chain"].append(bench.time_gpu(torch, chain, a.iters))
            times["fused"].append(bench.time_gpu(torch, fused, a.iters))
        single_ms = {k: bench.time_gpu(torch, fn, a.iters) for k, fn in singles.items()}
        nin, nout = iw * ih, ow * oh
        fused_bytes = 16 * nin + 16 * nout
        chain_bytes = 32 * nin + (16 * nin + 16 * nout) + 32 * nout
        row = {"in": f"{iw}x{ih}", "out": f"{ow}x{oh}", "same_bits": same,
               "intermediate_mb_saved": round((16 * nin + 16 * nout) / 1e6, 1),
               "fused_algorithmic_mb": round(fused_bytes / 1e6, 1), "chain_algorithmic_mb": round(chain_bytes / 1e6, 1),
               "singles_ms": {k: round(v, 4) for k, v in single_ms.items()}}
        for k, v in times.items():
            med = statistics.median(v)
            nb = fused_bytes if k == "fused" else chain_bytes
            row[k] = {"ms_median": round(med, 4), "ms_min": round(min(v), 4), "ms_max": round(max(v), 4),
                      "fraction_of_3.35TBps": round(nb / (med * 1e-3) / DATASHEET_BPS, 3)}
        row["speedup"] = round(row["chain"]["ms_median"] / row["fused"]["ms_median"], 3)
        res[name] = row
        print(name, json.dumps(row), flush=True)
        del src, t, e, r, f
        torch.cuda.empty_cache()
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
