"""GPU-box helper: the 21-tap Gaussian blur in one launch (vq_gaussian_blur) against the two calls it replaces
(vq_gaussian_blur_x into a temporary, then vq_gaussian_blur_y), and its band form (vq_gaussian_blur_multi_signal) on one rank's
band of equal_tiles(H, N), N = 2, 4, 8, into 1 and into N local destinations, at 3840x2160 and 7680x4320.

  python tools/perf_blur.py [--rounds 7] [--iters 50]

Per size, after warm-up, the two-call blur and the one-launch blur are timed alternately (`rounds` times each, CUDA events,
`iters` launches per timing); the median is reported with the spread, and the fraction of the data-sheet HBM bandwidth
(3.35 TB/s) the algorithmic bytes make: 32 B/px for the one-launch blur (each input pixel read once, each output pixel written
once; its recomputed 10-row halo, 20 rows per 64-row tile, is read again through L2 and not counted), 64 B/px for the two calls
(the temporary written and read again). The band call is timed on rank N/2's band (an interior band, with a halo on both
sides), alternating with the one-launch call, and compared with 1/N of that call. Also whether the two blurs give the same bits.
The card's name, power limit and SM clock (before and after the timings) are read in the same run."""
import argparse, json, os, statistics, subprocess, sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
import vqengine_b200 as vq
from vqengine_b200 import synth
from vqengine_b200.distributed import equal_tiles
import bench
from perf_multi_shading import card

DATASHEET_BPS = 3.35e12


def sm_clock():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=20).stdout.strip()
    return q


def stats(v, nbytes=None):
    med = statistics.median(v)
    row = {"ms_median": round(med, 4), "ms_min": round(min(v), 4), "ms_max": round(max(v), 4)}
    if nbytes is not None:
        row["fraction_of_3.35TBps"] = round(nbytes / (med * 1e-3) / DATASHEET_BPS, 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    ctx = vq.Context(0)
    res = {"card": card(0), "clock_before": sm_clock(), "lib": vq.LIB_PATH}
    for name, (w, h) in {"3840x2160": (3840, 2160), "7680x4320": (7680, 4320)}.items():
        src = torch.from_numpy(synth.hdr_image(w, h)).cuda()
        p = vq.BlurParams(w, h)
        tmp, out2, out1 = (torch.empty((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(3))

        def two_calls():
            ctx.gaussian_blur(src, tmp, vertical=False)
            ctx.gaussian_blur(tmp, out2, vertical=True)

        def one_launch():
            ctx.gaussian_blur2d(p, src, out1)

        two_calls(); one_launch()
        torch.cuda.synchronize()
        same = bool(torch.equal(out1.view(torch.int32), out2.view(torch.int32)))
        times = {"two_calls": [], "one_launch": []}
        for _ in range(a.rounds):                      # alternate: both see the same clocks and neighbours
            times["two_calls"].append(bench.time_gpu(torch, two_calls, a.iters))
            times["one_launch"].append(bench.time_gpu(torch, one_launch, a.iters))
        npx = w * h
        row = {"same_bits": same, "temporary_mb_saved": round(16 * npx / 1e6, 1),
               "two_calls": stats(times["two_calls"], 64 * npx), "one_launch": stats(times["one_launch"], 32 * npx)}
        row["speedup"] = round(row["two_calls"]["ms_median"] / row["one_launch"]["ms_median"], 3)
        bands = {}
        for n in (2, 4, 8):
            r0, r1 = equal_tiles(h, n)[n // 2]
            peers = [torch.empty((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(n - 1)]
            for nd in (1, n):
                dests = [vq.image_of(out1)] + [vq.image_of(t) for t in peers[:nd - 1]]

                def band():
                    ctx.gaussian_blur_multi(p, src, dests, r0, r1)

                tb, tf = [], []
                for _ in range(a.rounds):
                    tb.append(bench.time_gpu(torch, band, a.iters))
                    tf.append(bench.time_gpu(torch, one_launch, a.iters))
                rows = r1 - r0
                nbytes = 16 * w * (min(r1 + 10, h) - max(r0 - 10, 0)) + 16 * w * rows * nd
                bands[f"N{n}_dests{nd}"] = {"rows": [r0, r1], **stats(tb, nbytes), "one_launch_ms_median": round(statistics.median(tf), 4),
                                            "ideal_ms": round(statistics.median(tf) / n, 4)}
            del peers
        row["band"] = bands
        res[name] = row
        print(name, json.dumps(row), flush=True)
        del src, tmp, out1, out2
        torch.cuda.empty_cache()
    res["clock_after"] = sm_clock()
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
