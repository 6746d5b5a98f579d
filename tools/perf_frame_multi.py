"""GPU-box helper: the band forms of the skydome and the reflection composite (vq_skydome_multi_signal,
vq_apply_reflections_multi_signal) on one GPU.

  python tools/perf_frame_multi.py [--iters 10]

Workload: a 7680x4320 frame of bench.py's synthetic G-buffer whose top 40 % is cleared sky (normal 0), bench.py's registered
environment and its 2048x1024 HDRI (level 0 is what the sky samples). Timed with CUDA events (bench.time_gpu):
  * the full-frame vq_skydome under the G-buffer's normal plane, and vq_apply_reflections (bounding volumes off and on);
  * the band calls for even_tiles(4320, N), N = 2, 4, 8: each rank's band (the slowest rank is reported) into 1 destination and into
    N local destinations (local stand-ins for the peers' frames: the stores stay in this GPU's HBM, so no NVLink time is in them);
  * the scene-colour step of a rank: vq_forward_lighting_multi into its local frame + vq_skydome_multi_signal into N frames, against
    vq_forward_lighting_multi into N frames alone.
No signal is passed: a rendezvous needs the other ranks. A multi-GPU step time needs two or more GPUs and is not taken here. The
card's name and power limit are read in the same run."""
import argparse, json, os, sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
import vqengine_b200 as vq
from vqengine_b200 import synth
from vqengine_b200.distributed import even_tiles
import bench
from perf_multi_shading import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "perf_frame_multi.py needs a CUDA device"
    W, H = bench.W8K, bench.H8K
    ctx = vq.Context(0)
    envk = bench.build_env_maps_gpu(ctx, vq, torch)
    planes = [torch.from_numpy(p).cuda() for p in synth.gbuffer(W, H)]
    sky_rows = int(0.4 * H)
    planes[1][:sky_rows, :, :3] = 0.0
    gb = vq.GBuffer(vq.image_of(planes[0]), vq.image_of(planes[1]), vq.image_of(planes[2]), vq.null_image())
    pf, pv = synth.scene_constants(W, H, envk["spec_mips"])
    env = envk["env"]
    _, inv = synth.sky_view_proj(0.7, 0.1, 1.0, W / H)
    m = inv.astype(np.float32).reshape(16)
    pyr = vq.Pyramid(envk["pyr_t"].data_ptr(), envk["hdri_w"], envk["hdri_h"], 1)
    mask = planes[1]
    frames = [torch.zeros((H, W, 4), dtype=torch.float32, device="cuda") for _ in range(8)]
    imgs = [vq.image_of(f) for f in frames]
    refl, bvol = torch.rand((H, W, 4), device="cuda"), torch.rand((H, W, 4), device="cuda")

    def t(fn):
        return round(bench.time_gpu(torch, fn, a.iters), 4)

    res = {"card": card(0), "frame": f"{W}x{H}", "sky_rows": sky_rows, "iters": a.iters,
           "full_frame": {"skydome": t(lambda: ctx.skydome(m, pyr, frames[0], normal_mask=mask)),
                          "apply_reflections": t(lambda: ctx.apply_reflections(frames[0], refl)),
                          "apply_reflections_bv": t(lambda: ctx.apply_reflections(frames[0], refl, bvol)),
                          "forward_lighting": t(lambda: ctx.forward_lighting(pf, pv, gb, env, frames[0]))}}
    print("full_frame", json.dumps(res["full_frame"]), flush=True)
    for n in (2, 4, 8):
        bands = even_tiles(H, n)
        row = {}
        for dests in (1, n):
            outs = imgs[:dests]
            # the slowest band: the sky covers the top 40 %, so the first ranks' bands are mostly sky
            row[f"skydome_{dests}_dest"] = max(
                t(lambda: ctx.skydome_multi(m, pyr, outs, 0, normal_mask=mask, row_begin=b0, row_end=b1)) for b0, b1 in bands)
            row[f"apply_reflections_{dests}_dest"] = max(
                t(lambda: ctx.apply_reflections_multi(refl[b0:b1], outs, b0)) for b0, b1 in bands)
        step_sky, step_fwd = [], []
        for b0, b1 in bands:
            step_sky.append(t(lambda: (ctx.forward_lighting_multi(pf, pv, gb, env, imgs[:1], 0, row_begin=b0, row_end=b1),
                                       ctx.skydome_multi(m, pyr, imgs[:n], 0, normal_mask=mask, row_begin=b0, row_end=b1))))
            step_fwd.append(t(lambda: ctx.forward_lighting_multi(pf, pv, gb, env, imgs[:n], 0, row_begin=b0, row_end=b1)))
        row["step_forward_1_dest_plus_skydome_n_dest"] = max(step_sky)
        row["step_forward_n_dest"] = max(step_fwd)
        row["per_band_step_forward_1_plus_skydome_n"] = step_sky
        row["per_band_step_forward_n"] = step_fwd
        res[f"n{n}"] = row
        print(f"n{n}", json.dumps(row), flush=True)
    res["multi_gpu_step"] = "not measured (needs torchrun on two or more GPUs)"
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
