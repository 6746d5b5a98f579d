"""GPU-box helper: how much of K1's time is the size of its IBL sampling copies? Times the unchanged forward pass at 4K (the
bench's G-buffer and lights) over a grid of BRDF LUT and specular cube sizes. The instruction stream is the same at every point
(9 specular mips, so the same mip selection); only the bytes the gathers spread over change, and with them how much of the copies
L2 can hold next to the streamed G-buffer. Each point is prepared (vq_environment_prepare) before it is timed. The whole grid runs
twice; the card, its power limit and the SM clock right after each timing are printed with it."""
import os, subprocess, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import vqengine_b200 as vq
from vqengine_b200 import synth
import bench

W, H = bench.W4K, bench.H4K
DIFF_RES, SPEC_MIPS = 64, 9
LUTS, SPECS = (1024, 724, 512, 256), (512, 256)


def up(b):
    return (b + 255) // 256 * 256


def cube_copy_bytes(res, mips):          # vq_forward.cu padded_bytes: bordered texels + one mip-0 row and a texel of slack
    return (sum(6 * ((res >> m) + 2) ** 2 for m in range(mips)) + res + 3) * 16


def lut_copy_bytes(n):                   # vq_forward.cu lut_pair_bytes: (W+2) x (H+1) column-pair texels of 16 bytes
    return (n + 2) * (n + 1) * 16


def gpu_query(fields):
    r = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else "nvidia-smi unavailable"


def main():
    print(f"card: {gpu_query('name,power.limit,clocks.max.sm')}", flush=True)
    ctx = vq.Context(0)
    planes = synth.gbuffer(W, H, seed=synth.SEED_BASE + 3)
    pf, pv = synth.scene_constants(W, H, SPEC_MIPS)
    dpl = [torch.from_numpy(p).cuda() for p in planes]
    gb = vq.GBuffer(vq.image_of(dpl[0]), vq.image_of(dpl[1]), vq.image_of(dpl[2]), vq.null_image())
    out = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
    envs = {(l, s): bench.build_env_maps_gpu(ctx, vq, torch, diff_res=DIFF_RES, spec_res=s, spec_mips=SPEC_MIPS, lut=l)
            for l in LUTS for s in SPECS}
    for rep in range(2):
        us = {}
        for (l, s), envk in envs.items():
            ctx.environment_prepare(envk["env"])
            ms = bench.time_gpu(torch, lambda: ctx.forward_lighting(pf, pv, gb, envk["env"], out), 30, warmup=5)
            clk = gpu_query("clocks.sm")
            mb = (up(cube_copy_bytes(DIFF_RES, 1)) + up(cube_copy_bytes(s, SPEC_MIPS)) + up(lut_copy_bytes(l))) / 1e6
            us[(l, s)] = ms * 1e3
            print(f"run {rep}  lut {l:4d}^2  spec {s:3d}^2 x{SPEC_MIPS}  copies {mb:5.1f} MB (LUT {lut_copy_bytes(l) / 1e6:4.1f})  "
                  f"{ms * 1e3:7.1f} us  {W * H / ms / 1e3:7.0f} Mpx/s  sm clock {clk}", flush=True)
        print(f"run {rep}  (1024, 512) vs (724, 512): {us[(1024, 512)] / us[(724, 512)] - 1.0:+.2%}", flush=True)


if __name__ == "__main__":
    main()
