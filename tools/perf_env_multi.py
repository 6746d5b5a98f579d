"""GPU-box helper: the band forms of the environment prefilter (vq_diffuse_irradiance_multi_signal,
vq_brdf_integration_lut_multi_signal) and the one-launch cube blur (vq_gaussian_blur_cube) on one GPU.

  python tools/perf_env_multi.py [--iters 10]

Workload: bench.py's 2048x1024 synthetic HDRI and its pyramid, a 64-texel diffuse cube (the engine's) and a 1024^2 LUT at 2048
samples. Timed with CUDA events (bench.time_gpu):
  * K2 over the whole cube, and each band of equal_tiles(384, N), N = 2, 4, 8 (the slowest band is reported, with the ideal
    full / N beside it), into 1 and into N local destinations (local stand-ins for the peers' cubes: the stores stay in this GPU's
    HBM, so no NVLink time is in them); at bench.py's 64 x 16 grid and at the engine's step of 0.010 (629 x 158 samples);
  * K4 over the whole LUT and its bands for equal_tiles(1024, N);
  * the diffuse cube's blur: 12 launches (vq_gaussian_blur_x / _y per face, through a temporary) against vq_gaussian_blur_cube.
No signal is passed: a rendezvous needs the other ranks. A multi-GPU step time needs two or more GPUs and is not taken here. The
card's name, power limit and SM clock limit are read in the same run."""
import argparse, json, os, sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
import vqengine_b200 as vq
from vqengine_b200.distributed import equal_tiles
import bench
from perf_multi_shading import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "perf_env_multi.py needs a CUDA device"
    ctx = vq.Context(0)
    envk = bench.build_env_maps_gpu(ctx, vq, torch)
    pyr, res = envk["pyr"], envk["diff_res"]
    cubes = [torch.zeros((6 * res * res, 4), dtype=torch.float32, device="cuda") for _ in range(8)]
    cms = [vq.cubemap_of(c, res, 1) for c in cubes]
    luts = [torch.zeros((1024, 1024, 2), dtype=torch.float32, device="cuda") for _ in range(8)]
    lis = [vq.image_of(t, 2) for t in luts]

    def t(fn):
        return round(bench.time_gpu(torch, fn, a.iters), 4)

    out = {"card": card(0), "iters": a.iters, "diffuse": {}, "lut": {}}
    for mode, kw in (("grid 64x16", dict(n_phi=64, n_theta=16, src_mip=3)), ("step 0.010", dict(step=0.010, src_mip=3))):
        full = t(lambda: ctx.diffuse_irradiance(pyr, cms[0], **kw))
        r = {"full": full, "full_multi_1": t(lambda: ctx.diffuse_irradiance_multi(pyr, cms[:1], **kw))}
        for n in (2, 4, 8):
            bands = equal_tiles(6 * res, n)
            for k in (1, n):
                worst = max(t(lambda b=b: ctx.diffuse_irradiance_multi(pyr, cms[:k], row_begin=b[0], row_end=b[1], **kw)) for b in bands)
                r[f"n{n}_into{k}"] = {"slowest_band_ms": worst, "ideal_ms": round(full / n, 4), "vs_ideal": round(worst / (full / n), 2)}
        out["diffuse"][mode] = r
        print("diffuse", mode, json.dumps(r), flush=True)
    full = t(lambda: ctx.brdf_integration_lut(luts[0], 2048))
    r = {"full": full}
    for n in (2, 4, 8):
        for k in (1, n):
            worst = max(t(lambda b=b: ctx.brdf_integration_lut_multi(lis[:k], 2048, row_begin=b[0], row_end=b[1]))
                        for b in equal_tiles(1024, n))
            r[f"n{n}_into{k}"] = {"slowest_band_ms": worst, "ideal_ms": round(full / n, 4), "vs_ideal": round(worst / (full / n), 2)}
    out["lut"] = r
    print("lut", json.dumps(r), flush=True)
    faces, blurred = cubes[0].view(6, res, res, 4), cubes[1].view(6, res, res, 4)
    tmp = torch.empty_like(faces[0])

    def twelve():
        for f in range(6):
            ctx.gaussian_blur(faces[f], tmp, False)
            ctx.gaussian_blur(tmp, blurred[f], True)
    out["blur"] = {"twelve_launches": t(twelve), "blur_cube": t(lambda: ctx.gaussian_blur_cube(cms[0], cms[1])),
                   "blur_cube_in_place": t(lambda: ctx.gaussian_blur_cube(cms[2], cms[2]))}
    print("blur", json.dumps(out["blur"]), flush=True)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
