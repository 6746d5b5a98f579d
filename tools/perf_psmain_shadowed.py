"""GPU-box helper: shadowed PSMain end to end at 4K, the fused call (vq_forward_lighting_shadowed_from_materials, one launch, no
G-buffer, no PCF records) against the calls it replaces back to back (vq_gbuffer_from_materials with an emissive plane, then
vq_forward_lighting_shadowed: the PCF kernel and the shadowed forward kernel).

  python tools/perf_psmain_shadowed.py [--repeats 3] [--json]

Workload: tools/perf_psmain.py's 4K material frame (bench.surface_scene_gpu) lit with the casters and maps of bench.shadow_passes:
one point caster with 1024^2 cube faces (20-tap cube PCF), one spot caster and a shadowing directional light with 2048^2 maps (5x5
PCF), plus the scene's unshadowed point and spot lights; bench.py's environment maps, registered. The two paths are timed with CUDA
events, alternated in one process, `--repeats` times each; the card's name and power limit are read in the same run. The fused
result is checked bit for bit against the two-pass result on the timed frame first."""
import argparse, json, os, sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import vqengine_b200 as vq
from vqengine_b200 import synth
import bench
from perf_psmain import B_GBUF, B_IN, B_OUT, card

B_PCF_IN = 32            # the PCF kernel reads position and normal back from the G-buffer
B_REC = 8                # one 64-bit PCF record per pixel, written by the PCF kernel and read by the forward kernel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_psmain_shadowed.py needs a CUDA device"
    w, h = bench.W4K, bench.H4K
    ctx = vq.Context(0)
    envk = bench.build_env_maps_gpu(ctx, vq, torch)
    sc = bench.surface_scene_gpu(ctx, vq, torch, w, h)
    # the casters and maps of bench.shadow_passes
    pf, pv = synth.scene_constants(w, h, envk["spec_mips"], n_point=2, n_spot=1, casters=True)
    pf.fAmbientLightingFactor = 0.3
    L = pf.Lights
    m = np.zeros(16, np.float32); m[0] = 1 / 25; m[5] = 1 / 25; m[14] = 0.5; m[15] = 1.0
    for c in range(L.numSpotCasters):
        for k in range(16): L.shadowViews[c].m[k] = float(m[k])
    for k in range(16): L.shadowViewDirectional.m[k] = float(m[k])
    L.directional.shadowing = 1
    res_pt, res_2d = 1024, 2048
    pf.f2SpotLightShadowMapDimensions.x = pf.f2SpotLightShadowMapDimensions.y = float(res_2d)
    pf.f2DirectionalLightShadowMapDimensions.x = pf.f2DirectionalLightShadowMapDimensions.y = float(res_2d)
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    cubes = torch.rand((max(L.numPointCasters, 1), 6, res_pt, res_pt), device="cuda", generator=g) * 1.2
    spots = torch.rand((max(L.numSpotCasters, 1), res_2d, res_2d), device="cuda", generator=g) * 0.4 + 0.3
    dmap = torch.rand((res_2d, res_2d), device="cuda", generator=g) * 0.4 + 0.3

    out_two = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    out_fused = torch.empty_like(out_two)
    before = torch.cuda.memory_allocated()
    gp = [torch.empty((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(4)]
    gbuf_bytes = torch.cuda.memory_allocated() - before
    rec_bytes = w * h * B_REC          # the context's PCF-record scratch the two-pass path grows to
    gb = vq.GBuffer(*(vq.image_of(t) for t in gp))

    def two_pass():
        ctx.gbuffer_from_materials(sc["inputs"], sc["table"], pf.fAmbientLightingFactor, gb)
        ctx.forward_lighting_shadowed(pf, pv, gb, envk["env"], out_two, cubes, spots, dmap)

    def fused():
        ctx.forward_lighting_shadowed_from_materials(pf, pv, sc["inputs"], sc["table"], envk["env"], out_fused, cubes, spots, dmap)

    two_pass(); fused(); torch.cuda.synchronize()
    same = bool(torch.equal(out_two.view(torch.int32), out_fused.view(torch.int32)))
    n0 = vq.launch_count(); fused(); launches_fused = vq.launch_count() - n0
    n0 = vq.launch_count(); two_pass(); launches_two = vq.launch_count() - n0

    runs = {"fused": [], "two_pass": []}
    for _ in range(args.repeats):
        runs["fused"].append(bench.time_gpu(torch, fused, 10))
        runs["two_pass"].append(bench.time_gpu(torch, two_pass, 10))
    px = w * h
    res = {"card": card(), "frame": f"{w}x{h}", "bit_identical": same,
           "casters": f"{L.numPointCasters} point ({res_pt}^2 cube faces) + {L.numSpotCasters} spot + directional ({res_2d}^2)",
           "paths": {}}
    for name, launches, bpx, dev_bytes in (("fused", launches_fused, B_IN + B_OUT, 0),
                                            ("two_pass", launches_two, B_IN + 2 * B_GBUF + B_PCF_IN + 2 * B_REC + B_OUT,
                                             gbuf_bytes + rec_bytes)):
        ms = sorted(runs[name])
        res["paths"][name] = {"ms": [round(x, 4) for x in runs[name]], "ms_median": round(ms[len(ms) // 2], 4),
                              "Mpx_per_s": round(px / ms[len(ms) // 2] / 1e3, 1), "launches": launches,
                              "algorithmic_bytes_per_px": bpx, "device_bytes_allocated": dev_bytes}
    f, t = res["paths"]["fused"]["ms_median"], res["paths"]["two_pass"]["ms_median"]
    res["fused_over_two_pass"] = round(f / t, 4)
    sc["table"].close()
    ctx.close()
    if args.json:
        print(json.dumps(res))
        return
    print(f"{res['card']}  frame {res['frame']}  {res['casters']}  fused == two-pass bit for bit: {same}")
    for name, r in res["paths"].items():
        print(f"  {name:9s} {r['ms_median']:.4f} ms (runs {r['ms']})  {r['Mpx_per_s']:.1f} Mpx/s  {r['launches']} launch(es)  "
              f"{r['algorithmic_bytes_per_px']} B/px  G-buffer + PCF records {r['device_bytes_allocated'] / 1e6:.1f} MB")
    print(f"  fused / two-pass time: {res['fused_over_two_pass']:.3f}")


if __name__ == "__main__":
    main()
