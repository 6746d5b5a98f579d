"""GPU-box helper: PSMain end to end at 4K, the fused call (vq_forward_lighting_from_materials, one launch, no G-buffer) against
the two calls it replaces back to back (vq_gbuffer_from_materials with an emissive plane, then vq_forward_lighting).

  python tools/perf_psmain.py [--repeats 3] [--json]

Workload: bench.surface_producer_pass's 4K material frame (bench.surface_scene_gpu: 4 materials, 1024^2 RGBA8 maps, SSAO) lit by
bench.py's lights (synth.scene_constants) and environment maps (bench.build_env_maps_gpu, registered). The two paths are timed
with CUDA events, alternated in one process, `--repeats` times each; the card's name and power limit are read in the same run.
The fused result is checked bit for bit against the two-pass result on the timed frame first."""
import argparse, json, os, subprocess, sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import vqengine_b200 as vq
from vqengine_b200 import synth
import bench

# algorithmic bytes per pixel that cross HBM
B_IN = 48 + 4            # three float4 interpolant planes + the R32F SSAO texel
B_OUT = 16               # the float4 colour
B_GBUF = 64              # four float4 G-buffer planes (with emissive), written by the first pass and read by the second


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, clk = (c.strip() for c in q.split(","))
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as ex:
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({type(ex).__name__})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_psmain.py needs a CUDA device"
    w, h = bench.W4K, bench.H4K
    ctx = vq.Context(0)
    envk = bench.build_env_maps_gpu(ctx, vq, torch)
    sc = bench.surface_scene_gpu(ctx, vq, torch, w, h)
    pf, pv = synth.scene_constants(w, h, envk["spec_mips"])
    pf.fAmbientLightingFactor = 0.3
    out_two = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    out_fused = torch.empty_like(out_two)
    before = torch.cuda.memory_allocated()
    g = [torch.empty((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(4)]
    gbuf_bytes = torch.cuda.memory_allocated() - before
    gb = vq.GBuffer(*(vq.image_of(t) for t in g))

    def two_pass():
        ctx.gbuffer_from_materials(sc["inputs"], sc["table"], pf.fAmbientLightingFactor, gb)
        ctx.forward_lighting(pf, pv, gb, envk["env"], out_two)

    def fused():
        ctx.forward_lighting_from_materials(pf, pv, sc["inputs"], sc["table"], envk["env"], out_fused)

    two_pass(); fused(); torch.cuda.synchronize()
    same = bool(torch.equal(out_two.view(torch.int32), out_fused.view(torch.int32)))
    n0 = vq.launch_count(); fused(); launches_fused = vq.launch_count() - n0
    n0 = vq.launch_count(); two_pass(); launches_two = vq.launch_count() - n0

    runs = {"fused": [], "two_pass": []}
    for _ in range(args.repeats):
        runs["fused"].append(bench.time_gpu(torch, fused, 20))
        runs["two_pass"].append(bench.time_gpu(torch, two_pass, 20))
    px = w * h
    res = {"card": card(), "frame": f"{w}x{h}", "bit_identical": same, "paths": {}}
    for name, launches, bpx, dev_bytes in (("fused", launches_fused, B_IN + B_OUT, 0),
                                            ("two_pass", launches_two, B_IN + 2 * B_GBUF + B_OUT, gbuf_bytes)):
        ms = sorted(runs[name])
        res["paths"][name] = {"ms": [round(m, 4) for m in runs[name]], "ms_median": round(ms[len(ms) // 2], 4),
                              "Mpx_per_s": round(px / ms[len(ms) // 2] / 1e3, 1), "launches": launches,
                              "algorithmic_bytes_per_px": bpx, "device_bytes_allocated": dev_bytes}
    f, t = res["paths"]["fused"]["ms_median"], res["paths"]["two_pass"]["ms_median"]
    res["fused_over_two_pass"] = round(f / t, 4)
    sc["table"].close()
    ctx.close()
    if args.json:
        print(json.dumps(res))
        return
    print(f"{res['card']}  frame {res['frame']}  fused == two-pass bit for bit: {same}")
    for name, r in res["paths"].items():
        print(f"  {name:9s} {r['ms_median']:.4f} ms (runs {r['ms']})  {r['Mpx_per_s']:.1f} Mpx/s  {r['launches']} launch(es)  "
              f"{r['algorithmic_bytes_per_px']} B/px  G-buffer {r['device_bytes_allocated'] / 1e6:.1f} MB")
    print(f"  fused / two-pass time: {res['fused_over_two_pass']:.3f}")


if __name__ == "__main__":
    main()
