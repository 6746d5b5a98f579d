"""GPU-box helper: strong scaling of the shadowed and the from-materials shading calls over GPUs, in their multi-destination form
(vq_forward_lighting_shadowed_multi_signal, vq_forward_lighting_from_materials_multi_signal).

  torchrun --nproc-per-node N tools/perf_multi_shading.py [--iters 10] [--json]      (N = 2..8)
  python tools/perf_multi_shading.py [--iters 10] [--json]                           (one GPU)

Workload: BASELINE config 5's 7680x4320 frame of bench.py's material scene (bench.surface_scene_gpu), lit with the casters and maps of
bench.shadow_passes (one point caster with 1024^2 cube faces, one spot caster and a shadowing directional light with 2048^2 maps, plus
the scene's unshadowed point and spot lights) and bench.py's registered environment. Rank r shades the band even_tiles(4320, N)[r],
from inputs that hold just its band (attribute planes; for the G-buffer call the G-buffer the surface producer makes of them).
Three paths: the shadowed G-buffer call ("shadowed": PCF pre-pass + forward kernel), and the from-materials call with the maps bound
("from_materials_shadowed") and without ("from_materials").

Per path and rank: the kernel-only time of the rank's band into a local frame. With N > 1 GPUs also: the fused step (one call per
rank that stores every pixel into every rank's frame over NVLink and runs the rendezvous in its last CTA), the NCCL step (the same
call into the local band, then all_gather_into_tensor), and whether the two frames are identical. With one GPU: the band times for
N = 1, 2, 4, 8, and the full frame into two local destinations against one. CUDA events; the card's name and power limit are read
in the same run."""
import argparse, json, os, sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import numpy as np
import vqengine_b200 as vq
from vqengine_b200 import synth
from vqengine_b200.distributed import allgather_ranges, even_tiles
import bench

PATHS = ("shadowed", "from_materials_shadowed", "from_materials")


def card(local):
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", f"--id={local}", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, clk = (c.strip() for c in q.split(","))
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as ex:
        return {"name": torch.cuda.get_device_name(local), "power_limit": f"unknown ({type(ex).__name__})"}


def shadow_setup(w, h, spec_mips):
    """bench.shadow_passes's lights, shadow views and maps (that function times them but does not return them)"""
    pf, pv = synth.scene_constants(w, h, spec_mips, n_point=2, n_spot=1, casters=True)
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
    maps = {"point_cubes": torch.rand((max(L.numPointCasters, 1), 6, res_pt, res_pt), device="cuda", generator=g) * 1.2,
            "spot_maps": torch.rand((max(L.numSpotCasters, 1), res_2d, res_2d), device="cuda", generator=g) * 0.4 + 0.3,
            "directional_map": torch.rand((res_2d, res_2d), device="cuda", generator=g) * 0.4 + 0.3}
    return pf, pv, maps


class Band:
    """the inputs of rows [a, b) of the frame: band attribute planes (and the G-buffer made of them), with the frame's table"""

    def __init__(self, ctx, sc, a, b, w, pf, pv, maps, env):
        self.ctx, self.pf, self.pv, self.maps, self.env, self.a, self.b = ctx, pf, pv, maps, env, a, b
        self.table = sc["table"]
        p = [t[a:b] for t in sc["planes"]]
        self.si = vq.SurfaceInputs(vq.image_of(p[0]), vq.image_of(p[1]), vq.image_of(p[2]), vq.null_image())
        self.gbt = [torch.empty((b - a, w, 4), dtype=torch.float32, device="cuda") for _ in range(4)]
        self.gb = vq.GBuffer(*(vq.image_of(t) for t in self.gbt))
        ctx.gbuffer_from_materials(self.si, self.table, pf.fAmbientLightingFactor, self.gb)

    def call(self, path, images, offset, signal=None):
        c = self.ctx
        if path == "shadowed":
            c.forward_lighting_shadowed_multi(self.pf, self.pv, self.gb, self.env, images, offset, signal=signal, **self.maps)
        else:
            maps = self.maps if path == "from_materials_shadowed" else {}
            c.forward_lighting_from_materials_multi(self.pf, self.pv, self.si, self.table, self.env, images, offset, signal=signal, **maps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_multi_shading.py needs a CUDA device"
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0")))
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    FW, FH = bench.W8K, bench.H8K
    ctx = vq.Context(local)
    envk = bench.build_env_maps_gpu(ctx, vq, torch)
    sc = bench.surface_scene_gpu(ctx, vq, torch, FW, FH)
    sc["planes"] = [t for t in sc["keep"] if t.dim() == 3 and t.shape[:2] == (FH, FW)]
    pf, pv, maps = shadow_setup(FW, FH, envk["spec_mips"])
    env = envk["env"]

    def timed(fn, n=args.iters):
        """device time per call, max over ranks"""
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        if dist: dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record(); torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1) / n], dtype=torch.float64, device="cuda")
        if dist: dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return round(float(t.item()), 4)

    res = {"card": card(local), "frame": f"{FW}x{FH}", "world": world, "iters": args.iters,
           "casters": f"{pf.Lights.numPointCasters} point (1024^2 cube faces) + {pf.Lights.numSpotCasters} spot + directional (2048^2)",
           "paths": {}}
    tiles = even_tiles(FH, world)
    a, b = tiles[rank]
    band = Band(ctx, sc, a, b, FW, pf, pv, maps, env)
    local_band = torch.empty((b - a, FW, 4), dtype=torch.float32, device="cuda")
    frame = hdl = flags = None
    if world > 1:
        import torch.distributed._symmetric_memory as symm
        frame = symm.empty((FH, FW, 4), dtype=torch.float32, device=torch.device("cuda", local))
        hdl = symm.rendezvous(frame, dist.group.WORLD)
        frame.zero_(); torch.cuda.synchronize(); dist.barrier()
        flags = bench.PeerFlags(vq, torch, dist, rank, world)
        peer_imgs = [vq.Image(int(hdl.buffer_ptrs[r]), FW, FH, FW * 16) for r in flags.order]
        full = torch.empty((FH, FW, 4), dtype=torch.float32, device="cuda")
    else:                            # the first band of each world size, and a second full-frame destination
        bands = {n: band if n == 1 else Band(ctx, sc, *even_tiles(FH, n)[0], FW, pf, pv, maps, env) for n in (1, 2, 4, 8)}
        outs = {n: torch.empty((bd.b - bd.a, FW, 4), dtype=torch.float32, device="cuda") for n, bd in bands.items()}
        out2 = torch.empty((FH, FW, 4), dtype=torch.float32, device="cuda")
    for path in PATHS:
        r = {"rows_per_rank": b - a}
        kernel_only = lambda: band.call(path, [vq.image_of(local_band)], 0)
        r["kernel_only_ms_per_rank"] = timed(kernel_only)
        n0 = vq.launch_count(); kernel_only(); r["launches_per_call"] = vq.launch_count() - n0
        if world > 1:
            fused = lambda: band.call(path, peer_imgs, a, signal=flags.next())

            def nccl():
                band.call(path, [vq.image_of(full[a:b])], 0)
                allgather_ranges(full, tiles)
            r["fused_p2p_ms"] = timed(fused)
            r["nccl_allgather_ms"] = timed(nccl)
            fused(); nccl(); torch.cuda.synchronize(); dist.barrier()
            same = torch.tensor([1.0 if torch.equal(frame.view(torch.int32), full.view(torch.int32)) else 0.0], device="cuda")
            dist.all_reduce(same, op=dist.ReduceOp.MIN)
            r["equals_nccl_allgather"] = bool(same.item() == 1.0)
            r["nvlink_ingress_bytes_per_rank"] = (FH - (b - a)) * FW * 16
        else:
            r["band_ms_by_world"] = {str(n): timed(lambda: bd.call(path, [vq.image_of(outs[n])], 0)) for n, bd in bands.items()}
            two = [vq.image_of(local_band), vq.image_of(out2)]
            r["full_frame_two_local_destinations_ms"] = timed(lambda: band.call(path, two, 0))
            r["second_destination_cost"] = round(r["full_frame_two_local_destinations_ms"] / r["kernel_only_ms_per_rank"] - 1.0, 4)
            band.call(path, two, 0); torch.cuda.synchronize()
            r["two_destinations_identical"] = bool(torch.equal(local_band.view(torch.int32), out2.view(torch.int32)))
        res["paths"][path] = r
    if rank == 0:
        if args.json:
            print(json.dumps(res))
        else:
            print(f"{res['card']}  frame {res['frame']}  world {world}  {res['casters']}")
            for path, r in res["paths"].items():
                print(f"  {path}: {json.dumps(r)}")
    sc["table"].close()
    if dist:
        dist.barrier()
        dist.destroy_process_group()
    ctx.close()


if __name__ == "__main__":
    main()
