"""GPU-box helper: strong scaling of the post chain over GPUs (vq_tonemap_multi_signal, vq_cas_multi_signal, vq_fsr_easu_multi_signal,
vq_fsr_rcas_multi_signal), each rank running its distributed.post_chain_rows plan.

  python tools/perf_post_multi.py [--iters 50] [--json]                            (one GPU)
  torchrun --nproc-per-node N tools/perf_post_multi.py [--iters 50] [--json]      (N = 2..8)

Workloads:
  fsr_performance : the engine's FSR "performance" chain, a 3840x2160 HDR frame -> tonemap -> EASU 2x -> RCAS at 7680x4320;
  tonemap_8k      : the tonemapper alone on BASELINE config 5's 7680x4320 frame.
With one GPU, per workload: the single-GPU chain (vq_tonemap, vq_fsr_easu, vq_fsr_rcas, each also timed alone); one rank's band
chain for N = 2, 4, 8 and the first, a middle and the last band (intermediates in local full-size scratch, one destination); and the
middle band's chain with N local destinations standing in for the peers' frames, against one. With N > 1 GPUs also the real step:
the band chain whose last pass stores into every rank's symmetric-memory display frame and runs the rendezvous in its last CTA, and
whether every rank's frame equals the single-GPU chain bit for bit. CUDA events; the card's name and power limit are read in the
same run."""
import argparse, json, os, sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
import numpy as np
import vqengine_b200 as vq
from vqengine_b200 import synth
from vqengine_b200.distributed import equal_tiles, post_chain_rows
import bench
from perf_multi_shading import card

W4K, H4K, W8K, H8K = bench.W4K, bench.H4K, bench.W8K, bench.H8K


class Chain:
    """one workload: the HDR frame, the passes' constants, full-size scratch for the intermediates, and the single-GPU chain"""

    def __init__(self, ctx, fsr, in_w, in_h):
        self.ctx, self.fsr = ctx, fsr
        self.in_w, self.in_h = in_w, in_h
        self.out_w, self.out_h = (2 * in_w, 2 * in_h) if fsr else (in_w, in_h)
        g = torch.Generator(device="cuda"); g.manual_seed(11)
        self.hdr = torch.rand((in_h, in_w, 4), device="cuda", generator=g) * 3.0
        self.tm = synth.default_tonemapper()
        self.easu_con = vq.fsr_easu_con(in_w, in_h, in_w, in_h, self.out_w, self.out_h) if fsr else None
        self.rcas_con = vq.fsr_rcas_con(0.2)
        new = lambda h, w: torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
        self.ldr, self.up = new(in_h, in_w), (new(self.out_h, self.out_w) if fsr else None)
        self.single_out = new(self.out_h, self.out_w)

    def single(self):
        c = self.ctx
        if not self.fsr:
            c.tonemap(self.tm, self.hdr, self.single_out)
            return
        c.tonemap(self.tm, self.hdr, self.ldr)
        c.fsr_easu(self.easu_con, self.ldr, self.up)
        c.fsr_rcas(self.rcas_con, self.up, self.single_out)

    def singles(self):
        """each single call alone"""
        c = self.ctx
        if not self.fsr:
            return {"vq_tonemap": lambda: c.tonemap(self.tm, self.hdr, self.single_out)}
        return {"vq_tonemap": lambda: c.tonemap(self.tm, self.hdr, self.ldr),
                "vq_fsr_easu": lambda: c.fsr_easu(self.easu_con, self.ldr, self.up),
                "vq_fsr_rcas": lambda: c.fsr_rcas(self.rcas_con, self.up, self.single_out)}

    def band(self, band, dests, signal=None):
        """the rank's plan for `band` of the display frame: intermediates into local scratch, the last pass into `dests`"""
        c = self.ctx
        plan = post_chain_rows(self.in_h, self.out_h, band, fsr_con=self.easu_con)
        if not self.fsr:
            c.tonemap_multi(self.tm, self.hdr, dests, *plan["tonemap"][0], signal=signal)
            return
        for rows in plan["tonemap"]:
            c.tonemap_multi(self.tm, self.hdr, [vq.image_of(self.ldr)], *rows)
        c.fsr_easu_multi(self.easu_con, self.ldr, [vq.image_of(self.up)], *plan["fsr_easu"][0])
        c.fsr_rcas_multi(self.rcas_con, self.up, dests, *plan["fsr_rcas"][0], signal=signal)

    def plan_rows(self, band):
        plan = post_chain_rows(self.in_h, self.out_h, band, fsr_con=self.easu_con)
        return {k: sum(b - a for a, b in v) for k, v in plan.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "perf_post_multi.py needs a CUDA device"
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0")))
    torch.cuda.set_device(local)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ctx = vq.Context(local)

    def timed(fn, n=args.iters):
        """device time per call in ms, max over ranks"""
        for _ in range(3):
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

    res = {"card": card(local), "world": world, "iters": args.iters, "workloads": {}}
    for name, fsr, iw, ih in (("fsr_performance", True, W4K, H4K), ("tonemap_8k", False, W8K, H8K)):
        ch = Chain(ctx, fsr, iw, ih)
        r = {"hdr": f"{iw}x{ih}", "display": f"{ch.out_w}x{ch.out_h}"}
        r["single_gpu_chain_ms"] = timed(ch.single)
        r["single_calls_ms"] = {k: timed(f) for k, f in ch.singles().items()}
        local_out = torch.empty((ch.out_h, ch.out_w, 4), dtype=torch.float32, device="cuda")
        ch.single(); torch.cuda.synchronize()
        want = ch.single_out.clone()
        if world == 1:
            r["band_chain_ms"] = {}
            for n in (2, 4, 8):
                tiles = equal_tiles(ch.out_h, n)
                for which, band in (("first", tiles[0]), ("middle", tiles[n // 2]), ("last", tiles[-1])):
                    t = timed(lambda: ch.band(band, [vq.image_of(local_out)]))
                    r["band_chain_ms"][f"N={n} {which} {band}"] = {"ms": t, "rows_per_pass": ch.plan_rows(band)}
            r["band_chain_local_destinations_ms"] = {}
            frames = [local_out] + [torch.empty_like(local_out) for _ in range(7)]
            for n in (2, 4, 8):
                band = equal_tiles(ch.out_h, n)[n // 2]
                one = timed(lambda: ch.band(band, [vq.image_of(frames[0])]))
                many = timed(lambda: ch.band(band, [vq.image_of(f) for f in frames[:n]]))
                r["band_chain_local_destinations_ms"][f"N={n} {band}"] = {"1": one, str(n): many}
            # every band of an 8-way split into one frame assembles the single-GPU chain
            local_out.zero_()
            for band in equal_tiles(ch.out_h, 8):
                ch.band(band, [vq.image_of(local_out)])
            torch.cuda.synchronize()
            r["bands_assemble_single_chain"] = bool(torch.equal(local_out.view(torch.int32), want.view(torch.int32)))
            r["multi_gpu_step"] = "not measured (one GPU)"
        else:
            import torch.distributed._symmetric_memory as symm
            frame = symm.empty((ch.out_h, ch.out_w, 4), dtype=torch.float32, device=torch.device("cuda", local))
            hdl = symm.rendezvous(frame, dist.group.WORLD)
            frame.zero_(); torch.cuda.synchronize(); dist.barrier()
            flags = bench.PeerFlags(vq, torch, dist, rank, world)
            peers = [vq.Image(int(hdl.buffer_ptrs[q]), ch.out_w, ch.out_h, ch.out_w * 16) for q in flags.order]
            band = equal_tiles(ch.out_h, world)[rank]
            r["rank_band"] = band
            r["band_chain_one_destination_ms"] = timed(lambda: ch.band(band, [vq.image_of(local_out)]))
            r["multi_gpu_step_ms"] = timed(lambda: ch.band(band, peers, signal=flags.next()))
            ch.band(band, peers, signal=flags.next()); torch.cuda.synchronize(); dist.barrier()
            same = torch.tensor([1.0 if torch.equal(frame.view(torch.int32), want.view(torch.int32)) else 0.0], device="cuda")
            dist.all_reduce(same, op=dist.ReduceOp.MIN)
            r["every_frame_equals_single_gpu_chain"] = bool(same.item() == 1.0)
        res["workloads"][name] = r
        del ch
        torch.cuda.empty_cache()
    if rank == 0:
        if args.json:
            print(json.dumps(res))
        else:
            print(f"{res['card']}  world {world}  iters {args.iters}")
            for name, r in res["workloads"].items():
                print(f"  {name}: {json.dumps(r)}")
    if dist:
        dist.barrier()
        dist.destroy_process_group()
    ctx.close()


if __name__ == "__main__":
    main()
