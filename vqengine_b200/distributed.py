"""Multi-GPU plumbing: tile partitioning + the final gather of tiles (SURVEY.md §8(e)).

The passes shard naturally — every output texel depends only on read-only inputs — so each rank runs
the SAME kernels on a contiguous range of rows and the only communication is one all-gather of the
finished tiles at the end (NCCL over NVLink on the GPU box; gloo in the CPU tests). One process per
GPU, torch.distributed for the plumbing. Nothing here computes pixels.

Row spaces:
  forward / post passes : image rows                      -> equal contiguous row blocks (post chain halos: post_chain_rows,
                                                             with the blur in front: blur_rows)
  diffuse irradiance    : face*res + row                  -> equal contiguous row blocks
  specular prefilter    : flattened (mip, face, row)      -> contiguous blocks of equal COST
                          (a row of mip m has (res>>m) texels; mip 0 is roughness 0 = ~1 % of a full texel,
                          every other mip costs `samples` samples/texel)
Because both cubemap layouts are packed mip-major/face-minor/row-major, a contiguous row range is a
contiguous texel range of the packed buffer, so the gather needs no strided copies.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple


def equal_tiles(n_rows: int, world: int) -> List[Tuple[int, int]]:
    """`world` contiguous [begin,end) row ranges whose sizes differ by at most one (some may be empty)."""
    return [((n_rows * r) // world, (n_rows * (r + 1)) // world) for r in range(world)]


def even_tiles(n_rows: int, world: int) -> List[Tuple[int, int]]:
    """`world` contiguous [begin,end) row ranges whose inner boundaries are even rows and whose sizes differ by at most two (some
    may be empty): the bands of the from-materials shading calls, whose 2x2 quads must start on even rows of the frame. Row pairs
    are shared out with the larger shares first, so that an odd last row goes to a band of the smaller size."""
    pairs = n_rows // 2
    cuts = [2 * (-(-pairs * r // world)) for r in range(world)] + [n_rows]
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def post_chain_rows(in_height: int, out_height: int, band: Tuple[int, int], fsr_con=None, address_mode: int = 0,
                    cas: bool = False) -> Dict[str, List[Tuple[int, int]]]:
    """The [begin, end) rows each post pass must produce so that the chain's last pass can write rows `band` of the display frame
    (DESIGN.md §6). Plumbing only: nothing is launched. The stages come in the order RenderPostProcess runs them, the last one
    writing the display frame:
      fsr_con given (FSR on): tonemap -> fsr_easu -> fsr_rcas; CAS is not run, its output is unused when FSR is on;
      cas (FSR off, CAS on):  tonemap -> cas;
      otherwise:              tonemap.
    in_height is the HDR frame's height, out_height the display frame's (equal without FSR); address_mode is EASU's sampler
    addressing (0 = WRAP, the engine's). RCAS and CAS read rows y-1 .. y+1 of their source: the band plus one row each side,
    clipped to the image. EASU's source rows are vq_fsr_easu_source_rows's: one or, under WRAP at the top and bottom of the frame,
    two ranges, so the tonemapper may run twice. An empty band gives empty lists."""
    a, b = band
    assert 0 <= a <= b <= out_height
    if fsr_con is None:
        assert in_height == out_height, "without FSR the display frame has the HDR frame's size"
    if a == b:
        stages = ("tonemap", "fsr_easu", "fsr_rcas") if fsr_con is not None else ("tonemap", "cas") if cas else ("tonemap",)
        return {s: [] for s in stages}
    halo = (max(a - 1, 0), min(b + 1, out_height))
    if fsr_con is not None:
        from . import fsr_easu_source_rows
        return {"tonemap": fsr_easu_source_rows(fsr_con, in_height, out_height, *halo, address_mode=address_mode),
                "fsr_easu": [halo], "fsr_rcas": [(a, b)]}
    if cas:
        return {"tonemap": [halo], "cas": [(a, b)]}
    return {"tonemap": [(a, b)]}


def blur_rows(in_height: int, out_height: int, band: Tuple[int, int], fsr_con=None, address_mode: int = 0,
              cas: bool = False) -> Dict[str, List[Tuple[int, int]]]:
    """post_chain_rows with the Gaussian blur of the HDR frame in front of the chain: a "gaussian_blur" stage whose output rows are
    the tonemapper's source rows (the band plus the halo EASU, RCAS or CAS read), which vq_gaussian_blur_multi_signal produces from
    the whole source frame (it reads rows 10 beyond each range, clamped, itself). in_height is also the blur's iImageSizeY."""
    plan = post_chain_rows(in_height, out_height, band, fsr_con, address_mode, cas)
    return {"gaussian_blur": list(plan["tonemap"]), **plan}


def weighted_tiles(costs: Sequence[float], world: int) -> List[Tuple[int, int]]:
    """contiguous ranges over rows with per-row `costs`, cut where the cumulative cost crosses k/world."""
    total = float(sum(costs))
    cuts, acc, r = [0], 0.0, 1
    for i, c in enumerate(costs):
        acc += c
        while r < world and acc >= total * r / world - 1e-9:
            cuts.append(i + 1)
            r += 1
    while len(cuts) < world:
        cuts.append(len(costs))
    cuts.append(len(costs))
    return [(cuts[i], cuts[i + 1]) for i in range(world)]


def specular_row_costs(res: int, mips: int, samples: int = 512) -> List[float]:
    costs = []
    for m in range(mips):
        n = res >> m
        # mip 0 is roughness 0: one HDRI sample + a 4 x samples FADD replay, a small fraction of a full texel
        per_texel = 0.012 * float(samples) if m == 0 else float(samples)
        costs += [n * per_texel] * (6 * n)
    return costs


def specular_row_to_texel(res: int, mips: int, row: int) -> int:
    """texel offset (in the packed cubemap) of the first texel of flattened row `row` (row == total -> end)."""
    off = 0
    for m in range(mips):
        n = res >> m
        if row <= 6 * n:
            return off + row * n
        off += 6 * n * n
        row -= 6 * n
    return off


def specular_tiles(res: int, mips: int, world: int, samples: int = 512):
    rows = weighted_tiles(specular_row_costs(res, mips, samples), world)
    texels = [(specular_row_to_texel(res, mips, a), specular_row_to_texel(res, mips, b)) for a, b in rows]
    return rows, texels


def allgather_ranges(buf, ranges: Sequence[Tuple[int, int]], group=None):
    """In-place all-gather of UNEQUAL contiguous ranges of dim 0 of `buf` (same shape on every rank):
    on entry rank r has filled buf[ranges[r]]; on exit every rank has every range.
    Equal ranges covering the buffer use one all_gather_into_tensor straight into `buf`; unequal ranges use one
    broadcast per owner rank (no padding to the largest range)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    assert len(ranges) == world
    sizes = [b - a for a, b in ranges]
    if world == 1:
        return buf
    contiguous_cover = all(ranges[i][1] == ranges[i + 1][0] for i in range(world - 1))
    if len(set(sizes)) == 1 and contiguous_cover and ranges[0][0] == 0 and ranges[-1][1] == buf.shape[0]:
        dist.all_gather_into_tensor(buf, buf[ranges[rank][0]:ranges[rank][1]].clone(), group=group)
        return buf
    # unequal ranges: one broadcast per owner, all issued asynchronously (NCCL runs them back to back on its stream).
    # Every rank receives exactly the bytes it is missing - no padding to the largest range (mip 0 of the specular
    # cubemap is 75 % of the texels but 1 % of the cost, so ranges differ by 50x in size).
    works = []
    for r, (a, b) in enumerate(ranges):
        if b > a:
            works.append(dist.broadcast(buf[a:b], src=dist.get_global_rank(group, r) if group is not None else r,
                                        group=group, async_op=True))
    for w in works:
        w.wait()
    return buf


class InterleavedSpecularPlan:
    """Equal-cost AND equal-size partition of the specular prefilter for one all-gather.

    Cost-balanced contiguous ranges differ 50x in size (mip 0 is 75 % of the texels and 1 % of the cost), which forces
    either padding or one broadcast per owner (8 collectives ~ 0.3 ms of launch latency at 8 GPUs, measured). Instead
    every mip whose 6*n rows divide by `world` is split into `world` equal row blocks (rank r takes block r of EVERY such
    mip: equal cost and equal bytes by construction); the few tiny mips that do not divide are simply computed by every
    rank (a few dozen texels). The gather is then: pack my blocks -> ONE all_gather_into_tensor -> one strided copy per
    split mip back into the packed cubemap.
    """

    def __init__(self, res: int, mips: int, world: int):
        self.res, self.mips, self.world = res, mips, world
        self.split, self.replicated = [], []      # (mip, row0 (flattened), rows_per_rank, n) / (mip, row0, rows, n)
        row0 = 0
        for m in range(mips):
            n = res >> m
            rows = 6 * n
            if rows % world == 0 and world > 1:
                self.split.append((m, row0, rows // world, n))
            else:
                self.replicated.append((m, row0, rows, n))
            row0 += rows
        self.total_rows = row0
        self.chunk_texels = sum(k * n for (_, _, k, n) in self.split)

    def row_ranges(self, rank: int):
        """flattened (mip, face, row) ranges this rank computes"""
        out = [(r0 + rank * k, r0 + (rank + 1) * k) for (_, r0, k, _) in self.split]
        out += [(r0, r0 + rows) for (_, r0, rows, _) in self.replicated]
        return sorted((a, b) for a, b in out if b > a)     # increasing and disjoint: what vq_specular_prefilter_ranges takes

    def texel_range(self, row_a: int, row_b: int):
        return specular_row_to_texel(self.res, self.mips, row_a), specular_row_to_texel(self.res, self.mips, row_b)

    def gather(self, cube_t, rank: int, group=None):
        """cube_t: [texels, 4] packed cubemap; on entry this rank's row_ranges are filled; on exit all are."""
        import torch
        import torch.distributed as dist
        if self.world == 1 or not self.split:
            return cube_t
        parts = []
        for (_, r0, k, _) in self.split:
            a, b = self.texel_range(r0 + rank * k, r0 + (rank + 1) * k)
            parts.append(cube_t[a:b])
        send = torch.cat(parts, dim=0)
        recv = torch.empty((self.world * self.chunk_texels,) + tuple(cube_t.shape[1:]), dtype=cube_t.dtype, device=cube_t.device)
        dist.all_gather_into_tensor(recv, send, group=group)
        recv = recv.view(self.world, self.chunk_texels, *cube_t.shape[1:])
        off = 0
        for (_, r0, k, n) in self.split:
            a, b = self.texel_range(r0, r0 + self.world * k)          # the whole mip: rank blocks are contiguous, in rank order
            cube_t[a:b].view(self.world, k * n, *cube_t.shape[1:]).copy_(recv[:, off:off + k * n])
            off += k * n
        return cube_t


def _signal_at(signal, epoch: int):
    """a copy of the VqPeerSignal `signal` with `epoch` (None stays None: no rendezvous)"""
    if signal is None:
        return None
    import ctypes as C
    s = type(signal)()
    C.memmove(C.addressof(s), C.addressof(signal), C.sizeof(s))
    s.epoch = epoch & 0xFFFFFFFF
    return s


class EnvironmentStep:
    """One rank's share of PreFilterEnvironmentMap across GPUs, with no collective library: every pass stores its band into every
    rank's buffers over peer mappings, and the kernels' last CTAs run the rendezvous (DESIGN.md §6). In stream order:
      1. diffuse(): K2 on this rank's rows of equal_tiles(6 * res, world) (every texel costs the same) into every rank's diffuse
         cube, rendezvous with epoch e;
      2. finish(): K5 on the local diffuse cube into the local blurred cube (one launch), then K3 on plan.row_ranges(rank) into
         every rank's specular cube, rendezvous with epoch e + 1, then vq_environment_prepare of the local maps (when `env` is given).
    run() is both; it returns the next free epoch, e + 2. The blurred cube must not be a peer destination of any call: the next
    step's diffuse stores may land while this rank still reads its blurred cube."""

    def __init__(self, ctx, hdri, diffuse_cubes, blurred, spec_cubes, rank: int, world: int, plan: "InterleavedSpecularPlan" = None,
                 diffuse_params=None, num_samples: int = 512, env=None):
        """diffuse_cubes / spec_cubes: Cubemap descriptors, the local one first, then the peers' mapped ones; blurred: the local
        blurred diffuse cube; diffuse_params: the keyword arguments of Context.diffuse_irradiance (step, n_phi, n_theta, src_mip);
        env: the local EnvironmentMaps to prepare after the step, or None"""
        assert len(diffuse_cubes) == len(spec_cubes) == world and 0 <= rank < world
        self.ctx, self.hdri, self.diffuse_cubes, self.blurred, self.spec_cubes = ctx, hdri, list(diffuse_cubes), blurred, list(spec_cubes)
        self.rows = equal_tiles(6 * diffuse_cubes[0].res, world)[rank]
        plan = plan if plan is not None else InterleavedSpecularPlan(spec_cubes[0].res, spec_cubes[0].mips, world)
        self.spec_ranges = plan.row_ranges(rank)
        self.diffuse_params = dict(diffuse_params or {})
        self.num_samples, self.env = num_samples, env

    def diffuse(self, epoch: int, signal=None, stream=None):
        self.ctx.diffuse_irradiance_multi(self.hdri, self.diffuse_cubes, row_begin=self.rows[0], row_end=self.rows[1], stream=stream,
                                          signal=_signal_at(signal, epoch), **self.diffuse_params)

    def finish(self, epoch: int, signal=None, stream=None):
        self.ctx.gaussian_blur_cube(self.diffuse_cubes[0], self.blurred, stream=stream)
        self.ctx.specular_prefilter_ranges(self.hdri, self.spec_cubes, self.spec_ranges, self.num_samples,
                                           signal=_signal_at(signal, epoch + 1), stream=stream)
        if self.env is not None:
            self.ctx.environment_prepare(self.env, stream=stream)

    def run(self, epoch: int, signal=None, stream=None) -> int:
        self.diffuse(epoch, signal, stream)
        self.finish(epoch, signal, stream)
        return epoch + 2
