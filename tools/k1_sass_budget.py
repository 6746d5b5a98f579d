"""CPU-only: K1's instruction budget and the two models that say where its issue slots and L1 wavefronts go.

  python tools/k1_sass_budget.py [--src vq_forward.cu] [--models] [--json]

SASS budget: compiles vq_forward.cu for sm_90a into a temporary directory (nvcc -cubin -Xptxas -v), disassembles it with
cuobjdump and splits the bench's instantiation (forward_kernel<false,false,false>) into segments along its control flow:
  set-up        from the row's mbarrier wait to the TINY warp vote (LDS of the texels, V, N, k, Smith-G of V)
  point light   the body of the (non-TINY) point-light loop, and its hot path (without the blocks that call exact_ndoth)
  spot light    the body of the spot loop (no spot light in bench.py's frame)
  directional   the directional light
  env+compose   the environment gathers, exchanges, blends, composition and stores of the pair (full IBL and diffuse-only)
  callees       every out-of-line function, named after the call sites that reach it
Each row gives the instruction count and the SHFL, FSEL/SEL, MOV, BSSY/BSYNC, MUFU, LDG and IMAD.WIDE counts; registers and
spills come from ptxas for every forward_kernel instantiation. Counts are static: each segment runs once per pixel pair (the
light bodies once per light), the callees only for the flagged pixels.

--models adds two float64 models of bench.py's 4K frame (synth.gbuffer, synth.scene_constants; K1's pixel -> warp mapping:
pixel A = x0 + 32w + lane, pixel B = A + 128):
  exact paths   the share of pixel-light pairs with t < T_EXACT and N.L > 0, and of warps in which at least one lane of pixel A
                (or B) takes exact_ndoth; the same for |N.V| < NV_EXACT (exact_nv)
  L1 lines      distinct 128-byte lines per gather instruction, per pixel, for the diffuse cube, the specular cube and the LUT:
                one lane per 32-byte record (two LDG.128, each reading every lane's half) against lane pairs (each LDG.128
                reading two lanes' records whole)
"""
import argparse, json, os, re, subprocess, sys, tempfile
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vqengine_b200", "csrc")      # headers, also for a --src copied elsewhere (e.g. an older revision)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")
BENCH_KERNEL = "forward_kernelILb0ELb0ELb0E"
INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")


def compile_sass(src):
    with tempfile.TemporaryDirectory() as td:
        cubin = os.path.join(td, "k1.cubin")
        r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                            "-Xptxas", "-v", "-cubin", "-I", CSRC, "-o", cubin, src], capture_output=True, text=True)
        if r.returncode:
            sys.exit(r.stdout + r.stderr)
        sass = subprocess.run([CUOBJDUMP, "-sass", cubin], capture_output=True, text=True, check=True).stdout
    return r.stderr, sass


def ptxas_resources(log):
    """{instantiation: (registers, spill store bytes, spill load bytes)} of every forward_kernel"""
    res, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1) if "forward_kernel" in m.group(1) else None
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            res.setdefault(cur, [0, 0, 0])[1:] = [int(m.group(1)), int(m.group(2))]
        m = re.search(r"Used (\d+) registers", line)
        if m:
            res.setdefault(cur, [0, 0, 0])[0] = int(m.group(1))
    out = {}
    for name, v in res.items():
        m = re.search(r"forward_kernelILb(\d)ELb(\d)E(?:Lb(\d)E)?", name)
        out["<%s,%s,%s>" % tuple({"0": "false", "1": "true", None: "false"}[g] for g in m.groups())] = tuple(v)
    return out


def function_insns(sass, key):
    """[(pc, text)] of the function whose name contains `key`"""
    parts = re.split(r"\n\s*Function : ", sass)
    for p in parts[1:]:
        if key in p.split("\n", 1)[0]:
            return [(int(m.group(1), 16), m.group(2)) for m in INSN.finditer(p)]
    sys.exit("instantiation %s not found in the SASS" % key)


def opcode(text):
    t = re.sub(r"^@!?U?P[T0-9]+\s+", "", text)
    return t.split()[0]


def branch_target(text):
    m = re.search(r"\b(?:BRA|CALL\.REL\.NOINC)\b.*?(0x[0-9a-f]+)\s*$", text)
    return int(m.group(1), 16) if m else None


def classify(insns):
    c = Counter()
    for _, t in insns:
        op = opcode(t)
        base = op.split(".")[0]
        c["insns"] += 1
        if base == "SHFL": c["SHFL"] += 1
        if base in ("FSEL", "SEL"): c["SEL"] += 1
        if base in ("MOV", "UMOV"): c["MOV"] += 1
        if base in ("BSSY", "BSYNC"): c["BSSY"] += 1
        if base == "MUFU": c["MUFU"] += 1
        if base == "LDG": c["LDG"] += 1
        if op.startswith("IMAD.WIDE"): c["IMAD.WIDE"] += 1
    return c


def segments(ins):
    pcs = [p for p, _ in ins]
    idx = {p: i for i, p in enumerate(pcs)}
    text = dict(ins)
    vote = next(i for i, (_, t) in enumerate(ins) if opcode(t).startswith("VOTE"))
    wait = max(i for i in range(vote) if opcode(ins[i][1]).startswith("SYNCS.PHASECHK"))
    tiny = next(branch_target(t) for _, t in ins[vote:] if opcode(t) == "BRA")          # the TINY instantiation of the lights
    seg = {"set-up": ins[wait + 2:vote + 1]}
    # backward branches of the non-TINY light region: the point loop, then the spot loop
    loops = [(branch_target(t), p) for p, t in ins[vote:idx[tiny]] if opcode(t) == "BRA" and branch_target(t) < p]
    (p0, p1), (s0, s1) = loops[0], loops[1]
    body = lambda a, b: ins[idx[a]:idx[b] + 1]
    seg["point light"] = body(p0, p1)
    seg["spot light"] = body(s0, s1)
    # directional: after the spot loop up to the unconditional branch to the environment code
    j = idx[s1] + 1
    while not (opcode(ins[j][1]) == "BRA" and not ins[j][1].startswith("@")):
        j += 1
    env = branch_target(ins[j][1])
    d0 = idx[s1] + 1
    while opcode(ins[d0][1]) != "BRA" or branch_target(ins[d0][1]) != env:      # the dirEnabled guard
        d0 += 1
    seg["directional"] = ins[d0 + 1:j + 1]
    # environment: [env, split) and [split, end), end = the target of the first variant's closing branch
    e = idx[env]
    split = next(branch_target(t) for _, t in ins[e:] if opcode(t) == "BRA" and t.startswith("@"))
    close = next(i for i in range(e, idx[split]) if opcode(ins[i][1]) == "BRA" and not ins[i][1].startswith("@")
                 and branch_target(ins[i][1]) > split) if any(opcode(t) == "BRA" and not t.startswith("@") and branch_target(t) > split
                                                            for _, t in ins[e:idx[split]]) else None
    first = ins[e:idx[split]]
    end = branch_target(ins[close][1]) if close is not None else None
    if end is None:     # the first variant falls through: the second one ends with a branch past it
        end = next(branch_target(t) for _, t in ins[idx[split]:] if opcode(t) == "BRA" and not t.startswith("@"))
    second = ins[idx[split]:idx[end]]
    a, b = sorted((first, second), key=lambda s: classify(s)["LDG"])
    seg["env+compose (diffuse-only)"] = a
    seg["env+compose (full IBL)"] = b
    # callees, named by the segments that call them
    calls = {}
    for name in ("set-up", "point light", "spot light"):
        for p, t in seg[name]:
            if opcode(t) == "CALL.REL.NOINC":
                calls.setdefault(branch_target(t), name)
    names = {"set-up": "exact_nv", "point light": "exact_ndoth", "spot light": "exact_spot_cos"}
    for tgt, who in sorted(calls.items()):
        k = idx[tgt]
        r = next(i for i in range(k, len(ins)) if opcode(ins[i][1]).startswith("RET"))
        seg["callee " + names[who]] = ins[k:r + 1]
    seg["point light, hot path"] = hot_path(seg["point light"])
    seg["directional, hot path"] = hot_path(seg["directional"])
    return seg


def hot_path(body_ins):
    """a light body without the forward-branched blocks that contain a CALL (the exact paths, taken by few warps)"""
    hot, i = [], 0
    while i < len(body_ins):
        p, t = body_ins[i]
        tg = branch_target(t) if opcode(t) == "BRA" and t.startswith("@") else None
        if tg is not None and tg > p and tg <= body_ins[-1][0] and any(
                opcode(x) == "CALL.REL.NOINC" for q, x in body_ins[i + 1:] if q < tg):
            hot.append((p, t))
            while i < len(body_ins) and body_ins[i][0] < tg:
                i += 1
            continue
        hot.append((p, t)); i += 1
    return hot


ORDER = ["set-up", "point light", "point light, hot path", "spot light", "directional", "directional, hot path", "env+compose (full IBL)",
         "env+compose (diffuse-only)", "callee exact_ndoth", "callee exact_nv", "callee exact_spot_cos"]
COLS = ["insns", "SHFL", "SEL", "MOV", "BSSY", "MUFU", "LDG", "IMAD.WIDE"]


def budget(src):
    log, sass = compile_sass(src)
    seg = segments(function_insns(sass, BENCH_KERNEL))
    return {k: dict(classify(seg[k])) for k in ORDER if k in seg}, ptxas_resources(log)


# ------------------------------------------------------------------------------------------------------------------
# CPU models of bench.py's 4K frame
# ------------------------------------------------------------------------------------------------------------------
def load_synth():
    import importlib, types
    pkg = types.ModuleType("_vq_models"); pkg.__path__ = [os.path.join(ROOT, "vqengine_b200")]
    sys.modules["_vq_models"] = pkg
    return importlib.import_module("_vq_models.synth")


def frame(rows_every):
    import numpy as np
    synth = load_synth()
    W, H = 3840, 2160
    pf, pv = synth.scene_constants(W, H, 9)
    pos, nr, _ = synth.gbuffer(W, H)
    sel = np.arange(0, H, rows_every)
    P = pos[sel, :, :3].astype(np.float64); Ns = nr[sel, :, :3].astype(np.float64); r = nr[sel, :, 3].astype(np.float64)
    cam = np.array([pv.CameraPosition.x, pv.CameraPosition.y, pv.CameraPosition.z])
    return W, pf, P, Ns, r, cam


def warp_any(flag, W):
    """share of (row, warp) with any lane flagged, for pixel A and pixel B of K1's 256-pixel tiles"""
    import numpy as np
    x = np.arange(W); half = (x % 256) // 128; key = (x // 256) * 4 + (x % 128) // 32
    out = []
    for h in (0, 1):
        f = np.zeros((flag.shape[0], key.max() + 1), bool)
        np.logical_or.at(f, (slice(None), key[half == h]), flag[:, half == h])
        out.append(f.mean())
    return out


def model_exact(rows_every=10):
    import numpy as np
    W, pf, P, Ns, r, cam = frame(rows_every)
    L = pf.Lights
    V = cam - P; V /= np.linalg.norm(V, axis=-1, keepdims=True)
    N = Ns / np.linalg.norm(Ns, axis=-1, keepdims=True)
    a2m1 = r ** 4 - 1
    lights = [("point%d" % i, np.array([l.position.x, l.position.y, l.position.z]))
              for i, l in enumerate(L.point_lights[:L.numPointLights])]
    if L.directional.enabled:
        d = -np.array([L.directional.lightDirection.x, L.directional.lightDirection.y, L.directional.lightDirection.z])
        lights.append(("directional", d / np.linalg.norm(d)))
    rows = []
    for name, lp in lights:
        Wi = np.broadcast_to(lp, P.shape) if name == "directional" else lp - P
        Wi = Wi / np.linalg.norm(Wi, axis=-1, keepdims=True)
        Hh = V + Wi; Hh /= np.linalg.norm(Hh, axis=-1, keepdims=True)
        nh = np.clip((N * Hh).sum(-1), 0, 1)
        flag = (nh * nh * a2m1 + 1 < 0.02) & ((N * Wi).sum(-1) > 0)
        rows.append((name, flag.mean(), *warp_any(flag, W)))
    g = np.abs((N * V).sum(-1)) < 1e-3
    rows.append(("|N.V| < 1e-3", g.mean(), *warp_any(g, W)))
    return rows


def model_lines(rows_every=40):
    import numpy as np
    W, pf, P, Ns, rough, cam = frame(rows_every)
    V = cam - P; V /= np.linalg.norm(V, axis=-1, keepdims=True)

    def cube_rec(d, N, base):
        ax, ay, az = np.abs(d[..., 0]), np.abs(d[..., 1]), np.abs(d[..., 2])
        isX = (ax >= ay) & (ax >= az); isY = ~isX & (ay >= az)
        ma = np.where(isX, ax, np.where(isY, ay, az)); mv = np.where(isX, d[..., 0], np.where(isY, d[..., 1], d[..., 2]))
        pos = mv > 0
        u = np.where(isX, np.where(pos, -d[..., 2], d[..., 2]), np.where(isY, d[..., 0], np.where(pos, d[..., 0], -d[..., 0])))
        v = np.where(isY, np.where(pos, -d[..., 2], d[..., 2]), d[..., 1])
        face = np.where(isX, 0, np.where(isY, 2, 4)) + np.where(pos, 0, 1)
        Pp = N + 2
        x = u / ma * N / 2 + N / 2 - 0.5; y = -v / ma * N / 2 + N / 2 - 0.5
        return base + face * Pp * Pp + (np.floor(y).astype(np.int64) + 1) * Pp + np.floor(x).astype(np.int64) + 1, Pp

    dr, dP = cube_rec(Ns, 64, 0)                                   # bench: diffuse 64^2, specular 512^2 x 9 mips, LUT 1024^2
    offs = [0]
    for m in range(9):
        offs.append(offs[-1] + 6 * ((512 >> m) + 2) ** 2)
    mip = np.clip((rough * 8).astype(np.int64), 0, 8)
    R = -V - 2 * ((-V * Ns).sum(-1, keepdims=True)) * Ns
    sr = np.zeros_like(mip); sP = np.zeros_like(mip)
    for m in range(9):
        r_, p_ = cube_rec(R, 512 >> m, offs[m]); sr = np.where(mip == m, r_, sr); sP = np.where(mip == m, p_, sP)
    nsnv = np.clip((Ns * V).sum(-1), 0, 1)
    lx = np.clip(np.floor(nsnv * 1024 - 0.5).astype(np.int64) + 1, 0, 1024)
    ly = np.clip(np.floor(rough * 1024 - 0.5).astype(np.int64) + 1, 0, 1024)
    lr = ly * 1026 + lx

    def distinct(lines):
        s = np.sort(lines, axis=-1)
        return (1 + (np.diff(s, axis=-1) != 0).sum(-1)).sum()

    def count(rec_rows):
        own = pair = n = 0
        for rec in rec_rows:
            for half in (0, 1):
                for w in range(4):
                    cols = np.arange(W // 256)[:, None] * 256 + half * 128 + w * 32 + np.arange(32)[None, :]
                    r = rec[:, cols]
                    own += distinct((r * 16) // 128) + distinct((r * 16 + 16) // 128)
                    for par in (0, 1):
                        rr = r[..., par::2]
                        pair += distinct(np.concatenate([(rr * 16) // 128, (rr * 16 + 16) // 128], axis=-1))
                    n += r.shape[0] * r.shape[1] * 32
        return own / n, pair / n

    return [(name,) + count(rows) for name, rows in (("diffuse cube", [dr, dr + dP]), ("specular cube", [sr, sr + sP]),
                                                     ("BRDF LUT", [lr]))]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--src", default=os.path.join(CSRC, "vq_forward.cu"),
                    help="the K1 source to count, e.g. `git show REV:vqengine_b200/csrc/vq_forward.cu > /tmp/k1.cu` for a before/after")
    ap.add_argument("--models", action="store_true", help="also run the exact-path and L1-line models of the 4K frame")
    ap.add_argument("--json", action="store_true", help="one JSON object instead of tables")
    a = ap.parse_args()
    seg, res = budget(a.src)
    # what one pixel pair of bench.py's frame issues outside the exact paths: 4 point lights, the directional light, full IBL
    common = (seg["set-up"]["insns"] + 4 * seg["point light, hot path"]["insns"] + seg["directional, hot path"]["insns"] +
              seg["env+compose (full IBL)"]["insns"])
    out = {"segments": seg, "bench_pair_common_path": common,
           "resources": {k: dict(zip(("registers", "spill_stores", "spill_loads"), v)) for k, v in res.items()}}
    if a.models:
        out["exact_paths"] = [dict(zip(("case", "pairs", "warps_A", "warps_B"), r)) for r in model_exact()]
        out["l1_lines_per_px"] = [dict(zip(("gather", "one_lane_per_record", "lane_pairs"), r)) for r in model_lines()]
    if a.json:
        print(json.dumps(out))
        return
    print("K1 SASS budget, forward_kernel<false,false,false> (static instructions per segment; a pixel pair per thread)")
    print("%-28s" % "segment" + "".join("%10s" % c for c in COLS))
    for k, c in seg.items():
        print("%-28s" % k + "".join("%10d" % c.get(col, 0) for col in COLS))
    print("bench.py's pixel pair outside the exact paths (set-up + 4 point + directional + full IBL): %d" % common)
    print("\nptxas: registers / spill stores / spill loads")
    for k, v in sorted(res.items()):
        print("  forward_kernel%-20s %4d %6d %6d" % (k, *v))
    if a.models:
        print("\nexact paths (bench.py 4K frame): share of pixel-light pairs flagged, of warps calling for pixel A / B")
        for r in out["exact_paths"]:
            print("  %-14s %7.3f %%   %5.1f %%  %5.1f %%" % (r["case"], 100 * r["pairs"], 100 * r["warps_A"], 100 * r["warps_B"]))
        print("\nL1 wavefronts per pixel (distinct 128-byte lines per gather): one lane per record / lane pairs")
        for r in out["l1_lines_per_px"]:
            print("  %-14s %5.2f  %5.2f" % (r["gather"], r["one_lane_per_record"], r["lane_pairs"]))


if __name__ == "__main__":
    main()
