"""Seeded scenes for the shadowed pass (SURVEY §8(f).4) over the whole domain of its PCF decisions.

Every scene keeps all eleven casters active (5 point, 5 spot, the directional light), so every 5-bit slot of the per-pixel record
is in use, and lays its pixels out in warps of 32 (a row is 128 pixels = 4 warps) so that the device's warp vote sees what each
group was built for:

  * point casters: warps around caster 0 that take each of the six cube faces' axis paths (+Y included: pixels ABOVE the light),
    warps that mix axes, warps partly or wholly out of range, warps whose axis gap sits just above / just below the
    `cube_axis_is_certain` bound (2.01 r) or well inside it (r .. 2 r, where some taps do change face), and pixels on cube edges
    and corners (|x| = |y| exactly, where the tie rule X > Y > Z decides);
  * spot casters: perspective views (left-handed perspective times a look-at, uploaded row-major) with varied fov / near / far,
    and pixels behind the light, between the light and the near plane, on the frustum's edges and at the light itself (w = 0);
  * the directional light: an axis-aligned orthographic view with exact power-of-two scales, so that the exact probes (one warp) put
    taps exactly on texel boundaries, a pixel exactly on the frustum's edge (px = 1), and map texels equal to the fp32 value
    being compared (`>` false, one ulp away true).

Map sizes vary per scene: cubes 1, 2, 5, 8, 33; directional maps 1x1, 7x5, 16x16, 33x17, 64x64."""
import numpy as np

W = 128                        # pixels per row: four warps
N_POINT, N_SPOT = 5, 5
SIZES = [  # (cube resolution, (directional w, h), (spot w, h))
    (1, (1, 1), (16, 16)),
    (2, (7, 5), (20, 12)),
    (5, (16, 16), (9, 9)),
    (8, (33, 17), (32, 32)),
    (33, (64, 64), (13, 31)),
]
GROUND_Y = -8.0               # the height-field patch under the spot lights and the directional view
DIR_SCALE = 1.0 / 32.0         # directional view: px = x / 32, py = z / 32, pz = 0.5 - y / 64 (all exact for dyadic x, y, z)


def look_at_lh(eye, at, up):
    z = np.asarray(at, np.float64) - eye; z /= np.linalg.norm(z)
    x = np.cross(up, z); x /= np.linalg.norm(x)
    y = np.cross(z, x)
    V = np.eye(4)
    V[:3, 0], V[:3, 1], V[:3, 2] = x, y, z
    V[3, :3] = [-x @ eye, -y @ eye, -z @ eye]
    return V


def perspective_fov_lh(fov, aspect, near, far):
    h = 1.0 / np.tan(fov / 2); w = h / aspect; q = far / (far - near)
    P = np.zeros((4, 4))
    P[0, 0], P[1, 1], P[2, 2], P[2, 3], P[3, 2] = w, h, q, 1.0, -q * near
    return P


def dir_matrix():
    """row-major, row vector: (x, y, z, 1) -> (x/32, z/32, 0.5 - y/64, 1): the light looks down -Y, orthographic"""
    m = np.zeros((4, 4))
    m[0, 0] = DIR_SCALE; m[2, 1] = DIR_SCALE; m[1, 2] = -DIR_SCALE / 2; m[3, 2] = 0.5; m[3, 3] = 1.0
    return m


def _set_matrix(dst, M):
    f = np.asarray(M, np.float32).reshape(16)
    for k in range(16):
        dst.m[k] = float(f[k])


def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def disk_r(P, cam, far):
    """the offset radius bound of cube_axis_is_certain: b * (1 + |P - cam| / far) / 8"""
    return 0.7071067811865475 * (1.0 + np.linalg.norm(np.asarray(P, np.float64) - cam, axis=-1) / far) * 0.125


class Scene:
    """pf / pv constant blocks, G-buffer planes [H, W, 4] x3, and the maps (numpy float32); `groups` names each warp's purpose"""

    def __init__(self, idx, seed=0):
        from vqengine_b200 import synth
        self.idx = idx
        self.cube_res, (self.dir_w, self.dir_h), (self.spot_w, self.spot_h) = SIZES[idx % len(SIZES)]
        rng = np.random.default_rng(4000 + 97 * idx + seed)
        self.rng = rng
        pf, pv = synth.scene_constants(W, 8, 5, seed=idx + 1, n_point=2, n_spot=1, casters=True)
        self.pf, self.pv = pf, pv
        self.cam = np.array([0.0, 5.0, -17.0])
        pv.CameraPosition.x, pv.CameraPosition.y, pv.CameraPosition.z = self.cam
        L = pf.Lights
        L.numPointCasters, L.numSpotCasters = N_POINT, N_SPOT
        L.directional.enabled = 1; L.directional.shadowing = 1
        L.directional.depthBias = float(rng.integers(1, 41)) / 4096.0        # dyadic: pz - bias is exact for the exact probes
        # point casters: 0 is the axis light at the origin; the others are scattered around the pixels
        self.point_pos = np.zeros((N_POINT, 3))
        self.point_range = np.zeros(N_POINT)
        for i in range(N_POINT):
            l = L.point_casters[i]
            p = np.zeros(3) if i == 0 else rng.uniform(-12, 12, 3)
            l.position.x, l.position.y, l.position.z = (float(np.float32(c)) for c in p)
            l.range = float(rng.uniform(24, 40)) if i else 30.0
            l.color.x, l.color.y, l.color.z = rng.uniform(0.4, 1.0, 3)
            l.brightness = float(rng.uniform(300, 900))
            l.depthBias = float(rng.uniform(0.0, 0.05))
            self.point_pos[i] = [l.position.x, l.position.y, l.position.z]
            self.point_range[i] = l.range
        # spot casters: perspective views. Caster 0 sits at the origin, so that a pixel there has (x, y, w) = 0 exactly in fp32;
        # in scene 0 its near plane is 0 as well (z = 0 too: every quotient NaN, the texel coordinates NaN)
        self.spot_views = []
        for i in range(N_SPOT):
            s = L.spot_casters[i]
            eye = np.zeros(3) if i == 0 else np.array([rng.uniform(-10, 10), rng.uniform(9, 16), rng.uniform(-10, 10)])
            eye = eye.astype(np.float32).astype(np.float64)
            at = np.array([rng.uniform(-4, 4), GROUND_Y, rng.uniform(-4, 4)])
            d = _unit(at - eye)
            s.position.x, s.position.y, s.position.z = eye
            s.spotDir.x, s.spotDir.y, s.spotDir.z = d
            s.innerConeAngle = float(rng.uniform(0.4, 0.6)); s.outerConeAngle = s.innerConeAngle + float(rng.uniform(0.2, 0.4))
            s.color.x, s.color.y, s.color.z = rng.uniform(0.4, 1.0, 3)
            s.brightness = float(rng.uniform(300, 900))
            s.depthBias = float(rng.uniform(0.0005, 0.01))
            s.range = 100.0
            fov = float(rng.uniform(0.5, 1.6) if i else rng.uniform(1.3, 1.6)); near = float(rng.choice([0.05, 0.5, 2.0, 6.0])); far = float(rng.uniform(30, 80))
            if i == 0 and idx == 0:
                near = 0.0
            V = look_at_lh(eye, at, np.array([0.0, 0.0, 1.0]) if abs(d[1]) > 0.9 else np.array([0.0, 1.0, 0.0]))
            Pr = perspective_fov_lh(fov, self.spot_w / self.spot_h, near, far)
            M = V @ Pr
            _set_matrix(L.shadowViews[i], M)
            self.spot_views.append(dict(eye=eye, at=at, near=near, far=far, fov=fov, V=V, Pr=Pr,
                                        M=np.asarray(M, np.float32).astype(np.float64)))
        _set_matrix(L.shadowViewDirectional, dir_matrix())
        pf.f2SpotLightShadowMapDimensions.x, pf.f2SpotLightShadowMapDimensions.y = float(self.spot_w), float(self.spot_h)
        pf.f2DirectionalLightShadowMapDimensions.x, pf.f2DirectionalLightShadowMapDimensions.y = float(self.dir_w), float(self.dir_h)
        self._layout()
        self._maps()

    # ---- pixels ------------------------------------------------------------------------------------------------------------
    def _layout(self):
        rng = self.rng
        warps, groups = [], []
        far0 = self.point_range[0]

        def add(name, P, N=None):
            P = np.asarray(P, np.float32).reshape(-1, 3)
            assert len(P) == 32
            if N is None:                                          # facing caster 0 (observable for it), unit length
                N = _unit(self.point_pos[0] + 1e-3 - P)
            warps.append((P, np.asarray(N, np.float32).reshape(-1, 3))); groups.append(name)

        # the six faces of caster 0: tap directions -(Lw + o) = P - light, major axis +-X, +-Y, +-Z with a wide gap
        for a in range(3):
            for sgn in (1.0, -1.0):
                for _ in range(2):
                    P = rng.uniform(-1.5, 1.5, (32, 3)); P[:, a] = sgn * rng.uniform(8, 14, 32)
                    add(f"axis{2 * a + (0 if sgn > 0 else 1)}", P)
        # mixed axes: directions all over the sphere
        for _ in range(3):
            add("mixed", _unit(rng.normal(size=(32, 3))) * rng.uniform(4, 20, (32, 1)))
        # some lanes (lane 0 included) out of caster 0's range, the rest on one axis; and a warp with every lane out of range
        P = rng.uniform(-1.5, 1.5, (32, 3)); P[:, 1] = rng.uniform(8, 14, 32)
        out = rng.uniform(size=32) < 0.4; out[0] = True
        P[out] = _unit(rng.normal(size=(out.sum(), 3))) * (far0 + rng.uniform(0.5, 5, (out.sum(), 1)))
        add("partial_out", P)
        P = _unit(rng.normal(size=(32, 3))) * (far0 + rng.uniform(0.5, 5, (32, 1)))
        add("all_out", P)
        # the certainty gap: major - second = 2.01 r (1 +- 2^-10) + 1e-5 major, and r .. 2r (taps do change face there)
        for name, lo, hi in (("gap_above", 1 + 2 ** -10, 1 + 2 ** -9), ("gap_below", 1 - 2 ** -9, 1 - 2 ** -10), ("gap_inside", 0.5 / 2.01, 1.9 / 2.01)):
            P = np.zeros((32, 3))
            major = rng.uniform(8, 12, 32); second = rng.uniform(0.2, 0.9, 32) * major
            for _ in range(3):                                     # r depends on P itself: iterate to the fixed point
                P[:, 0], P[:, 1], P[:, 2] = rng.uniform(-0.5, 0.5, 32) * second, -major, second
                r = disk_r(P, self.cam, far0)
                f = rng.uniform(lo, hi, 32)
                second = major - (2.01 * f * r + 1e-5 * major)
            P[:, 0] = np.sign(P[:, 0]) * np.minimum(np.abs(P[:, 0]), 0.5 * second)
            P[:, 2] = second
            add(name, P)
        # cube edges and corners: |x| = |y| (and = |z|) exactly in fp32, the light at the origin so Lw = -P exactly
        E = []
        for k in range(32):
            m = float(rng.integers(3, 12)); s = rng.choice([-1.0, 1.0], 3)
            if k % 4 == 0: v = [m, m, m]                            # corner
            elif k % 4 == 1: v = [m, m, rng.uniform(-0.5, 0.5) * m]   # X/Y edge
            elif k % 4 == 2: v = [m, rng.uniform(-0.5, 0.5) * m, m]   # X/Z edge
            else: v = [rng.uniform(-0.5, 0.5) * m, m, m]              # Y/Z edge
            E.append(np.array(v) * s)
        add("edges", E)
        # spot caster 0 probes: at the light (w = 0), beside it (w = 0, x != 0), behind it, between it and the near plane,
        # and on the frustum's edges
        sv = self.spot_views[0]
        Vinv = np.linalg.inv(sv["V"])
        S = [sv["eye"], sv["eye"] + [3.0, 0.0, 0.0]]
        zdir = _unit(sv["at"] - sv["eye"])
        for t in (-0.5, -3.0, 0.3 * sv["near"], 0.9 * sv["near"]):
            S.append(sv["eye"] + zdir * t + rng.uniform(-0.05, 0.05, 3) * abs(t))
        while len(S) < 32:                                        # clip-space points on the frustum's faces, back to world
            c = rng.uniform(-1, 1, 3); c[2] = rng.uniform(0.2, 0.95)
            c[rng.integers(0, 2)] = rng.choice([-1.0, 1.0])
            z = sv["near"] + c[2] * 20.0                                                   # view depth
            h = np.array([c[0] * z / sv["Pr"][0, 0], c[1] * z / sv["Pr"][1, 1], z, 1.0]) @ Vinv
            S.append(h[:3])
        add("spot_probes", S, _unit(sv["eye"] - np.asarray(S) + 1e-3))
        # directional probes (exact): see exact_probes
        self.n_ground_rows = 2
        rows = (len(warps) + 3) // 4 + self.n_ground_rows
        H = rows
        pos = np.zeros((H, W, 4), np.float32); nrm = np.zeros((H, W, 4), np.float32)
        for i, (P, N) in enumerate(warps):
            r, c = divmod(i, 4)
            pos[r, 32 * c:32 * c + 32, :3] = P; nrm[r, 32 * c:32 * c + 32, :3] = N
        self.groups = groups + ["ground"] * (rows * 4 - len(groups))
        # the rest: a height-field patch under the spot lights and the directional view, normals jittered (not unit)
        first = len(warps)
        for i in range(first, rows * 4):
            r, c = divmod(i, 4)
            x = rng.uniform(-14, 14, 32); z = rng.uniform(-14, 14, 32)
            y = GROUND_Y + 2.0 * np.sin(0.3 * x) * np.cos(0.25 * z)
            n = _unit(np.stack([-0.6 * np.cos(0.3 * x) * np.cos(0.25 * z), np.ones(32), 0.5 * np.sin(0.3 * x) * np.sin(0.25 * z)], -1))
            n = n * rng.uniform(0.7, 1.3, (32, 1)) + rng.normal(0, 0.1, (32, 3))
            pos[r, 32 * c:32 * c + 32, :3] = np.stack([x, y, z], -1); nrm[r, 32 * c:32 * c + 32, :3] = n
        self._exact_probe_pixels(pos, nrm)
        pos[..., 3] = rng.uniform(0, 0.3, (H, W)); nrm[..., 3] = rng.uniform(0.05, 1.0, (H, W))
        alb = np.empty((H, W, 4), np.float32)
        alb[..., :3] = rng.uniform(0.1, 0.9, (H, W, 3)); alb[..., 3] = rng.uniform(0, 1, (H, W)) * (rng.uniform(size=(H, W)) < 0.3)
        self.planes = [pos, nrm, alb]
        self.H = H

    def _exact_probe_pixels(self, pos, nrm):
        """the last row's first warp: directional taps on exact texel boundaries / the frustum's edge (x, z dyadic)"""
        r = pos.shape[0] - 1
        rng = self.rng
        P = np.zeros((32, 3))
        for k in range(32):
            x = float(rng.integers(-32, 33)) if k > 3 else [32.0, -32.0, 32.0, 0.0][k]     # px = x/32: exactly +-1 on lanes 0..2
            z = float(rng.integers(-32, 33)) if k > 3 else [0.0, 5.0, -32.0, 32.0][k]
            y = float(rng.integers(-64, 64)) / 8.0
            P[k] = [x, y, z]
        pos[r, :32, :3] = P
        nrm[r, :32, :3] = [0.0, 1.0, 0.0]
        self.exact_idx = r * W + np.arange(32)
        self.groups[r * 4] = "exact"

    # ---- maps ----------------------------------------------------------------------------------------------------------------
    def _maps(self):
        import pcf_ref
        rng = self.rng
        R = self.cube_res
        self.cubes = rng.uniform(0.15, 0.7, (N_POINT, 6, R, R)).astype(np.float32)      # x far: both sides of the pixels' distances
        # spot maps: texels spread over the depths the in-frustum pixels actually have, so that the comparisons split
        P = self.planes[0][..., :3].reshape(-1, 3).astype(np.float64)
        self.spots = np.empty((N_SPOT, self.spot_h, self.spot_w), np.float32)
        for i, sv in enumerate(self.spot_views):
            h = np.concatenate([P, np.ones((len(P), 1))], 1) @ sv["M"]
            with np.errstate(all="ignore"):
                pz = h[:, 2] / h[:, 3]
            pz = pz[np.isfinite(pz) & (pz > 0) & (pz < 1)]
            lo, hi = (np.quantile(pz, [0.05, 0.95]) if len(pz) > 8 else (0.3, 0.99))
            self.spots[i] = rng.uniform(lo, hi, (self.spot_h, self.spot_w))
        self.dmap = rng.uniform(0.35, 0.65, (self.dir_h, self.dir_w)).astype(np.float32)
        # the exact probes: every texel a probe's directional taps read holds exactly its fp32 pz - bias (on the lanes that
        # are on a boundary; lanes 0..3 keep the random texels so that the frustum-edge lanes count a mix)
        ex = self.planes[0].reshape(-1, 4)[self.exact_idx, :3].astype(np.float64)
        t = pcf_ref.dir_taps(self, ex)
        for k in range(4, len(ex), 2):
            self.dmap[t["ty"][k][None, :], t["tx"][k][:, None]] = t["pzb32"][k]
        # the lanes whose 25 texels all still hold their own value (later lanes may have overwritten shared texels)
        self.eq_lanes = np.array([k for k in range(4, len(ex), 2)
                                  if (self.dmap[t["ty"][k][None, :], t["tx"][k][:, None]] == t["pzb32"][k]).all()], np.int64)

    # ---- for the library calls ---------------------------------------------------------------------------------------------
    def shadow_maps_struct(self, vq, cubes=None, spots=None, dmap=None):
        """VqShadowMaps over host or device buffers (pointers given), or over this scene's numpy maps"""
        sm = vq.ShadowMaps()
        self._keep = [np.ascontiguousarray(a) for a in (self.cubes, self.spots, self.dmap)]
        sm.point_cubes, sm.point_res = cubes if cubes is not None else self._keep[0].ctypes.data, self.cube_res
        sm.spot_maps, sm.spot_width, sm.spot_height = spots if spots is not None else self._keep[1].ctypes.data, self.spot_w, self.spot_h
        sm.directional_map, sm.directional_width, sm.directional_height = dmap if dmap is not None else self._keep[2].ctypes.data, self.dir_w, self.dir_h
        return sm

    def warp_groups(self):
        """[H * W / 32] group names, warp index = pixel index // 32"""
        return np.array(self.groups)


def scenes():
    return [Scene(i) for i in range(len(SIZES))]
