"""Crafted, seeded scenes for the colour renderer (renderPointsInRecentVoxel -> getSubPixel<Vec3b> -> updateRgb), each built
on the restatement of `render_reference`, which asserts the scene's defining property while the scene is built.

Exact projection, as projection_cases.HALVES_CAM: with fx = fy = 256, the camera-frame depth pcz = 4 and cx, cy on a 1/64
grid, u = (pcx * 256) / 4 + cx = 64 * pcx + cx is exact, so a point placed at pcx = (u - cx) / 64 lands on u exactly.  Two
camera rotations are used: the identity, and q = (1/2, 1/2, 1/2, 1/2), whose matrix is exactly the cyclic permutation
camera = (z, x, y) of the world point.

Every scene loads its points through addPoints once (one rendering sweep, so each voxel is in the recent list once) into a
colour map of 0.25 m voxels with at most 128 points and 1 mm fine cells; the scenes keep at most 64 points per voxel, so
every point is stored.  A scene is rendered several times; its state is compared after each rendering.

  * ties:        tap products exactly k + 1/2 (k even and odd) at the fractions 1/2 / 1/2, 1/4 / 3/4 and 3/4 / 1/4;
  * saturation:  2x2 blocks of 253, 254, 255 whose rounded products sum to 256 at the first, second or third saturated
                 addition.  256 is the largest sum there is: each tap rounds up by at most 1/2 over an exact mean <= 255,
                 and 257 would need four ties k + 1/2 over 255s, which no dyadic weight gives;
  * bounds:      u and v exactly on fl(fov * n) + 1 and one ulp below, ceil(u) just below and just at (1 - fov) * n, and
                 the zero-weight taps at u = cols - 1, v = rows - 1, for fov 0, 0.0001, 0.005 and 0.25 at 640x480, 752x480
                 and 1280x1024;
  * depth:       pcz exactly 0.001 and one ulp either side, found by walking t_camera_world[2] by ulps;
  * gate:        a second rendering whose distance is exactly fl(obs_dist * 1.2), and one a ulp above it;
  * dist0:       t_world_camera on a stored point: obs_dist = 0 switches the distance gate off for good;
  * backwards:   a rendering 150 s and 200 s before the first observation (covariance exactly 0, then negative);
  * chain:       40 renderings with different images and poses.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

import render_reference as RR

VOXEL, CAP, FINE = 0.25, 128, 0.001
IDENTITY = (0.0, 0.0, 0.0, 1.0)
CYCLIC = (0.5, 0.5, 0.5, 0.5)          # camera = (z, x, y) of the world point
SIZES = ((480, 640), (480, 752), (1024, 1280))
FOVS = (0.0, 0.0001, 0.005, 0.25)
F = 256.0
Z = 4.0


@dataclass
class Render:
    cam: RR.Camera
    img: np.ndarray
    obs_time: float


@dataclass
class Scene:
    name: str
    points: np.ndarray                                   # (n, 3) float64, each coordinate a float32
    renders: list = field(default_factory=list)
    # filled by run(): per rendering the restatement's count, observations and the state of every point after it
    counts: list = field(default_factory=list)
    observations: list = field(default_factory=list)
    states: list = field(default_factory=list)

    def run(self):
        st = [RR.PointState() for _ in range(self.points.shape[0])]
        for r in self.renders:
            n, obs = RR.render(st, self.points, r.cam, r.img, r.obs_time)
            self.counts.append(n)
            self.observations.append(obs)
            self.states.append([RR.PointState(list(s.rgb), s.n_rgb, list(s.cov), s.obs_dist, s.last_obs) for s in st])
        return self


def camera(rows, cols, cx=0.0, cy=0.0, fov=0.005, q=IDENTITY, t_cw=(0.0, 0.0, 0.0), t_wc=(0.0, 0.0, 0.0), fx=F, fy=F):
    return RR.Camera(np.r_[q, t_cw, t_wc, [fx, fy, cx, cy, fov]], rows, cols)


def to_world(pc, q=IDENTITY):
    """the world point whose camera-frame coordinates are pc (t_camera_world = 0)"""
    x, y, z = pc
    return (x, y, z) if tuple(q) == IDENTITY else (y, z, x)


def on_pixel(u, v, cx, cy, q=IDENTITY):
    """the world point (float32-exact) that projects exactly to (u, v) at depth 4"""
    pc = ((u - cx) / 64.0, (v - cy) / 64.0, Z)
    assert all(float(np.float32(a)) == a for a in pc), (u, v)
    return to_world(pc, q)


def noise(rng, rows, cols):
    return rng.integers(0, 256, (rows, cols, 3), dtype=np.uint8)


def _unique(points):
    p = np.asarray(points, np.float64).reshape(-1, 3)
    assert np.array_equal(p, p.astype(np.float32).astype(np.float64))
    assert len({r.tobytes() for r in p.astype(np.float32)}) == p.shape[0], "two points share a stored position"
    keys = np.trunc(p.astype(np.float32).astype(np.float64) / VOXEL).astype(np.int64)
    _, per_voxel = np.unique(keys, axis=0, return_counts=True)
    assert per_voxel.max() <= 64
    return p


def _obs(scene, k, i):
    return scene.observations[k][i]


# ---- rounding ties ----------------------------------------------------------------------------------------------------
# pixel values whose product with each weight of a fraction pair is exactly k + 1/2
TIE_PIXELS = {(0.5, 0.5): [4 * k + 2 for k in range(64)],          # x 1/4
              (0.25, 0.75): [16 * k + 8 for k in range(16)],       # x 1/16, 3/16, 9/16
              (0.75, 0.25): [16 * k + 8 for k in range(16)]}


def ties(seed=1):
    rng = np.random.default_rng(seed)
    rows, cols, cx, cy = 480, 640, 3.25, 1.5
    img = noise(rng, rows, cols)
    pts, where = [], []
    for fi, (fv, fu) in enumerate(TIE_PIXELS):
        for j in range(12):
            a, b = 20 + 3 * j + 40 * fi, 30 + 3 * (j % 4) + 12 * (j // 4)
            u, v = a + fu, b + fv
            pts.append(on_pixel(u, v, cx, cy))
            where.append((fv, fu, a, b))
            vals = TIE_PIXELS[(fv, fu)]
            img[b:b + 2, a:a + 2, :] = rng.choice(vals, (2, 2, 3))
    cam = camera(rows, cols, cx, cy)
    sc = Scene("ties", _unique(pts), [Render(cam, img, 2.0), Render(cam, img[::-1, ::-1].copy(), 2.5)])
    # the second image is the first rotated by 180 degrees, noise where the ties were: the fusion branch on the tie colours
    sc.run()
    even = odd = 0
    for i, (fv, fu, a, b) in enumerate(where):
        o = _obs(sc, 0, i)
        assert o.why == "in" and o.uv == (a + fu, b + fv)
        for ch in range(3):
            for x in RR.exact_tap_products(img, *o.uv)[ch]:
                assert RR.is_tie(x), (i, ch, x)                         # every tap is exactly k + 1/2
                k = int(x - Fraction(1, 2))
                even += k % 2 == 0
                odd += k % 2 == 1
    assert even > 100 and odd > 100
    return sc


# ---- saturated sums -----------------------------------------------------------------------------------------------------
def saturation(seed=2):
    rng = np.random.default_rng(seed)
    rows, cols, cx, cy = 480, 640, 0.5, 0.25
    img = noise(rng, rows, cols)
    pts = []
    j = 0
    for (fv, fu) in ((0.5, 0.5), (0.5, 0.0), (0.0, 0.5), (0.25, 0.75), (0.75, 0.25)):
        for block in ([253] * 4, [254] * 4, [255] * 4, [255, 254, 254, 255], [253, 255, 255, 253], [254, 253, 255, 254]):
            a, b = 40 + 3 * (j % 20), 40 + 3 * (j // 20)
            j += 1
            img[b:b + 2, a:a + 2, :] = np.array(block, np.uint8).reshape(2, 2, 1)
            pts.append(on_pixel(a + fu, b + fv, cx, cy, CYCLIC))
    cam = camera(rows, cols, cx, cy, q=CYCLIC)
    sc = Scene("saturation", _unique(pts), [Render(cam, img, 5.0), Render(cam, img, 5.25)]).run()
    where = set()
    for i in range(len(pts)):
        o = _obs(sc, 0, i)
        assert o.why == "in"
        for t, s in zip(o.sample.taps, o.sample.raw_sums):
            assert s <= 256
            if s == 256:
                # the partial sum that first passes 255: 1, 2 or 3
                acc = 0
                for n, x in enumerate(t):
                    acc += x
                    if acc > 255:
                        where.add(n)
                        break
    assert where == {1, 2, 3}, where
    return sc


# ---- window bounds ------------------------------------------------------------------------------------------------------
def _below(x):
    return float(np.nextafter(x, -np.inf))


def bounds(rows, cols, seed=3):
    """for every margin in FOVS two renderings: A with cx, cy on the lower bounds, B with cx = cy = 0 for the upper ones"""
    rng = np.random.default_rng(seed + cols)
    pts, plan = [], []
    mid_u, mid_v = cols / 2.0 + 0.5, rows / 2.0 + 0.25

    def add(p):
        p = tuple(float(np.float32(a)) for a in p)
        if p not in pts:
            pts.append(p)
        return pts.index(p)

    for fov in FOVS:
        cam_a0 = camera(rows, cols, fov=fov)
        u_lo, u_hi, v_lo, v_hi = RR.window(cam_a0)
        # A: cx = u_lo, cy = v_lo.  x = 0 lands on u_lo exactly, x = -(u_lo - prev(u_lo)) / 64 one ulp below
        du, dv = u_lo - _below(u_lo), v_lo - _below(v_lo)
        y_mid, x_mid = np.float32((mid_v - v_lo) / 64.0), np.float32((mid_u - u_lo) / 64.0)
        a_pts = {"u=lo": add((0.0, y_mid, Z)), "u=lo-ulp": add((-du / 64.0, y_mid, Z)),
                 "v=lo": add((x_mid, 0.0, Z)), "v=lo-ulp": add((x_mid, -dv / 64.0, Z)), "corner": add((0.0, 0.0, Z))}
        # B: cx = cy = 0, u = 64 x.  K is the largest integer below the upper bound
        ku, kv = math.ceil(u_hi) - 1, math.ceil(v_hi) - 1
        b_pts = {"ceil(u)=K": add((ku / 64.0, mid_v / 64.0, Z)), "u=K-1/64": add(((ku - 1 / 64) / 64.0, mid_v / 64.0, Z)),
                 "ceil(u)=K+1": add(((ku + 1 / 64) / 64.0, mid_v / 64.0, Z)),
                 "ceil(v)=K": add((mid_u / 64.0, kv / 64.0, Z)), "v=K-1/64": add((mid_u / 64.0, (kv - 1 / 64) / 64.0, Z)),
                 "ceil(v)=K+1": add((mid_u / 64.0, (kv + 1 / 64) / 64.0, Z))}
        if fov in (0.0, 0.0001):   # the zero-weight taps: u = cols - 1, v = rows - 1 exactly, and both
            assert ku == cols - 1 and kv == rows - 1
            b_pts.update({"u=cols-1": add(((cols - 1) / 64.0, mid_v / 64.0, Z)), "v=rows-1": add((mid_u / 64.0, (rows - 1) / 64.0, Z)),
                          "u,v=last": add(((cols - 1) / 64.0, (rows - 1) / 64.0, Z))})
        plan.append((fov, camera(rows, cols, u_lo, v_lo, fov), a_pts, camera(rows, cols, 0.0, 0.0, fov), b_pts, (u_lo, u_hi, v_lo, v_hi, ku, kv)))
    renders = []
    for k, (fov, cam_a, _, cam_b, _, _) in enumerate(plan):
        renders += [Render(cam_a, noise(rng, rows, cols), 1.0 + k), Render(cam_b, noise(rng, rows, cols), 1.5 + k)]
    sc = Scene(f"bounds-{cols}x{rows}", _unique(pts), renders).run()
    for k, (fov, cam_a, a_pts, cam_b, b_pts, (u_lo, u_hi, v_lo, v_hi, ku, kv)) in enumerate(plan):
        oa = {n: _obs(sc, 2 * k, i) for n, i in a_pts.items()}
        ob = {n: _obs(sc, 2 * k + 1, i) for n, i in b_pts.items()}
        assert oa["u=lo"].why == "in" and oa["u=lo"].uv[0] == u_lo
        assert oa["v=lo"].why == "in" and oa["v=lo"].uv[1] == v_lo
        assert oa["corner"].why == "in" and oa["corner"].uv == (u_lo, v_lo)
        assert oa["u=lo-ulp"].why == "window" and RR.camera_point(cam_a, pts[a_pts["u=lo-ulp"]])[0] * F / Z + u_lo == _below(u_lo)
        assert oa["v=lo-ulp"].why == "window" and RR.camera_point(cam_a, pts[a_pts["v=lo-ulp"]])[1] * F / Z + v_lo == _below(v_lo)
        assert ob["ceil(u)=K"].why == "in" and ob["ceil(u)=K"].uv[0] == ku and ob["u=K-1/64"].why == "in"
        assert ob["ceil(v)=K"].why == "in" and ob["ceil(v)=K"].uv[1] == kv and ob["v=K-1/64"].why == "in"
        # ceil(u) = K + 1 reaches the bound while u itself is still below it: `u < bound` would take the point
        u_out = RR.camera_point(cam_b, pts[b_pts["ceil(u)=K+1"]])[0] * F / Z
        v_out = RR.camera_point(cam_b, pts[b_pts["ceil(v)=K+1"]])[1] * F / Z
        assert ob["ceil(u)=K+1"].why == "window" and math.ceil(u_out) >= u_hi > u_out
        assert ob["ceil(v)=K+1"].why == "window" and math.ceil(v_out) >= v_hi > v_out
        if "u=cols-1" in ob:
            for n in ("u=cols-1", "v=rows-1", "u,v=last"):
                assert ob[n].why == "in"
            w = ob["u,v=last"].sample.weights
            assert ob["u,v=last"].uv == (cols - 1, rows - 1) and w[1:] == (0.0, 0.0, 0.0)
    return sc


# ---- the depth cut --------------------------------------------------------------------------------------------------------
def walk(f, t0, want, steps=4096):
    """the double t nearest t0 (by ulps) with f(t) == want"""
    lo = hi = t0
    for _ in range(steps):
        for t in (lo, hi):
            if f(t) == want:
                return t
        lo, hi = float(np.nextafter(lo, -np.inf)), float(np.nextafter(hi, np.inf))
    raise AssertionError(f"no t within {steps} ulps of {t0} gives {want!r}")


def depth(seed=4):
    rng = np.random.default_rng(seed)
    rows, cols, cx, cy = 480, 640, 320.25, 240.5
    zs = (0.0, 2.0 ** -11, float(np.float32(7.3e-4)))
    pts = [(0.0, 0.0, z) for z in zs] + [(0.0, 2.0 ** -20, zs[1]), (2.0 ** -20, 0.0, zs[2])]
    targets = (_below(0.001), 0.001, float(np.nextafter(0.001, np.inf)))
    renders, plan = [], []
    for i, z in enumerate(zs):
        for want in targets:
            t = walk(lambda t: z + t, 0.001 - z, want)
            cam = camera(rows, cols, cx, cy, t_cw=(0.0, 0.0, t), t_wc=(0.0, 0.0, -t))
            plan.append((i, want))
            renders.append(Render(cam, noise(rng, rows, cols), 3.0 + 0.25 * len(renders)))
    sc = Scene("depth", _unique(pts), renders).run()
    for k, (i, want) in enumerate(plan):
        assert RR.camera_point(sc.renders[k].cam, pts[i])[2] == want
        assert _obs(sc, k, i).why == ("depth" if want < 0.001 else "in"), (k, i, want)
    return sc


# ---- the distance gate ------------------------------------------------------------------------------------------------------
def gate(seed=5):
    rng = np.random.default_rng(seed)
    rows, cols, cx, cy = 480, 640, 320.0, 240.0
    pts = _unique([on_pixel(300.25, 200.5, cx, cy), on_pixel(350.5, 260.75, cx, cy), on_pixel(100.0, 100.0, cx, cy)])
    A, B = 0, 1
    r1 = Render(camera(rows, cols, cx, cy), noise(rng, rows, cols), 10.0)
    sc = Scene("gate", pts, [r1]).run()
    renders = [r1]

    def t_for(i, want):
        p = RR.stored(pts[i])
        t0 = p[2] - math.sqrt(want * want - p[0] * p[0] - p[1] * p[1])
        return walk(lambda t: RR.distance(camera(rows, cols, t_wc=(0.0, 0.0, t)), p), t0, want)

    # rendering 2: A exactly on its gate; rendering 3: B one ulp past its gate (B's obs_dist as rendering 2 left it)
    gA = sc.states[0][A].obs_dist * 1.2
    renders.append(Render(camera(rows, cols, cx, cy, t_wc=(0.0, 0.0, t_for(A, gA))), noise(rng, rows, cols), 10.5))
    sc = Scene("gate", pts, list(renders)).run()
    gB = sc.states[1][B].obs_dist * 1.2
    renders.append(Render(camera(rows, cols, cx, cy, t_wc=(0.0, 0.0, t_for(B, float(np.nextafter(gB, np.inf))))), noise(rng, rows, cols), 11.0))
    renders.append(Render(camera(rows, cols, cx, cy), noise(rng, rows, cols), 11.5))
    sc = Scene("gate", pts, renders).run()
    assert _obs(sc, 1, A).dist == gA and _obs(sc, 1, A).fused == 1
    assert _obs(sc, 2, B).dist == float(np.nextafter(gB, np.inf)) and _obs(sc, 2, B).fused == 0 and _obs(sc, 2, B).why == "in"
    return sc


def dist0(seed=6):
    rng = np.random.default_rng(seed)
    rows, cols, cx, cy = 480, 640, 320.0, 240.0
    pts = _unique([on_pixel(310.5, 230.25, cx, cy, CYCLIC), on_pixel(330.0, 250.0, cx, cy, CYCLIC)])
    P, Q = 0, 1
    cams = [camera(rows, cols, cx, cy, q=CYCLIC, t_wc=RR.stored(pts[P])), camera(rows, cols, cx, cy, q=CYCLIC, t_wc=(0.0, -96.0, 0.0)),
            camera(rows, cols, cx, cy, q=CYCLIC, t_wc=(50.0, 500.0, 50.0))]
    sc = Scene("dist0", pts, [Render(c, noise(rng, rows, cols), 20.0 + k) for k, c in enumerate(cams)]).run()
    assert _obs(sc, 0, P).dist == 0.0 and sc.states[0][P].obs_dist == 0.0
    assert [_obs(sc, k, P).fused for k in (1, 2)] == [1, 1] and sc.states[2][P].n_rgb == 3
    assert _obs(sc, 1, Q).fused == 0 and _obs(sc, 1, Q).why == "in"          # Q keeps its gate
    return sc


def backwards(dt, seed=7):
    """first observation at 1000, then a rendering at 1000 + dt (dt < 0), then forward again"""
    rng = np.random.default_rng(seed)
    rows, cols, cx, cy = 480, 640, 320.0, 240.0
    pts = _unique([on_pixel(300.0 + 7.25 * i, 220.0 + 5.5 * i, cx, cy) for i in range(6)])
    cam = camera(rows, cols, cx, cy)
    times = (1000.0, 1000.0 + dt, 1010.0, 1010.5)
    sc = Scene(f"backwards{int(dt)}", pts, [Render(cam, noise(rng, rows, cols), t) for t in times]).run()
    pre = float(np.float32(15.0 + 0.1 * dt))          # float(cov + 0.1 * dt) with cov = 15
    for i in range(len(pts)):
        assert _obs(sc, 1, i).fused == 1
        if dt == -150:       # float(15) + 0.1 * (-150) == 0: cov 0, n2 * mix = 0 * inf or 0 / 0 = NaN, the colour (short)(int)NaN = 0
            assert pre == 0.0 and sc.states[1][i].cov == [0.0] * 3 and sc.states[1][i].rgb == [0, 0, 0]
        else:
            assert pre < 0.0 and all(c > 0 for c in sc.states[1][i].cov)
    return sc


def chain(seed=8, n_render=40):
    """one scene rendered 40 times with different images and poses (small rotations and translations, increasing times)"""
    from sr_livo_b200 import synth
    rng = np.random.default_rng(seed)
    rows, cols = 480, 752
    pts = np.stack([rng.uniform(-2.0, 2.0, 320), rng.uniform(-1.2, 1.2, 320), rng.uniform(3.5, 4.5, 320)], axis=1)
    pts = _unique(pts.astype(np.float32).astype(np.float64))
    renders, t = [], 30.0
    for k in range(n_render):
        q = synth.quat_from_rotvec(rng.normal(0, 0.01, 3))
        t_cw = rng.normal(0, 0.03, 3)
        t_wc = -synth.quat_to_rot(q).T @ t_cw
        cam = RR.Camera(np.r_[q, t_cw, t_wc, [300.0, 300.0, 376.25, 240.5, 0.005]], rows, cols)
        renders.append(Render(cam, noise(rng, rows, cols), t))
        t += float(rng.choice([0.0, 0.05, 0.1, 0.5]))
    sc = Scene("chain", pts, renders).run()
    assert max(s.n_rgb for s in sc.states[-1]) >= 30
    return sc


# ---- comparing a stored colour state with the restatement -------------------------------------------------------------
PAD = 2
FIELDS = ("rgb", "n_rgb", "cov", "obs_dist", "last_obs")


def padded(img):
    """img inside a buffer PAD rows taller, the extra rows a pattern no tap may weigh"""
    out = np.full((img.shape[0] + PAD, img.shape[1], 3), 0xA5, np.uint8)
    out[: img.shape[0]] = img
    return out


def want_state(sc, k):
    """the restatement's state after rendering k, keyed by the stored float32 position"""
    out = {}
    for p, s in zip(sc.points, sc.states[k]):
        out[np.asarray(p, np.float32).tobytes()] = dict(rgb=np.array(s.rgb, np.int16), n_rgb=np.int16(s.n_rgb),
                                                        cov=np.array(s.cov, np.float32), obs_dist=np.float64(s.obs_dist),
                                                        last_obs=np.float64(s.last_obs))
    return out


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def assert_state(snap, sc, k, who):
    """every stored point of a snapshot (oracle, reference or device download) equals the restatement after rendering k"""
    want = want_state(sc, k)
    seen = set()
    for i, c in enumerate(snap["counts"].tolist()):
        for j in range(c):
            key = np.asarray(snap["xyz"][i, j], np.float32).tobytes()
            w = want[key]
            seen.add(key)
            for f in FIELDS:
                assert bits(snap[f][i, j]) == bits(w[f]), (who, sc.name, k, f, snap["xyz"][i, j], snap[f][i, j], w[f])
    assert seen == set(want), (who, sc.name, "stored points differ")


SCENES = {"ties": ties, "saturation": saturation, "depth": depth, "gate": gate, "dist0": dist0,
          "backwards-150": lambda: backwards(-150.0), "backwards-200": lambda: backwards(-200.0), "chain": chain}
SCENES.update({f"bounds-{c}x{r}": (lambda r=r, c=c: bounds(r, c)) for r, c in SIZES})
PROJECTION_SCENES = ["depth"] + [f"bounds-{c}x{r}" for r, c in SIZES]

_cache = {}


def scene(name) -> Scene:
    if name not in _cache:
        _cache[name] = SCENES[name]()
    return _cache[name]
