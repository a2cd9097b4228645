"""Every entry point the header documents as "host or device, detected per pointer", fed with each buffer as pageable numpy,
pinned torch, CUDA torch and managed (cudaMallocManaged) memory: outputs and map state are byte-identical to the all-pageable
call.  Device and managed memory are used in place, pinned and pageable memory are staged through the ctx scratch."""
import ctypes as C

import numpy as np
import pytest

from color_map_cases import camera, sweep
from sweep_prep_cases import raw_points, track

pytestmark = pytest.mark.gpu

KINDS = ("pageable", "pinned", "device", "managed")
VARIANTS = KINDS[1:] + ("mixed",)   # each against the all-pageable call; "mixed" gives the buffers of one call different kinds

_cudart = None


def cudart():
    """the CUDA runtime torch loaded (for cudaMallocManaged)"""
    global _cudart
    if _cudart is None:
        import torch
        torch.cuda.init()
        path = next(p for p in open("/proc/self/maps").read().split() if "libcudart.so" in p)
        _cudart = C.CDLL(path)
        _cudart.cudaMallocManaged.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, C.c_uint]
        _cudart.cudaFree.argtypes = [C.c_void_p]
    return _cudart


class Buf:
    """a copy of `a` (or zeros) in memory of one kind; .ptr for the C ABI, .get() reads it back"""

    def __init__(self, kind, a):
        import torch
        a = np.ascontiguousarray(a)
        self.kind, self.shape, self.dtype = kind, a.shape, a.dtype
        raw = a.reshape(-1).view(np.uint8)
        self._managed = None
        if kind == "pageable":
            self._np = raw.copy()
            self.ptr = self._np.ctypes.data
        elif kind == "pinned":
            self._t = torch.from_numpy(raw.copy()).pin_memory()
            self._np = self._t.numpy()
            self.ptr = self._t.data_ptr()
        elif kind == "device":
            self._t = torch.from_numpy(raw.copy()).cuda()
            self.ptr = self._t.data_ptr()
        else:
            p = C.c_void_p()
            assert cudart().cudaMallocManaged(C.byref(p), raw.nbytes, 1) == 0   # cudaMemAttachGlobal
            self._managed = p.value
            self._np = np.frombuffer((C.c_char * raw.nbytes).from_address(p.value), np.uint8)
            self._np[:] = raw
            self.ptr = p.value

    def get(self):
        import torch
        torch.cuda.synchronize()
        raw = self._t.cpu().numpy() if self.kind == "device" else self._np.copy()
        return raw.view(self.dtype).reshape(self.shape)

    def free(self):
        if self._managed is not None:
            cudart().cudaFree(self._managed)
            self._managed = None


def kinds_for(variant, names):
    if variant == "mixed":
        return {n: KINDS[(i + 1) % len(KINDS)] for i, n in enumerate(names)}
    return {n: variant for n in names}


class Api:
    def __init__(self):
        from sr_livo_b200 import capi
        self.capi, self.L = capi, capi.lib()
        self.ctx = C.c_void_p()
        assert self.L.srl_ctx_create(0, None, C.byref(self.ctx)) == 0
        self.bufs = []

    def ok(self, rc):
        assert rc == 0, self.L.srl_last_error(self.ctx).decode()

    def buf(self, kind, a):
        b = Buf(kind, a)
        self.bufs.append(b)
        return b

    def close(self):
        for b in self.bufs:
            b.free()
        self.L.srl_ctx_destroy(self.ctx)


@pytest.fixture
def api():
    a = Api()
    yield a
    a.close()


def i64():
    return C.c_int64(0)


def map_bytes(api, m, cap=20):
    nv, npts = i64(), i64()
    api.ok(api.L.srl_map_stats(m, C.byref(nv), C.byref(npts)))
    k = max(nv.value, 1)
    keys, counts, xyz = np.zeros((k, 3), np.int16), np.zeros(k, np.int32), np.zeros((k, cap, 3), np.float32)
    api.ok(api.L.srl_map_download(m, keys.ctypes.data, counts.ctypes.data, xyz.ctypes.data, k, C.byref(nv)))
    return npts.value, keys.tobytes() + counts.tobytes() + xyz.tobytes()


def world_points(seed, n=6000):
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.uniform(-8, 8, (n // 2, 3)), rng.normal(0, 0.6, (n - n // 2, 3))])


# ---- the LIO map ---------------------------------------------------------------------------------------------------------
def run_insert(api, fn, kinds):
    m = C.c_void_p()
    api.ok(api.L.srl_map_create(api.ctx, 1.0, 20, 1 << 14, C.byref(m)))
    out = []
    try:
        for k in range(2):
            xyz = api.buf(kinds["xyz"], world_points(k))
            added = i64()
            api.ok(getattr(api.L, fn)(m, xyz.ptr, xyz.shape[0], 0.1, 0 if k == 0 else 2, C.byref(added)))
            out.append(added.value)
        return out, map_bytes(api, m)
    finally:
        api.L.srl_map_destroy(m)


@pytest.mark.parametrize("fn", ["srl_map_insert", "srl_map_insert_device"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_map_insert(api, fn, variant):
    base = run_insert(api, fn, kinds_for("pageable", ["xyz"]))
    assert base[0][0] > 0
    assert run_insert(api, fn, kinds_for(variant, ["xyz"])) == base


def run_insert_published(api, kinds, sweep_source):
    m, sw = C.c_void_p(), C.c_void_p()
    api.ok(api.L.srl_map_create(api.ctx, 1.0, 20, 1 << 14, C.byref(m)))
    api.ok(api.L.srl_sweep_create(api.ctx, 1 << 13, C.byref(sw)))
    out = []
    q, R_il, t_il = np.array([0.0, 0, 0, 1]), np.eye(3).reshape(-1), np.zeros(3)
    try:
        for k in range(2):
            pts = world_points(10 + k)
            n = pts.shape[0]
            cloud = api.buf(kinds["xyzi_out"], np.full((n, 4), np.nan, np.float32))
            added, published = i64(), i64()
            mnp = 0 if k == 0 else 2
            if sweep_source:
                t = np.array([0.25, -0.5, 0.75])
                raw = np.ascontiguousarray(pts - t)
                api.ok(api.L.srl_sweep_upload(sw, raw.ctypes.data, n))
                api.ok(api.L.srl_map_insert_sweep_published(m, sw, q.ctypes.data, t.ctypes.data, R_il.ctypes.data, t_il.ctypes.data, 0.1, mnp,
                                                            cloud.ptr, n, C.byref(added), C.byref(published)))
            else:
                xyz = api.buf(kinds["xyz"], pts)
                api.ok(api.L.srl_map_insert_published(m, xyz.ptr, n, 0.1, mnp, 0.5, cloud.ptr, n, C.byref(added), C.byref(published)))
            out.append((added.value, published.value, cloud.get()[:published.value].tobytes()))
        return out, map_bytes(api, m)
    finally:
        api.L.srl_sweep_destroy(sw)
        api.L.srl_map_destroy(m)


@pytest.mark.parametrize("sweep_source", [False, True])
@pytest.mark.parametrize("variant", VARIANTS)
def test_map_insert_published(api, sweep_source, variant):
    names = ["xyzi_out"] if sweep_source else ["xyz", "xyzi_out"]
    base = run_insert_published(api, kinds_for("pageable", names), sweep_source)
    assert base[0][1][1] > 0
    assert run_insert_published(api, kinds_for(variant, names), sweep_source) == base


@pytest.mark.parametrize("variant", VARIANTS)
def test_grid_sampling(api, variant):
    pts = world_points(20, 20000)

    def run(kinds):
        xyz = api.buf(kinds["xyz"], pts)
        out, n_out = np.zeros(pts.shape[0], np.uint32), C.c_size_t(0)
        api.ok(api.L.srl_grid_sampling(api.ctx, xyz.ptr, pts.shape[0], 0.5, out.ctypes.data, C.byref(n_out)))
        return out[:n_out.value].tobytes()

    base = run(kinds_for("pageable", ["xyz"]))
    assert len(base) > 0
    assert run(kinds_for(variant, ["xyz"])) == base


# ---- the colour map -------------------------------------------------------------------------------------------------------
CAM = camera((0.0, 0.0, 0.0))


def cam_c(api):
    c = api.capi.Camera()
    c.q_camera_world[:] = CAM[0:4].tolist(); c.t_camera_world[:] = CAM[4:7].tolist(); c.t_world_camera[:] = CAM[7:10].tolist()
    c.fx, c.fy, c.cx, c.cy, c.fov_margin = CAM[10:15].tolist()
    c.cols, c.rows = 640, 480
    return c


def image(seed=3):
    return np.random.default_rng(seed).integers(0, 256, (480, 640, 3), dtype=np.uint8)


def color_state(api, cm):
    st = [i64() for _ in range(5)]
    api.ok(api.L.srl_color_map_stats(cm, *[C.byref(s) for s in st]))
    nv, nrgb, nrec = st[0].value, st[2].value, st[3].value
    cap = 50
    arrs = [np.zeros(nv * cap * 3, np.int16), np.zeros(nv * cap, np.int16), np.zeros(nv * cap * 3, np.float32), np.zeros(nv * cap),
            np.zeros(nv * cap), np.zeros(nv)]
    api.ok(api.L.srl_color_map_download_state(cm, nv, *[a.ctypes.data for a in arrs]))
    lists = [np.zeros(max(nrgb, 1) * 4, np.int16), np.zeros(max(nrec, 1) * 3, np.int16)]
    api.ok(api.L.srl_color_map_download_lists(cm, *[a.ctypes.data for a in lists]))
    vm = api.L.srl_color_map_voxels(cm)
    return [s.value for s in st], b"".join(a.tobytes() for a in arrs + lists), map_bytes(api, vm, cap)


def color_scene(api, xyz_kind="pageable", image_kind="pageable", render=True):
    cm = C.c_void_p()
    api.ok(api.L.srl_color_map_create_growable(api.ctx, 0.1, 50, 1 << 10, 1 << 16, 0.01, C.byref(cm)))
    stored = []
    for k in range(2):
        pts = sweep(30 + k, n_dense=4000)
        xyz = api.buf(xyz_kind, pts)
        n = i64()
        api.ok(api.L.srl_color_map_add_points(cm, xyz.ptr, pts.shape[0], 1 + k, 1.0 + k, float(k), 1, C.byref(n)))
        stored.append(n.value)
    if render:   # a point's first observation only sets its colour; the second one is counted
        for k in range(2):
            img = api.buf(image_kind, image(k))
            rendered = i64()
            api.ok(api.L.srl_color_map_render_recent(cm, C.byref(cam_c(api)), img.ptr, 2.5 + k, C.byref(rendered)))
            stored.append(rendered.value)
    return cm, stored


@pytest.mark.parametrize("variant", VARIANTS)
def test_color_map_add_points_and_render(api, variant):
    def run(kinds):
        cm, counts = color_scene(api, kinds["xyz"], kinds["image"])
        try:
            return counts, color_state(api, cm)
        finally:
            api.L.srl_color_map_destroy(cm)

    base = run(kinds_for("pageable", ["xyz", "image"]))
    assert base[0][0] > 0 and base[0][3] > 0
    assert run(kinds_for(variant, ["xyz", "image"])) == base


@pytest.fixture
def scene(api):
    cm, _ = color_scene(api)
    yield cm
    api.L.srl_color_map_destroy(cm)


@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("variant", VARIANTS)
def test_color_map_export(api, scene, order, variant):
    n = i64()
    api.ok(api.L.srl_color_map_export(scene, 0, order, None, None, 0, C.byref(n)))
    total = n.value
    assert total > 0

    def run(kinds):
        xyz = api.buf(kinds["xyz"], np.zeros((total, 3), np.float32))
        rgb = api.buf(kinds["rgb"], np.zeros((total, 3), np.uint8))
        got = i64()
        api.ok(api.L.srl_color_map_export(scene, 0, order, xyz.ptr, rgb.ptr, total, C.byref(got)))
        return got.value, xyz.get().tobytes(), rgb.get().tobytes()

    base = run(kinds_for("pageable", ["xyz", "rgb"]))
    assert run(kinds_for(variant, ["xyz", "rgb"])) == base


def select(api, cm, kinds, max_points):
    prm = api.capi.ProjectionParams()
    prm.minimum_dis, prm.skip_step, prm.use_all_points, prm.minimum_depth, prm.maximum_depth = 5.0, 1, 0, 0.1, 200.0
    ids = api.buf(kinds["ids"], np.zeros(max_points, np.uint32))
    xyz = api.buf(kinds["xyz"], np.zeros((max_points, 3), np.float32))
    uv = api.buf(kinds["uv"], np.zeros((max_points, 2), np.float32))
    n = i64()
    api.ok(api.L.srl_color_map_select_for_projection(cm, C.byref(cam_c(api)), C.byref(prm), ids.ptr, xyz.ptr, uv.ptr, max_points, C.byref(n)))
    k = n.value
    return k, ids.get()[:k], xyz.get()[:k].tobytes(), uv.get()[:k].tobytes()


@pytest.mark.parametrize("variant", VARIANTS)
def test_select_for_projection(api, scene, variant):
    names = ["ids", "xyz", "uv"]
    base = select(api, scene, kinds_for("pageable", names), 1 << 16)
    assert base[0] > 0
    got = select(api, scene, kinds_for(variant, names), 1 << 16)
    assert got[0] == base[0] and got[1].tobytes() == base[1].tobytes() and got[2:] == base[2:]


@pytest.mark.parametrize("variant", VARIANTS)
def test_gather_points(api, scene, variant):
    ids = select(api, scene, kinds_for("pageable", ["ids", "xyz", "uv"]), 1 << 16)[1]
    n = ids.shape[0]
    names = ["ids", "xyz", "rgb", "n_rgb", "cov", "key_index"]

    def run(kinds):
        d_ids = api.buf(kinds["ids"], ids)
        outs = [api.buf(kinds["xyz"], np.zeros((n, 3), np.float32)), api.buf(kinds["rgb"], np.zeros((n, 3), np.int16)),
                api.buf(kinds["n_rgb"], np.zeros(n, np.int16)), api.buf(kinds["cov"], np.zeros((n, 3), np.float32)),
                api.buf(kinds["key_index"], np.zeros((n, 4), np.int16))]
        api.ok(api.L.srl_color_map_gather_points(scene, d_ids.ptr, n, *[o.ptr for o in outs]))
        return [o.get().tobytes() for o in outs]

    base = run(kinds_for("pageable", names))
    assert run(kinds_for(variant, names)) == base


# ---- the per-sweep point transforms ---------------------------------------------------------------------------------------
def imu_states(api, seed, t0=100.0, span=0.1, n_states=21):
    states = track(np.random.default_rng(seed), np.linspace(t0, t0 + span, n_states))
    arr = (api.capi.ImuState * n_states)()
    for s, d in zip(arr, states):
        s.timestamp = d["timestamp"]
        s.quat[:] = d["quat"].tolist(); s.trans[:] = d["trans"].tolist(); s.vel[:] = d["vel"].tolist()
        s.un_acc[:] = d["un_acc"].tolist(); s.un_gyr[:] = d["un_gyr"].tolist()
    return arr


@pytest.mark.parametrize("fn", ["srl_distort_frame_by_constant", "srl_distort_frame_by_imu"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_distort_frame(api, fn, variant):
    rng = np.random.default_rng(7)
    n = 5000
    raw = raw_points(rng, n)
    rel = np.sort(rng.uniform(0.0, 110.0, n))          # the last ~10 ms lie past the IMU track: the walk stops there
    prior = rng.normal(0, 50, (n, 3))                  # in/out for the IMU walk: points it never reaches keep these
    states = imu_states(api, 8)
    R_il, t_il = np.eye(3).reshape(-1), np.array([0.05, -0.02, 0.1])
    names = ["raw", "rel", "imu"]

    def run(kinds):
        b_raw, b_rel, b_imu = api.buf(kinds["raw"], raw), api.buf(kinds["rel"], rel), api.buf(kinds["imu"], prior)
        args = [api.ctx, b_raw.ptr, b_rel.ptr, n, states, len(states), 100.0, R_il.ctypes.data, t_il.ctypes.data, b_imu.ptr]
        written = i64()
        if fn == "srl_distort_frame_by_imu":
            args.append(C.byref(written))
        api.ok(getattr(api.L, fn)(*args))
        return written.value, b_imu.get().tobytes()

    base = run(kinds_for("pageable", names))
    if fn == "srl_distort_frame_by_imu":
        assert 0 < base[0] < n
    assert run(kinds_for(variant, names)) == base


@pytest.mark.parametrize("variant", VARIANTS)
def test_transform_all_imu_point(api, variant):
    imu = raw_points(np.random.default_rng(9), 5000)
    last = imu_states(api, 10)[-1]
    R_il, t_il = np.eye(3).reshape(-1), np.array([0.05, -0.02, 0.1])
    names = ["imu", "raw_out"]

    def run(kinds):
        b_in, b_out = api.buf(kinds["imu"], imu), api.buf(kinds["raw_out"], np.zeros_like(imu))
        api.ok(api.L.srl_transform_all_imu_point(api.ctx, b_in.ptr, imu.shape[0], C.byref(last), R_il.ctypes.data, t_il.ctypes.data, b_out.ptr))
        return b_out.get().tobytes()

    base = run(kinds_for("pageable", names))
    assert run(kinds_for(variant, names)) == base

