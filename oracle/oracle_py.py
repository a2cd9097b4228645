"""ctypes binding of the CPU ORACLE (oracle/srl_oracle.cpp).

TEST INFRASTRUCTURE ONLY — importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package sr_livo_b200 never imports this.

PARITY: pinned against the reference's own compiled code (oracle/reference_py.py, tests/test_reference_pin.py) except for the
arithmetic inside Eigen / OpenCV calls, which stays unpinned — see oracle/srl_oracle.h.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
NS = 17


class IcpParams(C.Structure):
    """orc_icp_params — the icpOptions fields the hot path reads (include/parameters.h:8-56)."""
    _fields_ = [
        ("size_voxel_map", C.c_double),
        ("power_planarity", C.c_double),
        ("max_dist_to_plane_icp", C.c_double),
        ("weight_alpha", C.c_double),
        ("weight_neighborhood", C.c_double),
        ("threshold_orientation_norm", C.c_double),
        ("threshold_translation_norm", C.c_double),
        ("laser_point_cov", C.c_double),
        ("voxel_neighborhood", C.c_int32),
        ("min_number_neighbors", C.c_int32),
        ("max_number_neighbors", C.c_int32),
        ("threshold_voxel_occupancy", C.c_int32),
        ("max_num_residuals", C.c_int32),
        ("num_iters_icp", C.c_int32),
        ("init_num_frames", C.c_int32),
        ("frame_id", C.c_int32),
    ]


def r3live_params(**kw) -> IcpParams:
    """config/r3live.yaml:57-69 + compiled defaults (include/parameters.h) + laser_point_cov
    (src/lioOptimization.cpp:364).  frame_id defaults to 100 (steady state: nb=1, 5 iterations)."""
    p = IcpParams(
        size_voxel_map=1.0, power_planarity=2.0, max_dist_to_plane_icp=0.3, weight_alpha=0.9,
        weight_neighborhood=0.1, threshold_orientation_norm=0.1, threshold_translation_norm=0.01,
        laser_point_cov=0.001, voxel_neighborhood=1, min_number_neighbors=20, max_number_neighbors=20,
        threshold_voxel_occupancy=1, max_num_residuals=600, num_iters_icp=5, init_num_frames=20, frame_id=100)
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, v)
    return p


class EskfState(C.Structure):
    _fields_ = [("p", C.c_double * 3), ("q", C.c_double * 4), ("v", C.c_double * 3), ("ba", C.c_double * 3),
                ("bg", C.c_double * 3), ("g", C.c_double * 3), ("cov", C.c_double * (NS * NS))]


class NormalEq(C.Structure):
    _fields_ = [
        ("HTH", C.c_double * 36), ("HTh", C.c_double * 6), ("loss_sum", C.c_double),
        ("num_residuals", C.c_int64), ("num_full_neighborhoods", C.c_int64), ("sum_candidates", C.c_int64),
        ("sum_probes_hit", C.c_int64), ("num_visited", C.c_int64), ("num_fragile", C.c_int64),
        ("success", C.c_int32), ("nan_planarity", C.c_int32),
    ]


class DebugOut(C.Structure):
    _fields_ = [("world_xyz", C.c_void_p), ("status", C.c_void_p), ("nbr", C.c_void_p), ("nbr_dist", C.c_void_p),
                ("plane", C.c_void_p), ("num_candidates", C.c_void_p)]


def build(verbose: bool = False) -> None:
    """Compile the oracle (and oracle/_ref when /root/reference is present). Building the checker is not using it."""
    r = subprocess.run(["make", "-C", _HERE], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout, r.stderr)
    if r.returncode != 0:
        raise RuntimeError("oracle build failed")


_lib = None
_lib_kind = None


def lib(prefer_tsl: bool = True):
    global _lib, _lib_kind
    if _lib is not None:
        return _lib
    cands = []
    if prefer_tsl:
        cands.append((os.path.join(_HERE, "_ref", "libsrl_oracle_tsl.so"), "tsl"))
    cands.append((os.path.join(_HERE, "_build", "libsrl_oracle.so"), "std"))
    if not any(os.path.exists(p) for p, _ in cands):
        build()
    for path, kind in cands:
        if os.path.exists(path):
            L = C.CDLL(path)
            _lib_kind = kind
            break
    else:
        raise RuntimeError("oracle library missing; run `make -C oracle`")
    L.orc_map_create.restype = C.c_void_p
    L.orc_map_destroy.argtypes = [C.c_void_p]
    L.orc_map_backend.restype = C.c_char_p
    L.orc_map_num_voxels.argtypes = [C.c_void_p]
    L.orc_map_num_voxels.restype = C.c_int64
    L.orc_map_num_points.argtypes = [C.c_void_p]
    L.orc_map_num_points.restype = C.c_int64
    L.orc_map_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_int32, C.c_double, C.c_int32]
    L.orc_map_add_points.restype = C.c_int64
    L.orc_map_remove_far.argtypes = [C.c_void_p, C.c_void_p, C.c_double]
    L.orc_map_remove_far.restype = C.c_int64
    L.orc_map_snapshot.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_map_snapshot.restype = C.c_int64
    L.orc_map_load.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32]
    L.orc_build_plane_residuals.argtypes = [C.c_void_p, C.c_void_p, C.c_int64] + [C.c_void_p] * 5 + [
        C.POINTER(IcpParams), C.c_int32, C.POINTER(NormalEq), C.POINTER(DebugOut)]
    L.orc_build_plane_residuals.restype = C.c_int32
    L.orc_update_iekf.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(EskfState)] + [C.c_void_p] * 5 + [
        C.POINTER(IcpParams), C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_void_p, C.c_int32]
    L.orc_update_iekf.restype = C.c_int32
    L.orc_grid_sampling.argtypes = [C.c_void_p, C.c_int64, C.c_double, C.c_void_p]
    L.orc_grid_sampling.restype = C.c_int64
    L.orc_distort_frame_by_constant.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_distort_frame_by_constant.restype = None
    L.orc_distort_frame_by_imu.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_distort_frame_by_imu.restype = C.c_int64
    L.orc_transform_all_imu_point.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_transform_all_imu_point.restype = None
    L.orc_quat_slerp.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]
    L.orc_quat_slerp.restype = None
    L.orc_quat_to_rot.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_eig3_sym.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_eskf_observe.argtypes = [C.POINTER(EskfState), C.c_void_p]
    L.orc_mat17_inverse.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_mat17_inverse.restype = C.c_int32
    L.orc_voxel_hash.argtypes = [C.c_int16, C.c_int16, C.c_int16]
    L.orc_voxel_hash.restype = C.c_uint64
    _lib = L
    return L


def backend() -> str:
    return lib().orc_map_backend().decode()


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


@dataclass
class PassResult:
    HTH: np.ndarray
    HTh: np.ndarray
    loss_sum: float
    num_residuals: int
    num_full_neighborhoods: int
    sum_candidates: int
    sum_probes_hit: int
    num_visited: int
    num_fragile: int
    success: bool
    nan_planarity: bool
    world_xyz: np.ndarray | None = None
    status: np.ndarray | None = None
    nbr: np.ndarray | None = None
    nbr_dist: np.ndarray | None = None
    plane: np.ndarray | None = None
    num_candidates: np.ndarray | None = None


class OracleMap:
    """voxelHashMap (include/cloudMap.h:171) + addPointsToMap (src/lioOptimization.cpp:520-554)."""

    def __init__(self):
        self._h = lib().orc_map_create()

    def __del__(self):
        try:
            if self._h:
                lib().orc_map_destroy(self._h)
                self._h = None
        except Exception:
            pass

    @property
    def num_voxels(self) -> int:
        return int(lib().orc_map_num_voxels(self._h))

    @property
    def num_points(self) -> int:
        return int(lib().orc_map_num_points(self._h))

    def add_points(self, xyz, voxel_size=1.0, max_num_points_in_voxel=20, min_distance_points=0.15,
                   min_num_points=0) -> int:
        xyz = _f64(xyz).reshape(-1, 3)
        return int(lib().orc_map_add_points(self._h, _ptr(xyz), xyz.shape[0], voxel_size, max_num_points_in_voxel,
                                            min_distance_points, min_num_points))

    def remove_far(self, location, distance: float) -> int:
        """removePointsFarFromLocation (src/lioOptimization.cpp:556-572)."""
        loc = _f64(location).reshape(3)
        return int(lib().orc_map_remove_far(self._h, _ptr(loc), float(distance)))

    def snapshot(self, cap=20):
        n = self.num_voxels
        keys = np.zeros((n, 3), np.int16)
        counts = np.zeros(n, np.int32)
        xyz = np.zeros((n, cap, 3), np.float32)
        got = lib().orc_map_snapshot(self._h, cap, _ptr(keys), _ptr(counts), _ptr(xyz))
        assert got == n
        return keys, counts, xyz

    def load(self, keys, counts, xyz):
        keys = np.ascontiguousarray(keys, np.int16)
        counts = np.ascontiguousarray(counts, np.int32)
        xyz = np.ascontiguousarray(xyz, np.float32)
        cap = xyz.shape[1]
        lib().orc_map_load(self._h, _ptr(keys), _ptr(counts), _ptr(xyz), keys.shape[0], cap)

    # lioOptimization::buildPlaneResiduals + H_x/h assembly + HTH/HTh (src/optimize.cpp:18-131,160-170,235,239)
    def build_plane_residuals(self, raw_xyz, q_cur, t_cur, t_last, params: IcpParams, R_il=None, t_il=None,
                              nthreads=1, debug=False) -> PassResult:
        raw = _f64(raw_xyz).reshape(-1, 3)
        n = raw.shape[0]
        q = _f64(q_cur); t = _f64(t_cur); tl = _f64(t_last)
        R = _f64(np.eye(3) if R_il is None else R_il).reshape(9)
        ti = _f64(np.zeros(3) if t_il is None else t_il)
        ne = NormalEq()
        dbg = None
        arrs = {}
        if debug:
            K = params.max_number_neighbors
            arrs = dict(world_xyz=np.zeros((n, 3)), status=np.zeros(n, np.int32), nbr=np.zeros((n, K, 4), np.int16),
                        nbr_dist=np.zeros((n, K)), plane=np.zeros((n, 16)), num_candidates=np.zeros(n, np.int32))
            dbg = DebugOut(*[_ptr(arrs[k]) for k in ("world_xyz", "status", "nbr", "nbr_dist", "plane",
                                                     "num_candidates")])
        rc = lib().orc_build_plane_residuals(self._h, _ptr(raw), n, _ptr(q), _ptr(t), _ptr(tl), _ptr(R), _ptr(ti),
                                             C.byref(params), nthreads, C.byref(ne),
                                             C.byref(dbg) if dbg is not None else None)
        if rc != 0:
            raise RuntimeError(f"orc_build_plane_residuals rc={rc}")
        return PassResult(
            HTH=np.array(ne.HTH).reshape(6, 6), HTh=np.array(ne.HTh), loss_sum=ne.loss_sum,
            num_residuals=ne.num_residuals, num_full_neighborhoods=ne.num_full_neighborhoods,
            sum_candidates=ne.sum_candidates, sum_probes_hit=ne.sum_probes_hit, num_visited=ne.num_visited,
            num_fragile=ne.num_fragile, success=bool(ne.success), nan_planarity=bool(ne.nan_planarity), **arrs)

    # lioOptimization::updateIEKF (src/optimize.cpp:133-314)
    def update_iekf(self, raw_xyz, eskf: "Eskf", t_last, params: IcpParams, frame_q=None, frame_t=None,
                    R_il=None, t_il=None, nthreads=1, max_trace=32):
        raw = _f64(raw_xyz).reshape(-1, 3)
        fq = _f64(eskf.q if frame_q is None else frame_q).copy()
        ft = _f64(eskf.p if frame_t is None else frame_t).copy()
        tl = _f64(t_last)
        R = _f64(np.eye(3) if R_il is None else R_il).reshape(9)
        ti = _f64(np.zeros(3) if t_il is None else t_il)
        st = eskf.to_c()
        passes = C.c_int32(0)
        used = C.c_int32(0)
        trace = np.zeros((max_trace, 24))
        rc = lib().orc_update_iekf(self._h, _ptr(raw), raw.shape[0], C.byref(st), _ptr(fq), _ptr(ft), _ptr(tl),
                                   _ptr(R), _ptr(ti), C.byref(params), nthreads, C.byref(passes), C.byref(used),
                                   _ptr(trace), max_trace)
        if rc < 0:
            raise RuntimeError(f"orc_update_iekf rc={rc}")
        out = Eskf.from_c(st)
        return dict(success=bool(rc), passes=passes.value, num_residuals_used=used.value, eskf=out, frame_q=fq,
                    frame_t=ft, trace=trace[:min(passes.value, max_trace)].copy())


@dataclass
class Eskf:
    """eskfEstimator state (src/eskfEstimator.cpp:3-21); q is (x,y,z,w)."""
    p: np.ndarray = field(default_factory=lambda: np.zeros(3))
    q: np.ndarray = field(default_factory=lambda: np.array([0.0, 0.0, 0.0, 1.0]))
    v: np.ndarray = field(default_factory=lambda: np.zeros(3))
    ba: np.ndarray = field(default_factory=lambda: np.zeros(3))
    bg: np.ndarray = field(default_factory=lambda: np.zeros(3))
    g: np.ndarray = field(default_factory=lambda: np.array([0.0, 0.0, 9.81]))
    cov: np.ndarray = field(default_factory=lambda: np.eye(NS))

    def to_c(self) -> EskfState:
        s = EskfState()
        for name in ("p", "q", "v", "ba", "bg", "g"):
            a = _f64(getattr(self, name))
            for i in range(a.size):
                getattr(s, name)[i] = a[i]
        c = _f64(self.cov).reshape(-1)
        for i in range(NS * NS):
            s.cov[i] = c[i]
        return s

    @staticmethod
    def from_c(s: EskfState) -> "Eskf":
        return Eskf(p=np.array(s.p), q=np.array(s.q), v=np.array(s.v), ba=np.array(s.ba), bg=np.array(s.bg),
                    g=np.array(s.g), cov=np.array(s.cov).reshape(NS, NS))

    def observe(self, dx) -> "Eskf":
        st = self.to_c()
        d = _f64(dx)
        lib().orc_eskf_observe(C.byref(st), _ptr(d))
        return Eskf.from_c(st)


def grid_sampling(xyz, size_voxel_subsampling: float) -> np.ndarray:
    """gridSampling (src/utility.cpp:188-201): frame indices of the keypoints, reference order."""
    xyz = _f64(xyz).reshape(-1, 3)
    out = np.zeros(xyz.shape[0], np.int32)
    m = lib().orc_grid_sampling(_ptr(xyz), xyz.shape[0], size_voxel_subsampling, _ptr(out))
    return out[:m].copy()


def imu_states_array(states) -> np.ndarray:
    """orc_imu_state[]: rows of 17 doubles (timestamp, quat xyzw, trans, vel, un_acc, un_gyr) from dicts."""
    a = np.zeros((len(states), 17))
    for r, s in zip(a, states):
        r[0] = s["timestamp"]; r[1:5] = s["quat"]; r[5:8] = s["trans"]; r[8:11] = s["vel"]; r[11:14] = s["un_acc"]; r[14:17] = s["un_gyr"]
    return a


def distort_frame_by_constant(raw_xyz, relative_time_ms, states, time_frame_begin, R_il=None, t_il=None) -> np.ndarray:
    """distortFrameByConstant (src/utility.cpp:203-236)."""
    raw = _f64(raw_xyz).reshape(-1, 3); rel = _f64(relative_time_ms).reshape(-1); st = imu_states_array(states)
    R = _f64(np.eye(3) if R_il is None else R_il).reshape(9); t = _f64(np.zeros(3) if t_il is None else t_il)
    out = np.zeros_like(raw)
    lib().orc_distort_frame_by_constant(_ptr(raw), _ptr(rel), raw.shape[0], _ptr(st), st.shape[0], float(time_frame_begin), _ptr(R), _ptr(t), _ptr(out))
    return out


def distort_frame_by_imu(raw_xyz, relative_time_ms, states, time_frame_begin, R_il=None, t_il=None, imu_xyz_in=None):
    """distortFrameByImu (src/utility.cpp:238-312): (imu_xyz, number of leading points the iterator reached)."""
    raw = _f64(raw_xyz).reshape(-1, 3); rel = _f64(relative_time_ms).reshape(-1); st = imu_states_array(states)
    R = _f64(np.eye(3) if R_il is None else R_il).reshape(9); t = _f64(np.zeros(3) if t_il is None else t_il)
    out = np.zeros_like(raw) if imu_xyz_in is None else _f64(imu_xyz_in).reshape(-1, 3).copy()
    m = lib().orc_distort_frame_by_imu(_ptr(raw), _ptr(rel), raw.shape[0], _ptr(st), st.shape[0], float(time_frame_begin), _ptr(R), _ptr(t), _ptr(out))
    return out, int(m)


def transform_all_imu_point(imu_xyz, last_state, R_il=None, t_il=None) -> np.ndarray:
    """transformAllImuPoint (src/utility.cpp:320-332)."""
    imu = _f64(imu_xyz).reshape(-1, 3); st = imu_states_array([last_state])
    R = _f64(np.eye(3) if R_il is None else R_il).reshape(9); t = _f64(np.zeros(3) if t_il is None else t_il)
    out = np.zeros_like(imu)
    lib().orc_transform_all_imu_point(_ptr(imu), imu.shape[0], _ptr(st), _ptr(R), _ptr(t), _ptr(out))
    return out


def quat_slerp(a, t, b) -> np.ndarray:
    a = _f64(a); b = _f64(b); out = np.zeros(4)
    lib().orc_quat_slerp(_ptr(a), float(t), _ptr(b), _ptr(out))
    return out


def quat_to_rot(q) -> np.ndarray:
    q = _f64(q)
    R = np.zeros(9)
    lib().orc_quat_to_rot(_ptr(q), _ptr(R))
    return R.reshape(3, 3)


def eig3_sym(S):
    S = _f64(S).reshape(9)
    ev = np.zeros(3)
    evec = np.zeros(9)
    lib().orc_eig3_sym(_ptr(S), _ptr(ev), _ptr(evec))
    return ev, evec.reshape(3, 3)


def mat17_inverse(A):
    A = _f64(A).reshape(-1)
    out = np.zeros(NS * NS)
    ok = lib().orc_mat17_inverse(_ptr(A), _ptr(out))
    return bool(ok), out.reshape(NS, NS)


def voxel_hash(x, y, z) -> int:
    return int(lib().orc_voxel_hash(int(x), int(y), int(z)))


class OracleColorMap:
    """Row N4 oracle: the colour branch of addPointsToMap + renderPointsInRecentVoxel (see srl_oracle.cpp)."""

    def __init__(self, voxel_size=1.0, max_num_points_in_voxel=20, min_distance_points=0.15):
        L = lib()
        L.orc_color_create.restype = C.c_void_p
        L.orc_color_destroy.argtypes = [C.c_void_p]
        L.orc_color_add_points.restype = C.c_int64
        L.orc_color_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_int32, C.c_double, C.c_int32,
                                           C.c_double, C.c_double, C.c_int32]
        L.orc_color_render.restype = C.c_int64
        L.orc_color_render.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_double]
        for f in ("orc_color_num_voxels", "orc_color_num_rgb_points", "orc_color_num_recent", "orc_color_num_new_recent"):
            getattr(L, f).restype = C.c_int64
            getattr(L, f).argtypes = [C.c_void_p]
        L.orc_color_snapshot.restype = C.c_int64
        L.orc_color_snapshot.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p] * 9
        L.orc_color_lists.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        self._h = C.c_void_p(L.orc_color_create())
        self.voxel_size, self.cap, self.min_dist = voxel_size, max_num_points_in_voxel, min_distance_points

    def __del__(self):
        try:
            if self._h:
                lib().orc_color_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def add_points(self, xyz, add_point_step=1, time_sweep_end=1.0, time_last_process=0.0, to_rendering=True) -> int:
        xyz = _f64(xyz).reshape(-1, 3)
        return int(lib().orc_color_add_points(self._h, _ptr(xyz), xyz.shape[0], self.voxel_size, self.cap, self.min_dist,
                                              add_point_step, time_sweep_end, time_last_process, 1 if to_rendering else 0))

    def render(self, cam15, image_bgr, obs_time, rows=None) -> int:
        """rows: the frame's image_rows when image_bgr holds more rows than the frame (a buffer padded below the image, so the
        zero-weight taps of row `rows` are read from memory the caller owns); default image_bgr.shape[0]."""
        cam = _f64(cam15).reshape(15)
        img = np.ascontiguousarray(image_bgr, np.uint8)
        rows = img.shape[0] if rows is None else int(rows)
        assert rows <= img.shape[0]
        return int(lib().orc_color_render(self._h, _ptr(cam), _ptr(img), rows, img.shape[1], float(obs_time)))

    def counts(self):
        L = lib()
        return dict(voxels=int(L.orc_color_num_voxels(self._h)), rgb_points=int(L.orc_color_num_rgb_points(self._h)),
                    recent=int(L.orc_color_num_recent(self._h)), new_recent=int(L.orc_color_num_new_recent(self._h)))

    def snapshot(self):
        nv, cap = self.counts()["voxels"], self.cap
        out = dict(keys=np.zeros((nv, 3), np.int16), counts=np.zeros(nv, np.int32), xyz=np.zeros((nv, cap, 3), np.float32),
                   rgb=np.zeros((nv, cap, 3), np.int16), n_rgb=np.zeros((nv, cap), np.int16), cov=np.zeros((nv, cap, 3), np.float32),
                   obs_dist=np.zeros((nv, cap)), last_obs=np.zeros((nv, cap)), last_visited=np.zeros(nv))
        got = lib().orc_color_snapshot(self._h, cap, *[_ptr(out[k]) for k in ("keys", "counts", "xyz", "rgb", "n_rgb", "cov", "obs_dist",
                                                                                "last_obs", "last_visited")])
        assert got == nv
        return out

    def lists(self):
        c = self.counts()
        rgb_points = np.zeros((c["rgb_points"], 4), np.int16)
        recent = np.zeros((c["recent"], 3), np.int32)
        lib().orc_color_lists(self._h, _ptr(rgb_points), _ptr(recent))
        return rgb_points, recent
