"""The optical-flow tracker's bookkeeping on the device (srl_flow_tracker_*, row N9) against the plain restatement
(tests/flow_tracker_reference.py), bit for bit: the match list, cur (ids, uv, velocity), last (ids, uv), their order and every
point's is_out_lier_count, after every call.

The restatement's Lucas-Kanade is a second LKOpticalFlowKernel on the same images (row N6 pins it bit for bit), called when
the restatement calls it, so a device that tracks at another time (below 30 points, say) sees other pyramids and other points.
Images come from tests/lk_cases.py; the scene (tests/flow_tracker_cases.py) has points in front of and behind the camera and a
grid whose projections are exact, for the crafted reprojection errors and cells."""
import numpy as np
import pytest

import flow_tracker_cases as FC
import flow_tracker_ref as RF
import flow_tracker_reference as FR
import lk_cases as LC

pytestmark = pytest.mark.gpu


class _Positions(dict):
    """point id -> stored position, gathered from the map for ids first met as candidates"""

    def __init__(self, cm):
        super().__init__()
        self.cm = cm

    def __missing__(self, i):
        p = tuple(self.cm.gatherPoints(np.array([i], np.uint32))["xyz"][0].astype(np.float64))
        self[i] = p
        return p


@pytest.fixture(scope="module")
def env():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from sr_livo_b200 import capi, lio
    ctx = lio.Context(0)
    cm = lio.ColorVoxelMap(ctx, 0.5, 20, 1 << 15, 0.01)
    front, behind, exact = FC.scene_points()
    cm.addPoints(behind[: len(behind) // 2], time_sweep_end=1.0)       # low ids: leading entries behind the camera
    cm.addPoints(np.r_[front, exact, behind[len(behind) // 2:]], time_sweep_end=1.0)
    ids = []
    for c15 in (FC.cam15(fov=-0.4), FC.cam15(fov=-0.4, q_cw=(0.0, 1.0, 0.0, 0.0))):
        got, _, _ = cm.selectPointsForProjection(FC.device_camera(capi, c15), minimum_dis=1.0, use_all_points=True)
        ids.append(got)
    ids = np.unique(np.concatenate(ids))
    xyz = cm.gatherPoints(ids)["xyz"].astype(np.float64)
    pos = _Positions(cm)
    pos.update({int(i): tuple(p) for i, p in zip(ids, xyz)})
    frames = LC.frames(FC.COLS, FC.ROWS, 31, count=len(FC.SEQUENCE) + 2)
    yield dict(torch=torch, lio=lio, capi=capi, ctx=ctx, cm=cm, pos=pos, ids=ids, xyz=xyz, frames=frames)
    cm.close()
    ctx.close()


def _pair(env, max_points=300):
    lio = env["lio"]
    lk = lio.LKOpticalFlowKernel(env["ctx"], **lio.tracker_lk_params())
    twin = lio.LKOpticalFlowKernel(env["ctx"], **lio.tracker_lk_params())
    t = lio.OpticalFlowTracker(env["ctx"], env["cm"], lk, max_points)
    m = FR.FlowTrackerModel(env["pos"], max_points)
    # is_out_lier_count lives with the map's points, so earlier tests on the same map leave theirs
    m.count = {int(i): int(c) for i, c in zip(env["ids"], t.outlierCounts(env["ids"]))}
    return t, m, lk, twin


def _lk(twin, gray):
    def f(pts):
        curr, status, _ = twin.trackImage(gray, np.ascontiguousarray(pts, np.float32).reshape(-1, 2))
        return curr, status
    return f


class _Replay:
    """the twin's Lucas-Kanade results as the restatement got them, handed to the compiled reference for the same input"""

    def __init__(self):
        self.calls = []

    def record(self, lk):
        def f(pts):
            out = lk(pts)
            self.calls.append((np.array(pts, np.float32), out))
            return out
        return f

    def replay(self, pts):
        want, out = self.calls.pop(0)
        assert np.array_equal(np.asarray(pts, np.float32).view(np.uint32), want.view(np.uint32)), "Lucas-Kanade input differs"
        return out


def _ref_check(env, ref, m):
    _same(ref.last_arrays(), m.last_arrays(), "compiled reference: last")
    _same(ref.cur_arrays(), m.cur_arrays(), "compiled reference: cur")
    ids = env["ids"]
    assert np.array_equal(ref.counts(ids), np.array([m.count.get(int(i), 0) for i in ids], np.int16)), "compiled reference: counts"


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64 if a.dtype == np.float64 else a.dtype)


def _same(dev, ref, what):
    assert len(dev) == len(ref), what
    for k, (d, r) in enumerate(zip(dev, ref)):
        assert d.shape == r.shape, (what, k, d.shape, r.shape)
        assert np.array_equal(_bits(d), _bits(r)), (what, k)


def _check(env, t, m):
    _same(t.last(), m.last_arrays(), "last")
    _same(t.current(), m.cur_arrays(), "cur")
    _same(t.matches(), m.match_arrays(), "matches")
    ids = np.array(sorted(set(env["ids"].tolist()) | set(m.count)), np.uint32)
    want = np.array([m.count.get(int(i), 0) for i in ids], np.int16)
    got = t.outlierCounts(ids)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, ("is_out_lier_count", [(int(ids[k]), int(got[k]), int(want[k])) for k in bad[:8]])


def _candidates(env, c15, min_dis=10.0):
    cam = FC.device_camera(env["capi"], FC.cam15(c15[4:7], fov=-0.4))    # refreshPointsForProjection's camera (fov -0.4)
    got, _, _ = env["cm"].selectPointsForProjection(cam, minimum_dis=min_dis)
    return got


def _init_from_selection(env, t, m, twin, gray, time, c15):
    cam = FC.device_camera(env["capi"], c15)
    ids, _, uv = env["cm"].selectPointsForProjection(cam, minimum_dis=40.0)
    t.init(gray, time, ids, uv)
    m.init(time, ids, uv, _lk(twin, gray))
    return ids, uv


def test_sequence_against_the_restatement(env):
    """init, then every image: trackImage, the mask, the PnP inliers, updateAndAppendTrackPoints with the refresh selection, over
    the time steps, masks, inlier lists and camera drifts of FC.SEQUENCE; where oracle/_ref/libsrl_flow_tracker_ref.so was built,
    the reference's own compiled tracker runs the same calls and gives the same sets and counts"""
    t, m, lk, twin = _pair(env)
    rng = np.random.default_rng(5)
    ref, rp = None, _Replay()
    if RF.available():
        ref = RF.FlowTrackerReference(env["cm"].download()["xyz"].reshape(-1, 3), 300)   # row = point id (block * 20 + index)
        ref.set_counts(env["ids"], t.outlierCounts(env["ids"]))
    try:
        frames = env["frames"]
        time = 10.0
        c15 = FC.cam15()
        ids0, _, uv0 = env["cm"].selectPointsForProjection(FC.device_camera(env["capi"], c15), minimum_dis=40.0)
        t.init(frames[0], time, ids0, uv0)
        m.init(time, ids0, uv0, rp.record(_lk(twin, frames[0])))
        if ref:
            ref.init(time, ids0, uv0, rp.replay)
            _ref_check(env, ref, m)
        # the first frame's init followed by trackImage on the same image: dt = 0
        steps = [(0.0, None, "skip", 0.0)] + list(FC.SEQUENCE)
        erased_total = appended_total = 0
        for k, (dt, mk, ik, drift) in enumerate(steps):
            time += dt
            gray = frames[max(k, 0)]
            mask = None
            called = t.trackImage(gray, time)
            assert called == m.track_image(time, rp.record(_lk(twin, gray)), FC.COLS, FC.ROWS)
            _check(env, t, m)
            mask = FC.mask_for(mk, len(m.matches), rng)
            if mk is not None:
                t.rejectMatches(mask)
                m.reject_matches(mask)
                _check(env, t, m)
            if ref:
                ref.track_image(time, rp.replay, FC.COLS, FC.ROWS, None if mask is None else (lambda n, mask=mask: mask))
                _ref_check(env, ref, m)
            inl = FC.inliers_for(ik, len(m.cur), rng)
            if not (isinstance(inl, str) and inl == "skip"):
                assert t.removeOutlierUsingRansacPnp(inl) == m.remove_outliers(inl)
                _check(env, t, m)
                if ref:
                    ref.remove_outliers(inl)
                    _ref_check(env, ref, m)
            c15 = FC.cam15((drift, 0.0, 0.0))
            before = set(m.last)
            cand = _candidates(env, c15)
            t.updateAndAppendTrackPoints(FC.device_camera(env["capi"], c15), cand, 40.0)
            m.update_and_append(FC.model_camera(c15), cand, 40.0)
            _check(env, t, m)
            if ref:
                assert m.leading_unprojected == 0
                ref.update_and_append(c15, FC.COLS, FC.ROWS, cand, 40.0)
                _ref_check(env, ref, m)
            erased_total += len(before - set(m.last))
            appended_total += len(set(m.last) - before)
        assert erased_total > 0 and appended_total > 0
        assert m.lk_calls >= 6
    finally:
        t.close(); lk.close(); twin.close()
        if ref:
            ref.close()


def test_sets_larger_than_one_block_tile(env):
    """about 2000 points in last: the one-block set kernels carry their scans (and loop 1 its projection) across tiles of 1024"""
    t, m, lk, twin = _pair(env, max_points=4000)
    try:
        frames = env["frames"]
        ids = env["ids"]
        cam = FC.model_camera(FC.cam15())
        uv = []
        for i in ids:
            z_ok, _, u, v = FR.project_full(cam, env["pos"][int(i)])
            uv.append((u + 0.25 * (int(i) % 9), v) if z_ok else (60.0, 60.0))
        uv = np.array(uv, np.float32)
        assert len(ids) > 2048
        t.init(frames[0], 1.0, ids, uv)
        m.init(1.0, ids, uv, _lk(twin, frames[0]))
        assert t.trackImage(frames[1], 1.1) and m.track_image(1.1, _lk(twin, frames[1]), FC.COLS, FC.ROWS)
        _check(env, t, m)
        pos = np.searchsorted(np.array(sorted(m.last)), np.array(sorted(m.cur)))
        assert pos.min() < 1024 <= pos.max(), "cur must take entries from both tiles of last"
        mask = (np.arange(len(m.matches)) % 5 != 1).astype(np.uint8)
        t.rejectMatches(mask)
        m.reject_matches(mask)
        _check(env, t, m)
        c15 = FC.cam15((0.004, 0.0, 0.0))
        cand = _candidates(env, c15, min_dis=5.0)
        t.updateAndAppendTrackPoints(FC.device_camera(env["capi"], c15), cand, 10.0)
        m.update_and_append(FC.model_camera(c15), cand, 10.0)
        _check(env, t, m)
        assert len(m.last) > 1024
        assert t.removeOutlierUsingRansacPnp(None) == m.remove_outliers(None)
        _check(env, t, m)
    finally:
        t.close(); lk.close(); twin.close()


@pytest.mark.parametrize("n", [29, 30, 31])
@pytest.mark.parametrize("dt", [0.0, 9.99e-6, 1e-5, -0.25, 0.1])
def test_point_count_and_time_step_edges(env, n, dt):
    """29 points: no Lucas-Kanade, and the next image is tracked against the older pyramid; 30 and 31 track.  dt below 1e-5
    (negative included) gives velocity 1e-3f"""
    t, m, lk, twin = _pair(env)
    try:
        frames = env["frames"]
        ids, uv = _init_from_selection(env, t, m, twin, frames[0], 0.0, FC.cam15())
        assert len(ids) > 40
        sub_ids, sub_uv = ids[:n].copy(), uv[:n].copy()
        t.init(frames[0], 0.0, sub_ids, sub_uv)                      # from time 0, k * dt - (k - 1) * dt is dt exactly
        m.init(0.0, sub_ids, sub_uv, _lk(twin, frames[0]))
        for k in (1, 2):
            called = t.trackImage(frames[k], k * dt)
            assert called == m.track_image(k * dt, _lk(twin, frames[k]), FC.COLS, FC.ROWS) == (n >= 30)
            _check(env, t, m)
            if n >= 30 and dt < 1e-5:
                assert np.all(t.current()[2] == np.float64(np.float32(1e-3)))
        assert t.lastImageTime() == 2 * dt
        if n < 30:
            # 29 points never consumed frames 1 and 2: grown past 30 by updateAndAppendTrackPoints (no Lucas-Kanade call), the
            # tracker tracks frame 3 against frame 0's pyramid
            c15 = FC.cam15()
            cand = _candidates(env, c15)
            t.updateAndAppendTrackPoints(FC.device_camera(env["capi"], c15), cand, 40.0)
            m.update_and_append(FC.model_camera(c15), cand, 40.0)
            assert len(m.last) >= 30
            assert t.trackImage(frames[3], 5.1) and m.track_image(5.1, _lk(twin, frames[3]), FC.COLS, FC.ROWS)
            _check(env, t, m)
    finally:
        t.close(); lk.close(); twin.close()


def _exact_ids(env):
    """ids of the exact grid (z = 2) and their projections under the unmoved camera"""
    xyz = env["xyz"]
    sel = np.flatnonzero(xyz[:, 2] == 2.0)
    cam = FC.model_camera(FC.cam15())
    out = []
    for k in sel:
        z_ok, res, u, v = FR.project_full(cam, xyz[k])
        if res:
            out.append((int(env["ids"][k]), u, v))
    return out


def test_crafted_append_edges(env):
    """errors exactly at thr and 2 thr and one float above, with count 0 and count 1 (a second update); leading and interior
    entries behind the camera; an erased point that is also a candidate; cells shared between tracked points and candidates"""
    t, m, lk, twin = _pair(env, max_points=400)
    try:
        thr = 2.0 * FC.COLS / 320.0
        assert thr == 4.0
        ex = _exact_ids(env)
        assert len(ex) >= 40
        offsets = [0.0, thr, float(np.nextafter(np.float32(thr), np.float32(10))), 2 * thr,
                   float(np.nextafter(np.float32(2 * thr), np.float32(10))), 0.5 * thr, 1.5 * thr]
        ids, uv = [], []
        for k, (i, u, v) in enumerate(ex):
            ids.append(i)
            uv.append((u + offsets[k % len(offsets)], v))
        xyz = env["xyz"]
        behind = [int(env["ids"][k]) for k in np.flatnonzero(xyz[:, 2] < 0)]
        front_min = min(ids)
        lead = [i for i in behind if i < front_min]
        inner = [i for i in behind if i > front_min]
        assert lead and inner, "the scene must put points behind the camera before and among the tracked ids"
        ids += lead[:3] + inner[:3]
        uv += [(100.0, 100.0)] * 6
        ids, uv = np.array(ids, np.uint32), np.array(uv, np.float32)
        t.init(env["frames"][0], 1.0, ids, uv)
        m.init(1.0, ids, uv, _lk(twin, env["frames"][0]))
        c15 = FC.cam15()
        # candidates: the exact grid itself (members, skipped), the erased ones come straight back, then the refresh selection
        cand = np.r_[np.array([i for i, _, _ in ex], np.uint32)[::-1], _candidates(env, c15)]
        for _ in range(3):                                         # count 1 entries reach count 2 on the second update
            t.updateAndAppendTrackPoints(FC.device_camera(env["capi"], c15), cand, 40.0)
            m.update_and_append(FC.model_camera(c15), cand, 40.0)
            _check(env, t, m)
        # half-way cells: mini_distance 100 puts u = 3.125 + 320 + 50 j on and next to odd multiples of 50
        t.updateAndAppendTrackPoints(FC.device_camera(env["capi"], c15), cand, 100.0)
        m.update_and_append(FC.model_camera(c15), cand, 100.0)
        _check(env, t, m)
    finally:
        t.close(); lk.close(); twin.close()


@pytest.mark.parametrize("size0", ["max-1", "max", "max+1"])
def test_set_size_edges(env, size0):
    """loop 1 leaves max - 1, max or max + 1 points: the size check after each non-member candidate lets max - size0
    candidates in, or only the first non-member when size0 >= max"""
    ex = _exact_ids(env)
    n0 = 60
    max_points = {"max-1": n0 + 1, "max": n0, "max+1": n0 - 1}[size0]
    t, m, lk, twin = _pair(env, max_points=max_points)
    try:
        ids = np.array([i for i, _, _ in ex[:n0]], np.uint32)
        uv = np.array([(u, v) for _, u, v in ex[:n0]], np.float32)
        c15 = FC.cam15()
        cand = _candidates(env, c15)
        # a candidate that wins its cell against the tracked points: put first among the non-members, it must enter even when
        # the set is already full
        probe = FR.FlowTrackerModel(env["pos"], 1 << 30)
        probe.last = {int(i): (np.float32(a), np.float32(b)) for i, (a, b) in zip(ids, uv)}
        probe.update_and_append(FC.model_camera(c15), cand, 40.0)
        winner = next(int(i) for i in cand if int(i) in probe.last and int(i) not in set(ids.tolist()))
        for first_member in (False, True):                          # a member as the first candidate is skipped before the check
            t.init(env["frames"][0], 1.0, ids, uv)
            m.init(1.0, ids, uv, _lk(twin, env["frames"][0]))
            c = np.r_[ids[:1] if first_member else ids[:0], np.uint32(winner), cand].astype(np.uint32)
            t.updateAndAppendTrackPoints(FC.device_camera(env["capi"], c15), c, 40.0)
            m.update_and_append(FC.model_camera(c15), c, 40.0)
            _check(env, t, m)
            assert winner in m.last and len(m.last) == max(max_points, n0 + 1)
    finally:
        t.close(); lk.close(); twin.close()


def test_host_and_device_inputs_give_the_same_bytes(env):
    torch = env["torch"]
    out = []
    for on_device in (False, True):
        t, m, lk, twin = _pair(env)
        try:
            frames = env["frames"]
            cam = FC.device_camera(env["capi"], FC.cam15())
            ids, _, uv = env["cm"].selectPointsForProjection(cam, minimum_dis=40.0)
            dv = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if on_device else (lambda a: a)
            t.init(dv(frames[0]), 1.0, dv(ids.view(np.int32)) if on_device else ids, dv(uv))
            t.trackImage(dv(frames[1]), 1.1)
            n = t.counts()["match"]
            t.rejectMatches(dv((np.arange(n) % 3 != 0).astype(np.uint8)))
            k = t.counts()["cur"]
            t.removeOutlierUsingRansacPnp(dv(np.arange(k, dtype=np.int32)[::-1].copy()))
            cand = _candidates(env, FC.cam15((0.01, 0, 0)))
            t.updateAndAppendTrackPoints(FC.device_camera(env["capi"], FC.cam15((0.01, 0, 0))), dv(cand.view(np.int32)) if on_device else cand,
                                         40.0)
            out.append((t.matches(), t.current(), t.last()))
        finally:
            t.close(); lk.close(); twin.close()
    for a, b in zip(out[0], out[1]):
        _same(a, b, "host vs device")


def test_bad_arguments_change_nothing(env):
    lio = env["lio"]
    t, m, lk, twin = _pair(env)
    try:
        frames = env["frames"]
        ids, uv = _init_from_selection(env, t, m, twin, frames[0], 1.0, FC.cam15())
        t.trackImage(frames[1], 1.1)
        before = (t.matches(), t.current(), t.last())
        counts = t.outlierCounts(env["ids"])
        bad = ids.copy()
        bad[3] = 0xfffffff0
        for call in (lambda: t.init(frames[0], 2.0, bad, uv),
                     lambda: t.rejectMatches(np.ones(t.counts()["match"] + 1, np.uint8)),
                     lambda: t.removeOutlierUsingRansacPnp(np.array([0, t.counts()["cur"]], np.int32)),
                     lambda: t.removeOutlierUsingRansacPnp(np.array([-1], np.int32)),
                     lambda: t.updateAndAppendTrackPoints(FC.device_camera(env["capi"], FC.cam15()), bad, 40.0),
                     lambda: t.updateAndAppendTrackPoints(FC.device_camera(env["capi"], FC.cam15()), ids, 0.0),
                     lambda: t.init(np.ascontiguousarray(frames[0][:-8]), 2.0, ids, uv)):     # an image of another size

            with pytest.raises(lio.SrlError) as e:
                call()
            assert e.value.code == 4
            after = (t.matches(), t.current(), t.last())
            for a, b in zip(before, after):
                _same(a, b, "unchanged")
        assert np.array_equal(t.outlierCounts(env["ids"]), counts) and t.lastImageTime() == 1.1
    finally:
        t.close(); lk.close(); twin.close()


def test_chained_frames_on_the_device(env):
    """ten images of process -> trackImage -> rejectMatches -> removeOutlierUsingRansacPnp -> vioEsikf / vioPhotometric on
    current(device=True) -> render -> refresh selection -> updateAndAppendTrackPoints, every list on the device and only counts
    read back; the same calls on host copies of every input, on a second map and tracker, give the same bits"""
    import vio_cases as VC
    torch, lio, capi = env["torch"], env["lio"], env["capi"]
    cam = VC.CAMERAS["ntu"]
    c = VC.make_case(611, "ntu", n=1500, zmin=3.0, zmax=12.0)
    raw = VC.textured_image(cam["image_height"], cam["image_width"], 612)
    results = []
    for on_device in (True, False):
        ip = lio.ImageProcessing(env["ctx"], **cam)
        cols, rows = ip.output_size()
        cm = lio.ColorVoxelMap(env["ctx"], 1.0, 20, 1 << 15, 0.05)
        lk = lio.LKOpticalFlowKernel(env["ctx"], **lio.tracker_lk_params())
        t = lio.OpticalFlowTracker(env["ctx"], cm, lk)
        try:
            dv = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if on_device else (lambda a: np.ascontiguousarray(a))
            host = (lambda a: a.cpu().numpy()) if on_device else (lambda a: a)

            def select(camera, min_dis):
                """the selection's ids and uv, into device tensors on the device run"""
                if not on_device:
                    ids, _, uv = cm.selectPointsForProjection(camera, minimum_dis=min_dis)
                    return ids, uv
                k = cm.countPointsForProjection(camera, minimum_dis=min_dis)
                ids = torch.empty(k, dtype=torch.int32, device="cuda")
                uv = torch.empty((k, 2), dtype=torch.float32, device="cuda")
                cm.selectPointsForProjection(camera, minimum_dis=min_dis, out=(ids, None, uv))
                return ids, uv

            st = lio.CameraState(c["state"][0:4], c["state"][4:7], c["state"][7:16].reshape(3, 3), c["state"][16:19], *c["state"][19:24])
            ip.setCovariance(VC.initial_covariance())
            cm.addPoints(dv(c["xyz"].astype(np.float64)), time_sweep_end=1.0)
            trace = []
            for k in range(10):
                img = np.roll(raw, shift=(k % 3, 2 * k), axis=(0, 1))
                rgb, gray = ip.process(dv(img), out=(dv(np.empty((rows, cols, 3), np.uint8)), dv(np.empty((rows, cols), np.uint8))))
                camera = st.camera(cols, rows, 0.005)
                time = 1.0 + 0.1 * k
                if k == 0:
                    cm.renderPointsInRecentVoxel(camera, rgb, time)
                    ids, uv = select(camera, 40.0 / ip.scale_factor())
                    t.init(gray, time, ids, uv)
                    continue
                t.trackImage(gray, time)
                n = t.counts()["match"]
                t.rejectMatches(dv((np.arange(n) % 7 != 3).astype(np.uint8)))
                ncur = t.counts()["cur"]
                t.removeOutlierUsingRansacPnp(dv(np.arange(0, ncur, 1 + (k % 2), dtype=np.int32)))
                cids, cuv, cvel = t.current(device=on_device)
                ip.vioEsikf(cm, st, cids, cuv, cvel, 40)
                ip.vioPhotometric(cm, st, cids, cvel, 40, rgb)
                camera = st.camera(cols, rows, 0.005)
                cm.renderPointsInRecentVoxel(camera, rgb, time)
                cand, _ = select(st.camera(cols, rows, -0.4), 10.0)
                t.updateAndAppendTrackPoints(camera, cand, 40.0 / ip.scale_factor())
                trace.append((VC.state_array(st), tuple(host(a) for a in t.last(device=on_device)), t.counts()))
            results.append(trace)
        finally:
            t.close(); lk.close(); cm.close(); ip.close()
    for (s0, l0, n0), (s1, l1, n1) in zip(*results):
        assert np.array_equal(s0, s1) and n0 == n1
        _same(l0, l1, "chained")
    assert any(n["cur"] >= 10 for _, _, n in results[0])
