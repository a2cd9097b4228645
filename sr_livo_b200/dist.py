"""Multi-GPU scan matching: one process per GPU, map replicated, keypoints sharded by contiguous index range,
one 32-double all-reduce of the normal equations per ESIKF pass (SURVEY.md §8(e)).

torch.distributed is plumbing only (NCCL over NVLink on GPUs, gloo in the CPU tests).  Every rank runs the same
17x17 host update on the reduced block, so no state broadcast is needed and all ranks stay bit-identical.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import capi
from .capi import IcpParams, IekfIter, NormalEq, SrlError, lib, ptr
from .lio import _check


def shard_range(n: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous keypoint range of `rank`; boundaries fall on multiples of 32 (whole warp groups) so every rank
    keeps keypoint order (needed for deterministic sums and for the residual-cap semantics)."""
    groups = (n + 31) // 32
    b = (groups * rank) // world * 32
    e = (groups * (rank + 1)) // world * 32
    return min(b, n), min(e, n)


def allreduce_block(block, group=None):
    """Sum the 32-double result block over ranks, in place. `block` is a torch tensor (cuda for NCCL, cpu for gloo)."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        if block.is_cuda and dist.get_backend(group) == "gloo":     # gloo reduces host tensors: stage the 256 bytes
            host = block.cpu()
            dist.all_reduce(host, op=dist.ReduceOp.SUM, group=group)
            block.copy_(host)
        else:
            dist.all_reduce(block, op=dist.ReduceOp.SUM, group=group)
    return block


def unpack_block(block64: np.ndarray) -> NormalEq:
    ne = NormalEq()
    b = np.ascontiguousarray(block64, np.float64)
    _check(None, lib().srl_normal_eq_unpack(ptr(b), C.byref(ne)), what="srl_normal_eq_unpack")
    return ne


def iekf_loop(pass_fn, eskf_c, frame_q: np.ndarray, frame_t: np.ndarray, prm: IcpParams, group=None, max_trace: int = 32):
    """The updateIEKF loop (src/optimize.cpp:147-311) with a sharded pass:
    pass_fn(frame_q, frame_t) -> torch tensor of 32 doubles holding THIS rank's partial sums
    (device tensor filled asynchronously is fine).  Returns dict(success, passes, converged, trace)."""
    it = IekfIter()
    _check(None, lib().srl_iekf_begin(C.byref(eskf_c), C.byref(prm), C.byref(it)), what="srl_iekf_begin")
    passes = 0
    trace = []
    success = True
    converged = False
    num_res = 0
    while True:
        block = pass_fn(frame_q, frame_t)
        allreduce_block(block, group)
        host = block.detach().to("cpu").numpy().astype(np.float64, copy=True)   # D2H of 256 B (syncs the stream)
        ne = unpack_block(host)
        passes += 1
        num_res = ne.num_residuals
        if ne.nan_planarity:
            raise RuntimeError("error")                                  # src/optimize.cpp:348-350
        if ne.num_residuals < prm.min_number_neighbors:                  # :110-123, :155
            success = False
            break
        d_x = np.zeros(17)
        done = C.c_int32(0)
        div = C.c_int32(0)
        _check(None, lib().srl_iekf_step(C.byref(it), C.byref(ne), C.byref(prm), C.byref(eskf_c), ptr(frame_q), ptr(frame_t),
                                         ptr(d_x), C.byref(done), C.byref(div)), what="srl_iekf_step")
        if len(trace) < max_trace:
            trace.append(np.concatenate([d_x, frame_t, frame_q]))
        if done.value:
            converged = done.value == 2
            break
    return dict(success=success, passes=passes, converged=converged, num_residuals_used=int(num_res),
                trace=np.array(trace))


class DistributedLio:
    """A LioOptimization per rank + the sharded iterated update.

    native=True (default): the exchange of the 32 sums is fused into the pass's last kernel over NVLink peer memory
    (srl_comm_*, CUDA IPC mailboxes) and the whole loop runs in C (srl_update_iekf_dist); torch.distributed is used
    once, to hand the 64-byte IPC handles around.  native=False: one NCCL all-reduce per pass from Python (baseline)."""

    def __init__(self, lio_opt, rank: int, world: int, group=None, native: bool = True):
        import torch
        self.L = lio_opt
        self.rank, self.world, self.group = rank, world, group
        self.block = torch.zeros(32, dtype=torch.float64, device=f"cuda:{lio_opt.ctx.device}")
        self.comm = None
        if native and world > 1:
            import torch.distributed as tdist
            h = C.c_void_p()
            _check(None, lib().srl_comm_create(lio_opt.ctx.h, rank, world, C.byref(h)), what="srl_comm_create")
            mine = np.zeros(64, np.uint8)
            _check(lio_opt.ctx.h, lib().srl_comm_export(h, ptr(mine)))
            gathered = [None] * world
            tdist.all_gather_object(gathered, mine.tobytes(), group=group)
            allh = np.frombuffer(b"".join(gathered), np.uint8).copy()
            _check(lio_opt.ctx.h, lib().srl_comm_connect(h, ptr(allh)))
            tdist.barrier(group=group)
            self.comm = h
            # every rank must run the same form of the loop (the device-resident and the host-driven form agree to rounding,
            # not bit for bit, and the ranks' states are meant to stay bit-identical): if the device-resident loop is not
            # usable on some rank (kernels serialised by a tool, a GPU shared with other processes), all ranks use the host form
            active = [None] * world
            tdist.all_gather_object(active, int(lio_opt.ctx.counter("device_loop_active")), group=group)
            if min(active) == 0:
                lio_opt.ctx.set_option("device_loop", 0)

    def close(self):
        if self.comm is not None:
            lib().srl_comm_destroy(self.comm)
            self.comm = None

    def set_keypoints(self, raw_xyz):
        """This rank's contiguous range of the sweep's keypoints becomes its local sweep (uploaded, Morton-ordered and
        registered as a whole): H2D and ordering shrink with the number of ranks, and the per-pass exchange of the 32 sums
        makes every rank see the normal equations of the whole sweep."""
        raw = capi.f64(raw_xyz).reshape(-1, 3)
        b, e = shard_range(raw.shape[0], self.rank, self.world)
        self.range = (b, e)
        self.L.setKeypoints(raw[b:e])

    def set_keypoints_device(self, d_ptr: int, n: int):
        """Same from a device array of the whole sweep (n x 3 float64): a device-to-device copy of this rank's range."""
        b, e = shard_range(n, self.rank, self.world)
        self.range = (b, e)
        self.L.sweep.set_device(d_ptr + 24 * b, e - b)

    def optimize(self, raw_xyz, prm: IcpParams, t_last, world_out=None, frame_q=None, frame_t=None):
        """optimize() with HOST buffers on all ranks (srl_optimize_host_dist, all in C): H2D of this rank's range, the
        sharded iterated update, the final re-transform and D2H of this rank's rows into world_out[b:e]."""
        from .lio import EskfEstimator
        if self.comm is None:
            raise SrlError(capi.SRL_BAD_ARG, "DistributedLio.optimize needs the native exchange (native=True, world > 1)")
        raw = capi.f64(raw_xyz).reshape(-1, 3)
        n = raw.shape[0]
        bufs = self.L._call_buffers()
        self.L._marshal(bufs, t_last, frame_q, frame_t)
        b, e = C.c_size_t(0), C.c_size_t(0)
        rc = lib().srl_optimize_host_dist(self.L.ctx.h, self.comm, self.L.voxel_map.h, self.L.sweep.h, ptr(raw), n, bufs["st_ref"],
                                          bufs["p_fq"], bufs["p_ft"], bufs["p_tl"], bufs["p_R"], bufs["p_ti"], C.byref(prm), bufs["summ_ref"],
                                          ptr(world_out) if world_out is not None else None, C.byref(b), C.byref(e))
        self.range = (b.value, e.value)
        self.L.sweep.n = e.value - b.value
        out = self._result(bufs, rc)
        out["range"] = self.range
        return out

    def _pass(self, prm: IcpParams, t_last):
        from .lio import make_frame

        def fn(frame_q, frame_t):
            fr = make_frame(frame_q, frame_t, t_last, self.L.R_imu_lidar, self.L.t_imu_lidar)
            _check(self.L.ctx.h, lib().srl_build_plane_residuals_async(self.L.ctx.h, self.L.voxel_map.h, self.L.sweep.h, C.byref(fr),
                                                                       C.byref(prm), C.c_void_p(self.block.data_ptr())))
            # the pass ran on the ctx stream, the all-reduce and the D2H read run on torch's current stream: order them
            self.L.ctx.synchronize()
            return self.block
        return fn

    def _result(self, b, rc):
        summ, fq, ft = self.L._unmarshal(b, rc)
        return dict(success=summ.success, passes=summ.passes_run, converged=summ.converged, num_residuals_used=summ.num_residuals_used,
                    trace=summ.trace, frame_q=fq, frame_t=ft)

    def updateIEKF(self, prm: IcpParams, t_last, frame_q=None, frame_t=None):
        from .lio import EskfEstimator
        if self.comm is not None:
            b = self.L._call_buffers()
            self.L._marshal(b, t_last, frame_q, frame_t)
            rc = lib().srl_update_iekf_dist(self.L.ctx.h, self.comm, self.L.voxel_map.h, self.L.sweep.h, b["st_ref"], b["p_fq"], b["p_ft"],
                                            b["p_tl"], b["p_R"], b["p_ti"], C.byref(prm), b["summ_ref"])
            return self._result(b, rc)
        st = self.L.eskf_pro.to_c()
        fq = capi.f64(self.L.eskf_pro.q if frame_q is None else frame_q).copy()
        ft = capi.f64(self.L.eskf_pro.p if frame_t is None else frame_t).copy()
        out = iekf_loop(self._pass(prm, capi.f64(t_last)), st, fq, ft, prm, self.group)
        self.L.eskf_pro = EskfEstimator.from_c(st)
        out["frame_q"], out["frame_t"] = fq, ft
        return out
