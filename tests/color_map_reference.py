"""A plain restatement of the colour map's insertion: the colour branch of addPointsToMap with addPointToColorMap and
voxelBlock (src/lioOptimization.cpp:448-551, include/cloudMap.h:147-165), one point at a time.

Stored positions are numpy float32 (rgbPoint keeps position.cast<float>()); everything else is a Python float, one IEEE
double rounding per operation:
  * both keys are static_cast<short>(double(float(x)) / size): (int16)(int32)trunc(q) for |q| < 2^31 (map_reference's
    short_key).  NaN, +-inf and |q| >= 2^31 in either grid drop the point; it still counts toward point_idx % add_point_step;
  * min_num_points is 0, so a point whose voxel is absent creates it; a voxel refuses a point when IsFull();
  * the fine cell is tested (if_exist) before the point is stored; a point enters rgb_points_vec as (voxel key, index in
    block) only when it was stored and its cell was free, and then claims the cell;
  * found and new voxels alike are listed when fabs(t_end - t_last_process) > 1e-5 and fabs(last_visited - t_end) > 1e-5,
    which then sets last_visited = t_end; a new voxel starts at last_visited 0.0;
  * a rendering call clears voxels_recent_visited_temp first and publishes it at the end, with number_of_new_visited_voxel.

`events` counts what each call reached, so that the cases can show that they reach their edges.
"""
from __future__ import annotations

from collections import Counter

import numpy as np

from map_reference import f32, voxel_of

TIME_GATE = 1e-5
NEAR_GATE = (float(np.nextafter(TIME_GATE, 0.0)), TIME_GATE, float(np.nextafter(TIME_GATE, 1.0)))


class Block:
    def __init__(self):
        self.pts: list[tuple] = []
        self.last_visited = 0.0


class ColorMapRef:
    def __init__(self, voxel_size: float = 0.1, cap: int = 50, min_distance_points: float = 0.01):
        self.size, self.cap, self.fine = float(voxel_size), int(cap), float(min_distance_points)
        self.vox: dict[tuple, Block] = {}          # insertion order = creation order
        self.cells: dict[tuple, tuple] = {}        # hashmap_3d_points: fine cell -> voxel of the point that claimed it
        self.rgb: list[tuple] = []                 # rgb_points_vec as (kx, ky, kz, index in block)
        self.recent_temp: list[tuple] = []         # voxels_recent_visited_temp
        self.recent: list[tuple] = []              # map_tracker->voxels_recent_visited
        self.new_recent = 0                        # number_of_new_visited_voxel
        # bookkeeping for `events` only
        self.events: Counter = Counter()
        self.refused_free_cells: set = set()       # cells that were free when a full voxel refused a point in them
        self.first_voxel_of_cell: dict = {}        # cell -> voxel of the first point offered in it
        self.call_stored: dict[tuple, bool] = {}   # this call: voxel -> whether any of its points was stored

    @property
    def num_points(self) -> int:
        return sum(len(b.pts) for b in self.vox.values())

    def add_point(self, xyz, t_end: float, t_last: float) -> bool:
        p = tuple(f32(c) for c in xyz)
        key, cell = voxel_of(p, self.size), voxel_of(p, self.fine)
        if key is None or cell is None:
            self.events["dropped"] += 1
            return False
        free = cell not in self.cells
        blk = self.vox.get(key)
        if blk is None:
            blk = self.vox[key] = Block()
        stored = len(blk.pts) < self.cap
        if stored:
            blk.pts.append(p)
            if free:
                self.rgb.append(key + (len(blk.pts) - 1,))
                if cell in self.refused_free_cells:
                    self.events["cell_claimed_after_refusal"] += 1
                if self.first_voxel_of_cell.setdefault(cell, key) != key:
                    self.events["cell_won_across_voxels"] += 1
                self.cells[cell] = key
            else:
                self.events["stored_in_claimed_cell"] += 1
            if len(blk.pts) == self.cap:
                self.events["index_cap_minus_1"] += 1
        else:
            self.events["refused"] += 1
            if free:
                self.refused_free_cells.add(cell)
            self.first_voxel_of_cell.setdefault(cell, key)
        self.call_stored[key] = self.call_stored.get(key, False) or stored
        if abs(t_end - t_last) in NEAR_GATE or abs(blk.last_visited - t_end) in NEAR_GATE:
            self.events["gate_within_one_double"] += 1
        if abs(t_end - t_last) > TIME_GATE and abs(blk.last_visited - t_end) > TIME_GATE:
            blk.last_visited = t_end
            self.recent_temp.append(key)
            self.events["listed"] += 1
            if not self.call_stored[key]:
                self.events["listed_without_a_stored_point"] += 1
        return stored

    def add_points(self, xyz, add_point_step: int = 1, time_sweep_end: float = 1.0, time_last_process: float = 0.0,
                   to_rendering: bool = True) -> int:
        """addPointsToMap's colour branch: the number of points stored."""
        if to_rendering:
            self.recent_temp = []
        before = len(self.recent_temp)
        self.call_stored = {}
        stored = 0
        for point_idx, row in enumerate(np.asarray(xyz, np.float64).reshape(-1, 3).tolist()):
            if point_idx % add_point_step == 0:
                stored += self.add_point(row, time_sweep_end, time_last_process)
        if to_rendering:
            self.recent = list(self.recent_temp)
            self.new_recent = len(self.recent) - before
        return stored

    # ---- what the device and the oracle report
    def stats(self) -> dict:
        return dict(voxels=len(self.vox), points=self.num_points, rgb_points=len(self.rgb), recent=len(self.recent),
                    new_recent=self.new_recent)

    def lists(self):
        return np.array(self.rgb, np.int16).reshape(-1, 4), np.array(self.recent, np.int32).reshape(-1, 3)

    def voxels(self) -> dict:
        """key -> ((count, 3) float32 positions, last_visited)"""
        return {k: (np.array(b.pts, np.float32).reshape(-1, 3), b.last_visited) for k, b in self.vox.items()}

