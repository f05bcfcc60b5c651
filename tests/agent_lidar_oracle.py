"""Float64 statement of the per-agent lidar (DESIGN.md section 1 "Per-agent lidar"; ``t2d_lidar_scan_agents``): the
reference's ``SingleLineLidar`` bound to each row's slot (``bind_with(j)``, sensor/lidar.py:146-148 skips it), with the
scan itself the pinned ``oracle.lidar.scan``.  This module only chooses the sensor pose and the obstacle rings of a row:

* row (n, q) is observed by slot j = observers[n, q]; j outside [0, M) or ``type_id[n, j] >= n_types`` is an absent row,
  every beam ``inf``;
* the sensor is slot j's (x, y, heading), whatever j's shape;
* the obstacles are the scenario's tile segments and the pose rings of every other active box-shaped slot, slot 0
  included; disc and shapeless slots are no obstacles (:149-153: a Pedestrian's pose is not a ring).

The reference drops obstacles farther than the range before the scan (:117-124); so does this statement, with a wider
margin (a box whose centre lies beyond range + its circumradius + 1e-3): such a box's edges only produce distances above
the range, which the scan maps to ``inf``, so the drop never changes a beam and a row observed by slot 0 is
``oracle.lidar.scan_world``'s row bit for bit.
"""

from __future__ import annotations

import numpy as np

from oracle import geometry as G
from oracle import lidar as OL
from oracle.scenario import OBB


def _seg_rings(segments):
    return [] if segments is None else [np.asarray(s, dtype=np.float64).reshape(2, 2) for s in segments]


def scan_agents(x, y, heading, type_id, table, n_beams, max_range, observers=None, segments=None, tiles=None,
                tile_id=None):
    """x, y, heading: [N, M] (the fp32 device state, as float64); type_id uint8 [N, M]; table: ``as_oracle_table()``;
    observers: int [N, Q] (None: every slot, Q = M); segments: [S, 4] of every scenario, or ``tiles`` (a list of [S_t, 4]
    arrays or None) with ``tile_id`` [N] (None: tile 0).  Returns float64 [N, Q, n_beams]."""
    x, y, h = (np.asarray(a, np.float64) for a in (x, y, heading))
    tid = np.asarray(type_id, np.int64)
    N, M = tid.shape
    obs = np.broadcast_to(np.arange(M), (N, M)) if observers is None else np.asarray(observers, np.int64).reshape(N, -1)
    Q = obs.shape[1]
    shape = np.asarray(table["shape"])
    hl_t, hw_t = np.asarray(table["half_len"], np.float64), np.asarray(table["half_wid"], np.float64)
    n_types = len(shape)
    if tiles is None:
        tile_rings = [_seg_rings(segments)]
    else:
        tile_rings = [_seg_rings(t) for t in tiles]
    tids = np.zeros(N, np.int64) if tile_id is None else np.asarray(tile_id, np.int64).reshape(N)
    out = np.full((N, Q, int(n_beams)), np.inf)
    for n in range(N):
        boxes = {}   # slot -> (closed ring, circumradius)
        for i in range(M):
            t = tid[n, i]
            if t < n_types and shape[t] == OBB:
                c = G.obb_corners(x[n, i], y[n, i], h[n, i], hl_t[t], hw_t[t])
                boxes[i] = (np.concatenate([c, c[:1]], 0), float(np.hypot(hl_t[t], hw_t[t])))
        done = {}
        for q in range(Q):
            j = int(obs[n, q])
            if j < 0 or j >= M or tid[n, j] >= n_types:
                continue
            if j in done:   # a duplicate row: the same computation
                out[n, q] = out[n, done[j]]
                continue
            rings = list(tile_rings[tids[n]])
            for i, (ring, rb) in boxes.items():
                if i != j and np.hypot(x[n, i] - x[n, j], y[n, i] - y[n, j]) <= max_range + rb + 1e-3:
                    rings.append(ring)
            out[n, q] = OL.scan((x[n, j], y[n, j], h[n, j]), rings, n_beams, max_range)
            done[j] = q
    return out


def compare(got, ref, max_range):
    """The GPU criterion of the lidar tests: the same ``inf`` pattern, hit distances within fp32 output rounding."""
    got = np.asarray(got, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert np.array_equal(np.isinf(got), np.isinf(ref))
    hit = np.isfinite(ref)
    if hit.any():
        assert np.abs(got[hit] - ref[hit]).max() < 2e-6 * max_range + 1e-6
    return hit
