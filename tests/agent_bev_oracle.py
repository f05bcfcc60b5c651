"""Float64 statement of the per-agent BEV (DESIGN.md section 1 "Per-agent BEV"; ``t2d_bev_render_agents``): the
reference's ``BEVCamera`` bound to each row's slot (sensor_base.py:89-95), drawing every participant, its own body
included (camera.py:247-331).  The drawing is ``tests/bev_oracle.py``'s; this module only chooses a row's view and goal:

* row (n, q) is observed by slot j = observers[n, q]; j outside [0, M) or ``type_id[n, j] >= n_types`` (the number of
  type styles) is an absent row, all background (class 0), without the ego image's no-ego view;
* the view is slot j's fp32 (x, y, heading), whatever j's shape;
* the goal rectangle: ``goals[n, q]`` when per-row goals are given (NaN cx: none), else the scenario's target for the
  rows observed by slot 0 and none for the others.

A row observed by slot 0 without goals is therefore ``bev_oracle.render_world_scenario``'s image whenever slot 0 is
present.
"""

from __future__ import annotations

import numpy as np

from tests import bev_oracle as B


def row_goal(n, q, j, target=None, goals=None):
    """The goal rectangle row (n, q), observed by slot j, draws, or None."""
    if goals is not None:
        g = np.asarray(goals[n, q])
        return None if np.isnan(g[0]) else g
    if j == 0 and target is not None:
        return np.asarray(target[n])
    return None


def render_row(n, j, state, type_id, table, type_style, z, lw, width, height, rng, tile=None, seg_style=None, goal=None,
               target_style=B.NOT_DRAWN):
    """Class image uint8 [H, W] of scenario n seen from slot j (any int); state = dict of [N, M] arrays x, y, heading;
    tile = dict(segments, poly_start); ``goal``: the row's goal rectangle (``row_goal``) or None."""
    tile = tile or {}
    M = type_id.shape[1]
    if j < 0 or j >= M or int(type_id[n, j]) >= len(type_style):
        return np.zeros((height, width), np.uint8)
    view = B.view_of(state["x"][n, j], state["y"][n, j], state["heading"][n, j], True)
    win = B.window(width, height, rng)
    prims = B.primitives(state["x"][n], state["y"][n], state["heading"][n], type_id[n], table, type_style, z, lw, win[2],
                         tile.get("segments"), tile.get("poly_start"), seg_style, goal, target_style)
    return B.render(prims, view, width, height, rng)


def render_agents(state, type_id, table, type_style, z, lw, width, height, rng, observers=None, rows=None, tiles=None,
                  seg_styles=None, target=None, goals=None, target_style=B.NOT_DRAWN):
    """{(n, q): class image} for the rows ``rows`` (default: all) of the observer list ``observers`` int [N, Q] (None:
    row q is slot q, Q = M).  ``tiles`` / ``seg_styles``: per scenario (lists of length N) or None."""
    N, M = type_id.shape
    obs = np.broadcast_to(np.arange(M), (N, M)) if observers is None else np.asarray(observers, np.int64)
    if rows is None:
        rows = [(n, q) for n in range(N) for q in range(obs.shape[1])]
    out = {}
    for n, q in rows:
        j = int(obs[n, q])
        out[(n, q)] = render_row(n, j, state, type_id, table, type_style, z, lw, width, height, rng,
                                 None if tiles is None else tiles[n], None if seg_styles is None else seg_styles[n],
                                 row_goal(n, q, j, target, goals), target_style)
    return out
