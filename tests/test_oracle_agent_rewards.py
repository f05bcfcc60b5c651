"""The float64 per-agent status / reward oracle (tests/agent_reward_oracle.py) against the ego's oracle it generalises
(oracle.scenario), on hand-built priority cases, absent / duplicate / out-of-range rows, retirement and the done rule over
several steps, and the restore on reset.  No GPU needed."""

import numpy as np

from oracle import scenario as O
from tests import agent_reward_oracle as R

# a box (medium car) and a disc (pedestrian) row, as the device sees them
TABLE = dict({k: np.asarray([4.0, 0.3], np.float64) for k in O.TABLE_FLOAT_FIELDS},
             half_len=np.asarray([2.4, 0.3]), half_wid=np.asarray([0.95, 0.3]), radius=np.asarray([0.0, 0.3]),
             model=np.asarray([O.KINEMATICS, O.POINTMASS_NEWTON]), shape=np.asarray([O.OBB, O.CIRCLE]))
N_TYPES = 2


def _scene(seed, n=40, m=6, empty=0.15):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-20, 20, (n, m)).astype(np.float32)
    y = rng.uniform(-20, 20, (n, m)).astype(np.float32)
    h = rng.uniform(-3, 3, (n, m)).astype(np.float32)
    types = rng.integers(0, 2, (n, m)).astype(np.uint8)
    types[rng.random((n, m)) < empty] = 255
    flags = np.where(rng.random((n, m)) < 0.1, rng.integers(1, 8, (n, m)), 0).astype(np.uint8)
    steps = rng.integers(1, 30, n)
    return x, y, h, types, flags, steps


def _near_goals(x, y, h, slot, rng, nan_frac=0.3):
    """Goals next to each row's slot, some exactly on it (IoU 1), some NaN."""
    g = np.stack([np.take_along_axis(x, slot, 1) + rng.normal(0, 0.6, slot.shape),
                  np.take_along_axis(y, slot, 1) + rng.normal(0, 0.6, slot.shape),
                  np.take_along_axis(h, slot, 1) + rng.normal(0, 0.1, slot.shape),
                  np.full(slot.shape, 2.4), np.full(slot.shape, 0.95)], -1).astype(np.float32)
    exact = rng.random(slot.shape) < 0.2
    g[exact, 0] = np.take_along_axis(x, slot, 1)[exact]
    g[exact, 1] = np.take_along_axis(y, slot, 1)[exact]
    g[exact, 2] = np.take_along_axis(h, slot, 1)[exact]
    g[rng.random(slot.shape) < nan_frac, 0] = np.nan
    return g


def test_one_row_on_slot_zero_is_the_ego_chain():
    rng = np.random.default_rng(1)
    x, y, h, types, flags, steps = _scene(1)
    n = x.shape[0]
    types[:, 0] = 0   # a box ego
    target = _near_goals(x, y, h, np.zeros((n, 1), np.int64), rng, nan_frac=0.0)[:, 0]
    lp, cnt = np.zeros((n, 4)), np.zeros(n, np.int64)
    lp_r, cnt_r = np.zeros((n, 1, 4)), np.zeros((n, 1), np.int64)
    mi, md = np.full(n, -np.inf), np.full(n, np.inf)
    mi_r, md_r = np.full((n, 1), -np.inf), np.full((n, 1), np.inf)
    for t in range(6):
        steps_t = steps + t
        arrived, noact, iou, lp, cnt = O.goal_events(x, y, h, types, TABLE, target, lp, cnt, 0.95, 2)
        st, done = O.status_with_goal(flags, types, steps_t, arrived, noact, max_step=20)
        e = O.env_epilogue(flags, st, steps_t, 20, iou=iou, ego_xy=np.stack([x[:, 0], y[:, 0]], 1).astype(np.float64),
                           target=target.astype(np.float64), max_iou=mi, min_dist=md)
        mi, md = e["max_iou"], e["min_dist"]
        a = R.agents_epilogue(flags, types, x, y, h, steps_t, TABLE, N_TYPES, observers=np.zeros((n, 1), np.int16),
                              goals=target[:, None], last_pose=lp_r, noact_count=cnt_r, max_iou=mi_r, min_dist=md_r,
                              max_step=20, no_action_max=2)
        lp_r, cnt_r, mi_r, md_r = a["last_pose"], a["noact_count"], a["max_iou"], a["min_dist"]
        assert np.array_equal(a["status"][:, 0], st) and np.array_equal(a["iou"][:, 0], iou)
        assert np.array_equal(a["reward"][:, 0], e["reward"]) and np.array_equal(a["done"], e["done"])
        assert np.array_equal(a["terminated"][:, 0], e["terminated"]) and np.array_equal(a["truncated"][:, 0], e["truncated"])
        assert np.array_equal(mi_r[:, 0], mi) and np.array_equal(md_r[:, 0], md)
        assert np.array_equal(a["traffic"], e["traffic_status"])
        x = x + np.float32(0.3) * (np.arange(n) % 3 != 0)[:, None]   # a third of the scenarios stand still (NoAction)
    assert set(np.unique(a["status"])) >= {O.NORMAL}


def test_priority_chain_row_by_row():
    # one scenario, one row per slot; every slot a box sitting exactly on its goal (IoU 1 -> arrival)
    m = 5
    x = np.arange(m, dtype=np.float32)[None] * 10
    y = np.zeros((1, m), np.float32)
    h = np.zeros((1, m), np.float32)
    types = np.zeros((1, m), np.uint8)
    goals = np.stack([x, y, h, np.full((1, m), 2.4), np.full((1, m), 0.95)], -1).astype(np.float32)
    flags = np.asarray([[0, O.F_DYNAMIC, O.F_STATIC | O.F_DYNAMIC, O.F_OUTBOUND | O.F_STATIC, 0]], np.uint8)
    a = R.agents_epilogue(flags, types, x, y, h, [1], TABLE, N_TYPES, goals=goals, max_step=5)
    C, F, OB = O.COMPLETED, O.FAILED, O.OUT_BOUND
    assert list(a["status"][0]) == [C, F, F, OB, C]
    assert list(a["reward"][0]) == [5.0, -5.0, -5.0, -5.0, 5.0]
    assert list(a["terminated"][0]) == [True, False, False, False, True]
    assert list(a["truncated"][0]) == [False, True, True, True, False]
    assert a["done"][0] == 1 and (a["type_id"] == 255).all() and np.array_equal(a["retired"], types)
    # the time limit beats everything
    a = R.agents_epilogue(flags, types, x, y, h, [6], TABLE, N_TYPES, goals=goals, max_step=5)
    assert (a["status"] == O.TIME_EXCEEDED).all() and (a["reward"] == -1.0).all()
    # no action beats out of bound and collision, but not the time limit
    a0 = R.agents_epilogue(flags, types, x, y, h, [1], TABLE, N_TYPES, goals=goals, max_step=5, no_action_max=1)
    assert a0["last_pose"][..., 3].all() and (a0["noact_count"] == 0).all()
    a = R.agents_epilogue(flags, types, x, y, h, [2], TABLE, N_TYPES, goals=goals, max_step=5, no_action_max=1,
                          last_pose=a0["last_pose"], noact_count=a0["noact_count"] + 1)   # 2 > 1 still ticks
    assert (a["status"] == O.NO_ACTION).all() and (a["reward"] == -1.0).all() and (a["truncated"]).all()
    # far from the goal and no flags: NORMAL, the time penalty + IoU gain (0) + nothing on the first distance
    far = goals.copy()
    far[..., 0] += 100
    a = R.agents_epilogue(np.zeros_like(flags), types, x, y, h, [3], TABLE, N_TYPES, goals=far, max_step=5)
    assert (a["status"] == O.NORMAL).all() and a["done"][0] == 0 and (a["type_id"] == 0).all()
    assert np.allclose(a["reward"], -np.tanh(3 / 5) * 0.001) and np.allclose(a["min_dist"], 100)
    # a row without a goal gets only the time penalty and keeps its extrema
    a = R.agents_epilogue(np.zeros_like(flags), types, x, y, h, [3], TABLE, N_TYPES, max_step=5)
    assert np.allclose(a["reward"], -np.tanh(3 / 5) * 0.001) and (a["iou"] == 0).all()
    assert np.isinf(a["min_dist"]).all() and np.isneginf(a["max_iou"]).all()


def test_absent_duplicate_and_out_of_range_rows():
    x, y, h, types, flags, steps = _scene(3, n=4, m=4, empty=0.0)
    types[0, 2] = 255
    flags[:] = 0
    flags[0, 1] = O.F_DYNAMIC
    obs = np.asarray([[-1, 4, 2, 1, 1, 0]] * 4, np.int16)   # out of range, out of range, empty (row 0), dup, dup, slot 0
    a = R.agents_epilogue(flags, types, x, y, h, steps, TABLE, N_TYPES, observers=obs, max_step=100)
    assert (a["status"][:, :2] == 0).all() and a["status"][0, 2] == 0 and a["status"][1, 2] == O.NORMAL
    assert (a["reward"][:, :2] == 0).all() and not a["terminated"][:, :2].any() and not a["truncated"][:, :2].any()
    assert np.array_equal(a["status"][:, 3], a["status"][:, 4]) and np.array_equal(a["reward"][:, 3], a["reward"][:, 4])
    assert a["status"][0, 3] == O.FAILED and a["type_id"][0, 1] == 255 and a["retired"][0, 1] == types[0, 1]
    # a scenario whose rows are all absent is done
    a = R.agents_epilogue(flags, types, x, y, h, steps, TABLE, N_TYPES, observers=np.full((4, 3), -1, np.int16))
    assert (a["done"] == 1).all() and (a["status"] == 0).all() and np.array_equal(a["type_id"], types)


def test_retirement_and_done_over_several_steps_then_restore():
    x, y, h, types, flags, steps = _scene(4, n=3, m=3, empty=0.0)
    flags[:] = 0
    st = dict(types=types, retired=None, lp=None, cnt=None)
    plan = [(0, 0), (0, 1), (1, 1)]   # (scenario, slot) that collides at step t
    for t, (n_hit, m_hit) in enumerate(plan):
        f = flags.copy()
        f[n_hit, m_hit] = O.F_STATIC
        a = R.agents_epilogue(f, st["types"], x, y, h, steps + t, TABLE, N_TYPES, retired=st["retired"], max_step=100)
        st.update(types=a["type_id"], retired=a["retired"])
        assert a["status"][n_hit, m_hit] == O.FAILED and a["type_id"][n_hit, m_hit] == 255
    # scenario 0 lost slots 0 and 1 (absent now), scenario 1 slot 1; nobody is done while a NORMAL row remains
    assert (a["status"][0, :2] == 0).all() and a["status"][1, 1] == O.FAILED and a["done"].tolist() == [0, 0, 0]
    f = flags.copy()
    f[0, 2] = O.F_OUTBOUND   # the last agent of scenario 0 settles: done
    a = R.agents_epilogue(f, st["types"], x, y, h, steps + 3, TABLE, N_TYPES, retired=st["retired"], max_step=100)
    assert a["done"].tolist() == [1, 0, 0] and (a["type_id"][0] == 255).all()
    a2 = R.agents_epilogue(flags, a["type_id"], x, y, h, steps + 4, TABLE, N_TYPES, retired=a["retired"], max_step=100)
    assert a2["done"].tolist() == [1, 0, 0] and (a2["status"][0] == 0).all()   # all absent: done at every step
    # a masked reset restores the masked scenarios only
    types_r, retired_r, lp, cnt = R.reset([1, 0, 0], a["type_id"], a["retired"], np.ones((3, 3, 4)), np.ones((3, 3), np.int64))
    assert np.array_equal(types_r[0], types[0]) and (retired_r[0] == 255).all()
    assert types_r[1, 1] == 255 and retired_r[1, 1] == types[1, 1]
    assert (lp[0, :, 3] == 0).all() and (lp[1:, :, 3] == 1).all() and (cnt[0] == 0).all() and (cnt[1:] == 1).all()
