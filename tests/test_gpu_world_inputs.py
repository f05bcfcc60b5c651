"""What ``BatchedWorld`` accepts and rejects wherever it hands an array to the library, as a table.

Every entry point is tried with one array in each form a caller may hold: a device tensor, a CPU tensor, NumPy, a list,
another dtype, another shape with the same element count, another element count and a non-contiguous view (and None
where None means something).  A row either names the exception class the call raises, or is accepted; an accepted row
must give, bit for bit, what the entry point gives for its reference form (the device tensor; NumPy for the host steps;
the equivalent array for None).

The BEV tests below hold the per-type styles to the current type table across ``set_type_table``."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N, M, Q = 8, 4, 3
SKIP = "skip"   # a None row's reference: the entry point is not called at all
STATE = ("x", "y", "heading", "speed", "vx", "vy", "type_id")


def _scene():
    from tactics2d_b200 import synthetic

    return synthetic.config2(N, M, seed=31, size=24.0)


def _world(dev, drift=False):
    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.types import TypeParams, TypeTable

    s = _scene()
    table = TypeTable([TypeParams.vehicle("medium_car", "drift")]) if drift else s.table
    w = BatchedWorld(N, M, table, device=dev, max_step=40)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=np.zeros((N, M), np.uint8) if drift else s.type_id)
    return w


def _actions(k, rows=M):
    from tactics2d_b200 import synthetic

    return synthetic.random_actions(200 + k, (N, rows))


def _dev(a, w):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).to(w.device)


OBSERVERS = np.array([[0, 2, 2]] * (N // 2) + [[3, 1, 0]] * (N // 2), np.int16)


def _pool(w, speed=None):
    s = _scene()
    p = {k: _dev(getattr(s, k)[::-1], w) for k in ("x", "y", "heading", "speed")}
    if speed is not None:
        p["speed"] = speed
    return p


def _controllers(w, ctrl_id, lead_index=None, last_accel=None):
    from tactics2d_b200.controller import IDMController, PurePursuitController

    w.set_paths([np.array([[0, 0], [12, 4], [24, 24]], np.float32)])
    w.set_controllers([IDMController(), PurePursuitController(min_pre_aiming_distance=4.0, target_speed=6.0)], ctrl_id,
                      lead_index, np.zeros((N, M), np.int16), last_accel)
    act = _dev(_actions(9), w)
    w.control(act)
    return dict(act=act, last_accel=w.last_accel)


CTRL_ID = np.tile(np.array([255, 0, 1, 0], np.uint8), (N, 1))
LEAD = np.tile(np.array([-1, 0, 1, 2], np.int16), (N, 1))


def _pid(w, pid_target=None, pid_state=None):
    import torch

    from tactics2d_b200.controller import PIDController

    tgt = np.stack([np.full((N, M), 6.0), np.full((N, M), 0.3)], 2).astype(np.float32) if pid_target is None else pid_target
    w.set_controllers([PIDController()], np.where(CTRL_ID == 255, 255, 0).astype(np.uint8), pid_target=tgt,
                      pid_state=pid_state)
    act = torch.zeros((N, M, 2), dtype=torch.float32, device=w.device)
    w.control(act)
    return dict(act=act, pid_state=w.pid_state)


def _goal_target():
    s = _scene()
    return np.stack([s.x[:, 0] + 1.0, s.y[:, 0], s.heading[:, 0], np.full(N, 2.5), np.full(N, 1.2)], 1).astype(np.float32)


def _tiles():
    s = _scene()
    ring = np.array([[6, 6, 10, 6], [10, 6, 10, 10], [10, 10, 6, 10], [6, 10, 6, 6]], np.float32)
    return [dict(segments=s.segments, bounds=s.bounds), dict(segments=ring, bounds=None, poly_start=[0, 4])]


def _step_zero(w):
    import torch

    r = w.step(torch.zeros((N, M, 2), dtype=torch.float32, device=w.device))
    return {} if r.iou is None else dict(iou=r.iou)


def _set_ego_action(w, v):
    if v is not SKIP:
        w.set_ego_action(v)
    return _step_zero(w)


def _scatter(w, agent_action=None, action=None, observers=None):
    import torch

    agent_action = _dev(_actions(3, Q), w) if agent_action is None else agent_action
    action = torch.zeros((N, M, 2), dtype=torch.float32, device=w.device) if action is None else action
    observers = _dev(OBSERVERS, w) if observers is None else observers
    return dict(out=w.scatter_agent_action(agent_action, action, observers))


GOALS = np.stack([np.full((N, Q), 5.0), np.full((N, Q), 5.0), np.zeros((N, Q)), np.full((N, Q), 2.5), np.full((N, Q), 1.2)],
                 -1).astype(np.float32)


def _agents_goals(w, v):
    w.set_agents(_dev(OBSERVERS, w), v)
    w.step(_dev(_actions(4), w))
    e = w.agents_epilogue()
    return dict(agent_reward=e.reward, agent_status=e.status, agent_iou=e.iou)


def _host_agents(w, agent_action=None, action=None):
    w.set_agents(_dev(OBSERVERS, w))
    return dict(zip("abcde", w.step_host_agents(_actions(5, Q) if agent_action is None else agent_action, action)))


def _set_goal(w, v):
    if v is not SKIP:
        w.set_goal(v, arrival_threshold=0.5)
    return _step_zero(w)


def _reset_mask(w, v):
    w.reset(v, _pool(w))
    return {}


def _reset_index(w, v):
    w.reset(_dev(np.ones(N, np.uint8), w), _pool(w), v)
    return {}


def _set_state_x(w, v):
    s = _scene()
    w.set_state(v, s.y, s.heading, s.speed, type_id=s.type_id)
    return {}


def _set_state_type_id(w, v):
    s = _scene()
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=v)
    return {}


def _wheels(w, v):
    w.set_wheel_state(v, np.full((N, M), 3.0, np.float32))
    return dict(front=w.omega_front, rear=w.omega_rear)


SPEED = (np.arange(N * M, dtype=np.float32).reshape(N, M) % 7) * 0.5
MASK = (np.arange(N) % 3 != 1).astype(np.uint8)
POOL_INDEX = np.array([5, 0, 7, 2, 2, 1, 6, 3], np.int32)
TILE_ID = np.array([0, 1, 1, 0, 1, 0, 0, 1], np.int64)

# entry: (kind, reference array, call(world, value) -> dict of outputs, the array None stands for (None: not tried),
#         world options)
ENTRIES = {
    "step.action": ("strict", _actions(0), lambda w, v: (w.step(v), {})[1], None, {}),
    "control.action": ("strict", _actions(1), lambda w, v: (_controllers(w, CTRL_ID), dict(out=w.control(v)))[1], None, {}),
    "set_ego_action": ("strict", _actions(2, 1)[:, 0].copy(), _set_ego_action, SKIP, {}),
    "scatter_agent_action.agent_action": ("strict", _actions(3, Q), lambda w, v: _scatter(w, agent_action=v), None, {}),
    "scatter_agent_action.action": ("strict", np.full((N, M, 2), 0.5, np.float32), lambda w, v: _scatter(w, action=v), None, {}),
    "scatter_agent_action.observers": ("strict", OBSERVERS, lambda w, v: _scatter(w, observers=v), None, {}),
    "set_agents.goals": ("strict", GOALS, _agents_goals, None, {}),
    "set_controllers.pid_state": ("strict", np.linspace(-0.1, 0.1, N * M * 6).reshape(N, M, 6),
                                  lambda w, v: _pid(w, pid_state=v), None, {}),
    "reset.pool": ("strict", SPEED, lambda w, v: (w.reset(_dev(np.ones(N, np.uint8), w), _pool(w, v)), {})[1], None, {}),
    "step_host_ego.action": ("strict", np.full((N, M, 2), 0.25, np.float32),
                             lambda w, v: dict(zip("ds", w.step_host_ego(_actions(6, 1)[:, 0].copy(), v))),
                             np.zeros((N, M, 2), np.float32), {}),
    "step_host_agents.action": ("strict", np.full((N, M, 2), 0.25, np.float32), lambda w, v: _host_agents(w, action=v),
                                np.zeros((N, M, 2), np.float32), {}),
    "step_host.action": ("host", _actions(7), lambda w, v: dict(zip("ds", w.step_host(v))), None, {}),
    "step_host_ego.ego_action": ("host", _actions(8, 1)[:, 0].copy(), lambda w, v: dict(zip("ds", w.step_host_ego(v))), None, {}),
    "step_host_agents.agent_action": ("host", _actions(5, Q), lambda w, v: _host_agents(w, agent_action=v), None, {}),
    "set_goal.target": ("convert", _goal_target(), _set_goal, SKIP, {}),
    "set_controllers.ctrl_id": ("convert", CTRL_ID, lambda w, v: _controllers(w, v, LEAD), None, {}),
    "set_controllers.lead_index": ("convert", LEAD, lambda w, v: _controllers(w, CTRL_ID, v), None, {}),
    "set_controllers.last_accel": ("convert", np.full((N, M), 0.75, np.float32), lambda w, v: _controllers(w, CTRL_ID, LEAD, v),
                                   np.zeros((N, M), np.float32), {}),
    "set_controllers.pid_target": ("convert", np.stack([np.full((N, M), 4.0), np.full((N, M), -0.2)], 2).astype(np.float32),
                                   lambda w, v: _pid(w, pid_target=v), None, {}),
    "set_map_table.tile_id": ("tile", TILE_ID, lambda w, v: (w.set_map_table(_tiles(), v), _step_zero(w))[1], None, {}),
    "set_state.x": ("convert", _scene().x, _set_state_x, None, {}),
    "set_state.type_id": ("convert", _scene().type_id, _set_state_type_id, None, {}),
    "set_wheel_state": ("convert", SPEED + 1.0, _wheels, None, dict(drift=True)),
    "reset.mask": ("count", MASK, _reset_mask, None, {}),
    "reset.pool_index": ("count", POOL_INDEX, _reset_index, np.arange(N, dtype=np.int32), {}),
}

# the outcome of every form, by the kind of entry point; "ok" = accepted with the reference form's outputs
OUTCOMES = {
    "strict": dict(device="ok", cpu=ValueError, numpy=ValueError, list=ValueError, dtype=ValueError, shape=ValueError,
                   size=ValueError, strided=ValueError),
    "host": dict(numpy="ok", list="ok", cpu="ok", dtype="ok", strided_numpy="ok", device=ValueError,
                 dtype_tensor=ValueError, shape=ValueError, size=ValueError, strided=ValueError),
    "convert": dict(device="ok", cpu="ok", numpy="ok", list="ok", dtype="ok", shape="ok", strided="ok", size=RuntimeError),
    "tile": dict(device="ok", cpu="ok", numpy="ok", list="ok", dtype="ok", shape="ok", strided="ok", size=ValueError,
                 range=ValueError),
    "count": dict(device="ok", cpu="ok", dtype="ok", shape="ok", strided="ok", numpy=ValueError, list=ValueError,
                  size=ValueError),
}


def _forms(a, kind, dev):
    """Every form of the reference array ``a`` the kind's table names."""
    import torch

    other = {np.float32: np.float64, np.float64: np.float32}.get(a.dtype.type, np.int64 if kind != "tile" else np.float64)
    wide = np.ascontiguousarray(np.stack([a, a], -1))
    f = dict(numpy=lambda: a.copy(), list=lambda: a.tolist(), cpu=lambda: torch.from_numpy(a.copy()),
             device=lambda: torch.from_numpy(a.copy()).to(dev), dtype=lambda: torch.from_numpy(a.astype(other)).to(dev),
             shape=lambda: torch.from_numpy(a.reshape((-1, 1) if a.ndim == 1 else -1).copy()).to(dev),
             size=lambda: torch.from_numpy(a.reshape(-1)[:-1].copy()).to(dev),
             strided=lambda: torch.from_numpy(wide).to(dev)[..., 0],
             range=lambda: torch.from_numpy(np.where(np.arange(len(a)) == 3, 2, a)).to(dev))
    if kind == "host":
        f.update(dtype=lambda: a.astype(np.float64), dtype_tensor=lambda: torch.from_numpy(a.astype(np.float64)),
                 shape=lambda: a.reshape(-1).copy(), size=lambda: a.reshape(-1)[:-1].copy(), strided_numpy=lambda: wide[..., 0],
                 strided=lambda: torch.from_numpy(wide)[..., 0])
    return f


def _rows():
    rows = []
    for name, (kind, a, _, none_as, _) in ENTRIES.items():
        rows += [(name, form) for form in OUTCOMES[kind]]
        if none_as is not None:
            rows.append((name, "none"))
    return rows


def _outputs(w, out):
    import torch

    torch.cuda.synchronize()
    r = w.result
    got = {k: getattr(w, k) for k in STATE}
    got.update(flags=r.flags, hit_index=r.hit_index, hit_segment=r.hit_segment, status=r.status, done=r.done, **out)
    return {k: np.ascontiguousarray(v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in got.items()}


def _run(dev, name, value):
    _, _, call, _, opts = ENTRIES[name]
    w = _world(dev, **opts)
    try:
        return _outputs(w, call(w, value))
    finally:
        w.close()


@pytest.mark.parametrize("name,form", _rows(), ids=[f"{n}-{f}" for n, f in _rows()])
def test_entry_point_input_forms(cuda_device, name, form):
    kind, a, _, none_as, _ = ENTRIES[name]
    expected = "ok" if form == "none" else OUTCOMES[kind][form]
    ref_form = "numpy" if kind == "host" else "device"
    if form == "none":
        value = None
        ref_value = none_as if none_as is SKIP else _forms(none_as, kind, cuda_device)[ref_form]()
    else:
        value = _forms(a, kind, cuda_device)[form]()
        ref_value = _forms(a, kind, cuda_device)[ref_form]()
    if expected != "ok":
        with pytest.raises(Exception) as e:
            _run(cuda_device, name, value)
        assert e.type is expected, (name, form, e.type, str(e.value))
        return
    got, ref = _run(cuda_device, name, value), _run(cuda_device, name, ref_value)
    assert got.keys() == ref.keys()
    for k in ref:
        assert got[k].shape == ref[k].shape and np.array_equal(got[k].view(np.uint8), ref[k].view(np.uint8)), (name, form, k)


def test_wheel_state_needs_a_drift_row(cuda_device):
    w = _world(cuda_device)
    with pytest.raises(ValueError):
        w.set_wheel_state(np.zeros((N, M), np.float32), np.zeros((N, M), np.float32))
    w.close()


# ---------------------------------------------------------------------------------------------------- BEV type styles
def _bev_scene():
    """Slot 0 an ego at the origin; slots 1..5 of types 0, 1, 2 around it, all within 12 m."""
    x = np.tile(np.array([0.0, 6.0, -6.0, 0.0, 8.0, -4.0], np.float32), (2, 1))
    y = np.tile(np.array([0.0, 2.0, -3.0, 7.0, -6.0, 9.0], np.float32), (2, 1))
    h = np.tile(np.array([0.0, 0.5, 1.0, -1.0, 2.0, 0.2], np.float32), (2, 1))
    tid = np.tile(np.array([0, 1, 2, 1, 2, 0], np.uint8), (2, 1))
    return x, y, h, np.zeros_like(x), tid


def _table(*rows):
    from tactics2d_b200.types import TypeParams, TypeTable

    make = dict(car=lambda: TypeParams.vehicle("medium_car"), suv=lambda: TypeParams.vehicle("sports_utility_car"),
                cyclist=lambda: TypeParams.cyclist("cyclist"), pedestrian=lambda: TypeParams.pedestrian("adult_male"))
    return TypeTable([make[r]() for r in rows])


def _bev_world(dev, table):
    from tactics2d_b200 import BatchedWorld

    return BatchedWorld(2, 6, table, device=dev)


def _image(w):
    import torch

    img = w.bev(resolution=(64, 48), perception_range=15.0, rgb=False).clone()
    torch.cuda.synchronize()
    return img.cpu().numpy()


RING = np.array([[-10, -10, 10, -10], [10, -10, 10, 10], [10, 10, -10, 10], [-10, 10, -10, -10]], np.float32)


def test_bev_styles_follow_a_larger_type_table(cuda_device):
    """Styles chosen for a 1-row table, then a 3-row table: the new rows are drawn in their default styles and the goal in
    the chosen target style, as in a world built with the 3-row table, and stay so after the next set_map."""
    from tactics2d_b200.sensor.camera import STYLE_KEYS

    big = _table("car", "cyclist", "pedestrian")
    a = _bev_world(cuda_device, _table("car"))
    a.set_bev_styles(target="keepout")
    a.set_type_table(big)
    b = _bev_world(cuda_device, big)
    b.set_bev_styles(target="keepout")
    for w in (a, b):
        w.set_state(*_bev_scene()[:4], type_id=_bev_scene()[4])
        w.set_goal(np.array([[3.0, -8.0, 0.3, 2.0, 1.0]] * 2, np.float32))
    ia, ib = _image(a), _image(b)
    for key in ("vehicle", "cyclist", "pedestrian", "keepout"):
        assert (ib == STYLE_KEYS.index(key)).any(), key
    assert np.array_equal(ia, ib)
    for w in (a, b):
        w.set_map(RING, (-20.0, 20.0, -20.0, 20.0), poly_start=[0, 4])
    ia, ib = _image(a), _image(b)
    assert (ib == STYLE_KEYS.index("obstacle")).any()
    assert np.array_equal(ia, ib)
    a.close()
    b.close()


def test_bev_styles_kept_by_a_table_of_as_many_rows(cuda_device):
    """Explicit styles survive a swap to another table with as many rows."""
    from tactics2d_b200.sensor.camera import STYLE_KEYS

    explicit = ["pedestrian", "vehicle", "cyclist"]
    a = _bev_world(cuda_device, _table("car", "cyclist", "pedestrian"))
    a.set_bev_styles(explicit, target=None)
    a.set_type_table(_table("suv", "car", "cyclist"))
    b = _bev_world(cuda_device, _table("suv", "car", "cyclist"))
    b.set_bev_styles(explicit, target=None)
    for w in (a, b):
        w.set_state(*_bev_scene()[:4], type_id=_bev_scene()[4])
    ia, ib = _image(a), _image(b)
    assert (ib == STYLE_KEYS.index("pedestrian")).any() and np.array_equal(ia, ib)
    a.close()
    b.close()
