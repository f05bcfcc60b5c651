"""The oracle is pinned to the UNMODIFIED reference: golden vectors written by
oracle/make_golden.py (which imports the reference's tactics2d/physics) and the survey's
known-answer table (SURVEY.md section 8c)."""

import os

import numpy as np
import pytest

from oracle import physics as P

GOLD = os.path.join(os.path.dirname(__file__), "golden")
INF = (-np.inf, np.inf)
TOL = 1e-12


def _rel(got, ref):
    return np.abs(got - ref) / np.maximum(1.0, np.abs(ref))


def test_bicycle_golden():
    g = np.load(os.path.join(GOLD, "physics_bicycle.npz"))
    st, ac = g["states"], g["actions"]
    n_cases = 0
    for k in g.files:
        if not (k.startswith("kin_") or k.startswith("dyn_")):
            continue
        tag, name, interval, dt = k.split("_")
        interval = int(interval)
        dt = P.effective_delta_t(None if dt == "None" else int(dt), interval)
        rng = (tuple(g["steer_range"]), tuple(g["speed_range"]), tuple(g["accel_range"])) if name == "con" else (INF,) * 3
        if tag == "kin":
            o = P.step_kinematics(st[:, 0], st[:, 1], st[:, 2], st[:, 3], ac[:, 0], ac[:, 1], g["lf"], g["lr"], *rng,
                                  interval=interval, delta_t=dt)
        else:
            o = P.step_dynamics(st[:, 0], st[:, 1], st[:, 2], st[:, 3], ac[:, 0], ac[:, 1], g["lf"], g["lr"], g["mass"],
                                g["mass_height"], 0.7, 1500, 20.89, 20.89, *rng, interval=interval, delta_t=dt)
        got = np.stack([o[c] for c in ("x", "y", "heading", "speed", "vx", "vy", "accel", "delta")], 1)
        assert _rel(got, g[k]).max() <= TOL, k
        n_cases += 1
    assert n_cases == 20


def test_pointmass_golden():
    g = np.load(os.path.join(GOLD, "physics_pointmass.npz"))
    st, ac = g["states"], g["actions"]
    ranges = {"ped": (-7.0, 7.0), "band": (1.0, 3.0), "flt": 4.0, "unc": None}
    n_cases = 0
    for k in g.files:
        if not k.startswith("pm_"):
            continue
        _, name, backend, interval, dt = k.split("_")
        interval, dt = int(interval), int(dt)
        sr = P.normalize_range_pointmass(ranges[name])
        if backend == "newton":
            o = P.step_pointmass_newton(st[:, 0], st[:, 1], st[:, 2], st[:, 3], ac[:, 0], ac[:, 1], sr, interval)
        else:
            o = P.step_pointmass_euler(st[:, 0], st[:, 1], np.arctan2(st[:, 3], st[:, 2]), st[:, 2], st[:, 3], ac[:, 0],
                                       ac[:, 1], sr, interval, dt)
        got = np.stack([o[c] for c in ("x", "y", "heading", "vx", "vy", "speed")], 1)
        assert _rel(got, g[k]).max() <= TOL, k
        n_cases += 1
    assert n_cases == 24


def test_rollouts_free_running():
    """tests/test_physics.py:77-110 simulate_actions over VEHICLE/PEDESTRIAN_ACTION_LIST, free-running."""
    g = np.load(os.path.join(GOLD, "physics_rollouts.npz"))
    b = np.load(os.path.join(GOLD, "physics_bicycle.npz"))
    rng = (tuple(b["steer_range"]), tuple(b["speed_range"]), tuple(b["accel_range"]))
    for tag in ("kin", "dyn"):
        for interval, dt in [(100, 5), (50, 3), (9, 5)]:
            traj, act = g[f"{tag}_{interval}_{dt}_traj"], g[f"{tag}_{interval}_{dt}_act"]
            s = traj[0].copy()
            for i in range(len(act)):
                if tag == "kin":
                    o = P.step_kinematics(s[0], s[1], s[2], s[3], act[i, 0], act[i, 1], b["lf"], b["lr"], *rng,
                                          interval=interval, delta_t=dt)
                else:
                    o = P.step_dynamics(s[0], s[1], s[2], s[3], act[i, 0], act[i, 1], b["lf"], b["lr"], b["mass"],
                                        b["mass_height"], 0.7, 1500, 20.89, 20.89, *rng, interval=interval, delta_t=dt)
                s = np.array([o["x"], o["y"], o["heading"], o["speed"]], dtype=np.float64)
                assert _rel(s, traj[i + 1]).max() <= 1e-9, (tag, interval, dt, i)
    for backend in ("newton", "euler"):
        traj, act = g[f"pm_{backend}_traj"], g[f"pm_{backend}_act"]
        s = traj[0].copy()
        for i in range(len(act)):
            if backend == "newton":
                o = P.step_pointmass_newton(s[0], s[1], s[3], s[4], act[i, 0], act[i, 1], (0.0, 7.0), 100)
            else:
                o = P.step_pointmass_euler(s[0], s[1], s[2], s[3], s[4], act[i, 0], act[i, 1], (0.0, 7.0), 100, 5)
            s = np.array([o["x"], o["y"], o["heading"], o["vx"], o["vy"]], dtype=np.float64)
            assert _rel(s, traj[i + 1]).max() <= 1e-9, (backend, i)


# SURVEY.md section 8(c): values measured from the reference code (medium_car, lf=1.262, lr=1.375).
KIN = dict(lf=1.262, lr=1.375)
RNG = ((-0.524, 0.524), (-16.67, 69.44), (-11.0, 3.121))


def test_known_answers_kinematics():
    o = P.step_kinematics(10, 10, 0.3, 5, 1.0, 0.2, KIN["lf"], KIN["lr"], *RNG)
    np.testing.assert_allclose([o["x"], o["y"], o["heading"], o["speed"], o["vx"], o["vy"]],
                               [10.460101899439735, 10.207478447324114, 0.3385859239425399, 5.099999999999998,
                                4.810449024453569, 1.693983525047891], rtol=1e-13)
    o2 = P.step_kinematics(o["x"], o["y"], o["heading"], o["speed"], 5.0, -0.9, KIN["lf"], KIN["lr"], *RNG)
    np.testing.assert_allclose([o2["x"], o2["y"], o2["heading"], o2["speed"], o2["accel"], o2["delta"]],
                               [10.984652234013904, 10.204125170899955, 0.22846394026452768, 5.412099999999995, 3.121, -0.524],
                               rtol=1e-13)
    o3 = P.step_kinematics(10, 10, 0.3, 5, 1.0, 0.2, KIN["lf"], KIN["lr"], *RNG, interval=9)
    np.testing.assert_allclose([o3["x"], o3["y"], o3["heading"], o3["speed"]],
                               [10.04135741781754, 10.017786583803838, 0.30344158156690076, 5.0089999999999995], rtol=1e-13)


def test_known_answers_dynamics():
    dyn = lambda *a, **k: P.step_dynamics(*a, KIN["lf"], KIN["lr"], 1620, 0.726, 0.7, 1500, 20.89, 20.89, *RNG, **k)
    o = dyn(10, 10, 0.3, 5, 1.0, 0.2)
    np.testing.assert_allclose([o["x"], o["y"], o["heading"], o["speed"]],
                               [10.454044498400336, 10.220136047786687, 0.33888560266154016, 5.099999999999998], rtol=1e-13)
    o2 = dyn(o["x"], o["y"], o["heading"], o["speed"], 5.0, -0.9)
    np.testing.assert_allclose([o2["x"], o2["y"], o2["heading"], o2["speed"]],
                               [10.976942116208368, 10.188167832708386, 0.2287557008757041, 5.412099999999995], rtol=1e-13)
    o3 = dyn(10, 10, 0.3, 0.05, 1.0, 0.2)  # low-speed branch: heading jumps
    np.testing.assert_allclose([o3["x"], o3["y"], o3["heading"], o3["speed"]],
                               [10.003277244831548, 10.002000985139086, 5.781714387949648, 0.15000000000000008], rtol=1e-12)
    o4 = dyn(10, 10, 0.3, 5, 1.0, 0.2, interval=9)  # no remainder sub-step
    np.testing.assert_allclose([o4["x"], o4["y"], o4["heading"], o4["speed"]],
                               [10.021728059527945, 10.012364927381514, 0.30194726104561803, 5.005], rtol=1e-13)


def test_known_answers_pointmass():
    sr = P.normalize_range_pointmass((-7, 7))
    assert sr == (0.0, 7.0)  # Pedestrian's (-7, 7) becomes [0, 7]
    o = P.step_pointmass_newton(10, 10, 1, 0.5, 0.5, 0.2, sr)
    np.testing.assert_allclose([o["x"], o["y"], o["heading"], o["speed"], o["vx"], o["vy"]],
                               [10.1025, 10.051, 0.45983083364175814, 1.1717081547894084, 1.05, 0.52], rtol=1e-13)
    o = P.step_pointmass_newton(10, 10, 6.9, 0.5, 3, 1, sr)  # speed-limit branch
    np.testing.assert_allclose([o["x"], o["y"], o["heading"], o["speed"], o["vx"], o["vy"]],
                               [10.696944716341092, 10.052314905447028, 0.07531667613487306, 7.0, 6.980155277631122,
                                0.5267184258770407], rtol=1e-13)


def test_range_normalisation_rules():
    assert P.normalize_range_bicycle(0.5) == (-0.5, 0.5)
    assert P.normalize_range_bicycle(-0.5) == (-np.inf, np.inf)
    assert P.normalize_range_bicycle(1) == (-np.inf, np.inf)  # an int is NOT a float -> None
    assert P.normalize_range_bicycle((1.0, 1.0)) == (-np.inf, np.inf)
    assert P.normalize_range_bicycle((-1, 2)) == (-1.0, 2.0)
    assert P.normalize_range_bicycle(None) == (-np.inf, np.inf)
    assert P.normalize_range_pointmass(3.0) == (0.0, 3.0)
    assert P.normalize_range_pointmass((-2, -1)) == (-np.inf, np.inf)
    assert P.effective_delta_t(None, 100) == 5 and P.effective_delta_t(0, 100) == 1 and P.effective_delta_t(50, 9) == 9


def test_verify_state_golden():
    g = np.load(os.path.join(GOLD, "verify_state.npz"))
    got = [P.verify_state_bicycle(tuple(r[4:]), tuple(r[:4]), KIN["lr"] * 0 + (4.284 / 2 - 0.767),
                                  (4.284 / 2 - 0.880) + (4.284 / 2 - 0.767), RNG[0], RNG[1], RNG[2], 100)
           for r in g["inputs"]]
    assert np.array_equal(np.array(got), g["valid"])
    assert 0 < g["valid"].sum() < len(g["valid"])


@pytest.mark.parametrize("name", ["con", "unc"])
@pytest.mark.parametrize("interval,delta_t", [(100, 5), (9, 5), (50, 3)])
def test_drift_restatement_equals_reference(name, interval, delta_t):
    """SingleTrackDrift: two chained steps (the second consumes the wheel speeds of the first)."""
    from oracle import physics as P

    g = np.load(os.path.join(GOLD, "physics_drift.npz"))
    inf = (-np.inf, np.inf)
    rng = {k: (tuple(g[k]) if name == "con" else inf) for k in ("steer_range", "speed_range", "accel_range")}
    st, om = g["states"], g["omega"]
    want = g[f"drift_{name}_{interval}_{delta_t}"]
    cur = dict(x=st[:, 0], y=st[:, 1], heading=st[:, 2], speed=st[:, 3], omega_wf=om[:, 0], omega_wr=om[:, 1])
    for k, act in enumerate((g["actions"], g["actions2"])):
        cur = P.step_drift(cur["x"], cur["y"], cur["heading"], cur["speed"], cur["omega_wf"], cur["omega_wr"], act[:, 0], act[:, 1],
                           float(g["lf"]), float(g["lr"]), float(g["mass"]), 0.344, 0.76, 1.0, 1500.0, 1.7,
                           rng["steer_range"], rng["speed_range"], rng["accel_range"], interval, delta_t)
        got = np.stack([cur[f] for f in ("x", "y", "heading", "speed", "omega_wf", "omega_wr", "accel", "delta")], 1)
        np.testing.assert_allclose(got, want[:, k], rtol=1e-9, atol=1e-9)
