"""Generate golden physics vectors from the UNMODIFIED reference.

TEST INFRASTRUCTURE ONLY.  Run where a checkout of the reference (WoodOxen/tactics2d @ d7095aa) exists:

    T2D_REFERENCE=<reference checkout> python oracle/make_golden.py     # writes tests/golden/*.npz

The reference's ``tactics2d.physics`` and ``tactics2d.participant.trajectory`` import
with NumPy alone (SURVEY.md section 8c); nothing else of the reference is importable in
an environment without shapely / gymnasium.  The vectors are committed so that the tests
hold both the oracle and the CUDA path to the reference's own numbers without the reference.  Action scripts replayed below are the reference test
suite's ``VEHICLE_ACTION_LIST`` / ``PEDESTRIAN_ACTION_LIST`` (tests/test_physics.py:52-73).
"""

from __future__ import annotations

import os
import sys

import numpy as np

REF = os.environ.get("T2D_REFERENCE")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")

# medium_car, participant_template.py:78-95 ; ranges as Vehicle.load_from_template sets them
MEDIUM = dict(lf=4.284 / 2 - 0.880, lr=4.284 / 2 - 0.767, mass=1620.0, mass_height=1.452 / 2)
RANGES = dict(steer_range=(-0.524, 0.524), speed_range=(-16.67, 69.44), accel_range=(-11.0, 3.121))

VEHICLE_ACTION_LIST = [((0, 0), 1000), ((1, 0), 1000), ((-1, 0), 1000), ((4, 0), 1000),
                       ((-4, 0), 1000), ((15, 0), 2000), ((-15, 0), 500), ((1, 0), 1000),
                       ((0.1, 0.3), 5000), ((0.1, -0.3), 5000), ((0.1, 0.6), 5000),
                       ((0.1, -0.6), 5000)]
PEDESTRIAN_ACTION_LIST = [((0, 0), 100), ((1, 0), 500), ((-1, 0), 500), ((1, 0), 500),
                          ((0, 1), 500), ((0, -1), 500), ((1, 1), 500), ((2, 2), 500),
                          ((-2, -2), 2000), ((-1, 2), 500), ((2, -1), 500)]


def main():
    if not REF or not os.path.isdir(os.path.join(REF, "tactics2d")):
        sys.exit("set T2D_REFERENCE to a checkout of the reference (the directory that holds tactics2d/)")
    sys.path.insert(0, REF)
    from tactics2d.participant.trajectory import State
    from tactics2d.physics import PointMass, SingleTrackDynamics, SingleTrackKinematics

    os.makedirs(OUT, exist_ok=True)
    rng = np.random.default_rng(20260924)

    def rec_bicycle(model, states, actions, interval):
        out = np.zeros((len(states), 8))
        for i, ((x, y, h, v), (a, d)) in enumerate(zip(states, actions)):
            s, a_c, d_c = model.step(State(0, x=x, y=y, heading=h, speed=v), a, d, interval)
            vx, vy = s.velocity
            out[i] = (s.x, s.y, s.heading, s.speed, vx, vy, a_c, d_c)
        return out

    n = 192
    states = np.stack([rng.uniform(-500, 500, n), rng.uniform(-500, 500, n),
                       rng.uniform(0, 2 * np.pi, n), rng.uniform(-15, 60, n)], 1)
    # a slice of low / zero speeds and out-of-range speeds
    states[:16, 3] = rng.uniform(-0.3, 0.3, 16)
    states[16:20, 3] = 0.0
    states[20:24, 3] = (80.0, -30.0, 69.44, -16.67)
    actions = np.stack([rng.uniform(-14, 6, n), rng.uniform(-0.8, 0.8, n)], 1)
    actions[24:28] = 0.0

    cases = {}
    for name, kw in [("con", RANGES), ("unc", dict())]:
        for interval, delta_t in [(100, 5), (9, 5), (50, 3), (100, None), (33, 10)]:
            m = SingleTrackKinematics(lf=MEDIUM["lf"], lr=MEDIUM["lr"], interval=interval,
                                      delta_t=delta_t, **kw)
            cases[f"kin_{name}_{interval}_{delta_t}"] = rec_bicycle(m, states, actions, interval)
            m = SingleTrackDynamics(lf=MEDIUM["lf"], lr=MEDIUM["lr"], mass=MEDIUM["mass"],
                                    mass_height=MEDIUM["mass_height"], interval=interval,
                                    delta_t=delta_t, **kw)
            cases[f"dyn_{name}_{interval}_{delta_t}"] = rec_bicycle(m, states, actions, interval)
    np.savez(os.path.join(OUT, "physics_bicycle.npz"), states=states, actions=actions,
             lf=MEDIUM["lf"], lr=MEDIUM["lr"], mass=MEDIUM["mass"],
             mass_height=MEDIUM["mass_height"], steer_range=RANGES["steer_range"],
             speed_range=RANGES["speed_range"], accel_range=RANGES["accel_range"], **cases)

    # ---- point mass
    pstates = np.stack([rng.uniform(-50, 50, n), rng.uniform(-50, 50, n),
                        rng.uniform(-5, 5, n), rng.uniform(-5, 5, n)], 1)  # x y vx vy
    pstates[:8, 2:] = 0.0
    pstates[8:16, 2:] *= 2.0  # some above the 7 m/s limit already
    pact = np.stack([rng.uniform(-4, 4, n), rng.uniform(-4, 4, n)], 1)
    pact[:4] = 0.0
    pact[16:20] = 1e-7
    pcases = {}
    for name, sr in [("ped", (-7.0, 7.0)), ("band", (1.0, 3.0)), ("flt", 4.0), ("unc", None)]:
        for backend in ("newton", "euler"):
            for interval, delta_t in [(100, 5), (9, 5), (50, 3)]:
                m = PointMass(speed_range=sr, accel_range=(-1.5, 1.5), interval=interval,
                              delta_t=delta_t, backend=backend)
                out = np.zeros((n, 6))
                for i in range(n):
                    x, y, vx, vy = pstates[i]
                    st = State(0, x=x, y=y, heading=float(np.arctan2(vy, vx)), vx=vx, vy=vy)
                    s = m.step(st, tuple(pact[i]), interval)
                    out[i] = (s.x, s.y, s.heading, s.vx, s.vy, s.speed)
                pcases[f"pm_{name}_{backend}_{interval}_{delta_t}"] = out
    np.savez(os.path.join(OUT, "physics_pointmass.npz"), states=pstates, actions=pact, **pcases)

    # ---- scripted rollouts (tests/test_physics.py:77-110 simulate_actions), free-running
    roll = {}
    for tag, cls, extra in [("kin", SingleTrackKinematics, {}),
                            ("dyn", SingleTrackDynamics, dict(mass=MEDIUM["mass"],
                                                              mass_height=MEDIUM["mass_height"]))]:
        for interval, delta_t in [(100, 5), (50, 3), (9, 5)]:
            m = cls(lf=MEDIUM["lf"], lr=MEDIUM["lr"], interval=interval, delta_t=delta_t,
                    **extra, **RANGES)
            s = State(0, x=10.0, y=10.0, heading=0.3, speed=5.0)
            traj = [(s.x, s.y, s.heading, s.speed)]
            acts = []
            for action, duration in VEHICLE_ACTION_LIST:
                for _ in np.arange(0, duration, interval):
                    s, _, _ = m.step(s, action[0], action[1], interval)
                    traj.append((s.x, s.y, s.heading, s.speed))
                    acts.append(action)
            roll[f"{tag}_{interval}_{delta_t}_traj"] = np.array(traj)
            roll[f"{tag}_{interval}_{delta_t}_act"] = np.array(acts, dtype=np.float64)
    for backend in ("newton", "euler"):
        m = PointMass(speed_range=(-7.0, 7.0), accel_range=(-1.5, 1.5), interval=100,
                      delta_t=5, backend=backend)
        s = State(0, x=0.0, y=0.0, heading=0.0, vx=0.0, vy=0.0)
        traj = [(s.x, s.y, s.heading, s.vx, s.vy)]
        acts = []
        for action, duration in PEDESTRIAN_ACTION_LIST:
            for _ in np.arange(0, duration, 100):
                s = m.step(s, action, 100)
                traj.append((s.x, s.y, s.heading, s.vx, s.vy))
                acts.append(action)
        roll[f"pm_{backend}_traj"] = np.array(traj)
        roll[f"pm_{backend}_act"] = np.array(acts, dtype=np.float64)
    np.savez(os.path.join(OUT, "physics_rollouts.npz"), **roll)

    # ---- verify_state truth table (single_track_kinematics.py:200-250)
    m = SingleTrackKinematics(lf=MEDIUM["lf"], lr=MEDIUM["lr"], **RANGES)
    vs_in, vs_out = [], []
    for _ in range(256):
        last = (rng.uniform(-50, 50), rng.uniform(-50, 50), rng.uniform(0, 2 * np.pi),
                rng.uniform(-5, 30))
        a, d = rng.uniform(-12, 4), rng.uniform(-0.6, 0.6)
        s, _, _ = m.step(State(0, x=last[0], y=last[1], heading=last[2], speed=last[3]), a, d, 100)
        cand = np.array([s.x, s.y, s.heading, s.speed]) + rng.normal(0, 1, 4) * rng.choice(
            [0.0, 1e-3, 0.05, 0.5])
        cand[2] = np.mod(cand[2], 2 * np.pi)
        ok = m.verify_state(State(100, x=cand[0], y=cand[1], heading=cand[2], speed=cand[3]),
                            State(0, x=last[0], y=last[1], heading=last[2], speed=last[3]), 100)
        vs_in.append(np.concatenate([last, cand]))
        vs_out.append(bool(ok))
    np.savez(os.path.join(OUT, "verify_state.npz"), inputs=np.array(vs_in),
             valid=np.array(vs_out))
    controllers_golden(rng)
    drift_golden(rng)
    lidar_golden(rng)
    print("golden vectors written to", os.path.normpath(OUT))


def drift_golden(rng):
    """SingleTrackDrift (single_track_drift.py:340-465): two consecutive steps per case (the second one consumes the
    wheel speeds the first one returned), fp32-representable inputs."""
    from tactics2d.participant.trajectory import State
    from tactics2d.physics import SingleTrackDrift

    n = 160
    st = np.stack([rng.uniform(-200, 200, n), rng.uniform(-200, 200, n), rng.uniform(0, 2 * np.pi, n),
                   rng.uniform(0.5, 30, n)], 1)
    st[:12, 3] = rng.uniform(-0.09, 0.09, 12)               # the |v| < 0.1 kinematic branch
    st[12:20, 3] = rng.uniform(-8, -0.5, 8)                 # reversing
    act = np.stack([rng.uniform(-6, 4, n), rng.uniform(-0.6, 0.6, n)], 1)
    act[20:24] = 0.0
    act2 = np.stack([rng.uniform(-6, 4, n), rng.uniform(-0.6, 0.6, n)], 1)
    st, act, act2 = (a.astype(np.float32).astype(np.float64) for a in (st, act, act2))
    radius = 0.344
    om = np.stack([st[:, 3] / radius * rng.uniform(0.9, 1.1, n), st[:, 3] / radius * rng.uniform(0.9, 1.1, n)], 1)
    om = om.astype(np.float32).astype(np.float64)
    out = dict(states=st, actions=act, actions2=act2, omega=om, lf=MEDIUM["lf"], lr=MEDIUM["lr"], mass=MEDIUM["mass"],
               mass_height=MEDIUM["mass_height"], steer_range=RANGES["steer_range"], speed_range=RANGES["speed_range"],
               accel_range=RANGES["accel_range"])
    for name, kw in [("con", RANGES), ("unc", dict())]:
        for interval, delta_t in [(100, 5), (9, 5), (50, 3)]:
            m = SingleTrackDrift(lf=MEDIUM["lf"], lr=MEDIUM["lr"], mass=MEDIUM["mass"], mass_height=MEDIUM["mass_height"],
                                 interval=interval, delta_t=delta_t, **kw)
            rec = np.zeros((n, 2, 8))
            for i in range(n):
                s = State(0, x=st[i, 0], y=st[i, 1], heading=st[i, 2], speed=st[i, 3])
                wf, wr = om[i]
                for k, a in enumerate((act[i], act2[i])):
                    s, wf, wr, a_c, d_c = m.step(s, wf, wr, a[0], a[1], interval)
                    rec[i, k] = (s.x, s.y, s.heading, s.speed, wf, wr, a_c, d_c)
            out[f"drift_{name}_{interval}_{delta_t}"] = rec
    np.savez(os.path.join(OUT, "physics_drift.npz"), **out)


def lidar_golden(rng):
    """``SingleLineLidar._scan_obstacles`` (sensor/lidar.py:128-221) of the unmodified reference.

    The module imports ``shapely.affinity.affine_transform``, ``shapely.geometry.{LinearRing, Point, Polygon}`` and
    ``tactics2d.map.element.Map`` (:11-14), none importable here.  The generator loads ``lidar.py`` / ``sensor_base.py``
    by path with stand-ins that provide exactly what the scan touches: ring coordinates, ``affine_transform`` of a ring
    (x' = a x + b y + xoff, y' = d x + e y + yoff - shapely's documented matrix order [a, b, d, e, xoff, yoff]),
    ``ring.distance(point)`` (only used to skip far obstacles, :122-125) and a ``Map`` with an ``areas`` dict.  The whole
    ray / edge arithmetic (:160-221) that the kernel reproduces is the reference's own NumPy code."""
    import importlib.util
    import types

    class Point:
        def __init__(self, *a):
            a = a[0] if len(a) == 1 else a
            self.x, self.y = float(a[0]), float(a[1])

    class LinearRing:
        def __init__(self, coords):
            c = [(float(x), float(y)) for x, y in coords]
            if c[0] != c[-1]:
                c.append(c[0])
            self.coords = c

        def distance(self, pt):
            c = np.asarray(self.coords)
            p1, p2 = c[:-1], c[1:]
            d = p2 - p1
            dd = (d * d).sum(1)
            t = np.clip(((np.array([pt.x, pt.y]) - p1) * d).sum(1) / np.where(dd > 0, dd, 1.0), 0, 1)
            e = p1 + t[:, None] * d - np.array([pt.x, pt.y])
            return float(np.sqrt((e * e).sum(1)).min())

    class Polygon:
        def __init__(self, coords):
            self.exterior = LinearRing(coords)

    def affine_transform(geom, m):
        a, b, d, e, xo, yo = m
        return LinearRing([(a * x + b * y + xo, d * x + e * y + yo) for x, y in geom.coords])

    saved = {k: sys.modules.get(k) for k in ("shapely", "shapely.geometry", "shapely.affinity", "tactics2d.map", "tactics2d.map.element")}
    shp, geo, aff = types.ModuleType("shapely"), types.ModuleType("shapely.geometry"), types.ModuleType("shapely.affinity")
    geo.Point, geo.LinearRing, geo.Polygon, geo.LineString = Point, LinearRing, Polygon, LinearRing
    aff.affine_transform = affine_transform
    shp.geometry, shp.affinity = geo, aff
    mp, mpe = types.ModuleType("tactics2d.map"), types.ModuleType("tactics2d.map.element")

    class Map:
        def __init__(self):
            self.areas = {}

    mpe.Map = Map
    mp.element = mpe
    sys.modules.update({"shapely": shp, "shapely.geometry": geo, "shapely.affinity": aff, "tactics2d.map": mp, "tactics2d.map.element": mpe})
    try:
        pkg = types.ModuleType("t2d_ref_sensor")
        pkg.__path__ = [os.path.join(REF, "tactics2d", "sensor")]
        sys.modules["t2d_ref_sensor"] = pkg
        for name in ("sensor_base", "lidar"):
            spec = importlib.util.spec_from_file_location(f"t2d_ref_sensor.{name}", os.path.join(REF, "tactics2d", "sensor", f"{name}.py"))
            mod = importlib.util.module_from_spec(spec)
            sys.modules[f"t2d_ref_sensor.{name}"] = mod
            spec.loader.exec_module(mod)
        SingleLineLidar = sys.modules["t2d_ref_sensor.lidar"].SingleLineLidar

        class Area:
            type_ = "obstacle"

            def __init__(self, ring):
                self.geometry = LinearRing(ring)

        class Body:
            def __init__(self, x, y, h, hl, hw):   # Vehicle.get_pose, vehicle.py:133-140,272-281
                c, s = np.cos(h), np.sin(h)
                loc = [(hl, -hw), (hl, hw), (-hl, hw), (-hl, -hw)]
                self.pose = Polygon([(x + cx * c - cy * s, y + cx * s + cy * c) for cx, cy in loc])

            def get_pose(self, frame):
                return self.pose

        n_scene, n_other = 12, 14
        f32 = lambda a: np.asarray(a, np.float32).astype(np.float64)
        ego = f32(np.stack([rng.uniform(10, 50, n_scene), rng.uniform(10, 50, n_scene), rng.uniform(0, 2 * np.pi, n_scene)], 1))
        others = f32(np.stack([rng.uniform(0, 60, (n_scene, n_other)), rng.uniform(0, 60, (n_scene, n_other)),
                               rng.uniform(0, 2 * np.pi, (n_scene, n_other)), rng.uniform(1.5, 3.0, (n_scene, n_other)),
                               rng.uniform(0.7, 1.1, (n_scene, n_other))], 2))
        others[:3, 0, :2] = ego[:3, :2] + f32([[0.4, -0.3]])          # a body overlapping the sensor
        walls = f32([[[0, 0], [60, 0], [60, 1], [0, 1]], [[0, 59], [60, 59], [60, 60], [0, 60]],
                     [[28, 20], [32, 20], [32, 40], [28, 40]], [[5, 30], [9, 34], [5, 38], [1, 34]]])
        out = dict(ego=ego, others=others, walls=walls)
        world = Map()
        world.areas = {i: Area(w) for i, w in enumerate(walls)}
        for n_beams, max_range in ((360, 20.0), (500, 12.0), (37, 30.0), (1100, 9.0)):
            res = np.zeros((n_scene, n_beams))
            for k in range(n_scene):
                lid = SingleLineLidar(1, world, perception_range=max_range, freq_scan=1.0, freq_detect=float(n_beams))
                assert lid.point_density == n_beams
                lid._position, lid._heading = Point(ego[k, 0], ego[k, 1]), float(ego[k, 2])
                lid.bind_with(0)
                bodies = {0: None}
                bodies.update({j + 1: Body(*others[k, j]) for j in range(n_other)})
                lid._scan_obstacles(0, bodies, list(bodies))
                res[k] = lid.scan_result
            out[f"scan_{n_beams}_{int(max_range)}"] = res
        np.savez(os.path.join(OUT, "lidar.npz"), **out)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def _shapely_stand_in():
    """``tactics2d.controller`` imports ``shapely.geometry.{LineString, Point}`` (pure_pursuit_controller.py:8) and
    uses exactly one method of them, ``LineString.interpolate`` (:92).  shapely is not installable in this image, so
    the generator provides that one method (arc-length walk from the first vertex, clamped to the last) and nothing
    else; every other line executed below is the reference's own."""
    import types

    class Point:
        def __init__(self, x, y):
            self.x, self.y = float(x), float(y)

    class LineString:
        def __init__(self, coords):
            self.coords = [(float(a), float(b)) for a, b in coords]

        def interpolate(self, d):
            acc = 0.0
            for (x0, y0), (x1, y1) in zip(self.coords[:-1], self.coords[1:]):
                L = float(np.hypot(x1 - x0, y1 - y0))
                if d <= acc + L and L > 0:
                    t = (d - acc) / L
                    return Point(x0 + t * (x1 - x0), y0 + t * (y1 - y0))
                acc += L
            return Point(*self.coords[-1])

    shp, geo = types.ModuleType("shapely"), types.ModuleType("shapely.geometry")
    geo.LineString, geo.Point = LineString, Point
    shp.geometry = geo
    sys.modules.setdefault("shapely", shp)
    sys.modules.setdefault("shapely.geometry", geo)
    return LineString


def controllers_golden(rng):
    """IDMController / AccelerationController / PurePursuitController outputs of the unmodified reference."""
    LineString = _shapely_stand_in()
    from tactics2d.controller.acceleration_controller import AccelerationController
    from tactics2d.controller.idm_controller import IDMController
    from tactics2d.controller.pure_pursuit_controller import PurePursuitController
    from tactics2d.participant.trajectory import State

    n = 256
    ego = np.stack([rng.uniform(-100, 100, n), rng.uniform(-100, 100, n), rng.uniform(0, 2 * np.pi, n),
                    rng.uniform(0, 25, n), rng.uniform(-4, 3, n)], 1)            # x y heading speed accel(signed)
    ego[:8, 3] = 0.0
    ego[8:16, 3] = rng.uniform(-3, 0, 8)                                         # reversing
    gap = rng.uniform(0.5, 120, n)
    gap[16:20] = 0.0                                                             # leader exactly on top (distance 0)
    ang = rng.uniform(0, 2 * np.pi, n)
    lead = np.stack([ego[:, 0] + gap * np.cos(ang), ego[:, 1] + gap * np.sin(ang), rng.uniform(0, 2 * np.pi, n),
                     rng.uniform(0, 25, n), rng.uniform(-4, 3, n)], 1)
    lead[16:20, :2] = ego[16:20, :2]
    # fp32-representable inputs: the device holds the state in fp32, so its outputs can be held to these vectors directly
    ego, lead = ego.astype(np.float32).astype(np.float64), lead.astype(np.float32).astype(np.float64)

    def st(row):
        return State(0, x=row[0], y=row[1], heading=row[2], speed=row[3], accel=row[4])

    out = dict(ego=ego, lead=lead)
    idm_cfgs = [dict(), dict(desired_speed=0.0), dict(desired_speed=20.0, time_headway=1.0, min_spacing=1.0,
                                                      max_acceleration=2.0, comfortable_deceleration=4.0, delta=4.0)]
    for ci, cfg in enumerate(idm_cfgs):
        c = IDMController(**cfg)
        out[f"idm{ci}_free"] = np.array([c.step(st(e))[1] for e in ego], np.float64)
        out[f"idm{ci}_follow"] = np.array([c.step(st(e), st(l))[1] for e, l in zip(ego, lead)], np.float64)
    out["idm_cfgs"] = np.array([[IDMController(**c).__dict__[k] for k in
                                 ("desired_speed", "time_headway", "min_spacing", "max_acceleration",
                                  "comfortable_deceleration", "delta")] for c in idm_cfgs], np.float64)
    acc_rows = []
    for si, style in enumerate([None, -1.0, 0.3, 1.0]):
        c = AccelerationController(target_speed=8.0)
        if style is not None:
            c.update_driving_style(style)
        acc_rows.append([c.target_speed, float(c.kp), float(c.accel_change_rate), float(c.delta_t), float(c.max_accel),
                         float(c.min_accel), float(c.interval)])
        out[f"acc{si}_cruise"] = np.array([c.step(st(e))[1] for e in ego], np.float64)
        out[f"acc{si}_follow"] = np.array([c.step(st(e), front_state=st(l))[1] for e, l in zip(ego, lead)], np.float64)
    out["acc_cfgs"] = np.array(acc_rows, np.float64)
    # pure pursuit: three paths, ego anywhere near them (the look-ahead is measured from the path's first vertex)
    paths = [np.array([[0.0, 0.0], [30.0, 0.0], [60.0, 20.0], [60.0, 80.0]]),
             np.array([[-50.0, -50.0], [-40.0, -50.0]]),                          # shorter than the look-ahead
             np.stack([40 * np.cos(np.linspace(0, np.pi, 33)), 40 * np.sin(np.linspace(0, np.pi, 33))], 1)]
    paths = [q.astype(np.float32).astype(np.float64) for q in paths]
    pid = rng.integers(0, len(paths), n)
    pp_rows, steer, accel = [], [], []
    for si, (style, kw) in enumerate([(None, dict()), (0.5, dict(min_pre_aiming_distance=4.0, target_speed=12.0))]):
        c = PurePursuitController(**kw)
        if style is not None:
            c.update_driving_style(style)
        wb = 2.637 if si == 0 else 2.9
        lc = c._longitudinal_control
        pp_rows.append([lc.target_speed, float(lc.kp), float(lc.accel_change_rate), float(lc.delta_t), float(lc.max_accel),
                        float(lc.min_accel), float(lc.interval), c.min_pre_aiming_distance, float(c.interval), wb])
        r = [c.step(st(e), LineString(paths[k]), wheel_base=wb) for e, k in zip(ego, pid)]
        r2 = [c.step(st(e), LineString(paths[k]), wheel_base=wb, front_state=st(l)) for e, k, l in zip(ego, pid, lead)]
        out[f"pp{si}_steer"] = np.array([a[0] for a in r], np.float64)
        out[f"pp{si}_accel"] = np.array([a[1] for a in r], np.float64)
        out[f"pp{si}_accel_follow"] = np.array([a[1] for a in r2], np.float64)
    out["pp_cfgs"] = np.array(pp_rows, np.float64)
    out["path_id"] = pid.astype(np.int64)
    for k, pth in enumerate(paths):
        out[f"path{k}"] = pth
    np.savez(os.path.join(OUT, "controllers.npz"), **out)


if __name__ == "__main__":
    main()
