"""Write tests/golden/lidar_bound.npz from the UNMODIFIED reference's ``SingleLineLidar`` bound to a body other than 0.

TEST INFRASTRUCTURE ONLY.  Run where a checkout of the reference (WoodOxen/tactics2d @ d7095aa) exists:

    T2D_REFERENCE=<reference checkout> python tests/make_lidar_bound_golden.py

The fixture pins the binding rule of the per-agent lidar (DESIGN.md section 1 "Per-agent lidar") to the reference's own
code: ``bind_with(k)`` with k != 0 at k's pose among several bodies, ``_scan_obstacles`` skips k and sees every other
body, body 0 included (sensor/lidar.py:146-153).  It has its own seeded generator and touches no other fixture.

``sensor/lidar.py`` imports ``shapely.affinity.affine_transform``, ``shapely.geometry.{LinearRing, Point, Polygon}`` and
``tactics2d.map.element.Map`` (:11-14), none importable here.  As ``oracle/make_golden.py`` does for ``lidar.npz``, this
loads ``lidar.py`` / ``sensor_base.py`` by path with stand-ins that provide exactly what the scan touches: ring
coordinates, ``affine_transform`` of a ring (x' = a x + b y + xoff, y' = d x + e y + yoff - shapely's documented matrix
order [a, b, d, e, xoff, yoff]), ``ring.distance(point)`` (only used to skip far obstacles, :122-125) and a ``Map`` with an
``areas`` dict.  The ray / edge arithmetic (:160-221) is the reference's own NumPy code.
"""

from __future__ import annotations

import contextlib
import importlib.util
import os
import sys
import types

import numpy as np

REF = os.environ.get("T2D_REFERENCE")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lidar_bound.npz")

WALLS = [[[0, 0], [60, 0], [60, 1], [0, 1]], [[0, 59], [60, 59], [60, 60], [0, 60]],
         [[28, 20], [32, 20], [32, 40], [28, 40]], [[5, 30], [9, 34], [5, 38], [1, 34]]]
SETTINGS = ((360, 20.0), (500, 12.0), (37, 30.0), (1100, 9.0))


@contextlib.contextmanager
def reference_lidar():
    """Yields ``(SingleLineLidar, Map, Area, Body, Point)``: the reference's sensor class, and stand-ins for a map, an
    obstacle area of a ring and a box body whose pose is ``Vehicle.get_pose``'s polygon."""

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

    class Map:
        def __init__(self):
            self.areas = {}

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

    names = ("shapely", "shapely.geometry", "shapely.affinity", "tactics2d.map", "tactics2d.map.element", "t2d_ref_sensor",
             "t2d_ref_sensor.sensor_base", "t2d_ref_sensor.lidar")
    saved = {k: sys.modules.get(k) for k in names}
    shp, geo, aff = types.ModuleType("shapely"), types.ModuleType("shapely.geometry"), types.ModuleType("shapely.affinity")
    geo.Point, geo.LinearRing, geo.Polygon, geo.LineString = Point, LinearRing, Polygon, LinearRing
    aff.affine_transform = affine_transform
    shp.geometry, shp.affinity = geo, aff
    mp, mpe = types.ModuleType("tactics2d.map"), types.ModuleType("tactics2d.map.element")
    mpe.Map = Map
    mp.element = mpe
    sys.modules.update({"shapely": shp, "shapely.geometry": geo, "shapely.affinity": aff, "tactics2d.map": mp,
                        "tactics2d.map.element": mpe})
    try:
        pkg = types.ModuleType("t2d_ref_sensor")
        pkg.__path__ = [os.path.join(REF, "tactics2d", "sensor")]
        sys.modules["t2d_ref_sensor"] = pkg
        for name in ("sensor_base", "lidar"):
            spec = importlib.util.spec_from_file_location(f"t2d_ref_sensor.{name}",
                                                          os.path.join(REF, "tactics2d", "sensor", f"{name}.py"))
            mod = importlib.util.module_from_spec(spec)
            sys.modules[f"t2d_ref_sensor.{name}"] = mod
            spec.loader.exec_module(mod)
        yield sys.modules["t2d_ref_sensor.lidar"].SingleLineLidar, Map, Area, Body, Point
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def lidar_bound_golden(rng):
    """``bodies`` [scene, body, 5] = (x, y, heading, half_len, half_wid), ``bound`` [scene] (the body carrying the
    sensor), ``walls`` and one scan array ``scan_{beams}_{range}`` [scene, beams] per setting."""
    with reference_lidar() as (SingleLineLidar, Map, Area, Body, Point):
        n_scene, n_body = 12, 10
        f32 = lambda a: np.asarray(a, np.float32).astype(np.float64)
        bodies = f32(np.stack([rng.uniform(5, 55, (n_scene, n_body)), rng.uniform(5, 55, (n_scene, n_body)),
                               rng.uniform(0, 2 * np.pi, (n_scene, n_body)), rng.uniform(1.5, 3.0, (n_scene, n_body)),
                               rng.uniform(0.7, 1.1, (n_scene, n_body))], 2))
        bound = rng.integers(1, n_body, n_scene)
        rows = np.arange(n_scene)
        # the sensor away from the inner walls, body 0 within 3 - 4.5 m of it (in reach of every setting's range), every
        # other body at least 9 m away: nothing stands between the sensor and body 0, whose ring the scan must show; in
        # three scenes body 0 overlaps the sensor instead
        bodies[rows, bound, 0] = f32(rng.uniform(38, 52, n_scene))
        bodies[rows, bound, 1] = f32(rng.uniform(10, 50, n_scene))
        for k in range(n_scene):
            sx, sy = bodies[k, bound[k], :2]
            for j in range(1, n_body):
                while j != bound[k] and np.hypot(bodies[k, j, 0] - sx, bodies[k, j, 1] - sy) < 9.0:
                    bodies[k, j, :2] = f32(rng.uniform(5, 55, 2))
        ang = rng.uniform(0, 2 * np.pi, n_scene)
        dist = np.where(rows < 3, 0.5, rng.uniform(3.0, 4.5, n_scene))
        bodies[:, 0, 0] = f32(bodies[rows, bound, 0] + dist * np.cos(ang))
        bodies[:, 0, 1] = f32(bodies[rows, bound, 1] + dist * np.sin(ang))
        walls = f32(WALLS)
        out = dict(bodies=bodies, bound=bound.astype(np.int64), walls=walls)
        world = Map()
        world.areas = {i: Area(w) for i, w in enumerate(walls)}
        for n_beams, max_range in SETTINGS:
            res = np.zeros((n_scene, n_beams))
            for k in range(n_scene):
                lid = SingleLineLidar(1, world, perception_range=max_range, freq_scan=1.0, freq_detect=float(n_beams))
                assert lid.point_density == n_beams
                b = int(bound[k])
                lid._position, lid._heading = Point(bodies[k, b, 0], bodies[k, b, 1]), float(bodies[k, b, 2])
                lid.bind_with(b)
                parts = {j: Body(*bodies[k, j]) for j in range(n_body)}
                lid._scan_obstacles(0, parts, list(parts))
                res[k] = lid.scan_result
            out[f"scan_{n_beams}_{int(max_range)}"] = res
        return out


def main():
    if not REF or not os.path.isdir(os.path.join(REF, "tactics2d")):
        sys.exit("set T2D_REFERENCE to a checkout of the reference (the directory that holds tactics2d/)")
    np.savez(OUT, **lidar_bound_golden(np.random.default_rng(20261016)))
    print("written", os.path.normpath(OUT))


if __name__ == "__main__":
    main()
