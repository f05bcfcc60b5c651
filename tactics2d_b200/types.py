"""Participant type table: the per-type constants the kernels read from shared memory.

A row is what the reference spreads over a participant object and its physics model:
dimensions (``ParticipantBase.length/width``, participant_base.py:33-39), collision shape
(``Vehicle._bbox`` vehicle.py:132-142 / ``Pedestrian._radius`` pedestrian.py:85-88) and the
physics constructor arguments (single_track_kinematics.py:62-124, single_track_dynamics.py:58-138,
point_mass.py:33-81).  Mirrors ``t2d_type_params`` in ``include/t2d_b200.h``.
"""

from __future__ import annotations

import math
from dataclasses import dataclass, fields
from typing import Iterable, List, Sequence

import numpy as np

from ._lib import TypeParamsC

MODEL_KINEMATICS, MODEL_DYNAMICS, MODEL_POINTMASS_NEWTON, MODEL_POINTMASS_EULER, MODEL_STATIC, MODEL_DRIFT = range(6)
SHAPE_OBB, SHAPE_CIRCLE, SHAPE_NONE = range(3)
TYPE_INACTIVE = 255
MAX_TYPES = 64
INF = math.inf


def normalize_range_bicycle(r):
    """Range rule of the three bicycles (single_track_kinematics.py:87-115): a Python float
    r >= 0 -> (-r, r), negative -> unconstrained; a 2-sequence lo < hi is kept, else
    unconstrained; anything else (None, or an ``int``) -> unconstrained = (-inf, inf)."""
    if isinstance(r, float):
        return (-INF, INF) if r < 0 else (-r, r)
    if hasattr(r, "__len__") and len(r) == 2:
        return (-INF, INF) if r[0] >= r[1] else (float(r[0]), float(r[1]))
    return (-INF, INF)


def normalize_range_pointmass(r):
    """PointMass rule (point_mass.py:50-66): float r >= 0 -> (0, r); tuple ->
    (max(0, lo), max(0, hi)), unconstrained when empty."""
    if isinstance(r, float):
        return (-INF, INF) if r < 0 else (0.0, r)
    if hasattr(r, "__len__") and len(r) == 2:
        lo, hi = max(0, r[0]), max(0, r[1])
        return (-INF, INF) if lo >= hi else (float(lo), float(hi))
    return (-INF, INF)


@dataclass
class TypeParams:
    half_len: float = 0.0
    half_wid: float = 0.0
    radius: float = 0.0
    lf: float = 1.0
    lr: float = 1.0
    steer_lo: float = -INF
    steer_hi: float = INF
    speed_lo: float = -INF
    speed_hi: float = INF
    accel_lo: float = -INF
    accel_hi: float = INF
    mass: float = 1.0
    mass_height: float = 0.0
    mu: float = 0.7
    I_z: float = 1500.0
    cf: float = 20.89
    cr: float = 20.89
    model: int = MODEL_KINEMATICS
    shape: int = SHAPE_OBB
    wheel_radius: float = 0.344     # SingleTrackDrift defaults, single_track_drift.py:98-107
    T_sb: float = 0.76
    T_se: float = 1.0
    I_yw: float = 1.7
    name: str = ""

    def to_c(self) -> TypeParamsC:
        c = TypeParamsC()
        for f, _ in TypeParamsC._fields_:
            setattr(c, f, getattr(self, f))
        return c

    # ---- constructors following the reference's participant classes -------------------------
    @classmethod
    def vehicle(cls, type_name: str = "medium_car", model: str = "kinematics", **override) -> "TypeParams":
        """``Vehicle`` + ``load_from_template`` (vehicle.py:107-142,179-221): steer +-round(pi/6, 3),
        speed (-16.67, max_speed), accel (-max_decel, max_accel = round(27.78/t_0_100, 3));
        physics as ``_auto_construct_physics_model`` (:148-157): lf = L/2 - front_overhang,
        lr = L/2 - rear_overhang.  ``model="dynamics"`` / ``"drift"`` use kerb_weight and height/2
        (single_track_dynamics.py:79-80 docstring); drift keeps the wheel defaults of single_track_drift.py:98-107."""
        from .participant.element.participant_template import VEHICLE_TEMPLATE

        t = dict(VEHICLE_TEMPLATE[type_name])
        t.update(override)
        max_accel = t.get("max_accel", float(np.round(100 * 1000 / 3600 / t["0_100_km/h"], 3)))
        max_steer = t.get("max_steer", float(np.round(np.pi / 6, 3)))
        return cls(half_len=t["length"] / 2, half_wid=t["width"] / 2,
                   lf=t["length"] / 2 - t["front_overhang"], lr=t["length"] / 2 - t["rear_overhang"],
                   steer_lo=-max_steer, steer_hi=max_steer, speed_lo=-16.67, speed_hi=t["max_speed"],
                   accel_lo=-t["max_decel"], accel_hi=max_accel, mass=t["kerb_weight"],
                   mass_height=t["height"] / 2,
                   model={"dynamics": MODEL_DYNAMICS, "drift": MODEL_DRIFT}.get(model, MODEL_KINEMATICS),
                   shape=SHAPE_OBB, name=type_name)

    @classmethod
    def cyclist(cls, type_name: str = "cyclist") -> "TypeParams":
        """``Cyclist`` (cyclist.py:76-105): steer +-max_steer, speed (0, max_speed),
        accel (-max_decel, max_accel), kinematics with lf = lr = L/2."""
        from .participant.element.participant_template import CYCLIST_TEMPLATE

        t = CYCLIST_TEMPLATE[type_name]
        return cls(half_len=t["length"] / 2, half_wid=t["width"] / 2, lf=t["length"] / 2, lr=t["length"] / 2,
                   steer_lo=-t["max_steer"], steer_hi=t["max_steer"], speed_lo=0.0, speed_hi=t["max_speed"],
                   accel_lo=-t["max_decel"], accel_hi=t["max_accel"], model=MODEL_KINEMATICS,
                   shape=SHAPE_OBB, name=type_name)

    @classmethod
    def pedestrian(cls, type_name: str = "adult_male", backend: str = "newton") -> "TypeParams":
        """``Pedestrian`` (pedestrian.py:70-88): PointMass(speed_range=(-vmax, vmax)) which the
        constructor normalises to [0, vmax] (point_mass.py:52-55); pose = disc of width/2."""
        from .participant.element.participant_template import PEDESTRIAN_TEMPLATE

        t = PEDESTRIAN_TEMPLATE[type_name]
        lo, hi = normalize_range_pointmass((-t["max_speed"], t["max_speed"]))
        alo, ahi = normalize_range_pointmass((-t["max_accel"], t["max_accel"]))
        return cls(half_len=t["length"] / 2, half_wid=t["width"] / 2, radius=t["width"] / 2,
                   speed_lo=lo, speed_hi=hi, accel_lo=alo, accel_hi=ahi,
                   model=MODEL_POINTMASS_EULER if backend == "euler" else MODEL_POINTMASS_NEWTON,
                   shape=SHAPE_CIRCLE, name=type_name)

    @classmethod
    def obstacle(cls, length: float, width: float) -> "TypeParams":
        """``Obstacle`` / static ``Other`` (other.py:105-126, obstacle.py:14-19): a box that never moves."""
        return cls(half_len=length / 2, half_wid=width / 2, model=MODEL_STATIC, shape=SHAPE_OBB, name="obstacle")


class TypeTable:
    """An ordered list of :class:`TypeParams`; ``type_id`` of a participant indexes it."""

    def __init__(self, rows: Iterable[TypeParams]):
        self.rows: List[TypeParams] = list(rows)
        if not 1 <= len(self.rows) <= MAX_TYPES:
            raise ValueError(f"a type table holds 1..{MAX_TYPES} rows, got {len(self.rows)}")

    def __len__(self):
        return len(self.rows)

    def index(self, name: str) -> int:
        for i, r in enumerate(self.rows):
            if r.name == name:
                return i
        raise KeyError(name)

    def with_static_twins(self, rows: Iterable[int]):
        """This table plus one ``MODEL_STATIC`` copy of each of ``rows`` (same shape, extents and name, so BEV styles and the
        lidar treat it like its class): the rows replayed participants take (``BatchedWorld.set_log``).  Returns
        ``(table, twin)`` with ``twin[row]`` the index of row's twin; a row that is static already is its own twin."""
        from dataclasses import replace

        out, twin = list(self.rows), {}
        for r in sorted({int(v) for v in rows}):
            if self.rows[r].model == MODEL_STATIC:
                twin[r] = r
                continue
            twin[r] = len(out)
            out.append(replace(self.rows[r], model=MODEL_STATIC))
        if len(out) > MAX_TYPES:
            raise ValueError(f"static twins of {len(twin)} rows do not fit a {MAX_TYPES}-row table ({len(out)} rows)")
        return TypeTable(out), twin

    def to_c_array(self):
        arr = (TypeParamsC * len(self.rows))()
        for i, r in enumerate(self.rows):
            arr[i] = r.to_c()
        return arr

    def as_oracle_table(self) -> dict:
        """Column arrays holding the fp32-ROUNDED values the device sees (for the test oracle)."""
        out = {}
        for f in fields(TypeParams):
            if f.name == "name":
                continue
            col = [getattr(r, f.name) for r in self.rows]
            if f.name in ("model", "shape"):
                out[f.name] = np.asarray(col, dtype=np.int32)
            else:
                out[f.name] = np.asarray(col, dtype=np.float32).astype(np.float64)
        return out

    @classmethod
    def vehicles(cls, vehicle_model: str = "kinematics") -> "TypeTable":
        """The 9 vehicle templates only (a table without point-mass rows lets the kinematics-only kernel run)."""
        from .participant.element.participant_template import VEHICLE_TEMPLATE

        return cls([TypeParams.vehicle(k, vehicle_model) for k in VEHICLE_TEMPLATE])

    @classmethod
    def from_templates(cls, vehicle_model: str = "kinematics", pedestrian_backend: str = "newton") -> "TypeTable":
        """All 16 template types: 9 vehicles, 3 cyclists, 4 pedestrians (participant_template.py:42-257)."""
        from .participant.element.participant_template import (CYCLIST_TEMPLATE, PEDESTRIAN_TEMPLATE,
                                                               VEHICLE_TEMPLATE)

        rows = [TypeParams.vehicle(k, vehicle_model) for k in VEHICLE_TEMPLATE]
        rows += [TypeParams.cyclist(k) for k in CYCLIST_TEMPLATE]
        rows += [TypeParams.pedestrian(k, pedestrian_backend) for k in PEDESTRIAN_TEMPLATE]
        return cls(rows)
