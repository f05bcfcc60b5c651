"""LevelX-series trajectory files (highD, inD, rounD, exiD, uniD) -> participants, and -> pools of initial states.

Follows the reference's ``LevelXParser`` (tactics2d/dataset_parser/parse_levelx.py:20-333): same constructor, ``get_location``,
``get_time_range`` and ``parse_trajectory(file, folder, time_range, ids)`` with the same file naming (``%02d_tracks.csv``,
``%02d_tracksMeta.csv``, ``%02d_recordingMeta.csv``), column names, class / type mapping, 40 ms frames, heading conversion and -
for highD - the bounding-box-centre and lane-marking calibration arithmetic (:248-279).  Differences: pandas replaces polars (not in
this image); the UTM projection the highD calibration needs comes from ``_utm_northing`` below instead of pyproj (not in this image
either; the Krueger series agrees with PROJ's transverse Mercator to well below a millimetre at these latitudes, but that could
not be checked against pyproj here).

``initial_state_pool`` is what the batched path adds: it cuts the parsed log at a list of time stamps into rows of a pool
``x, y, heading, speed, vx, vy [P, M]`` + ``type_id [P, M]`` that ``BatchedWorld.reset(mask, pool, pool_index)`` draws from -
log-seeded resets (SURVEY.md 8f rank 3)."""

from __future__ import annotations

import math
import os
import re
from typing import Tuple, Union

import numpy as np

from ..participant.element import Cyclist, Pedestrian, Vehicle
from ..participant.trajectory import State, Trajectory


def _utm_northing(lon_deg: float, lat_deg: float, zone: int = 31) -> float:
    """Northing of WGS84 (lon, lat) in the given UTM zone (northern-hemisphere convention: no false northing), Krueger's
    n-series to the 6th order - what ``Proj(proj="utm", ellps="WGS84", zone=31)(lon, lat)[1]`` returns (parse_levelx.py:113,119-120)."""
    a, f = 6378137.0, 1 / 298.257223563
    n = f / (2 - f)
    A = a / (1 + n) * (1 + n**2 / 4 + n**4 / 64 + n**6 / 256)
    al = [n / 2 - 2 * n**2 / 3 + 5 * n**3 / 16 + 41 * n**4 / 180 - 127 * n**5 / 288 + 7891 * n**6 / 37800,
          13 * n**2 / 48 - 3 * n**3 / 5 + 557 * n**4 / 1440 + 281 * n**5 / 630 - 1983433 * n**6 / 1935360,
          61 * n**3 / 240 - 103 * n**4 / 140 + 15061 * n**5 / 26880 + 167603 * n**6 / 181440,
          49561 * n**4 / 161280 - 179 * n**5 / 168 + 6601661 * n**6 / 7257600,
          34729 * n**5 / 80640 - 3418889 * n**6 / 1995840,
          212378941 * n**6 / 319334400]
    lat, dlon = math.radians(lat_deg), math.radians(lon_deg - (zone * 6 - 183))
    e = math.sqrt(f * (2 - f))
    t = math.sinh(math.atanh(math.sin(lat)) - e * math.atanh(e * math.sin(lat)))
    xi = math.atan2(t, math.cos(dlon))
    eta = math.atanh(math.sin(dlon) / math.sqrt(1 + t * t))
    y = xi + sum(al[j] * math.sin(2 * (j + 1) * xi) * math.cosh(2 * (j + 1) * eta) for j in range(6))
    return 0.9996 * A * y


class LevelXParser:
    _REGISTERED_DATASET = ["highd", "ind", "round", "exid", "unid"]
    _TYPE_MAPPING = {"car": "car", "Car": "car", "van": "van", "truck": "truck", "Truck": "truck", "truck_bus": "bus", "bus": "bus",
                     "trailer": "trailer", "motorcycle": "motorcycle", "bicycle": "bicycle", "cycle": "bicycle", "pedestrian": "pedestrian"}
    _CLASS_MAPPING = {"car": Vehicle, "Car": Vehicle, "van": Vehicle, "truck": Vehicle, "Truck": Vehicle, "truck_bus": Vehicle, "bus": Vehicle,
                      "trailer": Vehicle, "motorcycle": Cyclist, "bicycle": Cyclist, "cycle": Cyclist, "pedestrian": Pedestrian}
    _HIGHD_BOUNDS = {1: [-0.00025899967, 0], 2: [-0.00018397412, 0], 3: [-0.00021942279, 0], 4: [-0.00024320481, 0],
                     5: [-0.00018558951, 0], 6: [-0.00024051251, 0.0000336538]}   # parse_levelx.py:65-72

    def __init__(self, dataset: str):
        self.dataset = dataset.lower()
        if self.dataset not in self._REGISTERED_DATASET:
            raise KeyError(f"{dataset} is not an available LevelX-series dataset. The available datasets are {self._REGISTERED_DATASET}.")
        self.id_key = "id" if self.dataset == "highd" else "trackId"                 # :110-112
        self.key_length = "width" if self.dataset == "highd" else "length"
        self.key_width = "height" if self.dataset == "highd" else "width"

    def _get_calibrate_params(self, df_meta):   # :116-129
        location = int(df_meta.iloc[0]["locationId"])
        lower_bound = _utm_northing(0.0, self._HIGHD_BOUNDS[location][0])
        upper_bound = _utm_northing(0.0, self._HIGHD_BOUNDS[location][1])
        lower = [float(v) for v in str(df_meta.iloc[0]["lowerLaneMarkings"]).split(";")]
        upper = [float(v) for v in str(df_meta.iloc[0]["upperLaneMarkings"]).split(";")]
        k = (upper_bound - lower_bound) / (upper[0] - lower[-1])
        return k, upper_bound - k * upper[0]

    @staticmethod
    def _get_file_id(file: Union[int, str]) -> int:   # :131-139
        if isinstance(file, str):
            return int(re.findall(r"\d+", file)[0])
        if isinstance(file, int):
            return file
        raise TypeError("The input file must be an integer or a string.")

    def get_location(self, file, folder: str) -> int:
        import pandas as pd

        return pd.read_csv(os.path.join(folder, "%02d_recordingMeta.csv" % self._get_file_id(file))).iloc[0]["locationId"]

    def get_time_range(self, file, folder: str) -> Tuple[int, int]:   # :160-180
        import pandas as pd

        meta = pd.read_csv(os.path.join(folder, "%02d_tracksMeta.csv" % self._get_file_id(file)))
        return int(meta["initialFrame"].min() * 40), int(meta["finalFrame"].max() * 40)

    def _frames(self, file, folder: str, time_range=None, ids=None):
        """The filtered track table with ``time_stamp``, ``heading_``, ``xCenter``, ``yCenter`` columns (:215-279) and the meta table."""
        import pandas as pd

        fid = self._get_file_id(file)
        tracks = pd.read_csv(os.path.join(folder, "%02d_tracks.csv" % fid), low_memory=False)
        meta = pd.read_csv(os.path.join(folder, "%02d_tracksMeta.csv" % fid))
        rec = pd.read_csv(os.path.join(folder, "%02d_recordingMeta.csv" % fid))
        lo, hi = (-np.inf, np.inf) if time_range is None else time_range
        meta = meta[(meta["finalFrame"] * 40 >= lo) & (meta["initialFrame"] * 40 <= hi)]
        if ids is not None:
            meta = meta[meta[self.id_key].isin({int(v) for v in ids})]
        t = tracks[tracks[self.id_key].isin(set(meta[self.id_key]))].copy()
        t["time_stamp"] = t["frame"] * 40
        t = t[(t["time_stamp"] >= lo) & (t["time_stamp"] <= hi)]
        if self.dataset == "highd":
            k, b = self._get_calibrate_params(rec)
            t["heading_"] = np.round(np.arctan2(-t["yVelocity"], t["xVelocity"]), 5)                     # :240-245
            theta = np.round(np.arctan(t["yVelocity"] / t["xVelocity"]), 5)                               # :255-257
            L, W = t[self.key_length], t[self.key_width]
            t["xCenter"] = t["x"] + L * np.cos(theta) / 2 - W * np.sin(theta) / 2                         # :258-270
            t["yCenter"] = (t["y"] + L * np.sin(theta) / 2 + W * np.cos(theta) / 2) * k + b               # :264-274
        else:
            t["heading_"] = t["heading"] * 2 * np.pi / 360                                                 # :246-249
        return t, meta

    def parse_trajectory(self, file, folder: str, time_range: Tuple[int, int] = None, ids: list = None):
        t, meta = self._frames(file, folder, time_range, ids)
        participants = {}
        for _, info in meta.iterrows():                                                                   # :216-237
            id_ = int(info[self.id_key])
            cls = self._CLASS_MAPPING[info["class"]]
            participants[id_] = cls(id_=id_, type_=self._TYPE_MAPPING[info["class"]], length=float(info[self.key_length]),
                                    width=float(info[self.key_width]))
        actual = (int(t["time_stamp"].min()), int(t["time_stamp"].max())) if len(t) else (0, 0)
        for id_, g in t.groupby(self.id_key):                                                             # :284-320
            traj = Trajectory(id_=int(id_), fps=25.0)
            for row in g.sort_values("time_stamp").itertuples(index=False):
                d = row._asdict()
                traj.add_state(State(int(d["time_stamp"]), x=float(d["xCenter"]), y=float(d["yCenter"]), heading=float(d["heading_"]),
                                     vx=float(d["xVelocity"]), vy=float(d["yVelocity"]), ax=float(d["xAcceleration"]),
                                     ay=float(d["yAcceleration"])))
            participants[int(id_)].bind_trajectory(traj)
        return participants, actual


def template_row(rows, cls, length: float, width: float) -> int:
    """The type-table row of a LevelX road user: among the rows of its class (vehicle, cyclist = lf == lr and narrow,
    pedestrian = disc), the one nearest to its logged length and width."""
    kind = {Vehicle: 0, Cyclist: 1, Pedestrian: 2}[cls]
    best, score = 0, np.inf
    for i, r in enumerate(rows):
        r_kind = 2 if r.shape == 1 else (1 if abs(r.lf - r.lr) < 1e-9 and r.half_wid < 0.6 else 0)
        if r_kind != kind:
            continue
        s = abs(2 * (r.radius if r.shape == 1 else r.half_len) - length) + abs(2 * (r.radius if r.shape == 1 else r.half_wid) - width)
        if s < score:
            best, score = i, s
    return best


def initial_state_pool(parser: LevelXParser, file, folder: str, m_participants: int, stamps, type_table=None, ids=None):
    """Rows of initial states for ``BatchedWorld.reset``: row p holds the up-to-``m_participants`` road users present in the
    log at time ``stamps[p]`` (ms; lowest track ids first), the rest of the row is empty slots (type 255).

    Returns ``(pool, type_id, table)``: ``pool`` = dict of float32 arrays ``x, y, heading, speed, vx, vy`` [P, M] (heading wrapped to
    [0, 2 pi), speed = |(vx, vy)| as ``State.speed`` derives it, state.py:143-146), ``type_id`` uint8 [P, M] indexing ``table``
    (default: the template table with one row per LevelX class - vehicles as SingleTrackKinematics, cyclists with lf = lr = L/2,
    pedestrians as PointMass - ``TypeTable.from_templates("kinematics")``; the logged length / width of a track picks the nearest row
    of its class)."""
    from ..types import TYPE_INACTIVE, TypeTable

    t, meta = parser._frames(file, folder, (min(stamps), max(stamps)), ids)
    table = type_table if type_table is not None else TypeTable.from_templates("kinematics")
    rows = table.rows
    cls_of = {int(r[parser.id_key]): (parser._CLASS_MAPPING[r["class"]], float(r[parser.key_length]), float(r[parser.key_width]))
              for _, r in meta.iterrows()}

    type_of = {k: template_row(rows, *v) for k, v in cls_of.items()}
    P, M = len(stamps), int(m_participants)
    pool = {k: np.zeros((P, M), np.float32) for k in ("x", "y", "heading", "speed", "vx", "vy")}
    tid = np.full((P, M), TYPE_INACTIVE, np.uint8)
    by_stamp = {s: g for s, g in t.groupby("time_stamp")}
    for p, s in enumerate(stamps):
        g = by_stamp.get(int(s))
        if g is None:
            continue
        g = g.sort_values(parser.id_key).head(M)
        k = len(g)
        pool["x"][p, :k] = g["xCenter"].to_numpy()
        pool["y"][p, :k] = g["yCenter"].to_numpy()
        pool["heading"][p, :k] = np.mod(g["heading_"].to_numpy(), 2 * np.pi)
        pool["vx"][p, :k] = g["xVelocity"].to_numpy()
        pool["vy"][p, :k] = g["yVelocity"].to_numpy()
        pool["speed"][p, :k] = np.hypot(g["xVelocity"].to_numpy(), g["yVelocity"].to_numpy())
        tid[p, :k] = [type_of[int(i)] for i in g[parser.id_key]]
    return pool, tid, table
