"""Static map geometry for the batched tick: Lanelet2-OSM -> collidable segment tiles.

The kernels take the scenario's static geometry as a flat tile ``float32 [S, 4] = (x1, y1, x2, y2)``
plus the out-of-bound box.  This module is the (offline, host-side) compiler from the reference's
on-disk format to that tile; it follows the reference's own parsing rules:

* node projection without pyproj: ``x = (lon - lon0) * 111320 * cos(lat0)``, ``y = (lat - lat0) * 110540``
  with the first non-deleted node as origin   (tactics2d/map/parser/parse_osm.py:259-278, :589-597);
* a Lanelet2 ``way`` is a RoadLine whose geometry is the LineString of its ``nd`` refs in order and
  whose ``type`` / ``subtype`` tags classify it                       (parse_osm.py:384-403, :82-120);
* barrier kinds (no lane change, physically blocking): type ``curbstone`` / ``road_border`` and
  ``guard_rail`` / ``wall`` / ``fence`` ...                     (tactics2d/map/element/roadline.py:107-123);
* ``Map.boundary`` = (floor(xmin), ceil(xmax), floor(ymin), ceil(ymax)) over all nodes
                                                              (tactics2d/map/element/map.py:92-167);
* a Lanelet2 ``multipolygon`` / ``area`` relation is an Area: its ``outer`` member ways chained end to end into the
  exterior ring, its ``inner`` member ways chained into holes, a new hole starting whenever the current one closes
                                                              (parse_osm.py:461-510, chaining rule :37-60).

The tiles of the reference's 13 bundled maps (``data/{highD,inD,rounD}_map/*.osm``) are compiled once in
advance (``python -m tactics2d_b200.map <reference>/data`` -> ``tactics2d_b200/map/tiles/*.npz``) and ship with the
package, so that nothing at run time needs the reference's map files.
"""

from __future__ import annotations

import math
import os
import xml.etree.ElementTree as ET
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

TILE_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tiles")

# RoadLine kinds that are physical structures a vehicle cannot drive through.  The reference gives every one of them the
# lane-change rule (False, False): type curbstone / road_border at roadline.py:109-110, subtypes guard_rail, wall, fence,
# jersey_barrier, gate, door, rail at roadline.py:111-124.  The PAINTED members of that same list (zebra_marking,
# pedestrian_marking, bike_marking, keepout, roadline.py:115-118) carry the same rule but are not obstacles and stay out.
BARRIER_TYPES = ("curbstone", "road_border", "guard_rail", "wall", "fence", "jersey_barrier", "gate", "door", "rail")


@dataclass
class Way:
    id_: int
    type_: Optional[str]
    subtype: Optional[str]
    points: np.ndarray   # float64 [P, 2]


@dataclass
class Area:
    """One static object of ``StaticCollision`` (``Area.geometry`` = Polygon(outer, inners), area.py:13-125).  Rings are
    stored without the repeated closing vertex; ``closed`` says whether the chained outer ways met their own start
    (the reference only warns when they do not, parse_osm.py:491-492, and shapely closes the ring itself)."""
    id_: int
    type_: Optional[str]
    subtype: Optional[str]
    outer: np.ndarray            # float64 [V, 2]
    inners: List[np.ndarray]     # each float64 [W, 2]
    closed: bool = True


@dataclass
class OsmMap:
    nodes: Dict[int, Tuple[float, float]]
    ways: List[Way]
    areas: List[Area] = field(default_factory=list)

    @property
    def boundary(self) -> Tuple[float, float, float, float]:
        """Map.boundary, map.py:92-167."""
        if not self.nodes:
            return (0.0, 0.0, 0.0, 0.0)
        xy = np.asarray(list(self.nodes.values()), dtype=np.float64)
        return (float(np.floor(xy[:, 0].min())), float(np.ceil(xy[:, 0].max())), float(np.floor(xy[:, 1].min())),
                float(np.ceil(xy[:, 1].max())))


def parse_osm_lanelet2(path: str) -> OsmMap:
    """OSMParser(lanelet2=True).parse without a projector (parse_osm.py:536-619): nodes and ways only."""
    root = ET.parse(path).getroot()
    all_nodes = [n for n in root.findall("node") if n.get("action") != "delete"]
    lat0 = float(all_nodes[0].attrib["lat"]) if all_nodes else 0.0
    lon0 = float(all_nodes[0].attrib["lon"]) if all_nodes else 0.0
    k = 111320.0 * math.cos(math.radians(lat0))
    nodes = {int(n.attrib["id"]): ((float(n.attrib["lon"]) - lon0) * k, (float(n.attrib["lat"]) - lat0) * 110540.0)
             for n in all_nodes}
    ways = []
    for w in root.findall("way"):
        if w.get("action") == "delete":
            continue
        tags = {t.attrib["k"]: t.attrib["v"] for t in w.findall("tag")}
        pts = np.asarray([nodes[int(nd.attrib["ref"])] for nd in w.findall("nd")], dtype=np.float64).reshape(-1, 2)
        ways.append(Way(int(w.attrib["id"]), tags.get("type"), tags.get("subtype"), pts))
    by_id = {w.id_: w for w in ways}
    areas = []
    for rel in root.findall("relation"):
        if rel.get("action") == "delete":
            continue
        tags = {t.attrib["k"]: t.attrib["v"] for t in rel.findall("tag")}
        if not any(v in ("multipolygon", "area") for v in tags.values()):   # parse_osm.py:608-612 looks at every tag value
            continue
        areas.append(_chain_area(rel, tags, by_id))
    return OsmMap(nodes, ways, areas)


def _chain(chain: list, nxt: list, rel_id: int) -> None:
    """Append the way ``nxt`` to the open ring ``chain`` wherever the two share an end point, turning either around if
    that is what makes them meet (the four cases of parse_osm.py:48-60); ways that do not touch are a SyntaxError there
    and here."""
    if chain[-1] == nxt[0]:
        pass
    elif chain[0] == nxt[0]:
        chain.reverse()
    elif chain[0] == nxt[-1]:
        chain.reverse()
        nxt.reverse()
    elif chain[-1] == nxt[-1]:
        nxt.reverse()
    else:
        raise SyntaxError(f"the member ways of relation {rel_id} do not form a continuous ring")
    chain += nxt[1:]


def _chain_area(rel: ET.Element, tags: Dict[str, str], ways: Dict[int, Way]) -> Area:
    """``_load_area_lanelet2`` (parse_osm.py:461-510)."""
    rel_id = int(rel.attrib["id"])
    members = {"outer": [], "inner": []}
    for m in rel.findall("member"):
        if m.attrib.get("role") in members:
            members[m.attrib["role"]].append(int(m.attrib["ref"]))

    def pts(way_id):
        return [tuple(p) for p in ways[way_id].points.tolist()]

    if not members["outer"]:
        raise IndexError(f"area relation {rel_id} has no outer member")    # line_ids["outer"][0], parse_osm.py:485
    outer = pts(members["outer"][0])
    for wid in members["outer"][1:]:
        _chain(outer, pts(wid), rel_id)
    closed = outer[0] == outer[-1]
    rings, cur = [], []
    for wid in members["inner"]:
        if not cur:
            cur = pts(wid)
        else:
            _chain(cur, pts(wid), rel_id)
        if cur[0] == cur[-1]:
            rings.append(cur)
            cur = []
    if cur:
        rings.append(cur)

    def ring(points):
        v = np.asarray(points, dtype=np.float64).reshape(-1, 2)
        return v[:-1] if len(v) >= 2 and np.array_equal(v[0], v[-1]) else v

    return Area(rel_id, tags.get("type"), tags.get("subtype"), ring(outer), [ring(r) for r in rings], bool(closed))


def collidable_segments(map_: OsmMap, barrier_types: Sequence[str] = BARRIER_TYPES, solid_lines: Optional[bool] = None) -> np.ndarray:
    """Flatten the blocking RoadLines into segments, ways in file order, pieces in vertex order.

    ``solid_lines``: also treat ``subtype == "solid"`` markings as the road edge; default = only when the map
    has no barrier-type way at all (the highD maps are nothing but ``line_thin`` solid/dashed markings)."""
    def blocking(w):
        return (w.type_ in barrier_types) or (w.subtype in barrier_types)

    if solid_lines is None:
        solid_lines = not any(blocking(w) for w in map_.ways)
    segs = []
    for w in map_.ways:
        if not (blocking(w) or (solid_lines and w.subtype == "solid")):
            continue
        for a, b in zip(w.points[:-1], w.points[1:]):
            segs.append((a[0], a[1], b[0], b[1]))
    return np.asarray(segs, dtype=np.float32).reshape(-1, 4)


def compile_tiles(src_root: str, out_dir: str = TILE_DIR) -> List[str]:
    """Compile every ``*.osm`` below ``src_root`` into ``out_dir/<name>.npz`` (segments, bounds, counts)."""
    os.makedirs(out_dir, exist_ok=True)
    written = []
    for d, _, files in sorted(os.walk(src_root)):
        for f in sorted(files):
            if not f.endswith(".osm"):
                continue
            m = parse_osm_lanelet2(os.path.join(d, f))
            seg = collidable_segments(m)
            n_all = int(sum(max(0, len(w.points) - 1) for w in m.ways))
            name = f[:-4]
            rings = [r for a in m.areas for r in [a.outer] + a.inners]
            np.savez(os.path.join(out_dir, name + ".npz"), segments=seg, bounds=np.asarray(m.boundary, dtype=np.float32),
                     n_all_segments=n_all, n_ways=len(m.ways),
                     # the Areas: ring vertices back to back, ring r = area_xy[area_ring_start[r] : area_ring_start[r + 1]],
                     # area a owns rings [area_first_ring[a], area_first_ring[a + 1]), the first of them its exterior
                     area_xy=np.concatenate(rings, 0) if rings else np.zeros((0, 2), np.float64),
                     area_ring_start=np.cumsum([0] + [len(r) for r in rings]).astype(np.int32),
                     area_first_ring=np.cumsum([0] + [1 + len(a.inners) for a in m.areas]).astype(np.int32),
                     area_id=np.asarray([a.id_ for a in m.areas], dtype=np.int64),
                     area_subtype=np.asarray([a.subtype or "" for a in m.areas], dtype="U32"),
                     area_type=np.asarray([a.type_ or "" for a in m.areas], dtype="U32"),
                     area_closed=np.asarray([a.closed for a in m.areas], dtype=bool))
            written.append(name)
    return written


def load_collidable_segments(name: str):
    """(segments float32 [S, 4], bounds (xmin, xmax, ymin, ymax)) of a packaged tile, e.g. ``"inD_1"``."""
    path = os.path.join(TILE_DIR, name + ".npz")
    if not os.path.exists(path):
        raise FileNotFoundError(f"map tile {name!r} not found in {TILE_DIR}; compile it with `python -m tactics2d_b200.map <osm dir>`")
    z = np.load(path)
    return np.ascontiguousarray(z["segments"], dtype=np.float32), tuple(float(v) for v in z["bounds"])


def load_areas(name: str, subtypes: Optional[Sequence[str]] = None) -> List[Area]:
    """The Areas of a packaged map in file order - the list an env hands to ``StaticCollision.reset`` (the parking env
    passes every area but the target, envs/parking.py:438-440).  ``subtypes``: keep only these (e.g. ``("vegetation",
    "traffic_island")``); None keeps all."""
    path = os.path.join(TILE_DIR, name + ".npz")
    if not os.path.exists(path):
        raise FileNotFoundError(f"map tile {name!r} not found in {TILE_DIR}; compile it with `python -m tactics2d_b200.map <osm dir>`")
    z = np.load(path)
    xy, rs, fr = z["area_xy"], z["area_ring_start"], z["area_first_ring"]
    out = []
    for a in range(len(z["area_id"])):
        sub = str(z["area_subtype"][a]) or None
        if subtypes is not None and sub not in subtypes:
            continue
        rings = [np.array(xy[rs[r]:rs[r + 1]], dtype=np.float64) for r in range(fr[a], fr[a + 1])]
        out.append(Area(int(z["area_id"][a]), str(z["area_type"][a]) or None, sub, rings[0], rings[1:], bool(z["area_closed"][a])))
    return out


def list_tiles() -> List[str]:
    return sorted(f[:-4] for f in os.listdir(TILE_DIR) if f.endswith(".npz")) if os.path.isdir(TILE_DIR) else []


def polygons_to_segments(polygons, polylines=()):
    """Flatten static objects into the tile format of ``BatchedWorld.set_map`` / ``set_map_table``.

    ``polygons``: in the order ``StaticCollision.reset`` receives the areas, each either a [V, 2] vertex array
    (``Area.geometry.exterior``, with or without the repeated closing vertex) or an ``Area`` (exterior plus holes);
    ``polylines``: list of [V, 2] arrays (``RoadLine.geometry``), appended after them.  Returns ``(segments [S, 4] float32,
    poly_start [P + 1] int32)``: object p = segments [poly_start[p], poly_start[p + 1]), its rings back to back, every ring
    closed on itself.  An object with holes needs nothing more: a pose intersects ``Polygon(outer, holes)`` when it crosses
    any edge of any ring, or touches none and its centre is inside the exterior and outside every hole - which is the
    parity of the edges of all the rings together that a ray from the centre crosses."""
    segs, starts = [], [0]

    def ring_edges(ring):
        v = np.asarray(ring, dtype=np.float32).reshape(-1, 2)
        if len(v) >= 2 and np.array_equal(v[0], v[-1]):
            v = v[:-1]
        if len(v) < 3:
            raise ValueError("a polygon ring needs at least 3 vertices")
        return np.concatenate([v, np.roll(v, -1, axis=0)], 1)

    for poly in polygons:
        rings = [poly.outer] + list(poly.inners) if isinstance(poly, Area) else [poly]
        edges = [ring_edges(r) for r in rings]
        segs.extend(edges)
        starts.append(starts[-1] + sum(len(e) for e in edges))
    for line in polylines:
        v = np.asarray(line, dtype=np.float32).reshape(-1, 2)
        if len(v) >= 2:
            segs.append(np.concatenate([v[:-1], v[1:]], 1))
    seg = np.concatenate(segs, 0).astype(np.float32) if segs else np.zeros((0, 4), np.float32)
    return np.ascontiguousarray(seg), np.asarray(starts, dtype=np.int32)


def area_style_key(area: Area) -> str:
    """The BEV style key of an Area as ``BEVCamera._get_type`` picks it (sensor/camera.py:56-87): its subtype, else its
    type, else ``"area"``.  A key without a row in ``sensor.camera.BEV_STYLES`` draws as ``"area"``."""
    from ..sensor.camera import BEV_STYLES

    key = area.subtype or area.type_ or "area"
    return key if key in BEV_STYLES else "area"


def segment_style_keys(polygons, polylines=(), polyline_key: str = "road_border"):
    """Per-segment BEV style keys in the layout :func:`polygons_to_segments` returns for the same arguments: every
    edge of an Area gets :func:`area_style_key` (a bare vertex array: ``"obstacle"``), every polyline piece
    ``polyline_key``.  Pass the result as the ``"style"`` of a tile (``BatchedWorld.set_map`` / ``set_map_table``)."""
    seg, ps = polygons_to_segments(polygons, polylines)
    keys = []
    for p, poly in enumerate(polygons):
        k = area_style_key(poly) if isinstance(poly, Area) else "obstacle"
        keys += [k] * int(ps[p + 1] - ps[p])
    keys += [polyline_key] * (len(seg) - len(keys))
    return keys
