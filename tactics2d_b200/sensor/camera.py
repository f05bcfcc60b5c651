"""``BEVCamera``: the bird's-eye-view observation of every scenario's ego, rendered on the device.

The reference's ``BEVCamera.update`` (``tactics2d/sensor/camera.py:333-386``) returns geometry dicts that a
``MatplotlibRenderer`` then draws into the 200 x 200 x 3 ``uint8`` observation of ``ParkingEnv`` / ``RacingEnv``
(``envs/parking.py:130``).  This class returns the rendered batch instead: ``render(world)`` is one launch of the
K6 kernel (``t2d_bev_render``) and yields ``uint8 [N, H, W, 3]``; ``render_agents(world, observers)`` renders the same view
from every observer row (``t2d_bev_render_agents``) as ``uint8 [N, Q, H, W, 3]``.  The drawing contract, and where it deliberately
differs from the reference's renderer, is DESIGN.md section 1 "BEV observation".

``BEV_STYLES`` restates the rows of the reference's style tables that this renderer uses, as
``key: (colour, z order, stroke width in points)``.  Rows 0-3 have fixed meanings in the C ABI: background, heading
arrow, default style of a map ring object and of an open map segment.
"""

from __future__ import annotations

from typing import Sequence, Tuple, Union

BEV_STYLES = {
    "background": ("#ffffff", -128, 1.0),      # the figure's white face
    "heading_arrow": ("#2f3542", 7, 1.0),      # camera.py:283-297 colour black; matplotlib_config.py:28,154
    "obstacle": ("#b2bec3", 5, 1.0),           # matplotlib_config.py:26,79,144
    "road_border": ("#a5b1c2", 4, 1.0),        # :25,84,149; width 1 pt, camera.py:190
    "area": ("#2f3542", 2, 1.0),               # :28,68,135
    "parking": ("#2f3542", 3, 1.0),            # :28,70,137
    "vegetation": ("#20bf6b", 3, 1.0),         # :14,74,140
    "keepout": ("#fc5c65", 3, 1.0),            # :8,75,141
    "traffic_island": ("#4b6584", 3, 1.0),     # :27,78,143
    "building": ("#b2bec3", 5, 1.0),           # :26,77,142
    "roadline": ("#f1f2f6", 4, 1.0),           # :24,81,146; width 1 pt, camera.py:190
    "curbstone": ("#a5b1c2", 5, 0.5),          # :25,83,150; width 0.5 pt, camera.py:191-192
    "vehicle": ("#2bcbba", 6, 1.0),            # :17,86,151
    "cyclist": ("#fd9644", 6, 1.0),            # :11,91,159
    "pedestrian": ("#45aaf2", 6, 1.0),         # :19,94,162
    # generate_parking_lot.py:40,114 colours the target area #EE766E; "target_area" is in neither table, so
    # _resolve_style gives it z order 1
    "target_area": ("#EE766E", 1, 1.0),
}
STYLE_KEYS = list(BEV_STYLES)
NOT_DRAWN = 255


def style_rgb(key: str) -> Tuple[int, int, int]:
    h = BEV_STYLES[key][0].lstrip("#")
    return int(h[0:2], 16), int(h[2:4], 16), int(h[4:6], 16)


def palette():
    """uint8 [len(BEV_STYLES), 3]: the colour of every style index (RGB output = palette[class output])."""
    import numpy as np

    return np.asarray([style_rgb(k) for k in STYLE_KEYS], dtype=np.uint8)


def default_type_style(row) -> Union[str, None]:
    """The style key of a type-table row, by its template name (camera.py:56-87 types participants by class):
    vehicle / cyclist / pedestrian templates, ``obstacle`` -> not drawn (camera.py:318-319); other names fall back on
    the collision shape (box -> vehicle, disc -> pedestrian, none -> not drawn)."""
    from ..participant.element.participant_template import CYCLIST_TEMPLATE, PEDESTRIAN_TEMPLATE, VEHICLE_TEMPLATE
    from ..types import SHAPE_CIRCLE, SHAPE_NONE

    if row.shape == SHAPE_NONE or row.name == "obstacle":
        return None
    if row.name in VEHICLE_TEMPLATE:
        return "vehicle"
    if row.name in CYCLIST_TEMPLATE:
        return "cyclist"
    if row.name in PEDESTRIAN_TEMPLATE:
        return "pedestrian"
    return "pedestrian" if row.shape == SHAPE_CIRCLE else "vehicle"


class BEVCamera:
    """Bird's-eye view of participant ``id_`` (only the ego, participant 0, is supported) of every scenario.

    ``perception_range``: a scalar R or ``(left, right, front, back)`` in metres (camera.py:31-38); ``resolution``:
    ``(width, height)`` in pixels (the reference's default ``(200, 200)``, envs/parking.py:412-416)."""

    def __init__(self, id_: int = 0, perception_range: Union[float, Sequence[float]] = 20.0,
                 resolution: Tuple[int, int] = (200, 200)):
        if id_ != 0:
            raise ValueError("the batched BEV camera is mounted on the ego, participant 0")
        self.id_ = id_
        self.perception_range = perception_range
        self.resolution = (int(resolution[0]), int(resolution[1]))
        self.observation = None

    def render(self, world, rgb: bool = True):
        """``uint8 [N, H, W, 3]`` (``rgb``) or the style indices ``uint8 [N, H, W]``; a view of a buffer the world
        reuses on the next render of the same shape."""
        self.observation = world.bev(self.resolution, self.perception_range, rgb=rgb)
        return self.observation

    def render_agents(self, world, observers=None, goals=None, rgb: bool = True):
        """This camera's view bound to every observer row's slot (``BatchedWorld.bev_agents``; DESIGN.md section 1
        "Per-agent BEV"): ``uint8 [N, Q, H, W, 3]`` (``rgb``) or ``[N, Q, H, W]`` style indices.  ``observers`` int16
        ``[N, Q]`` and ``goals`` fp32 ``[N, Q, 5]`` as in ``BatchedWorld.observe_agents``; an absent row is all
        background.  A view of a buffer the world reuses on the next call with the same shape."""
        self.observation = world.bev_agents(self.resolution, self.perception_range, rgb=rgb, observers=observers,
                                            goals=goals)
        return self.observation
