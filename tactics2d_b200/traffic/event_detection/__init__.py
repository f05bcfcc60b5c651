"""Detectors on this hot path (reference ``tactics2d/traffic/event_detection/__init__.py:7-26``), including the
IoU based ``Arrival`` / ``NoAction`` (SURVEY.md section 8(f) rank 2) and ``OffRoute`` against a route per slot
(``BatchedWorld.set_routes``).  ``OffLane`` is a stub in the reference and is not built here."""

from .detectors import Arrival, DynamicCollision, NoAction, OffRoute, OutBound, StaticCollision, TimeExceed
from .event_base import EventBase

__all__ = ["EventBase", "DynamicCollision", "StaticCollision", "OutBound", "TimeExceed", "Arrival", "NoAction", "OffRoute"]
