"""tactics2d_b200 - a GPU-native (H100, sm_90a) batched ``env.step()`` for tactics2d.

One hot path, built from scratch for sm_90a behind the reference's class surface:
per-participant physics (``tactics2d.physics``), pose (``tactics2d.participant``), collision /
out-of-bound / time-limit events (``tactics2d.traffic``) and the Gym-style batched step/reset
(``tactics2d.envs``), for N scenarios x M participants per call.  Host code is Python over a
C ABI (``include/t2d_b200.h``, ``ctypes``); PyTorch tensors are only the device-memory container.
"""

__version__ = "0.1.0"

from . import _lib  # noqa: F401
from .types import (  # noqa: F401
    MODEL_DYNAMICS, MODEL_KINEMATICS, MODEL_POINTMASS_EULER, MODEL_POINTMASS_NEWTON, MODEL_STATIC,
    SHAPE_CIRCLE, SHAPE_NONE, SHAPE_OBB, TYPE_INACTIVE, TypeParams, TypeTable)
from .world import (  # noqa: F401
    AGENT_FIELDS, EGO_FIELDS, GOAL_FIELDS, HIST_FIELDS, SEGMENT_FIELDS, AgentEnvResult, AgentObservation, BatchedWorld, StepResult,
    VectorObservation, vector_obs_width)
