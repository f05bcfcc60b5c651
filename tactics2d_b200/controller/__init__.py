"""NPC controllers evaluated on the device (``tactics2d.controller`` surface).

``IDMController``, ``AccelerationController``, ``PurePursuitController`` and ``PIDController`` keep the reference's constructor arguments,
attributes, ``update_driving_style`` / ``configure`` and ``step(ego_state, ...) -> (steering, acceleration)``
(tactics2d/controller/*.py).  They are parameter holders: ``BatchedWorld.set_controllers`` turns a list of them into the
controller table of ``t2d_control``, which evaluates every controlled participant of every scenario in one launch;
``step`` on a single ``State`` goes through the same kernel with a batch of one.  ``PIDController`` also carries
per-slot state (``BatchedWorld.pid_state``), which a scenario reset clears.
"""

from .acceleration_controller import AccelerationController
from .controller_base import CTRL_CRUISE, CTRL_EXTERNAL, CTRL_IDM, CTRL_PID, CTRL_PURE_PURSUIT, ControllerBase
from .idm_controller import IDMController
from .pid_controller import PIDController
from .pure_pursuit_controller import PurePursuitController

__all__ = ["ControllerBase", "AccelerationController", "IDMController", "PurePursuitController", "PIDController",
           "CTRL_EXTERNAL", "CTRL_IDM", "CTRL_CRUISE", "CTRL_PURE_PURSUIT", "CTRL_PID"]
