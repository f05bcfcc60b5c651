"""``Trajectory``: the time-ordered states of one participant.

Interface and error behaviour of the reference's ``tactics2d/participant/trajectory/trajectory.py:15-188``:
``add_state`` raises ``ValueError`` for a non-State and ``KeyError`` when time goes backwards (:127-138),
warns and overwrites when the frame already exists, flips ``stable_freq`` when the sampling interval
changes (:139-144); ``reset(state, keep_history)`` as :170-188.  (One deliberate deviation: overwriting an
existing frame does not append the frame a second time to ``frames``.)

The batched engine keeps the current state of every participant in HBM and, with ``BatchedWorld.set_history``, a
ring of its last H states on the device (DESIGN.md section 1 "Trajectory history"); ``BatchedWorld.trajectory(n, m)``
reads a slot's valid entries back as a Trajectory.  A Trajectory is also the host-side history of the
reference-shaped participant objects.
"""

from __future__ import annotations

import logging
from typing import Any, List, Tuple

import numpy as np

from .state import State


class Trajectory:
    def __init__(self, id_: Any, fps: float = None, stable_freq: bool = True):
        self.id_ = id_
        self.fps = fps
        self.stable_freq = stable_freq
        self._states = {}
        self._frames: List[int] = []
        self._current_state = None

    def __len__(self):
        return len(self._frames)

    @property
    def frames(self) -> List[int]:
        return self._frames

    @property
    def history_states(self) -> dict:
        return self._states

    @property
    def initial_state(self):
        return self._states[self._frames[0]] if self._frames else None

    @property
    def last_state(self):
        return self._states[self._frames[-1]] if self._frames else None

    @property
    def first_frame(self):
        return self._frames[0] if self._frames else None

    @property
    def last_frame(self):
        return self._frames[-1] if self._frames else None

    @property
    def current_state(self):
        return self._current_state

    @property
    def average_speed(self):
        speeds = [s.speed for s in self._states.values()]
        return float(np.mean(speeds)) if speeds else float("nan")

    def has_state(self, frame: int) -> bool:
        return frame in self._states

    def get_state(self, frame: int = None) -> State:
        if frame is None:
            return self._current_state
        if frame not in self._states:
            raise KeyError(f"Time stamp {frame} is not found in the trajectory {self.id_}.")
        return self._states[frame]

    def add_state(self, state: State):
        if not isinstance(state, State):
            raise ValueError("The input state is not a valid State object.")
        if self._frames and state.frame < self._frames[-1]:
            raise KeyError(f"Trying to insert an early time stamp {state.frame} happening before the last stamp "
                           f"{self._frames[-1]} in trajectory {self.id_}")
        if state.frame in self._states:
            logging.warning(f"State at time stamp {state.frame} is already in trajectory {self.id_}. It will be overwritten.")
            self._states[state.frame] = state
            self._current_state = state
            return
        if len(self._frames) > 1 and self.stable_freq:
            if state.frame - self._frames[-1] != self._frames[-1] - self._frames[-2]:
                self.stable_freq = False
                logging.warning(f"The time interval of the trajectory {self.id_} is uneven.")
        self._frames.append(state.frame)
        self._states[state.frame] = state
        self._current_state = state

    append_state = add_state

    def get_trace(self, frame_range: Tuple[int, int] = None) -> list:
        if not self._frames:
            return []
        lo = self.first_frame if frame_range is None else frame_range[0]
        hi = self.last_frame if frame_range is None else frame_range[1]
        return [self._states[f].location for f in self._frames if lo <= f <= hi]

    def reset(self, state: State = None, keep_history: bool = False):
        if state is None:
            first = self.initial_state
            if keep_history:
                self._current_state = first
                return
            state = first
        self._states.clear()
        self._frames.clear()
        self.add_state(state)
