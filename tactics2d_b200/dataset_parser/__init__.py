"""Dataset parsers on the path's input side: logged trajectories -> initial-state pools for ``BatchedWorld.reset``, and
recorded tracks for log replay (``BatchedWorld.set_log``)."""
from .parse_levelx import LevelXParser, initial_state_pool  # noqa: F401
from .replay import ReplayEpisodes, ReplayLog, build_replay_episodes  # noqa: F401
