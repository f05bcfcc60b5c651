"""``BatchedTrafficEnv`` - Gym-style ``step`` / ``reset`` over N scenarios x M participants.

Keeps the contract of the reference's single-ego envs (``tactics2d/envs/parking.py:219-298``,
``racing.py:145-202``):

* ``reset(seed, options) -> (observation, info)``; ``step(action) -> (observation, reward, terminated,
  truncated, info)``;
* the action order is ``[steering, accel]`` (parking.py:239); out-of-range actions are clipped by the physics
  model, not rejected (single_track_kinematics.py:192-193);
* ``terminated`` iff the scenario status is COMPLETED; ``truncated`` iff the scenario or the ego's traffic
  status is not NORMAL (parking.py:243-248); without a ``target`` a scenario never completes, so every ``done``
  is a truncation;
* the status priority time-exceed -> out-of-bound -> collision (parking.py:361-392);
* the reward chain of ``ParkingEnv._get_reward`` (parking.py:148-190), in its order: -5 collision, -1 time exceeded / no
  action, -5 out of bound, +5 completed, else the time penalty ``-tanh(t / max_step) * 0.001`` + the IoU gain over the
  episode's best + 0.1 x the progress towards the target centre (``_max_iou`` / ``_min_dist_to_target`` are kept per
  scenario on the device).  Two deliberate differences, both where the reference misbehaves: its check_status stores
  NO_ACTION into the *traffic* status (parking.py:372), here it is a scenario status and earns the -1 the reward chain
  intends; its first step adds ``(inf - d) * 0.1`` to the reward, here the first step only records the distance.

What differs, deliberately: the environment is *vectorised* (every quantity has a leading N axis and lives on
the GPU), all M participants are simulated (the ego is participant 0; the others take ``npc_action`` or zeros),
the observation is the state tensors themselves by default, with ``observation="bev"`` the reference's bird's-eye
view image of every ego rendered on the device (``BatchedWorld.bev``), or with ``observation="vector"`` the ego-frame vector
of its motion, goal, nearest participants and nearest map segments (``BatchedWorld.observe``), and scenarios are drawn from a pool of initial states instead of the reference's map generators.
The reference envs construct a ``render_manager`` that is commented out at this commit and crash on the
first ``update`` (SURVEY.md section 3.4); this class follows their documented contract, not the crash.
"""

from __future__ import annotations

from typing import Optional

import numpy as np

from ..traffic import BatchedScenarioManager, ScenarioStatus, TrafficStatus
from ..world import BatchedWorld


class InvalidAction(Exception):
    """Raised when an action does not have the batched action shape (parking.py:235-236 raises it for
    actions outside the action space)."""


class BatchedTrafficEnv:
    metadata = {"render_modes": []}

    def __init__(self, scene, device="cuda:0", max_step: int = 1000, step_size: int = 100, delta_t: int = 5,
                 any_participant: bool = False, auto_reset: bool = True, target=None, arrival_threshold: float = 0.95,
                 no_action_max_step: int = 100, observation: str = "state", bev_resolution=(200, 200),
                 bev_range=(20.0, 20.0, 20.0, 20.0), replay=None, vector_obs: Optional[dict] = None,
                 agent_rewards: bool = False, agent_actions: bool = False, lidar: Optional[dict] = None,
                 route: Optional[dict] = None, sampler: Optional[dict] = None, history: Optional[dict] = None,
                 camera: Optional[dict] = None, leaders: Optional[dict] = None, lane_change: Optional[dict] = None,
                 reactive: Optional[dict] = None, yielding: Optional[dict] = None):
        """``scene``: a :class:`tactics2d_b200.synthetic.Scene` (initial states, types, map tile, bounds);
        ``replay``: optional :class:`tactics2d_b200.dataset_parser.ReplayEpisodes` - one scenario per episode row, the
        ego (participant 0) driven by the policy and the other slots by the recording (``BatchedWorld.set_log``); the
        initial states and the type table then come from it and only the map and bounds from ``scene`` (which may be None);
        an auto-reset restarts the scenario's row, ``reset(options={"shuffle": True})`` deals the rows out anew; episodes
        with slot schedules (``build_replay_episodes(..., reuse_slots=True)``) add ``info["track"]``, the int32 [N, M]
        track each slot shows after the step's auto-reset (``BatchedWorld.replay_track``);
        ``target``: optional [N, 5] target areas (cx, cy, heading, half_len, half_wid) for the egos - enables the
        ``Arrival`` (-> COMPLETED / ``terminated``) and ``NoAction`` detectors and the IoU reward terms of
        ``ParkingEnv._get_reward`` (parking.py:148-190); ``observation``: ``"state"`` (the state tensors) or ``"bev"``
        (``uint8 [N, H, W, 3]``, the view of ``BatchedWorld.bev(bev_resolution, bev_range)``, rendered after the
        auto-reset so that a finished scenario shows its new episode; one more launch per step) or ``"vector"`` (fp32 [N, F], the
        ``flat`` row of ``BatchedWorld.observe(**vector_obs)``, also computed after the auto-reset; ``vector_obs`` takes its
        keyword arguments ``k_agents``, ``k_segments``, ``agent_range``, ``segment_range``) or ``"agents"`` (fp32 [N, Q, F],
        the ``flat`` rows of ``BatchedWorld.observe_agents(**vector_obs)``, one per observer slot, for multi-agent control,
        also computed after the auto-reset; ``vector_obs`` may then also hold ``observers`` and ``goals``);
        ``agent_rewards``: with ``observation="agents"``, score every observer row as an agent (``BatchedWorld.set_agents``
        with the same ``observers`` / ``goals``, ``arrival_threshold`` and ``no_action_max_step``): ``step`` returns
        ``[N, Q]`` reward / terminated / truncated, ``info`` adds ``agent_status`` and ``agent_iou``, a settled agent's slot
        leaves the world until its scenario resets, and a scenario auto-resets when none of its agents is NORMAL.  The
        per-row goals replace ``target``, which is then rejected;
        ``agent_actions``: with ``observation="agents"``, ``step`` takes one (steering, accel) per observer row, ``[N, Q,
        2]``, and scatters it on the device into the slots the rows observe (``BatchedWorld.scatter_agent_action``; the
        lowest row naming a slot wins, empty and retired slots take nothing);
        ``lidar``: e.g. ``dict(n_beams=360, max_range=20.0)`` (``ParkingEnv``'s lidar, parking.py:303-304) adds
        ``info["lidar"]`` to ``reset`` and ``step``, the reference env's ``infos["lidar"]`` (parking.py:206-217), scanned
        after the auto-reset like the observation: fp32 ``[N, n_beams]`` from every ego (``BatchedWorld.lidar_scan``), or
        with ``observation="agents"`` ``[N, Q, n_beams]`` from every observer row (``BatchedWorld.lidar_scan_agents`` on
        ``vector_obs["observers"]``);
        ``route``: e.g. ``dict(paths=[...], route_id=..., threshold=3.0)`` gives participants a route to follow
        (``BatchedWorld.set_paths`` + ``set_routes``; DESIGN.md section 1 "Route following"): ``route_id`` indexes ``paths``
        per pool row, ``[P, M]`` or ``[P]`` for the ego only (-1: none); ``threshold`` is the ``OffRoute`` distance,
        ``progress_weight`` (0.1) and ``off_route_reward`` (-5) the reward terms; an off-route ego or agent row is
        truncated.  The routes follow their rows like the types do (an auto-reset keeps a scenario's route; a shuffle of a
        replay deals them out with the rows).  ``info["route"]`` is the route observation after the auto-reset
        (``BatchedWorld.route_observe`` with ``n_points`` (8) and ``spacing`` (2.0)): ``[N, F]`` from every ego, or with
        ``observation="agents"`` ``[N, Q, F]`` from every observer row;
        ``sampler``: e.g. ``dict(seed=0, jitter=..., tries=8, sample_rows=True, avoid_target=False)`` draws every episode
        (``BatchedWorld.set_reset_sampler``; DESIGN.md section 1 "Sampled resets"; envs/parking.py:397-441): every reset
        and auto-reset runs a pool row drawn from a seeded stream and moves the start states by ``jitter`` ([M, 4, 2]
        ranges) where the move is collision-free; the row's types, ``target`` and routes follow it.  ``reset(seed=s)``
        re-keys the stream and restarts the episode counters, ``reset()`` keeps drawing; ``info["pool_row"]`` is the row
        each scenario runs after the step's auto-reset.  A shuffle is then rejected, as are jitter on the replayed slots
        (with ``replay``, only slot 0 may move) and per-row goals with ``sample_rows`` (they belong to scenarios, not rows);
        ``history``: e.g. ``dict(length=16)`` keeps the last ``length`` states of every slot on the device
        (``BatchedWorld.set_history``; DESIGN.md section 1 "Trajectory history") and adds ``info["history"]`` to ``reset``
        and ``step``, computed after the auto-reset like the observation (``BatchedWorld.observe_history``): with
        ``observation="vector"`` the ego's past and that of the agents of its observation (``[N, 1 + K, H, 7]``), with
        ``"agents"`` every observer row's and its agents' (``[N, Q, 1 + K, H, 7]``), else the ego's own past
        (``[N, 1, H, 7]``).  A scenario that auto-reset shows one valid entry per present slot, its new start state;
        ``camera``: e.g. ``dict(resolution=(200, 200), perception_range=20.0, rgb=True)`` adds ``info["bev"]`` to ``reset``
        and ``step``, rendered after the auto-reset like the lidar: with ``observation="agents"`` ``uint8 [N, Q, H, W(,
        3)]`` from every observer row (``BatchedWorld.bev_agents`` on ``vector_obs["observers"]`` and ``["goals"]``;
        DESIGN.md section 1 "Per-agent BEV"), else ``[N, H, W(, 3)]`` from every ego (``BatchedWorld.bev``).  It is
        rejected with ``observation="bev"``, whose observation already is that image;
        ``leaders``: e.g. ``dict(half_width=1.8, max_range=100.0)`` binds a leader search (``BatchedWorld.set_leader_search``;
        DESIGN.md section 1 "Leader search"), so the controllers set on ``env.world`` follow the participant ahead of them
        every step instead of a fixed ``lead_index``, and adds ``info["leader"]`` (int16 [N, M], -1 for none) and
        ``info["leader_gap"]`` (fp32 [N, M], +inf for none) to ``reset`` and ``step``: the leaders of the state after the
        auto-reset (``BatchedWorld.find_leaders``);
        ``lane_change``: e.g. ``dict(left=[1, -1], right=[-1, 0], politeness=0.0)`` (the keywords of
        ``BatchedWorld.set_lane_change``; needs ``leaders``) lets the IDM rows with a lateral channel change lanes with
        MOBIL (DESIGN.md section 1 "Lane changes").  It is bound after the search, at ``reset`` - set the paths and the
        controllers (with ``path_id``) on ``env.world`` first - and bound again there whenever ``set_controllers`` or
        ``set_paths`` dropped it.  It adds ``info["lane_path"]`` (int16 [N, M], every slot's current lane) and
        ``info["lane_change"]`` (int8 [N, M], the decisions of the step) to ``reset`` and ``step``, after the auto-reset,
        which restarts the reset scenarios from their ``path_id``;
        ``reactive``: e.g. ``dict(controller=IDMController(..., lateral=PIDController(lateral_error="path_cross_track")),
        tolerance=0.1, extend=30.0)`` (needs ``replay`` and ``leaders``) makes the replayed traffic react (DESIGN.md
        section 1 "Reactive replay"): every moving track follows its own logged path (``ReplayLog.track_paths``, appended
        to the ``route`` paths) with the controller from its first sample on, braking for whatever the leader search finds
        ahead of it, the ego included.  Every slot but the ego's gets the controller row (``world.set_controllers``); the
        reactive replay is bound at ``reset``, and bound again there whenever a later setter dropped it.  It adds
        ``yielding``: e.g. ``dict(critical_gap=3.0, priority=[...])`` (the keywords of ``BatchedWorld.set_yielding``; needs
        ``leaders``) makes the path-following IDM traffic yield at the conflict zones of the bound paths (DESIGN.md section 1
        "Yielding at conflict zones"); with ``reactive`` the zones are those of the track paths and the route paths (the ego
        routes), so a reactive track also yields to the ego.  It is bound at ``reset``, and bound again there whenever a
        later setter dropped it.  It adds ``info["yield_to"]`` (int16 [N, M], the slot each car yields to, -1 for none) and
        ``info["stop_gap"]`` (fp32 [N, M], +inf for none) to ``reset`` and ``step``: the yields of the state after the
        auto-reset (``BatchedWorld.find_yields``);
        ``info["reactive"]`` (bool [N, M], the slots that show a reactive track, ``BatchedWorld.reactive``) to ``reset``
        and ``step``, after the auto-reset."""
        import torch

        if observation not in ("state", "bev", "vector", "agents"):
            raise ValueError(f"observation must be 'state', 'bev', 'vector' or 'agents', got {observation!r}")
        if agent_rewards and observation != "agents":
            raise ValueError("agent_rewards needs observation='agents' (its observer list names the agents)")
        if agent_actions and observation != "agents":
            raise ValueError("agent_actions needs observation='agents' (its observer list names the agents)")
        if agent_rewards and target is not None:
            raise ValueError("agent_rewards takes per-row goals in vector_obs['goals'], not target")
        self.agent_rewards = bool(agent_rewards)
        self.agent_actions = bool(agent_actions)
        self.observation = observation
        self.vector_obs = dict(vector_obs or {})
        keys = {"k_agents", "k_segments", "agent_range", "segment_range"}
        if observation == "agents":
            keys |= {"observers", "goals"}
        unknown = set(self.vector_obs) - keys
        if unknown:
            raise ValueError(f"vector_obs: unknown keys {sorted(unknown)}")
        self.lidar = None if lidar is None else dict(lidar)
        if self.lidar is not None:
            unknown = set(self.lidar) - {"n_beams", "max_range"}
            if unknown:
                raise ValueError(f"lidar: unknown keys {sorted(unknown)}")
        self.route = None if route is None else dict(route)
        if self.route is not None:
            unknown = set(self.route) - {"paths", "route_id", "threshold", "progress_weight", "off_route_reward", "n_points",
                                         "spacing"}
            if unknown:
                raise ValueError(f"route: unknown keys {sorted(unknown)}")
            missing = {"paths", "route_id", "threshold"} - set(self.route)
            if missing:
                raise ValueError(f"route: missing keys {sorted(missing)}")
        self.sampler = None if sampler is None else dict(sampler)
        if self.sampler is not None:
            unknown = set(self.sampler) - {"seed", "jitter", "tries", "sample_rows", "avoid_target"}
            if unknown:
                raise ValueError(f"sampler: unknown keys {sorted(unknown)}")
            jit = self.sampler.get("jitter")
            if replay is not None and jit is not None and np.any(np.asarray(jit)[1:] != 0):
                raise ValueError("sampler: with replay only slot 0 may have jitter (the log drives the others)")
            if agent_rewards and self.vector_obs.get("goals") is not None and self.sampler.get("sample_rows", True):
                raise ValueError("sampler: per-row goals belong to scenarios, not pool rows: use sample_rows=False")
        self.history = None if history is None else dict(history)
        if self.history is not None:
            unknown = set(self.history) - {"length"}
            if unknown:
                raise ValueError(f"history: unknown keys {sorted(unknown)}")
            if "length" not in self.history:
                raise ValueError("history: missing key 'length'")
        self.camera = None if camera is None else dict(camera)
        if self.camera is not None:
            if observation == "bev":
                raise ValueError("camera: the 'bev' observation already is the ego's image; use bev_resolution / bev_range")
            unknown = set(self.camera) - {"resolution", "perception_range", "rgb"}
            if unknown:
                raise ValueError(f"camera: unknown keys {sorted(unknown)}")
        self.leaders = None if leaders is None else dict(leaders)
        if self.leaders is not None:
            unknown = set(self.leaders) - {"half_width", "max_range"}
            if unknown:
                raise ValueError(f"leaders: unknown keys {sorted(unknown)}")
            self.leaders = dict(half_width=float(self.leaders.get("half_width", 1.8)),
                                max_range=float(self.leaders.get("max_range", 100.0)))
        self.lane_change = None if lane_change is None else dict(lane_change)
        if self.lane_change is not None:
            if self.leaders is None:
                raise ValueError("lane_change needs a leader search: pass leaders=dict(...)")
            unknown = set(self.lane_change) - {"left", "right", "politeness", "threshold", "b_safe", "min_gap", "cooldown"}
            if unknown:
                raise ValueError(f"lane_change: unknown keys {sorted(unknown)}")
            if "left" not in self.lane_change or "right" not in self.lane_change:
                raise ValueError("lane_change needs the 'left' and 'right' neighbour tables")
        self.reactive = None if reactive is None else dict(reactive)
        if self.reactive is not None:
            if replay is None or leaders is None:
                raise ValueError("reactive needs a log and a leader search: pass replay=... and leaders=dict(...)")
            if lane_change is not None:
                raise ValueError("reactive does not take lane changes (lane_change)")
            unknown = set(self.reactive) - {"controller", "tolerance", "extend"}
            if unknown:
                raise ValueError(f"reactive: unknown keys {sorted(unknown)}")
            if "controller" not in self.reactive:
                raise ValueError("reactive needs the 'controller' its tracks drive with")
        self.yielding = None if yielding is None else dict(yielding)
        if self.yielding is not None:
            if self.leaders is None:
                raise ValueError("yielding needs a leader search: pass leaders=dict(...)")
            unknown = set(self.yielding) - {"priority", "width", "margin", "critical_gap", "commit_decel", "v_min"}
            if unknown:
                raise ValueError(f"yielding: unknown keys {sorted(unknown)}")
        self.bev_resolution = (int(bev_resolution[0]), int(bev_resolution[1]))
        self.bev_range = bev_range

        self.replay = replay
        if replay is not None:
            scene = replay.scene() if scene is None else replay.scene(scene.segments, scene.bounds, scene.name)
        self.scene = scene
        n, m = scene.shape
        self.num_envs, self.num_participants = n, m
        self.max_step = int(max_step)
        self.auto_reset = auto_reset
        self.world = BatchedWorld(n, m, scene.table, device=device, interval=step_size, delta_t=delta_t, max_step=max_step,
                                  any_participant=any_participant, steer_first=True)
        self.world.set_map(scene.segments, scene.bounds)
        self.scenario_manager = BatchedScenarioManager(self.world, max_step=max_step, step_size=step_size)
        dev = self.world.device
        self._pool = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in scene.state().items()}
        self._type_id = torch.from_numpy(scene.type_id).to(dev)
        self.scenario_manager.set_initial_state(self._pool)
        if replay is not None:
            self.world.set_log(replay.log, replay.t0, **replay.binding())
        self._action = torch.zeros((n, m, 2), dtype=torch.float32, device=dev)
        self._rng = np.random.default_rng(0)
        if target is not None:
            self.world.set_goal(target, arrival_threshold, no_action_max_step)
        if self.agent_rewards:
            self.world.set_agents(self.vector_obs.get("observers"), self.vector_obs.get("goals"), arrival_threshold,
                                  no_action_max_step)
        self._route_pool = None
        if self.route is not None:
            rt = self.route
            rid = np.asarray(rt["route_id"].cpu() if torch.is_tensor(rt["route_id"]) else rt["route_id"]).astype(np.int64)
            if rid.shape == (n,):
                rid = np.concatenate([rid[:, None], np.full((n, m - 1), -1, np.int64)], 1)
            if rid.shape != (n, m):
                raise ValueError(f"route['route_id'] must be [{n}, {m}] or [{n}] (one row per pool row)")
            self.world.set_paths(rt["paths"])
            self._route_pool = torch.from_numpy(rid.astype(np.int16)).to(dev)
            self.world.set_routes(self._route_pool.clone(), rt["threshold"], rt.get("progress_weight", 0.1),
                                  rt.get("off_route_reward", -5.0))
            self._route_observers = None
            if observation == "agents":
                obs = self.vector_obs.get("observers")
                self._route_observers = obs if obs is not None else \
                    torch.arange(m, dtype=torch.int16, device=dev).expand(n, m).contiguous()
        self._target_pool = None if target is None else self.world._goal["target"].clone()
        if self.sampler is not None:
            self._bind_sampler(self.sampler.get("seed", 0))
        if self.history is not None:
            self.world.set_history(self.history["length"])
        if self.leaders is not None:
            self.world.set_leader_search(**self.leaders)
        self._reactive_tracks = None
        if self.reactive is not None:
            rc = self.reactive
            paths, track_path, speed = replay.log.track_paths(rc.get("tolerance", 0.1), rc.get("extend", 30.0))
            base = [] if self.route is None else list(self.route["paths"])
            self.world.set_paths(base + paths)
            ctrl = np.zeros((n, m), np.uint8)
            ctrl[:, 0] = 255                                   # the ego is the policy's
            self.world.set_controllers([rc["controller"]], ctrl)
            self._reactive_tracks = dict(track_path=track_path, desired_speed=speed, path_base=len(base))
        self._last_obs = None
        if observation == "bev":
            w, h = self.bev_resolution
            self.observation_space = {"shape": (n, h, w, 3), "dtype": "uint8", "low": 0, "high": 255}
        elif observation == "vector":
            self.observation_space = {"shape": (n, self.world.observe(**self.vector_obs).flat.shape[1]), "dtype": "float32"}
        elif observation == "agents":
            self.observation_space = {"shape": tuple(self.world.observe_agents(**self.vector_obs).flat.shape),
                                      "dtype": "float32"}
        else:
            self.observation_space = {"shape": (n, m, 6), "dtype": "float32"}
        self.action_space = {"shape": (n, 2), "low": (-np.inf, -np.inf), "high": (np.inf, np.inf)}
        if self.agent_actions:
            obs = self.vector_obs.get("observers")
            self.action_space["shape"] = (n, m if obs is None else int(obs.shape[1]), 2)

    # ------------------------------------------------------------------ helpers
    def _bind_sampler(self, seed):
        """(Re)key the reset sampler (zeroes the episode counters); the pool rows' types, targets and routes follow them."""
        sp = self.sampler
        self.world.set_reset_sampler(seed, jitter=sp.get("jitter"), tries=sp.get("tries", 8),
                                     sample_rows=sp.get("sample_rows", True), avoid_target=sp.get("avoid_target", False),
                                     type_id=self._type_id, target=self._target_pool, route_id=self._route_pool)

    def _obs(self):
        if self.observation == "bev":
            return self.world.bev(self.bev_resolution, self.bev_range, rgb=True)
        if self.observation == "vector":
            self._last_obs = self.world.observe(**self.vector_obs)
            return self._last_obs.flat
        if self.observation == "agents":
            self._last_obs = self.world.observe_agents(**self.vector_obs)
            return self._last_obs.flat
        return self.scenario_manager.get_observation()

    def _info(self, status, traffic, flags, hit_index, hit_segment):
        info = {"scenario_status": status, "traffic_status": traffic, "flags": flags, "hit_index": hit_index,
                "hit_segment": hit_segment, "step_count": self.world.step_count}
        if self.world.replay_track is not None:   # scheduled replay: the track each slot shows (-1: none)
            info["track"] = self.world.replay_track
        if self.sampler is not None:
            info["pool_row"] = self.world.pool_row
        return info

    def _add_lidar(self, info):
        """``info["lidar"]`` / ``info["bev"]`` / ``info["route"]`` / ``info["history"]`` / ``info["leader"]`` and
        ``info["leader_gap"]`` when the env has a lidar / a camera / routes / a history / a leader search; called after the
        auto-reset and the observation, so that they see the new episodes and the observation's agents."""
        if self.route is not None:
            info["route"] = self.world.route_observe(self.route.get("n_points", 8), self.route.get("spacing", 2.0),
                                                     self._route_observers)
        if self.lidar is not None:
            if self.observation == "agents":
                info["lidar"] = self.world.lidar_scan_agents(**self.lidar, observers=self.vector_obs.get("observers"))
            else:
                info["lidar"] = self.world.lidar_scan(**self.lidar)
        if self.camera is not None:
            cam = dict(resolution=self.camera.get("resolution", (200, 200)),
                       perception_range=self.camera.get("perception_range", 20.0), rgb=self.camera.get("rgb", True))
            if self.observation == "agents":
                info["bev"] = self.world.bev_agents(**cam, observers=self.vector_obs.get("observers"),
                                                    goals=self.vector_obs.get("goals"))
            else:
                info["bev"] = self.world.bev(**cam)
        if self.history is not None:
            if self.observation == "vector":
                info["history"] = self.world.observe_history(self._last_obs.agent_index)
            elif self.observation == "agents":
                info["history"] = self.world.observe_history(self._last_obs.agent_index, self.vector_obs.get("observers"))
            else:
                info["history"] = self.world.observe_history()
        if self.leaders is not None:
            info["leader"], info["leader_gap"] = self.world.find_leaders(**self.leaders)
        if self.lane_change is not None:
            info["lane_path"], info["lane_change"] = self.world.lane_path, self.world.lane_change
        if self.reactive is not None:
            info["reactive"] = self.world.reactive
        if self.yielding is not None:
            info["yield_to"], info["stop_gap"] = self.world.find_yields()
        return info

    # ------------------------------------------------------------------ gym surface
    def reset(self, seed: int = None, options: dict = None):
        import torch

        if self.sampler is not None and options and options.get("shuffle"):
            raise ValueError("a sampled env draws its rows: options={'shuffle': True} is not taken")
        if seed is not None:
            self._rng = np.random.default_rng(seed)
            if self.sampler is not None:
                self._bind_sampler(seed)
        perm = None
        if options and options.get("shuffle"):
            perm = torch.from_numpy(self._rng.permutation(self.num_envs).astype(np.int32)).to(self.world.device)
        if self.lane_change is not None and self.world.lane_path is None:   # bound after the search, on the set controllers
            self.world.set_lane_change(**self.lane_change)
        if self.reactive is not None and self.world.drive_path is None:   # the reset below hands the present tracks over
            self.world.set_reactive_replay(**self._reactive_tracks)
        if self.yielding is not None and self.world.yield_to is None:   # on the bound paths, controllers and search
            self.world.set_yielding(**self.yielding)
        if self.agent_rewards:   # every slot takes its pool row's type below; no retired type of the old episodes survives
            self.world.retired_type.fill_(255)
            self.world.reset_agent_trackers()
        if self.sampler is not None:                        # K13 copies the drawn rows' types and routes
            self.scenario_manager.reset(sample=True)
        elif self.replay is not None and perm is not None:   # the rows' own types (the replayed slots' are rewritten anyway)
            self.world.type_id.copy_(self._type_id[perm.long()])
            if self._route_pool is not None:                # ... and routes
                self.world.route_id.copy_(self._route_pool[perm.long()])
        else:
            self.world.type_id.copy_(self._type_id)
            if self._route_pool is not None:
                self.world.route_id.copy_(self._route_pool)
        if self.sampler is None:
            self.scenario_manager.reset(pool_index=perm)
        self.world.reset_env_trackers()
        status = torch.full((self.num_envs,), int(ScenarioStatus.NORMAL), dtype=torch.uint8, device=self.world.device)
        traffic = torch.full((self.num_envs, self.num_participants), int(TrafficStatus.NORMAL), dtype=torch.uint8,
                             device=self.world.device)
        o = self.world._out
        obs = self._obs()
        info = self._info(status, traffic, torch.zeros_like(o.flags), torch.full_like(o.hit_index, -1),
                          torch.full_like(o.hit_segment, -1))
        return obs, self._add_lidar(info)

    def step(self, action, npc_action=None):
        """``action``: fp32 device tensor [N, 2] = (steering, accel) of the ego (participant 0), or [N, M, 2] for
        all participants; ``npc_action`` [N, M-1, 2] optionally drives the others (otherwise they keep their rows of the
        internal action array: zeros, or what ``world.set_controllers`` computes on the device every tick).

        Launches per call: the controllers (if set), the fused tick, the env epilogue (reward / terminated / truncated /
        TrafficStatus / done in one kernel) and the masked reset - no elementwise PyTorch.  The tensors in the returned
        tuple and in ``info`` are views of buffers owned by the env: they hold this step's values until the next ``step``.

        With ``agent_actions``: ``action`` is exactly ``[N, Q, 2]``, one (steering, accel) per observer row, scattered into
        the internal action array by one more launch in front of the controllers; ``npc_action`` [N, M, 2] optionally
        fills that array first (the slots no agent row drives keep its rows)."""
        w = self.world
        if self.agent_actions:
            if tuple(action.shape) != self.action_space["shape"]:
                raise InvalidAction(f"Action of shape {tuple(action.shape)} is not in the action space.")
            full = self._action
            if npc_action is not None:
                full.copy_(npc_action)
            w.set_ego_action(None)
            w.scatter_agent_action(action.to(device=w.device, dtype=full.dtype).contiguous(), full,
                                   self.vector_obs.get("observers"))
        elif action.dim() == 3:
            if tuple(action.shape) != (self.num_envs, self.num_participants, 2):
                raise InvalidAction(f"Action of shape {tuple(action.shape)} is not in the action space.")
            full = action.contiguous()
            w.set_ego_action(None)
        else:
            if tuple(action.shape) != (self.num_envs, 2):
                raise InvalidAction(f"Action of shape {tuple(action.shape)} is not in the action space.")
            full = self._action
            w.set_ego_action(action.to(device=w.device, dtype=full.dtype).contiguous())   # read by the kernels, not scattered
            if npc_action is not None:
                full[:, 1:, :] = npc_action
        if w.last_accel is not None:
            w.control(full)
        self.scenario_manager.update(full)
        if self.agent_rewards:   # one K10 launch instead of the ego's epilogue; retired slots ignore their action rows
            a = w.agents_epilogue(reset_trackers_on_done=self.scenario_manager.reset_trackers_on_done)
            r = w.result
            info = self._info(r.status, a.traffic, r.flags, r.hit_index, r.hit_segment)
            info["agent_status"], info["agent_iou"] = a.status, a.iou
            if self.auto_reset:
                self._auto_reset(a.done)
            obs = self._obs()
            return obs, a.reward, a.terminated, a.truncated, self._add_lidar(info)
        status, traffic = self.scenario_manager.check_status()
        e = self.scenario_manager.env_result
        r = w.result
        info = self._info(status, traffic, r.flags, r.hit_index, r.hit_segment)
        if r.iou is not None:
            info["iou"] = r.iou
        if self.auto_reset:
            self._auto_reset(e.done)
        obs = self._obs()
        return obs, e.reward, e.terminated, e.truncated, self._add_lidar(info)

    def _auto_reset(self, done):
        """The masked reset of the finished scenarios: a new draw with a sampler, else the scenario's row again (with a
        log: its episode row)."""
        if self.sampler is not None:
            self.scenario_manager.reset(mask=done, sample=True)
        else:
            self.scenario_manager.reset(mask=done, pool_index=self.world.log_row)

    def render(self):
        raise NotImplementedError("rendering is outside this hot path")

    def close(self):
        self.world.close()
