"""CPU oracle for the tactics2d batched env.step() hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``oracle/`` is part of the product:
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline /
``--impl reference`` legs may import or execute it, and there only as the
checker (or as the timed CPU baseline), never as the thing shipped.  The
product path (``tactics2d_b200``) fails loudly when its CUDA library is missing.

What it is: a float64 restatement of the reference's per-participant algorithm

* ``oracle.physics``   - SingleTrackKinematics / SingleTrackDynamics / PointMass
  (reference ``tactics2d/physics/*.py``), vectorised NumPy float64;
* ``oracle.scalar_port`` - the same, written as the reference writes it (one
  Python call per participant, NumPy *scalar* arithmetic) - the CPU baseline;
* ``oracle.geometry``  - pose (``participant/element/vehicle.py:263-281``) and
  the closed-set ``intersects`` / ``contains`` predicates the reference gets
  from shapely/GEOS (``traffic/event_detection/collision.py``, ``out_bound.py``);
* ``oracle.scenario``  - the whole tick: physics -> pose -> collisions ->
  out-of-bound -> status priority chain (``envs/parking.py:352-392``);
* ``oracle/c/``        - the same tick in plain C (gcc), for full-size checks;
* ``oracle.lidar``     - ``SingleLineLidar._scan_obstacles`` (``sensor/lidar.py:128-221``);
* ``oracle.controllers`` - IDM / cruise / adaptive cruise / pure pursuit (``controller/*.py``).

Parity pinning
--------------
* Physics (all four models, SingleTrackDrift included): PINNED.
  ``oracle/make_golden.py`` imports the *unmodified* reference
  (``tactics2d/physics`` of a reference checkout) and writes
  ``tests/golden/physics_*.npz``; ``tests/test_oracle_golden.py`` holds the
  oracle to those vectors (<=1e-12 relative) and to the survey's KATs.
* Controllers and lidar: PINNED to outputs of the unmodified reference classes
  (``tests/golden/controllers.npz``, ``lidar.npz``).  Those modules import a few
  shapely containers; the generator supplies stand-ins for exactly the members
  they touch (``LineString.interpolate``; ring coordinates, ``affine_transform``,
  ``distance``) and says so - the arithmetic the kernels reproduce is the
  reference's own code.  ``tests/test_oracle_controllers.py``,
  ``tests/test_oracle_lidar.py``.
* Collision / out-of-bound / status / Arrival-NoAction IoU: PARITY UNPINNED.  The reference computes
  these with shapely/GEOS (third-party, ``shapely>=2.0.7,<2.1.0``,
  requirements.txt:18), which is not installable here, and the reference's own
  tests pin no value at that boundary (tests/test_traffic.py is empty,
  tests/test_env.py is all skipped).  The oracle restates the documented GEOS
  semantics (closed sets; touching counts) and is cross-checked against an
  independent exact-rational edge-crossing definition in
  ``tests/test_oracle_geometry.py``.
"""
