"""The trajectory history without a device: the ring semantics of ``tests/history_oracle.py`` on hand-built sequences, its
lag-0 blocks against the vector-observation oracles' agent rows, the argument checks that need no device, and
``bench_history.py --help``."""

from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import agent_obs_oracle as AO
from tests import history_oracle as HO
from tests import vector_obs_oracle as VO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE = [dict(shape=0, half_len=2.0, half_wid=1.0, radius=1.0), dict(shape=1, half_len=0.4, half_wid=0.4, radius=0.4),
         dict(shape=2, half_len=0.0, half_wid=0.0, radius=0.0)]


def _state(rng, N, M):
    st = {k: rng.uniform(-30, 30, (N, M)).astype(np.float32) for k in ("x", "y")}
    st["heading"] = rng.uniform(-np.pi, np.pi, (N, M)).astype(np.float32)
    st["speed"] = rng.uniform(0, 10, (N, M)).astype(np.float32)
    st["vx"] = (st["speed"] * np.cos(st["heading"])).astype(np.float32)
    st["vy"] = (st["speed"] * np.sin(st["heading"])).astype(np.float32)
    return st


def _expected(states, types, H):
    """The view of a ring that saw ``states`` (one per entry of the current episode, oldest first), by brute force."""
    N, M = types[-1].shape
    out = {k: np.zeros((N, M, H), np.float32) for k in HO.FIELDS}
    valid = np.zeros((N, M, H), bool)
    for lag in range(min(H, len(states))):
        st, t = states[-1 - lag], types[-1 - lag]
        ok = (t == types[-1]) & (t < len(TABLE))
        valid[:, :, lag] = ok
        for k in HO.FIELDS:
            out[k][:, :, lag] = np.where(ok, st[k], 0)
    return out, valid


@pytest.mark.parametrize("H", [1, 2, 5])
def test_ring_lengths_below_at_and_above_H(H):
    rng = np.random.default_rng(H)
    N, M = 3, 5
    t = rng.integers(0, 2, (N, M)).astype(np.uint8)
    ring = HO.Ring(N, M, H)
    v = ring.view(t, len(TABLE))
    assert not v["valid"].any() and (v["count"] == 0).all()   # a new binding is empty
    st = _state(rng, N, M)
    ring.restart(np.ones(N), st, t)
    states, types = [st], [t]
    for L in range(1, 3 * H + 2):
        v = ring.view(t, len(TABLE))
        ref, valid = _expected(states, types, H)
        assert (v["count"] == L).all()
        assert np.array_equal(v["valid"], valid)
        assert v["valid"][:, :, :min(L, H)].all() and not v["valid"][:, :, min(L, H):].any()
        for k in HO.FIELDS:
            assert np.array_equal(v[k], ref[k]), (L, k)
        st = _state(rng, N, M)
        ring.append(st, t)
        states.append(st); types.append(t)


def test_restart_mid_ring_keeps_the_unmasked_scenarios():
    rng = np.random.default_rng(7)
    N, M, H = 4, 3, 4
    t = np.zeros((N, M), np.uint8)
    ring = HO.Ring(N, M, H)
    st = _state(rng, N, M)
    ring.restart(np.ones(N), st, t)
    for _ in range(6):
        ring.append(_state(rng, N, M), t)
    before = ring.view(t, len(TABLE))
    mask = np.array([0, 1, 0, 1])
    st = _state(rng, N, M)
    ring.restart(mask, st, t)
    after = ring.view(t, len(TABLE))
    assert list(after["count"]) == [7, 1, 7, 1]
    for n in (0, 2):
        for k in ("x", "valid"):
            assert np.array_equal(after[k][n], before[k][n])
    for n in (1, 3):
        assert after["valid"][n, :, 0].all() and not after["valid"][n, :, 1:].any()
        assert np.array_equal(after["x"][n, :, 0], st["x"][n])
    ring.append(_state(rng, N, M), t)
    assert list(ring.view(t, len(TABLE))["count"]) == [8, 2, 8, 2]


def test_type_and_track_changes_invalidate_entries():
    rng = np.random.default_rng(3)
    N, M, H = 2, 4, 6
    t = np.array([[0, 1, 0, 255], [0, 0, 1, 1]], np.uint8)
    tr = np.array([[-1, 3, 4, -1], [-1, -1, 5, 6]], np.int32)
    ring = HO.Ring(N, M, H)
    ring.restart(np.ones(N), _state(rng, N, M), t, tr)
    ring.append(_state(rng, N, M), t, tr)
    t2 = t.copy(); t2[0, 1] = 255          # slot retired (K10) or its track absent
    t2[1, 3] = 0                           # another type moved in
    tr2 = tr.copy(); tr2[0, 2] = 9         # a schedule's track switch
    ring.append(_state(rng, N, M), t2, tr2)
    v = ring.view(t2, len(TABLE), tr2)
    assert v["valid"][0, 0].tolist() == [True, True, True, False, False, False]
    assert not v["valid"][0, 1].any()      # an empty slot has no history
    assert v["valid"][0, 2].tolist() == [True, False, False, False, False, False]
    assert not v["valid"][0, 3].any()
    assert v["valid"][1, 3].tolist() == [True, False, False, False, False, False]
    assert v["valid"][1, 2].tolist() == [True, True, True, False, False, False]
    # the slot takes its old type and track back: the old entries count again, the foreign one does not
    ring.append(_state(rng, N, M), t, tr)
    v = ring.view(t, len(TABLE), tr)
    assert v["valid"][0, 2].tolist() == [True, False, True, True, False, False]
    assert v["type_id"][0, 2, 1] == 255 and v["x"][0, 2, 1] == 0


@pytest.mark.parametrize("K", [0, 3, 7])
def test_lag0_block_is_the_vector_observation_agent_row(K):
    rng = np.random.default_rng(K + 11)
    N, M, H = 5, 9, 3
    t = rng.integers(0, 3, (N, M)).astype(np.uint8)
    t[0, 0] = 255
    t[1, 4] = 255
    ring = HO.Ring(N, M, H)
    ring.restart(np.ones(N), _state(rng, N, M), t)
    st = _state(rng, N, M)
    ring.append(st, t)                      # the newest entry is the current state
    flat, aidx, _ = VO.observe(st, t, TABLE, K, 0, 1e4, 1.0)
    got, dist = HO.observe(ring, st, t, len(TABLE), agent_index=aidx)
    agents = VO.split(flat, K, 0)[2]
    assert got.shape == (N, 1 + K, H, HO.HIST_F)
    for n in range(N):
        for k in range(K):
            if aidx[n, k] < 0:
                assert (got[n, 1 + k] == 0).all()
                continue
            assert np.array_equal(got[n, 1 + k, 0, :].view(np.uint32), agents[n, k, :7].view(np.uint32)), (n, k)
            assert np.isclose(dist[n, 1 + k, 0], agents[n, k, 10], rtol=1e-6)
    assert (got[0] == 0).all()              # no ego: a zero row
    # K9-style rows: observers with duplicates, -1 and M in the list
    obs = np.array([[0, 2, 2, -1, M], [3, 1, 0, 8, 5]] * 2 + [[4, 4, 0, 1, 2]], np.int16)
    flat, aidx, _ = AO.observe_agents(st, t, TABLE, K, 0, 1e4, 1.0, observers=obs)
    got, dist = HO.observe(ring, st, t, len(TABLE), agent_index=aidx, observers=obs, Q=obs.shape[1])
    agents = AO.split(flat, K, 0)[2].reshape(N * obs.shape[1], K, VO.AGENT_F)
    got_rows = got.reshape(N * obs.shape[1], 1 + K, H, HO.HIST_F)
    for rid in range(N * obs.shape[1]):
        for k in range(K):
            if aidx.reshape(-1, K)[rid, k] >= 0:
                assert np.array_equal(got_rows[rid, 1 + k, 0].view(np.uint32), agents[rid, k, :7].view(np.uint32))
    for rid in np.nonzero((obs.reshape(-1) < 0) | (obs.reshape(-1) >= M))[0]:
        assert (got_rows[rid] == 0).all()


def test_observer_block_holds_its_own_past():
    rng = np.random.default_rng(5)
    N, M, H = 2, 3, 4
    t = np.zeros((N, M), np.uint8)
    ring = HO.Ring(N, M, H)
    st0 = _state(rng, N, M)
    ring.restart(np.ones(N), st0, t)
    st1 = _state(rng, N, M)
    ring.append(st1, t)
    got, dist = HO.observe(ring, st1, t, len(TABLE))
    assert got.shape == (N, 1, H, HO.HIST_F)
    assert (got[:, 0, 0, 1:3] == 0).all() and (got[:, 0, 0, 3] == 1).all() and (got[:, 0, 0, 4] == 0).all()
    assert (got[:, 0, :2, 0] == 1).all() and (got[:, 0, 2:] == 0).all()
    c, s = np.cos(st1["heading"][:, 0].astype(np.float64)), np.sin(st1["heading"][:, 0].astype(np.float64))
    dx = st0["x"][:, 0].astype(np.float64) - st1["x"][:, 0]
    dy = st0["y"][:, 0].astype(np.float64) - st1["y"][:, 0]
    assert np.array_equal(got[:, 0, 1, 1], (c * dx + s * dy).astype(np.float32))


def test_oracle_rejects_lengths_outside_the_abi():
    for H in (0, 65):
        with pytest.raises(ValueError):
            HO.Ring(1, 1, H)


def test_abi_rejections_that_need_no_device():
    from tactics2d_b200 import _lib

    lib = _lib.load()
    null = C.c_void_p(0)
    assert lib.t2d_set_history(null, 8) == -1
    assert lib.t2d_observe_history(null, null, 0, null, 0, null, null) == -1
    assert lib.t2d_history_view(null, None) == -1
    assert _lib.SYMBOLS["t2d_set_history"] == (C.c_int, [C.c_void_p, C.c_int32])


def test_env_rejects_unknown_history_keys():
    from tactics2d_b200.envs import BatchedTrafficEnv

    with pytest.raises(ValueError, match="history: unknown keys"):
        BatchedTrafficEnv(None, history=dict(length=4, stride=2))
    with pytest.raises(ValueError, match="history: missing key"):
        BatchedTrafficEnv(None, history=dict())


def test_hist_fields_are_exported():
    import tactics2d_b200

    assert tactics2d_b200.HIST_FIELDS == ("valid", "ex", "ey", "cos_dh", "sin_dh", "v_x", "v_y")
    assert tactics2d_b200.AGENT_FIELDS[:7] == tactics2d_b200.HIST_FIELDS


def test_bench_history_help_without_a_device():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench_history.py"), "--help"], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "usage:" in r.stdout
