"""Known answers for the per-agent action oracle (tests/agent_action_oracle.py, DESIGN.md section 1 "Per-agent
action"): the lowest row naming a slot wins, rows out of range and slots that are empty or retired take nothing, the
rows no agent names keep their values, and the fp32 bits pass through unchanged."""

import numpy as np

from tests.agent_action_oracle import owner_rows, scatter_agent_action

N_TYPES = 3


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _rows(Q, base=10.0):
    """agent_action [1, Q, 2] whose row q is (base + q, -(base + q))."""
    v = base + np.arange(Q, dtype=np.float32)
    return np.stack([v, -v], -1)[None]


def test_duplicates_lowest_row_wins():
    types = np.zeros((1, 4), np.uint8)
    act = np.zeros((1, 4, 2), np.float32)
    obs = np.array([[2, 1, 2, 1, 2]])
    out = scatter_agent_action(act, _rows(5), types, N_TYPES, obs)
    assert np.array_equal(out[0, 2], [10, -10]) and np.array_equal(out[0, 1], [11, -11])
    assert np.array_equal(out[0, [0, 3]], np.zeros((2, 2)))
    assert np.array_equal(owner_rows(types, 5, obs)[0], [5, 1, 0, 5])


def test_rows_out_of_range_write_nothing():
    types = np.zeros((1, 3), np.uint8)
    act = np.full((1, 3, 2), 7.0, np.float32)
    obs = np.array([[-1, 3, 100, -32768, 1]])
    out = scatter_agent_action(act, _rows(5), types, N_TYPES, obs)
    assert np.array_equal(out[0, 1], [14, -14])
    assert np.array_equal(out[0, [0, 2]], np.full((2, 2), 7.0))


def test_empty_and_retired_slots_take_nothing():
    types = np.array([[0, 255, N_TYPES, 2]], np.uint8)   # 255 empty or retired, n_types: no such row either
    act = np.full((1, 4, 2), -3.0, np.float32)
    out = scatter_agent_action(act, _rows(4), types, N_TYPES, None)
    assert np.array_equal(out[0, 0], [10, -10]) and np.array_equal(out[0, 3], [13, -13])
    assert np.array_equal(out[0, 1:3], np.full((2, 2), -3.0))
    # a retired slot's row is not handed to the next row naming it: the first row owns the slot either way
    out = scatter_agent_action(act, _rows(2), types, N_TYPES, np.array([[1, 1]]))
    assert np.array_equal(out, act)


def test_no_observer_list_is_row_q_on_slot_q():
    rng = np.random.default_rng(0)
    N, M, Q = 5, 8, 6
    types = rng.integers(0, N_TYPES, (N, M)).astype(np.uint8)
    act = rng.normal(size=(N, M, 2)).astype(np.float32)
    rows = rng.normal(size=(N, Q, 2)).astype(np.float32)
    out = scatter_agent_action(act, rows, types, N_TYPES, None)
    assert np.array_equal(out[:, :Q], rows) and np.array_equal(out[:, Q:], act[:, Q:])
    explicit = scatter_agent_action(act, rows, types, N_TYPES, np.broadcast_to(np.arange(Q), (N, Q)))
    assert np.array_equal(_bits(out), _bits(explicit))


def test_one_row_and_128_rows_above_m():
    types = np.zeros((2, 4), np.uint8)
    act = np.zeros((2, 4, 2), np.float32)
    out = scatter_agent_action(act, _rows(1).repeat(2, 0), types, N_TYPES, np.array([[3], [0]]))
    assert np.array_equal(out[0, 3], [10, -10]) and np.array_equal(out[1, 0], [10, -10])
    assert np.count_nonzero(out) == 4
    obs = np.arange(128)[None].repeat(2, 0) % 6 - 1   # -1, 0, 1, 2, 3, 4 (out of range), -1, 0, ...
    out = scatter_agent_action(act, _rows(128).repeat(2, 0), types, N_TYPES, obs)
    assert np.array_equal(out[:, :, 0], np.array([[11, 12, 13, 14]] * 2, np.float32))


def test_non_agent_rows_are_untouched_bit_for_bit():
    rng = np.random.default_rng(1)
    N, M, Q = 16, 32, 12
    types = rng.integers(0, N_TYPES + 1, (N, M)).astype(np.uint8)
    types[types == N_TYPES] = 255
    act = rng.normal(size=(N, M, 2)).astype(np.float32)
    act[0, 0] = [np.float32(-0.0), np.nan]
    obs = rng.integers(-2, M + 2, (N, Q))
    out = scatter_agent_action(act, rng.normal(size=(N, Q, 2)).astype(np.float32), types, N_TYPES, obs)
    written = (owner_rows(types, Q, obs) < Q) & (types < N_TYPES)
    assert written.any() and (~written).any()
    assert np.array_equal(_bits(out)[~written], _bits(act)[~written])


def test_nan_payloads_and_negative_zero_pass_through():
    types = np.zeros((1, 3), np.uint8)
    src = np.zeros((1, 3, 2), np.uint32)
    src[0, 0] = [0x80000000, 0x7FC00001]   # -0.0, a quiet NaN with a payload
    src[0, 1] = [0xFFBADBAD, 0x7F800001]   # negative NaN with a payload, a signalling NaN
    src[0, 2] = [0xFF800000, 0x00000001]   # -inf, the smallest subnormal
    out = scatter_agent_action(np.ones((1, 3, 2), np.float32), src.view(np.float32), types, N_TYPES, None)
    assert np.array_equal(_bits(out), src)
