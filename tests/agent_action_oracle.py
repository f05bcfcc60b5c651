"""NumPy restatement of DESIGN.md section 1 "Per-agent action" (K11, ``t2d_scatter_agent_action``).

Slot m of scenario n takes row q* of ``agent_action``, the lowest q with ``observers[n, q] == m``, when its type is active
(``type_id[n, m] < n_types``); every other row of ``action`` keeps its value.  The copy is of the fp32 bits, so NaN
payloads and -0.0 pass through."""

import numpy as np


def owner_rows(type_id, Q, observers=None):
    """int64 [N, M]: the row q* that owns each slot (the lowest q naming it), Q where no row names the slot."""
    N, M = type_id.shape
    obs = np.broadcast_to(np.arange(Q), (N, Q)) if observers is None else np.asarray(observers, dtype=np.int64)
    assert obs.shape == (N, Q)
    if observers is None:
        assert Q <= M
    owner = np.full((N, M), Q, dtype=np.int64)
    n, q = np.nonzero((obs >= 0) & (obs < M))
    np.minimum.at(owner, (n, obs[n, q]), q)
    return owner


def scatter_agent_action(action, agent_action, type_id, n_types, observers=None):
    """The action array after the scatter (a new array; ``action`` is not changed).

    action [N, M, 2] fp32, agent_action [N, Q, 2] fp32, type_id [N, M] uint8, observers [N, Q] int or None (row q is slot
    q, Q <= M)."""
    out = np.array(action, dtype=np.float32, copy=True)
    src = np.ascontiguousarray(agent_action, dtype=np.float32).view(np.uint32)
    N, M = type_id.shape
    Q = src.shape[1]
    assert src.shape == (N, Q, 2) and out.shape == (N, M, 2)
    owner = owner_rows(type_id, Q, observers)
    n, m = np.nonzero((owner < Q) & (np.asarray(type_id) < n_types))
    out.view(np.uint32)[n, m] = src[n, owner[n, m]]
    return out
