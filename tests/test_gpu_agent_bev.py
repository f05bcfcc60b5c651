"""The per-agent BEV (t2d_bev_render_agents, BatchedWorld.bev_agents) against the float64 statement in
tests/agent_bev_oracle.py: class images bit for bit on sampled rows, RGB = palette[class], slot-0 rows = the ego image,
absent and retired rows all background, the dense-scene fallback from a slot other than 0, odd and ragged shapes, an output
past 2^31 bytes, CUDA graph = eager, the C-level rejections and the env's info["bev"].  Every output starts as a sentinel
fill, so that a skipped row or pixel fails."""

import ctypes as C

import numpy as np
import pytest

from tests import agent_bev_oracle as AB
from tests import bev_oracle as B
from tests.test_gpu_bev import _c2_world, _ind_tiles, _styles

SENTINEL = 0x5A   # no style index, and no palette colour is (90, 90, 90)


def _i16(a, device="cuda"):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, np.int16)).to(device)


def _f32(a, device="cuda"):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(device)


def _render(w, res, rng, rgb, observers=None, goals=None):
    """bev_agents into its buffer after a sentinel fill; returns the buffer (synchronised)."""
    import torch

    out = w.bev_agents(res, rng, rgb=rgb, observers=observers, goals=goals)
    out.fill_(SENTINEL)
    out = w.bev_agents(res, rng, rgb=rgb, observers=observers, goals=goals)
    torch.cuda.synchronize()
    return out


def _oracle_rows(w, res, rng, rows, observers=None, goals=None, tiles=None, seg_styles=None, target=None, target_style=None):
    idx, ts, z, lw = _styles(w)
    rng = (rng,) * 4 if np.ndim(rng) == 0 else rng
    if target_style is None:
        target_style = idx["target_area"]
    obs = None if observers is None else observers.cpu().numpy()
    g = None if goals is None else goals.cpu().numpy()
    return AB.render_agents(w.state_numpy(), w.type_id.cpu().numpy(), w.type_table.as_oracle_table(), ts, z, lw, res[0],
                            res[1], rng, obs, rows, tiles, seg_styles, target, g, target_style)


def _check(w, res, rng, rows, observers=None, goals=None, rgb_too=True, **kw):
    """Class images of ``rows`` bit for bit against the oracle, every class pixel a style, and RGB = palette[class] on
    every row.  Returns the class images (device)."""
    import torch
    from tactics2d_b200.sensor.camera import palette

    cls = _render(w, res, rng, False, observers, goals).clone()
    assert (cls != SENTINEL).all()
    if rgb_too:
        rgb = _render(w, res, rng, True, observers, goals)
        pal = torch.from_numpy(palette()).to(cls.device)
        for i in range(0, w.N, 256):   # in slices: the index tensor of a whole C2 batch would take 8 bytes a pixel
            assert torch.equal(pal[cls[i:i + 256].long()], rgb[i:i + 256]), (res, rng, i)
    got = cls.cpu().numpy()
    for (n, q), ref in _oracle_rows(w, res, rng, rows, observers, goals, **kw).items():
        assert np.array_equal(got[n, q], ref), (res, rng, n, q, int((got[n, q] != ref).sum()))
    return cls


# ------------------------------------------------------------------------------------------------------------- C2
@pytest.mark.gpu
def test_c2_observer_list_bit_exact_and_slot_zero_rows_equal_the_ego_image(cuda_device):
    import torch

    w, s = _c2_world()
    n, m, q = 4096, 64, 8
    rs = np.random.default_rng(7)
    obs = rs.integers(1, m, (n, q))
    obs[:, 0] = 0
    obs[:, 1] = -1
    obs[:, 2] = m
    obs[:, 3] = obs[:, 4]     # a duplicate
    obs[::3, 5] = 0           # slot 0 again in another column
    t = _i16(obs)
    tile = dict(segments=s.segments, poly_start=None)
    rows = [(int(a), int(b)) for a, b in zip(rs.choice(n, 40, replace=False), rs.integers(0, q, 40))]
    rows += [(n - 1, k) for k in range(q)]   # the last rows, past 2^31 bytes in RGB
    cls = _check(w, (200, 200), 20.0, rows, t, tiles=[tile] * n)
    ego = w.bev((200, 200), 20.0, rgb=False).clone()
    ego_rgb = w.bev((200, 200), 20.0, rgb=True).clone()
    assert (s.type_id[:, 0] < 255).all()
    assert torch.equal(cls[:, 0], ego) and torch.equal(cls[::3, 5], ego[::3])
    rgb = w.bev_agents((200, 200), 20.0, rgb=True, observers=t)
    assert rgb.shape == (n, q, 200, 200, 3) and rgb.numel() > 2**31
    assert torch.equal(rgb[:, 0], ego_rgb)
    assert not cls[:, 1:3].any()                     # -1 and M: absent
    assert torch.equal(cls[:, 3], cls[:, 4])         # duplicates
    assert (cls[:, 6:] != 0).float().mean() > 0.01   # the other rows draw
    # every slot (no list): row q is slot q
    full = _render(w, (48, 48), 20.0, False)
    assert full.shape == (n, m, 48, 48) and torch.equal(full[:, 0], w.bev((48, 48), 20.0, rgb=False))
    got = full.cpu().numpy()
    for (a, b), ref in _oracle_rows(w, (48, 48), 20.0, [(5, 63), (4095, 17), (4095, 63)], tiles=[tile] * n).items():
        assert np.array_equal(got[a, b], ref)
    del rgb, full
    w.close()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ mixed, map, goals
@pytest.mark.gpu
def test_mixed_types_on_ind_map_table_with_per_row_goals(cuda_device):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic
    from tactics2d_b200.sensor.camera import STYLE_KEYS
    from tactics2d_b200.types import SHAPE_NONE, TypeParams, TypeTable

    n, m, q = 48, 24, 10
    s = synthetic.with_inactive(synthetic.config4(n, m, seed=41, size=40.0), 0.2, seed=3)
    table = TypeTable(list(s.table.rows) + [TypeParams(shape=SHAPE_NONE, name="marker")])   # a shapeless type
    s.type_id[:, 0] = np.where(np.arange(n) % 4 == 1, len(table) - 1, s.type_id[:, 0])       # observes, is not drawn
    s.type_id[::7, 3] = len(table) - 1
    shapes = table.as_oracle_table()["shape"]
    assert set(shapes[s.type_id[s.type_id < 255]]) == {0, 1, 2} and (s.type_id == 255).any()
    tiles = _ind_tiles()
    rs = np.random.default_rng(4)
    tid = rs.integers(0, 2, n)
    w = BatchedWorld(n, m, table)
    w.set_map_table(tiles, tid)
    x, y = s.x.copy(), s.y.copy()
    for i in range(n):   # the participants around each tile's centre
        b = tiles[tid[i]]["bounds"]
        x[i] += (b[0] + b[1]) / 2 - x[i].mean()
        y[i] += (b[2] + b[3]) / 2 - y[i].mean()
    w.set_state(x, y, s.heading, s.speed, type_id=s.type_id)
    target = np.stack([x[:, 0] + 2, y[:, 0] - 1, s.heading[:, 0], np.full(n, 2.5), np.full(n, 1.2)], 1).astype(np.float32)
    w.set_goal(target)
    w.set_bev_styles()
    idx = {k: i for i, k in enumerate(STYLE_KEYS)}
    seg_style = [np.asarray([idx[k] for k in t["style"]], np.uint8) for t in tiles]
    obs = rs.integers(-2, m + 2, (n, q))
    obs[:, 0] = 0
    goals = np.full((n, q, 5), np.nan, np.float32)
    js = np.clip(obs, 0, m - 1)
    near = rs.random((n, q)) < 0.7   # a goal next to its observer, else NaN
    goals[near] = np.stack([x[np.arange(n)[:, None], js] + 3, y[np.arange(n)[:, None], js] + 1,
                            np.full((n, q), 0.4), np.full((n, q), 2.0), np.full((n, q), 1.0)], -1)[near]
    t, g = _i16(obs), _f32(goals)
    ts = [tiles[k] for k in tid]
    ss = [seg_style[k] for k in tid]
    rows = [(i, k) for i in range(0, n, 5) for k in range(q)]
    for res, rng in (((200, 200), 20.0), ((160, 96), (12.0, 25.0, 30.0, 8.0))):
        # without goals: slot 0's rows draw the target and equal the ego image
        cls = _check(w, res, rng, rows, t, tiles=ts, seg_styles=ss, target=target)
        present = torch.from_numpy(s.type_id[:, 0] < 255).to(cuda_device)
        assert torch.equal(cls[present, 0], w.bev(res, rng, rgb=False)[present])
        assert not cls[~present, 0].any()   # no slot 0: an absent row, not the ego image's no-ego view
        # with per-row goals
        cls = _check(w, res, rng, rows, t, g, tiles=ts, seg_styles=ss)
        assert (cls == idx["target_area"]).any()
    # goals hidden by their style
    w.set_bev_styles(target=None)
    cls = _check(w, (200, 200), 20.0, rows, t, g, tiles=ts, seg_styles=ss, target_style=B.NOT_DRAWN)
    assert not (cls == idx["target_area"]).any()
    w.close()


# -------------------------------------------------------------------------------------------------------- retirement
@pytest.mark.gpu
def test_retired_rows_are_background_and_their_bodies_gone_until_reset(cuda_device):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    N, M = 512, 16
    s = synthetic.config2(N, M, seed=21)
    w = BatchedWorld(N, M, s.table, max_step=1000)
    w.set_map(s.segments, s.bounds)
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in s.state().items()}
    w.type_id.copy_(torch.from_numpy(s.type_id).cuda())
    w.reset(torch.ones(N, dtype=torch.uint8, device=cuda_device), pool)
    w.set_agents()
    types0 = w.type_id.clone()
    res, rng = (96, 96), 25.0
    before = _render(w, res, rng, False).clone()
    for k in range(6):
        w.step(torch.from_numpy(synthetic.random_actions(900 + k, (N, M))).cuda())
        w.agents_epilogue()
    gone = w.type_id == 255
    assert gone.sum() > 20
    cls = _render(w, res, rng, False).clone()
    assert not cls[gone].any()
    tile = dict(segments=s.segments, poly_start=None)
    sel = torch.nonzero(gone.any(1)).flatten().cpu().numpy()[:12]
    rows = [(int(a), k) for a in sel for k in range(M)]
    _check(w, res, rng, rows, tiles=[tile] * N, rgb_too=False)
    # the same poses with the retired slots back in place: some present row saw a retired body
    w.type_id.copy_(types0)
    back = _render(w, res, rng, False).clone()
    assert not torch.equal(back[~gone], cls[~gone])
    w.type_id.copy_(torch.where(gone, torch.full_like(types0, 255), types0))
    mask = torch.zeros(N, dtype=torch.uint8, device=cuda_device)
    mask[::2] = 1
    w.reset(mask, pool)
    mk = mask.bool()
    after = _render(w, res, rng, False).clone()
    assert torch.equal(after[mk], before[mk])   # the reset scenarios are back at their first episode's images
    assert (gone & mk[:, None]).any() and after[gone & mk[:, None]].any()
    _check(w, res, rng, rows, tiles=[tile] * N, rgb_too=False)
    w.close()


# --------------------------------------------------------------------------------------------------- dense fallback
@pytest.mark.gpu
def test_dense_fallback_seen_from_a_slot_other_than_zero(cuda_device):
    """The four scenes of test_gpu_bev_rare_paths' dense world, with a pedestrian on the ego's centre facing back in slot
    20: seen from it (the view turned by pi) they hold 317, 513, 513 and 687 visible primitives, so rows 1..3 take the
    fallback that rebuilds every candidate at every pixel."""
    import torch
    from tests import test_gpu_bev_rare_paths as R

    rs = np.random.default_rng(11)   # the fixture's scenes, drawn in its order
    m = 128
    tiles = [R._dense_tile(rs, 100), R._dense_tile(rs, 470)]
    plan = [(0, 96, 10, True), (1, 10, 8, False), (1, 10, 8, True), (1, 96, 10, True)]
    slots = {}
    x, y, h = (np.zeros((4, m), np.float32) for _ in range(3))
    types = np.zeros((4, m), np.uint8)
    target = np.zeros((4, 5), np.float32)
    for n, (t, n_fill, n_ped, goal) in enumerate(plan):
        if (n_fill, n_ped) not in slots:
            slots[(n_fill, n_ped)] = R._dense_slots(rs, m, n_fill, n_ped)
        x[n], y[n], h[n], types[n] = slots[(n_fill, n_ped)]
        gx, gy = R._rot(R.EGO, -16.0 if goal else -R.FAR - 30, 6.0)
        target[n] = (gx, gy, R.EGO[2] + 0.2, 2.5, 1.2)
    assert (types[:, 20] == R.EMPTY).all()
    x[:, 20], y[:, 20], h[:, 20], types[:, 20] = x[:, 0], y[:, 0], np.float32(R.EGO[2] + np.pi), R.PED
    tid = np.asarray([p[0] for p in plan])
    w = R._world(4, m, x, y, h, types, tiles, tid, target)
    idx, ts, z, lw = _styles(w)
    tab = w.type_table.as_oracle_table()
    ss = [np.asarray([idx[k] for k in tiles[k]["style"]], np.uint8) for k in tid]
    P = []
    for n in range(4):
        args = (x[n], y[n], h[n], types[n], tab, ts, z, lw, B.window(*R.FB_RES, R.FB_RNG)[2], tiles[tid[n]]["segments"],
                tiles[tid[n]]["poly_start"], ss[n], None, B.NOT_DRAWN)
        P.append(R.count_visible(args, B.view_of(x[n, 20], y[n, 20], h[n, 20], True), *R.FB_RES, R.FB_RNG))
    assert P == [317, 513, 513, 687]
    obs = _i16(np.tile([20, 0, 20, 7], (4, 1)))
    rows = [(n, k) for n in range(4) for k in range(4)]
    cls = _check(w, R.FB_RES, R.FB_RNG, rows, obs, tiles=[tiles[k] for k in tid], seg_styles=ss, target=target)
    assert torch.equal(cls[:, 0], cls[:, 2]) and torch.equal(cls[:, 1], w.bev(R.FB_RES, R.FB_RNG, rgb=False))
    assert not torch.equal(cls[:, 0], cls[:, 1])
    # per-row goals: slot 20 draws one in front of it (514 in scene 2)
    goals = np.full((4, 4, 5), np.nan, np.float32)
    goals[:, 0] = target
    cls = _check(w, R.FB_RES, R.FB_RNG, rows, obs, _f32(goals), tiles=[tiles[k] for k in tid], seg_styles=ss)
    assert (cls[:, 0] == idx["target_area"]).any() and not (cls[:, 1:] == idx["target_area"]).any()
    w.close()


# ------------------------------------------------------------------------------------------------ odd and ragged shapes
def _small_world(n, m, seed, size=30.0):
    from tactics2d_b200 import BatchedWorld, synthetic

    s = synthetic.with_inactive(synthetic.config4(n, m, seed=seed, size=size), 0.15, seed=seed)
    w = BatchedWorld(n, m, s.table)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    return w, dict(segments=s.segments, poly_start=None)


@pytest.mark.gpu
@pytest.mark.parametrize("res", [(37, 23), (1, 1), (1024, 1), (1, 1024), (129, 17)])
def test_odd_image_sizes(cuda_device, res):
    w, tile = _small_world(5, 12, seed=8)
    obs = _i16(np.random.default_rng(1).integers(-1, 13, (5, 3)))
    rows = [(n, k) for n in range(5) for k in range(3)]
    _check(w, res, (15.0, 10.0, 20.0, 12.0), rows, obs, tiles=[tile] * 5)
    w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 33, 128])
@pytest.mark.parametrize("q", [1, 33, 128])
def test_ragged_rows_and_slots_at_odd_n(cuda_device, m, q):
    n = 7
    w, tile = _small_world(n, m, seed=m + q, size=25.0 + m / 4)
    rs = np.random.default_rng(m * 1000 + q)
    obs = rs.integers(-1, m + 1, (n, q))
    rows = [(n - 1, q - 1), (0, 0)] + [(int(a), int(b)) for a, b in zip(rs.integers(0, n, 10), rs.integers(0, q, 10))]
    _check(w, (48, 40), 18.0, rows, _i16(obs), tiles=[tile] * n)
    if q == m:   # no list: row k is slot k
        _check(w, (48, 40), 18.0, [(n - 1, q - 1), (3, 0)], None, tiles=[tile] * n)
    w.close()


# ------------------------------------------------------------------------------------------------ beyond 2^31 bytes
@pytest.mark.gpu
def test_class_output_beyond_2_to_the_31_bytes(cuda_device):
    import torch

    free, _ = torch.cuda.mem_get_info()
    if free < 8 * 2**30:
        pytest.skip(f"needs 8 GB of free device memory, {free / 2**30:.1f} GB free")
    n, m, q = 4096, 64, 16
    assert n * q * 200 * 200 > 2**31
    w, s = _c2_world(n, m, seed=3)
    obs = np.random.default_rng(9).integers(0, m, (n, q))
    obs[-1, -1] = 0
    t = _i16(obs)
    got = _render(w, (200, 200), 20.0, False, t)
    assert (got[-2:] != SENTINEL).all()
    tile = dict(segments=s.segments, poly_start=None)
    cpu = got[-2:].cpu().numpy()
    for (a, b), ref in _oracle_rows(w, (200, 200), 20.0, [(n - 2, k) for k in range(q)] + [(n - 1, k) for k in range(q)],
                                    t, tiles=[tile] * n).items():
        assert np.array_equal(cpu[a - (n - 2), b], ref), (a, b)
    assert torch.equal(got[-1, -1], w.bev((200, 200), 20.0, rgb=False)[-1])
    del got
    w._agent_bev.clear()
    w.close()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------ graph capture
@pytest.mark.gpu
def test_graph_capture_equals_eager(cuda_device):
    import torch

    w, _ = _c2_world(256, 64)
    rs = np.random.default_rng(2)
    obs = _i16(rs.integers(-1, 64, (256, 12)))
    goals = np.full((256, 12, 5), np.nan, np.float32)
    goals[:, ::2] = (0.0, 0.0, 0.3, 3.0, 2.0)
    for kw in (dict(rgb=True), dict(rgb=False, observers=obs), dict(rgb=True, observers=obs, goals=_f32(goals))):
        eager = w.bev_agents((200, 200), 20.0, **kw).clone()
        g = torch.cuda.CUDAGraph()
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            w.bev_agents((200, 200), 20.0, **kw)
        torch.cuda.current_stream().wait_stream(st)
        with torch.cuda.graph(g):
            out = w.bev_agents((200, 200), 20.0, **kw)
        out.fill_(SENTINEL)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)
    w.close()


# ------------------------------------------------------------------------------------------------------ rejections
@pytest.mark.gpu
def test_c_level_rejections_launch_nothing(cuda_device):
    import torch
    from tactics2d_b200 import _lib

    w, _ = _c2_world(8, 8)
    lib = w.lib
    obs = _i16(np.zeros((8, 4)))
    ego = w.bev((32, 32), 20.0, rgb=False).clone()
    rows = w.bev_agents((32, 32), 20.0, rgb=False, observers=obs).clone()
    out = torch.full((8 * 128 * 64 * 64 * 3,), 7, dtype=torch.uint8, device=cuda_device)
    p = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731
    r20 = np.full(4, 20.0, np.float32)
    rng = lambda r: C.c_void_p(r.ctypes.data)   # noqa: E731

    def call(ctx=w._ctx, o=p(obs), q=4, goals=None, width=32, height=32, r=r20, o_=p(out)):
        return lib.t2d_bev_render_agents(ctx, o, q, goals, width, height, None if r is None else rng(r), 1, o_, None)

    def still_works():
        assert torch.equal(w.bev((32, 32), 20.0, rgb=False), ego)
        assert torch.equal(w.bev_agents((32, 32), 20.0, rgb=False, observers=obs), rows)

    n0 = lib.t2d_launch_count()
    cases = [dict(q=0), dict(q=-1), dict(q=129), dict(o=None, q=9),                  # rows
             dict(width=0), dict(height=-1), dict(width=1025), dict(height=2000),       # sizes
             dict(r=None), dict(o_=None), dict(ctx=None)]
    cases += [dict(r=np.asarray(v, np.float32)) for v in ((0, 20, 20, 20), (20, -1, 20, 20), (20, 20, np.nan, 20),
                                                          (20, 20, 20, 1e6))]
    for kw in cases:
        assert call(**kw) == -1, kw
        still_works()
    n1 = lib.t2d_launch_count()
    ctx = C.c_void_p()   # a context whose state is not bound
    _lib.check(lib.t2d_create(C.byref(ctx), 0, 8, 8, C.byref(_lib.Config(100, 5, 0, 0))))
    _lib.check(lib.t2d_set_type_table(ctx, w.type_table.to_c_array(), len(w.type_table)))
    assert call(ctx=ctx) == -4
    lib.t2d_destroy(ctx)
    w2, _ = _c2_world(8, 8)   # a world whose styles are not set
    assert call(ctx=w2._ctx) == -4
    w2.close()
    torch.cuda.synchronize()
    assert n1 == n0 + 2 * len(cases) and lib.t2d_launch_count() == n1 and (out == 7).all()
    still_works()
    # the limits themselves are accepted, and Q > M with a list
    big = _i16(np.zeros((8, 128)))
    assert call(o=p(big), q=128) == 0 and call(o=None, q=8) == 0
    # the Python checks keep host tensors, wrong dtypes and shapes away from the kernel
    for bad in (torch.zeros((8, 2), dtype=torch.int16), torch.zeros((8, 2), dtype=torch.int32, device=cuda_device),
                torch.zeros((8, 129), dtype=torch.int16, device=cuda_device),
                torch.zeros((4, 2), dtype=torch.int16, device=cuda_device),
                torch.zeros((2, 8), dtype=torch.int16, device=cuda_device).t()):
        with pytest.raises(ValueError):
            w.bev_agents(observers=bad)
    with pytest.raises(ValueError):
        w.bev_agents(observers=obs, goals=torch.zeros((8, 3, 5), device=cuda_device))
    with pytest.raises(ValueError):
        w.bev_agents((2048, 200), observers=obs)
    with pytest.raises(_lib.T2DError):
        w.bev_agents(perception_range=0.0, observers=obs)
    still_works()
    w.close()


@pytest.mark.gpu
def test_more_rows_than_the_grid_holds_is_unsupported(cuda_device):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    free, _ = torch.cuda.mem_get_info()
    if free < 8 * 2**30:
        pytest.skip(f"needs 8 GB of free device memory, {free / 2**30:.1f} GB free")

    n = 2**24 + 1   # N · 128 > 2^31 - 1
    w = BatchedWorld(n, 1, synthetic.config2(4, 1).table)
    w.set_bev_styles()
    one = torch.zeros(16, dtype=torch.int16, device=cuda_device)
    r = np.full(4, 20.0, np.float32)
    n0 = w.lib.t2d_launch_count()
    code = w.lib.t2d_bev_render_agents(w._ctx, C.c_void_p(one.data_ptr()), 128, None, 8, 8, C.c_void_p(r.ctypes.data), 0,
                                       C.c_void_p(one.data_ptr()), None)
    assert code == -3 and b"2^31" in w.lib.t2d_last_error()
    assert w.lib.t2d_launch_count() == n0
    w.close()
    torch.cuda.empty_cache()


# -------------------------------------------------------------------------------------------------------- camera, env
@pytest.mark.gpu
def test_camera_render_agents(cuda_device):
    import torch
    from tactics2d_b200.sensor import BEVCamera

    w, _ = _c2_world(32, 16)
    cam = BEVCamera(perception_range=15.0, resolution=(64, 48))
    got = cam.render_agents(w)
    assert got.shape == (32, 16, 48, 64, 3) and cam.observation is got
    assert torch.equal(got[:, 0], cam.render(w))
    obs = _i16(np.tile([3, 0], (32, 1)))
    assert torch.equal(cam.render_agents(w, obs, rgb=False)[:, 1], w.bev((64, 48), 15.0, rgb=False))
    with pytest.raises(ValueError):
        BEVCamera(id_=2)
    w.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["vector", "agents"])
def test_env_info_bev_after_auto_resets(cuda_device, mode):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    n, m = 64, 16
    s = synthetic.config2(n, m, seed=2)
    rs = np.random.default_rng(3)
    obs = _i16(rs.integers(0, m, (n, 5)))
    goals = np.full((n, 5, 5), np.nan, np.float32)
    goals[:, 1] = (0.0, 0.0, 0.0, 2.0, 1.0)
    cam = dict(resolution=(64, 48), perception_range=15.0, rgb=False)
    kw = dict(observation=mode, camera=cam, vector_obs=dict(k_agents=4, k_segments=6))
    if mode == "agents":
        kw["vector_obs"].update(observers=obs, goals=_f32(goals))
        kw.update(agent_rewards=True, agent_actions=True)
    env = BatchedTrafficEnv(s, max_step=3, **kw)
    _, info = env.reset()
    shape = (n, 5, 48, 64) if mode == "agents" else (n, 48, 64)
    assert info["bev"].shape == shape and info["bev"].dtype == torch.uint8
    act = torch.full(env.action_space["shape"], 0.1, device=cuda_device)
    reset_seen = False
    for _ in range(5):   # max_step 3: every scenario ends and auto-resets within these steps
        info = env.step(act)[4]
        got = info["bev"].clone()
        w = env.world
        want = (w.bev_agents((64, 48), 15.0, rgb=False, observers=obs, goals=kw["vector_obs"]["goals"])
                if mode == "agents" else w.bev((64, 48), 15.0, rgb=False))
        assert got.shape == shape and torch.equal(got, want)
        reset_seen = reset_seen or bool((w.step_count == 0).any())
    assert reset_seen
    env.close()


def test_env_camera_arguments_rejected():
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = synthetic.config2(4, 4, seed=2)
    with pytest.raises(ValueError):
        BatchedTrafficEnv(s, observation="bev", camera=dict(resolution=(64, 64)))
    with pytest.raises(ValueError):
        BatchedTrafficEnv(s, camera=dict(resolution=(64, 64), range=20.0))
