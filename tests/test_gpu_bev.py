"""K6, the BEV observation (t2d_bev_render), against the float64 oracle in tests/bev_oracle.py: class images bit-exact,
RGB = palette[class], eager = CUDA graph, invalid arguments rejected, and the env's "bev" observation."""

import numpy as np
import pytest

from tests import bev_oracle as B

pytestmark = pytest.mark.gpu


def _styles(world):
    from tactics2d_b200.sensor.camera import BEV_STYLES, STYLE_KEYS, default_type_style

    idx = {k: i for i, k in enumerate(STYLE_KEYS)}
    ts = [B.NOT_DRAWN if default_type_style(r) is None else idx[default_type_style(r)] for r in world.type_table.rows]
    z = [BEV_STYLES[k][1] for k in STYLE_KEYS]
    lw = [BEV_STYLES[k][2] for k in STYLE_KEYS]
    return idx, ts, z, lw


def _oracle(world, n, width, height, rng, tile=None, seg_style=None, target=None, target_style=B.NOT_DRAWN):
    idx, ts, z, lw = _styles(world)
    st = world.state_numpy()
    return B.render_world_scenario(n, st, world.type_id.cpu().numpy(), world.type_table.as_oracle_table(), ts, z, lw,
                                   width, height, rng, tile, seg_style, target, target_style)


def _c2_world(n=4096, m=64, seed=1):
    from tactics2d_b200 import BatchedWorld, synthetic

    s = synthetic.config2(n, m, seed=seed)
    w = BatchedWorld(n, m, s.table)
    w.set_map(s.segments, s.bounds)
    w.set_state(s.x, s.y, s.heading, s.speed, type_id=s.type_id)
    return w, s


def test_c2_class_image_bit_exact_and_rgb_is_palette(cuda_device):
    import torch
    from tactics2d_b200.sensor.camera import palette

    w, s = _c2_world()
    cls = w.bev(rgb=False).clone()
    rgb = w.bev(rgb=True)
    torch.cuda.synchronize()
    assert cls.shape == (4096, 200, 200) and rgb.shape == (4096, 200, 200, 3) and rgb.dtype == torch.uint8
    pal = torch.from_numpy(palette()).to(cls.device)
    assert torch.equal(pal[cls.long()], rgb)
    got = cls.cpu().numpy()
    tile = dict(segments=s.segments, poly_start=None, bounds=s.bounds)
    for n in np.random.default_rng(5).choice(4096, 64, replace=False):
        ref = _oracle(w, int(n), 200, 200, (20, 20, 20, 20), tile)
        assert np.array_equal(got[n], ref), (n, int((got[n] != ref).sum()))
    assert (got != 0).mean() > 0.01   # the scene draws something (1.7 % of the pixels at C2)
    w.close()


def test_graph_capture_equals_eager(cuda_device):
    import torch

    w, _ = _c2_world(256, 64)
    eager = w.bev(rgb=True).clone()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        w.bev(rgb=True)
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(g):
        out = w.bev(rgb=True)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    w.close()


def test_invalid_sizes_and_ranges_rejected(cuda_device):
    import ctypes as C

    import torch
    from tactics2d_b200 import _lib

    w, _ = _c2_world(4, 8)
    w.bev()
    buf = torch.empty(4 * 2048 * 2048 * 3, dtype=torch.uint8, device=cuda_device)
    for width, height, rng in ((0, 200, (20,) * 4), (200, -1, (20,) * 4), (1025, 200, (20,) * 4), (200, 2000, (20,) * 4),
                               (200, 200, (0, 20, 20, 20)), (200, 200, (20, -1, 20, 20)), (200, 200, (20, 20, float("nan"), 20)),
                               (200, 200, (20, 20, 20, 1e6))):
        r = np.asarray(rng, np.float32)
        code = w.lib.t2d_bev_render(w._ctx, width, height, C.c_void_p(r.ctypes.data), 1, C.c_void_p(buf.data_ptr()), None)
        assert code == -1, (width, height, rng)
    with pytest.raises(ValueError):
        w.bev(resolution=(2048, 200))
    with pytest.raises(_lib.T2DError):
        w.bev(perception_range=(20, 20, 0, 20))
    w.close()


def _ind_tiles():
    from tactics2d_b200.map import load_areas, polygons_to_segments, segment_style_keys

    tiles = []
    for name in ("inD_1", "inD_2"):
        areas = load_areas(name)
        xy = np.concatenate([a.outer for a in areas])
        b = (float(xy[:, 0].min()), float(xy[:, 0].max()), float(xy[:, 1].min()), float(xy[:, 1].max()))
        line = [(b[0] + 5, b[2] + 5), (b[1] - 5, b[3] - 5)]
        seg, ps = polygons_to_segments(areas, [line])
        tiles.append(dict(segments=seg, poly_start=ps, bounds=b, style=segment_style_keys(areas, [line], "roadline")))
    return tiles


def test_mixed_scene_on_ind_map_table_with_tile_rewrite(cuda_device):
    import torch
    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.sensor.camera import STYLE_KEYS
    from tactics2d_b200.types import TypeParams, TypeTable

    table = TypeTable([TypeParams.vehicle("medium_car"), TypeParams.cyclist("cyclist"), TypeParams.pedestrian("adult_male"),
                       TypeParams.obstacle(2.0, 1.0)])
    n, m = 32, 24
    tiles = _ind_tiles()
    rng = np.random.default_rng(3)
    tid = rng.integers(0, 2, n)
    w = BatchedWorld(n, m, table)
    w.set_map_table(tiles, tid)
    x, y = np.zeros((n, m), np.float32), np.zeros((n, m), np.float32)
    for i in range(n):
        b = tiles[tid[i]]["bounds"]
        cx, cy = (b[0] + b[1]) / 2, (b[2] + b[3]) / 2
        x[i] = cx + rng.uniform(-25, 25, m)
        y[i] = cy + rng.uniform(-25, 25, m)
    h = rng.uniform(-np.pi, np.pi, (n, m)).astype(np.float32)
    types = rng.integers(0, 4, (n, m)).astype(np.uint8)
    types[rng.random((n, m)) < 0.1] = 255
    types[5, 0] = 255   # one scenario without an ego: the view centres on its tile's bounds
    w.set_state(x, y, h, np.zeros((n, m), np.float32), type_id=types)
    target = np.stack([x[:, 0] + 3, y[:, 0] - 2, h[:, 0], np.full(n, 2.5), np.full(n, 1.2)], 1).astype(np.float32)
    w.set_goal(target)
    w.set_bev_styles()
    idx = {k: i for i, k in enumerate(STYLE_KEYS)}
    seg_style = [np.asarray([idx[k] for k in t["style"]], np.uint8) for t in tiles]
    for rewrite in (False, True):
        if rewrite:
            tid = 1 - tid
            w.tile_id.copy_(torch.from_numpy(tid.astype(np.int16)).to(cuda_device))
        for res, rng_ in (((200, 200), (20, 20, 20, 20)), ((160, 96), (12, 25, 30, 8))):
            got = w.bev(res, rng_, rgb=False).cpu().numpy()
            for i in range(n):
                ref = _oracle(w, i, res[0], res[1], rng_, tiles[tid[i]], seg_style[tid[i]], target, idx["target_area"])
                assert np.array_equal(got[i], ref), (rewrite, res, i, int((got[i] != ref).sum()))
    w.close()


def test_band_scene_pixel_centres_on_and_next_to_boundaries(cuda_device):
    """Range 16 at 256 px: pitch 0.125 m, pixel centres at 0.0625 + 0.125 k.  Box edges, disc rims (radius 0.625 about a
    pixel centre passes through the centres at offsets (0.375, 0.5)), ring edges and a stroke lie exactly on centres and
    1 float32 ulp to either side."""
    from tactics2d_b200 import BatchedWorld
    from tactics2d_b200.map import polygons_to_segments
    from tactics2d_b200.sensor.camera import STYLE_KEYS
    from tactics2d_b200.types import MODEL_POINTMASS_NEWTON, SHAPE_CIRCLE, SHAPE_OBB, TypeParams, TypeTable

    f32 = np.float32
    box = [f32(0.9375), np.nextafter(f32(0.9375), f32(2)), np.nextafter(f32(0.9375), f32(0))]
    rad = [f32(0.625), np.nextafter(f32(0.625), f32(2)), np.nextafter(f32(0.625), f32(0))]
    rows = [TypeParams(half_len=float(e), half_wid=float(e), shape=SHAPE_OBB, name="medium_car") for e in box]
    rows += [TypeParams(radius=float(r), half_len=float(r), half_wid=float(r), shape=SHAPE_CIRCLE,
                        model=MODEL_POINTMASS_NEWTON, name="adult_male") for r in rad]
    rows += [TypeParams.pedestrian("adult_male")]
    table = TypeTable(rows)
    n, m = 3, 4
    tiles = []
    for k in range(n):
        e = box[k]
        ring = np.asarray([(-e, -e), (-e - 3, -e), (-e - 3, -e - 3), (-e, -e - 3)], np.float32)
        seg, ps = polygons_to_segments([ring], [[(2.0, 2 * e), (6.0, 2 * e)], [(-6.0, 6.0 + e), (-6.0, 6.0 + e)]])
        tiles.append(dict(segments=seg, poly_start=ps, bounds=(-10.0, 10.0, -10.0, 10.0),
                          style=["keepout"] * 4 + ["roadline", "curbstone"]))
    w = BatchedWorld(n, m, table)
    w.set_map_table(tiles, np.arange(n))
    x = np.zeros((n, m), np.float32); y = np.zeros((n, m), np.float32)
    types = np.full((n, m), 255, np.uint8)
    for k in range(n):
        types[k, 0] = 6                                   # a pedestrian ego at the origin, heading 0
        x[k, 1], y[k, 1], types[k, 1] = 4.0, -4.0, k      # box edges at 4 +- 0.9375: pixel centres
        x[k, 2], y[k, 2], types[k, 2] = -3.9375, 4.0625, 3 + k
    w.set_state(x, y, np.zeros((n, m), np.float32), np.zeros((n, m), np.float32), type_id=types)
    got = w.bev((256, 256), (16, 16, 16, 16), rgb=False).cpu().numpy()
    idx = {k: i for i, k in enumerate(STYLE_KEYS)}
    for k in range(n):
        ss = np.asarray([idx[s] for s in tiles[k]["style"]], np.uint8)
        ref = _oracle(w, k, 256, 256, (16, 16, 16, 16), tiles[k], ss)
        assert np.array_equal(got[k], ref), (k, int((got[k] != ref).sum()))
    # on the edge counts, one ulp outside does not: the three scenarios differ exactly at the boundary centres
    assert not np.array_equal(got[0], got[2])
    w.close()


def test_env_bev_observation_after_auto_reset(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    s = synthetic.config2(64, 16, seed=2)
    env = BatchedTrafficEnv(s, max_step=3, observation="bev", bev_resolution=(120, 80), bev_range=(15, 15, 20, 10))
    assert env.observation_space["shape"] == (64, 80, 120, 3)
    obs, _ = env.reset()
    assert obs.shape == (64, 80, 120, 3) and obs.dtype == torch.uint8
    for _ in range(4):   # max_step 3: every scenario truncates and auto-resets within these steps
        obs, reward, term, trunc, info = env.step(torch.zeros((64, 2), device=cuda_device))
    first = obs.clone()
    assert torch.equal(first, env.world.bev((120, 80), (15, 15, 20, 10)))
    # the default env keeps the state observation
    env2 = BatchedTrafficEnv(s, max_step=3)
    o2, _ = env2.reset()
    assert env2.observation_space["dtype"] == "float32" and not (torch.is_tensor(o2) and o2.dtype == torch.uint8)
    env.close(); env2.close()
