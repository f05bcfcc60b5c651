"""K7, log replay (t2d_set_log), on the device: replayed state and type ids bit-exact against oracle/replay.py through ticks and
masked resets, teacher-forced ticks with replayed and kinematic participants mixed against the float64 tick oracle, the
BEV of a freshly reset scenario, the env over a log, CUDA-graph / host-path / unbinding equivalences, and the C-level
rejections of malformed logs."""

import numpy as np
import pytest

from oracle import replay as R
from oracle import scenario as O
from tests import bev_oracle as B
from tests.util import assert_state_close

pytestmark = pytest.mark.gpu

KEYS = ("x", "y", "heading", "speed", "vx", "vy")


def _world(ep, interval=100, **kw):
    import torch
    from tactics2d_b200 import BatchedWorld

    P, M = ep.type_id.shape
    w = BatchedWorld(P, M, ep.table, interval=interval, **kw)
    w.set_log(ep.log, ep.t0, ep.row_track)
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in ep.pool.items()}
    w.type_id.copy_(torch.from_numpy(ep.type_id).cuda())
    w.reset(torch.ones(P, dtype=torch.uint8, device="cuda"), pool)
    return w, pool


def _snap(w):
    st = w.state_numpy()
    row = None if w.log_row is None else w.log_row.cpu().numpy()
    return st, w.type_id.cpu().numpy(), w.step_count.cpu().numpy(), row


def _check_replay(ep, w, pre_state, pre_tid, offset, what, mask=None):
    """The world's replayed slots equal the oracle applied to the pre-replay state, bit for bit (the other slots' types
    untouched).  Returns the oracle's presence mask."""
    st, tid, cnt, row = _snap(w)
    step = cnt - offset   # K7 ran with the step count before K1 incremented it (tick) or after K2 zeroed it (reset)
    ref, ref_tid = R.apply(pre_state, pre_tid, ep.log, ep.t0, ep.row_track, row, step, w.interval, offset, mask)
    rep, pres, _, _ = R.sample(ep.log, ep.t0, ep.row_track, row, step, w.interval, offset)
    if mask is not None:
        rep = rep & np.asarray(mask, bool)[:, None]
        pres = pres & np.asarray(mask, bool)[:, None]
    assert np.array_equal(tid[rep], ref_tid[rep]), what
    assert np.array_equal(tid[~rep], np.asarray(pre_tid)[~rep]), what
    for k in KEYS:
        assert np.array_equal(st[k][rep].view(np.uint32), ref[k][rep].view(np.uint32)), (what, k)
    return pres


@pytest.mark.parametrize("interval", [40, 100, 120])
def test_replayed_state_bit_exact_through_ticks_and_shuffled_resets(cuda_device, interval):
    import torch
    from tactics2d_b200 import synthetic

    N, M = 512, 64
    ep = synthetic.replay_episodes(N, M, 3000, seed=interval, duration_ms=20000, max_frames=60, horizon_ms=3000)
    w, pool = _world(ep, interval)
    pres_hist = []
    rng = np.random.default_rng(interval)
    st0 = {k: v for k, v in ep.pool.items()}
    pres_hist.append(_check_replay(ep, w, st0, ep.type_id, 0, "initial reset"))
    for t in range(36):
        st, tid, _, _ = _snap(w)
        if t % 9 == 8:   # masked reset onto shuffled rows
            mask = rng.uniform(0, 1, N) < 0.4
            idx = rng.permutation(N).astype(np.int32)
            w.reset(torch.from_numpy(mask.astype(np.uint8)).cuda(), pool, torch.from_numpy(idx).cuda())
            torch.cuda.synchronize()
            row = w.log_row.cpu().numpy()
            assert np.array_equal(row[mask], idx[mask])
            pre = {k: np.where(mask[:, None], ep.pool[k][idx], st[k]).astype(np.float32) for k in KEYS}
            pres_hist.append(_check_replay(ep, w, pre, tid, 0, f"reset {t}", mask))
            assert (w.step_count.cpu().numpy()[mask] == 0).all()
            continue
        act = torch.from_numpy(synthetic.random_actions(t, (N, M))).cuda()
        w.step(act)
        torch.cuda.synchronize()
        pres_hist.append(_check_replay(ep, w, st, tid, 1, f"tick {t}"))
    h = np.stack(pres_hist)
    assert (~h[:-1] & h[1:]).sum() > 100 and (h[:-1] & ~h[1:]).sum() > 100   # tracks appear and vanish mid-episode
    assert h.mean() > 0.03
    w.close()


def _events_by_tile(st, tid, table, tiles, tile_id):
    N, M = tid.shape
    fl = np.zeros((N, M), np.uint8); hi = np.full((N, M), -1, np.int16); hs = np.full((N, M), -1, np.int16)
    for k, t in enumerate(tiles):
        sel = tile_id == k
        if sel.any():
            f, i, s = O.events(st["x"][sel], st["y"][sel], st["heading"][sel], tid[sel], table, t["segments"], t["bounds"])
            fl[sel], hi[sel], hs[sel] = f, i, s
    return fl, hi, hs


@pytest.mark.parametrize("tables", ["kin_only", "fp64_models"])
def test_teacher_forced_ticks_mixed_replay_and_kinematics(cuda_device, tables):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.types import MODEL_KINEMATICS, TypeTable

    N, M = 256, 32
    base = TypeTable.vehicles() if tables == "kin_only" else TypeTable.from_templates("kinematics")
    ep = synthetic.replay_episodes(N, M, 1500, seed=11, table=base, size=80.0, duration_ms=15000, max_frames=80, horizon_ms=2000)
    # half of each row's NPC slots are kinematic participants instead of replayed ones
    rt = ep.row_track.copy()
    tid0 = ep.type_id.copy()
    free = np.zeros_like(rt, bool)
    free[:, 1::2] = True
    free[:, 0] = False
    rt[free] = -1
    rng = np.random.default_rng(3)
    tid0[free] = rng.integers(0, 9, free.sum())
    for k in KEYS:
        ep.pool[k][free] = rng.uniform(0, 80, free.sum()).astype(np.float32) if k in ("x", "y") else ep.pool[k][0, 0]
    ep.row_track, ep.type_id = rt, tid0
    tiles = [dict(segments=synthetic.grid_wall_segments(80.0, 40.0, 8.0), bounds=(-5.0, 85.0, -5.0, 85.0)),
             dict(segments=np.asarray([[0, 40, 80, 40]], np.float32), bounds=(-20.0, 100.0, -20.0, 100.0))]
    tile_id = (np.arange(N) % 2).astype(np.int64)
    w, pool = _world(ep, 100, max_step=8)
    w.set_map_table(tiles, tile_id)
    table = ep.table.as_oracle_table()
    model = np.asarray(table["model"])
    n_fl = 0
    for t in range(10):
        st, tid, cnt, row = _snap(w)
        act = synthetic.random_actions(50 + t, (N, M))
        r = w.step(torch.from_numpy(act).cuda())
        torch.cuda.synchronize()
        _check_replay(ep, w, st, tid, 1, f"tick {t}")
        got, gtid, gcnt, _ = _snap(w)
        ref = O.physics_tick(st, gtid, act, table, 100, 5)
        kin = (gtid != 255) & (model[np.where(gtid == 255, 0, gtid)] == MODEL_KINEMATICS)
        assert_state_close(got, ref, kin, what=f"tick {t}")
        fl, hi, hs = _events_by_tile(got, gtid, table, tiles, tile_id)
        assert np.array_equal(fl, r.flags.cpu().numpy()) and np.array_equal(hi, r.hit_index.cpu().numpy())
        assert np.array_equal(hs, r.hit_segment.cpu().numpy())
        stt, done = O.status(fl, gtid, gcnt, 8)
        assert np.array_equal(stt, r.status.cpu().numpy()) and np.array_equal(done, r.done.cpu().numpy())
        n_fl += int((fl[kin | (gtid != 255)] != 0).sum())
    assert n_fl > 0
    w.close()


def _styles(world):
    from tactics2d_b200.sensor.camera import BEV_STYLES, STYLE_KEYS, default_type_style

    idx = {k: i for i, k in enumerate(STYLE_KEYS)}
    ts = [B.NOT_DRAWN if default_type_style(r) is None else idx[default_type_style(r)] for r in world.type_table.rows]
    return ts, [BEV_STYLES[k][1] for k in STYLE_KEYS], [BEV_STYLES[k][2] for k in STYLE_KEYS]


def test_reset_scenario_shows_its_t0_traffic_in_the_bev(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    ep = synthetic.replay_episodes(64, 24, 800, seed=4, size=60.0, duration_ms=8000, max_frames=100)
    env = BatchedTrafficEnv(None, replay=ep, max_step=3, observation="bev", bev_resolution=(120, 100), bev_range=(25, 25, 25, 25))
    obs, _ = env.reset(options={"shuffle": True})
    w = env.world
    torch.cuda.synchronize()
    row = w.log_row.cpu().numpy()
    st, tid, cnt, _ = _snap(w)
    assert (cnt == 0).all() and len(set(row.tolist())) == 64
    _, pres, s, rtid = R.sample(ep.log, ep.t0, ep.row_track, row, cnt, w.interval, 0)
    assert pres.sum() > 64
    for k in KEYS:
        assert np.array_equal(st[k][pres], s[k][pres]), k
    assert np.array_equal(tid[pres], rtid[pres]) and np.array_equal(tid[:, 0], ep.type_id[row, 0])
    cls = w.bev((120, 100), (25, 25, 25, 25), rgb=False).cpu().numpy()
    ts, z, lw = _styles(w)
    table = w.type_table.as_oracle_table()
    for n in range(0, 64, 5):
        ref = B.render_world_scenario(n, st, tid, table, ts, z, lw, 120, 100, (25, 25, 25, 25), None, None, None, B.NOT_DRAWN)
        assert np.array_equal(cls[n], ref), n
    env.close()


def test_env_over_a_log_across_auto_resets(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    N, M = 128, 16
    ep = synthetic.replay_episodes(N, M, 1200, seed=8, size=100.0, duration_ms=10000, max_frames=120)
    env = BatchedTrafficEnv(None, replay=ep, max_step=5)
    env.reset(seed=1, options={"shuffle": True})
    w = env.world
    table = w.type_table.as_oracle_table()
    rng = np.random.default_rng(0)
    resets = 0
    for t in range(14):
        st, tid, cnt, row = _snap(w)
        a = rng.uniform(-0.5, 0.5, (N, 2)).astype(np.float32)
        _, _, term, trunc, _ = env.step(torch.from_numpy(a).cuda())
        torch.cuda.synchronize()
        done = (term | trunc).cpu().numpy()
        resets += int(done.sum())
        got, gtid, gcnt, grow = _snap(w)
        assert np.array_equal(grow, row)                                          # an auto-reset restarts the same row
        assert (gcnt[done] == 0).all() and (gcnt[~done] == cnt[~done] + 1).all()
        _, pres, s, rtid = R.sample(ep.log, ep.t0, ep.row_track, grow, gcnt, w.interval, 0)
        for k in KEYS:
            assert np.array_equal(got[k][pres], s[k][pres]), (t, k)             # the NPC slots follow the log
        rep = ep.row_track[grow] >= 0
        assert np.array_equal(gtid[rep], rtid[rep])
        act = np.zeros((N, M, 2), np.float32)
        act[:, 0] = a
        ref = O.physics_tick(st, tid, act, table, 100, 5, steer_first=True)   # the ego follows the policy
        ego = np.zeros((N, M), bool)
        ego[~done, 0] = True
        assert_state_close(got, ref, ego, what=f"ego step {t}")
        for k in KEYS:
            assert np.array_equal(got[k][done, 0], ep.pool[k][grow[done], 0]), k
    assert resets >= N   # every scenario ran past max_step at least once
    env.close()


def test_graph_host_paths_and_unbinding(cuda_device, monkeypatch):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    monkeypatch.setenv("T2D_HOST_CHUNKS", "4")   # step_host in four chunks of 128 scenarios
    N, M = 512, 32
    ep = synthetic.replay_episodes(N, M, 2000, seed=9, duration_ms=15000, max_frames=80)
    ws = [_world(ep, 100)[0] for _ in range(4)]
    ego_eager, _ = _world(ep, 100)
    acts = [torch.from_numpy(synthetic.random_actions(200 + t, (N, M))).cuda() for t in range(6)]
    # eager / CUDA graph / step_host / step_host_ego (zero NPC actions: the eager world gets the same); one warm-up tick
    # each on a side stream before the capture
    static = torch.zeros_like(acts[0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ws[0].step(static); ws[1].step(static); ego_eager.step(static)
        ws[2].step_host(static.cpu().numpy()); ws[3].step_host_ego(static[:, 0].cpu().numpy())
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ws[1].step(static)
    for t, a in enumerate(acts):
        ws[0].step(a)
        static.copy_(a)
        g.replay()
        ws[2].step_host(a.cpu().numpy())
    for t, a in enumerate(acts):
        full = torch.zeros_like(a)
        full[:, 0] = a[:, 0]
        ego_eager.step(full)
        ws[3].step_host_ego(a[:, 0].cpu().numpy())
    torch.cuda.synchronize()
    ref = _snap(ws[0])
    assert int(ref[2][0]) == 7
    for other in (ws[1], ws[2]):
        got = _snap(other)
        for k in KEYS:
            assert np.array_equal(got[0][k], ref[0][k]), k
        assert np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2])
    ge, gh = _snap(ego_eager), _snap(ws[3])
    for k in KEYS:
        assert np.array_equal(ge[0][k], gh[0][k]), k
    assert np.array_equal(ge[1], gh[1])
    for snap in (ref, gh):   # every path replayed: the slots hold the log at the current step
        _, pres, smp, _ = R.sample(ep.log, ep.t0, ep.row_track, snap[3], snap[2], 100, 0)
        assert pres.sum() > 1000
        for k in KEYS:
            assert np.array_equal(snap[0][k][pres], smp[k][pres]), k
    # set_log(None): the world then ticks like one that never had a log
    plain = BatchedWorld(N, M, ep.table, interval=100)
    st, tid, cnt, _ = _snap(ws[0])
    plain.set_state(st["x"], st["y"], st["heading"], st["speed"], st["vx"], st["vy"], type_id=tid)
    plain.step_count.copy_(torch.from_numpy(cnt).cuda())
    ws[0].set_log(None)
    assert ws[0].log_row is None
    for a in acts[:3]:
        ws[0].step(a); plain.step(a)
    torch.cuda.synchronize()
    a_, b_ = _snap(ws[0]), _snap(plain)
    for k in KEYS:
        assert np.array_equal(a_[0][k], b_[0][k]), k
    assert np.array_equal(a_[1], b_[1])
    for x in ws + [ego_eager, plain]:
        x.close()


def test_set_log_rejects_malformed_logs_without_a_launch(cuda_device):
    import ctypes as C
    import torch
    from dataclasses import replace
    from tactics2d_b200 import _lib, synthetic
    from tactics2d_b200.types import TypeTable

    ep = synthetic.replay_episodes(16, 8, 40, seed=2, duration_ms=4000, max_frames=20)
    w, _ = _world(ep, 100)
    lib = _lib.load()
    log = ep.log
    rec = log.records

    def rejected(lg=log, t0=ep.t0, rt=ep.row_track, match=""):
        n0 = lib.t2d_launch_count()
        with pytest.raises(_lib.T2DError, match=match):
            w.set_log(lg, t0, rt)
        assert lib.t2d_launch_count() == n0

    rejected(replace(log, type_row=np.where(np.arange(len(log)) == 3, 0, log.type_row).astype(np.uint8)), match="T2D_MODEL_STATIC")
    rejected(replace(log, type_row=np.full(len(log), 200, np.uint8)), match="outside the type table")
    bad = ep.row_track.copy(); bad[2, 3] = len(log)
    rejected(rt=bad, match="outside")
    bad = ep.row_track.copy(); bad[2, 3] = -2
    rejected(rt=bad, match="outside")
    bad = ep.row_track.copy(); bad[5, 1] = 7; bad[5, 6] = 7
    rejected(rt=bad, match="bound twice")
    rejected(replace(log, period_ms=np.where(np.arange(len(log)) == 1, 0, log.period_ms).astype(np.int32)), match="period")
    rejected(replace(log, period_ms=np.where(np.arange(len(log)) == 1, -40, log.period_ms).astype(np.int32)), match="period")
    nf = log.n_frames.copy(); k = int(np.argmax(nf > 0)); cut = int(log.rec_off[k])
    rejected(replace(log, n_frames=np.where(np.arange(len(log)) == k, 0, nf).astype(np.int32),
                     records=np.delete(rec, np.s_[cut:cut + nf[k]], 0)), match="no frames")
    for v in (np.nan, np.inf):
        r2 = rec.copy(); r2[17, 2] = v
        rejected(replace(log, records=r2), match="not finite")
    # the type_id pointer must be the bound one
    keep = dict(first=log.first_ms, n_frames=log.n_frames, period=log.period_ms, type_row=log.type_row, records=rec,
                t0=ep.t0, row_track=ep.row_track)
    other = torch.zeros_like(w.type_id)
    n0 = lib.t2d_launch_count()
    code = lib.t2d_set_log(w._ctx, C.byref(w._log_struct(keep, w.log_row, other)))
    assert code == -1 and b"bound" in lib.t2d_last_error() and lib.t2d_launch_count() == n0
    # the good log stays bound; a type table that makes a replayed track's row non-static is rejected
    with pytest.raises(_lib.T2DError, match="T2D_MODEL_STATIC"):
        w.set_type_table(TypeTable(list(ep.table.rows[:9]) + [replace(r, model=0) for r in ep.table.rows[9:]]))
    w.step(torch.zeros((16, 8, 2), device="cuda"))
    torch.cuda.synchronize()
    st, tid, cnt, row = _snap(w)
    _, pres, s, _ = R.sample(ep.log, ep.t0, ep.row_track, row, cnt, 100, 0)
    assert np.array_equal(st["x"][pres], s["x"][pres])
    w.close()
