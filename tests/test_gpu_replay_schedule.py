"""K7 with slot schedules (t2d_set_log_schedule) on the device: replayed state, type ids and ``replay_track`` bit-exact against
tests/schedule_oracle.py through ticks and masked resets onto shuffled rows, equivalence of a one-entry schedule with the
row_track binding, teacher-forced mixed ticks against the float64 tick oracle, CUDA-graph / host-path / unbinding
equivalences, the env over scheduled episodes, and the C-level rejections of malformed schedules."""

import numpy as np
import pytest

from oracle import replay as R
from oracle import scenario as O
from tests import schedule_oracle as S
from tests.util import assert_state_close

pytestmark = pytest.mark.gpu

KEYS = ("x", "y", "heading", "speed", "vx", "vy")


def _walk_episodes(n, m, seed, table=None, size=200.0, duration_ms=20000, n_tracks=3000, max_frames=60, horizon_ms=4000):
    """Scheduled rows over the random-walk recording of ``synthetic.replay_episodes`` (wandering headings, a quarter of the
    tracks starting off the 40 ms grid, 1..max_frames frames): short tracks, so slots switch often."""
    from tactics2d_b200 import synthetic
    from tactics2d_b200.dataset_parser import build_replay_episodes

    src = synthetic.replay_episodes(2, m, n_tracks, seed=seed, table=table, size=size, duration_ms=duration_ms,
                                    max_frames=max_frames).log
    rng = np.random.default_rng(seed)
    first = src.first_ms.astype(np.int64)
    ok = np.nonzero((first % 40 == 0) & (src.n_frames >= 8) & (first >= 0) & (first < duration_ms - horizon_ms))[0]
    ego = rng.choice(ok, n)
    t0 = first[ego] + 40 * rng.integers(0, 4, n)
    kw = {} if table is None else dict(type_table=table)
    return build_replay_episodes(src, m, t0.tolist(), src.ids[ego].tolist(), horizon_ms=horizon_ms, reuse_slots=True, **kw)


def _as_schedule(row_track):
    """A row_track binding as a schedule of at most one entry per slot."""
    flat = np.asarray(row_track).reshape(-1)
    off = np.concatenate([[0], np.cumsum(flat >= 0)]).astype(np.int32)
    return off, flat[flat >= 0].astype(np.int32)


def _world(ep, interval=100, binding=None, **kw):
    import torch
    from tactics2d_b200 import BatchedWorld

    P, M = ep.type_id.shape
    w = BatchedWorld(P, M, ep.table, interval=interval, **kw)
    w.set_log(ep.log, ep.t0, **(binding if binding is not None else ep.binding()))
    pool = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in ep.pool.items()}
    w.type_id.copy_(torch.from_numpy(ep.type_id).cuda())
    w.reset(torch.ones(P, dtype=torch.uint8, device="cuda"), pool)
    return w, pool


def _snap(w):
    st = w.state_numpy()
    trk = None if w.replay_track is None else w.replay_track.cpu().numpy()
    return st, w.type_id.cpu().numpy(), w.step_count.cpu().numpy(), w.log_row.cpu().numpy(), trk


def _check(ep, w, pre_state, pre_tid, pre_track, offset, what, mask=None):
    """The world's replayed slots and replay_track equal the schedule oracle applied to the pre-replay state, bit for bit."""
    st, tid, cnt, row, trk = _snap(w)
    step = cnt - offset
    ref, ref_tid = S.apply(pre_state, pre_tid, ep.log, ep.t0, *ep.schedule, row, step, w.interval, offset, mask)
    rep, _, _, _, ref_trk = S.sample(ep.log, ep.t0, *ep.schedule, row, step, w.interval, offset)
    sel = np.ones(len(cnt), bool) if mask is None else np.asarray(mask, bool)
    rep = rep & sel[:, None]
    assert np.array_equal(tid[rep], ref_tid[rep]), what
    assert np.array_equal(tid[~rep], np.asarray(pre_tid)[~rep]), what
    for k in KEYS:
        assert np.array_equal(st[k][rep].view(np.uint32), ref[k][rep].view(np.uint32)), (what, k)
    assert np.array_equal(trk[sel], ref_trk[sel]), what
    assert np.array_equal(trk[~sel], pre_track[~sel]), what
    return trk


@pytest.mark.parametrize("interval", [40, 100, 120])
def test_scheduled_state_bit_exact_through_ticks_and_shuffled_resets(cuda_device, interval):
    import torch
    from tactics2d_b200 import synthetic

    N, M = 512, 64
    ep = _walk_episodes(N, M, seed=interval)
    off = ep.schedule[0]
    assert (np.diff(off).max()) >= 4                                              # slots with several entries
    w, pool = _world(ep, interval)
    rng = np.random.default_rng(interval)
    trk = _check(ep, w, dict(ep.pool), ep.type_id, np.full((N, M), -1), 0, "initial reset")
    seen = np.where(trk >= 0, trk, -1)
    switches = 0
    for t in range(40):
        st, tid, _, _, trk0 = _snap(w)
        if t % 9 == 8:   # masked reset onto shuffled rows
            mask = rng.uniform(0, 1, N) < 0.4
            idx = rng.permutation(N).astype(np.int32)
            w.reset(torch.from_numpy(mask.astype(np.uint8)).cuda(), pool, torch.from_numpy(idx).cuda())
            torch.cuda.synchronize()
            assert np.array_equal(w.log_row.cpu().numpy()[mask], idx[mask])
            pre = {k: np.where(mask[:, None], ep.pool[k][idx], st[k]).astype(np.float32) for k in KEYS}
            trk = _check(ep, w, pre, tid, trk0, 0, f"reset {t}", mask)
            seen[mask] = trk[mask]
            continue
        w.step(torch.from_numpy(synthetic.random_actions(t, (N, M))).cuda())
        torch.cuda.synchronize()
        trk = _check(ep, w, st, tid, trk0, 1, f"tick {t}")
        switches += int(((trk >= 0) & (seen >= 0) & (trk != seen)).sum())   # a slot shows another track than before
        seen = np.where(trk >= 0, trk, seen)
    assert switches > 200, switches
    w.close()


def test_one_entry_schedule_equals_row_track(cuda_device):
    import torch
    from tactics2d_b200 import synthetic

    N, M = 256, 32
    ep = synthetic.replay_episodes(N, M, 2000, seed=21, size=60.0, duration_ms=15000, max_frames=80, horizon_ms=3000)
    a, pool = _world(ep, 100, dict(row_track=ep.row_track))
    b, _ = _world(ep, 100, dict(schedule=_as_schedule(ep.row_track)))
    assert a.replay_track is None and b.replay_track is not None
    rng = np.random.default_rng(2)
    n_fl = 0
    for t in range(24):
        if t % 7 == 6:
            mask = torch.from_numpy((rng.uniform(0, 1, N) < 0.5).astype(np.uint8)).cuda()
            idx = torch.from_numpy(rng.permutation(N).astype(np.int32)).cuda()
            a.reset(mask, pool, idx); b.reset(mask, pool, idx)
            continue
        act = torch.from_numpy(synthetic.random_actions(300 + t, (N, M))).cuda()
        ra, rb = a.step(act), b.step(act)
        torch.cuda.synchronize()
        for f in ("flags", "hit_index", "hit_segment", "status", "done"):
            assert torch.equal(getattr(ra, f), getattr(rb, f)), (t, f)
        n_fl += int((ra.flags != 0).sum())
        sa, sb = _snap(a), _snap(b)
        for k in KEYS:
            assert np.array_equal(sa[0][k].view(np.uint32), sb[0][k].view(np.uint32)), (t, k)
        assert np.array_equal(sa[1], sb[1]) and np.array_equal(sa[2], sb[2]) and np.array_equal(sa[3], sb[3])
        _, pres, _, _ = R.sample(ep.log, ep.t0, ep.row_track, sa[3], sa[2] - 1, 100, 1)
        assert np.array_equal(sb[4], np.where(pres, ep.row_track[sa[3]], -1))
    assert n_fl > 0
    a.close(); b.close()


def _events_by_tile(st, tid, table, tiles, tile_id):
    N, M = tid.shape
    fl = np.zeros((N, M), np.uint8); hi = np.full((N, M), -1, np.int16); hs = np.full((N, M), -1, np.int16)
    for k, t in enumerate(tiles):
        sel = tile_id == k
        if sel.any():
            f, i, s = O.events(st["x"][sel], st["y"][sel], st["heading"][sel], tid[sel], table, t["segments"], t["bounds"])
            fl[sel], hi[sel], hs[sel] = f, i, s
    return fl, hi, hs


def test_teacher_forced_ticks_mixed_schedules_and_kinematics(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.types import MODEL_KINEMATICS, TypeTable

    N, M = 256, 32
    ep = _walk_episodes(N, M, seed=11, table=TypeTable.from_templates("kinematics"), size=80.0, duration_ms=15000,
                        n_tracks=1500, max_frames=40, horizon_ms=2000)
    # every other NPC slot becomes a kinematic participant: its schedule is emptied
    off, trk = ep.schedule
    keep = np.ones(N * M, bool)
    keep[np.arange(N * M) % M % 2 == 1] = False
    keep[np.arange(N * M) % M == 0] = False
    lens = np.where(keep, np.diff(off), 0)
    trk = np.concatenate([trk[off[s]:off[s + 1]] for s in range(N * M) if keep[s]] + [np.zeros(0, np.int32)]).astype(np.int32)
    ep.schedule = (np.concatenate([[0], np.cumsum(lens)]).astype(np.int32), trk)
    free = ~keep.reshape(N, M)
    free[:, 0] = False
    rng = np.random.default_rng(3)
    ep.type_id = ep.type_id.copy()
    ep.type_id[free] = rng.integers(0, 9, free.sum())
    for k in KEYS:
        ep.pool[k][free] = rng.uniform(0, 80, free.sum()).astype(np.float32) if k in ("x", "y") else ep.pool[k][0, 0]
    tiles = [dict(segments=synthetic.grid_wall_segments(80.0, 40.0, 8.0), bounds=(-5.0, 85.0, -5.0, 85.0)),
             dict(segments=np.asarray([[0, 40, 80, 40]], np.float32), bounds=(-20.0, 100.0, -20.0, 100.0))]
    tile_id = (np.arange(N) % 2).astype(np.int64)
    w, _ = _world(ep, 100, max_step=8)
    w.set_map_table(tiles, tile_id)
    table = ep.table.as_oracle_table()
    model = np.asarray(table["model"])
    n_fl = n_sched = 0
    for t in range(10):
        st, tid, _, _, trk0 = _snap(w)
        act = synthetic.random_actions(50 + t, (N, M))
        r = w.step(torch.from_numpy(act).cuda())
        torch.cuda.synchronize()
        trk = _check(ep, w, st, tid, trk0, 1, f"tick {t}")
        got, gtid, gcnt, _, _ = _snap(w)
        ref = O.physics_tick(st, gtid, act, table, 100, 5)
        kin = (gtid != 255) & (model[np.where(gtid == 255, 0, gtid)] == MODEL_KINEMATICS)
        assert_state_close(got, ref, kin, what=f"tick {t}")
        fl, hi, hs = _events_by_tile(got, gtid, table, tiles, tile_id)
        assert np.array_equal(fl, r.flags.cpu().numpy()) and np.array_equal(hi, r.hit_index.cpu().numpy())
        assert np.array_equal(hs, r.hit_segment.cpu().numpy())
        stt, done = O.status(fl, gtid, gcnt, 8)
        assert np.array_equal(stt, r.status.cpu().numpy()) and np.array_equal(done, r.done.cpu().numpy())
        n_fl += int((fl[gtid != 255] != 0).sum())
        n_sched += int((trk >= 0).sum())
    assert n_fl > 0 and n_sched > 1000
    w.close()


def test_graph_host_paths_and_unbinding(cuda_device, monkeypatch):
    import torch
    from tactics2d_b200 import BatchedWorld, synthetic

    monkeypatch.setenv("T2D_HOST_CHUNKS", "4")   # step_host in four chunks of 128 scenarios
    N, M = 512, 32
    ep = _walk_episodes(N, M, seed=9, duration_ms=15000, n_tracks=2000, max_frames=40, horizon_ms=3000)
    ws = [_world(ep, 100)[0] for _ in range(4)]
    ego_eager, _ = _world(ep, 100)
    acts = [torch.from_numpy(synthetic.random_actions(200 + t, (N, M))).cuda() for t in range(8)]
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
    for a in acts:
        ws[0].step(a)
        static.copy_(a)
        g.replay()
        ws[2].step_host(a.cpu().numpy())
    for a in acts:
        full = torch.zeros_like(a)
        full[:, 0] = a[:, 0]
        ego_eager.step(full)
        ws[3].step_host_ego(a[:, 0].cpu().numpy())
    torch.cuda.synchronize()
    ref = _snap(ws[0])
    assert int(ref[2][0]) == 9
    for other in (ws[1], ws[2]):
        got = _snap(other)
        for k in KEYS:
            assert np.array_equal(got[0][k], ref[0][k]), k
        for i in (1, 2, 4):
            assert np.array_equal(got[i], ref[i])
    ge, gh = _snap(ego_eager), _snap(ws[3])
    for k in KEYS:
        assert np.array_equal(ge[0][k], gh[0][k]), k
    assert np.array_equal(ge[1], gh[1]) and np.array_equal(ge[4], gh[4])
    for snap in (ref, gh):   # every path replayed: the slots hold the log at the current step
        _, pres, smp, _, trk = S.sample(ep.log, ep.t0, *ep.schedule, snap[3], snap[2], 100, 0)
        assert pres.sum() > 1000 and np.array_equal(snap[4], trk)
        for k in KEYS:
            assert np.array_equal(snap[0][k][pres], smp[k][pres]), k
    # set_log(None): the world then ticks like one that never had a log
    plain = BatchedWorld(N, M, ep.table, interval=100)
    st, tid, cnt, _, _ = _snap(ws[0])
    plain.set_state(st["x"], st["y"], st["heading"], st["speed"], st["vx"], st["vy"], type_id=tid)
    plain.step_count.copy_(torch.from_numpy(cnt).cuda())
    ws[0].set_log(None)
    assert ws[0].log_row is None and ws[0].replay_track is None
    for a in acts[:3]:
        ra, rb = ws[0].step(a), plain.step(a)
        torch.cuda.synchronize()
        assert torch.equal(ra.flags, rb.flags) and torch.equal(ra.hit_index, rb.hit_index)
    a_, b_ = ws[0].state_numpy(), plain.state_numpy()
    for k in KEYS:
        assert np.array_equal(a_[k], b_[k]), k
    assert torch.equal(ws[0].type_id, plain.type_id)
    for x in ws + [ego_eager, plain]:
        x.close()


def test_env_over_scheduled_episodes_across_auto_resets(cuda_device):
    import torch
    from tactics2d_b200 import synthetic
    from tactics2d_b200.envs import BatchedTrafficEnv

    N, M = 128, 48
    ep = synthetic.highway_episodes(N, M, seed=4, duration_ms=60000, horizon_ms=20000, length_m=150.0, rate_per_s=4.0)
    assert (ep.dropped == 0).all()
    env = BatchedTrafficEnv(None, replay=ep, max_step=6)
    _, info = env.reset(seed=1, options={"shuffle": True})
    w = env.world
    assert "track" in info and info["track"] is w.replay_track
    rng = np.random.default_rng(0)
    resets = shown = 0
    for t in range(20):
        st, tid, cnt, row, _ = _snap(w)
        a = rng.uniform(-0.5, 0.5, (N, 2)).astype(np.float32)
        _, _, term, trunc, info = env.step(torch.from_numpy(a).cuda())
        torch.cuda.synchronize()
        done = (term | trunc).cpu().numpy()
        resets += int(done.sum())
        got, gtid, gcnt, grow, gtrk = _snap(w)
        assert np.array_equal(grow, row)                                          # an auto-reset restarts the same row
        assert (gcnt[done] == 0).all() and (gcnt[~done] == cnt[~done] + 1).all()
        assert np.array_equal(info["track"].cpu().numpy(), gtrk)
        rep, pres, s, rtid, rtrk = S.sample(ep.log, ep.t0, *ep.schedule, grow, gcnt, w.interval, 0)
        assert np.array_equal(gtrk, rtrk), t                                     # a finished scenario: its schedule at t0
        for k in KEYS:
            assert np.array_equal(got[k][pres], s[k][pres]), (t, k)
        assert np.array_equal(gtid[rep], rtid[rep])
        act = np.zeros((N, M, 2), np.float32)
        act[:, 0] = a
        ref = O.physics_tick(st, tid, act, ep.table.as_oracle_table(), 100, 5, steer_first=True)
        ego = np.zeros((N, M), bool)
        ego[~done, 0] = True
        assert_state_close(got, ref, ego, what=f"ego step {t}")
        shown += int((gtrk >= 0).sum())
    assert resets >= 2 * N and shown > 20 * N * 5
    # an env over one-track-per-slot episodes returns no "track"
    ep0 = synthetic.highway_episodes(8, 16, seed=4, duration_ms=60000, horizon_ms=20000, reuse_slots=False)
    env0 = BatchedTrafficEnv(None, replay=ep0, max_step=6)
    _, info0 = env0.reset()
    _, _, _, _, info1 = env0.step(torch.zeros((8, 2), device="cuda"))
    assert "track" not in info0 and "track" not in info1 and env0.world.replay_track is None
    env.close(); env0.close()


def test_set_log_schedule_rejects_malformed_schedules_without_a_launch(cuda_device):
    import ctypes as C
    import torch
    from dataclasses import replace
    from tactics2d_b200 import _lib

    N, M = 16, 8
    ep = _walk_episodes(N, M, seed=2, duration_ms=6000, n_tracks=300, max_frames=30, horizon_ms=2000)
    w, _ = _world(ep, 100)
    lib = _lib.load()
    off, trk = ep.schedule
    first, last = ep.log.first_ms.astype(np.int64), ep.log.last_ms
    n_ent = np.diff(off)
    # a slot with two entries or more, followed by a non-empty slot of the same row
    multi, other = next((s, s2) for s in range(N * M) if n_ent[s] >= 2
                        for s2 in range(s + 1, (s // M + 1) * M) if n_ent[s2] >= 1)
    e0 = int(off[multi])

    def rejected(o=off, t=trk, lg=ep.log, match=""):
        n0 = lib.t2d_launch_count()
        with pytest.raises(_lib.T2DError, match=match):
            w.set_log(lg, ep.t0, schedule=(o, t))
        assert lib.t2d_launch_count() == n0

    bad = off.copy(); bad[multi + 1] = bad[multi] - 1
    rejected(o=bad, match="monotone")
    bad = off.copy(); bad[0] = 1
    rejected(o=bad, match="from 0 to n_entries")
    bad = off.copy(); bad[-1] -= 1
    rejected(o=bad, match="from 0 to n_entries")
    for v in (-1, len(ep.log)):
        bad = trk.copy(); bad[e0] = v
        rejected(t=bad, match="outside")
    a, b = int(trk[e0]), int(trk[e0 + 1])
    bad = trk.copy(); bad[e0], bad[e0 + 1] = b, a                                # out of order
    rejected(t=bad, match="does not start after")
    # overlapping / touching: B moved to start on or before A's last stamp
    for shift in (0, -40):
        fm = ep.log.first_ms.copy(); fm[b] = last[a] + shift
        rejected(lg=replace(ep.log, first_ms=fm.astype(np.int32)), match="does not start after")
    bad = trk.copy()                                                              # the same track in two slots of a row
    bad[off[other]] = a
    rejected(t=bad, match="twice")
    fm = ep.log.first_ms.copy(); fm[int(trk[-1])] = np.iinfo(np.int32).max - 10   # the last stamp overflows int32 ms
    rejected(lg=replace(ep.log, first_ms=fm.astype(np.int32)), match="int32")
    with pytest.raises(ValueError, match="exactly one"):
        w.set_log(ep.log, ep.t0, row_track=np.full((N, M), -1), schedule=ep.schedule)
    # a row_track next to a schedule is refused at the C level
    lg = ep.log
    i32 = lambda x: np.ascontiguousarray(x, dtype=np.int32)
    keep = dict(first=i32(lg.first_ms), n_frames=i32(lg.n_frames), period=i32(lg.period_ms), type_row=lg.type_row,
                records=lg.records, t0=i32(ep.t0), row_track=np.full((N, M), -1, np.int32))
    so, st_ = i32(off), i32(trk)
    n0 = lib.t2d_launch_count()
    code = lib.t2d_set_log_schedule(w._ctx, C.byref(w._log_struct(keep, w.log_row, w.type_id)), C.c_void_p(so.ctypes.data),
                                    C.c_void_p(st_.ctypes.data), len(st_), C.c_void_p(w.replay_track.data_ptr()))
    assert code == -1 and b"row_track must be NULL" in lib.t2d_last_error() and lib.t2d_launch_count() == n0
    # the good schedule stays bound and replays bit-exact
    for t in range(3):
        st, tid, _, _, trk0 = _snap(w)
        w.step(torch.zeros((N, M, 2), device="cuda"))
        torch.cuda.synchronize()
        _check(ep, w, st, tid, trk0, 1, f"tick {t}")
    w.close()
