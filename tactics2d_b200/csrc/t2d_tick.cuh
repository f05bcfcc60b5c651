// t2d_tick.cuh - K1 t2d_step_kernel (the fused tick), its static phase and phase timeline, the SingleTrackDrift
// pre-pass t2d_drift_kernel, and K3 t2d_physics_kernel (a flat batch through one physics model).
//
// Work decomposition of K1: a scenario (M <= 128 participants) is owned by a group of G lanes of
// one warp, 4 consecutive participants per lane (one float4 per state array per lane: coalesced
// 128-bit loads, 4 independent Euler chains per thread for ILP).  G = pow2 >= ceil(M/4), so a
// warp holds 32/G scenarios and every exchange inside a scenario is warp-synchronous: poses go
// through a per-warp shared-memory tile + __syncwarp, reductions through shuffles.  CTAs are
// persistent (grid = SMs x resident CTAs) and stage the static map tile (segments + broadphase
// grid) into shared memory ONCE with a TMA bulk copy (cp.async.bulk + mbarrier) that overlaps
// the first tile's physics.
#pragma once

#include "t2d_world.cuh"

namespace t2d {

struct StepArgs {
  float *x, *y, *h, *v, *vx, *vy;
  const uint8_t* type_id;
  int32_t* step_count;
  const float* action;
  const float* ego_action;         // [N][2] action of participant 0 of every scenario (overrides its row of `action`), or nullptr
  uint8_t* flags;
  int16_t* hit_index;
  int16_t* hit_segment;
  uint8_t* scn_status;
  uint8_t* done;
  const unsigned char* map_blob;   // device: the tiles' blobs, one after the other; nullptr when no tile has segments
  const uint32_t* tile_off;        // [n_tiles] byte offset of every tile's blob (map table mode)
  const uint16_t* tile_id;         // [N] the tile of every scenario, or nullptr: every scenario uses tile 0
  MapHeader mh;                    // copy of the blob header (grid geometry, section offsets): constant bank
  const Params* table;             // device
  int map_bytes, map_in_smem;
  int n_types;
  int N, M, G;                     // G = lanes per scenario
  int g_shift, mp_shift, unused1, n_tiles, wpc, table_bytes;   // launch-shape constants (see the kernel prologue)
  int off_poseA, off_poseB, off_hit, off_queue, off_sorted, unused0, off_qcount, off_bar;   // shared-memory carve
  // (unused0, unused1: free slots that keep the parameter layout the drift pre-pass shares with K1)
  int n_steps;
  float dt, dt_rem;
  double dt_d, dt_rem_d, interval_d;   // the same steps in double (dynamics / point mass run in fp64)
  int max_step, cfg_flags;
  int do_physics, has_bounds, vec_ok, needs_vel_in;
  int prefetch;                    // L2 prefetch of tile inputs ahead of their loads (see the kernel prologue)
  float bxmin, bxmax, bymin, bymax;
  float rb_max;                    // largest bounding radius in the type table (broadphase threshold)
  GoalArgs goal;                   // the ego's; goal.target == nullptr: no goal
  float *wheel_f, *wheel_r;        // [N][M] wheel angular speeds of the SingleTrackDrift participants, or nullptr
  uint8_t* order;                  // [N][64] the world's x-order hint (FIXED instance only; see the sort)
  unsigned long long* order_fallbacks;   // the device's fallback counters (FIXED instance only)
};

// Every model except the fp32 kinematic fast path (one copy of the fp64 code per kernel).  SingleTrackDrift is NOT
// integrated here: its fp64 tyre model needs far more registers than K1's budget (inlined, or even called, from K1 it
// pushed the whole kernel into spilling and cost the other models 3 - 9 %), so t2d_drift_kernel advances those
// participants in a pre-pass and K1 only builds their pose.
__device__ __noinline__ void other_model_step(OneIO& io, const Params& p, int n_steps, double dt, double dt_rem, double interval) {
  if (p.model() == MODEL_DYNAMICS) {
    dynamics_step(io, p, n_steps, dt);
  } else if (p.model() == MODEL_POINTMASS_NEWTON) {
    pointmass_newton_step(io, p, interval);
  } else if (p.model() == MODEL_POINTMASS_EULER) {
    pointmass_euler_step(io, p, n_steps, dt, dt_rem);
  } else {
    sincos_fast(io.h, &io.sh, &io.ch);
  }
}

// Static broadphase, level 1: the clearance field.  One shared-memory load tells whether the pose's
// bounding circle can reach any segment at all (most participants are nowhere near a wall).
// The test is split in two so that the global byte load can be issued early and consumed late:
// near_fetch returns the quantised clearance under the participant (0 = treat as near: outside the grid but within
// reach of it; 255 = far), near_decide compares it with the bounding radius.
__device__ __forceinline__ unsigned near_fetch(const float ax, const float ay, const float rbound, const MapHeader& mh, const uint8_t* fine,
                                               unsigned& alt) {
  // branch-free (four of these run side by side per lane): the byte under the participant is fetched from a clamped,
  // always valid address and replaced afterwards when the position lies outside the grid.  The cell indices come
  // from the round-to-nearest magic number (rint(f - 1/2) = floor(f) up to a cell boundary, where either neighbour's
  // clearance is a valid lower bound) instead of float -> int conversions on the XU pipe.
  const float r = rbound * 1.0001f + 1e-3f;
  const float fx = (ax - mh.x0) * mh.inv_cell, fy = (ay - mh.y0) * mh.inv_cell;
  const float gxf = (float)mh.gx, gyf = (float)mh.gy;
  const bool inside = fx >= 0.0f && fy >= 0.0f && fx < gxf && fy < gyf;
  const float kf = (float)mh.fine;
  const int nx = mh.gx * mh.fine, ny = mh.gy * mh.fine;
  const float ux = fmaf(inside ? fx : 0.0f, kf, -0.5f), uy = fmaf(inside ? fy : 0.0f, kf, -0.5f);
  int ix = __float_as_int(ux + RINT_MAGIC) - 0x4B400000, iy = __float_as_int(uy + RINT_MAGIC) - 0x4B400000;
  ix = min(max(ix, 0), nx - 1); iy = min(max(iy, 0), ny - 1);
  const unsigned q = (unsigned)__ldg(fine + (size_t)iy * nx + ix);
  // outside the grid: reachable only within r of its box (NaN position: 255, never near)
  const float ox = fmaxf(fmaxf(-fx, fx - gxf), 0.0f), oy = fmaxf(fmaxf(-fy, fy - gyf), 0.0f);
  const unsigned q_out = fmaxf(ox, oy) * mh.cell <= r ? 0u : 255u;
  // The loaded byte is NOT touched here (its first use would stall the lane on the L2 round trip): it is returned as
  // loaded; `alt` says what to take instead - 0xffffffff: nothing (inside the grid), else the value for outside.
  alt = inside ? 0xffffffffu : q_out;
  return q;
}
__device__ __forceinline__ bool near_decide(unsigned q, unsigned alt, const float rbound) {
  const unsigned v = alt == 0xffffffffu ? q : alt;
  return (float)v * CLEAR_QUANT <= rbound * 1.0001f + 1e-3f;
}

// Own pose of participant `idx` back from the warp's shared-memory tile (the hot loops keep only x, y
// and the bounding radius in registers; the rare exact paths re-read the rest).
// The warp's pose tile is addressed by participant slot (scenario slot x padded participants + participant), but laid
// out lane-minor: slot = lane * PPL + i lives at word i * 32 + lane, so that the lanes' stores of their own PPL
// participants are conflict-free (consecutive lanes, consecutive 16-byte words).
static_assert(PPL == 4, "pslot's masks and shifts are those of 4 participants per lane");
__device__ __forceinline__ int pslot(int slot) { return ((slot & 3) << 5) | (slot >> 2); }

__device__ __forceinline__ Pose load_pose(const float4* poseA, const float4* poseB, int slot) {
  const int idx = pslot(slot);
  const float4 a = poseA[idx], b = poseB[idx];
  Pose p;
  p.x = a.x; p.y = a.y; p.h = a.w; p.c = b.x; p.s = b.y; p.l = b.z; p.w = b.w;
  return p;
}

constexpr int QCAP = 192;   // per-warp queue: candidate pairs, then static participants (0..127) + undecided segments (128..191)

// Exact test of one candidate pair (tile indices ti, tj of the same scenario); a hit is recorded for both
// ends as the minimum partner index (scenario-local), which is what "first hit in list order" means.  Inlined into the
// drain: an out-of-line call taking the poses by value made every draining lane spill around an ABI call; only the rare
// fp64 fallback (pair_exact) stays out of line, keeping its register footprint out of the kernel.
__device__ __forceinline__ void pair_resolve(int ti, int tj, int mp_shift, const float4* poseA, const float4* poseB, int* hitmin) {
  const Pose a = load_pose(poseA, poseB, ti), b = load_pose(poseA, poseB, tj);
  if (pair_hit(a, b)) {
    const int mask = (1 << mp_shift) - 1;
    atomicMin(&hitmin[pslot(ti)], tj & mask);
    atomicMin(&hitmin[pslot(tj)], ti & mask);
  }
}

// Minus the squared broadphase reach of an owner of bounding radius rb: conservative, since any partner's bounding
// radius is <= rb_max.
__device__ __forceinline__ float neg_reach2(float rb, float rb_max) {
  const float rr = rb + rb_max;
  return -fmaf(rr * rr, 1.00001f, 1e-12f);
}

// Order-preserving map of a float (not NaN) to uint32 and back: a < b  <=>  f2ord(a) < f2ord(b) (-0 sorts before +0).
__device__ __forceinline__ unsigned f2ord(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }

// One entry of a scenario's x-sorted list (the tick's broadphase): position, minus the squared reach (neg_reach2) and
// the sort key as bits; the key's low 7 bits are the participant's slot in its scenario.
// The exact broadphase test of one pair {a, b} of a scenario: the circular enumeration's owner is the end from which the
// other lies at circular offset 1 .. Mh (Mh = M / 2; at even M the pair at offset M / 2 is owned by BOTH ends, each
// testing it with its own reach).  The margin d^2 - thr of owner o against partner r is fma(dx, dx, fma(dy, dy, -thr_o))
// with dx = fl(x_r - x_o), dy = fl(y_r - y_o): for the other orientation fl(x_o - x_r) = -dx exactly, so both squares are
// shared.  A pair whose owner's margin is <= 0 goes on the warp's queue as (owner, partner) tile indices; when the queue
// is full the count keeps growing, and the caller then falls back to the exhaustive pass.  No function call may appear in
// here: it is inlined into the scan loop, and a CALL makes the compiler keep only callee-saved registers live across it.
__device__ __forceinline__ void sweep_pair(const float4& a, const float4& b, int tb, int M, int Mh, unsigned* queue, int* qcount) {
  const int sa = (int)(__float_as_uint(a.w) & 127u), sb = (int)(__float_as_uint(b.w) & 127u);
  int d = sb - sa;   // circular offset of b from a (the slots differ: 1 .. M - 1)
  if (d < 0) d += M;
  const float dx = b.x - a.x, dy = b.y - a.y;
  if (d <= Mh && fmaf(dx, dx, fmaf(dy, dy, a.z)) <= 0.0f) {
    const int slot = atomicAdd(qcount, 1);
    if (slot < QCAP) queue[slot] = ((unsigned)(tb + sa) << 16) | (unsigned)(tb + sb);
  }
  if (d >= M - Mh && fmaf(dx, dx, fmaf(dy, dy, b.z)) <= 0.0f) {
    const int slot = atomicAdd(qcount, 1);
    if (slot < QCAP) queue[slot] = ((unsigned)(tb + sb) << 16) | (unsigned)(tb + sa);
  }
}

// The smallest margin a pair can have under any owner's reach (nglob = neg_reach2(rb_max, rb_max) <= every -thr, and the
// margin is monotone in -thr): > 0 rules out a candidate in both orientations.  NaN positions give NaN, which fminf drops.
__device__ __forceinline__ float pair_min_margin(const float4& a, const float4& b, float nglob) {
  const float dx = b.x - a.x, dy = b.y - a.y;
  return fmaf(dx, dx, fmaf(dy, dy, nglob));
}

// Dense-scene fallback (the candidate queue overflowed): every lane resolves all pairs of its own participants
// against all partners of the scenario directly.  Correct for any density, slow, and never on the hot path.
__device__ __noinline__ void pair_exhaustive(int t0, int tb, int m0, int M, int mp_shift, float rb_max, const float4* poseA,
                                             const float4* poseB, int* hitmin) {
  for (int i = 0; i < PPL; ++i) {
    if (m0 + i >= M) break;
    const float4 a = poseA[pslot(t0 + i)];
    if (!(a.x == a.x)) continue;
    const float rr = a.z + rb_max;
    for (int j = m0 + i + 1; j < M; ++j) {
      const float4 b = poseA[pslot(tb + j)];
      const float dx = b.x - a.x, dy = b.y - a.y;
      if (fmaf(dx, dx, dy * dy) <= fmaf(rr * rr, 1.00001f, 1e-12f)) pair_resolve(t0 + i, tb + j, mp_shift, poseA, poseB, hitmin);
    }
  }
}

// Static level 2 for ONE participant (tile index ti), run by one lane: walk the grid cells under the bounding
// circle, fp32-filtered segment test per listed segment, keep the lowest hit.  No function call in here (see
// sweep_pair): a segment the filter cannot decide is pushed on the exact queue (entries QX0 .. QCAP-1
// of the warp's queue, counter qcount) and decided after the loop; if that queue is full the participant is
// marked (returns -2) for the out-of-line exact walk.
constexpr int QX0 = 128;   // first exact-queue entry (entries below hold the compacted participant list)

// Static level 2 for ONE participant whose reach is <= the map's dilation: ONE cell look-up (the cell under the centre)
// and one loop over its dilated list.  Returns the lowest hit, 0x7fffffff for none, -2 when the participant needs the
// out-of-line walk (reach beyond the dilation, or the exact queue is full).
__device__ __forceinline__ int static_walk(int ti, const Pose& a, float rbound, const MapHeader& mh, const MapView& mv, unsigned* queue,
                                           int* qcount) {
  const float r = rbound * 1.0001f + 1e-3f;
  if (!(r <= mh.dil)) return -2;
  const float fx = (a.x - mh.x0) * mh.inv_cell, fy = (a.y - mh.y0) * mh.inv_cell;
  if (!(fx >= 0.0f && fy >= 0.0f && fx < (float)mh.gx && fy < (float)mh.gy)) return 0x7fffffff;   // beyond the grown box: out of reach
  const int cx = min((int)fx, mh.gx - 1), cy = min((int)fy, mh.gy - 1);
  const int cidx = cy * mh.gx + cx;
  const uint32_t b = mv.dcell_start[cidx], e = mv.dcell_start[cidx + 1];
  int best = 0x7fffffff;
  bool overflow = false;
  // the pose's bounding circle as a box: a listed segment whose own box misses it (most of a dilated list in a dense map)
  // is skipped for 8 instructions instead of running the 35-instruction filtered test to the same "disjoint" verdict
  const float bx0 = a.x - r, bx1 = a.x + r, by0 = a.y - r, by1 = a.y + r;
  for (uint32_t k = b; k < e; ++k) {
    const int sidx = mv.ditems[k];
    const float4 sg = mv.seg[sidx];
    if (fmaxf(sg.x, sg.z) < bx0 || fminf(sg.x, sg.z) > bx1 || fmaxf(sg.y, sg.w) < by0 || fminf(sg.y, sg.w) > by1) continue;
    const int rr = a.w < 0.0f ? circle_segment_f32(a.x, a.y, a.l, sg.x, sg.y, sg.z, sg.w)
                              : obb_segment_f32(a.x, a.y, a.c, a.s, a.l, a.w, sg.x, sg.y, sg.z, sg.w);
    if (rr > 0) {
      best = sidx;   // the list is ascending: the first hit is the lowest
      break;
    } else if (rr < 0) {
      const int slot = atomicAdd(qcount, 1);
      if (slot < QCAP - QX0) queue[QX0 + slot] = ((unsigned)ti << 16) | (unsigned)sidx;
      else overflow = true;
    }
  }
  return overflow ? -2 : best;
}

// The static phase of one warp tile.  (1) every lane decides with the clearance field which of its participants
// can reach a wall at all; (2) those participants are compacted into a list with warp ballots; (3) the list is
// processed one participant per lane (static_walk), so the divergent cell walks of ~15 % of the participants run
// side by side instead of one after the other; (4) the few filter-undecided segments are settled in fp64.
// Where a participant's tile lives: one tile for everybody (header in the kernel's constant bank, sections in shared or
// global memory), or a table of tiles indexed by the participant's scenario (headers and sections in global memory).
struct TileRef {
  const MapHeader* mh;         // header (constant bank, or global)
  const unsigned char* sec;    // where the sections up to the fine field are read from (shared or global)
  const unsigned char* blob;   // the blob in global memory (fine field, polygon data)
};

template <bool MAP_TABLE>
__device__ __forceinline__ void static_phase(unsigned near_bits, int t0, int lane, int tile_first_scn, int mp_shift, const StepArgs& A,
                                             const unsigned char* s_map, const float4* poseA, const float4* poseB, int* segmin,
                                             unsigned* queue, int* qcount) {
  int base = 0;
#pragma unroll
  for (int i = 0; i < PPL; ++i) {
    const bool near = (near_bits >> i) & 1u;
    const unsigned m = __ballot_sync(0xffffffffu, near);
    if (near) queue[base + __popc(m & ((1u << lane) - 1u))] = (unsigned)(t0 + i);
    base += __popc(m);
  }
  // the tile of participant slot ti (its scenario = the warp tile's first scenario + ti / padded participants)
  auto tile_of = [&](int ti) {
    TileRef t;
    if constexpr (MAP_TABLE) {
      const long long n = (long long)tile_first_scn + (ti >> mp_shift);
      const unsigned char* blob = A.map_blob + A.tile_off[n < A.N ? A.tile_id[n] : 0];
      t.mh = reinterpret_cast<const MapHeader*>(blob); t.sec = blob; t.blob = blob;
    } else {
      t.mh = &A.mh; t.sec = A.map_in_smem ? s_map : A.map_blob; t.blob = A.map_blob;
    }
    return t;
  };
  __syncwarp();
  for (int k = lane; k < base; k += 32) {
    const int ti = (int)queue[k];
    const TileRef t = tile_of(ti);
    const Pose a = load_pose(poseA, poseB, ti);
    const int best = t.mh->n_seg > 0 ? static_walk(ti, a, poseA[pslot(ti)].z, *t.mh, map_view(t.sec, *t.mh), queue, qcount) : 0x7fffffff;
    segmin[pslot(ti)] = best;   // one lane per participant: plain store (-2 = needs the exact walk)
  }
  __syncwarp();
  const int n_x = min(*qcount, QCAP - QX0);
  for (int k = lane; k < n_x; k += 32) {   // undecided (participant, segment) pairs: exact test
    const unsigned e = queue[QX0 + k];
    const int ti = (int)(e >> 16), sidx = (int)(e & 0xffffu);
    int* sm = &segmin[pslot(ti)];
    if (*sm != -2 && sidx < *sm) {
      const TileRef t = tile_of(ti);
      if (seg_exact(load_pose(poseA, poseB, ti), reinterpret_cast<const float4*>(t.sec + t.mh->off_seg)[sidx])) atomicMin(sm, sidx);
    }
  }
  __syncwarp();
  for (int k = lane; k < base; k += 32) {   // the out-of-line walk where needed; then edges -> objects, polygon containment
    const int ti = (int)queue[k];
    int* sm = &segmin[pslot(ti)];
    const TileRef t = tile_of(ti);
    if (*sm == -2) {
      const MapView mv = map_view(t.sec, *t.mh);
      *sm = static_walk_exact(load_pose(poseA, poseB, ti), poseA[pslot(ti)].z, *t.mh, mv.seg, mv.cell_start, mv.items);
    }
    if (t.mh->n_poly > 0) {
      const float4 pa = poseA[pslot(ti)];
      *sm = static_objects(*sm, pa.x, pa.y, *t.mh, t.blob);
    }
  }
  __syncwarp();
}

__device__ __noinline__ bool oob_slow(const float4* poseA, const float4* poseB, int idx, float xmin, float xmax, float ymin, float ymax) {
  const Pose a = load_pose(poseA, poseB, idx);
  int r = out_of_bound_f32(a.x, a.y, a.c, a.s, a.l, a.w, a.w < 0.0f, xmin, xmax, ymin, ymax);
  if (r < 0) r = out_of_bound_f64(a.x, a.y, a.h, a.l, a.w, a.w < 0.0f, xmin, xmax, ymin, ymax) ? 1 : 0;
  return r != 0;
}

// The launch shape K1's FIXED instance is compiled for (C2: M = 64 participants, so G = 16 lanes and MP = 64 padded
// slots per scenario; kinematic physics on, vector access, no velocity inputs, no ego action, no goal).  The host
// launches it exactly when a tick has this shape and the generic instance otherwise.
constexpr int FIX_M = 64, FIX_G = 16, FIX_G_SHIFT = 4, FIX_MP_SHIFT = 6;

// Load cohorts of the FIXED instance.  Its tick is one wave, so every warp issues its loads within a fraction of a
// microsecond of the others and then waits for the whole transfer, and the SMs have nothing to issue meanwhile.  The
// first half of every CTA's warps (cohort A) issue their first tile's loads and then arrive on this named barrier; the
// second half (cohort B) wait on it before issuing theirs, so their requests queue behind A's and A runs its physics
// while B's bytes stream in.  Only A prefetches into L2 before griddepcontrol.wait, for the same reason.  The barrier
// counts every thread of the CTA, so each thread must reach it exactly once (see the tile loop).
constexpr int COHORT_BAR = 1;   // (0 is __syncthreads')
__device__ __forceinline__ void cohort_arrive(int threads) {
  asm volatile("barrier.arrive %0, %1;" ::"n"(COHORT_BAR), "r"(threads) : "memory");
}
__device__ __forceinline__ void cohort_wait(int threads) {
  asm volatile("barrier.sync %0, %1;" ::"n"(COHORT_BAR), "r"(threads) : "memory");
}

// The FIXED instance's x sort starts from the order the scenario's slots had after the previous tick (the world's
// [N][64] order hint) and repairs it with T2D_ORDER_PASSES odd-even transposition passes; a warp whose order is still not
// strictly ascending falls back to the sort network (see the sort).  At C2 a participant moves at most about 1.5 m per
// tick, and two passes sort nearly every warp from the previous tick's order.  A warp that falls back counts itself in
// StepArgs::order_fallbacks, spread over ORDER_COUNTERS 128-byte lines (by CTA) so that a tick where every warp falls
// back does not queue its atomics on one address; t2d_tick_order_fallback_count sums them.
#ifndef T2D_ORDER_PASSES
#define T2D_ORDER_PASSES 2
#endif
constexpr int ORDER_COUNTERS = 64, ORDER_COUNTER_STRIDE = 16;   // (16 counters of 8 bytes: one per 128-byte line)

// L2 prefetch of the lines a lane's PPL participants will load (state, action, type ids; order hint in FIXED).
template <bool FIXED>
__device__ __forceinline__ void prefetch_tile_l2(const StepArgs& A, long long i) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(A.x + i));
  asm volatile("prefetch.global.L2 [%0];" ::"l"(A.y + i));
  asm volatile("prefetch.global.L2 [%0];" ::"l"(A.h + i));
  asm volatile("prefetch.global.L2 [%0];" ::"l"(A.v + i));
  if (FIXED || A.action) asm volatile("prefetch.global.L2 [%0];" ::"l"(A.action + 2 * i));
  asm volatile("prefetch.global.L2 [%0];" ::"l"(A.type_id + i));
  if (FIXED) asm volatile("prefetch.global.L2 [%0];" ::"l"(A.order + i));   // (M = 64: the hint's index is the state's)
  if (!FIXED && A.needs_vel_in) {
    asm volatile("prefetch.global.L2 [%0];" ::"l"(A.vx + i));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(A.vy + i));
  }
}

// ---------------------------------------------------------------------------- K1 phase timeline (measurement build)
// Built with -DT2D_TICK_TIMELINE (bench_tick_phases.py compiles such a library on the side), lane 0 of every warp
// records %globaltimer and %clock64 at TL_POINTS points of its first tile: entry, after griddepcontrol.wait, loads
// consumed, physics done, sort done, sweep done, drain done, static done, exit.  A point waits for the value `dep` it is
// given, so that it marks when that value was available rather than when its instruction was issued.  In the shipped
// build T2D_TL expands to nothing and the kernel is unchanged.
#ifdef T2D_TICK_TIMELINE
constexpr int TL_POINTS = 9, TL_MAX_WARPS = 4096;
__device__ unsigned long long t2d_timeline[TL_MAX_WARPS][TL_POINTS][2];
#define T2D_TL(k, on, slot, dep)                                                                                    \
  do {                                                                                                              \
    if ((on) && (slot) < TL_MAX_WARPS) {                                                                            \
      unsigned long long g_, c_;                                                                                    \
      asm volatile("mov.u64 %0, %%globaltimer;\n\tmov.u64 %1, %%clock64;" : "=l"(g_), "=l"(c_) : "f"(dep) : "memory"); \
      t2d_timeline[slot][k][0] = g_;                                                                                \
      t2d_timeline[slot][k][1] = c_;                                                                                \
    }                                                                                                               \
  } while (0)
#else
#define T2D_TL(k, on, slot, dep)
#endif

// ---------------------------------------------------------------------------- K1
// KIN_ONLY: every type in the table is SingleTrackKinematics or static - the fp64 models are compiled out
// (their register footprint would otherwise bound the occupancy of the whole kernel).
// MAP_TABLE: every scenario names its own static-geometry tile (t2d_set_map_table); the tiles are then read from global
// memory, header included.  Otherwise one tile serves all scenarios: header in the constant bank, sections staged into
// shared memory once per CTA.
// FIXED: the tick has the C2 launch shape (FIX_M ...): every shape value is a compile-time constant, so the sort network
// and the status reduction unroll, addresses fold, and the tests for features that shape excludes go away.  The
// physics and every other operation on the data are the generic instance's: only control flow and addresses differ.
// (The sub-step loop keeps its runtime trip count: unrolled, the compiler fuses multiplies and adds that the loop keeps
// in separate blocks into FMAs, which changes result bits.)
template <bool KIN_ONLY, bool MAP_TABLE, bool FIXED>
__global__ void __launch_bounds__(CTA_THREADS, 2) t2d_step_kernel(const __grid_constant__ StepArgs A) {
  extern __shared__ __align__(128) unsigned char smem[];
  T2D_TL(0, (threadIdx.x & 31) == 0, (int)(blockIdx.x * A.wpc + (threadIdx.x >> 5)), 0.0f);
  // carve: [map blob | 16B aligned] [type table] [pose tiles, hit mins, queues, positions] [mbarrier]; every
  // offset, shift and count that depends only on the launch shape comes precomputed from the host
  // (kernel-parameter constant bank) instead of integer divisions / loops per thread
  const int map_smem_bytes = (!MAP_TABLE && A.map_in_smem) ? A.map_bytes : 0;
  const int table_bytes = A.table_bytes;
  const int wpc = A.wpc;
  unsigned char* s_map = smem;
  Params* s_table = reinterpret_cast<Params*>(smem + map_smem_bytes);
  float4* s_poseA = reinterpret_cast<float4*>(smem + A.off_poseA);
  float4* s_poseB = reinterpret_cast<float4*>(smem + A.off_poseB);
  int* s_hit = reinterpret_cast<int*>(smem + A.off_hit);
  unsigned* s_queue = reinterpret_cast<unsigned*>(smem + A.off_queue);
  float4* s_sorted = reinterpret_cast<float4*>(smem + A.off_sorted);
  int* s_qcount = reinterpret_cast<int*>(smem + A.off_qcount);
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(smem + A.off_bar);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // Programmatic dependent launch: let the next tick's grid start launching now (its prologue - shared-memory
  // carve, mbarrier, TMA staging of the static table / map - overlaps this grid's tail) ...
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  // Stage the type table and the map tile with TMA bulk copies (UBLKCP) on one mbarrier; the wait sits after
  // the first tile's global loads have been issued, so the staging overlaps the cold HBM reads.
  if (tid == 0) {
    mbar_init(s_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(s_bar, (uint32_t)(table_bytes + map_smem_bytes));
    bulk_g2s(s_table, A.table, (uint32_t)table_bytes, s_bar);
    if (map_smem_bytes > 0) bulk_g2s(s_map, A.map_blob, (uint32_t)map_smem_bytes, s_bar);
  }
  bool staged = false;
  // L2 prefetch of the first tile's state / action lines while the previous grid drains (its CTAs retire over a
  // microsecond or two; ours take their places one by one and would otherwise just sit in griddepcontrol.wait): L2 is the
  // coherence point of the GPU, so a line fetched early can never be stale when it is loaded after the wait.  With a
  // peer-memory done exchange running under the tick the burst of prefetches competes with the exchange kernel's peer
  // stores and system-scope fence, and the exchange chain then sets the pace, so the host leaves it off while an
  // exchange object is alive in the process (T2D_PREFETCH=0 / 1 overrides).
  // a launch-shape parameter, or the constant it is in the FIXED instance (read where it is used, as before)
#define K1_SHAPE(field, fixed_value) (FIXED ? (fixed_value) : A.field)
  const bool cohorts = FIXED && wpc > 1;                 // warps [0, wpc / 2) are cohort A, the rest cohort B
  const bool cohort_b = cohorts && warp >= (wpc >> 1);
  {
    const long long n_ = ((long long)blockIdx.x * wpc + warp) * (32 >> K1_SHAPE(g_shift, FIX_G_SHIFT)) + (lane >> K1_SHAPE(g_shift, FIX_G_SHIFT));
    const int m_ = (lane & (K1_SHAPE(G, FIX_G) - 1)) * PPL;
    if (!cohort_b && A.prefetch && n_ < A.N && m_ < K1_SHAPE(M, FIX_M)) prefetch_tile_l2<FIXED>(A, n_ * K1_SHAPE(M, FIX_M) + m_);   // (inside the arrays: a hint, but no stray addresses)
  }
  // ... and wait here, before the first access to the state the previous tick wrote, until that grid has
  // completed and flushed (no-op when the kernel was not launched as a programmatic dependent).
  asm volatile("griddepcontrol.wait;" ::: "memory");
  T2D_TL(1, lane == 0, (int)blockIdx.x * wpc + warp, 0.0f);
  const int G = K1_SHAPE(G, FIX_G), M = K1_SHAPE(M, FIX_M);
  const int spw = 32 >> K1_SHAPE(g_shift, FIX_G_SHIFT);   // scenarios per warp
  const int sub = lane >> K1_SHAPE(g_shift, FIX_G_SHIFT);   // scenario slot inside the warp
  const int gl = lane & (G - 1);        // lane inside the group
  const int m0 = gl * PPL;              // first participant of this lane
  const int MP = G * PPL;               // padded participants per scenario
  // warp-level views of the pose tile; t0 = this lane's first slot in it, tb = its scenario's first slot
  float4* poseA = s_poseA + warp * POSE_PER_WARP;
  float4* poseB = s_poseB + warp * POSE_PER_WARP;
  int* hitmin = s_hit + warp * POSE_PER_WARP;
  unsigned* queue = s_queue + warp * QCAP;
  int* qcount = s_qcount + warp;
  const int tb = sub * MP, t0 = tb + m0;
  const int mp_shift = K1_SHAPE(mp_shift, FIX_MP_SHIFT);   // MP = 1 << mp_shift
  float4* sorted = s_sorted + warp * POSE_PER_WARP + tb;   // this scenario's x-sorted list (sweep_pair)
  const int Mh = M >> 1;                // partner offsets 1..Mh cover every unordered pair

  const int n_tiles = A.n_tiles;
  const int tile0 = (int)blockIdx.x * wpc + warp;
  // The cohort barrier, once per thread: B waits here, before its first tile; A arrives right after issuing its first
  // tile's loads, or here when it has no tile (a partial last CTA, where B has none either).  Later tiles of a
  // persistent launch do not touch it.
  if (cohort_b) cohort_wait(wpc * 32);
  else if (cohorts && tile0 >= n_tiles) cohort_arrive(wpc * 32);
  for (int tile = tile0; tile < n_tiles; tile += (int)gridDim.x * wpc) {
    const long long n = (long long)tile * spw + sub;
    const bool scn_ok = n < A.N;
    int nvalid = scn_ok ? (FIXED ? PPL : min(PPL, M - m0)) : 0;
    if (nvalid < 0) nvalid = 0;
    const long long idx0 = n * M + m0;
#ifdef T2D_TICK_TIMELINE
    const bool tl_on = lane == 0 && tile == (int)blockIdx.x * wpc + warp;
    const int tl_slot = tile;
#endif

    // ------------------------------------------------------------------ load
    float sx[PPL], sy[PPL], shd[PPL], sv[PPL], svx[PPL], svy[PPL], a0[PPL], a1[PPL];
    int tidv[PPL];
#pragma unroll
    for (int i = 0; i < PPL; ++i) {
      sx[i] = sy[i] = shd[i] = sv[i] = svx[i] = svy[i] = a0[i] = a1[i] = 0.0f;
      tidv[i] = T2D_TYPE_INACTIVE;
    }
    // FIXED: the order hint of entries 4 gl .. 4 gl + 3, one byte each (the identity outside the batch)
    uint32_t hint = 0x03020100u + 0x04040404u * (uint32_t)gl;
    if (nvalid == PPL && K1_SHAPE(vec_ok, 1)) {
      ld_vec<float, PPL>(A.x + idx0, sx);
      ld_vec<float, PPL>(A.y + idx0, sy);
      ld_vec<float, PPL>(A.h + idx0, shd);
      ld_vec<float, PPL>(A.v + idx0, sv);
      uint8_t tb8[PPL];
      ld_vec<uint8_t, PPL>(A.type_id + idx0, tb8);
      if constexpr (FIXED) hint = *reinterpret_cast<const uint32_t*>(A.order + idx0);   // (M = 64: the state's index)
#pragma unroll
      for (int i = 0; i < PPL; ++i) tidv[i] = tb8[i];
      if (K1_SHAPE(do_physics, 1)) {
        float2 act[PPL];
        float lo[4], hi[4];
        ld_vec<float, 4>(A.action + 2 * idx0, lo);
        ld_vec<float, 4>(A.action + 2 * idx0 + 4, hi);
        act[0] = make_float2(lo[0], lo[1]); act[1] = make_float2(lo[2], lo[3]);
        act[2] = make_float2(hi[0], hi[1]); act[3] = make_float2(hi[2], hi[3]);
#pragma unroll
        for (int i = 0; i < PPL; ++i) { a0[i] = act[i].x; a1[i] = act[i].y; }
        if (K1_SHAPE(needs_vel_in, 0)) {
          ld_vec<float, PPL>(A.vx + idx0, svx);
          ld_vec<float, PPL>(A.vy + idx0, svy);
        }
      }
    } else {
      // ragged / unaligned rows: predicated scalar loads, fully unrolled (a runtime-indexed loop would demote every
      // per-participant array of this kernel to local memory)
#pragma unroll
      for (int i = 0; i < PPL; ++i) {
        if (i < nvalid) {
          sx[i] = A.x[idx0 + i]; sy[i] = A.y[idx0 + i]; shd[i] = A.h[idx0 + i]; sv[i] = A.v[idx0 + i];
          tidv[i] = A.type_id[idx0 + i];
          if (K1_SHAPE(do_physics, 1)) {
            a0[i] = A.action[2 * (idx0 + i)]; a1[i] = A.action[2 * (idx0 + i) + 1];
            if (K1_SHAPE(needs_vel_in, 0)) { svx[i] = A.vx[idx0 + i]; svy[i] = A.vy[idx0 + i]; }
          }
        }
      }
    }
    if (cohorts && !cohort_b && tile == tile0) cohort_arrive(wpc * 32);   // issued, not landed: B's requests queue behind
    {   // several tiles per warp (persistent CTAs): the next tile's lines start their way to L2 now
      const long long n_next = n + (long long)gridDim.x * wpc * spw;
      if (A.prefetch && n_next < A.N && m0 < M) prefetch_tile_l2<FIXED>(A, n_next * M + m0);
    }
    if (K1_SHAPE(ego_action, nullptr) != nullptr && K1_SHAPE(do_physics, 1) && gl == 0 && scn_ok) {   // the ego's action comes from its own [N, 2] array
      const float2 ea = reinterpret_cast<const float2*>(K1_SHAPE(ego_action, nullptr))[n];
      a0[0] = ea.x; a1[0] = ea.y;
    }
    if (!staged) {   // table + map tile landed? (first tile only)
      mbar_wait(s_bar, 0);
      staged = true;
    }
    // the participant's type row; its third 16-byte group holds the collision shape and the model / shape ids
    float ch[PPL], sh[PPL];
    bool active[PPL], kin[PPL];
    const Params* pp[PPL];
    int model[PPL];
    bool lane_all_kin = true, lane_any_kin = false;
#pragma unroll
    for (int i = 0; i < PPL; ++i) {
      active[i] = tidv[i] < A.n_types;
      pp[i] = &s_table[active[i] ? tidv[i] : 0];
      model[i] = pp[i]->model_shape & 0xff;
      kin[i] = active[i] && (model[i] == MODEL_KINEMATICS);
      lane_all_kin = lane_all_kin && kin[i];
      lane_any_kin = lane_any_kin || kin[i];
      ch[i] = 1.0f; sh[i] = 0.0f;
    }
    T2D_TL(2, tl_on, tl_slot, sx[PPL - 1] + sy[PPL - 1] + shd[PPL - 1] + sv[PPL - 1] + a0[PPL - 1] + a1[PPL - 1] + (float)model[PPL - 1]);
    if (A.cfg_flags & T2D_CFG_STEER_FIRST) {
#pragma unroll
      for (int i = 0; i < PPL; ++i)
        if (model[i] <= MODEL_DYNAMICS || model[i] == MODEL_DRIFT) { float t = a0[i]; a0[i] = a1[i]; a1[i] = t; }
    }

    // ------------------------------------------------------------------ physics
    if (K1_SHAPE(do_physics, 1)) {
      // Kinematic participants of the whole warp advance together in the 4-chain loop; slots holding another
      // model (or nothing) ride along on a neutral row (zero speed / action, unbounded ranges) and are discarded.
      if (__any_sync(0xffffffffu, lane_any_kin)) {
        const Params* const null_row = &s_table[A.n_types];
        const Params* pk[PPL];
        KinIO<PPL> io;
#pragma unroll
        for (int i = 0; i < PPL; ++i) {
          pk[i] = kin[i] ? pp[i] : null_row;
          io.x[i] = kin[i] ? sx[i] : 0.0f; io.y[i] = kin[i] ? sy[i] : 0.0f;
          io.h[i] = kin[i] ? shd[i] : 0.0f; io.v[i] = kin[i] ? sv[i] : 0.0f;
          io.acc[i] = kin[i] ? a0[i] : 0.0f; io.steer[i] = kin[i] ? a1[i] : 0.0f;
        }
        kinematics_step<PPL>(io, pk, A.n_steps, A.dt, A.dt_rem);
#pragma unroll
        for (int i = 0; i < PPL; ++i) {
          if (kin[i]) {
            sx[i] = io.x[i]; sy[i] = io.y[i]; shd[i] = io.h[i]; sv[i] = io.v[i];
            svx[i] = io.vx[i]; svy[i] = io.vy[i]; ch[i] = io.ch[i]; sh[i] = io.sh[i];
          }
        }
      }
      if (!lane_all_kin) {
#pragma unroll
        for (int i = 0; i < PPL; ++i) {
          if (active[i] && !kin[i]) {
            if constexpr (!KIN_ONLY) {
              OneIO io;
              io.x = sx[i]; io.y = sy[i]; io.h = shd[i]; io.v = sv[i]; io.vx = svx[i]; io.vy = svy[i];
              io.a0 = a0[i]; io.a1 = a1[i];
              io.ch = 1.0f; io.sh = 0.0f;
              other_model_step(io, *pp[i], A.n_steps, A.dt_d, A.dt_rem_d, A.interval_d);
              sx[i] = io.x; sy[i] = io.y; shd[i] = io.h; sv[i] = io.v; svx[i] = io.vx; svy[i] = io.vy;
              ch[i] = io.ch; sh[i] = io.sh;
            } else {
              sincos_fast(shd[i], &sh[i], &ch[i]);   // static participant: the pose only
            }
          }
        }
      }
      // ---------------------------------------------------------------- store state
      bool all_active = true;
#pragma unroll
      for (int i = 0; i < PPL; ++i) all_active = all_active && active[i];
      if (nvalid == PPL && K1_SHAPE(vec_ok, 1) && all_active) {   // (an inactive slot keeps its state: vx, vy may not even be loaded)
        st_vec<float, PPL>(A.x + idx0, sx);
        st_vec<float, PPL>(A.y + idx0, sy);
        st_vec<float, PPL>(A.h + idx0, shd);
        st_vec<float, PPL>(A.v + idx0, sv);
        st_vec<float, PPL>(A.vx + idx0, svx);
        st_vec<float, PPL>(A.vy + idx0, svy);
      } else {
#pragma unroll
        for (int i = 0; i < PPL; ++i) {
          if (i < nvalid && active[i]) {
            A.x[idx0 + i] = sx[i]; A.y[idx0 + i] = sy[i]; A.h[idx0 + i] = shd[i]; A.v[idx0 + i] = sv[i];
            A.vx[idx0 + i] = svx[i]; A.vy[idx0 + i] = svy[i];
          }
        }
      }
    } else {
#pragma unroll
      for (int i = 0; i < PPL; ++i) sincos_fast(shd[i], &sh[i], &ch[i]);
    }
    T2D_TL(3, tl_on, tl_slot, sx[0] + sy[PPL - 1] + ch[0] + sh[PPL - 1]);

    // ------------------------------------------------------------------ poses -> shared
    // Only (x, y, bounding radius) stay in registers; the full pose lives in the warp's smem tile.
    float px[PPL], py[PPL], rb[PPL];
    unsigned solid_bits = 0;
#pragma unroll
    for (int i = 0; i < PPL; ++i) {
      const Vec4 g2 = params_group(pp[i], 2);             // (pose_l, pose_w, rbound, model | shape << 8): one 128-bit load
      const bool sol = active[i] && (__float_as_int(g2.w) >> 8) != SHAPE_NONE;
      solid_bits |= sol ? (1u << i) : 0u;
      rb[i] = g2.z;                                       // bounding radius, rounded up so the broadphase is conservative
      px[i] = sol ? sx[i] : __int_as_float(0x7fc00000);   // NaN: a non-solid slot never passes a distance test
      py[i] = sy[i];
      // (lane-minor layout, see pslot: these stores are conflict-free)
      poseA[i * 32 + lane] = make_float4(px[i], py[i], rb[i], shd[i]);
      poseB[i * 32 + lane] = make_float4(ch[i], sh[i], g2.x, g2.y);
    }
    if (lane == 0) *qcount = 0;
    __syncwarp();
    // the step counter of the status section: fetched here - behind the state stores, so it cannot be hoisted to the top
    // of the tile (where ptxas spilled it, stalling the warp on HBM before its state loads were even issued), and with
    // the whole collision phase in front of its first use
    const int cnt_in = (K1_SHAPE(do_physics, 1) && gl == 0 && scn_ok) ? A.step_count[n] : 0;

    // static broadphase level 1 (clearance field: one byte per participant through L1/L2), issued here so that
    // its global-load latency hides behind the partner loop
    unsigned near_q[PPL], near_alt[PPL];
#pragma unroll
    for (int i = 0; i < PPL; ++i) { near_q[i] = 255u; near_alt[i] = 255u; }   // 255 = far from every segment
    // this lane's tile (all PPL participants of a lane belong to one scenario)
    const MapHeader* lane_mh = &A.mh;
    const unsigned char* lane_blob = A.map_blob;
    if constexpr (MAP_TABLE) {
      lane_blob = A.map_blob + A.tile_off[scn_ok ? A.tile_id[n] : 0];
      lane_mh = reinterpret_cast<const MapHeader*>(lane_blob);
    }
    if (A.map_blob != nullptr && lane_mh->n_seg > 0) {
#pragma unroll
      for (int i = 0; i < PPL; ++i) {
        unsigned alt;
        near_q[i] = near_fetch(px[i], py[i], rb[i], *lane_mh, lane_blob + lane_mh->off_fine, alt);   // (a NaN position reads cell 0 and is "outside": alt = 255)
        near_alt[i] = ((solid_bits >> i) & 1u) ? alt : 255u;
      }
    }

    // ------------------------------------------------------------------ dynamic collision
    // Broadphase: every unordered pair of a scenario is tested in the orientation(s) of the circular enumeration - owner i,
    // partner (i + 1 .. i + M/2) mod M (sweep_pair) - but only the pairs that can be candidates are enumerated: the group
    // sorts its scenario's slots by x and each sorted entry is paired with the entries after it up to the reach.
    // Candidates (rare) go on the warp's queue; after the sweep all 32 lanes drain it (narrowphase), recording a hit for
    // both ends by atomicMin in shared memory on the scenario-local partner index.
    int hit[PPL];
    {
      // (1) Sort.  Key of slot m0 + i: f2ord(x) with its low 7 bits replaced by the slot (MP <= 128), so the keys are
      // distinct and one unsigned min / max moves key and payload together; a non-solid or padding slot (x NaN) takes
      // 0xffffff80 | slot, above every solid key.  Bitonic network over element e = 4 gl + k of the group: strides 1
      // and 2 are compare-exchanges inside the lane, larger strides __shfl_xor_sync inside the group (the group's lanes
      // are aligned to G, so lane ^ j stays in it).  A tie in x is ordered by slot, which the scan below does not need.
      unsigned key[PPL];
#pragma unroll
      for (int i = 0; i < PPL; ++i)
        key[i] = (px[i] == px[i] ? (f2ord(px[i]) & ~127u) : 0xffffff80u) | (unsigned)(m0 + i);
      auto cx = [&](int a, int b, bool desc) {
        const unsigned lo = min(key[a], key[b]), hi = max(key[a], key[b]);
        key[a] = desc ? hi : lo;
        key[b] = desc ? lo : hi;
      };
      // FIXED: start from the previous tick's order instead.  Entry e = 4 gl + k takes the slot s = hint byte k & 63 and
      // its key is built as above, from the x in the pose tile; T2D_ORDER_PASSES odd-even transposition passes (an even
      // phase: pairs (4 gl, 4 gl + 1), (4 gl + 2, 4 gl + 3); an odd phase: (4 gl + 1, 4 gl + 2) and, across lanes,
      // (4 gl + 3, 4 gl + 4)) repair it, and the result is kept if every key is strictly below its successor in every
      // scenario of the warp.  Otherwise the whole warp runs the network on the keys above (one decision per warp, so the
      // network's shuffles see every lane).
      //
      // Why the kept list is the network's output, bit for bit.  A key is a function of its slot alone, so keys of
      // distinct slots differ in their low bits and keys of equal slots are equal: 64 strictly ascending keys therefore
      // name 64 distinct slots of 0..63, every slot once, whatever the hint held (a stale, duplicated or corrupt hint
      // cannot pass).  The passes only compare-exchange, so the list is a permutation of the key set the network sorts;
      // a strictly ascending arrangement of a set is unique, and the network's output is one.  From (2) on the tick
      // sees the same keys in the same entries, so the scan, the queue, the drain and every output are unchanged.  A
      // stale hint costs time, never a result; it is stored back only where the sorted slots differ from it.
      bool hinted = false;
      if constexpr (FIXED) {
        unsigned hk[PPL];
#pragma unroll
        for (int i = 0; i < PPL; ++i) {
          const unsigned s = (hint >> (8 * i)) & 63u;
          const float x = poseA[pslot(tb + (int)s)].x;
          hk[i] = (x == x ? (f2ord(x) & ~127u) : 0xffffff80u) | s;
        }
        auto up = [&](int a, int b) {
          const unsigned lo = min(hk[a], hk[b]), hi = max(hk[a], hk[b]);
          hk[a] = lo;
          hk[b] = hi;
        };
#pragma unroll
        for (int pass = 0; pass < T2D_ORDER_PASSES; ++pass) {
          up(0, 1); up(2, 3);
          up(1, 2);
          const unsigned next = __shfl_down_sync(0xffffffffu, hk[0], 1);
          const unsigned prev = __shfl_up_sync(0xffffffffu, hk[PPL - 1], 1);
          if (gl != G - 1) hk[PPL - 1] = min(hk[PPL - 1], next);
          if (gl != 0) hk[0] = max(hk[0], prev);
        }
        const unsigned next = __shfl_down_sync(0xffffffffu, hk[0], 1);
        const bool ascending = hk[0] < hk[1] && hk[1] < hk[2] && hk[2] < hk[3] && (gl == G - 1 || hk[3] < next);
        hinted = __all_sync(0xffffffffu, ascending);
        if (hinted) {
#pragma unroll
          for (int i = 0; i < PPL; ++i) key[i] = hk[i];
        } else if (lane == 0) {
          atomicAdd(&A.order_fallbacks[(blockIdx.x & (ORDER_COUNTERS - 1)) * ORDER_COUNTER_STRIDE], 1ull);
        }
      }
      if (!hinted) {
        cx(0, 1, false); cx(2, 3, true);   // sorted runs of 2, alternating in direction (element bit 1)
        for (int S = PPL; S <= MP; S <<= 1) {           // merge into sorted runs of S (the last one, S = MP, ascending)
          const bool desc = (gl & (S >> 2)) != 0;       // element bit log2(S) = lane bit log2(S / 4)
          for (int j = S >> 3; j > 0; j >>= 1) {        // element stride 4 j = lane stride j
            const bool keep_max = ((gl & j) != 0) != desc;
#pragma unroll
            for (int i = 0; i < PPL; ++i) {
              const unsigned o = __shfl_xor_sync(0xffffffffu, key[i], j);
              key[i] = keep_max ? max(key[i], o) : min(key[i], o);
            }
          }
          cx(0, 2, desc); cx(1, 3, desc); cx(0, 1, desc); cx(2, 3, desc);
        }
      }
      if constexpr (FIXED) {
        const uint32_t sorted_slots = (key[0] & 127u) | (key[1] & 127u) << 8 | (key[2] & 127u) << 16 | (key[3] & 127u) << 24;
        if (scn_ok && sorted_slots != hint) *reinterpret_cast<uint32_t*>(A.order + idx0) = sorted_slots;
      }
      T2D_TL(4, tl_on, tl_slot, __uint_as_float(key[0] ^ key[PPL - 1]));
      // (2) Stage the sorted list: entry 4 gl + k = (x, y, -thr, key) of the slot the key names, from the pose tile.
      float4 own[PPL];
#pragma unroll
      for (int i = 0; i < PPL; ++i) {
        const float4 a = poseA[pslot(tb + (int)(key[i] & 127u))];
        own[i] = make_float4(a.x, a.y, neg_reach2(a.z, A.rb_max), __uint_as_float(key[i]));
        sorted[m0 + i] = own[i];
      }
      __syncwarp();
      // (3) Scan.  Entry p is paired with every entry q > p of its scenario up to the first q whose bucket floor
      // lo_q = ord2f(key_q & ~127) satisfies fl(lo_q - xmax) > T, where xmax >= x_p (the max over the lane's own entries)
      // and T = fl(fma(2 rb_max, 1.0001f, 1e-5f)).
      //
      // Why no pair beyond the stop is a candidate, in either orientation.  Let owner o, partner r have the margin
      // fma(dx, dx, fma(dy, dy, -thr_o)) <= 0 with dx = fl(x_r - x_o), as sweep_pair computes it.  A NaN or infinite
      // operand makes the margin NaN or +inf, so both positions are finite.  (a) Rounding is monotone and every
      // v >= 2^-149 rounds to >= 2^-149 > 0, so the margin <= 0 means dx^2 + e < 2^-149 for e = fl(dy^2 - thr_o) >= -thr_o
      // (thr_o is a float): |dx| < sqrt(thr_o) + 2^-74.  (b) dx rounds the exact x_r - x_o with relative error 2^-24
      // (absolute 2^-150 among subnormals), so |x_r - x_o| < (sqrt(thr_o) + 2^-74)(1 + 2^-23) + 2^-149.  (c) thr_o =
      // fl(fl(rr^2) * 1.00001f + 1e-12f) with rr = fl(rb_o + rb_max) <= 2 rb_max (exact doubling, monotone rounding), so
      // sqrt(thr_o) <= rr * 1.0000051 * (1 + 2^-24) + 1.0000001e-6 and |x_r - x_o| < D = 2 rb_max * 1.0000054 + 1.1e-6,
      // whichever end owns the pair.  (d) T >= (2 rb_max * 1.0001f + 1e-5f)(1 - 2^-24) > D.  (e) The keys are sorted, so
      // for q' >= q the bucket floors are ordered, lo_q' >= lo_q, and x_q' >= lo_q' (f2ord is monotone and clearing low
      // bits only lowers it); every own p has x_p <= xmax.  A stop with fl(lo_q - xmax) > T means lo_q - xmax > T exactly
      // (T is a float and rounding is monotone), so x_q' - x_p > T > D: no candidate, at any coordinate magnitude.  A NaN
      // test stops the scan too; that happens only when lo_q is NaN (q non-solid, so are all later entries; or x_q = -inf,
      // whose bucket holds no finite x, so every own x is -inf as well) or when lo_q = xmax = +inf: in each case every
      // remaining pair has a non-finite position.  An own entry that is not solid has x NaN, which fmaxf leaves out; a
      // lane with no solid entry has xmax NaN and stops at once (its own pairs have NaN margins).
      //
      // The pairs enumerated are each unordered pair of sorted ranks {p < q} at most once (by the lane holding p), and
      // sweep_pair decides owner and margin exactly as the circular sweep does, so the queue receives the same set of
      // (owner, partner) entries - only in another order, which the atomicMin drain does not see - and an overflow
      // triggers on the same count.  At C2 (64 participants over 200 m of x, T = 5.65 m) an entry has about 1.8
      // x-neighbours within T, so a lane scans its 6 own pairs and one group of 4 entries beyond them.
      const float T = fmaf(2.0f * A.rb_max, 1.0001f, 1e-5f);
      const float nglob = neg_reach2(A.rb_max, A.rb_max);
      const float xmax = fmaxf(fmaxf(own[0].x, own[1].x), fmaxf(own[2].x, own[3].x));
      {
        float m = INFINITY;
#pragma unroll
        for (int a = 0; a < PPL; ++a)
#pragma unroll
          for (int b = a + 1; b < PPL; ++b) m = fminf(m, pair_min_margin(own[a], own[b], nglob));
        if (m <= 0.0f) {
#pragma unroll
          for (int a = 0; a < PPL; ++a)
#pragma unroll
            for (int b = a + 1; b < PPL; ++b) sweep_pair(own[a], own[b], tb, M, Mh, queue, qcount);
        }
      }
      if (xmax == xmax) {
        for (int q0 = m0 + PPL; q0 < MP; q0 += PPL) {   // four entries per round, loaded together (MP is a multiple of 4)
          float4 e[PPL];
#pragma unroll
          for (int k = 0; k < PPL; ++k) e[k] = sorted[q0 + k];
          bool stop = false;
#pragma unroll
          for (int k = 0; k < PPL; ++k) {
            if (!(ord2f(__float_as_uint(e[k].w) & ~127u) - xmax <= T)) { stop = true; break; }
            float m = INFINITY;
#pragma unroll
            for (int a = 0; a < PPL; ++a) m = fminf(m, pair_min_margin(own[a], e[k], nglob));
            if (m <= 0.0f) {
#pragma unroll
              for (int a = 0; a < PPL; ++a) sweep_pair(own[a], e[k], tb, M, Mh, queue, qcount);
            }
          }
          if (stop) break;
        }
      }
      T2D_TL(5, tl_on, tl_slot, xmax);
#pragma unroll
      for (int i = 0; i < PPL; ++i) hitmin[i * 32 + lane] = 0x7fffffff;
      __syncwarp();   // the queue holds every candidate
      // narrowphase: the queued candidate pairs, one per lane (or the exhaustive pass if the queue overflowed)
      const int n_q = *qcount;
      if (n_q <= QCAP) {
        for (int k = lane; k < n_q; k += 32) {
          const unsigned e = queue[k];
          pair_resolve((int)(e >> 16), (int)(e & 0xffffu), mp_shift, poseA, poseB, hitmin);
        }
      } else {
        pair_exhaustive(t0, tb, m0, M, mp_shift, A.rb_max, poseA, poseB, hitmin);
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < PPL; ++i) {
        const int h = hitmin[i * 32 + lane];
        hit[i] = (h == 0x7fffffff) ? -1 : h;
        hitmin[i * 32 + lane] = 0x7fffffff;   // reused below as the per-participant first-hit segment
      }
      if (lane == 0) *qcount = 0;
      __syncwarp();
    }
    T2D_TL(6, tl_on, tl_slot, (float)(hit[0] + hit[PPL - 1]));

    // ------------------------------------------------------------------ static collision
    int hseg[PPL];
#pragma unroll
    for (int i = 0; i < PPL; ++i) hseg[i] = -1;
    if (A.map_blob != nullptr) {
      unsigned near_bits = 0;
#pragma unroll
      for (int i = 0; i < PPL; ++i)
        if (((solid_bits >> i) & 1u) && near_decide(near_q[i], near_alt[i], rb[i])) near_bits |= 1u << i;
      if (__any_sync(0xffffffffu, near_bits != 0)) {
        static_phase<MAP_TABLE>(near_bits, t0, lane, tile * spw, mp_shift, A, s_map, poseA, poseB, hitmin, queue, qcount);
#pragma unroll
        for (int i = 0; i < PPL; ++i) {
          const int h = hitmin[i * 32 + lane];
          hseg[i] = (h == 0x7fffffff) ? -1 : h;
        }
      }
    }
    T2D_TL(7, tl_on, tl_slot, (float)(hseg[0] + hseg[PPL - 1]));

    // ------------------------------------------------------------------ out of bound + flags
    // the boundary box of this lane's scenario (Map.boundary of its tile)
    float bxmin = A.bxmin, bxmax = A.bxmax, bymin = A.bymin, bymax = A.bymax;
    bool has_bounds = A.has_bounds != 0;
    if constexpr (MAP_TABLE) {
      has_bounds = lane_mh->has_bounds != 0;
      bxmin = lane_mh->bxmin; bxmax = lane_mh->bxmax; bymin = lane_mh->bymin; bymax = lane_mh->bymax;
    }
    uint8_t fl[PPL];
    unsigned oob_check = 0;   // participants whose bounding circle is not well inside the box (rare): settled below, once
#pragma unroll
    for (int i = 0; i < PPL; ++i) {
      uint8_t f = 0;
      if (hit[i] >= 0) f |= T2D_F_DYNAMIC;
      if (hseg[i] >= 0) f |= T2D_F_STATIC;
      // the bounding circle well inside the box: inside for sure (the common case)
      const float r = rb[i] * 1.0001f + 1e-3f;
      const bool clear_in = (px[i] - bxmin > r) && (bxmax - px[i] > r) && (py[i] - bymin > r) && (bymax - py[i] > r);
      if (has_bounds && ((solid_bits >> i) & 1u) && !clear_in) oob_check |= 1u << i;
      fl[i] = f;
    }
    if (oob_check) {
#pragma unroll
      for (int i = 0; i < PPL; ++i)
        if (((oob_check >> i) & 1u) && oob_slow(poseA, poseB, t0 + i, bxmin, bxmax, bymin, bymax)) fl[i] |= T2D_F_OUTBOUND;
    }
    if (nvalid == PPL && K1_SHAPE(vec_ok, 1)) {
      int16_t h16[PPL], s16[PPL];
#pragma unroll
      for (int i = 0; i < PPL; ++i) { h16[i] = (int16_t)hit[i]; s16[i] = (int16_t)hseg[i]; }
      if (A.flags) st_vec<uint8_t, PPL>(A.flags + idx0, fl);
      if (A.hit_index) st_vec<int16_t, PPL>(A.hit_index + idx0, h16);
      if (A.hit_segment) st_vec<int16_t, PPL>(A.hit_segment + idx0, s16);
    } else {
#pragma unroll
      for (int i = 0; i < PPL; ++i) {
        if (i < nvalid) {
          if (A.flags) A.flags[idx0 + i] = fl[i];
          if (A.hit_index) A.hit_index[idx0 + i] = (int16_t)hit[i];
          if (A.hit_segment) A.hit_segment[idx0 + i] = (int16_t)hseg[i];
        }
      }
    }

    // ------------------------------------------------------------------ scenario status
    if (K1_SHAPE(do_physics, 1)) {
      unsigned agg;
      if (A.cfg_flags & T2D_CFG_ANY_PARTICIPANT) {
        agg = 0;
#pragma unroll
        for (int i = 0; i < PPL; ++i) agg |= fl[i];
        for (int o = G >> 1; o > 0; o >>= 1) agg |= __shfl_xor_sync(0xffffffffu, agg, o);
      } else {
        agg = __shfl_sync(0xffffffffu, (unsigned)fl[0], sub * G);   // participant 0 = the ego
      }
      if (gl == 0 && scn_ok) {
        const int cnt = cnt_in + 1;                                  // parking.py:353 (loaded with the state)
        A.step_count[n] = cnt;
        uint8_t st = T2D_STATUS_NORMAL;
        unsigned goal = 0;
        if (K1_SHAPE(goal.target, nullptr) != nullptr) {   // the ego is participant 0 = this lane's first slot
          const float4 ea = poseA[pslot(t0)], eb = poseB[pslot(t0)];
          if (ea.x == ea.x && eb.w >= 0.0f) goal = ego_goal_events(A, n, ea.x, ea.y, ea.w, eb.z, eb.w);
        }
        if (goal & 1u) st = T2D_STATUS_COMPLETED;                    // parking.py:387-390 (lowest priority)
        if (agg & T2D_F_DYNAMIC) st = T2D_STATUS_FAILED;
        if (agg & T2D_F_STATIC) st = T2D_STATUS_FAILED;              // parking.py:381-385
        if (agg & T2D_F_OUTBOUND) st = T2D_STATUS_OUT_BOUND;         // parking.py:376-379
        if (goal & 2u) st = T2D_STATUS_NO_ACTION;                    // parking.py:371-374
        if (A.max_step > 0 && cnt > A.max_step) st = T2D_STATUS_TIME_EXCEEDED;  // parking.py:366-369
        if (A.scn_status) A.scn_status[n] = st;
        if (A.done) A.done[n] = st != T2D_STATUS_NORMAL;             // parking.py:243-248
      }
    }
    T2D_TL(8, tl_on, tl_slot, 0.0f);
    __syncwarp();   // pose tile is reused by the next tile
  }
  if (!staged) mbar_wait(s_bar, 0);   // never leave a bulk copy in flight at exit
#undef K1_SHAPE
}

// ---------------------------------------------------------------------------- drift pre-pass
// SingleTrackDrift participants of a tick, one per thread, before K1 (which then only builds their pose).
__global__ void __launch_bounds__(128) t2d_drift_kernel(const __grid_constant__ StepArgs A) {
  const long long total = (long long)A.N * A.M;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int tid = A.type_id[i];
    if (tid >= A.n_types) continue;
    const Params& p = A.table[tid];
    if (p.model() != MODEL_DRIFT) continue;
    OneIO io;
    io.x = A.x[i]; io.y = A.y[i]; io.h = A.h[i]; io.v = A.v[i]; io.vx = 0.0f; io.vy = 0.0f;
    float2 act = reinterpret_cast<const float2*>(A.action)[i];
    if (A.ego_action != nullptr && i % A.M == 0) act = reinterpret_cast<const float2*>(A.ego_action)[i / A.M];
    const bool sf = (A.cfg_flags & T2D_CFG_STEER_FIRST) != 0;
    io.a0 = sf ? act.y : act.x; io.a1 = sf ? act.x : act.y;
    io.ch = 1.0f; io.sh = 0.0f;
    io.w0 = A.wheel_f[i]; io.w1 = A.wheel_r[i];
    drift_step(io, p, A.n_steps, A.dt_d, A.dt_rem_d);
    A.x[i] = io.x; A.y[i] = io.y; A.h[i] = io.h; A.v[i] = io.v; A.vx[i] = io.vx; A.vy[i] = io.vy;
    A.wheel_f[i] = io.w0; A.wheel_r[i] = io.w1;
  }
}

// ---------------------------------------------------------------------------- K3
struct PhysArgs {
  Params p;
  float *x, *y, *h, *v, *vx, *vy;
  float *wheel_f, *wheel_r;
  const float* action;
  float* applied;
  int n, n_steps;
  float dt, dt_rem;
  double dt_d, dt_rem_d, interval_d;
};

__global__ void __launch_bounds__(256) t2d_physics_kernel(const __grid_constant__ PhysArgs A) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < A.n; i += (long long)gridDim.x * blockDim.x) {
    if (A.p.model() == MODEL_KINEMATICS) {
      KinIO<1> io;
      io.x[0] = A.x[i]; io.y[0] = A.y[i]; io.h[0] = A.h[i]; io.v[0] = A.v[i];
      io.acc[0] = A.action[2 * i]; io.steer[0] = A.action[2 * i + 1];
      const Params* const p1[1] = {&A.p};
      kinematics_step<1>(io, p1, A.n_steps, A.dt, A.dt_rem);
      A.x[i] = io.x[0]; A.y[i] = io.y[0]; A.h[i] = io.h[0]; A.v[i] = io.v[0]; A.vx[i] = io.vx[0]; A.vy[i] = io.vy[0];
      if (A.applied) { A.applied[2 * i] = io.acc[0]; A.applied[2 * i + 1] = io.steer[0]; }
    } else {
      OneIO io;
      io.x = A.x[i]; io.y = A.y[i]; io.h = A.h[i]; io.v = A.v[i]; io.vx = A.vx[i]; io.vy = A.vy[i];
      io.a0 = A.action[2 * i]; io.a1 = A.action[2 * i + 1];
      io.ch = 1.0f; io.sh = 0.0f;
      if (A.p.model() == MODEL_DRIFT) {
        io.w0 = A.wheel_f[i]; io.w1 = A.wheel_r[i];
        drift_step(io, A.p, A.n_steps, A.dt_d, A.dt_rem_d);
        A.wheel_f[i] = io.w0; A.wheel_r[i] = io.w1;
      } else {
        other_model_step(io, A.p, A.n_steps, A.dt_d, A.dt_rem_d, A.interval_d);
      }
      A.x[i] = io.x; A.y[i] = io.y; A.h[i] = io.h; A.v[i] = io.v; A.vx[i] = io.vx; A.vy[i] = io.vy;
      if (A.applied) { A.applied[2 * i] = io.a0; A.applied[2 * i + 1] = io.a1; }
    }
  }
}

}  // namespace t2d
