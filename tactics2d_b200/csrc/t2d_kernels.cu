// t2d_kernels.cu - sm_90a kernels and the C ABI (include/t2d_b200.h) of the batched tick.
//
// K1  t2d_step_kernel      fused physics -> pose -> dynamic collision (broadphase + filtered
//                          narrowphase) -> static collision against the map tile in shared
//                          memory (uniform-grid broadphase) -> out-of-bound -> status chain.
//                          (+ t2d_drift_kernel: pre-pass for SingleTrackDrift participants.)
// K2  t2d_reset_kernel     masked re-initialisation from a pool of initial states.
// K3  t2d_physics_kernel   flat batch through one physics model (PhysicsModelBase.step).
// K4  t2d_lidar_kernel     single-line lidar of every scenario's ego (per-edge beam windows).
// K5  t2d_control_kernel   NPC controllers: IDM, cruise / adaptive cruise, pure pursuit, PID.
// K7  t2d_replay_kernel    log replay: recorded tracks pose the replayed slots before K1 / after K2.
// K8  t2d_obs_kernel       the ego-frame vector observation (t2d_obs.cuh).
// K9  t2d_obs_agents_kernel the same observation from a list of observer slots per scenario (t2d_obs.cuh).
// K10 t2d_agents_epilogue_kernel status, reward and retirement of every agent row of an observer list.
// K11 t2d_agent_action_kernel    the action of every agent row of an observer list, scattered to its slot.
// K12 t2d_route_obs_kernel       the route of every observer row in its frame, with look-ahead points.
// K13 t2d_episode_draw_kernel    sampled resets: the seeded pool-row draw and the row-owned columns.
// K14 t2d_episode_place_kernel   sampled resets: collision-checked jitter of the start states, one warp per scenario.
// K15 t2d_history_append_kernel  trajectory history: append the state after a tick, restart it after a reset (t2d_history.cuh).
// K16 t2d_history_obs_kernel     trajectory history: past poses of an observer and its agents in its current frame.
//     t2d_exchange_allgather_kernel   all-gather of the done masks over NVLink peer memory.
//
// Work decomposition of K1: a scenario (M <= 128 participants) is owned by a group of G lanes of
// one warp, 4 consecutive participants per lane (one float4 per state array per lane: coalesced
// 128-bit loads, 4 independent Euler chains per thread for ILP).  G = pow2 >= ceil(M/4), so a
// warp holds 32/G scenarios and every exchange inside a scenario is warp-synchronous: poses go
// through a per-warp shared-memory tile + __syncwarp, reductions through shuffles.  CTAs are
// persistent (grid = SMs x resident CTAs) and stage the static map tile (segments + broadphase
// grid) into shared memory ONCE with a TMA bulk copy (cp.async.bulk + mbarrier) that overlaps
// the first tile's physics.
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/t2d_b200.h"
#include "t2d_math.cuh"

namespace t2d {

constexpr int MAX_WARPS_PER_CTA = 8;
constexpr int CTA_THREADS = MAX_WARPS_PER_CTA * 32;   // upper bound; the host picks the warps per CTA (pick_wpc)
constexpr int PPL = 4;                  // participants per lane of K1
constexpr int POSE_PER_WARP = 32 * PPL;
constexpr int MAP_SMEM_LIMIT = 120 * 1024;

struct MapHeader {   // 128 bytes, start of a tile's blob
  int32_t n_seg, gx, gy, n_items;
  float x0, y0, inv_cell, cell;
  uint32_t off_seg, off_cell, off_items, total_bytes;
  uint32_t off_clear;   // float per cell: lower bound of the distance from any point of the cell to any segment
  int32_t fine;         // the fine clearance field has (gx * fine) x (gy * fine) cells, one byte each (global memory)
  // "dilated" lists: cell c lists (ascending) every segment that comes within `dil` metres of the cell's box, so that a
  // participant whose bounding radius is <= dil finds all its candidates in the ONE cell under its centre (the grid
  // covers the segments' bounding box grown by dil: a centre outside it cannot reach a segment)
  uint32_t off_dcell, off_ditems;
  float dil;
  int32_t n_ditems;
  uint32_t off_objfirst;   // uint16 per segment: first segment of the object (polygon / polyline piece) it belongs to
  int32_t n_poly;          // closed rings among the segments (Area.geometry polygons)
  uint32_t off_poly;       // int32 [n_poly + 1]: ring p = segments [start[p], start[p + 1])
  uint32_t off_pbox;       // float4 per ring: xmin, xmax, ymin, ymax
  uint32_t off_fine;       // the fine clearance field (bytes), last section of the blob
  uint32_t smem_bytes;     // = off_fine: the part worth staging into shared memory
  float bxmin, bxmax, bymin, bymax;   // Map.boundary of the tile (OutBound)
  int32_t has_bounds;
  uint32_t pad[3];
};
constexpr float CLEAR_QUANT = 0.125f;   // metres per unit of the byte-quantised fine clearance field
static_assert(sizeof(MapHeader) == 128, "MapHeader must be 128 bytes");

// The bound world as t2d_ctx holds it (world_args): the state and the type table every kernel besides K1, its drift
// pre-pass and K7 reads.  Their argument structs derive from it.
struct WorldArgs {
  float *x, *y, *h, *v, *vx, *vy;  // [N][M]
  const uint8_t* type_id;          // [N][M]
  int32_t* step_count;             // [N]
  const Params* table;             // device
  int n_types, N, M;
};

// The bound map as K4, K6 and K8 / K9 read it (map_args); tile_blob finds a scenario's tile in it.
struct MapArgs {
  const unsigned char* map_blob;   // device: the tiles' blobs, one after the other; nullptr when no tile has segments
  const uint32_t* tile_off;        // [n_tiles] byte offset of every tile's blob
  const uint16_t* tile_id;         // [N] the tile of every scenario, or nullptr: every scenario uses tile 0
};

// The blob of scenario n's tile, or nullptr when no tile has geometry (tile 0 starts the blob: no table, no lookup)
__device__ __forceinline__ const unsigned char* tile_blob(const MapArgs& m, long long n) {
  return m.map_blob ? m.map_blob + (m.tile_id ? m.tile_off[m.tile_id[n]] : 0u) : nullptr;
}

// The Arrival / NoAction detector state of a set of rows (ego_goal_events): the ego of every scenario (t2d_set_goal,
// [N] rows) or every agent row (t2d_set_agents, [N][Q] rows).
struct GoalArgs {
  const float* target;             // [rows][5] cx, cy, heading, half_len, half_wid of the target area, or nullptr
  float* iou;                      // [rows]
  float* last_pose;                // [rows][4] x, y, heading, valid
  int32_t* noact_count;            // [rows]
  float threshold;
  int noact_max;
};

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

// ---------------------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA bulk copy global -> shared, completion signalled on the mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}

// ---------------------------------------------------------------------------- vector access
// N consecutive elements of an [N_scn, M] array as ONE load / store of sizeof(T) * N bytes (<= 16).
template <int BYTES> struct VecOf;
template <> struct VecOf<1> { using T = uint8_t; };
template <> struct VecOf<2> { using T = uint16_t; };
template <> struct VecOf<4> { using T = uint32_t; };
template <> struct VecOf<8> { using T = uint2; };
template <> struct VecOf<16> { using T = uint4; };

template <typename T, int N>
__device__ __forceinline__ void ld_vec(const T* p, T (&o)[N]) {
  using V = typename VecOf<sizeof(T) * N>::T;
  const V v = *reinterpret_cast<const V*>(p);
  memcpy(o, &v, sizeof(V));
}
template <typename T, int N>
__device__ __forceinline__ void st_vec(T* p, const T (&o)[N]) {
  using V = typename VecOf<sizeof(T) * N>::T;
  V v;
  memcpy(&v, o, sizeof(V));
  *reinterpret_cast<V*>(p) = v;
}

// ---------------------------------------------------------------------------- pair narrowphase
// A pose is (x, y, heading, c, s, l, w); w < 0 marks a disc of radius l.
struct Pose {
  float x, y, h, c, s, l, w;
};

__device__ __noinline__ bool pair_exact(const Pose a, const Pose b) {
  const bool ca = a.w < 0.0f, cb = b.w < 0.0f;
  if (!ca && !cb) return obb_obb_f64(a.x, a.y, a.h, a.l, a.w, b.x, b.y, b.h, b.l, b.w);
  if (!ca && cb) return obb_circle_f64(a.x, a.y, a.h, a.l, a.w, b.x, b.y, b.l);
  if (ca && !cb) return obb_circle_f64(b.x, b.y, b.h, b.l, b.w, a.x, a.y, a.l);
  return circle_circle_f64(a.x, a.y, a.l, b.x, b.y, b.l);
}

__device__ __forceinline__ bool pair_hit(const Pose& a, const Pose& b) {
  const bool ca = a.w < 0.0f, cb = b.w < 0.0f;
  int r;
  if (!ca && !cb) r = obb_obb_f32(a.x, a.y, a.c, a.s, a.l, a.w, b.x, b.y, b.c, b.s, b.l, b.w);
  else if (!ca && cb) r = obb_circle_f32(a.x, a.y, a.c, a.s, a.l, a.w, b.x, b.y, b.l);
  else if (ca && !cb) r = obb_circle_f32(b.x, b.y, b.c, b.s, b.l, b.w, a.x, a.y, a.l);
  else r = circle_circle_f32(a.x, a.y, a.l, b.x, b.y, b.l);
  if (r < 0) return pair_exact(a, b);
  return r != 0;
}

__device__ __noinline__ bool seg_exact(const Pose a, const float4 sg) {
  if (a.w < 0.0f) return circle_segment_f64(a.x, a.y, a.l, sg.x, sg.y, sg.z, sg.w);
  return obb_segment_f64(a.x, a.y, a.h, a.l, a.w, sg.x, sg.y, sg.z, sg.w);
}

__device__ __forceinline__ bool seg_hit(const Pose& a, const float4 sg) {
  int r = a.w < 0.0f ? circle_segment_f32(a.x, a.y, a.l, sg.x, sg.y, sg.z, sg.w)
                     : obb_segment_f32(a.x, a.y, a.c, a.s, a.l, a.w, sg.x, sg.y, sg.z, sg.w);
  if (r < 0) return seg_exact(a, sg);
  return r != 0;
}

__device__ __noinline__ bool oob_exact(const Pose a, float xmin, float xmax, float ymin, float ymax) {
  return out_of_bound_f64(a.x, a.y, a.h, a.l, a.w, a.w < 0.0f, xmin, xmax, ymin, ymax);
}

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

// The sections of a map blob (in shared or in global memory: the accessors are inlined, the address space is known).
struct MapView {
  const float4* seg;
  const uint32_t* cell_start;
  const uint16_t* items;
  const uint32_t* dcell_start;
  const uint16_t* ditems;
};
__device__ __forceinline__ MapView map_view(const unsigned char* blob, const MapHeader& mh) {
  MapView v;
  v.seg = reinterpret_cast<const float4*>(blob + mh.off_seg);
  v.cell_start = reinterpret_cast<const uint32_t*>(blob + mh.off_cell);
  v.items = reinterpret_cast<const uint16_t*>(blob + mh.off_items);
  v.dcell_start = reinterpret_cast<const uint32_t*>(blob + mh.off_dcell);
  v.ditems = reinterpret_cast<const uint16_t*>(blob + mh.off_ditems);
  return v;
}

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

// Area polygons (StaticCollision.update tests pose.intersects(area.geometry), collision.py:37-43): a pose that touches no
// edge still intersects the closed polygon when it lies inside it.  `best` = the lowest edge hit so far (0x7fffffff: none);
// returns the first segment of the first OBJECT hit: an edge hit is renamed to its object's first segment, and every ring
// that starts below that and contains the pose centre takes over.  The crossing-number test runs in fp32: it is only
// decisive for rings none of whose edges touch the pose, i.e. whose edges all stay at least the pose's inradius away from
// the centre - far beyond fp32 rounding.
__device__ __noinline__ int static_objects(int best, float px, float py, const MapHeader& mh, const unsigned char* blob) {
  if (best != 0x7fffffff && best >= 0) best = reinterpret_cast<const uint16_t*>(blob + mh.off_objfirst)[best];
  const int32_t* pstart = reinterpret_cast<const int32_t*>(blob + mh.off_poly);
  const float4* pbox = reinterpret_cast<const float4*>(blob + mh.off_pbox);
  const float4* seg = reinterpret_cast<const float4*>(blob + mh.off_seg);
  for (int p = 0; p < mh.n_poly; ++p) {
    const int s0 = pstart[p];
    if (s0 >= best) break;
    const float4 bb = pbox[p];
    if (!(px >= bb.x && px <= bb.y && py >= bb.z && py <= bb.w)) continue;
    bool in = false;
    for (int i = s0; i < pstart[p + 1]; ++i) {
      const float4 e = seg[i];
      if ((e.y > py) != (e.w > py) && px < (e.z - e.x) * (py - e.y) / (e.w - e.y) + e.x) in = !in;
    }
    if (in) { best = s0; break; }
  }
  return best;
}

// Out-of-line exact walk for a participant whose undecided segments did not fit the exact queue (never on the
// hot path): the same cells, every test through the fp32 filter + fp64 fallback.
__device__ __noinline__ int static_walk_exact(const Pose a, float rbound, const MapHeader mh, const float4* seg, const uint32_t* cell_start,
                                              const uint16_t* items) {
  const float r = rbound * 1.0001f + 1e-3f;
  int cx0 = max((int)floorf((a.x - r - mh.x0) * mh.inv_cell), 0), cx1 = min((int)floorf((a.x + r - mh.x0) * mh.inv_cell), mh.gx - 1);
  int cy0 = max((int)floorf((a.y - r - mh.y0) * mh.inv_cell), 0), cy1 = min((int)floorf((a.y + r - mh.y0) * mh.inv_cell), mh.gy - 1);
  int best = 0x7fffffff;
  for (int cy = cy0; cy <= cy1; ++cy)
    for (int cx = cx0; cx <= cx1; ++cx) {
      const int cidx = cy * mh.gx + cx;
      for (uint32_t k = cell_start[cidx]; k < cell_start[cidx + 1]; ++k) {
        const int sidx = items[k];
        if (sidx >= best) break;
        if (seg_hit(a, seg[sidx])) best = sidx;
      }
    }
  return best;
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

// Arrival (arrival.py:32-47) and NoAction (no_action.py:32-53) for row n of the detector record A.goal; returns bit0 =
// arrived, bit1 = no action for more than max_step consecutive ticks.  One lane per row, fp64, out of line: K1 (the ego)
// and K10 (the agent rows) run the same code, so that their detectors agree bit for bit.  It takes the kernel's whole
// argument block rather than &A.goal: the address of a member of a kernel parameter is loop-invariant, and K1 would hold
// it in two registers across its tile loop.
template <class Args>
__device__ __noinline__ unsigned ego_goal_events(const Args& A, long long n, float ex, float ey, float eh, float el, float ew) {
  const GoalArgs& G = A.goal;
  unsigned r = 0;
  float* last = G.last_pose + 4 * n;
  if (G.noact_max > 0) {
    int cnt = G.noact_count[n];
    if (last[3] != 0.0f) {                                          // no_action.py:40-50
      const double iou = rect_iou_f64(ex, ey, eh, el, ew, last[0], last[1], last[2], el, ew);
      cnt = iou > 0.999 ? cnt + 1 : 0;
    }
    G.noact_count[n] = cnt;
    if (cnt > G.noact_max) r |= 2u;                                 // no_action.py:53
  }
  last[0] = ex; last[1] = ey; last[2] = eh; last[3] = 1.0f;         // no_action.py:39,51
  const float* tg = G.target + 5 * n;
  const double iou = rect_iou_f64(ex, ey, eh, el, ew, tg[0], tg[1], tg[2], tg[3], tg[4]);   // arrival.py:42-44
  G.iou[n] = (float)iou;
  if (iou >= (double)G.threshold) r |= 1u;                          // arrival.py:45
  return r;
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

// ---------------------------------------------------------------------------- K2
struct ResetArgs : WorldArgs {
  const uint8_t* mask;
  const int32_t* pool_index;
  const float *px, *py, *ph, *pv, *pvx, *pvy;
  GoalArgs goal;                       // the ego's NoAction state starts fresh
  // per-participant state owned by the world besides x .. vy: the SingleTrackDrift wheel speeds and the controllers'
  // State.accel of the previous tick - a new episode must not inherit them from the old one
  float *wheel_f, *wheel_r;            // [N][M] or nullptr
  const float *pool_wf, *pool_wr;      // [n_pool][M] initial wheel speeds, or nullptr: free rolling, speed / wheel radius
  float* last_accel;                   // [N][M] or nullptr
  double* pid_state;                   // [N][M][6] or nullptr: the PID controllers' integral / previous error / derivative
  int n_pool;
  // t2d_set_agents: the slots K10 retired take their types back, and the per-row NoAction state starts fresh
  uint8_t* agent_type_id;              // writable alias of type_id, or nullptr: no agents bound
  uint8_t* agent_retired;              // [N][M], 255 = not retired
  GoalArgs agent;
  int agent_q;
};

__global__ void t2d_reset_kernel(const __grid_constant__ ResetArgs A) {
  const long long total = (long long)A.N * A.M;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / A.M), m = (int)(i - (long long)n * A.M);
    if (!A.mask[n]) continue;
    int r = A.pool_index ? A.pool_index[n] : n;
    r = min(max(r, 0), A.n_pool - 1);
    const long long s = (long long)r * A.M + m;
    A.x[i] = A.px[s]; A.y[i] = A.py[s]; A.h[i] = A.ph[s]; A.v[i] = A.pv[s];
    A.vx[i] = A.pvx ? A.pvx[s] : A.pv[s] * cosf(A.ph[s]);
    A.vy[i] = A.pvy ? A.pvy[s] : A.pv[s] * sinf(A.ph[s]);
    if (A.agent_type_id != nullptr) {
      const uint8_t rt = A.agent_retired[i];
      if (rt != 0xff) { A.agent_type_id[i] = rt; A.agent_retired[i] = 0xff; }
      for (int q = m; q < A.agent_q; q += A.M) {   // NoAction.reset of every row
        A.agent.last_pose[4 * ((long long)n * A.agent_q + q) + 3] = 0.0f;
        A.agent.noact_count[(long long)n * A.agent_q + q] = 0;
      }
    }
    if (A.wheel_f != nullptr) {
      float wf = 0.0f, wr = 0.0f;
      if (A.pool_wf != nullptr) {
        wf = A.pool_wf[s]; wr = A.pool_wr[s];
      } else {
        const int tid = A.type_id[i];
        if (tid < A.n_types && A.table[tid].model() == MODEL_DRIFT) wf = wr = A.pv[s] / A.table[tid].wheel_radius;   // zero slip
      }
      A.wheel_f[i] = wf; A.wheel_r[i] = wr;
    }
    if (A.last_accel != nullptr) A.last_accel[i] = 0.0f;   // a fresh State has no acceleration (state.py:171-185)
    if (A.pid_state != nullptr)                            // PIDController.reset, pid_controller.py:408-418
      for (int k = 0; k < 6; ++k) A.pid_state[6 * i + k] = 0.0;
    if (m == 0) {
      A.step_count[n] = 0;
      if (A.goal.last_pose) A.goal.last_pose[4 * (long long)n + 3] = 0.0f;   // NoAction.reset / last_pose = None
      if (A.goal.noact_count) A.goal.noact_count[n] = 0;
    }
  }
}

// ---------------------------------------------------------------------------- K13 / K14: sampled resets
// DESIGN.md section 1 "Sampled resets" (envs/parking.py:397-441, map/generator/generate_parking_lot.py:231-237).
// K13 draws the pool row of every masked scenario and copies the columns that belong to the row; K2 (and K7) then run
// with pool_index = pool_row; K14 moves the start states by seeded jitter, checked by the tick's own predicates.
struct DrawArgs {
  const uint8_t* mask;
  const uint32_t* episode;             // [N]
  int32_t* pool_row;                   // [N]
  uint64_t seed;
  int sample_rows, N, M, P;
  const uint8_t* pool_type;  uint8_t* type_id;  uint8_t* retired;   // [P][M] -> [N][M]; retired: [N][M] or nullptr
  const float* pool_target;  float* target;                         // [P][5] -> [N][5]
  const uint16_t* pool_tile; uint16_t* tile_id;                     // [P] -> [N]
  const int16_t* pool_route; int16_t* route_id;                     // [P][M] -> [N][M]
};

__global__ void __launch_bounds__(256) t2d_episode_draw_kernel(const __grid_constant__ DrawArgs A) {
  const long long total = (long long)A.N * A.M;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / A.M), m = (int)(i - (long long)n * A.M);
    if (!A.mask[n]) continue;
    const int r = A.sample_rows ? draw_row(episode_draw(A.seed, 0u, (uint32_t)n, A.episode[n]).x, A.P) : min(n, A.P - 1);
    const long long s = (long long)r * A.M + m;
    if (A.pool_type) {
      A.type_id[i] = A.pool_type[s];
      if (A.retired) A.retired[i] = 0xff;   // K2 would restore a retired type of the old episode over the new one
    }
    if (A.pool_route) A.route_id[i] = A.pool_route[s];
    if (m == 0) {
      A.pool_row[n] = r;
      if (A.pool_tile) A.tile_id[n] = A.pool_tile[r];
      if (A.pool_target)
        for (int k = 0; k < 5; ++k) A.target[5 * (long long)n + k] = A.pool_target[5 * (long long)r + k];
    }
  }
}

struct PlaceArgs : WorldArgs {
  const uint8_t* mask;
  uint32_t* episode;                   // [N]
  int8_t* reset_try;                   // [N][M]
  uint64_t seed;
  const float* jitter;                 // [M][8] (lo, hi) of dx, dy, dheading, dspeed, or nullptr: no slot is jittered
  int tries, avoid_target;
  const float* target;                 // [N][5] the t2d_set_goal target (avoid_target), or nullptr
  MapArgs map;
  MapHeader mh;                        // the single tile's header (its bounds also when no tile has segments)
  int has_bounds;
  float *wheel_f, *wheel_r;            // [N][M] or nullptr
  int pool_wheels;                     // t2d_bind_reset_wheel_pool is bound: K2's wheel speeds stay
};

// The tick's pose of a slot at (x, y, heading) with its type's shape (K1's pose tile: sincos_fast, pose_l, pose_w)
__device__ __forceinline__ Pose slot_pose(const Params& p, float x, float y, float h) {
  Pose a;
  a.x = x; a.y = y; a.h = h; a.l = p.pose_l; a.w = p.pose_w;
  sincos_fast(h, &a.s, &a.c);
  return a;
}

// Would check_events flag slot m of scenario n at pose a?  The same filtered predicates as K1: out of its tile's box,
// a collidable segment or Area of its tile, any other active slot at its current state; with avoid, the target box too.
__device__ __forceinline__ bool place_blocked(const PlaceArgs& A, long long n, int m, const Pose a, float rb, bool avoid,
                                              const float4* sa, const float4* sb) {
  const unsigned char* blob = tile_blob(A.map, n);
  const MapHeader* mh = (A.map.tile_id && blob) ? reinterpret_cast<const MapHeader*>(blob) : &A.mh;
  const bool bounded = A.map.tile_id && blob ? mh->has_bounds != 0 : A.has_bounds != 0;
  if (bounded) {
    int r = out_of_bound_f32(a.x, a.y, a.c, a.s, a.l, a.w, a.w < 0.0f, mh->bxmin, mh->bxmax, mh->bymin, mh->bymax);
    if (r < 0) r = out_of_bound_f64(a.x, a.y, a.h, a.l, a.w, a.w < 0.0f, mh->bxmin, mh->bxmax, mh->bymin, mh->bymax) ? 1 : 0;
    if (r) return true;
  }
  if (blob && mh->n_seg > 0) {
    // (the blob and its header as global addresses: the out-of-line walks K1 shares keep their global loads)
    const unsigned char* g = reinterpret_cast<const unsigned char*>(__cvta_global_to_generic(__cvta_generic_to_global(blob)));
    const MapHeader& gh = *reinterpret_cast<const MapHeader*>(g);   // (tile 0's header starts the blob)
    const MapView mv = map_view(g, gh);
    int best = static_walk_exact(a, rb, gh, mv.seg, mv.cell_start, mv.items);
    if (gh.n_poly > 0) best = static_objects(best, a.x, a.y, gh, g);
    if (best != 0x7fffffff) return true;
  }
  for (int j = 0; j < A.M; ++j) {   // the scenario's slots as K14 staged them (rb < 0: inactive, retired or no shape)
    const float4 pa = sa[j];
    if (j == m || !(pa.z >= 0.0f)) continue;
    const float dx = pa.x - a.x, dy = pa.y - a.y, rr = rb + pa.z;
    if (dx * dx + dy * dy > fmaf(rr * rr, 1.00001f, 1e-12f)) continue;   // bounding circles apart (conservative, as K1)
    const float4 pb = sb[j];
    Pose b;
    b.x = pa.x; b.y = pa.y; b.h = pa.w; b.c = pb.x; b.s = pb.y; b.l = pb.z; b.w = pb.w;
    if (pair_hit(a, b)) return true;
  }
  if (avoid) {
    const float* tg = A.target + 5 * n;
    Pose t;
    t.x = tg[0]; t.y = tg[1]; t.h = tg[2]; t.l = tg[3]; t.w = tg[4];
    sincos_fast(t.h, &t.s, &t.c);
    if (pair_hit(a, t)) return true;
  }
  return false;
}

// One warp per scenario: slots in order 0 .. M-1, lane t tries draw 1 + 32 m + t, the lowest accepted lane wins.  The
// scenario's poses are staged in the warp's shared memory (K1's pose tile layout, slot-major), so the partner loop of
// every try reads them there; the winner of a slot writes its new pose to both copies.
constexpr int K14_WARPS = 4;
__device__ __forceinline__ void stage_pose(const PlaceArgs& A, long long i, int tid, float x, float y, float h, float4* sa,
                                           float4* sb, int j) {
  const bool solid = tid < A.n_types && A.table[tid].shape() != SHAPE_NONE;
  const Params& p = A.table[solid ? tid : 0];
  float sn, cs;
  sincos_fast(h, &sn, &cs);
  sa[j] = make_float4(x, y, solid ? p.rbound : -1.0f, h);
  sb[j] = make_float4(cs, sn, p.pose_l, p.pose_w);
}

__global__ void __launch_bounds__(K14_WARPS * 32) t2d_episode_place_kernel(const __grid_constant__ PlaceArgs A) {
  __shared__ float4 s_pose[K14_WARPS][2][T2D_MAX_PARTICIPANTS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long n = (long long)blockIdx.x * K14_WARPS + warp;
  if (n >= A.N || !A.mask[n]) return;
  float4* sa = s_pose[warp][0];
  float4* sb = s_pose[warp][1];
  const uint32_t e = A.episode[n];
  const long long base = n * A.M;
  if (A.jitter != nullptr)
    for (int j = lane; j < A.M; j += 32) stage_pose(A, base + j, A.type_id[base + j], A.x[base + j], A.y[base + j], A.h[base + j], sa, sb, j);
  __syncwarp();
  for (int m = 0; m < A.M; ++m) {
    const long long i = base + m;
    const int tid = A.type_id[i];
    bool jittered = A.jitter != nullptr && tid < A.n_types;
    if (jittered) {
      bool any = false;
      for (int k = 0; k < 8; ++k) any = any || A.jitter[8 * m + k] != 0.0f;
      jittered = any;
    }
    if (!jittered) {
      if (lane == 0) A.reset_try[i] = -1;
      continue;
    }
    const Params& p = A.table[tid];
    bool ok = false;
    Cand cd{};
    if (lane < A.tries) {
      cd = jitter_candidate(episode_draw(A.seed, 1u + 32u * (uint32_t)m + (uint32_t)lane, (uint32_t)n, e), A.jitter + 8 * m,
                            A.x[i], A.y[i], A.h[i], A.v[i]);
      ok = p.shape() == SHAPE_NONE ||
           !place_blocked(A, n, m, slot_pose(p, cd.x, cd.y, cd.h), p.rbound, A.avoid_target && m == 0 && A.target != nullptr,
                          sa, sb);
    }
    const unsigned acc = __ballot_sync(0xffffffffu, ok);
    const int win = acc ? __ffs(acc) - 1 : -1;
    if (lane == (win < 0 ? 0 : win)) {
      if (win >= 0) {
        A.x[i] = cd.x; A.y[i] = cd.y; A.h[i] = cd.h; A.v[i] = cd.v;
        A.vx[i] = cd.v * cosf(cd.h); A.vy[i] = cd.v * sinf(cd.h);   // as K2 for a pool without velocities
        // free rolling, as K2 sets it without a wheel pool; with one, the slot keeps the pool's wheel speeds
        if (A.wheel_f != nullptr && !A.pool_wheels && p.model() == MODEL_DRIFT) A.wheel_f[i] = A.wheel_r[i] = cd.v / p.wheel_radius;
        stage_pose(A, i, tid, cd.x, cd.y, cd.h, sa, sb, m);
      }
      A.reset_try[i] = (int8_t)win;
    }
    __syncwarp();   // the next slot's tries read this one's placed pose
  }
  if (lane == 0) A.episode[n] = e + 1u;
}

// ---------------------------------------------------------------------------- route following
// DESIGN.md section 1 "Route following": the polyline table (t2d_set_paths) read by K5's PATH sources, the OffRoute
// detector and route progress of the epilogues, and K12.
struct PathVertex { double x, y, cum, len; };   // vertex, arc length up to it, length of the segment that starts here

// The closest point c of a polyline to (x, y): the first strict minimum of |p - c|^2 over the segments of non-zero
// length, c the clamped projection, and that segment's unit tangent u.  ARC adds d2 = |p - c|^2, the arc length s of c
// (the lengths of the earlier segments of non-zero length summed in list order, plus t len) and the total length L.
// fp64, one rounding per operation, in this order (tests/pid_oracle.py, tests/route_oracle.py).  false: no segment.
struct PathPoint { double cx, cy, ux, uy, d2, s, L; };

template <bool ARC>
__device__ __forceinline__ bool closest_on_path(const PathVertex* pv, int n_vert, double x, double y, PathPoint& c) {
  double best = 0.0, acc = 0.0;
  bool found = false;
  for (int i = 0; i + 1 < n_vert; ++i) {
    const double ax = pv[i].x, ay = pv[i].y;
    const double dx = __dsub_rn(pv[i + 1].x, ax), dy = __dsub_rn(pv[i + 1].y, ay);
    const double l2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
    if (!(l2 > 0.0)) continue;
    double t = __ddiv_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, ax), dx), __dmul_rn(__dsub_rn(y, ay), dy)), l2);
    t = fmin(fmax(t, 0.0), 1.0);
    const double qx = __dadd_rn(ax, __dmul_rn(t, dx)), qy = __dadd_rn(ay, __dmul_rn(t, dy));
    const double ex = __dsub_rn(x, qx), ey = __dsub_rn(y, qy);
    const double d2 = __dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey));
    if constexpr (ARC) {
      const double len = __dsqrt_rn(l2);
      if (!found || d2 < best) {
        best = d2; c.cx = qx; c.cy = qy; c.ux = __ddiv_rn(dx, len); c.uy = __ddiv_rn(dy, len);
        c.s = __dadd_rn(acc, __dmul_rn(t, len));
        found = true;
      }
      acc = __dadd_rn(acc, len);
    } else {
      if (!found || d2 < best) {
        const double len = __dsqrt_rn(l2);
        best = d2; c.cx = qx; c.cy = qy; c.ux = __ddiv_rn(dx, len); c.uy = __ddiv_rn(dy, len);
        found = true;
      }
    }
  }
  if constexpr (ARC) { c.d2 = best; c.L = acc; }
  return found;
}

// The bound routes (t2d_set_routes): route_id == nullptr when none are bound
struct RouteArgs {
  const int16_t* route_id;          // [N][M] path of every slot, -1 (or any id the table does not hold): none
  const PathVertex* path_v;
  const int* path_off;
  int n_paths;
  float off_reward;                 // the reward of an off-route step
  double threshold, weight;         // OffRoute threshold (m), progress weight (per m)
};

// The polyline of slot i's route, or nullptr
__device__ __forceinline__ const PathVertex* route_of(const RouteArgs& R, long long i, int& n_vert) {
  const int rid = R.route_id[i];
  if (rid < 0 || rid >= R.n_paths) return nullptr;
  n_vert = R.path_off[rid + 1] - R.path_off[rid];
  return R.path_v + R.path_off[rid];
}

enum : int { ROUTE_NONE = 0, ROUTE_ON = 1, ROUTE_OFF = 2 };
struct RouteHit { double s; int state; };

// OffRoute.update (off_route.py:24-35) for slot i at its fp32 centre: off when the distance to the route's closest point
// exceeds the threshold; s is that point's arc length.  Out of line: both epilogues run this one compiled copy.
__device__ __noinline__ RouteHit route_probe(const RouteArgs& R, long long i, float x, float y) {
  int n_vert = 0;
  const PathVertex* pv = route_of(R, i, n_vert);
  PathPoint c;
  if (pv == nullptr || !closest_on_path<true>(pv, n_vert, (double)x, (double)y, c)) return {0.0, ROUTE_NONE};
  return {c.s, __dsqrt_rn(c.d2) > R.threshold ? ROUTE_OFF : ROUTE_ON};
}

// ---------------------------------------------------------------------------- env epilogue
// What ParkingEnv.step does after check_status (envs/parking.py:240-256, _get_reward :148-190), for all N scenarios in
// one launch: TrafficStatus per participant from the event byte (status.py:52-61), terminated / truncated
// (parking.py:243-248), the reward chain in the reference's order, the two running extrema it keeps per episode
// (_max_iou, _min_dist_to_target) and the done mask that drives the masked reset.  One thread per participant slot;
// the thread of slot 0 also does the per-scenario part.  Reads the ego's flags through the same array, so the launch
// has no other input than the tick's outputs.
struct EnvArgs : WorldArgs {   // (the state after the tick: the ego's position for the distance shaping)
  const uint8_t* flags;        // [N][M] event byte of the tick
  const uint8_t* status;       // [N] ScenarioStatus of the tick
  const float* iou;            // [N] IoU(ego pose, target) of the tick, or nullptr (no goal)
  const float* target;         // [N][5] or nullptr
  float* max_iou;              // [N] in/out, or nullptr
  float* min_dist;             // [N] in/out, or nullptr
  float* reward;               // [N]
  uint8_t *terminated, *truncated, *done;   // [N]
  uint8_t* traffic_status;     // [N][M]
  RouteArgs route;
  double* s_best;              // [N] best arc length of the episode, or nullptr: no progress term
  int max_step, reset_trackers;
};

// The reward chain of _get_reward (parking.py:148-190) for one scored participant: st its ScenarioStatus, ts its
// TrafficStatus as check_status leaves it (only the collision and OffRoute detectors set it), step_count its scenario's
// tick count.  max_iou == nullptr skips the IoU term, min_dist == nullptr the progress term (target = the goal centre,
// (x, y) the participant's position), s_best == nullptr the route progress term (s the arc length on the route, weight
// its factor; an extension).  Out of line: the env epilogue and K10 run this one compiled copy, so that their rewards
// agree bit for bit whatever the compiler would contract in an inlined copy.
__device__ __noinline__ float reward_chain(int st, int ts, int step_count, int max_step, float iou, float* max_iou,
                                           const float* target, float* min_dist, float x, float y, float off_reward,
                                           double weight, double s, double* s_best) {
  float r;
  if (ts == 3 || ts == 4) r = -5.0f;                                             // :151-152 (+ dynamic collision, an extension)
  else if (ts == T2D_TRAFFIC_OFF_ROUTE) r = off_reward;                          // (an extension)
  else if (st == T2D_STATUS_TIME_EXCEEDED || st == T2D_STATUS_NO_ACTION) r = -1.0f;   // :153-157
  else if (st == T2D_STATUS_OUT_BOUND) r = -5.0f;                                // :158-159
  else if (st == T2D_STATUS_COMPLETED) r = 5.0f;                                 // :160-161
  else {
    r = max_step > 0 ? -tanhf((float)step_count / (float)max_step) * 0.001f : 0.0f;   // :163
    if (max_iou != nullptr) {
      const float best = *max_iou;
      r += (best == -INFINITY) ? iou : iou - best;                                 // :164-169
      *max_iou = fmaxf(best, iou);                                                 // :170
    }
    if (min_dist != nullptr) {
      const float dx = x - target[0], dy = y - target[1];
      const float d = sqrtf(dx * dx + dy * dy), best = *min_dist;                  // :172-185
      if (d < best) {                                                              // :186-188 (inf on the first step: the
        if (best != INFINITY) r += (best - d) * 0.1f;                              //  reference adds inf there; we add nothing)
        *min_dist = d;
      }
    }
    if (s_best != nullptr) {                                                       // route progress: weight (s - s_best)
      const double best = *s_best;                                                 // in fp64, one rounding to fp32; the
      if (s > best) {                                                              // first step only records s
        if (best != -INFINITY) r += __double2float_rn(__dmul_rn(weight, __dsub_rn(s, best)));
        *s_best = s;
      }
    }
  }
  return r;
}

__global__ void __launch_bounds__(256) t2d_env_epilogue_kernel(const __grid_constant__ EnvArgs A) {
  const long long total = (long long)A.N * A.M;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const unsigned f = A.flags[i];
    const uint8_t ts = (f & T2D_F_STATIC) ? 3 : ((f & T2D_F_DYNAMIC) ? 4 : 1);   // COLLISION_STATIC / COLLISION_DYNAMIC / NORMAL
    if (A.traffic_status) A.traffic_status[i] = ts;
    const int n = (int)(i / A.M);
    if (i - (long long)n * A.M != 0) continue;
    const int st = A.status[n];
    // check_status returns at the first detector that fires (parking.py:366-385): the ego's traffic status is only set
    // by the collision detector, i.e. when the scenario status says FAILED, and by OffRoute, which ranks below collision
    // and above completion
    int ego_ts = st == T2D_STATUS_FAILED ? ts : 1;
    RouteHit rh{0.0, ROUTE_NONE};
    if (A.route.route_id != nullptr && (st == T2D_STATUS_NORMAL || st == T2D_STATUS_COMPLETED)) {
      rh = route_probe(A.route, i, A.x[i], A.y[i]);
      if (rh.state == ROUTE_OFF) {
        ego_ts = T2D_TRAFFIC_OFF_ROUTE;
        if (A.traffic_status) A.traffic_status[i] = T2D_TRAFFIC_OFF_ROUTE;
      }
    }
    const bool term = st == T2D_STATUS_COMPLETED && ego_ts == 1;                   // :243-244
    const bool trunc = !term && (st != T2D_STATUS_NORMAL || ego_ts != 1);          // :245-248
    const bool scored_iou = A.iou != nullptr && A.max_iou != nullptr;
    const float r = reward_chain(st, ego_ts, A.step_count[n], A.max_step, scored_iou ? A.iou[n] : 0.0f,
                                 scored_iou ? A.max_iou + n : nullptr, A.target ? A.target + 5 * (long long)n : nullptr,
                                 (A.target && A.min_dist) ? A.min_dist + n : nullptr, A.x[i], A.y[i], A.route.off_reward,
                                 A.route.weight, rh.s, (rh.state == ROUTE_ON && A.s_best) ? A.s_best + n : nullptr);
    A.reward[n] = r;
    if (A.terminated) A.terminated[n] = term;
    if (A.truncated) A.truncated[n] = trunc;
    if (A.done) A.done[n] = term || trunc;
    if (A.reset_trackers && (term || trunc)) {   // the next episode starts fresh (ParkingEnv.reset, parking.py:276-277)
      if (A.max_iou) A.max_iou[n] = -INFINITY;
      if (A.min_dist) A.min_dist[n] = INFINITY;
      if (A.s_best) A.s_best[n] = -INFINITY;
    }
  }
}

// ---------------------------------------------------------------------------- K10 per-agent epilogue
// DESIGN.md section 1 "Per-agent status and reward": the status chain, terminated / truncated and the reward chain of the
// env epilogue for every row (n, q) of an observer list, retirement of the slots whose rows settle, and the done mask
// "no row of the scenario is NORMAL".  One warp per scenario; lane l takes rows l, l + 32, l + 64, l + 96.
// The state is the tick's result; a settled row's slot becomes 255 in type_id, the caller's writable array ...
struct AgentArgs : WorldArgs {
  GoalArgs goal;                // the rows' detectors, indexed by the row n·Q + q (target [N][Q][5] or nullptr)
  const uint8_t* flags;         // [N][M] event byte of the tick
  const int16_t* observers;     // [N][Q] or nullptr: row q is slot q
  uint8_t* retired;             // [N][M]: ... and keeps its type here (255: not retired)
  float *max_iou, *min_dist;    // [N][Q] per-episode extrema
  float* reward;                // [N][Q]
  uint8_t *terminated, *truncated, *status;   // [N][Q]
  uint8_t* done;                // [N]
  uint8_t* traffic_status;      // [N][M] or nullptr
  RouteArgs route;
  double* s_best;               // [N][Q] best arc length of the episode, or nullptr: no progress term
  int Q, max_step, reset_trackers;
};

constexpr int K10_WARPS = 8;
constexpr int K10_ROWS_PER_LANE = T2D_OBS_MAX_OBSERVERS / 32;   // Q <= 128

__global__ void __launch_bounds__(K10_WARPS * 32) t2d_agents_epilogue_kernel(const __grid_constant__ AgentArgs A) {
  const int lane = threadIdx.x & 31;
  const long long n = (long long)blockIdx.x * K10_WARPS + (threadIdx.x >> 5);
  if (n >= A.N) return;   // whole warps
  const long long s0 = n * A.M, r0 = n * A.Q;
  if (A.traffic_status) {
    for (int m = lane; m < A.M; m += 32) {
      const unsigned f = A.flags[s0 + m];
      A.traffic_status[s0 + m] = (f & T2D_F_STATIC) ? 3 : ((f & T2D_F_DYNAMIC) ? 4 : 1);
    }
    if (A.route.route_id != nullptr) __syncwarp();   // before an off-route row overwrites its slot's code
  }
  const int cnt = A.step_count[n];
  const bool time_up = A.max_step > 0 && cnt > A.max_step;                     // parking.py:366-369
  bool any_normal = false;
  unsigned settle = 0;                                                          // bit k: row lane + 32 k retires its slot
#pragma unroll 1
  for (int k = 0; k < K10_ROWS_PER_LANE; ++k) {
    const int q = lane + 32 * k;
    if (q >= A.Q) break;
    const long long r = r0 + q;
    const int j = A.observers ? A.observers[r] : q;
    const int t = (j >= 0 && j < A.M) ? A.type_id[s0 + j] : 0xff;
    if (t >= A.n_types) {   // absent row
      A.status[r] = 0; A.reward[r] = 0.0f; A.terminated[r] = 0; A.truncated[r] = 0; A.goal.iou[r] = 0.0f;
      continue;
    }
    const long long i = s0 + j;
    const float x = A.x[i], y = A.y[i];
    const float* goal = A.goal.target ? A.goal.target + 5 * r : nullptr;
    const bool has_goal = goal != nullptr && goal[0] == goal[0];
    unsigned ev = 0;
    float iou = 0.0f;
    const Vec4 g2 = params_group(A.table + t, 2);   // (pose_l, pose_w, rbound, model | shape << 8)
    // K1's condition for the ego: a solid box (pose tile: x not NaN, pose_w >= 0)
    if (has_goal && x == x && (__float_as_int(g2.w) >> 8) != SHAPE_NONE && g2.y >= 0.0f) {
      ev = ego_goal_events(A, r, x, y, A.h[i], g2.x, g2.y);   // writes goal.iou[r]
      iou = A.goal.iou[r];
    } else {
      A.goal.iou[r] = 0.0f;
    }
    const unsigned f = A.flags[i];
    int st = T2D_STATUS_NORMAL;                                                 // parking.py:366-390, lowest priority first
    if (ev & 1u) st = T2D_STATUS_COMPLETED;
    if (f & T2D_F_DYNAMIC) st = T2D_STATUS_FAILED;
    if (f & T2D_F_STATIC) st = T2D_STATUS_FAILED;
    if (f & T2D_F_OUTBOUND) st = T2D_STATUS_OUT_BOUND;
    if (ev & 2u) st = T2D_STATUS_NO_ACTION;
    if (time_up) st = T2D_STATUS_TIME_EXCEEDED;
    RouteHit rh{0.0, ROUTE_NONE};
    if (A.route.route_id != nullptr && (st == T2D_STATUS_NORMAL || st == T2D_STATUS_COMPLETED)) {   // OffRoute: below
      rh = route_probe(A.route, i, x, y);                                                            // collision, above
      if (rh.state == ROUTE_OFF) {                                                                   // completion
        st = T2D_STATUS_FAILED;
        if (A.traffic_status) A.traffic_status[i] = T2D_TRAFFIC_OFF_ROUTE;
      }
    }
    const int ts = st == T2D_STATUS_FAILED ? ((f & T2D_F_STATIC) ? 3 : ((f & T2D_F_DYNAMIC) ? 4 : T2D_TRAFFIC_OFF_ROUTE)) : 1;
    const bool term = st == T2D_STATUS_COMPLETED;
    const bool trunc = !term && st != T2D_STATUS_NORMAL;
    A.reward[r] = reward_chain(st, ts, cnt, A.max_step, iou, has_goal ? A.max_iou + r : nullptr, goal,
                               has_goal ? A.min_dist + r : nullptr, x, y, A.route.off_reward, A.route.weight, rh.s,
                               (rh.state == ROUTE_ON && A.s_best) ? A.s_best + r : nullptr);
    A.status[r] = (uint8_t)st; A.terminated[r] = term; A.truncated[r] = trunc;
    any_normal = any_normal || st == T2D_STATUS_NORMAL;
    if (st != T2D_STATUS_NORMAL) {   // retire the slot (duplicate rows store the same type)
      settle |= 1u << k;
      A.retired[i] = (uint8_t)t;
    }
  }
  // every row has read its slot's type before any slot leaves type_id
  const bool done = !__any_sync(0xffffffffu, any_normal);
  if (lane == 0) A.done[n] = done;
  __syncwarp();
#pragma unroll 1
  for (int k = 0; k < K10_ROWS_PER_LANE; ++k) {
    const int q = lane + 32 * k;
    if (q >= A.Q) break;
    if (A.reset_trackers && done) {
      A.max_iou[r0 + q] = -INFINITY; A.min_dist[r0 + q] = INFINITY;
      if (A.s_best) A.s_best[r0 + q] = -INFINITY;
    }
    if ((settle >> k) & 1u) const_cast<uint8_t*>(A.type_id)[s0 + (A.observers ? A.observers[r0 + q] : q)] = 0xff;
  }
}

// ---------------------------------------------------------------------------- K11 per-agent action
// DESIGN.md section 1 "Per-agent action": slot m of scenario n takes row q* of agent_action, the lowest q with
// observers[n][q] == m, when its type is active; nothing else is written.  One warp per scenario; lane l takes rows l,
// l + 32, l + 64, l + 96 and claims their slots with atomicMin on a per-slot owner in shared memory, so the first row
// wins whatever the order of the atomics.  Then one float2 copy per owned active slot (the fp32 bits as they are).
struct ActionArgs : WorldArgs {
  const int16_t* observers;     // [N][Q] or nullptr: row q is slot q
  const float* agent_action;    // [N][Q][2]
  float* action;                // [N][M][2]
  int Q;
};

constexpr int K11_WARPS = 8;

__global__ void __launch_bounds__(K11_WARPS * 32) t2d_agent_action_kernel(const __grid_constant__ ActionArgs A) {
  __shared__ int s_owner[K11_WARPS][T2D_MAX_PARTICIPANTS];
  const int lane = threadIdx.x & 31;
  const long long n = (long long)blockIdx.x * K11_WARPS + (threadIdx.x >> 5);
  if (n >= A.N) return;   // whole warps
  const long long s0 = n * A.M, r0 = n * A.Q;
  constexpr int K = T2D_MAX_PARTICIPANTS / 32;   // = T2D_OBS_MAX_OBSERVERS / 32: rows and slots per lane
  // every independent load first: the observer and type loads of a lane are in flight together
  int slot[K];
  unsigned type[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const int q = lane + 32 * k, m = q;
    slot[k] = q < A.Q ? (A.observers ? (int)A.observers[r0 + q] : q) : -1;
    type[k] = m < A.M ? A.type_id[s0 + m] : 0xffu;
  }
  int* owner = s_owner[threadIdx.x >> 5];
#pragma unroll
  for (int k = 0; k < K; ++k)
    if (lane + 32 * k < A.M) owner[lane + 32 * k] = A.Q;   // Q: no row names the slot
  __syncwarp();
#pragma unroll
  for (int k = 0; k < K; ++k)
    if (slot[k] >= 0 && slot[k] < A.M) atomicMin(&owner[slot[k]], lane + 32 * k);
  __syncwarp();
  const float2* src = reinterpret_cast<const float2*>(A.agent_action) + r0;
  float2* dst = reinterpret_cast<float2*>(A.action) + s0;
  float2 val[K];
  bool put[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {   // all loads, then all stores (the two arrays may alias as far as the compiler knows)
    const int m = lane + 32 * k;
    const int q = m < A.M ? owner[m] : A.Q;
    put[k] = q < A.Q && type[k] < (unsigned)A.n_types;
    if (put[k]) val[k] = src[q];
  }
#pragma unroll
  for (int k = 0; k < K; ++k)
    if (put[k]) dst[lane + 32 * k] = val[k];
}

// ---------------------------------------------------------------------------- K12 route observation
// DESIGN.md section 1 "Route following": row (n, q) describes the route of slot j = observers[n][q] (slot q without a
// list) in the frame of that slot (origin its centre, +x along its heading): has_route, the signed lateral offset
// (PATH_CROSS_TRACK's convention), the heading error to the closest segment's tangent in (-pi, pi], s / L, L - s, then P
// look-ahead points (x, y) at arc length min(s + k spacing, L), k = 1..P.  Absent rows (observer outside [0, M), empty or
// retired slot, no route) are zeros.  One warp per scenario; lane l takes rows l, l + 32, l + 64, l + 96.
struct RouteObsArgs : WorldArgs {
  RouteArgs route;              // route_id may be nullptr: every row is absent
  const int16_t* observers;     // [N][Q] or nullptr: row q is slot q
  float* out;                   // [N][Q][T2D_ROUTE_OBS_FIELDS + 2 P]
  int Q, P;
  double spacing;
};

constexpr int K12_WARPS = 8;

__global__ void __launch_bounds__(K12_WARPS * 32) t2d_route_obs_kernel(const __grid_constant__ RouteObsArgs A) {
  const int lane = threadIdx.x & 31;
  const long long n = (long long)blockIdx.x * K12_WARPS + (threadIdx.x >> 5);
  if (n >= A.N) return;   // whole warps
  const int F = T2D_ROUTE_OBS_FIELDS + 2 * A.P;
#pragma unroll 1
  for (int q = lane; q < A.Q; q += 32) {
    const long long r = n * A.Q + q;
    float* o = A.out + r * F;
    const int j = A.observers ? A.observers[r] : q;
    const long long i = n * A.M + j;
    int nv = 0;
    const PathVertex* pv = nullptr;
    PathPoint c;
    if (A.route.route_id != nullptr && j >= 0 && j < A.M && A.type_id[i] < A.n_types) pv = route_of(A.route, i, nv);
    if (pv == nullptr || !closest_on_path<true>(pv, nv, (double)A.x[i], (double)A.y[i], c)) {
      for (int k = 0; k < F; ++k) o[k] = 0.0f;
      continue;
    }
    const double x = A.x[i], y = A.y[i], h = A.h[i];
    double sn, cs;
    sincos(h, &sn, &cs);
    const double d_h = __dsub_rn(atan2(c.uy, c.ux), h);
    double err = atan2(sin(d_h), cos(d_h));
    constexpr double PI_D = 3.141592653589793;
    if (err == -PI_D) err = PI_D;   // (-pi, pi]
    o[0] = 1.0f;
    o[1] = (float)__dsub_rn(__dmul_rn(c.ux, __dsub_rn(c.cy, y)), __dmul_rn(c.uy, __dsub_rn(c.cx, x)));
    o[2] = (float)err;
    o[3] = (float)__ddiv_rn(c.s, c.L);
    o[4] = (float)__dsub_rn(c.L, c.s);
    int seg = 0;
    double acc = 0.0;   // arc length at the start of segment seg
    for (int k = 1; k <= A.P; ++k) {
      const double sig = fmin(__dadd_rn(c.s, __dmul_rn((double)k, A.spacing)), c.L);
      double px = pv[nv - 1].x, py = pv[nv - 1].y;
      for (; seg + 1 < nv; ++seg) {   // the first segment of non-zero length that ends at or beyond sig
        const double ax = pv[seg].x, ay = pv[seg].y;
        const double dx = __dsub_rn(pv[seg + 1].x, ax), dy = __dsub_rn(pv[seg + 1].y, ay);
        const double l2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
        if (!(l2 > 0.0)) continue;
        const double len = __dsqrt_rn(l2), end = __dadd_rn(acc, len);
        if (sig <= end) {
          const double t = __ddiv_rn(__dsub_rn(sig, acc), len);
          px = __dadd_rn(ax, __dmul_rn(t, dx)); py = __dadd_rn(ay, __dmul_rn(t, dy));
          break;
        }
        acc = end;
      }
      const double ex = __dsub_rn(px, x), ey = __dsub_rn(py, y);
      o[T2D_ROUTE_OBS_FIELDS + 2 * (k - 1)] = (float)__dadd_rn(__dmul_rn(ex, cs), __dmul_rn(ey, sn));
      o[T2D_ROUTE_OBS_FIELDS + 2 * (k - 1) + 1] = (float)__dsub_rn(__dmul_rn(ey, cs), __dmul_rn(ex, sn));
    }
  }
}

// ---------------------------------------------------------------------------- K3
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

// ---------------------------------------------------------------------------- K7
// Log replay (t2d_set_log): every replayed slot takes its track's state at the time the next tick produces (or, in
// reset mode, at the row's t0), before K1, which then only builds the pose of these static-model slots.  One thread
// per (scenario, slot), consecutive threads on consecutive slots: the [N, M] slot offset reads and the state / type_id
// stores coalesce; the schedule entries, the track entry and its two frame records are gathers.  A slot's schedule is
// a run of entries with strictly increasing, disjoint presence intervals; the thread takes the first entry whose last
// stamp is >= t (the slot's final entry if none is), so a schedule of L entries costs ceil(log2 L) dependent probes.
// When no schedule of the log holds more than one entry (t2d_set_log's row_track, and any such schedule), the host
// uploads the slots' tracks as one [n_rows][M] array instead and the offsets and the entry gather drop out of the
// dependent chain.  Whether the chosen track is present at t is then decided exactly as for a single track.  Interpolation in fp64 with explicit round-to-nearest operations (no FMA
// contraction), in the order oracle/replay.py states.
struct ReplayTrack { int32_t first_ms, period_ms, n_frames, rec_off; };
struct ReplayEntry { int32_t last_ms, track; };   // one 8-byte load per probe

struct ReplayArgs {
  float *x, *y, *h, *v, *vx, *vy;
  uint8_t* type_id;
  const int32_t* step_count;       // [N]
  const int32_t* log_row;          // [N] the row each scenario runs (tick mode)
  const uint8_t* mask;             // reset mode: [N] the scenarios being reset; nullptr in tick mode
  const int32_t* pool_index;       // reset mode: the new row of each masked scenario, nullptr = row n
  int32_t* log_row_out;            // reset mode: log_row, written for the masked scenarios
  const ReplayTrack* tracks;       // [n_tracks]
  const uint8_t* track_type;       // [n_tracks]
  const float* rec;                // [sum n_frames][5] x, y, heading, vx, vy
  const int32_t* t0;               // [n_rows] ms
  const int32_t* slot_off;         // [n_rows * M + 1] schedule of (row, m): entries [slot_off[row M + m], slot_off[row M + m + 1])
  const ReplayEntry* entries;      // [E]
  const int32_t* slot_track1;      // when no schedule has more than one entry: [n_rows * M] its track, -1 for none
                                   // (slot_off / entries then unused); nullptr otherwise
  int32_t* track_out;              // [N][M] the track each slot shows, -1 for none; nullptr: not written
  int N, M, n_rows, offset, interval_ms;
};

__device__ __forceinline__ float replay_lerp(float a, float b, double w) {   // a + w (b - a)
  return __double2float_rn(__dadd_rn((double)a, __dmul_rn(w, __dsub_rn((double)b, (double)a))));
}

__global__ void __launch_bounds__(256) t2d_replay_kernel(const __grid_constant__ ReplayArgs A) {
  constexpr double PI_D = 3.141592653589793, TWO_PI_D = 6.283185307179586;
  const long long total = (long long)A.N * A.M;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / A.M), m = (int)(i - (long long)n * A.M);
    int row;
    if (A.mask != nullptr) {
      if (!A.mask[n]) continue;
      row = A.pool_index ? A.pool_index[n] : n;
      row = min(max(row, 0), A.n_rows - 1);   // as K2 clamps its pool row (n_pool == n_rows)
      if (m == 0) A.log_row_out[n] = row;
    } else {
      row = min(max(A.log_row[n], 0), A.n_rows - 1);
    }
    const long long s = (long long)row * A.M + m;
    int k;
    long long t;
    if (A.slot_track1 != nullptr) {   // at most one entry per slot: the track itself, no offsets
      k = __ldg(A.slot_track1 + s);
      if (k < 0) {
        if (A.track_out) A.track_out[i] = -1;
        continue;
      }
      t = (long long)A.t0[row] + ((long long)A.step_count[n] + A.offset) * A.interval_ms;
    } else {
      int lo = __ldg(A.slot_off + s), hi = __ldg(A.slot_off + s + 1) - 1;
      if (hi < lo) {   // an empty schedule: the slot is not replayed
        if (A.track_out) A.track_out[i] = -1;
        continue;
      }
      t = (long long)A.t0[row] + ((long long)A.step_count[n] + A.offset) * A.interval_ms;
      while (lo < hi) {   // the first entry with last_ms >= t; the final one stands for "after every entry"
        const int mid = (lo + hi) >> 1;
        if ((long long)__ldg(&A.entries[mid].last_ms) >= t) hi = mid;
        else lo = mid + 1;
      }
      k = __ldg(&A.entries[lo].track);
    }
    const int4 tr4 = __ldg(reinterpret_cast<const int4*>(A.tracks) + k);
    const int first = tr4.x, period = tr4.y, n_frames = tr4.z, rec_off = tr4.w;
    const long long d = t - first;
    if (d < 0 || d > (long long)(n_frames - 1) * period) {   // the track is not in the scene at t
      A.type_id[i] = T2D_TYPE_INACTIVE;
      if (A.track_out) A.track_out[i] = -1;
      continue;
    }
    if (A.track_out) A.track_out[i] = k;
    const long long j = d / period;
    const int r = (int)(d - j * period);
    const float* a = A.rec + 5 * ((long long)rec_off + j);
    float x, y, h, vx, vy;
    if (r == 0) {   // on a frame: the record, bit for bit
      x = a[0]; y = a[1]; h = a[2]; vx = a[3]; vy = a[4];
    } else {        // between frames j and j + 1 (an extension: the reference has no state there)
      const float* b = a + 5;
      const double w = __ddiv_rn((double)r, (double)period);
      x = replay_lerp(a[0], b[0], w);
      y = replay_lerp(a[1], b[1], w);
      vx = replay_lerp(a[3], b[3], w);
      vy = replay_lerp(a[4], b[4], w);
      const double ha = (double)a[2];
      double dh = __dsub_rn((double)b[2], ha);   // the shorter arc: fold once into [-pi, pi]
      if (dh > PI_D) dh = __dsub_rn(dh, TWO_PI_D);
      else if (dh < -PI_D) dh = __dadd_rn(dh, TWO_PI_D);
      double hh = __dadd_rn(ha, __dmul_rn(w, dh));
      if (hh < 0.0) hh = __dadd_rn(hh, TWO_PI_D);   // wrap once into [0, 2 pi)
      else if (hh >= TWO_PI_D) hh = __dsub_rn(hh, TWO_PI_D);
      h = __double2float_rn(hh);
      if (h == (float)TWO_PI_D) h = 0.0f;   // just below 2 pi, rounded up to fp32(2 pi): the same direction as 0
    }
    // State.speed (state.py:143-146) from the fp32 velocity
    const float v = __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn((double)vx, (double)vx), __dmul_rn((double)vy, (double)vy))));
    A.x[i] = x; A.y[i] = y; A.h[i] = h; A.v[i] = v; A.vx[i] = vx; A.vy[i] = vy;
    A.type_id[i] = A.track_type[k];
  }
}

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

// ---------------------------------------------------------------------------- K4
// Single-line lidar of the ego (participant 0) of every scenario: SingleLineLidar._scan_obstacles
// (tactics2d/sensor/lidar.py:128-221).  Obstacle edges = the map's collidable segments (the reference takes the
// exteriors of `area.type_ == "obstacle"`, :137-143) + the pose rings of the other box-shaped participants (:146-153;
// a Pedestrian's pose is not a ring and is skipped there too), transformed into the ego frame (:105-126); per beam
// the reference's determinant intersection with its 1e-8 slack box filters (:160-213), min over edges, clip to the
// range, range -> inf.  One warp per scenario: sources are culled by distance, the surviving edges go to shared memory
// together with their beam window (beam_window below), and the warp walks the edges with its lanes sharing the beams of
// each window.  fp64 throughout (from the fp32 state): every tested pair gives exactly the float64 oracle's value, the
// untested pairs are ones the reference's own filters reject.
// The sensor may sit on any slot (t2d_lidar_scan_agents; the reference's SingleLineLidar bound with bind_with(j), whose
// scan skips participant j and sees every other one, :146-148): one warp per (scenario, observer) row n·Q + q, the rows
// of a scenario in adjacent warps so that they share its slots through L1.  t2d_lidar_scan is the row list {0} (Q = 1,
// no list): the walk over the other slots below visits exactly the slots 1 .. M-1 then, in the same rounds.
constexpr int LIDAR_EDGES = 144;   // edges per shared-memory chunk per warp (4 doubles + a beam window each)
constexpr int LIDAR_WARPS = 4;
constexpr int LIDAR_BEAMS = 512;   // beams per pass (running minima in shared memory)

struct LidarArgs : WorldArgs {
  MapArgs map;
  const double* beam_cs;      // [n_beams][2] cos, sin of the beam angles (host float64)
  const int16_t* observers;   // [N][Q]: the slot carrying the sensor of row n·Q + q, or nullptr: row q is slot q
  float* scan;                // [N][Q][n_beams]
  int Q, n_beams;
  double range;
};

__device__ __forceinline__ double point_segment_dist2(double x1, double y1, double x2, double y2) {   // from the origin
  const double dx = x2 - x1, dy = y2 - y1, dd = dx * dx + dy * dy;
  double t = dd > 0.0 ? -(x1 * dx + y1 * dy) / dd : 0.0;
  t = fmin(fmax(t, 0.0), 1.0);
  const double ex = x1 + t * dx, ey = y1 + t * dy;
  return ex * ex + ey * ey;
}

// (beam_window, the per-edge beam interval, lives in t2d_math.cuh so that tests/hostsim can check it on the host.)
__global__ void __launch_bounds__(LIDAR_WARPS * 32, 7) t2d_lidar_kernel(const __grid_constant__ LidarArgs A) {
  __shared__ double s_edge[LIDAR_WARPS][LIDAR_EDGES][4];
  __shared__ BeamWindow s_win[LIDAR_WARPS][LIDAR_EDGES];
  __shared__ float s_best[LIDAR_WARPS][LIDAR_BEAMS];
  __shared__ int s_cnt[LIDAR_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long row = (long long)blockIdx.x * LIDAR_WARPS + warp;
  if (row >= (long long)A.N * A.Q) return;
  // (the ego scan divides by nothing, and a 32-bit division serves every row index below 2^32)
  const long long n = A.Q == 1 ? row : row <= 0xffffffffll ? (long long)((unsigned)row / (unsigned)A.Q) : row / A.Q;
  const int q = (int)(row - n * A.Q);
  const int jo = A.observers ? (int)A.observers[row] : q;   // the slot carrying the sensor
  double(*edge)[4] = s_edge[warp];
  BeamWindow* win = s_win[warp];
  float* best = s_best[warp];
  int* cnt = &s_cnt[warp];
  const long long base = n * A.M;
  float* out = A.scan + row * A.n_beams;
  if (jo < 0 || jo >= A.M || A.type_id[base + jo] >= A.n_types) {   // not a slot, or an empty one: nothing is seen
    for (int b = lane; b < A.n_beams; b += 32) out[b] = INFINITY;
    return;
  }
  const double x0 = A.x[base + jo], y0 = A.y[base + jo], th = A.h[base + jo];
  double sa, ca;
  sincos(th, &sa, &ca);
  const double xoff = -x0 * ca - y0 * sa, yoff = x0 * sa - y0 * ca;   // lidar.py:116-121
  const double R = A.range, R2 = R * R;
  // the scenario's static-geometry tile (its header is read from global memory: one warp, a handful of words)
  const unsigned char* blob = tile_blob(A.map, n);
  const MapHeader* tmh = reinterpret_cast<const MapHeader*>(blob);
  const int n_seg = blob ? tmh->n_seg : 0;
  const float4* seg = n_seg > 0 ? reinterpret_cast<const float4*>(blob + tmh->off_seg) : nullptr;
  const int part_rounds = (A.M - 1 + 31) / 32, seg_rounds = (n_seg + 31) / 32;
  for (int b0 = 0; b0 < A.n_beams; b0 += LIDAR_BEAMS) {
    const int nb = min(LIDAR_BEAMS, A.n_beams - b0);      // beams b0 .. b0 + nb - 1 in this pass
    for (int k = lane; k < nb; k += 32) best[k] = INFINITY;
    if (lane == 0) *cnt = 0;
    __syncwarp();
    // Sources in rounds of 32: the other participants (a cheap centre-distance test first; a box in reach contributes
    // its four ring edges, :146-153), then the map segments (:137-143).  Edges within the range go to the shared chunk
    // with their beam window; the chunk is scanned whenever the next round might not fit.
    for (int r = 0; r < part_rounds + seg_rounds; ++r) {
      if (r < part_rounds) {
        const int i = r * 32 + lane;
        const int j = i < jo ? i : i + 1;   // the i-th slot other than the observer's
        const int tj = j < A.M ? (int)A.type_id[base + j] : 255;
        if (tj < A.n_types && A.table[tj].shape() == SHAPE_OBB) {
          const Params& pj = A.table[tj];
          const double xj = A.x[base + j], yj = A.y[base + j];
          const double reach = R + (double)pj.rbound * 1.000001 + 1e-6;
          if ((xj - x0) * (xj - x0) + (yj - y0) * (yj - y0) <= reach * reach) {
            double cx[4], cy[4], ex[4], ey[4];
            rect_corners_f64(xj, yj, A.h[base + j], pj.half_len, pj.half_wid, cx, cy);
#pragma unroll
            for (int k = 0; k < 4; ++k) {   // affine [a, b, -b, a, xoff, yoff]
              ex[k] = ca * cx[k] + sa * cy[k] + xoff;
              ey[k] = -sa * cx[k] + ca * cy[k] + yoff;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const double x1 = ex[k], y1 = ey[k], x2 = ex[(k + 1) & 3], y2 = ey[(k + 1) & 3];
              const double d2 = point_segment_dist2(x1, y1, x2, y2);
              if (d2 < R2 * 1.0000001 + 1e-9) {
                const int slot = atomicAdd(cnt, 1);
                edge[slot][0] = x1; edge[slot][1] = y1; edge[slot][2] = x2; edge[slot][3] = y2;
                win[slot] = beam_window(x1, y1, x2, y2, d2, A.n_beams);
              }
            }
          }
        }
      } else {
        const int si = (r - part_rounds) * 32 + lane;
        if (si < n_seg) {
          const float4 sg = seg[si];
          const double x1 = ca * sg.x + sa * sg.y + xoff, y1 = -sa * sg.x + ca * sg.y + yoff;
          const double x2 = ca * sg.z + sa * sg.w + xoff, y2 = -sa * sg.z + ca * sg.w + yoff;
          const double d2 = point_segment_dist2(x1, y1, x2, y2);
          if (d2 < R2 * 1.0000001 + 1e-9) {
            const int slot = atomicAdd(cnt, 1);
            edge[slot][0] = x1; edge[slot][1] = y1; edge[slot][2] = x2; edge[slot][3] = y2;
            win[slot] = beam_window(x1, y1, x2, y2, d2, A.n_beams);
          }
        }
      }
      __syncwarp();
      const int n_e = *cnt;
      if (n_e + 128 <= LIDAR_EDGES && r + 1 < part_rounds + seg_rounds) continue;   // the next round still fits
      // ---- edge by edge, the lanes share the beams of its window (lidar.py:160-213 for those pairs)
      for (int i = 0; i < n_e; ++i) {
        const double x1 = edge[i][0], y1 = edge[i][1], x2 = edge[i][2], y2 = edge[i][3];
        const BeamWindow w = win[i];
        const double d = y2 - y1, e = x1 - x2, f = y1 * x2 - x1 * y2;
        const double xlo = fmin(x1, x2) - 1e-8, xhi = fmax(x1, x2) + 1e-8, ylo = fmin(y1, y2) - 1e-8, yhi = fmax(y1, y2) + 1e-8;
        for (int t = lane; t < w.y; t += 32) {
          int b = w.x + t;
          if (b >= A.n_beams) b -= A.n_beams;
          const int k = b - b0;
          if (k < 0 || k >= nb) continue;
          const double cb = A.beam_cs[2 * b], sb = A.beam_cs[2 * b + 1];
          const double a_ = sb, b_ = -cb;
          const double det = a_ * e - b_ * d;
          if (det != 0.0) {
            const double rx = (b_ * f) / det, ry = (-a_ * f) / det;
            const double lx = cb * R, ly = sb * R;
            const bool okx = !(rx > fmax(1e-8, lx) + 1e-8) && !(rx < fmin(-1e-8, lx) - 1e-8) && !(rx > xhi) && !(rx < xlo);
            const bool oky = !(ry > fmax(1e-8, ly) + 1e-8) && !(ry < fmin(-1e-8, ly) - 1e-8) && !(ry > yhi) && !(ry < ylo);
            if (okx && oky) {
              const double dist = sqrt(rx * rx + ry * ry);
              if (dist < R) best[k] = fminf(best[k], (float)dist);   // clip to the range, range -> inf (:211-213)
            }
          }
        }
        __syncwarp();   // the next edge's window may hand the same beam to another lane
      }
      if (lane == 0) *cnt = 0;
      __syncwarp();
    }
    for (int k = lane; k < nb; k += 32) out[b0 + k] = best[k];
    __syncwarp();
  }
}

// ============================================================================ done exchange over peer memory
// All-gather of the per-rank done masks as ONE small kernel per rank and step, over NVLink / NVSwitch peer memory:
//   put     warp w serves the peers w, w + warps, ...: its lanes store 16-byte pieces of this rank's mask into slot
//           (step % slots), row `rank`, of that peer's gather ring (the own ring included);
//   signal  every lane fences its stores to system scope, the warp synchronises and lane 0 writes step + 1 into word
//           `rank` of the peer's flag array (a strong relaxed store behind the fence = a release): ONE fence round
//           trip per peer, all peers in parallel - not a chain of release stores issued by one thread;
//   wait    lanes 0 .. world-1 of warp 0 poll the OWN flag array (acquire, system scope) until every rank has signalled
//           step - lag; bounded (`timeout` SM cycles): on expiry the sticky error word is set and dst is filled with 0xFF;
//   copy    the slot of step - lag (all ranks' masks in rank order) goes to the caller's array.
// lag = 0 is the synchronous all-gather (the kernel cannot retire before the slowest rank's tick of this step has
// signalled).  lag >= 1 delivers the masks `lag` steps late: by then every signal has long arrived, the wait never spins
// and the kernel is a few microseconds of posted stores - the exchange leaves the critical path (the consumer of the
// gathered masks, a learner or reset scheduler, is behind the simulation anyway).  The kernels of one rank run in
// stream order and kernel k only completes after every rank has signalled step k - lag, i.e. after every rank's kernel
// k - lag - 1 has copied step k - 2 lag - 1 out: a ring of 2 lag + 2 slots is never overwritten before it was read.
struct AllGatherArgs {
  unsigned char* peer[T2D_MAX_RANKS];   // every rank's exchange allocation (own included)
  unsigned char* base;                  // = peer[rank]
  const unsigned char* local;           // this rank's done mask [n_real]
  unsigned char* dst;                   // [world * n_local]
  int world, rank, n_local, n_real, slots, lag;
  long long timeout;                    // SM cycles the wait may spin
};

__global__ void __launch_bounds__(512) t2d_exchange_allgather_kernel(const __grid_constant__ AllGatherArgs A) {
  __shared__ int s_ok;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  const size_t flag_off = (size_t)A.slots * A.world * A.n_local;
  unsigned* words = reinterpret_cast<unsigned*>(A.base + flag_off);      // [0, MAX_RANKS): flags; then step, -, -, error
  const unsigned step = words[T2D_MAX_RANKS];
  const size_t row = (size_t)(step % (unsigned)A.slots) * A.world * A.n_local + (size_t)A.rank * A.n_local;
  if (threadIdx.x == 0) s_ok = 1;
  // ---- put + signal, one warp per peer
  const int n16 = A.n_local / 16;   // n_local is a multiple of 16; the tail beyond n_real is zero
  for (int p = warp; p < A.world; p += warps) {
    uint4* out = reinterpret_cast<uint4*>(A.peer[p] + row);
    for (int i = lane; i < n16; i += 32) {
      uint4 v;
      if (16 * i + 16 <= A.n_real && (reinterpret_cast<uintptr_t>(A.local) & 15) == 0) {
        v = __ldcg(reinterpret_cast<const uint4*>(A.local) + i);
      } else {
        unsigned char b[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) b[k] = (16 * i + k < A.n_real) ? A.local[16 * i + k] : (unsigned char)0;
        memcpy(&v, b, 16);
      }
      out[i] = v;
    }
    __threadfence_system();
    __syncwarp();
    if (lane == 0) {
      unsigned* f = reinterpret_cast<unsigned*>(A.peer[p] + flag_off) + A.rank;
      asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(f), "r"(step + 1u) : "memory");
    }
  }
  // ---- wait for step - lag
  const bool deliver = step >= (unsigned)A.lag;
  const unsigned target = step - (unsigned)A.lag;     // the step whose masks this call delivers
  if (deliver && threadIdx.x < (unsigned)A.world) {
    const unsigned* f = words + threadIdx.x;
    const long long t0 = clock64();
    unsigned v;
    for (;;) {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
      if (v >= target + 1u) break;
      if (clock64() - t0 > A.timeout) { s_ok = 0; break; }
      __nanosleep(20);
    }
  }
  __syncthreads();
  const size_t bytes = (size_t)A.world * A.n_local;
  if (deliver) {
    if (s_ok) {
      // ---- copy
      const unsigned char* src = A.base + (size_t)(target % (unsigned)A.slots) * bytes;
      if ((reinterpret_cast<uintptr_t>(A.dst) & 15) == 0) {
        for (size_t i = threadIdx.x; i < bytes / 16; i += blockDim.x)
          reinterpret_cast<uint4*>(A.dst)[i] = __ldcg(reinterpret_cast<const uint4*>(src) + i);
      } else {
        for (size_t i = threadIdx.x; i < bytes; i += blockDim.x) A.dst[i] = __ldcg(src + i);
      }
    } else {
      // a rank never showed up: the caller must not mistake stale masks for this step's - 0xFF is no done value
      for (size_t i = threadIdx.x; i < bytes; i += blockDim.x) A.dst[i] = (unsigned char)0xFF;
      if (threadIdx.x == 0) words[T2D_MAX_RANKS + 3] = 1u;
    }
  }
  if (threadIdx.x == 0) words[T2D_MAX_RANKS] = step + 1u;
}

// ============================================================================ K5: NPC controllers
// One warp per scenario; lane l owns participants l, l + 32, ... .  fp64 on the fp32 state (a few dozen flops per
// participant: the kernel is bound by its ~30 B / participant of HBM traffic).  All reads of last_accel (own and the
// leader's, previous tick) happen before the warp barrier, all writes (this tick) after it.

// The leading fields of t2d_controller_params, the only ones the IDM / cruise / pure-pursuit laws read.  The row also
// holds doubles (the PID part), so it is 8-byte aligned; read through this 4-byte-aligned view, those laws load their
// fields one by one as they did before the row grew.
struct CtrlLawRow {
  int32_t kind;
  float desired_speed, time_headway, min_spacing, max_acceleration, comfortable_deceleration, delta;
  float target_speed, kp, accel_change_rate, delta_t, max_accel, min_accel, interval;
  float min_pre_aiming_distance, pp_interval, wheel_base;
};
static_assert(alignof(CtrlLawRow) == 4 && offsetof(CtrlLawRow, wheel_base) == offsetof(t2d_controller_params, wheel_base),
              "CtrlLawRow is the float prefix of t2d_controller_params");

struct CtrlArgs : WorldArgs {
  const t2d_controller_params* ctab;
  int n_ctrl;
  const uint8_t* ctrl_id;
  const int16_t* lead;
  const int16_t* path_id;
  const PathVertex* path_v;
  const int* path_off;
  int n_paths;
  float* last_accel;
  float* action;
  const float* ego_action;   // [N][2] or nullptr: participant 0's action (written into its row of `action` as well)
  int steer_first;
  const float* pid_target;   // [N][M][2] (target_speed, lateral target) or nullptr; read by the HAS_PID instance only
  double* pid_state;         // [N][M][6] or nullptr; read and written by the HAS_PID instance only
};

__device__ __forceinline__ double clip_np(double v, double lo, double hi) {   // np.clip: NaN propagates
  return v != v ? v : fmin(fmax(v, lo), hi);
}

// acceleration_controller.py:82-130: cruise, or adaptive cruise when a leader is given
__device__ double longitudinal_law(const CtrlLawRow& p, double v, double x, double y, double a_last, bool has_lead,
                                   double vl, double xl, double yl, double al) {
  const double kp = (double)p.kp;
  double a;
  if (has_lead) {
    const double d_front = sqrt((x - xl) * (x - xl) + (y - yl) * (y - yl));                  // :114
    const double d_target = clip_np(v * (double)p.interval + 5.0, 7.0, 80.0);                // :115-118, :42-45
    const double rel_speed = vl - v;                                                         // :120
    const double rel_target_speed = (d_target - d_front) / kp;                               // :121
    const double rel_accel = (rel_target_speed - rel_speed) / kp;                            // :122
    a = al - rel_accel;                                                                      // :124
  } else {
    a = ((double)p.target_speed - v) / kp;                                                   // :94
  }
  const double w = (double)p.accel_change_rate * (double)p.delta_t;
  a = clip_np(a, a_last - w, a_last + w);                                                    // :95-99, :126-130
  return clip_np(a, (double)p.min_accel, (double)p.max_accel);
}

// (v / v_des) ** delta: the IDM exponent is 4 by default - two multiplications instead of the general pow()
__device__ __forceinline__ double idm_pow(double r, double delta) {
  if (delta == 4.0) { const double r2 = r * r; return r2 * r2; }
  if (delta == 2.0) return r * r;
  return pow(r, delta);
}

// idm_controller.py:59-141
__device__ double idm_law(const CtrlLawRow& p, double v, double x, double y, bool has_lead, double vl, double xl,
                          double yl) {
  const double vd = (double)p.desired_speed, am = (double)p.max_acceleration, b = (double)p.comfortable_deceleration;
  double a;
  if (!has_lead) {
    a = vd > 0.0 ? am * (1.0 - idm_pow(v / vd, (double)p.delta)) : (v > 0.0 ? -b : 0.0);     // :74-82
  } else {
    const double dist = sqrt((xl - x) * (xl - x) + (yl - y) * (yl - y));                     // :107-109 (np.hypot, no overflow concern at map scale)
    const double dv = vl - v;                                                                // :112
    double s_star = (double)p.min_spacing + v * (double)p.time_headway + (v * dv) / (2.0 * sqrt(am * b));   // :116-120
    s_star = fmax(s_star, (double)p.min_spacing);                                            // :121
    if (dist > 0.0) {
      const double ratio = vd > 0.0 ? idm_pow(v / vd, (double)p.delta) : (v > 0.0 ? 1.0 : 0.0);  // :127-130
      const double q = s_star / dist;
      a = am * (1.0 - ratio - q * q);                                                        // :132-134
    } else {
      a = -b;                                                                                // :137
    }
  }
  return clip_np(a, -b, am);                                                                 // :89
}

// pure_pursuit_controller.py:51-74,90-92; LineString.interpolate = arc-length walk from the first vertex
__device__ double pure_pursuit_law(const CtrlLawRow& p, const PathVertex* pv, int n_vert, double v, double x, double y,
                                   double heading) {
  const double d = fmax(v * (double)p.pp_interval, (double)p.min_pre_aiming_distance);     // :90-91
  double px = pv[n_vert - 1].x, py = pv[n_vert - 1].y;
  for (int i = 0; i + 1 < n_vert; ++i) {
    const PathVertex q = pv[i];
    if (d <= q.cum + q.len && q.len > 0.0) {
      const double t = (d - q.cum) / q.len;
      px = q.x + t * (pv[i + 1].x - q.x);
      py = q.y + t * (pv[i + 1].y - q.y);
      break;
    }
  }
  const double ang = atan2(py - y, px - x);                                                 // :62-64
  const double dist = hypot(py - y, px - x);                                                // :65-67
  return atan(2.0 * (double)p.wheel_base * sin(ang - heading) / dist);                      // :68-70
}

// pid_controller.py:159-234, one channel.  s = (integral, prev_error, prev_derivative) is rewritten in place.  Every
// operation rounds once (no FMA contraction) in the reference's order; `limited` selects the output_limits branch.
__device__ double pid_channel(const t2d_controller_params& p, double e, double s[3], double kp, double ki, double kd,
                              bool limited, double lo, double hi) {
  const double alpha = p.derivative_filter_alpha;
  const double p_term = __dmul_rn(kp, e);                                                     // :191
  const double raw = __ddiv_rn(__dsub_rn(e, s[1]), p.dt);                                     // :194
  const double d = __dadd_rn(__dmul_rn(alpha, raw), __dmul_rn(__dsub_rn(1.0, alpha), s[2]));   // :195-198
  double out = __dadd_rn(p_term, __dmul_rn(kd, d));                                          // :199-202
  bool saturated = false;
  if (limited) {                                                                             // :205-214
    if (out > hi) { saturated = true; out = hi; }
    else if (out < lo) { saturated = true; out = lo; }
  }
  s[0] = saturated ? __dmul_rn(s[0], 0.99) : __dadd_rn(s[0], __dmul_rn(e, p.dt));            // :217-222
  out = __dadd_rn(out, __dmul_rn(ki, s[0]));                                                 // :224-227
  if (limited) out = clip_np(out, lo, hi);                                                   // :230-232
  s[1] = e;
  s[2] = d;
  return out;
}

// The lateral error of a PATH_* source (no reference counterpart), from the closest point c and its tangent u:
// PATH_CROSS_TRACK: e = u.x (c.y - y) - u.y (c.x - x), positive when the path lies to the left; PATH_HEADING:
// target_heading = atan2(u.y, u.x).  false: no segment.
__device__ bool path_lateral_error(const PathVertex* pv, int n_vert, double x, double y, double heading, bool cross,
                                   double& e) {
  PathPoint c;
  if (!closest_on_path<false>(pv, n_vert, x, y, c)) return false;
  if (cross) {
    e = __dsub_rn(__dmul_rn(c.ux, __dsub_rn(c.cy, y)), __dmul_rn(c.uy, __dsub_rn(c.cx, x)));
  } else {
    const double err = __dsub_rn(atan2(c.uy, c.ux), heading);
    e = atan2(sin(err), cos(err));
  }
  return true;
}

// pid_controller.py:309-406 for slot i: (steering, acceleration) into steer / acc; the slot's state row is rewritten
// for each channel that runs.  A channel whose source is NONE, or whose error is missing (a PATH source without a usable
// path: the combined mode's missing keyword), gives 0 and leaves its half of the row alone.
__device__ void pid_law(const t2d_controller_params& p, const CtrlArgs& A, size_t i, double x, double y, double v,
                        double heading, double& steer, double& acc) {
  double* st = A.pid_state + 6 * i;
  steer = 0.0;
  acc = 0.0;
  const int lat = p.pid_lateral;
  if (lat != T2D_PID_LAT_NONE) {
    double e = 0.0;
    bool have = true;
    if (lat == T2D_PID_LAT_HEADING) {                                                       // :267-274
      const double err = __dsub_rn((double)A.pid_target[2 * i + 1], heading);
      e = atan2(sin(err), cos(err));
    } else if (lat == T2D_PID_LAT_CROSS_TRACK) {                                             // :275-279
      e = (double)A.pid_target[2 * i + 1];
    } else {
      const int pid = A.path_id ? (int)A.path_id[i] : -1;
      have = pid >= 0 && pid < A.n_paths &&
             path_lateral_error(A.path_v + A.path_off[pid], A.path_off[pid + 1] - A.path_off[pid], x, y, heading,
                                lat == T2D_PID_LAT_PATH_CROSS_TRACK, e);
    }
    if (have) {
      double s[3] = {st[0], st[1], st[2]};
      const double out = pid_channel(p, e, s, p.kp_lat, p.ki_lat, p.kd_lat, false, 0.0, 0.0);   // :338-348
      const bool cross = lat == T2D_PID_LAT_CROSS_TRACK || lat == T2D_PID_LAT_PATH_CROSS_TRACK;
      steer = cross ? __dmul_rn(out, __ddiv_rn(2.0, (double)p.wheel_base)) : out;            // :355-365
      steer = clip_np(steer, -p.max_steering, p.max_steering);                               // :368
      st[0] = s[0]; st[1] = s[1]; st[2] = s[2];
    }
  }
  if (p.pid_longitudinal == T2D_PID_LON_TARGET) {
    const double e = __dsub_rn((double)A.pid_target[2 * i], v);                              // :306-307
    double s[3] = {st[3], st[4], st[5]};
    const double lo = (double)p.min_accel, hi = (double)p.max_accel;
    acc = clip_np(pid_channel(p, e, s, p.kp_lon, p.ki_lon, p.kd_lon, true, lo, hi), lo, hi);   // :383-397
    st[3] = s[0]; st[4] = s[1]; st[5] = s[2];
  }
}

__device__ __forceinline__ const CtrlLawRow& law_row(const t2d_controller_params* ctab, int cid) {
  return *reinterpret_cast<const CtrlLawRow*>(reinterpret_cast<const char*>(ctab) + (size_t)cid * sizeof(t2d_controller_params));
}

// HAS_PID: the instance with the PID law, launched when the bound table holds a PID row; the other one is today's K5.
template <bool HAS_PID>
__global__ void __launch_bounds__(128) t2d_control_kernel(const __grid_constant__ CtrlArgs A) {
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; n < A.N; n += warps) {
    const size_t base = (size_t)n * A.M;
    float2 out[4];
    float mag[4];
    bool ctl[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = lane + 32 * j;
      ctl[j] = false;
      mag[j] = 0.0f;
      out[j] = make_float2(0.0f, 0.0f);
      if (m >= A.M) continue;
      const int tid = A.type_id[base + m];
      if (tid >= A.n_types) continue;                  // inactive slot
      const Params& tp = A.table[tid];
      out[j] = reinterpret_cast<const float2*>(A.action)[base + m];
      if (m == 0 && A.ego_action != nullptr) { out[j] = reinterpret_cast<const float2*>(A.ego_action)[n]; ctl[j] = true; }   // row 0 <- the ego's action
      const int cid = A.ctrl_id[base + m];
      if (cid < A.n_ctrl && law_row(A.ctab, cid).kind != T2D_CTRL_EXTERNAL) {
        const CtrlLawRow& p = law_row(A.ctab, cid);
        const double x = A.x[base + m], y = A.y[base + m], v = A.v[base + m];
        const int li = A.lead ? (int)A.lead[base + m] : -1;
        const bool has = li >= 0 && li < A.M && li != m && A.type_id[base + li] < A.n_types;
        double xl = 0.0, yl = 0.0, vl = 0.0, al = 0.0;
        if (has) {
          xl = A.x[base + li]; yl = A.y[base + li]; vl = A.v[base + li]; al = A.last_accel[base + li];
        }
        double acc, steer = 0.0;
        if (HAS_PID && p.kind == T2D_CTRL_PID) {
          pid_law(A.ctab[cid], A, base + m, x, y, v, (double)A.h[base + m], steer, acc);
        } else if (p.kind == T2D_CTRL_IDM) {
          acc = idm_law(p, v, x, y, has, vl, xl, yl);
        } else {
          acc = longitudinal_law(p, v, x, y, (double)A.last_accel[base + m], has, vl, xl, yl, al);
          if (p.kind == T2D_CTRL_PURE_PURSUIT) {
            const int pid = A.path_id ? (int)A.path_id[base + m] : -1;
            if (pid >= 0 && pid < A.n_paths)
              steer = pure_pursuit_law(p, A.path_v + A.path_off[pid], A.path_off[pid + 1] - A.path_off[pid], v, x, y,
                                       (double)A.h[base + m]);
          }
        }
        out[j] = A.steer_first ? make_float2((float)steer, (float)acc) : make_float2((float)acc, (float)steer);
        ctl[j] = true;
      }
      // |a| the physics will apply: single_track_kinematics.py:192 clips to the accel range; point_mass.py takes (ax, ay) as is
      if (tp.model() <= T2D_MODEL_DYNAMICS || tp.model() == T2D_MODEL_DRIFT)
        mag[j] = fabsf(clampf(A.steer_first ? out[j].y : out[j].x, tp.accel_lo, tp.accel_hi));
      else if (tp.model() <= T2D_MODEL_POINTMASS_EULER)
        mag[j] = (float)hypot((double)out[j].x, (double)out[j].y);
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = lane + 32 * j;
      if (m >= A.M) continue;
      if (ctl[j]) reinterpret_cast<float2*>(A.action)[base + m] = out[j];
      A.last_accel[base + m] = mag[j];
    }
  }
}

}  // namespace t2d

#include "t2d_bev.cuh"
#include "t2d_obs.cuh"
#include "t2d_history.cuh"

// =============================================================================================
// C ABI
// =============================================================================================
using namespace t2d;

static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};
// K1 launches per instance (launch_step's `variant`), then the one-tile launches that read the map from global memory
static std::atomic<long long> g_tick_instances[7] = {};
static std::atomic<int> g_exchanges_alive{0};   // peer-memory done exchanges in this process (see StepArgs::prefetch)
static std::mutex g_smem_mutex;
// [device]: the fallback counters of K1's FIXED instance (ORDER_COUNTERS x ORDER_COUNTER_STRIDE, zeroed), allocated by
// the first t2d_create on the device and kept for the life of the process, as a __device__ variable would be
static unsigned long long* g_order_fallbacks[64] = {};
static std::mutex g_order_mutex;
static int g_smem_configured[64][6];   // [device][kernel variant]: dynamic shared memory opted in so far (process-wide)

static int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
#define CUDA_TRY(expr)                                                                           \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) return fail(T2D_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

// Owners of the context's device and pinned host buffers.  Dropping one frees its buffer, so whatever replaces or drops
// one runs with the context's device current.
struct CudaFree {
  void operator()(void* p) const { cudaFree(p); }
};
struct CudaFreeHost {
  void operator()(void* p) const { cudaFreeHost(p); }
};
template <class T> using dev_ptr = std::unique_ptr<T, CudaFree>;
template <class T> using host_ptr = std::unique_ptr<T, CudaFreeHost>;

template <class T> static int dev_alloc(dev_ptr<T>& out, size_t n) {
  T* p = nullptr;
  CUDA_TRY(cudaMalloc(&p, n * sizeof(T)));
  out.reset(p);
  return T2D_OK;
}

template <class T> static int host_alloc(host_ptr<T>& out, size_t n, unsigned flags = cudaHostAllocDefault) {
  T* p = nullptr;
  CUDA_TRY(cudaHostAlloc(&p, n * sizeof(T), flags));
  out.reset(p);
  return T2D_OK;
}

// n host elements copied to a fresh device buffer; `out` changes only on success
template <class T> static int upload(dev_ptr<T>& out, const T* src, size_t n) {
  dev_ptr<T> d;
  if (int r = dev_alloc(d, n)) return r;
  CUDA_TRY(cudaMemcpy(d.get(), src, n * sizeof(T), cudaMemcpyHostToDevice));
  out = std::move(d);
  return T2D_OK;
}

struct t2d_exchange {
  int device = 0, world = 0, rank = 0, n_local = 0, slots = 0;
  size_t bytes = 0;
  int n_real = 0;
  int threads = 256;                             // CTA size of the exchange kernel (T2D_EXCHANGE_THREADS, read once at create)
  long long timeout_cycles = 4000000000LL;       // how long a wait may spin (~2 s of SM clocks; T2D_EXCHANGE_TIMEOUT_MS)
  unsigned char* base = nullptr;                 // slots x world x n_local done bytes | MAX_RANKS flag words | step, -, -, error
  unsigned char* peer[T2D_MAX_RANKS] = {};       // every rank's base (own included), valid after t2d_exchange_connect
  bool connected = false;
  size_t flag_off() const { return (size_t)slots * world * n_local; }
  unsigned* word(int i) const { return reinterpret_cast<unsigned*>(base + flag_off()) + T2D_MAX_RANKS + i; }   // 0 steps done, 3 error
};

// The bound map (t2d_set_map_table), replaced as a whole: a new map also drops the per-segment BEV styles of the old one
struct DeviceMap {
  dev_ptr<unsigned char> blob;         // the tiles back to back, each 128-byte aligned
  dev_ptr<uint32_t> tile_off;          // [n_tiles] byte offsets of the tiles inside blob
  const uint16_t* tile_id = nullptr;   // caller-owned DEVICE [N]; nullptr unless there is more than one tile
  int n_tiles = 0;
  bool has_segments = false;
  bool has_bounds = false;             // any tile has a boundary box
  MapHeader mh{};                      // tile 0's header
  int smem_bytes = 0;                  // what a single tile stages into shared memory
  std::vector<int> tile_nseg;          // segments of every tile, in tile order
  dev_ptr<uint8_t> seg_style;          // BEV style per segment, tiles back to back; nullptr: the default ring / open styles
  dev_ptr<uint32_t> seg_base;          // [n_tiles] first entry of every tile in seg_style
};

// The bound log (t2d_set_log / K7), replaced as a whole
struct DeviceLog {
  dev_ptr<ReplayTrack> tracks;
  dev_ptr<uint8_t> track_type;
  dev_ptr<float> rec;
  dev_ptr<int32_t> t0;
  dev_ptr<int32_t> slot_off;           // [n_rows * M + 1] schedule offsets
  dev_ptr<ReplayEntry> entries;
  dev_ptr<int32_t> slot_track1;        // [n_rows * M] instead of the two above when no schedule has two entries
  int n_tracks = 0, n_rows = 0;
  int32_t* row = nullptr;              // caller-owned DEVICE [N]
  int32_t* track_out = nullptr;        // caller-owned DEVICE [N][M] or nullptr
  uint8_t* type_id = nullptr;          // writable alias of type_id, checked against the bound one before every launch
  std::vector<uint8_t> track_type_host;   // host copy: t2d_set_type_table keeps these rows static
};

// The bound reset sampler (t2d_set_reset_sampler), replaced as a whole: the caller's struct with the jitter table moved
// into the library's own device copy
struct DeviceSampler {
  t2d_reset_sampler s{};               // s.jitter: jitter.get() or nullptr
  dev_ptr<float> jitter;               // [M][8]
};

// The trajectory history ring (t2d_set_history), replaced as a whole; the track ring exists exactly while a log schedule
// with a track output is bound (history_tracks)
struct DeviceHistory {
  int H = 0;
  dev_ptr<float> f;                    // [6][N][H][M]: x, y, heading, speed, vx, vy
  dev_ptr<uint8_t> type;               // [N][H][M]
  dev_ptr<int32_t> track;              // [N][H][M] or nullptr
  dev_ptr<long long> count;            // [N]
};

// Staging of the host steps (t2d_step_host, t2d_step_host_ego, t2d_step_host_agents); every piece is created whole the
// first time a step needs it.
static constexpr int MAX_HOST_CHUNKS = 8;

struct ChunkedUpload {   // t2d_step_host: device copy of the actions, the copy stream and its events
  dev_ptr<float> action;               // [N][M][2]
  cudaStream_t copy = nullptr;
  cudaEvent_t begin = nullptr, chunk[MAX_HOST_CHUNKS] = {};
  ~ChunkedUpload() {
    if (begin) cudaEventDestroy(begin);
    for (cudaEvent_t e : chunk)
      if (e) cudaEventDestroy(e);
    if (copy) cudaStreamDestroy(copy);
  }
};

struct Mirror {   // a packed block of device outputs and its pinned host mirror
  dev_ptr<uint8_t> dev;
  host_ptr<uint8_t> host;
};

struct MappedEgo {   // t2d_step_host_ego: [N][2] pinned + mapped host staging of the ego actions ...
  host_ptr<float> host;
  const float* dev = nullptr;          // ... and its device-side address: the kernels read it over PCIe, no copy engine involved
};

struct AgentStaging {   // t2d_step_host_agents, sized for q rows per scenario
  int q = 0;
  dev_ptr<float> action;               // [N][Q][2]
  Mirror out;                          // device: [N][Q] fp32 reward, [3][N][Q] uint8, [N] uint8 done, then [N][Q] fp32 iou;
                                       // host: the part up to done
};

struct t2d_ctx {
  int device = 0, N = 0, M = 0, G = 0;
  t2d_config cfg{};
  int n_types = 0;
  bool has_pointmass = false;
  bool has_drift = false;
  bool kin_only = false;
  float *wheel_f = nullptr, *wheel_r = nullptr;
  const float *reset_pool_wf = nullptr, *reset_pool_wr = nullptr;   // t2d_bind_reset_wheel_pool
  dev_ptr<Params> d_table;
  DeviceMap map;
  float *x = nullptr, *y = nullptr, *h = nullptr, *v = nullptr, *vx = nullptr, *vy = nullptr;
  const uint8_t* type_id = nullptr;
  int32_t* step_count = nullptr;
  int sm_count = 0;                // set by t2d_create from the device
  int max_smem_optin = 0;
  float rb_max = 0.0f;
  const float* ego_action = nullptr;   // t2d_set_ego_action
  GoalArgs goal{};                     // t2d_set_goal
  // per-agent status and reward (t2d_set_agents / K10); agent_q == 0: not bound
  int agent_q = 0;
  const int16_t* agent_observers = nullptr;
  GoalArgs agent{};                    // iou: the t2d_agents_epilogue argument
  uint8_t* agent_retired = nullptr;
  bool use_pdl = true;            // T2D_PDL=0 disables programmatic dependent launch
  int prefetch_override = -1;      // T2D_PREFETCH=0 / 1 (experiments; -1 = on unless a done exchange is alive)
  int wpc_override = 0;            // T2D_WPC=w: warps per CTA of the tick (experiments; 0 = pick from the batch size)
  int grid_limit = 0;              // T2D_GRID_LIMIT=k: at most k CTAs of the persistent tick grid per SM (experiments; 0 = occupancy)
  bool tick_generic = false;       // T2D_TICK_GENERIC=1: never launch K1's FIXED instance (tests compare the two)
  int occ_smem[9] = {-1, -1, -1, -1, -1, -1, -1, -1, -1};   // per warps-per-CTA: smem the cached occupancy was computed for
  int occ_val[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  int occ_variant[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  // NPC controllers (t2d_set_controllers / t2d_set_paths / t2d_control)
  dev_ptr<t2d_controller_params> d_ctab;
  int n_ctrl = 0;
  const uint8_t* ctrl_id = nullptr;
  const int16_t* ctrl_lead = nullptr;
  const int16_t* ctrl_path = nullptr;
  float* ctrl_last_accel = nullptr;
  bool ctrl_has_pid = false;          // the table holds a T2D_CTRL_PID row: K5 runs its PID instance
  bool ctrl_pid_reads_target = false; // ... and one of them reads the target array
  const float* pid_target = nullptr;  // t2d_set_pid: [N][M][2]
  double* pid_state = nullptr;        // t2d_set_pid: [N][M][6]
  dev_ptr<PathVertex> d_path_v;
  dev_ptr<int> d_path_off;
  int n_paths = 0;
  // routes (t2d_set_routes / t2d_bind_route_trackers); route_id == nullptr: none bound
  const int16_t* route_id = nullptr;
  double route_threshold = 0.0, route_weight = 0.0;
  float route_off_reward = 0.0f;
  double* route_s_best = nullptr;        // [N] or nullptr
  double* route_agent_s_best = nullptr;  // [N][route_agent_rows] or nullptr
  int route_agent_rows = 0;
  // host steps
  std::unique_ptr<ChunkedUpload> hs_upload;
  Mirror hs_out;                       // [2][N] status, done (t2d_step_host and t2d_step_host_ego)
  MappedEgo hs_ego;
  AgentStaging ha;
  dev_ptr<uint8_t> ha_flags;           // [N][M]: the flags K10 needs when the caller keeps none
  int host_chunks = 0;                 // 0 = pick from the batch size
  // BEV observation (t2d_set_bev_styles / t2d_bev_render)
  int n_bev_styles = 0;                // 0: styles not set
  t2d_bev_style bev_style[bev::MAX_STYLES] = {};
  uint8_t bev_type_style[T2D_MAX_TYPES] = {};
  int bev_target_style = bev::NO_STYLE;
  std::unique_ptr<DeviceLog> log;      // nullptr: no log bound
  std::vector<int> type_model;         // host copy of the current type table's model ids
  dev_ptr<uint8_t> order;              // [N][64] x-order hint of K1's FIXED instance (t2d_create: the identity)
  std::unique_ptr<DeviceSampler> sampler;   // t2d_set_reset_sampler; nullptr: none bound
  std::unique_ptr<DeviceHistory> hist;      // t2d_set_history; nullptr: none bound
};

enum : unsigned { NEED_STATE = 1, NEED_TABLE = 2, NEED_TICK = 4 };

// The call-order preconditions, checked in this order: the bound state, the type table, and what a tick with physics
// needs besides (a caller that launches other kernels first checks them up front).
static int require(const t2d_ctx* c, unsigned need) {
  if ((need & NEED_STATE) && !c->x) return fail(T2D_E_STATE, "state not bound: call t2d_bind_state first");
  if ((need & NEED_TABLE) && (!c->d_table || c->n_types == 0))
    return fail(T2D_E_STATE, "type table not set: call t2d_set_type_table first");
  if (need & NEED_TICK) {
    if (c->has_drift && !(c->wheel_f && c->wheel_r))
      return fail(T2D_E_STATE, "the type table holds a SingleTrackDrift row: call t2d_bind_wheel_state first");
    if (c->log && c->log->type_id != c->type_id) return fail(T2D_E_STATE, "state rebound after t2d_set_log: call t2d_set_log again");
  }
  return T2D_OK;
}

static WorldArgs world_args(const t2d_ctx* c) {
  return {c->x, c->y, c->h, c->v, c->vx, c->vy, c->type_id, c->step_count, c->d_table.get(), c->n_types, c->N, c->M};
}

static RouteArgs route_args(const t2d_ctx* c) {
  return {c->route_id, c->d_path_v.get(), c->d_path_off.get(), c->n_paths, c->route_off_reward, c->route_threshold,
          c->route_weight};
}

// K10 reads its progress tracker by the bound agents' rows: a tracker bound for another Q is a call-order error
static int check_route_trackers(const t2d_ctx* c, const char* fn) {
  if (c->route_id && c->route_agent_s_best && c->route_agent_rows != c->agent_q)
    return fail(T2D_E_STATE, std::string(fn) + ": the agents' route tracker has another row count than the bound agents: "
                                               "call t2d_bind_route_trackers again");
  return T2D_OK;
}

// ---- trajectory history (t2d_set_history; K15 / K16)
static hist::Ring history_ring(const t2d_ctx* c) {
  const DeviceHistory& g = *c->hist;
  const size_t plane = (size_t)c->N * g.H * c->M;
  float* f = g.f.get();
  return {f, f + plane, f + 2 * plane, f + 3 * plane, f + 4 * plane, f + 5 * plane, g.type.get(), g.track.get(), g.count.get(), g.H};
}

// the track every slot shows now, when the ring records tracks
static const int32_t* history_track_now(const t2d_ctx* c) { return c->hist->track ? c->log->track_out : nullptr; }

// Gives `g` a fresh track ring filled with -1 (an entry recorded before the schedule counts as showing no track) when
// `track_out`, the bound schedule's track output, is set, and drops it otherwise
static int history_tracks(const t2d_ctx* c, DeviceHistory& g, const int32_t* track_out) {
  if (!track_out) {
    g.track.reset();
    return T2D_OK;
  }
  const size_t n = (size_t)c->N * g.H * c->M;
  dev_ptr<int32_t> t;
  if (int r = dev_alloc(t, n)) return r;
  CUDA_TRY(cudaMemset(t.get(), 0xff, n * sizeof(int32_t)));
  g.track = std::move(t);
  return T2D_OK;
}

// from scenario `first` on (t2d_set_map_table keeps tile_id only with more than one tile)
static MapArgs map_args(const DeviceMap& map, int first = 0) {
  return {map.blob.get(), map.tile_off.get(), map.tile_id ? map.tile_id + first : nullptr};
}

// after every launch: count it and report a launch error
static int launched() {
  g_launches.fetch_add(1);
  CUDA_TRY(cudaGetLastError());
  return T2D_OK;
}

// grid of a grid-stride kernel: one CTA per `per_cta` items, at most `per_sm` CTAs per SM
static int capped_grid(long long items, int per_cta, int sm_count, int per_sm) {
  return (int)std::max(1LL, std::min((items + per_cta - 1) / per_cta, (long long)sm_count * per_sm));
}

// K15 after a tick (mask == nullptr: every scenario appends) or a reset (the masked scenarios restart); no ring, no launch
static int launch_history(t2d_ctx* c, const uint8_t* mask, void* stream) {
  if (!c->hist) return T2D_OK;
  hist::AppendArgs A{world_args(c)};
  A.ring = history_ring(c); A.track_now = history_track_now(c); A.mask = mask;
  hist::t2d_history_append_kernel<<<(c->N + hist::K15_WARPS - 1) / hist::K15_WARPS, hist::K15_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

// the integration steps of one interval, for the tick and t2d_physics_step
template <class Args> static void set_time_step(Args& A, int interval_ms, int delta_t_ms) {
  const int delta_t = std::min(delta_t_ms, interval_ms);
  A.n_steps = interval_ms / delta_t;                            // single_track_kinematics.py:129
  A.dt = (float)((double)delta_t / 1000.0);                     // :128
  A.dt_rem = (float)((double)(interval_ms % delta_t) / 1000.0);   // :130,152
  A.dt_d = (double)delta_t / 1000.0;
  A.dt_rem_d = (double)(interval_ms % delta_t) / 1000.0;
  A.interval_d = (double)interval_ms / 1000.0;                  // point_mass.py:86
}

extern "C" {

int t2d_version(void) { return T2D_VERSION; }
const char* t2d_last_error(void) { return g_err.c_str(); }
int64_t t2d_launch_count(void) { return (int64_t)g_launches.load(); }
int64_t t2d_tick_fixed_count(void) { return (int64_t)(g_tick_instances[4].load() + g_tick_instances[5].load()); }
int64_t t2d_tick_order_fallback_count(void) {
  std::lock_guard<std::mutex> lock(g_order_mutex);
  int64_t sum = 0;
  for (unsigned long long* d : g_order_fallbacks) {
    if (!d) continue;
    unsigned long long n[ORDER_COUNTERS * ORDER_COUNTER_STRIDE];
    if (cudaMemcpy(n, d, sizeof(n), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    for (int i = 0; i < ORDER_COUNTERS; ++i) sum += (int64_t)n[i * ORDER_COUNTER_STRIDE];
  }
  return sum;
}
int64_t t2d_tick_instance_count(int k) { return k >= 0 && k < 7 ? (int64_t)g_tick_instances[k].load() : -1; }

#ifdef T2D_TICK_TIMELINE
// The phase timeline of the last tick (measurement build only): [TL_MAX_WARPS][TL_POINTS][globaltimer, clock64],
// zeroed after the copy when `clear` is set.
int t2d_tick_timeline(void* dst, int64_t bytes, int clear) {
  if (!dst || bytes != (int64_t)sizeof(t2d_timeline)) return fail(T2D_E_INVALID, "timeline buffer size");
  CUDA_TRY(cudaMemcpyFromSymbol(dst, t2d_timeline, sizeof(t2d_timeline)));
  if (clear) {
    void* p = nullptr;
    CUDA_TRY(cudaGetSymbolAddress(&p, t2d_timeline));
    CUDA_TRY(cudaMemset(p, 0, sizeof(t2d_timeline)));
  }
  return T2D_OK;
}
#endif

static int check_cfg(const t2d_config* cfg) {
  if (!cfg) return fail(T2D_E_INVALID, "cfg is NULL");
  if (cfg->interval_ms <= 0) return fail(T2D_E_INVALID, "interval_ms must be > 0");
  if (cfg->delta_t_ms <= 0) return fail(T2D_E_INVALID, "delta_t_ms must be > 0");
  return T2D_OK;
}

int t2d_create(t2d_ctx** out, int device, int n_scenarios, int m_participants, const t2d_config* cfg) {
  if (!out) return fail(T2D_E_INVALID, "out is NULL");
  *out = nullptr;
  if (int r = check_cfg(cfg)) return r;
  if (n_scenarios <= 0 || m_participants <= 0) return fail(T2D_E_INVALID, "n_scenarios and m_participants must be > 0");
  if (m_participants > T2D_MAX_PARTICIPANTS)
    return fail(T2D_E_UNSUPPORTED, "m_participants > 128: a scenario must fit one warp (4 participants per lane)");
  int count = 0;
  CUDA_TRY(cudaGetDeviceCount(&count));
  if (device < 0 || device >= count) return fail(T2D_E_INVALID, "no such CUDA device");
  CUDA_TRY(cudaSetDevice(device));
  t2d_ctx* c = new t2d_ctx();
  c->device = device;
  c->N = n_scenarios;
  c->M = m_participants;
  if (const char* e = getenv("T2D_PDL")) c->use_pdl = atoi(e) != 0;
  if (const char* e = getenv("T2D_GRID_LIMIT")) c->grid_limit = std::max(0, atoi(e));
  if (const char* e = getenv("T2D_TICK_GENERIC")) c->tick_generic = atoi(e) != 0;
  if (const char* e = getenv("T2D_PREFETCH")) c->prefetch_override = atoi(e) != 0 ? 1 : 0;
  if (const char* e = getenv("T2D_WPC")) {
    const int v = atoi(e);
    if (v >= 1 && v <= MAX_WARPS_PER_CTA) c->wpc_override = v;
  }
  if (const char* e = getenv("T2D_HOST_CHUNKS")) c->host_chunks = std::max(0, std::min(atoi(e), MAX_HOST_CHUNKS));
  int g = 1;
  while (g * PPL < m_participants) g <<= 1;
  c->G = g;
  c->cfg = *cfg;
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  c->sm_count = prop.multiProcessorCount;
  c->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  {
    std::lock_guard<std::mutex> lock(g_order_mutex);
    unsigned long long*& counters = g_order_fallbacks[device % 64];
    const size_t bytes = ORDER_COUNTERS * ORDER_COUNTER_STRIDE * sizeof(unsigned long long);
    if (!counters && (cudaMalloc(&counters, bytes) != cudaSuccess || cudaMemset(counters, 0, bytes) != cudaSuccess)) {
      cudaFree(counters);
      counters = nullptr;
      delete c;
      return fail(T2D_E_CUDA, "t2d_create: cannot allocate the order fallback counters");
    }
  }
  {
    std::vector<uint8_t> identity((size_t)n_scenarios * FIX_M);
    for (size_t i = 0; i < identity.size(); ++i) identity[i] = (uint8_t)(i % FIX_M);
    if (int r = upload(c->order, identity.data(), identity.size())) {
      delete c;
      return r;
    }
  }
  *out = c;
  return T2D_OK;
}

int t2d_order_hint(t2d_ctx* c, void* read_to, const void* write_from) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  const size_t bytes = (size_t)c->N * FIX_M;
  if (read_to) CUDA_TRY(cudaMemcpy(read_to, c->order.get(), bytes, cudaMemcpyDeviceToHost));
  if (write_from) CUDA_TRY(cudaMemcpy(c->order.get(), write_from, bytes, cudaMemcpyHostToDevice));
  return T2D_OK;
}

int t2d_destroy(t2d_ctx* c) {
  if (!c) return T2D_OK;
  cudaSetDevice(c->device);   // the owners free on the current device
  delete c;
  return T2D_OK;
}

int t2d_set_config(t2d_ctx* c, const t2d_config* cfg) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = check_cfg(cfg)) return r;
  c->cfg = *cfg;
  return T2D_OK;
}

int t2d_set_type_table(t2d_ctx* c, const t2d_type_params* table, int n_types) {
  if (!c || !table) return fail(T2D_E_INVALID, "ctx/table is NULL");
  if (n_types <= 0 || n_types > T2D_MAX_TYPES) return fail(T2D_E_INVALID, "n_types must be in 1..64");
  static_assert(sizeof(t2d_type_params) == sizeof(AbiParams), "type table layout");
  if (c->log)
    for (uint8_t row : c->log->track_type_host)   // a bound log's tracks must stay static rows (K1 would integrate on the log)
      if (row >= n_types || table[row].model != T2D_MODEL_STATIC)
        return fail(T2D_E_INVALID, "type table: row " + std::to_string(row) + " of a replayed track must exist and be T2D_MODEL_STATIC");
  bool has_pointmass = false, has_drift = false, kin_only = true;
  float rb_max = 0.0f;
  for (int i = 0; i < n_types; ++i) {
    const t2d_type_params& p = table[i];
    if (p.shape == T2D_SHAPE_OBB) rb_max = std::max(rb_max, sqrtf(p.half_len * p.half_len + p.half_wid * p.half_wid) * 1.000002f);
    if (p.shape == T2D_SHAPE_CIRCLE) rb_max = std::max(rb_max, p.radius);
    if (p.model < 0 || p.model > T2D_MODEL_DRIFT) return fail(T2D_E_INVALID, "type table: unknown model id");
    if (p.shape < 0 || p.shape > T2D_SHAPE_NONE) return fail(T2D_E_INVALID, "type table: unknown shape id");
    const bool bicycle = p.model <= T2D_MODEL_DYNAMICS || p.model == T2D_MODEL_DRIFT;
    if (bicycle && !(p.lf + p.lr > 0.0f)) return fail(T2D_E_INVALID, "type table: lf + lr must be > 0");
    if (p.model == T2D_MODEL_DYNAMICS && !(p.lf > 0.0f && p.I_z > 0.0f))
      return fail(T2D_E_INVALID, "type table: dynamics needs lf > 0 and I_z > 0");
    if (p.model == T2D_MODEL_DRIFT && !(p.lf > 0.0f && p.I_z > 0.0f && p.mass > 0.0f && p.wheel_radius > 0.0f && p.I_yw > 0.0f))
      return fail(T2D_E_INVALID, "type table: drift needs lf, I_z, mass, wheel_radius and I_yw > 0");
    if (p.model == T2D_MODEL_DRIFT) has_drift = true;
    if (p.shape == T2D_SHAPE_OBB && !(p.half_len >= 0.0f && p.half_wid >= 0.0f))
      return fail(T2D_E_INVALID, "type table: negative OBB half extent");
    if (p.shape == T2D_SHAPE_CIRCLE && !(p.radius >= 0.0f)) return fail(T2D_E_INVALID, "type table: negative radius");
    if (p.model == T2D_MODEL_POINTMASS_NEWTON || p.model == T2D_MODEL_POINTMASS_EULER) has_pointmass = true;
    if (p.model != T2D_MODEL_KINEMATICS && p.model != T2D_MODEL_STATIC) kin_only = false;
  }
  std::vector<Params> rows(n_types + 1);
  for (int i = 0; i < n_types; ++i) {
    AbiParams a;
    memcpy(&a, &table[i], sizeof(AbiParams));
    rows[i] = derive_params(a);
  }
  {
    // row n_types: the neutral kinematic row that K1's 4-chain loop gives to slots holding another model or nothing
    // (zero speed and action in, unbounded ranges: every product stays finite and the result is discarded)
    AbiParams a{};
    a.lf = 1.0f; a.lr = 1.0f;
    a.steer_lo = a.speed_lo = a.accel_lo = -INFINITY;
    a.steer_hi = a.speed_hi = a.accel_hi = INFINITY;
    a.model = MODEL_KINEMATICS; a.shape = SHAPE_NONE;
    rows[n_types] = derive_params(a);
  }
  CUDA_TRY(cudaSetDevice(c->device));
  if (int r = upload(c->d_table, rows.data(), rows.size())) return r;
  c->n_types = n_types;
  c->type_model.resize(n_types);
  for (int i = 0; i < n_types; ++i) c->type_model[i] = table[i].model;
  c->has_pointmass = has_pointmass;
  c->has_drift = has_drift;
  c->rb_max = rb_max;
  c->kin_only = kin_only;
  for (int w = 0; w < 9; ++w) c->occ_smem[w] = -1;
  return T2D_OK;
}
// Host-side build of one static-geometry tile: the segments in list order (+ which of them close up to polygons), a
// uniform grid over their bounding box grown by one cell, per cell the ascending list of the segments that touch it and
// the "dilated" list of those within one cell of it, the clearance fields, the tile's boundary box.
struct TileIn {
  const float* segments; int n_seg;
  const int32_t* poly_start; int n_poly;
  const float* bounds;
};

static bool point_in_ring(const float* seg, int s0, int s1, double px, double py) {   // even-odd over the ring's edges
  bool in = false;
  for (int i = s0; i < s1; ++i) {
    const double x1 = seg[4 * i], y1 = seg[4 * i + 1], x2 = seg[4 * i + 2], y2 = seg[4 * i + 3];
    if ((y1 > py) != (y2 > py) && px < (x2 - x1) * (py - y1) / (y2 - y1) + x1) in = !in;
  }
  return in;
}

static int build_tile(const TileIn& t, float cell_size, float reach, std::vector<unsigned char>& blob) {
  const float* segments = t.segments;
  const int n_seg = t.n_seg;
  if (n_seg < 0 || n_seg > T2D_MAX_SEGMENTS) return fail(T2D_E_INVALID, "n_seg must be in 0..32767");
  if (n_seg > 0 && !segments) return fail(T2D_E_INVALID, "segments is NULL");
  if (t.n_poly < 0 || (t.n_poly > 0 && !t.poly_start)) return fail(T2D_E_INVALID, "poly_start is NULL");
  if (t.bounds && !(t.bounds[0] <= t.bounds[1] && t.bounds[2] <= t.bounds[3])) return fail(T2D_E_INVALID, "bounds must be (xmin<=xmax, ymin<=ymax)");
  for (int p = 0; p < t.n_poly; ++p) {
    const int s0 = t.poly_start[p], s1 = t.poly_start[p + 1];
    if (s0 < 0 || s1 > n_seg || s1 - s0 < 3 || (p > 0 && s0 < t.poly_start[p])) return fail(T2D_E_INVALID, "poly_start: rings must be ascending, inside the segment list and have >= 3 edges");
    // one object = one or more closed rings back to back (an Area's exterior, then its holes): every edge ends where the
    // next one starts, except the edge that returns to its ring's first vertex - the next edge starts the next ring
    int r0 = s0;
    for (int i = s0; i < s1; ++i) {
      if (segments[4 * i + 2] == segments[4 * r0] && segments[4 * i + 3] == segments[4 * r0 + 1]) { r0 = i + 1; continue; }
      if (i + 1 == s1 || segments[4 * i + 2] != segments[4 * (i + 1)] || segments[4 * i + 3] != segments[4 * (i + 1) + 1])
        return fail(T2D_E_INVALID, "poly_start: a ring's edges must chain and close");
    }
  }
  MapHeader mh{};
  mh.n_seg = n_seg; mh.n_poly = t.n_poly;
  mh.has_bounds = t.bounds ? 1 : 0;
  if (t.bounds) { mh.bxmin = t.bounds[0]; mh.bxmax = t.bounds[1]; mh.bymin = t.bounds[2]; mh.bymax = t.bounds[3]; }
  if (n_seg == 0) {   // bounds only
    mh.gx = mh.gy = 0; mh.total_bytes = mh.smem_bytes = mh.off_fine = sizeof(MapHeader);
    blob.assign(sizeof(MapHeader), 0);
    memcpy(blob.data(), &mh, sizeof(mh));
    return T2D_OK;
  }
  float xmin = INFINITY, xmax = -INFINITY, ymin = INFINITY, ymax = -INFINITY;
  for (int i = 0; i < n_seg * 4; ++i)
    if (!std::isfinite(segments[i])) return fail(T2D_E_INVALID, "segments must be finite");
  for (int i = 0; i < n_seg; ++i) {
    const float* s = segments + 4 * i;
    xmin = std::min(xmin, std::min(s[0], s[2])); xmax = std::max(xmax, std::max(s[0], s[2]));
    ymin = std::min(ymin, std::min(s[1], s[3])); ymax = std::max(ymax, std::max(s[1], s[3]));
  }
  const float span = std::max(xmax - xmin, ymax - ymin);
  float cell = cell_size > 0.0f ? cell_size : 8.0f;
  // keep the grid small enough for shared memory: at most 64 x 64 cells over the box grown by one cell (the dilation)
  while (span / cell > 62.0f) cell *= 2.0f;
  // reach of the dilated lists: the largest bounding radius of the type table (as the kernel inflates it) when a table is
  // set - shorter lists in dense maps - else one cell; a participant that reaches further takes the out-of-line walk
  const float dil = reach > 0.0f ? std::min(cell, reach * 1.0002f + 2e-3f) : cell;
  const float margin = 1e-3f * std::max(1.0f, std::max(std::fabs(xmin) + std::fabs(xmax), std::fabs(ymin) + std::fabs(ymax)) * 1e-3f);
  const float x0 = xmin - dil - margin, y0 = ymin - dil - margin;
  const int gx = std::max(1, (int)std::floor((xmax + dil + margin - x0) / cell) + 1);
  const int gy = std::max(1, (int)std::floor((ymax + dil + margin - y0) / cell) + 1);
  const float inv = 1.0f / cell;
  // cells[c] lists (ascending) the segments that pass within `grow` of cell c's box (conservatively: the segment's line
  // against the box grown by `grow` on every side)
  auto bin_segments = [&](float grow) {
    std::vector<std::vector<uint16_t>> cells((size_t)gx * gy);
    for (int i = 0; i < n_seg; ++i) {
      const float* s = segments + 4 * i;
      const float g = grow + margin;
      const float sx0 = std::min(s[0], s[2]) - g, sx1 = std::max(s[0], s[2]) + g;
      const float sy0 = std::min(s[1], s[3]) - g, sy1 = std::max(s[1], s[3]) + g;
      int cx0 = std::max(0, (int)std::floor((sx0 - x0) * inv)), cx1 = std::min(gx - 1, (int)std::floor((sx1 - x0) * inv));
      int cy0 = std::max(0, (int)std::floor((sy0 - y0) * inv)), cy1 = std::min(gy - 1, (int)std::floor((sy1 - y0) * inv));
      for (int cy = cy0; cy <= cy1; ++cy)
        for (int cx = cx0; cx <= cx1; ++cx) {
          // exact-enough cull: does the segment's line pass within the grown cell box?
          const float bx0 = x0 + cx * cell - g, bx1 = x0 + (cx + 1) * cell + g;
          const float by0 = y0 + cy * cell - g, by1 = y0 + (cy + 1) * cell + g;
          const double dx = (double)s[2] - s[0], dy = (double)s[3] - s[1];
          const double hx = 0.5 * ((double)bx1 - bx0), hy = 0.5 * ((double)by1 - by0);
          const double mx = 0.5 * ((double)bx1 + bx0), my = 0.5 * ((double)by1 + by0);
          const double cr = std::fabs(((double)s[0] - mx) * dy - ((double)s[1] - my) * dx);
          if (cr > hx * std::fabs(dy) + hy * std::fabs(dx) + 1e-6 * (std::fabs(dx) + std::fabs(dy) + 1.0)) continue;
          cells[(size_t)cy * gx + cx].push_back((uint16_t)i);
        }
    }
    return cells;
  };
  const std::vector<std::vector<uint16_t>> cells = bin_segments(0.0f);
  // the dilated lists serve participants with reach r <= dil from the cell under their centre: every segment within r
  // of the centre is within dil of that cell's box (+ a 0.1 % + 1 mm guard for the fp32 cell index)
  const std::vector<std::vector<uint16_t>> dcells = bin_segments(dil * 1.001f + 1e-3f);
  size_t n_items = 0, n_ditems = 0;
  for (auto& v : cells) n_items += v.size();
  for (auto& v : dcells) n_ditems += v.size();
  int fine = 4;   // bounded host work: cells x segments <= ~1e8 distance evaluations
  while (fine > 1 && (double)gx * gy * fine * fine * n_seg > 1e8) fine >>= 1;
  mh.gx = gx; mh.gy = gy; mh.n_items = (int)n_items; mh.n_ditems = (int)n_ditems; mh.fine = fine;
  mh.x0 = x0; mh.y0 = y0; mh.inv_cell = inv; mh.cell = cell; mh.dil = dil;
  auto up16 = [](size_t v) { return (v + 15) / 16 * 16; };
  mh.off_seg = (uint32_t)up16(sizeof(MapHeader));
  mh.off_cell = (uint32_t)up16(mh.off_seg + (size_t)n_seg * 16);
  mh.off_items = (uint32_t)up16(mh.off_cell + ((size_t)gx * gy + 1) * 4);
  mh.off_dcell = (uint32_t)up16(mh.off_items + n_items * 2);
  mh.off_ditems = (uint32_t)up16(mh.off_dcell + ((size_t)gx * gy + 1) * 4);
  mh.off_objfirst = (uint32_t)up16(mh.off_ditems + n_ditems * 2);
  mh.off_poly = (uint32_t)up16(mh.off_objfirst + (size_t)n_seg * 2);
  mh.off_pbox = (uint32_t)up16(mh.off_poly + ((size_t)t.n_poly + 1) * 4);
  mh.off_clear = (uint32_t)up16(mh.off_pbox + (size_t)t.n_poly * 16);
  mh.off_fine = (uint32_t)up16(mh.off_clear + (size_t)gx * gy * 4);
  mh.smem_bytes = mh.off_fine;   // the fine field is read through L1 / L2, everything in front of it may be staged
  mh.total_bytes = (uint32_t)up16(mh.off_fine + (size_t)gx * fine * gy * fine);
  blob.assign(mh.total_bytes, 0);
  memcpy(blob.data(), &mh, sizeof(mh));
  memcpy(blob.data() + mh.off_seg, segments, (size_t)n_seg * 16);
  auto write_lists = [&](const std::vector<std::vector<uint16_t>>& lists, uint32_t off_start, uint32_t off_items) {
    uint32_t* cs = reinterpret_cast<uint32_t*>(blob.data() + off_start);
    uint16_t* it = reinterpret_cast<uint16_t*>(blob.data() + off_items);
    uint32_t acc = 0;
    for (size_t ci = 0; ci < lists.size(); ++ci) {
      cs[ci] = acc;
      for (uint16_t sg : lists[ci]) it[acc++] = sg;
    }
    cs[lists.size()] = acc;
  };
  write_lists(cells, mh.off_cell, mh.off_items);
  write_lists(dcells, mh.off_dcell, mh.off_ditems);
  // the object a segment belongs to, named by the object's first segment: an open polyline piece is its own object, the
  // edges of a polygon share the polygon's first edge (StaticCollision.update reports the first OBJECT hit, collision.py:37-43)
  uint16_t* objfirst = reinterpret_cast<uint16_t*>(blob.data() + mh.off_objfirst);
  for (int i = 0; i < n_seg; ++i) objfirst[i] = (uint16_t)i;
  int32_t* pstart = reinterpret_cast<int32_t*>(blob.data() + mh.off_poly);
  float* pbox = reinterpret_cast<float*>(blob.data() + mh.off_pbox);
  for (int p = 0; p < t.n_poly; ++p) {
    const int s0 = t.poly_start[p], s1 = t.poly_start[p + 1];
    pstart[p] = s0;
    float bx0 = INFINITY, bx1 = -INFINITY, by0 = INFINITY, by1 = -INFINITY;
    for (int i = s0; i < s1; ++i) {
      objfirst[i] = (uint16_t)s0;
      bx0 = std::min(bx0, segments[4 * i]); bx1 = std::max(bx1, segments[4 * i]);
      by0 = std::min(by0, segments[4 * i + 1]); by1 = std::max(by1, segments[4 * i + 1]);
    }
    pbox[4 * p] = bx0; pbox[4 * p + 1] = bx1; pbox[4 * p + 2] = by0; pbox[4 * p + 3] = by1;
  }
  pstart[t.n_poly] = t.n_poly > 0 ? t.poly_start[t.n_poly] : 0;
  // clearance fields: lower bound of the distance from any point of a cell to the nearest segment
  // (distance from the cell centre minus the half diagonal); ZERO inside a polygon - a pose deep inside an obstacle
  // touches no edge but intersects the Area all the same.  Coarse (float per cell) and fine (bytes of CLEAR_QUANT metres,
  // fine x fine per coarse cell, read through L1 / L2).
  auto centre_dist = [&](double px, double py) {
    for (int p = 0; p < t.n_poly; ++p)
      if (px >= pbox[4 * p] && px <= pbox[4 * p + 1] && py >= pbox[4 * p + 2] && py <= pbox[4 * p + 3] &&
          point_in_ring(segments, t.poly_start[p], t.poly_start[p + 1], px, py))
        return 0.0;
    double best = INFINITY;
    for (int i = 0; i < n_seg; ++i) {
      const float* sg = segments + 4 * i;
      const double dx = (double)sg[2] - sg[0], dy = (double)sg[3] - sg[1], ux = px - sg[0], uy = py - sg[1];
      const double dd = dx * dx + dy * dy;
      double tt = dd > 0.0 ? (ux * dx + uy * dy) / dd : 0.0;
      tt = std::min(1.0, std::max(0.0, tt));
      const double ex = ux - tt * dx, ey = uy - tt * dy;
      best = std::min(best, ex * ex + ey * ey);
    }
    return std::sqrt(best);
  };
  float* clr = reinterpret_cast<float*>(blob.data() + mh.off_clear);
  {
    const double half_diag = 0.5 * std::sqrt(2.0) * (double)cell * 1.0001 + 2.0 * margin;
    for (int cy = 0; cy < gy; ++cy)
      for (int cx = 0; cx < gx; ++cx) {
        const double d = centre_dist((double)x0 + (cx + 0.5) * (double)cell, (double)y0 + (cy + 0.5) * (double)cell) - half_diag;
        clr[(size_t)cy * gx + cx] = d > 0.0 ? (float)(d * 0.9999) : 0.0f;
      }
  }
  uint8_t* fine_field = blob.data() + mh.off_fine;
  {
    const double fc = (double)cell / fine;
    const double half_diag = 0.5 * std::sqrt(2.0) * fc * 1.001 + 2.0 * margin + 1e-3 * fc;
    for (int iy = 0; iy < gy * fine; ++iy)
      for (int ix = 0; ix < gx * fine; ++ix) {
        const double d = centre_dist((double)x0 + (ix + 0.5) * fc, (double)y0 + (iy + 0.5) * fc) - half_diag;
        const double q = std::floor(std::max(0.0, d) / CLEAR_QUANT);
        fine_field[(size_t)iy * gx * fine + ix] = (uint8_t)std::min(255.0, q);
      }
  }
  return T2D_OK;
}

int t2d_set_map_table(t2d_ctx* c, const t2d_map_tile* tiles, int n_tiles, const uint16_t* tile_id, float cell_size) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (n_tiles < 0 || n_tiles > T2D_MAX_TILES) return fail(T2D_E_INVALID, "n_tiles must be in 0..T2D_MAX_TILES");
  if (n_tiles > 0 && !tiles) return fail(T2D_E_INVALID, "tiles is NULL");
  if (n_tiles > 1 && !tile_id) return fail(T2D_E_INVALID, "tile_id is NULL (needed with more than one tile)");
  DeviceMap m;
  std::vector<unsigned char> all;
  std::vector<uint32_t> offs((size_t)n_tiles);
  for (int i = 0; i < n_tiles; ++i) {
    TileIn t{tiles[i].segments, tiles[i].n_seg, tiles[i].poly_start, tiles[i].n_poly, tiles[i].bounds};
    std::vector<unsigned char> blob;
    if (int r = build_tile(t, cell_size, c->rb_max, blob)) return r;
    offs[i] = (uint32_t)all.size();
    all.insert(all.end(), blob.begin(), blob.end());
    all.resize((all.size() + 127) / 128 * 128, 0);   // every tile starts 128-byte aligned
    m.has_bounds = m.has_bounds || tiles[i].bounds != nullptr;
    m.has_segments = m.has_segments || tiles[i].n_seg > 0;
    m.tile_nseg.push_back(tiles[i].n_seg);
    if (i == 0) memcpy(&m.mh, blob.data(), sizeof(MapHeader));
  }
  CUDA_TRY(cudaSetDevice(c->device));
  if (n_tiles > 0) {
    if (int r = upload(m.blob, all.data(), all.size())) return r;
    if (int r = upload(m.tile_off, offs.data(), offs.size())) return r;
  }
  m.n_tiles = n_tiles;
  m.tile_id = n_tiles > 1 ? tile_id : nullptr;
  m.smem_bytes = (int)m.mh.smem_bytes;   // what a single tile stages into shared memory
  c->map = std::move(m);
  return T2D_OK;
}

int t2d_set_map_polygons(t2d_ctx* c, const float* segments, int n_seg, const int32_t* poly_start, int n_poly, const float* bounds,
                         float cell_size) {
  if (n_seg == 0 && !bounds) return t2d_set_map_table(c, nullptr, 0, nullptr, cell_size);
  t2d_map_tile t{};
  t.segments = segments; t.n_seg = n_seg; t.poly_start = poly_start; t.n_poly = n_poly; t.bounds = bounds;
  return t2d_set_map_table(c, &t, 1, nullptr, cell_size);
}

int t2d_set_map(t2d_ctx* c, const float* segments, int n_seg, const float* bounds, float cell_size) {
  return t2d_set_map_polygons(c, segments, n_seg, nullptr, 0, bounds, cell_size);
}

int t2d_bind_state(t2d_ctx* c, float* x, float* y, float* heading, float* speed, float* vx, float* vy,
                   const uint8_t* type_id, int32_t* step_count) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!x || !y || !heading || !speed || !vx || !vy || !type_id || !step_count)
    return fail(T2D_E_INVALID, "t2d_bind_state: NULL array");
  c->x = x; c->y = y; c->h = heading; c->v = speed; c->vx = vx; c->vy = vy;
  c->type_id = type_id; c->step_count = step_count;
  return T2D_OK;
}

int t2d_bind_wheel_state(t2d_ctx* c, float* omega_front, float* omega_rear) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if ((omega_front == nullptr) != (omega_rear == nullptr)) return fail(T2D_E_INVALID, "t2d_bind_wheel_state: one array is NULL");
  c->wheel_f = omega_front; c->wheel_r = omega_rear;
  return T2D_OK;
}

int t2d_bind_reset_wheel_pool(t2d_ctx* c, const float* pool_omega_front, const float* pool_omega_rear) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if ((pool_omega_front == nullptr) != (pool_omega_rear == nullptr)) return fail(T2D_E_INVALID, "t2d_bind_reset_wheel_pool: one array is NULL");
  c->reset_pool_wf = pool_omega_front; c->reset_pool_wr = pool_omega_rear;
  return T2D_OK;
}

// t2d_set_log (row_track, slot_off == nullptr) and t2d_set_log_schedule: validate everything, then replace the bound log.
// A row_track binding becomes a schedule of at most one entry per slot.
static int set_log(t2d_ctx* c, const t2d_log* L, const char* who, const int32_t* slot_off, const int32_t* slot_track,
                   int n_entries, int32_t* track_out) {
  const std::string fn = who;
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (L->n_tracks <= 0 || L->n_rows <= 0) return fail(T2D_E_INVALID, fn + ": n_tracks and n_rows must be >= 1");
  if (!L->first_ms || !L->n_frames || !L->period_ms || !L->type_row || !L->records || !L->t0_ms || !L->log_row || !L->type_id)
    return fail(T2D_E_INVALID, fn + ": NULL array");
  if (slot_off == nullptr && !L->row_track) return fail(T2D_E_INVALID, fn + ": NULL array");
  if (slot_off != nullptr && L->row_track) return fail(T2D_E_INVALID, fn + ": row_track must be NULL (the schedule binds the slots)");
  if (L->type_id != c->type_id)
    return fail(T2D_E_INVALID, fn + ": type_id is not the array bound with t2d_bind_state");
  const int K = L->n_tracks, M = c->M;
  const long long PM = (long long)L->n_rows * M;
  std::vector<ReplayTrack> tracks((size_t)K);
  std::vector<long long> last((size_t)K);
  long long n_rec = 0;
  for (int k = 0; k < K; ++k) {
    if (L->period_ms[k] <= 0) return fail(T2D_E_INVALID, fn + ": track " + std::to_string(k) + ": period_ms must be > 0");
    if (L->n_frames[k] < 1) return fail(T2D_E_INVALID, fn + ": track " + std::to_string(k) + ": no frames");
    const int row = L->type_row[k];
    if (row >= c->n_types) return fail(T2D_E_INVALID, fn + ": track " + std::to_string(k) + ": type_row outside the type table");
    if (c->type_model[row] != T2D_MODEL_STATIC)
      return fail(T2D_E_INVALID, fn + ": track " + std::to_string(k) + ": type_row is not a T2D_MODEL_STATIC row");
    tracks[k] = ReplayTrack{L->first_ms[k], L->period_ms[k], L->n_frames[k], (int32_t)n_rec};
    last[k] = (long long)L->first_ms[k] + (long long)(L->n_frames[k] - 1) * L->period_ms[k];
    n_rec += L->n_frames[k];
    if (n_rec > INT32_MAX / 5) return fail(T2D_E_UNSUPPORTED, fn + ": too many records");
  }
  for (long long i = 0; i < 5 * n_rec; ++i)
    if (!std::isfinite(L->records[i])) return fail(T2D_E_INVALID, fn + ": record " + std::to_string(i / 5) + " is not finite");
  std::vector<int32_t> off((size_t)PM + 1, 0);
  std::vector<ReplayEntry> entries;
  std::vector<int> seen((size_t)K, -1);
  if (slot_off == nullptr) {
    for (int p = 0; p < L->n_rows; ++p)
      for (int m = 0; m < M; ++m) {
        const long long s = (long long)p * M + m;
        const int k = L->row_track[s];
        if (k < -1 || k >= K) return fail(T2D_E_INVALID, fn + ": row_track entry outside [-1, n_tracks)");
        if (k >= 0) {
          if (seen[k] == p) return fail(T2D_E_INVALID, fn + ": track " + std::to_string(k) + " bound twice in row " + std::to_string(p));
          seen[k] = p;
          // a slot's final entry is never probed: its last stamp only has to be an int32, not exact
          entries.push_back(ReplayEntry{(int32_t)std::min<long long>(last[k], INT32_MAX), k});
        }
        off[s + 1] = (int32_t)entries.size();
      }
  } else {
    if (!slot_track && n_entries > 0) return fail(T2D_E_INVALID, fn + ": NULL array");
    if (n_entries < 0) return fail(T2D_E_INVALID, fn + ": n_entries must be >= 0");
    if (slot_off[0] != 0 || slot_off[PM] != n_entries)
      return fail(T2D_E_INVALID, fn + ": slot_off must run from 0 to n_entries");
    for (long long s = 0; s < PM; ++s)
      if (slot_off[s + 1] < slot_off[s]) return fail(T2D_E_INVALID, fn + ": slot_off is not monotone at slot " + std::to_string(s));
    entries.resize((size_t)n_entries);
    for (int p = 0; p < L->n_rows; ++p)
      for (int m = 0; m < M; ++m) {
        const long long s = (long long)p * M + m;
        for (int e = slot_off[s]; e < slot_off[s + 1]; ++e) {
          const int k = slot_track[e];
          const std::string at = fn + ": row " + std::to_string(p) + " slot " + std::to_string(m) + ": ";
          if (k < 0 || k >= K) return fail(T2D_E_INVALID, at + "slot_track entry outside [0, n_tracks)");
          if (seen[k] == p) return fail(T2D_E_INVALID, at + "track " + std::to_string(k) + " scheduled twice in the row");
          seen[k] = p;
          if (e > slot_off[s] && (long long)L->first_ms[k] <= last[slot_track[e - 1]])
            return fail(T2D_E_INVALID, at + "track " + std::to_string(k) + " does not start after the previous entry ends");
          if (last[k] > INT32_MAX) return fail(T2D_E_UNSUPPORTED, at + "track " + std::to_string(k) + ": last stamp exceeds int32 ms");
          entries[e] = ReplayEntry{(int32_t)last[k], k};
        }
      }
    std::copy(slot_off, slot_off + PM + 1, off.begin());
  }
  // at most one entry per slot (every row_track binding): the slots' tracks as one array, no search
  bool single = true;
  for (long long s = 0; s < PM && single; ++s) single = off[s + 1] - off[s] <= 1;
  CUDA_TRY(cudaSetDevice(c->device));
  auto g = std::make_unique<DeviceLog>();
  if (single) {
    std::vector<int32_t> one((size_t)PM, -1);
    for (long long s = 0; s < PM; ++s)
      if (off[s + 1] > off[s]) one[s] = entries[off[s]].track;
    if (int r = upload(g->slot_track1, one.data(), one.size())) return r;
  } else {
    if (int r = upload(g->slot_off, off.data(), off.size())) return r;
    if (int r = upload(g->entries, entries.data(), entries.size())) return r;
  }
  if (int r = upload(g->tracks, tracks.data(), tracks.size())) return r;
  if (int r = upload(g->track_type, L->type_row, (size_t)K)) return r;
  if (int r = upload(g->rec, L->records, 5 * (size_t)n_rec)) return r;
  if (int r = upload(g->t0, L->t0_ms, (size_t)L->n_rows)) return r;
  g->track_type_host.assign(L->type_row, L->type_row + K);
  g->n_tracks = K; g->n_rows = L->n_rows;
  g->row = L->log_row; g->type_id = L->type_id; g->track_out = track_out;
  if (c->hist) {   // the ring's tracks restart with the log (a rejected call keeps both as they were)
    DeviceHistory tracks;
    tracks.H = c->hist->H;
    if (int r = history_tracks(c, tracks, track_out)) return r;
    c->hist->track = std::move(tracks.track);
  }
  c->log = std::move(g);
  return T2D_OK;
}

int t2d_set_log(t2d_ctx* c, const t2d_log* L) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!L) {
    CUDA_TRY(cudaSetDevice(c->device));
    c->log.reset();
    if (c->hist) c->hist->track.reset();
    return T2D_OK;
  }
  return set_log(c, L, "t2d_set_log", nullptr, nullptr, 0, nullptr);
}

int t2d_set_log_schedule(t2d_ctx* c, const t2d_log* L, const int32_t* slot_off, const int32_t* slot_track, int32_t n_entries,
                         int32_t* track_out) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!L || !slot_off) return fail(T2D_E_INVALID, "t2d_set_log_schedule: log / slot_off is NULL (t2d_set_log(ctx, NULL) unbinds)");
  return set_log(c, L, "t2d_set_log_schedule", slot_off, slot_track, n_entries, track_out);
}

// K7 over the scenarios [first, first + count): tick mode (mask == nullptr, offset 1) or reset mode (the masked scenarios
// take row pool_index[n] / n, offset 0).
static int launch_replay(t2d_ctx* c, void* stream, int first, int count, int offset, const uint8_t* mask, const int32_t* pool_index) {
  const DeviceLog& g = *c->log;
  if (g.type_id != c->type_id) return fail(T2D_E_STATE, "state rebound after t2d_set_log: call t2d_set_log again");
  const size_t p0 = (size_t)first * c->M;
  ReplayArgs R{};
  R.x = c->x + p0; R.y = c->y + p0; R.h = c->h + p0; R.v = c->v + p0; R.vx = c->vx + p0; R.vy = c->vy + p0;
  R.type_id = g.type_id + p0;
  R.step_count = c->step_count + first;
  R.log_row = g.row + first;
  R.mask = mask ? mask + first : nullptr;
  R.pool_index = pool_index ? pool_index + first : nullptr;
  R.log_row_out = mask ? g.row + first : nullptr;
  R.tracks = g.tracks.get(); R.track_type = g.track_type.get(); R.rec = g.rec.get();
  R.t0 = g.t0.get(); R.slot_off = g.slot_off.get(); R.entries = g.entries.get(); R.slot_track1 = g.slot_track1.get();
  R.track_out = g.track_out ? g.track_out + p0 : nullptr;
  R.N = count; R.M = c->M; R.n_rows = g.n_rows; R.offset = offset; R.interval_ms = c->cfg.interval_ms;
  t2d_replay_kernel<<<capped_grid((long long)count * c->M, 256, c->sm_count, 8), 256, 0, (cudaStream_t)stream>>>(R);
  return launched();
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Warps per CTA of the tick.  One wave (the usual case: every warp tile is resident at once and the kernel's duration is
// one tile's lifetime): the SM with the most warps sets the pace, and every CTA costs a launch + prologue (barrier
// init, TMA staging), weighed below as 0.42 of a warp on the fullest SM (1-warp CTAs are not considered: the prologue
// is paid per warp there).  Several waves: persistent CTAs of the largest size.  On an H100 (132 SMs) 4096 x 64 is 2048 warp
// tiles, more than the conservative 132 x 14, so it takes 8-warp CTAs; at the launch bounds' 2 CTAs per SM all 256 of them are
// resident at once anyway (one wave).  On an H100 80GB HBM3 SXM at a 400 W power limit (T2D_WPC, 40000 timed steps) 8 and 4 warps
// per CTA measured within 2 % of each other and 2 warps per CTA about 45 % slower.
static int pick_wpc(long long tiles, int sm_count) {
  const int resident_warps = 14;   // per SM at the kernel's register budget, rounded down to what every variant reaches
  if (tiles > (long long)sm_count * resident_warps) return MAX_WARPS_PER_CTA;
  int best = 2;
  double best_cost = 1e30;
  for (int w = 2; w <= MAX_WARPS_PER_CTA; ++w) {
    const long long ctas = (tiles + w - 1) / w;
    const long long per_sm = (ctas + sm_count - 1) / sm_count;
    const double cost = (double)(per_sm * w) + 0.42 * (double)per_sm;
    if (cost < best_cost - 1e-9 || (cost < best_cost + 1e-9 && w > best)) { best_cost = cost; best = w; }
  }
  return best;
}

// Launches K1 over the scenarios [first, first + count) of the bound state with the ego action `ego` (nullptr: row 0 of
// `action`); the per-participant / per-scenario pointers passed in (action, flags, ..., done) address scenario `first`
// already, `ego` scenario 0.
static int launch_step(t2d_ctx* c, const float* action, const float* ego, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment,
                       uint8_t* scn_status, uint8_t* done, void* stream, int do_physics, int first = 0, int count = -1) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (do_physics && !action) return fail(T2D_E_INVALID, "action is NULL");
  if (do_physics)
    if (int r = require(c, NEED_TICK)) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  if (count < 0) count = c->N - first;
  if (first < 0 || count <= 0 || first + count > c->N) return fail(T2D_E_INVALID, "scenario range out of bounds");
  const DeviceMap& map = c->map;
  const size_t p0 = (size_t)first * c->M;
  StepArgs A{};
  A.x = c->x + p0; A.y = c->y + p0; A.h = c->h + p0; A.v = c->v + p0; A.vx = c->vx + p0; A.vy = c->vy + p0;
  A.type_id = c->type_id + p0; A.step_count = c->step_count + first;
  A.wheel_f = c->wheel_f ? c->wheel_f + p0 : nullptr; A.wheel_r = c->wheel_r ? c->wheel_r + p0 : nullptr;
  A.action = action; A.ego_action = ego ? ego + 2 * (size_t)first : nullptr; A.flags = flags; A.hit_index = hit_index; A.hit_segment = hit_segment;
  A.scn_status = scn_status; A.done = done;
  A.order = c->order.get() + (size_t)first * FIX_M;
  A.order_fallbacks = g_order_fallbacks[c->device % 64];
  const bool map_table = map.n_tiles > 1;
  const MapArgs mp = map_args(map, first);
  A.map_blob = mp.map_blob; A.tile_off = mp.tile_off; A.tile_id = mp.tile_id; A.map_bytes = map.smem_bytes; A.mh = map.mh;
  A.map_in_smem = (!map_table && map.blob && map.mh.n_seg > 0 && map.smem_bytes <= MAP_SMEM_LIMIT) ? 1 : 0;
  A.table = c->d_table.get(); A.n_types = c->n_types;
  A.N = count; A.M = c->M; A.G = c->G;
  set_time_step(A, c->cfg.interval_ms, c->cfg.delta_t_ms);
  A.max_step = c->cfg.max_step; A.cfg_flags = c->cfg.flags;
  // the boundary box: tile 0's (with a map table every lane reads its own tile's)
  A.do_physics = do_physics; A.has_bounds = map.has_bounds ? 1 : 0;
  A.bxmin = map.mh.bxmin; A.bxmax = map.mh.bxmax; A.bymin = map.mh.bymin; A.bymax = map.mh.bymax;
  A.prefetch = c->prefetch_override >= 0 ? c->prefetch_override : (g_exchanges_alive.load() == 0 ? 1 : 0);
  // (drift / replay: K1 passes the pre-pass's vx, vy through)
  A.needs_vel_in = (c->has_pointmass || c->has_drift || (do_physics && c->log)) ? 1 : 0;
  bool vec = (c->M % PPL == 0) && aligned16(A.x) && aligned16(A.y) && aligned16(A.h) && aligned16(A.v) && aligned16(A.vx) &&
             aligned16(A.vy) && (reinterpret_cast<uintptr_t>(A.type_id) % 4 == 0) && (!action || aligned16(action)) &&
             (!flags || reinterpret_cast<uintptr_t>(flags) % 4 == 0) && (!hit_index || reinterpret_cast<uintptr_t>(hit_index) % 8 == 0) &&
             (!hit_segment || reinterpret_cast<uintptr_t>(hit_segment) % 8 == 0);
  A.vec_ok = vec ? 1 : 0;

  A.rb_max = c->rb_max;
  A.goal = c->goal;
  if (A.goal.target) {   // the rows from `first` on (t2d_set_goal binds the three outputs with every target)
    A.goal.target += 5 * (size_t)first; A.goal.iou += first; A.goal.last_pose += 4 * (size_t)first; A.goal.noact_count += first;
  }
  const int table_bytes = (((c->n_types + 1) * (int)sizeof(Params) + 15) / 16) * 16;   // + the neutral row
  const int spw = 32 / c->G;
  const long long tiles = ((long long)count + spw - 1) / spw;
  int wpc = pick_wpc(tiles, c->sm_count);
  if (c->wpc_override > 0) wpc = c->wpc_override;   // T2D_WPC (experiments), read once at t2d_create
  {
    int off = (A.map_in_smem ? A.map_bytes : 0) + table_bytes;
    A.off_poseA = off; off += wpc * POSE_PER_WARP * (int)sizeof(float4);
    A.off_poseB = off; off += wpc * POSE_PER_WARP * (int)sizeof(float4);
    A.off_hit = off; off += wpc * POSE_PER_WARP * (int)sizeof(int);
    A.off_queue = off; off += wpc * QCAP * 4;
    A.off_sorted = off; off += wpc * POSE_PER_WARP * (int)sizeof(float4);
    A.off_qcount = off; off += ((wpc + 3) & ~3) * 4;
    A.off_bar = off; off += 16;
    A.wpc = wpc;
    A.table_bytes = table_bytes;
    A.n_tiles = (int)tiles;
    A.g_shift = 0;
    while ((1 << A.g_shift) < c->G) ++A.g_shift;
    const int MP = c->G * PPL;
    A.mp_shift = 0;
    while ((1 << A.mp_shift) < MP) ++A.mp_shift;
  }
  const int smem = A.off_bar + 16;
  if (smem > c->max_smem_optin) return fail(T2D_E_UNSUPPORTED, "shared memory budget exceeded");
  using kernel_t = void (*)(StepArgs);
  kernel_t kern;
  // the C2-shaped instance exactly when this tick has the shape it is compiled for (FIX_M ...)
  const bool fixed = c->kin_only && !c->tick_generic && c->M == FIX_M && c->G == FIX_G && do_physics && A.vec_ok &&
                     !A.needs_vel_in && A.ego_action == nullptr && A.goal.target == nullptr;
  if (fixed) kern = map_table ? (kernel_t)t2d_step_kernel<true, true, true> : (kernel_t)t2d_step_kernel<true, false, true>;
  else if (c->kin_only) kern = map_table ? (kernel_t)t2d_step_kernel<true, true, false> : (kernel_t)t2d_step_kernel<true, false, false>;
  else kern = map_table ? (kernel_t)t2d_step_kernel<false, true, false> : (kernel_t)t2d_step_kernel<false, false, false>;
  const int variant = (fixed ? 4 : c->kin_only ? 2 : 0) + (map_table ? 1 : 0);
  {
    // cudaFuncSetAttribute applies to the kernel function for the whole process and SETS the value: worlds of
    // different sizes share it, so the opt-in is tracked per (device, kernel variant) and only ever raised.
    std::lock_guard<std::mutex> lock(g_smem_mutex);
    int& configured = g_smem_configured[c->device % 64][variant];
    if (smem > configured) {
      CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      configured = smem;
    }
  }
  if (do_physics && c->log)
    if (int r = launch_replay(c, stream, first, count, 1, nullptr, nullptr)) return r;
  if (do_physics && c->has_drift) {
    t2d_drift_kernel<<<capped_grid((long long)count * c->M, 128, c->sm_count, 16), 128, 0, (cudaStream_t)stream>>>(A);
    if (int r = launched()) return r;
  }
  const long long ctas_needed = (tiles + wpc - 1) / wpc;
  if (c->occ_smem[wpc] != smem || c->occ_variant[wpc] != variant) {
    int per_sm = 1;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, wpc * 32, smem));
    c->occ_val[wpc] = per_sm < 1 ? 1 : per_sm;
    c->occ_smem[wpc] = smem;
    c->occ_variant[wpc] = variant;
  }
  int per_sm_ctas = c->occ_val[wpc];
  if (c->grid_limit > 0) per_sm_ctas = std::min(per_sm_ctas, c->grid_limit);   // T2D_GRID_LIMIT: leave CTA slots to other streams
  const long long resident = (long long)c->sm_count * per_sm_ctas;
  const int grid = (int)std::max(1LL, std::min(ctas_needed, resident));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3((unsigned)(wpc * 32));
  cfg.dynamicSmemBytes = (size_t)smem;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = c->use_pdl ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, A));
  if (int r = launched()) return r;
  g_tick_instances[variant].fetch_add(1);
  if (!map_table && map.blob && map.mh.n_seg > 0 && !A.map_in_smem) g_tick_instances[6].fetch_add(1);
  return T2D_OK;
}

// K5 with the ego action `ego` (nullptr: row 0 of `action`)
// A call K5 could not complete is refused before anything is launched: PID rows without their state or target.
static int check_pid_binding(const t2d_ctx* c) {
  if (!c->ctrl_has_pid) return T2D_OK;
  if (!c->pid_state) return fail(T2D_E_INVALID, "a PID controller row is bound without its state: call t2d_set_pid first");
  if (c->ctrl_pid_reads_target && !c->pid_target)
    return fail(T2D_E_INVALID, "a PID controller row reads the target, and none is bound: call t2d_set_pid with one");
  return T2D_OK;
}

static int launch_control(t2d_ctx* c, float* action, const float* ego, void* stream) {
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (!c->d_ctab) return fail(T2D_E_STATE, "controllers not set: call t2d_set_controllers first");
  if (int r = check_pid_binding(c)) return r;
  if (!action) return fail(T2D_E_INVALID, "action is NULL");
  if (reinterpret_cast<uintptr_t>(action) % 8 != 0) return fail(T2D_E_INVALID, "action must be 8-byte aligned");
  CUDA_TRY(cudaSetDevice(c->device));
  CtrlArgs A{world_args(c)};
  A.ctab = c->d_ctab.get(); A.n_ctrl = c->n_ctrl; A.ctrl_id = c->ctrl_id; A.lead = c->ctrl_lead; A.path_id = c->ctrl_path;
  A.path_v = c->d_path_v.get(); A.path_off = c->d_path_off.get(); A.n_paths = c->n_paths;
  A.last_accel = c->ctrl_last_accel; A.action = action; A.ego_action = ego;
  A.steer_first = (c->cfg.flags & T2D_CFG_STEER_FIRST) ? 1 : 0;
  A.pid_target = c->pid_target; A.pid_state = c->pid_state;
  const int warps_per_cta = 4;
  auto kern = c->ctrl_has_pid ? t2d_control_kernel<true> : t2d_control_kernel<false>;
  kern<<<capped_grid(c->N, warps_per_cta, c->sm_count, 16), warps_per_cta * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

struct HostPart {   // a part of a packed read-back that goes to a caller's array (dst == nullptr: not wanted)
  void* dst;
  size_t off, bytes;
};

// Copies the first `bytes` of a packed device block to its pinned mirror, waits for the stream, and copies the parts out
static int read_back(const Mirror& m, size_t bytes, cudaStream_t s, std::initializer_list<HostPart> parts) {
  CUDA_TRY(cudaMemcpyAsync(m.host.get(), m.dev.get(), bytes, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (const HostPart& p : parts)
    if (p.dst) memcpy(p.dst, m.host.get() + p.off, p.bytes);
  return T2D_OK;
}

static int make_mirror(Mirror& out, size_t dev_bytes, size_t host_bytes) {
  Mirror m;
  if (int r = dev_alloc(m.dev, dev_bytes)) return r;
  if (int r = host_alloc(m.host, host_bytes)) return r;
  out = std::move(m);
  return T2D_OK;
}

// the [2][N] status / done block of t2d_step_host and t2d_step_host_ego
static int status_done_staging(t2d_ctx* c) {
  return c->hs_out.dev ? T2D_OK : make_mirror(c->hs_out, 2 * (size_t)c->N, 2 * (size_t)c->N);
}

int t2d_set_goal(t2d_ctx* c, const float* target, float arrival_threshold, int no_action_max_step, float* iou_out, float* last_pose,
                 int32_t* no_action_count) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (target && (!iou_out || !last_pose || !no_action_count)) return fail(T2D_E_INVALID, "t2d_set_goal: NULL output array");
  if (target && !(arrival_threshold > 0.0f && arrival_threshold <= 1.0f)) return fail(T2D_E_INVALID, "arrival_threshold must be in (0, 1]");
  c->goal = {target, iou_out, last_pose, no_action_count, arrival_threshold, no_action_max_step};
  return T2D_OK;
}

int t2d_step(t2d_ctx* c, const float* action, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment, uint8_t* scn_status,
             uint8_t* done, void* stream) {
  if (int r = launch_step(c, action, c ? c->ego_action : nullptr, flags, hit_index, hit_segment, scn_status, done, stream, 1))
    return r;
  return launch_history(c, nullptr, stream);
}

int t2d_step_host(t2d_ctx* c, const float* action_host, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment,
                  uint8_t* scn_status_host, uint8_t* done_host, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!action_host) return fail(T2D_E_INVALID, "action is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  const int N = c->N, M = c->M;
  if (!c->hs_upload) {
    auto u = std::make_unique<ChunkedUpload>();
    if (int r = dev_alloc(u->action, (size_t)N * M * 2)) return r;
    CUDA_TRY(cudaStreamCreateWithFlags(&u->copy, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&u->begin, cudaEventDisableTiming));
    for (cudaEvent_t& e : u->chunk) CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    c->hs_upload = std::move(u);
  }
  if (int r = status_done_staging(c)) return r;
  ChunkedUpload& u = *c->hs_upload;
  uint8_t* out = c->hs_out.dev.get();
  // Chunks of whole scenarios: the copy of chunk k + 1 (copy engine, own stream) runs under the kernel of chunk k.
  // A kernel that does not fill the GPU lasts one tile's lifetime whatever the batch, so splitting a small upload only
  // adds a fixed cost per chunk; it pays once a chunk alone fills the GPU, i.e. from ~1 M participants (8 MiB of
  // actions) per chunk upwards.
  int chunks = c->host_chunks;
  if (chunks <= 0) chunks = (int)std::min<long long>(MAX_HOST_CHUNKS, std::max<long long>(1, (long long)N * M / (1 << 20)));
  int per = (N + chunks - 1) / chunks;
  per = (per + 31) & ~31;   // whole warp tiles (<= 32 scenarios per warp): a chunked tick groups lanes exactly as t2d_step does
  cudaStream_t s = (cudaStream_t)stream;
  const bool split = per < N;   // a single chunk needs no second stream
  if (split) {
    CUDA_TRY(cudaEventRecord(u.begin, s));            // the copies follow whatever the caller queued on `stream`
    CUDA_TRY(cudaStreamWaitEvent(u.copy, u.begin, 0));
  }
  int k = 0;
  for (int first = 0; first < N; first += per, ++k) {
    const int count = std::min(per, N - first);
    const size_t a0 = (size_t)first * M * 2;
    CUDA_TRY(cudaMemcpyAsync(u.action.get() + a0, action_host + a0, (size_t)count * M * 2 * sizeof(float), cudaMemcpyHostToDevice,
                             split ? u.copy : s));
    if (split) {
      CUDA_TRY(cudaEventRecord(u.chunk[k], u.copy));
      CUDA_TRY(cudaStreamWaitEvent(s, u.chunk[k], 0));
    }
    const size_t p0 = (size_t)first * M;
    if (int r = launch_step(c, u.action.get() + a0, c->ego_action, flags ? flags + p0 : nullptr, hit_index ? hit_index + p0 : nullptr,
                            hit_segment ? hit_segment + p0 : nullptr, out + first, out + N + first, stream, 1, first, count))
      return r;
  }
  if (int r = launch_history(c, nullptr, stream)) return r;   // after the last chunk
  return read_back(c->hs_out, 2 * (size_t)N, s, {{scn_status_host, 0, (size_t)N}, {done_host, (size_t)N, (size_t)N}});
}

int t2d_set_prefetch(t2d_ctx* c, int mode) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (mode < -1 || mode > 1) return fail(T2D_E_INVALID, "prefetch mode must be -1 (policy), 0 (off) or 1 (on)");
  c->prefetch_override = mode;
  return T2D_OK;
}

int t2d_set_ego_action(t2d_ctx* c, const float* ego_action) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (ego_action && reinterpret_cast<uintptr_t>(ego_action) % 8 != 0) return fail(T2D_E_INVALID, "ego_action must be 8-byte aligned");
  c->ego_action = ego_action;
  return T2D_OK;
}

int t2d_step_host_ego(t2d_ctx* c, const float* ego_action_host, float* action, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment,
                      uint8_t* scn_status_host, uint8_t* done_host, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!ego_action_host || !action) return fail(T2D_E_INVALID, "ego_action / action is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  const int N = c->N;
  if (!c->hs_ego.host) {
    // pinned AND mapped: the first kernel of the step reads the 8 N bytes straight from host memory (one PCIe round trip
    // inside the kernel) instead of waiting for a copy-engine transfer and the stream dependency behind it
    MappedEgo e;
    if (int r = host_alloc(e.host, (size_t)N * 2, cudaHostAllocMapped)) return r;
    float* dev = nullptr;
    CUDA_TRY(cudaHostGetDevicePointer(&dev, e.host.get(), 0));
    e.dev = dev;
    c->hs_ego = std::move(e);
  }
  if (int r = status_done_staging(c)) return r;
  if (c->d_ctab)
    if (int r = check_pid_binding(c)) return r;
  memcpy(c->hs_ego.host.get(), ego_action_host, (size_t)N * 2 * sizeof(float));
  const float* ego = c->hs_ego.dev;
  if (c->d_ctab) {
    // the controllers' launch fetches the ego actions and writes them into row 0 of `action`; the other participants'
    // actions never leave the device; the tick then reads everything from `action`
    if (int r = launch_control(c, action, ego, stream)) return r;
    ego = nullptr;
  }
  uint8_t* out = c->hs_out.dev.get();
  if (int r = launch_step(c, action, ego, flags, hit_index, hit_segment, out, out + N, stream, 1)) return r;
  if (int r = launch_history(c, nullptr, stream)) return r;
  return read_back(c->hs_out, 2 * (size_t)N, (cudaStream_t)stream,
                   {{scn_status_host, 0, (size_t)N}, {done_host, (size_t)N, (size_t)N}});
}

int t2d_env_epilogue(t2d_ctx* c, const uint8_t* flags, const uint8_t* scn_status, float* reward, uint8_t* terminated,
                     uint8_t* truncated, uint8_t* traffic_status, uint8_t* done, float* max_iou, float* min_dist,
                     int reset_trackers_on_done, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE)) return r;
  if (!flags || !scn_status || !reward) return fail(T2D_E_INVALID, "t2d_env_epilogue: flags / scn_status / reward is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  EnvArgs A{world_args(c)};
  A.flags = flags; A.status = scn_status;
  A.iou = c->goal.target ? c->goal.iou : nullptr; A.target = c->goal.target;
  A.max_iou = max_iou; A.min_dist = min_dist;
  A.reward = reward; A.terminated = terminated; A.truncated = truncated; A.done = done; A.traffic_status = traffic_status;
  A.max_step = c->cfg.max_step; A.reset_trackers = reset_trackers_on_done ? 1 : 0;
  A.route = route_args(c); A.s_best = c->route_id ? c->route_s_best : nullptr;
  t2d_env_epilogue_kernel<<<capped_grid((long long)c->N * c->M, 256, c->sm_count, 8), 256, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_set_agents(t2d_ctx* c, const int16_t* observers, int32_t n_observers, const float* goals, float arrival_threshold,
                   int no_action_max_step, float* last_pose, int32_t* noact_count, uint8_t* retired_type) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!observers && n_observers == 0) {   // unbind
    c->agent_q = 0; c->agent_observers = nullptr; c->agent = {}; c->agent_retired = nullptr;
    return T2D_OK;
  }
  if (n_observers < 1 || n_observers > T2D_OBS_MAX_OBSERVERS) return fail(T2D_E_INVALID, "t2d_set_agents: n_observers must be in 1..128");
  if (!observers && n_observers > c->M) return fail(T2D_E_INVALID, "t2d_set_agents: without observers row q is slot q (n_observers <= M)");
  if (!last_pose || !noact_count || !retired_type) return fail(T2D_E_INVALID, "t2d_set_agents: NULL state array");
  if (goals && !(arrival_threshold > 0.0f && arrival_threshold <= 1.0f)) return fail(T2D_E_INVALID, "arrival_threshold must be in (0, 1]");
  c->agent_q = n_observers; c->agent_observers = observers; c->agent_retired = retired_type;
  c->agent = {goals, nullptr, last_pose, noact_count, arrival_threshold, no_action_max_step};
  return T2D_OK;
}

int t2d_agents_epilogue(t2d_ctx* c, const uint8_t* flags, float* reward, uint8_t* terminated, uint8_t* truncated,
                        uint8_t* agent_status, float* iou, uint8_t* done, float* max_iou, float* min_dist, uint8_t* traffic_status,
                        int reset_trackers_on_done, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (c->agent_q == 0) return fail(T2D_E_STATE, "t2d_agents_epilogue: no agents bound: call t2d_set_agents first");
  if (!flags || !reward || !terminated || !truncated || !agent_status || !iou || !done || !max_iou || !min_dist)
    return fail(T2D_E_INVALID, "t2d_agents_epilogue: NULL array");
  if (int r = check_route_trackers(c, "t2d_agents_epilogue")) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  AgentArgs A{world_args(c)};
  A.route = route_args(c); A.s_best = c->route_id ? c->route_agent_s_best : nullptr;
  A.goal = c->agent; A.goal.iou = iou;
  A.flags = flags; A.observers = c->agent_observers; A.retired = c->agent_retired;
  A.max_iou = max_iou; A.min_dist = min_dist; A.reward = reward; A.terminated = terminated; A.truncated = truncated;
  A.status = agent_status; A.done = done; A.traffic_status = traffic_status;
  A.Q = c->agent_q; A.max_step = c->cfg.max_step;
  A.reset_trackers = reset_trackers_on_done ? 1 : 0;
  t2d_agents_epilogue_kernel<<<(c->N + K10_WARPS - 1) / K10_WARPS, K10_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

static bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

// K11 over the bound state's type ids; the caller has checked the arguments
static int launch_agent_action(t2d_ctx* c, const int16_t* observers, int Q, const float* agent_action, float* action,
                               void* stream) {
  CUDA_TRY(cudaSetDevice(c->device));
  ActionArgs A{world_args(c)};
  A.observers = observers; A.agent_action = agent_action; A.action = action; A.Q = Q;
  t2d_agent_action_kernel<<<(c->N + K11_WARPS - 1) / K11_WARPS, K11_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_scatter_agent_action(t2d_ctx* c, const int16_t* observers, int32_t n_observers, const float* agent_action,
                             float* action, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (n_observers < 1 || n_observers > T2D_OBS_MAX_OBSERVERS)
    return fail(T2D_E_INVALID, "t2d_scatter_agent_action: n_observers must be in 1..128");
  if (!observers && n_observers > c->M)
    return fail(T2D_E_INVALID, "t2d_scatter_agent_action: without an observer list n_observers must not exceed the slots per scenario");
  if (!agent_action || !action) return fail(T2D_E_INVALID, "t2d_scatter_agent_action: agent_action / action is NULL");
  if (!aligned8(agent_action) || !aligned8(action))
    return fail(T2D_E_INVALID, "t2d_scatter_agent_action: agent_action and action must be 8-byte aligned");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  return launch_agent_action(c, observers, n_observers, agent_action, action, stream);
}

int t2d_step_host_agents(t2d_ctx* c, const float* agent_action_host, float* action, uint8_t* flags, int16_t* hit_index,
                         int16_t* hit_segment, float* max_iou, float* min_dist, int reset_trackers_on_done, float* reward_host,
                         uint8_t* terminated_host, uint8_t* truncated_host, uint8_t* agent_status_host, uint8_t* done_host,
                         void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!agent_action_host || !action || !max_iou || !min_dist || !done_host)
    return fail(T2D_E_INVALID, "t2d_step_host_agents: agent_action / action / max_iou / min_dist / done is NULL");
  if (!aligned8(action)) return fail(T2D_E_INVALID, "t2d_step_host_agents: action must be 8-byte aligned");
  if (int r = require(c, NEED_STATE | NEED_TABLE | NEED_TICK)) return r;
  if (c->agent_q == 0) return fail(T2D_E_STATE, "t2d_step_host_agents: no agents bound: call t2d_set_agents first");
  if (int r = check_route_trackers(c, "t2d_step_host_agents")) return r;
  if (c->d_ctab)
    if (int r = check_pid_binding(c)) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  const int N = c->N, M = c->M, Q = c->agent_q;
  const size_t nq = (size_t)N * Q;
  const size_t out_bytes = 7 * nq + N;                   // reward, terminated, truncated, status, done
  const size_t iou_off = (out_bytes + 15) & ~(size_t)15;
  if (c->ha.q != Q) {   // staging for the bound Q
    AgentStaging a;
    if (int r = dev_alloc(a.action, nq * 2)) return r;
    if (int r = make_mirror(a.out, iou_off + nq * sizeof(float), out_bytes)) return r;
    a.q = Q;
    c->ha = std::move(a);
  }
  if (!flags && !c->ha_flags)
    if (int r = dev_alloc(c->ha_flags, (size_t)N * M)) return r;
  uint8_t* fl = flags ? flags : c->ha_flags.get();
  uint8_t* o = c->ha.out.dev.get();
  float* d_reward = reinterpret_cast<float*>(o);
  uint8_t* d_term = o + 4 * nq;
  uint8_t* d_trunc = d_term + nq;
  uint8_t* d_status = d_trunc + nq;
  uint8_t* d_done = d_status + nq;
  float* d_iou = reinterpret_cast<float*>(o + iou_off);
  // One copy-engine transfer of the actions, as t2d_step_host (from pinned caller memory it is a DMA; pageable memory
  // goes through the driver's staging).  Staging them in mapped host memory for K11 to read over PCIe, as
  // t2d_step_host_ego does with its 8 N bytes, made the whole call about 1.5x slower at 2 MiB (DESIGN.md section 7).
  cudaStream_t s = (cudaStream_t)stream;
  CUDA_TRY(cudaMemcpyAsync(c->ha.action.get(), agent_action_host, nq * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
  if (int r = launch_agent_action(c, c->agent_observers, Q, c->ha.action.get(), action, stream)) return r;
  if (c->d_ctab)
    if (int r = launch_control(c, action, c->ego_action, stream)) return r;
  if (int r = launch_step(c, action, c->ego_action, fl, hit_index, hit_segment, nullptr, nullptr, stream, 1)) return r;
  if (int r = launch_history(c, nullptr, stream)) return r;   // the post-tick state, before K10 retires slots
  if (int r = t2d_agents_epilogue(c, fl, d_reward, d_term, d_trunc, d_status, d_iou, d_done, max_iou, min_dist, nullptr,
                                  reset_trackers_on_done, stream))
    return r;
  return read_back(c->ha.out, out_bytes, s,
                   {{reward_host, 0, 4 * nq}, {terminated_host, 4 * nq, nq}, {truncated_host, 5 * nq, nq},
                    {agent_status_host, 6 * nq, nq}, {done_host, 7 * nq, (size_t)N}});
}

int t2d_check_events(t2d_ctx* c, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment, void* stream) {
  return launch_step(c, nullptr, c ? c->ego_action : nullptr, flags, hit_index, hit_segment, nullptr, nullptr, stream, 0);
}

// The arguments t2d_reset and t2d_reset_sampled share
static int check_reset(t2d_ctx* c, const uint8_t* mask, int n_pool, const float* pool_x, const float* pool_y,
                       const float* pool_heading, const float* pool_speed) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE)) return r;
  if (!mask || !pool_x || !pool_y || !pool_heading || !pool_speed) return fail(T2D_E_INVALID, "t2d_reset: NULL array");
  if (n_pool <= 0) return fail(T2D_E_INVALID, "n_pool must be > 0");
  if (c->log && n_pool != c->log->n_rows) return fail(T2D_E_INVALID, "t2d_reset: with a log bound, pool row p is episode row p (n_pool == n_rows)");
  if (c->log && c->log->type_id != c->type_id) return fail(T2D_E_STATE, "state rebound after t2d_set_log: call t2d_set_log again");
  return T2D_OK;
}

// K2 (and K7) of t2d_reset, after check_reset; t2d_reset_sampled runs it between K13 and K14
static int launch_reset(t2d_ctx* c, const uint8_t* mask, const int32_t* pool_index, int n_pool, const float* pool_x,
                        const float* pool_y, const float* pool_heading, const float* pool_speed, const float* pool_vx,
                        const float* pool_vy, void* stream) {
  CUDA_TRY(cudaSetDevice(c->device));
  ResetArgs A{world_args(c)};
  A.mask = mask; A.pool_index = pool_index;
  A.px = pool_x; A.py = pool_y; A.ph = pool_heading; A.pv = pool_speed; A.pvx = pool_vx; A.pvy = pool_vy;
  A.goal = c->goal;
  A.wheel_f = c->wheel_f; A.wheel_r = c->wheel_r; A.pool_wf = c->reset_pool_wf; A.pool_wr = c->reset_pool_wr;
  A.last_accel = c->ctrl_last_accel; A.pid_state = c->pid_state; A.n_pool = n_pool;
  if (c->agent_q > 0) {   // the bound type_id is the caller's writable device array (K10 retires slots in it)
    A.agent_type_id = const_cast<uint8_t*>(c->type_id); A.agent_retired = c->agent_retired;
    A.agent = c->agent; A.agent_q = c->agent_q;
  }
  t2d_reset_kernel<<<capped_grid((long long)c->N * c->M, 256, c->sm_count, 8), 256, 0, (cudaStream_t)stream>>>(A);
  if (int r = launched()) return r;
  if (c->log) return launch_replay(c, stream, 0, c->N, 0, mask, pool_index);   // the new episode's traffic at t0
  return T2D_OK;
}

int t2d_reset(t2d_ctx* c, const uint8_t* mask, const int32_t* pool_index, int n_pool, const float* pool_x, const float* pool_y,
              const float* pool_heading, const float* pool_speed, const float* pool_vx, const float* pool_vy, void* stream) {
  if (int r = check_reset(c, mask, n_pool, pool_x, pool_y, pool_heading, pool_speed)) return r;
  if (int r = launch_reset(c, mask, pool_index, n_pool, pool_x, pool_y, pool_heading, pool_speed, pool_vx, pool_vy, stream))
    return r;
  return launch_history(c, mask, stream);   // entry 0 of the new episode: the state after the whole reset
}

// A row-owned pool needs what it writes into: checked when the sampler is bound and before every sampled reset (the
// goal, the map table or the routes may have been unbound since)
static int check_sampler_targets(const t2d_ctx* c, const t2d_reset_sampler& s) {
  if (s.pool_target && !c->goal.target) return fail(T2D_E_STATE, "reset sampler: a target pool needs a t2d_set_goal target");
  if (s.pool_tile_id && !c->map.tile_id) return fail(T2D_E_STATE, "reset sampler: a tile pool needs a map table of more than one tile");
  if (s.pool_route_id && !c->route_id) return fail(T2D_E_STATE, "reset sampler: a route pool needs t2d_set_routes");
  return T2D_OK;
}

int t2d_set_reset_sampler(t2d_ctx* c, const t2d_reset_sampler* s) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!s) {
    c->sampler.reset();
    return T2D_OK;
  }
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (s->tries < 1 || s->tries > 32) return fail(T2D_E_INVALID, "reset sampler: tries must be in 1..32");
  if (!s->episode || !s->pool_row || !s->reset_try) return fail(T2D_E_INVALID, "reset sampler: NULL episode / pool_row / reset_try");
  const bool pools = s->pool_type_id || s->pool_target || s->pool_tile_id || s->pool_route_id;
  if (pools && s->n_rows <= 0) return fail(T2D_E_INVALID, "reset sampler: row pools need n_rows > 0");
  if (s->jitter)
    for (int k = 0; k < c->M * 4; ++k) {
      const float lo = s->jitter[2 * k], hi = s->jitter[2 * k + 1];
      if (!(std::isfinite(lo) && std::isfinite(hi) && lo <= hi))
        return fail(T2D_E_INVALID, "reset sampler: every jitter range must be finite with lo <= hi");
    }
  if (int r = check_sampler_targets(c, *s)) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  auto d = std::make_unique<DeviceSampler>();
  d->s = *s;
  if (s->jitter) {
    if (int r = upload(d->jitter, s->jitter, (size_t)c->M * 8)) return r;
    d->s.jitter = d->jitter.get();
  }
  CUDA_TRY(cudaMemset(s->episode, 0, sizeof(uint32_t) * c->N));
  c->sampler = std::move(d);
  return T2D_OK;
}

int t2d_reset_sampled(t2d_ctx* c, const uint8_t* mask, int n_pool, const float* pool_x, const float* pool_y,
                      const float* pool_heading, const float* pool_speed, const float* pool_vx, const float* pool_vy,
                      void* stream) {
  if (int r = check_reset(c, mask, n_pool, pool_x, pool_y, pool_heading, pool_speed)) return r;
  if (!c->sampler) return fail(T2D_E_STATE, "t2d_reset_sampled: no reset sampler bound");
  if (int r = require(c, NEED_TABLE)) return r;
  const t2d_reset_sampler& s = c->sampler->s;
  if (int r = check_sampler_targets(c, s)) return r;
  if ((s.pool_type_id || s.pool_target || s.pool_tile_id || s.pool_route_id) && n_pool != s.n_rows)
    return fail(T2D_E_INVALID, "t2d_reset_sampled: the pool must have the sampler's n_rows rows");
  if (!s.sample_rows && n_pool < c->N) return fail(T2D_E_INVALID, "t2d_reset_sampled: without row draws the pool needs one row per scenario");
  CUDA_TRY(cudaSetDevice(c->device));
  DrawArgs D{};
  D.mask = mask; D.episode = s.episode; D.pool_row = s.pool_row; D.seed = s.seed; D.sample_rows = s.sample_rows;
  D.N = c->N; D.M = c->M; D.P = n_pool;
  // the row-owned columns are written into the caller's bound arrays (type_id, the goal target, the map table's tile_id,
  // the route ids), which the library documents as rewritable between ticks
  D.pool_type = s.pool_type_id; D.type_id = const_cast<uint8_t*>(c->type_id);
  D.retired = c->agent_q > 0 ? c->agent_retired : nullptr;
  D.pool_target = s.pool_target; D.target = const_cast<float*>(c->goal.target);
  D.pool_tile = s.pool_tile_id; D.tile_id = const_cast<uint16_t*>(c->map.tile_id);
  D.pool_route = s.pool_route_id; D.route_id = const_cast<int16_t*>(c->route_id);
  t2d_episode_draw_kernel<<<capped_grid((long long)c->N * c->M, 256, c->sm_count, 8), 256, 0, (cudaStream_t)stream>>>(D);
  if (int r = launched()) return r;
  if (int r = launch_reset(c, mask, s.pool_row, n_pool, pool_x, pool_y, pool_heading, pool_speed, pool_vx, pool_vy, stream))
    return r;
  PlaceArgs P{world_args(c)};
  P.mask = mask; P.episode = s.episode; P.reset_try = s.reset_try; P.seed = s.seed;
  P.jitter = s.jitter; P.tries = s.tries; P.avoid_target = s.avoid_target; P.target = c->goal.target;
  P.map = map_args(c->map); P.mh = c->map.mh; P.has_bounds = c->map.has_bounds ? 1 : 0;
  P.wheel_f = c->wheel_f; P.wheel_r = c->wheel_r; P.pool_wheels = c->reset_pool_wf != nullptr;
  t2d_episode_place_kernel<<<(unsigned)((c->N + K14_WARPS - 1) / K14_WARPS), K14_WARPS * 32, 0, (cudaStream_t)stream>>>(P);
  if (int r = launched()) return r;
  return launch_history(c, mask, stream);   // entry 0 of the new episode: the placed state
}

// K4 over the rows of an observer list (observers == nullptr: row q is slot q); the callers have checked their arguments
static int launch_lidar(t2d_ctx* c, const int16_t* observers, int Q, int n_beams, float max_range, const double* beam_cos_sin,
                        float* scan, void* stream) {
  CUDA_TRY(cudaSetDevice(c->device));
  LidarArgs A{world_args(c)};
  A.map = map_args(c->map);
  A.beam_cs = beam_cos_sin; A.observers = observers; A.scan = scan;
  A.Q = Q; A.n_beams = n_beams; A.range = (double)max_range;
  const long long grid = ((long long)c->N * Q + LIDAR_WARPS - 1) / LIDAR_WARPS;
  if (grid > INT32_MAX) return fail(T2D_E_UNSUPPORTED, "lidar: more than 2^33 rows (one warp per row)");
  t2d_lidar_kernel<<<(unsigned)grid, LIDAR_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_lidar_scan(t2d_ctx* c, int n_beams, float max_range, const double* beam_cos_sin, float* scan, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (n_beams <= 0 || !(max_range > 0.0f) || !beam_cos_sin || !scan) return fail(T2D_E_INVALID, "t2d_lidar_scan: bad argument");
  return launch_lidar(c, nullptr, 1, n_beams, max_range, beam_cos_sin, scan, stream);
}

int t2d_lidar_scan_agents(t2d_ctx* c, const int16_t* observers, int32_t n_observers, int n_beams, float max_range,
                          const double* beam_cos_sin, float* scan, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (n_observers < 1 || n_observers > T2D_OBS_MAX_OBSERVERS)
    return fail(T2D_E_INVALID, "t2d_lidar_scan_agents: n_observers must be in 1..128");
  if (n_beams <= 0 || !(max_range > 0.0f) || !beam_cos_sin || !scan)
    return fail(T2D_E_INVALID, "t2d_lidar_scan_agents: n_beams must be > 0, max_range > 0, beam_cos_sin and scan not NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (!observers && n_observers > c->M)
    return fail(T2D_E_INVALID, "t2d_lidar_scan_agents: without an observer list n_observers must not exceed the slots per scenario");
  return launch_lidar(c, observers, n_observers, n_beams, max_range, beam_cos_sin, scan, stream);
}

int t2d_set_bev_styles(t2d_ctx* c, const t2d_bev_style* table, int n_styles, const uint8_t* type_style, const uint8_t* seg_style,
                       int n_seg_total, int target_style) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_TABLE)) return r;
  if (!table || n_styles < 4 || n_styles > T2D_MAX_BEV_STYLES) return fail(T2D_E_INVALID, "n_styles must be in 4..64");
  if (!type_style) return fail(T2D_E_INVALID, "type_style is NULL");
  for (int i = 0; i < n_styles; ++i)
    if (!(table[i].line_width_pt >= 0.0f && table[i].line_width_pt <= 100.0f))
      return fail(T2D_E_INVALID, "style line width must be in [0, 100] pt");
  auto ok = [&](int s) { return s == bev::NO_STYLE || (s >= 0 && s < n_styles); };
  for (int t = 0; t < c->n_types; ++t)
    if (!ok(type_style[t])) return fail(T2D_E_INVALID, "type_style: no such style");
  if (!ok(target_style)) return fail(T2D_E_INVALID, "target_style: no such style");
  const std::vector<int>& nseg = c->map.tile_nseg;
  long long total = 0;
  for (int k : nseg) total += k;
  if (seg_style) {
    if (n_seg_total != total) return fail(T2D_E_INVALID, "n_seg_total differs from the segments of the map's tiles");
    for (long long s = 0; s < total; ++s)
      if (!ok(seg_style[s])) return fail(T2D_E_INVALID, "seg_style: no such style");
  }
  CUDA_TRY(cudaSetDevice(c->device));
  dev_ptr<uint8_t> d_style;
  dev_ptr<uint32_t> d_base;
  if (seg_style && total > 0) {
    std::vector<uint32_t> base(nseg.size());
    uint32_t acc = 0;
    for (size_t i = 0; i < base.size(); ++i) { base[i] = acc; acc += (uint32_t)nseg[i]; }
    if (int r = upload(d_style, seg_style, (size_t)total)) return r;
    if (int r = upload(d_base, base.data(), base.size())) return r;
  }
  // opt in to the kernel's shared memory here: t2d_bev_render must stay free of anything a graph capture rejects
  CUDA_TRY(cudaFuncSetAttribute(bev::t2d_bev_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(bev::Smem)));
  c->map.seg_style = std::move(d_style);
  c->map.seg_base = std::move(d_base);
  memcpy(c->bev_style, table, sizeof(t2d_bev_style) * (size_t)n_styles);
  memset(c->bev_type_style, bev::NO_STYLE, sizeof(c->bev_type_style));
  memcpy(c->bev_type_style, type_style, (size_t)c->n_types);
  c->bev_target_style = target_style;
  c->n_bev_styles = n_styles;
  return T2D_OK;
}

int t2d_bev_render(t2d_ctx* c, int width, int height, const float* range, int rgb, uint8_t* out, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE)) return r;
  if (c->n_bev_styles == 0) return fail(T2D_E_STATE, "BEV styles not set: call t2d_set_bev_styles first");
  if (!range || !out) return fail(T2D_E_INVALID, "t2d_bev_render: range / out is NULL");
  if (width < 1 || height < 1 || width > bev::MAX_SIDE || height > bev::MAX_SIDE)
    return fail(T2D_E_INVALID, "t2d_bev_render: width and height must be in 1..1024");
  for (int k = 0; k < 4; ++k)
    if (!(range[k] > 0.0f && range[k] <= 1.0e5f)) return fail(T2D_E_INVALID, "t2d_bev_render: every range must be in (0, 1e5] m");
  // the window (matplotlib_renderer.py:152-164, auto_scale :200-224), in the float64 oracle's operation order
  const double L = range[0], R = range[1], F = range[2], B = range[3];
  const double x_min = -L, x_max = R, y_min = -B, y_max = F;
  const double ww = x_max - x_min, wh = y_max - y_min;
  const double cx = (x_min + x_max) / 2, cy = (y_min + y_max) / 2;
  const double aspect = (double)height / (double)width;
  double nw, nh;
  if (wh / ww > aspect) { nw = wh / aspect; nh = wh; }
  else { nw = ww; nh = ww * aspect; }
  const double nx0 = cx - nw / 2, nx1 = cx + nw / 2, ny0 = cy - nh / 2, ny1 = cy + nh / 2;
  bev::Args A{world_args(c)};
  A.win.xmin = nx0; A.win.ymax = ny1;
  A.win.px = (nx1 - nx0) / width; A.win.py = (ny1 - ny0) / height;
  for (int s = 0; s < c->n_bev_styles; ++s) {
    const t2d_bev_style& st = c->bev_style[s];
    const double hw = (double)st.line_width_pt * 200.0 / 72.0 / 2.0 * A.win.px;   // points at the renderer's 200 dpi
    A.hw2[s] = hw * hw;
    A.style_rgb[s][0] = st.r; A.style_rgb[s][1] = st.g; A.style_rgb[s][2] = st.b;
    A.style_z[s] = st.z;
  }
  memcpy(A.type_style, c->bev_type_style, sizeof(A.type_style));
  A.map = map_args(c->map); A.seg_style = c->map.seg_style.get(); A.seg_base = c->map.seg_base.get();
  A.target = c->goal.target; A.target_style = c->bev_target_style;
  A.ring_style = T2D_BEV_STYLE_RING; A.open_style = T2D_BEV_STYLE_OPEN;
  A.W = width; A.H = height; A.rgb = rgb ? 1 : 0; A.out = out;
  CUDA_TRY(cudaSetDevice(c->device));
  bev::t2d_bev_kernel<<<c->N, bev::CTA, sizeof(bev::Smem), (cudaStream_t)stream>>>(A);
  return launched();
}

// What t2d_observe and t2d_observe_agents share: the checks of cfg and out (messages prefixed with fn) and K8's arguments
static int obs_args(const t2d_ctx* c, const std::string& fn, const t2d_obs_config* cfg, float* out, int16_t* agent_index,
                    int16_t* segment_index, obs::Args& A) {
  if (!cfg) return fail(T2D_E_INVALID, fn + ": cfg is NULL");
  if (cfg->k_agents < 0 || cfg->k_agents > T2D_OBS_MAX_AGENTS) return fail(T2D_E_INVALID, fn + ": k_agents must be in 0..127");
  if (cfg->k_segments < 0 || cfg->k_segments > T2D_OBS_MAX_SEGMENTS)
    return fail(T2D_E_INVALID, fn + ": k_segments must be in 0..256");
  if (!(cfg->agent_range > 0.0f && cfg->agent_range <= 1.0e5f) || !(cfg->segment_range > 0.0f && cfg->segment_range <= 1.0e5f))
    return fail(T2D_E_INVALID, fn + ": agent_range and segment_range must be in (0, 1e5] m");
  if (!out) return fail(T2D_E_INVALID, fn + ": out is NULL");
  static_assert(T2D_OBS_MAX_AGENTS == obs::MAX_K && T2D_OBS_MAX_SEGMENTS == obs::MAX_S, "K8's shared lists hold the ABI's limits");
  static_cast<WorldArgs&>(A) = world_args(c);
  A.max_step = c->cfg.max_step; A.map = map_args(c->map); A.target = c->goal.target;
  A.K = cfg->k_agents; A.S = cfg->k_segments;
  A.F = obs::EGO_F + obs::GOAL_F + obs::AGENT_F * A.K + obs::SEG_F * A.S;
  const double ra = cfg->agent_range, rs = cfg->segment_range;
  A.ra2 = ra * ra; A.rs2 = rs * rs;
  A.out = out; A.agent_index = agent_index; A.segment_index = segment_index;
  return T2D_OK;
}

int t2d_observe(t2d_ctx* c, const t2d_obs_config* cfg, float* out, int16_t* agent_index, int16_t* segment_index, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  obs::Args A{};
  if (int r = obs_args(c, "t2d_observe", cfg, out, agent_index, segment_index, A)) return r;
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  const int grid = (c->N + obs::WARPS - 1) / obs::WARPS;
  obs::t2d_obs_kernel<<<grid, obs::WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_observe_agents(t2d_ctx* c, const t2d_obs_config* cfg, const int16_t* observers, int32_t n_observers,
                       const float* goals, float* out, int16_t* agent_index, int16_t* segment_index, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  obs::AgentArgs G{};
  if (int r = obs_args(c, "t2d_observe_agents", cfg, out, agent_index, segment_index, G.a)) return r;
  if (n_observers < 1 || n_observers > T2D_OBS_MAX_OBSERVERS)
    return fail(T2D_E_INVALID, "t2d_observe_agents: n_observers must be in 1..128");
  if (!observers && n_observers > c->M)
    return fail(T2D_E_INVALID, "t2d_observe_agents: without an observer list n_observers must not exceed the slots per scenario");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  G.observers = observers; G.goals = goals; G.Q = n_observers;
  CUDA_TRY(cudaSetDevice(c->device));
  const long long rows = (long long)c->N * n_observers;
  const int grid = (int)std::min<long long>((rows + obs::WARPS - 1) / obs::WARPS, 1ll << 30);   // the kernel strides past 2^32 rows
  obs::t2d_obs_agents_kernel<<<grid, obs::WARPS * 32, 0, (cudaStream_t)stream>>>(G);
  return launched();
}

int t2d_set_history(t2d_ctx* c, int32_t length) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (length < 0 || length > T2D_HISTORY_MAX) return fail(T2D_E_INVALID, "t2d_set_history: length must be in 0..64");
  CUDA_TRY(cudaSetDevice(c->device));
  if (length == 0) {
    c->hist.reset();
    return T2D_OK;
  }
  static_assert(T2D_HISTORY_MAX == hist::MAX_H && T2D_HISTORY_FIELDS == hist::HIST_F, "K16's stage holds the ABI's limits");
  auto g = std::make_unique<DeviceHistory>();
  g->H = length;
  const size_t plane = (size_t)c->N * length * c->M;
  if (int r = dev_alloc(g->f, 6 * plane)) return r;
  if (int r = dev_alloc(g->type, plane)) return r;
  if (int r = dev_alloc(g->count, (size_t)c->N)) return r;
  CUDA_TRY(cudaMemset(g->f.get(), 0, 6 * plane * sizeof(float)));
  CUDA_TRY(cudaMemset(g->type.get(), 0xff, plane));
  CUDA_TRY(cudaMemset(g->count.get(), 0, (size_t)c->N * sizeof(long long)));
  if (int r = history_tracks(c, *g, c->log ? c->log->track_out : nullptr)) return r;
  c->hist = std::move(g);
  return T2D_OK;
}

int t2d_history_view(t2d_ctx* c, t2d_history_ring* out) {
  if (!c || !out) return fail(T2D_E_INVALID, "t2d_history_view: ctx / out is NULL");
  *out = t2d_history_ring{};
  if (!c->hist) return T2D_OK;
  const hist::Ring R = history_ring(c);
  out->length = R.H;
  out->x = R.x; out->y = R.y; out->heading = R.h; out->speed = R.v; out->vx = R.vx; out->vy = R.vy;
  out->type_id = R.type; out->track = R.track; out->count = reinterpret_cast<int64_t*>(R.count);
  return T2D_OK;
}

int t2d_observe_history(t2d_ctx* c, const int16_t* observers, int32_t n_observers, const int16_t* agent_index, int32_t k_agents,
                        float* out, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (n_observers < 0 || n_observers > T2D_OBS_MAX_OBSERVERS)
    return fail(T2D_E_INVALID, "t2d_observe_history: n_observers must be in 0..128");
  if (n_observers == 0 && observers) return fail(T2D_E_INVALID, "t2d_observe_history: an observer list needs n_observers >= 1");
  if (!observers && n_observers > c->M)
    return fail(T2D_E_INVALID, "t2d_observe_history: without an observer list n_observers must not exceed the slots per scenario");
  if (k_agents < 0 || k_agents > T2D_OBS_MAX_AGENTS) return fail(T2D_E_INVALID, "t2d_observe_history: k_agents must be in 0..127");
  if (k_agents > 0 && !agent_index) return fail(T2D_E_INVALID, "t2d_observe_history: agent_index is NULL");
  if (!out) return fail(T2D_E_INVALID, "t2d_observe_history: out is NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (!c->hist) return fail(T2D_E_STATE, "t2d_observe_history: no history bound: call t2d_set_history first");
  CUDA_TRY(cudaSetDevice(c->device));
  hist::ObsArgs A{world_args(c)};
  A.ring = history_ring(c); A.track_now = history_track_now(c);
  A.observers = observers; A.Q = n_observers; A.agent_index = agent_index; A.K = k_agents; A.out = out;
  const long long rows = (long long)c->N * std::max(1, n_observers);
  const int grid = (int)std::min<long long>((rows + hist::K16_WARPS - 1) / hist::K16_WARPS, 1ll << 30);   // the kernel strides
  hist::t2d_history_obs_kernel<<<grid, hist::K16_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_set_controllers(t2d_ctx* c, const t2d_controller_params* table, int n_rows, const uint8_t* ctrl_id,
                        const int16_t* lead_index, const int16_t* path_id, float* last_accel) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  if (!table) {
    c->d_ctab.reset();
    c->n_ctrl = 0; c->ctrl_id = nullptr; c->ctrl_lead = nullptr; c->ctrl_path = nullptr;
    c->ctrl_last_accel = nullptr;
    c->ctrl_has_pid = c->ctrl_pid_reads_target = false;
    return T2D_OK;
  }
  if (n_rows <= 0 || n_rows > T2D_MAX_CONTROLLERS) return fail(T2D_E_INVALID, "n_rows must be in 1..T2D_MAX_CONTROLLERS");
  if (!ctrl_id || !last_accel) return fail(T2D_E_INVALID, "t2d_set_controllers: ctrl_id / last_accel is NULL");
  bool has_pid = false, reads_target = false;
  for (int i = 0; i < n_rows; ++i) {
    const t2d_controller_params& p = table[i];
    if (p.kind < T2D_CTRL_EXTERNAL || p.kind > T2D_CTRL_PID) return fail(T2D_E_INVALID, "unknown controller kind");
    if (p.kind == T2D_CTRL_PID) {   // PIDController.__init__'s checks, pid_controller.py:81-102
      if (!(p.dt > 0.0)) return fail(T2D_E_INVALID, "PID row: dt must be positive");
      if (!(p.max_steering > 0.0)) return fail(T2D_E_INVALID, "PID row: max_steering must be positive");
      if (!(p.max_accel > 0.0f)) return fail(T2D_E_INVALID, "PID row: max_accel must be positive");
      if (!(p.min_accel < 0.0f)) return fail(T2D_E_INVALID, "PID row: min_accel must be negative (deceleration)");
      if (!(p.max_accel > p.min_accel)) return fail(T2D_E_INVALID, "PID row: max_accel must be greater than min_accel");
      if (!(p.derivative_filter_alpha > 0.0 && p.derivative_filter_alpha <= 1.0))
        return fail(T2D_E_INVALID, "PID row: derivative_filter_alpha must be in range (0, 1]");
      if (p.pid_lateral < T2D_PID_LAT_NONE || p.pid_lateral > T2D_PID_LAT_PATH_CROSS_TRACK)
        return fail(T2D_E_INVALID, "PID row: unknown lateral source");
      if (p.pid_longitudinal != T2D_PID_LON_NONE && p.pid_longitudinal != T2D_PID_LON_TARGET)
        return fail(T2D_E_INVALID, "PID row: unknown longitudinal source");
      if ((p.pid_lateral == T2D_PID_LAT_CROSS_TRACK || p.pid_lateral == T2D_PID_LAT_PATH_CROSS_TRACK) && !(p.wheel_base > 0.0f))
        return fail(T2D_E_INVALID, "PID row: wheel_base must be positive");   // pid_controller.py:357-358
      has_pid = true;
      reads_target = reads_target || p.pid_longitudinal == T2D_PID_LON_TARGET || p.pid_lateral == T2D_PID_LAT_HEADING ||
                     p.pid_lateral == T2D_PID_LAT_CROSS_TRACK;
    }
    if (p.kind == T2D_CTRL_PURE_PURSUIT && !(p.min_pre_aiming_distance > 0.0f))
      return fail(T2D_E_INVALID, "min_pre_aiming_distance must be positive");   // pure_pursuit_controller.py:30-31
    if (p.kind >= T2D_CTRL_CRUISE && p.target_speed < 0.0f)
      return fail(T2D_E_INVALID, "target_speed must be non-negative");          // acceleration_controller.py:48-49
  }
  if (int r = upload(c->d_ctab, table, (size_t)n_rows)) return r;
  c->n_ctrl = n_rows; c->ctrl_id = ctrl_id; c->ctrl_lead = lead_index; c->ctrl_path = path_id; c->ctrl_last_accel = last_accel;
  c->ctrl_has_pid = has_pid; c->ctrl_pid_reads_target = reads_target;
  return T2D_OK;
}

int t2d_set_pid(t2d_ctx* c, const float* target, double* state) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!state) {
    if (target) return fail(T2D_E_INVALID, "t2d_set_pid: a target needs a state");
    c->pid_target = nullptr; c->pid_state = nullptr;
    return T2D_OK;
  }
  if (reinterpret_cast<uintptr_t>(target) % 8 != 0 || reinterpret_cast<uintptr_t>(state) % 8 != 0)
    return fail(T2D_E_INVALID, "t2d_set_pid: target / state must be 8-byte aligned");
  c->pid_target = target; c->pid_state = state;
  return T2D_OK;
}

int t2d_set_paths(t2d_ctx* c, const float* xy, const int32_t* offsets, int n_paths) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  if (n_paths == 0 || !xy) {   // unbind
    c->d_path_v.reset(); c->d_path_off.reset(); c->n_paths = 0;
    return T2D_OK;
  }
  if (n_paths < 0 || !offsets) return fail(T2D_E_INVALID, "t2d_set_paths: bad argument");
  if (offsets[0] != 0) return fail(T2D_E_INVALID, "offsets[0] must be 0");
  for (int p = 0; p < n_paths; ++p)
    if (offsets[p + 1] - offsets[p] < 2) return fail(T2D_E_INVALID, "a path needs at least 2 vertices");
  const int V = offsets[n_paths];
  std::vector<PathVertex> pv((size_t)V);
  for (int p = 0; p < n_paths; ++p) {
    double acc = 0.0;   // the running arc length of LineString.interpolate's walk, in float64
    for (int i = offsets[p]; i < offsets[p + 1]; ++i) {
      pv[i].x = xy[2 * i]; pv[i].y = xy[2 * i + 1];
      pv[i].cum = acc;
      pv[i].len = 0.0;
      if (i + 1 < offsets[p + 1]) {
        pv[i].len = hypot((double)xy[2 * i + 2] - (double)xy[2 * i], (double)xy[2 * i + 3] - (double)xy[2 * i + 1]);
        acc += pv[i].len;
      }
    }
  }
  dev_ptr<PathVertex> d_v;
  dev_ptr<int> d_off;
  if (int r = upload(d_v, pv.data(), pv.size())) return r;
  if (int r = upload(d_off, offsets, (size_t)n_paths + 1)) return r;
  c->d_path_v = std::move(d_v); c->d_path_off = std::move(d_off); c->n_paths = n_paths;
  return T2D_OK;
}

int t2d_set_routes(t2d_ctx* c, const int16_t* route_id, double threshold, double progress_weight, float off_route_reward) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (route_id) {
    if (!(std::isfinite(threshold) && threshold >= 0.0))
      return fail(T2D_E_INVALID, "t2d_set_routes: threshold must be finite and >= 0");
    if (!std::isfinite(progress_weight) || !std::isfinite(off_route_reward))
      return fail(T2D_E_INVALID, "t2d_set_routes: progress_weight and off_route_reward must be finite");
  }
  c->route_id = route_id;
  c->route_threshold = route_id ? threshold : 0.0;
  c->route_weight = route_id ? progress_weight : 0.0;
  c->route_off_reward = route_id ? off_route_reward : 0.0f;
  return T2D_OK;
}

int t2d_bind_route_trackers(t2d_ctx* c, double* s_best, double* agent_s_best, int32_t n_agent_rows) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (agent_s_best && (n_agent_rows < 1 || n_agent_rows > T2D_OBS_MAX_OBSERVERS))
    return fail(T2D_E_INVALID, "t2d_bind_route_trackers: n_agent_rows must be in 1..128");
  if (!aligned8(s_best) || !aligned8(agent_s_best))
    return fail(T2D_E_INVALID, "t2d_bind_route_trackers: the trackers must be 8-byte aligned");
  c->route_s_best = s_best;
  c->route_agent_s_best = agent_s_best;
  c->route_agent_rows = agent_s_best ? n_agent_rows : 0;
  return T2D_OK;
}

int t2d_route_observe(t2d_ctx* c, const int16_t* observers, int32_t n_observers, int n_points, float spacing, float* out,
                      void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (n_observers < 1 || n_observers > T2D_OBS_MAX_OBSERVERS)
    return fail(T2D_E_INVALID, "t2d_route_observe: n_observers must be in 1..128");
  if (!observers && n_observers > c->M)
    return fail(T2D_E_INVALID, "t2d_route_observe: without an observer list n_observers must not exceed the slots per scenario");
  if (n_points < 0 || n_points > T2D_ROUTE_MAX_POINTS) return fail(T2D_E_INVALID, "t2d_route_observe: n_points must be in 0..256");
  if (!(spacing > 0.0f) || !std::isfinite(spacing)) return fail(T2D_E_INVALID, "t2d_route_observe: spacing must be finite and > 0");
  if (!out) return fail(T2D_E_INVALID, "t2d_route_observe: out is NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  RouteObsArgs A{world_args(c)};
  A.route = route_args(c); A.observers = observers; A.out = out; A.Q = n_observers; A.P = n_points;
  A.spacing = (double)spacing;
  t2d_route_obs_kernel<<<(c->N + K12_WARPS - 1) / K12_WARPS, K12_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_control(t2d_ctx* c, float* action, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  return launch_control(c, action, c->ego_action, stream);
}
int t2d_exchange_create(t2d_exchange** out, int device, int world, int rank, int n_local, int slots, void* ipc_handle_out) {
  if (!out || !ipc_handle_out) return fail(T2D_E_INVALID, "out / ipc_handle_out is NULL");
  *out = nullptr;
  if (world < 1 || world > T2D_MAX_RANKS || rank < 0 || rank >= world) return fail(T2D_E_INVALID, "bad world / rank");
  if (n_local <= 0 || slots < 2 || slots > 64) return fail(T2D_E_INVALID, "n_local must be > 0 and slots in 2..64");
  static_assert(sizeof(cudaIpcMemHandle_t) == T2D_IPC_HANDLE_BYTES, "IPC handle size");
  CUDA_TRY(cudaSetDevice(device));
  t2d_exchange* x = new t2d_exchange();
  x->device = device; x->world = world; x->rank = rank; x->n_real = n_local; x->n_local = (n_local + 15) & ~15; x->slots = slots;
  x->threads = std::min(256, 32 * world);                 // one warp per peer
  if (const char* e = getenv("T2D_EXCHANGE_THREADS")) {   // experiments: a smaller CTA finds a home on a busy SM sooner
    const int v = atoi(e);
    if (v >= 32 && v <= 512 && v % 32 == 0 && v >= world) x->threads = v;
  }
  if (const char* e = getenv("T2D_EXCHANGE_TIMEOUT_MS")) {
    const double ms = atof(e);
    if (ms > 0.0) x->timeout_cycles = (long long)(ms * 2.0e6);   // ~2 GHz SM clock
  }
  x->bytes = x->flag_off() + (T2D_MAX_RANKS + 4) * sizeof(unsigned);
  cudaError_t e = cudaMalloc(&x->base, x->bytes);
  if (e == cudaSuccess) e = cudaMemset(x->base, 0, x->bytes);
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, x->base);
  if (e != cudaSuccess) {
    if (x->base) cudaFree(x->base);
    delete x;
    return fail(T2D_E_CUDA, std::string("t2d_exchange_create: ") + cudaGetErrorString(e));
  }
  memcpy(ipc_handle_out, &h, sizeof(h));
  CUDA_TRY(cudaDeviceSynchronize());
  g_exchanges_alive.fetch_add(1);
  *out = x;
  return T2D_OK;
}

int t2d_exchange_connect(t2d_exchange* x, const void* handles) {
  if (!x || !handles) return fail(T2D_E_INVALID, "exchange / handles is NULL");
  CUDA_TRY(cudaSetDevice(x->device));
  for (int p = 0; p < x->world; ++p) {
    if (p == x->rank) { x->peer[p] = x->base; continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, static_cast<const unsigned char*>(handles) + (size_t)p * sizeof(h), sizeof(h));
    void* ptr = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {   // do not leak the mappings opened so far
      for (int q = 0; q < p; ++q)
        if (q != x->rank && x->peer[q]) { cudaIpcCloseMemHandle(x->peer[q]); x->peer[q] = nullptr; }
      return fail(T2D_E_CUDA, std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
    }
    x->peer[p] = static_cast<unsigned char*>(ptr);
  }
  x->connected = true;
  return T2D_OK;
}

int t2d_exchange_allgather_lagged(t2d_exchange* x, const uint8_t* done_local, uint8_t* dst, int lag, void* stream) {
  if (!x || !done_local || !dst) return fail(T2D_E_INVALID, "exchange / done_local / dst is NULL");
  if (!x->connected) return fail(T2D_E_STATE, "exchange not connected: call t2d_exchange_connect first");
  if (lag < 0 || 2 * lag + 2 > x->slots) return fail(T2D_E_INVALID, "lag needs a ring of at least 2 * lag + 2 slots");
  CUDA_TRY(cudaSetDevice(x->device));
  AllGatherArgs A{};
  for (int p = 0; p < x->world; ++p) A.peer[p] = x->peer[p];
  A.base = x->base; A.local = done_local; A.dst = dst;
  A.world = x->world; A.rank = x->rank; A.n_local = x->n_local; A.n_real = x->n_real; A.slots = x->slots;
  A.lag = lag; A.timeout = x->timeout_cycles;
  t2d_exchange_allgather_kernel<<<1, x->threads, 0, (cudaStream_t)stream>>>(A);
  g_launches.fetch_add(1);
  CUDA_TRY(cudaGetLastError());
  return T2D_OK;
}

int t2d_exchange_allgather(t2d_exchange* x, const uint8_t* done_local, uint8_t* dst, void* stream) {
  return t2d_exchange_allgather_lagged(x, done_local, dst, 0, stream);
}

int t2d_exchange_status(t2d_exchange* x, uint32_t* steps, uint32_t* timed_out) {
  if (!x) return fail(T2D_E_INVALID, "exchange is NULL");
  CUDA_TRY(cudaSetDevice(x->device));
  unsigned w[4];
  CUDA_TRY(cudaMemcpy(w, x->word(0), sizeof(w), cudaMemcpyDeviceToHost));
  if (steps) *steps = w[0];
  if (timed_out) *timed_out = w[3];
  return T2D_OK;
}

int t2d_exchange_destroy(t2d_exchange* x) {
  if (!x) return T2D_OK;
  cudaSetDevice(x->device);
  for (int p = 0; p < x->world; ++p)
    if (x->connected && p != x->rank && x->peer[p]) cudaIpcCloseMemHandle(x->peer[p]);
  if (x->base) cudaFree(x->base);
  g_exchanges_alive.fetch_sub(1);
  delete x;
  return T2D_OK;
}

int t2d_physics_step(int device, const t2d_type_params* params, int interval_ms, int delta_t_ms, int n, float* x, float* y,
                     float* heading, float* speed, float* vx, float* vy, float* omega_front, float* omega_rear,
                     const float* action, float* applied, void* stream) {
  if (!params) return fail(T2D_E_INVALID, "params is NULL");
  if (n < 0) return fail(T2D_E_INVALID, "n must be >= 0");
  if (n == 0) return T2D_OK;
  if (!x || !y || !heading || !speed || !vx || !vy || !action) return fail(T2D_E_INVALID, "t2d_physics_step: NULL array");
  if (interval_ms <= 0 || delta_t_ms <= 0) return fail(T2D_E_INVALID, "interval_ms and delta_t_ms must be > 0");
  if (params->model < 0 || params->model > T2D_MODEL_DRIFT) return fail(T2D_E_INVALID, "unknown model id");
  if (params->model == T2D_MODEL_DRIFT && !(omega_front && omega_rear))
    return fail(T2D_E_INVALID, "t2d_physics_step: SingleTrackDrift needs the wheel-speed arrays");
  CUDA_TRY(cudaSetDevice(device));
  PhysArgs A{};
  A.wheel_f = omega_front; A.wheel_r = omega_rear;
  {
    AbiParams a;
    memcpy(&a, params, sizeof(AbiParams));
    A.p = derive_params(a);
  }
  A.x = x; A.y = y; A.h = heading; A.v = speed; A.vx = vx; A.vy = vy; A.action = action; A.applied = applied;
  A.n = n;
  set_time_step(A, interval_ms, delta_t_ms);
  int sms = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  t2d_physics_kernel<<<capped_grid(n, 256, sms, 8), 256, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

}  // extern "C"
