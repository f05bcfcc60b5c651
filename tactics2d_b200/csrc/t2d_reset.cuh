// t2d_reset.cuh - K2 t2d_reset_kernel (masked reset from a pool of initial states) and the sampled resets: K13
// t2d_episode_draw_kernel (seeded pool-row draw) and K14 t2d_episode_place_kernel (collision-checked jitter).
#pragma once

#include "t2d_world.cuh"

namespace t2d {

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

}  // namespace t2d
