// t2d_leader.cuh - K17 t2d_leader_kernel: the leader of every participant slot, the nearest participant ahead of it in its
// corridor, which K5's car-following laws (IDM, adaptive cruise) take as `leading_state` / `front_state`.
//
// Contract: DESIGN.md section 1, "Leader search" (an extension: the reference leaves the leader to its caller).  fp64 with
// one rounding per operation, in the order tests/leader_oracle.py evaluates it.  A follower is every slot with a type
// < n_types at a position that is not NaN; a candidate is every other such slot whose shape is not SHAPE_NONE.
//   path frame     the follower's controller path_id names a path with a segment of non-zero length: the follower and every
//                  candidate are projected onto it with closest_on_path<true>; a candidate qualifies when its distance to
//                  the path is <= half_width and gap = s_j - s_i is in (0, max_range];
//   heading frame  every other follower: the candidate's offset in the follower's frame (K8's Frame, sincos_angle of its
//                  fp32 heading); it qualifies when ex > 0, |ey| <= half_width and ex <= max_range, and gap = ex.
// The leader is the qualifying candidate of smallest (gap, slot); lead = -1 and gap = +inf without one.
//
// One warp per scenario, lane l owns slots l, l + 32, l + 64, l + 96 (as K5).  The candidates' positions are staged in shared
// memory and every lane walks them in slot order, so a tie goes to the lower slot.  The projections depend on (candidate,
// path) only: the warp takes the distinct paths of its followers one at a time (smallest id first), projects every candidate
// onto that path once, and the followers of that path walk the staged arc lengths.
#pragma once

#include <stdint.h>

#include "t2d_obs.cuh"
#include "t2d_route.cuh"
#include "t2d_world.cuh"

namespace t2d {
namespace leader {

constexpr int WARPS = 4;                  // scenarios per CTA
constexpr int NO_PATH = 0x7fffffff;       // the follower takes the heading frame (or has no path left to walk)

struct Args : WorldArgs {
  const int16_t* path_id;                 // [N][M] the controllers' path of every slot, or nullptr: heading frame for all
  PathTable paths;
  double half_width, max_range;
  int16_t* lead;                          // [N][M]
  float* gap;                             // [N][M] or nullptr
};

struct Smem {   // per warp
  double s[128];                          // arc length of each slot on the path being walked
  float x[128], y[128];
  uint8_t cand[128];                      // the slot is a candidate
  uint8_t on[128];                        // ... within half_width of the path being walked
};

// The leaders of scenario n, written by one warp
__device__ __forceinline__ void find_row(const Args& A, Smem& sm, int lane, long long n) {
  const long long base = n * A.M;
  bool fol[4];
  int pend[4];            // the follower's usable path until it has walked it; NO_PATH for the heading frame and when done
  obs::Frame f[4];        // the heading frame
  double best[4];
  int bj[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int m = lane + 32 * k;
    fol[k] = false;
    pend[k] = NO_PATH;
    best[k] = __longlong_as_double(0x7ff0000000000000ll);   // +inf
    bj[k] = -1;
    sm.cand[m] = 0;
    if (m >= A.M) continue;
    const int t = A.type_id[base + m];
    if (t >= A.n_types) continue;   // empty or retired slot: no leader, no candidate
    const float x = A.x[base + m], y = A.y[base + m];
    sm.x[m] = x;
    sm.y[m] = y;
    sm.cand[m] = A.table[t].shape() != SHAPE_NONE;
    fol[k] = !(isnan(x) || isnan(y));
    if (!fol[k]) continue;
    if (A.path_id) {
      const int p = A.path_id[base + m];
      if (A.paths.usable(p)) pend[k] = p;
    }
    if (pend[k] == NO_PATH) {
      f[k].x0 = x;
      f[k].y0 = y;
      obs::sincos_angle((double)A.h[base + m], &f[k].s, &f[k].c);
    }
  }
  __syncwarp();

  // ---- heading frame: every candidate in slot order
  const bool heading = (fol[0] && pend[0] == NO_PATH) || (fol[1] && pend[1] == NO_PATH) ||
                       (fol[2] && pend[2] == NO_PATH) || (fol[3] && pend[3] == NO_PATH);
  if (__any_sync(0xffffffffu, heading)) {
    for (int j = 0; j < A.M; ++j) {
      if (!sm.cand[j]) continue;   // warp-uniform
      const double xj = sm.x[j], yj = sm.y[j];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!fol[k] || pend[k] != NO_PATH || j == lane + 32 * k) continue;
        const double dx = obs::dsub(xj, f[k].x0), dy = obs::dsub(yj, f[k].y0);
        const double ex = f[k].ex(dx, dy), ey = f[k].ey(dx, dy);
        if (ex > 0.0 && fabs(ey) <= A.half_width && ex <= A.max_range && ex < best[k]) {   // NaN fails every test
          best[k] = ex;
          bj[k] = j;
        }
      }
    }
  }

  // ---- path frame: the followers' distinct paths, smallest id first
  for (;;) {
    const int p = __reduce_min_sync(0xffffffffu, min(min(pend[0], pend[1]), min(pend[2], pend[3])));
    if (p == NO_PATH) break;
    const PathVertex* pv = A.paths.v + A.paths.off[p];
    const int nv = A.paths.off[p + 1] - A.paths.off[p];
    double si[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int m = lane + 32 * k;
      si[k] = 0.0;
      bool on = false;
      if (m < A.M && (sm.cand[m] || pend[k] == p)) {   // a follower of p needs its own arc length, candidates theirs
        PathPoint c;
        closest_on_path<true>(pv, nv, (double)sm.x[m], (double)sm.y[m], c);   // p has a segment: c is set
        sm.s[m] = c.s;
        si[k] = c.s;
        on = sm.cand[m] && __dsqrt_rn(c.d2) <= A.half_width;   // a NaN position gives d2 = NaN: never on
      }
      sm.on[m] = on;
    }
    __syncwarp();
    for (int j = 0; j < A.M; ++j) {
      if (!sm.on[j]) continue;   // warp-uniform
      const double sj = sm.s[j];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (pend[k] != p || j == lane + 32 * k) continue;
        const double g = __dsub_rn(sj, si[k]);
        if (g > 0.0 && g <= A.max_range && g < best[k]) {
          best[k] = g;
          bj[k] = j;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (pend[k] == p) pend[k] = NO_PATH;
    __syncwarp();
  }

#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int m = lane + 32 * k;
    if (m >= A.M) continue;
    A.lead[base + m] = (int16_t)bj[k];
    if (A.gap) A.gap[base + m] = __double2float_rn(best[k]);   // +inf without a leader
  }
}

// K17: one warp per scenario
__global__ void __launch_bounds__(WARPS * 32) t2d_leader_kernel(const __grid_constant__ Args A) {
  __shared__ Smem s_all[WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n = (long long)blockIdx.x * WARPS + warp;
  if (n >= A.N) return;   // whole warps
  find_row(A, s_all[warp], lane, n);
}

}  // namespace leader
}  // namespace t2d
