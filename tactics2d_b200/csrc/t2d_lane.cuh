// t2d_lane.cuh - K18 t2d_lane_change_kernel: MOBIL lane changes (Kesting, Treiber and Helbing 2007) for the IDM rows
// with a lateral channel, decided on the state K5 reads next and written into the slots' current path `lane_path`, which
// K17 and K5 then read instead of the controllers' path_id.  And t2d_lane_reset_kernel, which restarts the reset
// scenarios from their starting lanes.
//
// Contract: DESIGN.md section 1, "Lane changes" (an extension: the reference has no lane-change model).  fp64 with one
// rounding per operation, in the order tests/lane_change_oracle.py evaluates it, except the accelerations, which are
// K5's own idm_law, so that a predicted acceleration is what K5 computes for that pair.
//   candidate    K17's: type < n_types, a shape, a position that is not NaN; on path r when its distance to r (K17's
//                closest_on_path<true>) is <= half_width, s^r its arc length there;
//   changer      an IDM row with a lateral channel, at a position that is not NaN, cooldown 0, its current path p usable
//                (PathTable::usable), itself on p, and a usable neighbour q in {left[p], right[p]};
//   on q         blocked when a candidate on q has |s^q_j - s^q_c| < min_gap; the new leader l' is the candidate on q of
//                smallest s^q_j - s^q_c in (0, max_range], the new follower n the same behind (ties: lower slot); the old
//                leader l and follower o the same on p;
//   decision     a(f | L) = idm_law with f's IDM row (the changer's when f has none), free flow without L; a missing
//                follower gives 0 to both its terms.  Safe: a(n | c) >= -b_safe or no n.  Incentive:
//                (a(c | l') - a(c | l)) + politeness ((a(n | c) - a(n | l')) + (a(o | l) - a(o | c))).  The unblocked
//                safe side of larger incentive > threshold wins, a tie goes left.
// A change writes lane_path = q, cooldown = the bound cooldown, change = +1 (left) / -1 (right); every other slot gets
// change 0 and a positive cooldown counts down by 1.  Decisions are simultaneous: two cars may take the same gap.
//
// One warp per scenario, lane l owns slots l, l + 32, l + 64, l + 96 (as K17).  Positions and speeds are staged in shared
// memory; the warp takes the distinct paths its changers need (their own and their neighbours', smallest id first),
// projects every candidate onto each once, and the changers that need that path walk the staged arc lengths in slot order.
#pragma once

#include <stdint.h>

#include "t2d_control.cuh"
#include "t2d_route.cuh"
#include "t2d_world.cuh"

namespace t2d {
namespace lane {

constexpr int WARPS = 4;                  // scenarios per CTA
constexpr int NO_PATH = 0x7fffffff;       // nothing (left) to walk
constexpr unsigned NONE = 0xffu;          // no slot / no IDM row

struct Args : WorldArgs {
  const t2d_controller_params* ctab;
  int n_ctrl;
  const uint8_t* ctrl_id;                 // [N][M]
  PathTable paths;
  const int16_t* left;                    // [n_paths] device: the left / right neighbour of every path, -1 for none
  const int16_t* right;
  double half_width, max_range;           // the bound leader search's
  double politeness, threshold, b_safe, min_gap;
  int cooldown;
  int16_t* lane_path;                     // [N][M] read and rewritten
  int16_t* cool;                          // [N][M] read and rewritten
  int8_t* change;                         // [N][M] or nullptr
};

struct Smem {   // per warp
  double s[128];                          // arc length of each slot on the path being walked
  float x[128], y[128], v[128];
  uint8_t cand[128];                      // the slot is a candidate
  uint8_t on[128];                        // ... within half_width of the path being walked
  uint8_t row[128];                       // the slot's IDM row, NONE without one
};

// a(f | L): idm_law of slot f behind slot L (L == NONE: free flow), with f's IDM row or `own` when f has none
__device__ __forceinline__ double accel(const Args& A, const Smem& sm, unsigned own, unsigned f, unsigned L) {
  const unsigned r = sm.row[f] != NONE ? sm.row[f] : own;
  const bool has = L != NONE;
  const double xl = has ? (double)sm.x[L] : 0.0, yl = has ? (double)sm.y[L] : 0.0, vl = has ? (double)sm.v[L] : 0.0;
  return idm_law(law_row(A.ctab, (int)r), (double)sm.v[f], (double)sm.x[f], (double)sm.y[f], has, vl, xl, yl);
}

// The lane changes of scenario n, written by one warp
__device__ __forceinline__ void decide_row(const Args& A, Smem& sm, int lane, long long n) {
  const long long base = n * A.M;
  int p0[4], c0[4];       // lane_path and cooldown as read
  int need[4][3];         // the paths of changer k: its own, left, right (NO_PATH: none)
  unsigned pend[4];       // bit e: need[k][e] is still to be walked
  uint32_t near[4];       // l | o << 8 | l'_left << 16 | n_left << 24
  uint32_t far[4];        // l'_right | n_right << 8 | (on p, blocked left, blocked right) << 16
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int m = lane + 32 * k;
    p0[k] = -1; c0[k] = 0;
    need[k][0] = need[k][1] = need[k][2] = NO_PATH;
    pend[k] = 0;
    near[k] = 0xffffffffu; far[k] = 0x0000ffffu;
    sm.cand[m] = 0;
    sm.row[m] = NONE;
    if (m >= A.M) continue;
    p0[k] = A.lane_path[base + m];
    c0[k] = A.cool[base + m];
    const int cid = A.ctrl_id[base + m];
    const bool idm = cid < A.n_ctrl && A.ctab[cid].kind == T2D_CTRL_IDM;
    if (idm) sm.row[m] = (uint8_t)cid;
    const int t = A.type_id[base + m];
    if (t >= A.n_types) continue;   // empty or retired slot: no candidate, no changer
    const float x = A.x[base + m], y = A.y[base + m];
    sm.x[m] = x;
    sm.y[m] = y;
    sm.v[m] = A.v[base + m];
    const bool finite = !(isnan(x) || isnan(y));
    sm.cand[m] = finite && A.table[t].shape() != SHAPE_NONE;
    if (!(finite && idm && A.ctab[cid].pid_lateral != T2D_PID_LAT_NONE && c0[k] <= 0 && A.paths.usable(p0[k]))) continue;
    const int ql = A.left[p0[k]], qr = A.right[p0[k]];
    const bool hl = A.paths.usable(ql), hr = A.paths.usable(qr);
    if (!(hl || hr)) continue;
    need[k][0] = p0[k];
    need[k][1] = hl ? ql : NO_PATH;
    need[k][2] = hr ? qr : NO_PATH;
    pend[k] = 1u | (hl ? 2u : 0u) | (hr ? 4u : 0u);
  }
  __syncwarp();

  // ---- the changers' distinct paths, smallest id first
  for (;;) {
    int mine = NO_PATH;
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int e = 0; e < 3; ++e)
        if (pend[k] & (1u << e)) mine = min(mine, need[k][e]);
    const int r = __reduce_min_sync(0xffffffffu, mine);
    if (r == NO_PATH) break;
    const PathVertex* pv = A.paths.v + A.paths.off[r];
    const int nv = A.paths.off[r + 1] - A.paths.off[r];
    double sc[4];
    bool walk[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int m = lane + 32 * k;
      walk[k] = ((pend[k] & 1u) && need[k][0] == r) || ((pend[k] & 2u) && need[k][1] == r) ||
                ((pend[k] & 4u) && need[k][2] == r);
      sc[k] = 0.0;
      bool on = false;
      if (m < A.M && (sm.cand[m] || walk[k])) {   // a changer needs its own arc length, candidates theirs
        PathPoint c;
        closest_on_path<true>(pv, nv, (double)sm.x[m], (double)sm.y[m], c);   // r has a segment: c is set
        sm.s[m] = c.s;
        sc[k] = c.s;
        const bool within = __dsqrt_rn(c.d2) <= A.half_width;
        on = sm.cand[m] && within;
        if (need[k][0] == r && within) far[k] |= 1u << 16;   // the changer is on its own path
      }
      sm.on[m] = on;
    }
    __syncwarp();
    const double inf = __longlong_as_double(0x7ff0000000000000ll);
    double ba[4], bb[4];
    unsigned ja[4], jb[4];
    bool blk[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { ba[k] = bb[k] = inf; ja[k] = jb[k] = NONE; blk[k] = false; }
    for (int j = 0; j < A.M; ++j) {
      if (!sm.on[j]) continue;   // warp-uniform
      const double sj = sm.s[j];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!walk[k] || j == lane + 32 * k) continue;
        const double g = __dsub_rn(sj, sc[k]), gb = __dsub_rn(sc[k], sj);
        if (fabs(g) < A.min_gap) blk[k] = true;
        if (g > 0.0 && g <= A.max_range && g < ba[k]) { ba[k] = g; ja[k] = (unsigned)j; }
        if (gb > 0.0 && gb <= A.max_range && gb < bb[k]) { bb[k] = gb; jb[k] = (unsigned)j; }
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (!walk[k]) continue;
      const uint32_t pair = ja[k] | (jb[k] << 8);
      if (need[k][0] == r) near[k] = (near[k] & 0xffff0000u) | pair;
      if (need[k][1] == r) {
        near[k] = (near[k] & 0x0000ffffu) | (pair << 16);
        if (blk[k]) far[k] |= 1u << 17;
      }
      if (need[k][2] == r) {
        far[k] = (far[k] & 0xffff0000u) | pair;
        if (blk[k]) far[k] |= 1u << 18;
      }
#pragma unroll
      for (int e = 0; e < 3; ++e)
        if (need[k][e] == r) pend[k] &= ~(1u << e);
    }
    __syncwarp();
  }

  // ---- the decisions, then every slot's outputs
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int m = lane + 32 * k;
    if (m >= A.M) continue;
    int dir = 0, to = p0[k];
    if (need[k][0] != NO_PATH && (far[k] & (1u << 16))) {   // a changer on its own path
      const unsigned c = (unsigned)m, own = sm.row[m];
      const unsigned l = near[k] & 0xffu, o = (near[k] >> 8) & 0xffu;
      const double a_c = accel(A, sm, own, c, l);
      const double d_o = o != NONE ? __dsub_rn(accel(A, sm, own, o, l), accel(A, sm, own, o, c)) : 0.0;
      double best = 0.0;
#pragma unroll
      for (int side = 0; side < 2; ++side) {
        const int q = need[k][1 + side];
        if (q == NO_PATH || (far[k] & (1u << (17 + side)))) continue;   // no usable target, or blocked
        const uint32_t pair = side == 0 ? near[k] >> 16 : far[k] & 0xffffu;
        const unsigned ln = pair & 0xffu, nn = (pair >> 8) & 0xffu;
        const double at_c = accel(A, sm, own, c, ln);
        double d_n = 0.0;
        if (nn != NONE) {
          const double at_n = accel(A, sm, own, nn, c);
          if (!(at_n >= -A.b_safe)) continue;   // unsafe for the new follower
          d_n = __dsub_rn(at_n, accel(A, sm, own, nn, ln));
        }
        const double inc = __dadd_rn(__dsub_rn(at_c, a_c), __dmul_rn(A.politeness, __dadd_rn(d_n, d_o)));
        if (inc > A.threshold && (dir == 0 || inc > best)) {   // left first: a tie stays left
          best = inc;
          dir = side == 0 ? 1 : -1;
          to = q;
        }
      }
    }
    A.lane_path[base + m] = (int16_t)to;
    A.cool[base + m] = (int16_t)(dir != 0 ? A.cooldown : (c0[k] > 0 ? c0[k] - 1 : c0[k]));
    if (A.change) A.change[base + m] = (int8_t)dir;
  }
}

// K18: one warp per scenario
__global__ void __launch_bounds__(WARPS * 32) t2d_lane_change_kernel(const __grid_constant__ Args A) {
  __shared__ Smem s_all[WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n = (long long)blockIdx.x * WARPS + warp;
  if (n >= A.N) return;   // whole warps
  decide_row(A, s_all[warp], lane, n);
}

// The reset scenarios start again from their starting lanes: lane_path = path_id, cooldown = change = 0
struct ResetArgs {
  const uint8_t* mask;                    // [N]
  const int16_t* path_id;                 // [N][M] the controllers'
  int16_t* lane_path;
  int16_t* cool;
  int8_t* change;                         // or nullptr
  long long N;
  int M;
};

__global__ void __launch_bounds__(256) t2d_lane_reset_kernel(const __grid_constant__ ResetArgs A) {
  const long long total = A.N * A.M;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    if (!A.mask[i / A.M]) continue;
    A.lane_path[i] = A.path_id[i];
    A.cool[i] = 0;
    if (A.change) A.change[i] = 0;
  }
}

}  // namespace lane
}  // namespace t2d
