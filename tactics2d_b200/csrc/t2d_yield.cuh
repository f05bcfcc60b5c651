// t2d_yield.cuh - K19 t2d_yield_kernel: whom every path-following IDM car yields to at the conflict zones of its path, and
// where it stops, which K5's yielding instance takes as a stopped leader.
//
// Contract: DESIGN.md section 1, "Yielding at conflict zones" (an extension, with no reference counterpart).  fp64 with one
// rounding per operation, in the order tests/yield_oracle.py evaluates it.
//   slot path  the path K17 reads (current path: drive_path, lane_path or path_id) when it has a segment of non-zero
//              length; a slot without one takes its route (t2d_set_routes) when that has one: a partner only.  s_k is
//              the arc length of closest_on_path<true> on that path, u_k = max(v_k, v_min).
//   yielder    a slot with a type < n_types, a position that is not NaN, an IDM controller row and a usable current path p.
//              It considers the zones z of p with cd_i = v_i^2 / (2 commit_decel) < d_i = s_in_p - s_i <= max_range.
//   partner    every candidate of K17 (type < n_types, shape not SHAPE_NONE, position not NaN) with a slot path q = z.q;
//              d_j = s_in_q - s_j, t_j = max(d_j, 0) / u_j.  It is cleared when s_j > s_out_q and excluded when it is
//              within half_width of p ahead of i there (K17 already follows it).  i must yield to a partner that is
//              neither, when d_j <= v_j^2 / (2 commit_decel) (committed), or t_j <= critical_gap and priority[q] >
//              priority[p], or t_j <= critical_gap, the priorities are equal and (d_j, j) < (d_i, i).
// The yield zone is the considered zone of smallest d_i (then lowest row) with a must-yield partner: yield_to = its lowest
// such partner, stop_gap = d_i rounded once, stop_xy = the zone's stop point; -1 / +inf without one.
//
// One warp per scenario, four per CTA, lane l owns slots l, l + 32, l + 64, l + 96 (as K17).  Every slot is projected once,
// onto its own slot path, into shared memory; each yielder lane then walks its path's zones from the first one past its
// commit distance (a binary search: the table is sorted by s_in_p) and scans the staged slots for the zone's partners.
// Only a partner that would otherwise force a yield is projected onto p, for the exclusion.
#pragma once

#include <stdint.h>

#include "t2d_route.cuh"
#include "t2d_world.cuh"

namespace t2d {
namespace yield {

constexpr int WARPS = 4;                  // scenarios per CTA

// A zone row on the device: t2d_conflict_zone without s_out_p (no rule reads it), with its stop point
struct Zone {
  double s_in_p, s_in_q, s_out_q;
  double stop_x, stop_y;                  // p's point at arc length clamp(s_in_p, 0, L)
  int32_t q, reserved;
};

struct Args : WorldArgs {
  const int16_t* path_id;                 // [N][M] every slot's current path (K17's)
  const int16_t* route_id;                // [N][M] or nullptr: the routes of partner-only slots
  const uint8_t* ctrl_id;
  const t2d_controller_params* ctab;
  int n_ctrl;
  PathTable paths;
  const Zone* zones;
  const int* zone_off;                    // [n_paths + 1]
  const int16_t* priority;                // [n_paths]
  double half_width, max_range;           // the bound leader search's
  double critical_gap, two_commit_decel, v_min;
  int16_t* yield_to;                      // [N][M]
  float* stop_gap;                        // [N][M]
  double2* stop_xy;                       // [N][M], written where stop_gap is finite
};

struct Smem {   // per warp
  double s[128];                          // arc length of each partner on its slot path
  double cd[128];                         // ... and its commit distance
  float v[128];
  int16_t path[128];                      // the partner's slot path, -1 when the slot is no partner
};

// v^2 / (2 commit_decel): the distance slot speed v needs to stop at commit_decel
__device__ __forceinline__ double commit_distance(const Args& A, double v) {
  return __ddiv_rn(__dmul_rn(v, v), A.two_commit_decel);
}

// The yields of scenario n, written by one warp
__device__ __forceinline__ void find_row(const Args& A, Smem& sm, int lane, long long n) {
  const long long base = n * A.M;
  int own[4];             // the yielder's path, -1 for a slot that does not yield
  double si[4], vi[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int m = lane + 32 * k;
    own[k] = -1;
    si[k] = vi[k] = 0.0;
    if (m >= A.M) continue;
    sm.path[m] = -1;
    const int t = A.type_id[base + m];
    if (t >= A.n_types) continue;   // empty or retired slot
    const float x = A.x[base + m], y = A.y[base + m];
    if (isnan(x) || isnan(y)) continue;
    int p = A.path_id ? (int)A.path_id[base + m] : -1;
    const bool current = A.paths.usable(p);
    if (!current) p = A.route_id && A.paths.usable(A.route_id[base + m]) ? (int)A.route_id[base + m] : -1;
    if (p < 0) continue;
    PathPoint c;
    closest_on_path<true>(A.paths.v + A.paths.off[p], A.paths.off[p + 1] - A.paths.off[p], (double)x, (double)y, c);
    const float v = A.v[base + m];
    if (A.table[t].shape() != SHAPE_NONE) {
      sm.path[m] = (int16_t)p;
      sm.s[m] = c.s;
      sm.cd[m] = commit_distance(A, (double)v);
      sm.v[m] = v;
    }
    const int cid = A.ctrl_id[base + m];
    if (current && cid < A.n_ctrl && A.ctab[cid].kind == T2D_CTRL_IDM) {
      own[k] = p;
      si[k] = c.s;
      vi[k] = (double)v;
    }
  }
  __syncwarp();

#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int m = lane + 32 * k;
    if (m >= A.M) continue;
    int who = -1, zone = -1;
    double gap = __longlong_as_double(0x7ff0000000000000ll);   // +inf
    const int p = own[k];
    if (p >= 0) {
      const double cd = commit_distance(A, vi[k]);
      // the first zone past the commit distance: d_i grows with the row (the rows of p are sorted by s_in_p)
      int lo = A.zone_off[p], hi = A.zone_off[p + 1];
      const int end = hi;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__dsub_rn(A.zones[mid].s_in_p, si[k]) > cd) hi = mid; else lo = mid + 1;
      }
      const int prio_p = A.priority[p];
      const PathVertex* pv = A.paths.v + A.paths.off[p];
      const int nv = A.paths.off[p + 1] - A.paths.off[p];
      for (int z = lo; z < end && who < 0; ++z) {
        const Zone Z = A.zones[z];
        const double di = __dsub_rn(Z.s_in_p, si[k]);
        if (!(di <= A.max_range)) break;
        const int prio_q = A.priority[Z.q];
        for (int j = 0; j < A.M; ++j) {
          if (sm.path[j] != Z.q) continue;
          const double sj = sm.s[j];
          if (sj > Z.s_out_q) continue;   // cleared
          const double dj = __dsub_rn(Z.s_in_q, sj);
          bool must = dj <= sm.cd[j];   // committed
          // else the gap test, where the priorities or the (d, slot) order let it decide
          if (!must && (prio_q > prio_p || (prio_q == prio_p && (dj < di || (dj == di && j < m)))))
            must = __ddiv_rn(fmax(dj, 0.0), fmax((double)sm.v[j], A.v_min)) <= A.critical_gap;
          if (!must) continue;
          PathPoint c;   // excluded: within half_width of p, ahead of i there
          closest_on_path<true>(pv, nv, (double)A.x[base + j], (double)A.y[base + j], c);
          if (__dsqrt_rn(c.d2) <= A.half_width && c.s > si[k]) continue;
          who = j;
          break;
        }
        if (who >= 0) {
          zone = z;
          gap = di;
        }
      }
    }
    A.yield_to[base + m] = (int16_t)who;
    A.stop_gap[base + m] = __double2float_rn(gap);
    if (zone >= 0) A.stop_xy[base + m] = make_double2(A.zones[zone].stop_x, A.zones[zone].stop_y);
  }
}

// K19: one warp per scenario
__global__ void __launch_bounds__(WARPS * 32) t2d_yield_kernel(const __grid_constant__ Args A) {
  __shared__ Smem s_all[WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n = (long long)blockIdx.x * WARPS + warp;
  if (n >= A.N) return;   // whole warps
  find_row(A, s_all[warp], lane, n);
}

}  // namespace yield
}  // namespace t2d
