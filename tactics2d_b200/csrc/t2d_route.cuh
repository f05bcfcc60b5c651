// t2d_route.cuh - the polyline table and its path geometry (closest point, OffRoute probe) that K5, K17-K19, the
// epilogues and K12 read, and K12 t2d_route_obs_kernel (the route of every observer row in its frame).
#pragma once

#include "t2d_world.cuh"

namespace t2d {

// ---------------------------------------------------------------------------- route following
// DESIGN.md section 1 "Route following": the polyline table (t2d_set_paths) read by K5's PATH sources, the traffic
// stages K17-K19, the OffRoute detector and route progress of the epilogues, and K12.
struct PathVertex { double x, y, cum, len; };   // vertex, arc length up to it, length of the segment that starts here

// The bound polyline table: path p in [0, n) owns v[off[p] .. off[p + 1]); n == 0 when none is bound
struct PathTable {
  const PathVertex* v;
  const int* off;
  int n;

  // The polyline of path p into (pv, n_vert); false, with both left alone, when p is not a path of the table
  __device__ __forceinline__ bool vertices(int p, const PathVertex*& pv, int& n_vert) const {
    if (p < 0 || p >= n) return false;
    n_vert = off[p + 1] - off[p];
    pv = v + off[p];
    return true;
  }

  // p is a path of the table with a segment of non-zero length: closest_on_path's test, segment by segment
  __device__ __forceinline__ bool usable(int p) const {
    if (p < 0 || p >= n) return false;
    const PathVertex* pv = v + off[p];
    const int n_vert = off[p + 1] - off[p];
    for (int i = 0; i + 1 < n_vert; ++i) {
      const double dx = __dsub_rn(pv[i + 1].x, pv[i].x), dy = __dsub_rn(pv[i + 1].y, pv[i].y);
      if (__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)) > 0.0) return true;
    }
    return false;
  }
};

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
  PathTable paths;
  float off_reward;                 // the reward of an off-route step
  double threshold, weight;         // OffRoute threshold (m), progress weight (per m)
};

// The polyline of slot i's route, or nullptr
__device__ __forceinline__ const PathVertex* route_of(const RouteArgs& R, long long i, int& n_vert) {
  const PathVertex* pv = nullptr;
  R.paths.vertices(R.route_id[i], pv, n_vert);
  return pv;
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

}  // namespace t2d
