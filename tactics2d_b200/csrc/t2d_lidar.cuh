// t2d_lidar.cuh - K4 t2d_lidar_kernel: single-line lidar of every observer row (per-edge beam windows).
#pragma once

#include "t2d_world.cuh"

namespace t2d {

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

}  // namespace t2d
