// t2d_bev.cuh - K6: the bird's-eye-view observation of every scenario's ego (BEVCamera.update + MatplotlibRenderer,
// tactics2d/sensor/camera.py:333-386, renderer/matplotlib_renderer.py:542-768), rendered on the device.
//
// Contract: DESIGN.md section 1, "BEV observation".  A pixel takes the style of the top-most primitive (largest
// (z, draw index)) whose CLOSED set holds the pixel centre; no antialiasing.  Primitives are closed polygons (a box pose
// ring, its heading triangle, the goal rectangle, a map object's rings under the even-odd rule), discs (pedestrians) and
// strokes with round caps (open map segments).
//
// Every coverage test runs in fp64 with explicitly rounded adds and multiplies (no FMA contraction), on world
// coordinates, in the order the float64 oracle evaluates them: the class image is bit-exact against it.  On H100 fp64
// runs at half the fp32 rate, and the kernel is bound by its image stores, so no fp32 pre-filter is used.
//
// The same kernel renders the view of any list of observer slots per scenario (t2d_bev_render_agents, DESIGN.md section 1
// "Per-agent BEV"; the reference's BEVCamera bound to each row's slot): one CTA per row n·Q + q, centred on the row's slot,
// which draws the scenario's primitives exactly as the ego's view does.  A row differs from the ego's image only in its
// view, its goal rectangle and where it is stored; an absent row stages no primitive, so every pixel is the background.
//
// The predicates are __host__ __device__ so that a g++ build can check them against the oracle.
#pragma once

#include <stdint.h>

#include "t2d_world.cuh"

namespace t2d {
namespace bev {

constexpr int MAX_STYLES = 64;
constexpr int MAX_SIDE = 1024;       // largest image side t2d_bev_render accepts
constexpr int BIN = 16;              // pixel bins are BIN x BIN; the CTA works through the image in bands of BIN rows
constexpr int BINS_X = MAX_SIDE / BIN;
constexpr int MAX_PRIMS = 512;       // visible primitives staged per scenario; beyond that the CTA tests every candidate
constexpr int WORDS = MAX_PRIMS / 32;
constexpr int CTA = 256;
constexpr int STYLE_ARROW = 1;       // row 1 of the style table is the heading arrow, row 0 the background
constexpr uint8_t NO_STYLE = 255;

enum Kind : int { K_POLY = 0, K_DISC = 1, K_STROKE = 2, K_RING = 3 };

// ---- fp64 arithmetic with one rounding per operation (matches NumPy's elementwise float64 bit for bit)
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
#else
// host builds of this header must be compiled with -ffp-contract=off
inline double add(double a, double b) { return a + b; }
inline double sub(double a, double b) { return a - b; }
inline double mul(double a, double b) { return a * b; }
#endif

// Does the ray from (px, py) towards +x cross the edge (x1, y1) -> (x2, y2)?  The half-open rule (y1 > py) != (y2 > py)
// counts a vertex once; the intercept test px < x(py) is the sign of the edge function, free of a division.
T2D_HD bool ray_crosses(double x1, double y1, double x2, double y2, double px, double py) {
  if ((y1 > py) == (y2 > py)) return false;
  const double c = sub(mul(sub(x2, x1), sub(py, y1)), mul(sub(y2, y1), sub(px, x1)));
  return y2 > y1 ? c > 0.0 : c < 0.0;
}

// Squared distance from (px, py) to the segment <= hw2 (hw2 = 0: the point lies on the segment).
T2D_HD bool near_segment(double x1, double y1, double x2, double y2, double px, double py, double hw2) {
  const double dx = sub(x2, x1), dy = sub(y2, y1), ux = sub(px, x1), uy = sub(py, y1);
  const double t = add(mul(ux, dx), mul(uy, dy));
  if (t <= 0.0) return add(mul(ux, ux), mul(uy, uy)) <= hw2;
  const double dd = add(mul(dx, dx), mul(dy, dy));
  if (t >= dd) {
    const double vx = sub(px, x2), vy = sub(py, y2);
    return add(mul(vx, vx), mul(vy, vy)) <= hw2;
  }
  const double c = sub(mul(dx, uy), mul(dy, ux));
  return mul(c, c) <= mul(hw2, dd);
}

T2D_HD bool in_disc(double cx, double cy, double r2, double px, double py) {
  const double ux = sub(px, cx), uy = sub(py, cy);
  return add(mul(ux, ux), mul(uy, uy)) <= r2;
}

// Closed polygon of n vertices (a convex pose ring or triangle): inside by the even-odd rule, or on an edge.
T2D_HD bool in_polygon(const double* vx, const double* vy, int n, double px, double py) {
  bool in = false;
  for (int i = 0; i < n; ++i) {
    const int j = i + 1 == n ? 0 : i + 1;
    if (near_segment(vx[i], vy[i], vx[j], vy[j], px, py, 0.0)) return true;
    in ^= ray_crosses(vx[i], vy[i], vx[j], vy[j], px, py);
  }
  return in;
}

// Pose ring of a box (vehicle.py:133-140,272-281): corner i = (x + lx c - ly s, y + lx s + ly c).
T2D_HD void box_ring(double x, double y, double c, double s, double l, double w, double* vx, double* vy) {
  const double lx[4] = {l, l, -l, -l}, ly[4] = {-w, w, w, -w};
  for (int i = 0; i < 4; ++i) {
    vx[i] = sub(add(x, mul(lx[i], c)), mul(ly[i], s));
    vy[i] = add(add(y, mul(lx[i], s)), mul(ly[i], c));
  }
}

// Heading triangle (camera.py:263-268): midpoints of ring edges 0-1, 1-2 and 3-0.
T2D_HD void arrow_of(const double* rx, const double* ry, double* vx, double* vy) {
  const int a[3] = {0, 1, 3}, b[3] = {1, 2, 0};
  for (int i = 0; i < 3; ++i) {
    vx[i] = mul(add(rx[a[i]], rx[b[i]]), 0.5);
    vy[i] = mul(add(ry[a[i]], ry[b[i]]), 0.5);
  }
}

// Pixel centre (row r, column c) -> world: view coordinates (u, v) in the widened window, rotated by the view yaw
// and moved to the view centre.
struct View {
  double ex, ey, cs, sn;   // view centre and (cos, sin) of the view yaw
};
struct Window {
  double xmin, ymax, px, py;   // left edge, top edge (view frame), pixel pitch along x and y
};
T2D_HD void pixel_world(const View& v, const Window& w, int r, int c, double& X, double& Y) {
  const double u = add(w.xmin, mul((double)c + 0.5, w.px));
  const double q = sub(w.ymax, mul((double)r + 0.5, w.py));
  X = sub(add(v.ex, mul(v.cs, u)), mul(v.sn, q));
  Y = add(add(v.ey, mul(v.sn, u)), mul(v.cs, q));
}

}  // namespace bev

// ============================================================================ K6
#if defined(__CUDACC__)
namespace bev {

struct Args : WorldArgs {
  MapArgs map;
  const uint8_t* seg_style;        // per segment, tiles back to back (seg_base[tile] + segment), or nullptr: defaults
  const uint32_t* seg_base;        // [n_tiles]
  const float* target;             // [N][5] goal rectangles, or nullptr
  int target_style;                // NO_STYLE: the goal is not drawn
  int ring_style, open_style;      // defaults of a ring object and of an open segment
  int W, H, rgb;
  Window win;
  double hw2[MAX_STYLES];          // squared half-width of a stroke of each style, in metres
  uint8_t type_style[T2D_MAX_TYPES];
  uint8_t style_rgb[MAX_STYLES][3];
  int8_t style_z[MAX_STYLES];
  uint8_t* out;                    // [N][Q][H][W](3)
  // the rows of t2d_bev_render_agents (the ego's view reads none of these)
  const int16_t* observers;        // [N][Q] the slot observing row n·Q + q, or nullptr: row q is slot q
  const float* goals;              // [N][Q][5] the goal rectangle of every row (NaN cx: none), or nullptr
  int Q;                           // rows per scenario (1 for the ego's view)
};

struct Prim {
  uint32_t key;               // (z + 128) << 24 | draw index
  uint8_t kind, style, nv;
  int r0, r1, c0, c1;         // pixel rows / columns that may hold a covered centre
  int s0, s1;                 // K_RING: segment range in the blob
  double g[8];                // K_POLY: nv vertices (x[0..nv), then y at +4); K_DISC: cx, cy, r2; K_STROKE: x1, y1, x2, y2
};

struct Scene {   // per row, shared
  View view;
  const unsigned char* blob;
  const float4* seg;
  const int32_t* pstart;
  const float4* pbox;
  const uint8_t* sstyle;
  int n_seg, n_poly, ring_lo, ring_hi, n_cand;
};

__device__ __forceinline__ int seg_style_of(const Args& A, const Scene& S, int s, int dflt) {
  return S.sstyle ? S.sstyle[s] : dflt;
}

// Fractional pixel coordinates of a world point (for bounding boxes only; exactness is not needed there).
__device__ __forceinline__ void to_pixel(const Args& A, const View& v, double X, double Y, double& fc, double& fr) {
  const double dx = X - v.ex, dy = Y - v.ey;
  const double u = v.cs * dx + v.sn * dy, q = -v.sn * dx + v.cs * dy;
  fc = (u - A.win.xmin) / A.win.px;
  fr = (A.win.ymax - q) / A.win.py;
}

// Candidate i of the scenario in draw order: 0 the goal rectangle, then the rings, then the open segments, then per
// participant its body and heading arrow.  Returns false when the candidate draws nothing or misses the image.  The goal
// is the scenario's target, or with ROWS the row's goal `goal` (nullptr: none).
template <bool ROWS>
__device__ bool make_prim(const Args& A, const Scene& S, const float* goal, long long n, int i, Prim& p) {
  double bx0 = INFINITY, bx1 = -INFINITY, by0 = INFINITY, by1 = -INFINITY, grow = 0.0;
  auto pt = [&](double X, double Y) {
    double fc, fr;
    to_pixel(A, S.view, X, Y, fc, fr);
    bx0 = fmin(bx0, fc); bx1 = fmax(bx1, fc); by0 = fmin(by0, fr); by1 = fmax(by1, fr);
  };
  int z, draw;
  if (i == 0) {   // the goal rectangle
    if (!(ROWS ? goal : A.target) || A.target_style == NO_STYLE) return false;
    const float* t = ROWS ? goal : A.target + n * 5;
    double s, c;
    sincos((double)t[2], &s, &c);
    box_ring(t[0], t[1], c, s, t[3], t[4], p.g, p.g + 4);
    p.kind = K_POLY; p.nv = 4; p.style = (uint8_t)A.target_style; draw = 0;
    for (int k = 0; k < 4; ++k) pt(p.g[k], p.g[4 + k]);
  } else if (i < 1 + S.n_poly) {   // ring object p: its box from the blob; the edges stay in global memory
    const int q = i - 1;
    p.kind = K_RING; p.s0 = S.pstart[q]; p.s1 = S.pstart[q + 1];
    const int st = seg_style_of(A, S, p.s0, A.ring_style);
    if (st == NO_STYLE) return false;
    p.style = (uint8_t)st; draw = 1 + p.s0;
    const float4 b = S.pbox[q];
    pt(b.x, b.z); pt(b.x, b.w); pt(b.y, b.z); pt(b.y, b.w);
  } else if (i < 1 + S.n_poly + S.n_seg) {   // open segment
    const int s = i - 1 - S.n_poly;
    if (s >= S.ring_lo && s < S.ring_hi) return false;
    const int st = seg_style_of(A, S, s, A.open_style);
    if (st == NO_STYLE) return false;
    const float4 e = S.seg[s];
    p.kind = K_STROKE; p.style = (uint8_t)st; draw = 1 + s;
    p.g[0] = e.x; p.g[1] = e.y; p.g[2] = e.z; p.g[3] = e.w; p.g[4] = A.hw2[st];
    pt(e.x, e.y); pt(e.z, e.w);
    grow = sqrt(A.hw2[st]) / fmin(A.win.px, A.win.py);
  } else {   // participant j: body (even k) or heading arrow (odd k)
    const int k = i - 1 - S.n_poly - S.n_seg, j = k >> 1;
    const long long pj = n * A.M + j;
    const int t = A.type_id[pj];
    if (t >= A.n_types || A.type_style[t] == NO_STYLE) return false;
    const Params& tp = A.table[t];
    const int shape = tp.shape();
    draw = 1 + 32767 + k;
    const double x = A.x[pj], y = A.y[pj];
    if (shape == SHAPE_CIRCLE) {
      if (k & 1) return false;
      const double r = tp.pose_l;
      p.kind = K_DISC; p.style = A.type_style[t];
      p.g[0] = x; p.g[1] = y; p.g[2] = mul(r, r);
      pt(x - r, y - r); pt(x + r, y + r); pt(x - r, y + r); pt(x + r, y - r);
    } else if (shape == SHAPE_OBB) {
      double s, c, rx[4], ry[4];
      sincos((double)A.h[pj], &s, &c);
      box_ring(x, y, c, s, tp.pose_l, tp.pose_w, rx, ry);
      p.kind = K_POLY;
      if (k & 1) {
        arrow_of(rx, ry, p.g, p.g + 4);
        p.nv = 3; p.style = STYLE_ARROW;
      } else {
        for (int v = 0; v < 4; ++v) { p.g[v] = rx[v]; p.g[4 + v] = ry[v]; }
        p.nv = 4; p.style = A.type_style[t];
      }
      for (int v = 0; v < p.nv; ++v) pt(p.g[v], p.g[4 + v]);
    } else {
      return false;
    }
  }
  z = A.style_z[p.style];
  p.key = ((uint32_t)(z + 128) << 24) | (uint32_t)draw;
  // a pixel centre sits at (c + 0.5, r + 0.5): one pixel of slack covers the rounding of to_pixel
  grow += 1.0;
  if (!(bx1 + grow >= 0.0 && by1 + grow >= 0.0 && bx0 - grow <= (double)A.W && by0 - grow <= (double)A.H)) return false;
  p.c0 = max(0, (int)floor(bx0 - grow)); p.c1 = min(A.W - 1, (int)ceil(bx1 + grow));
  p.r0 = max(0, (int)floor(by0 - grow)); p.r1 = min(A.H - 1, (int)ceil(by1 + grow));
  return p.c0 <= p.c1 && p.r0 <= p.r1;
}

__device__ __forceinline__ bool covers(const Prim& p, const Scene& S, const Args& A, double X, double Y) {
  switch (p.kind) {
    case K_POLY: return in_polygon(p.g, p.g + 4, p.nv, X, Y);
    case K_DISC: return in_disc(p.g[0], p.g[1], p.g[2], X, Y);
    case K_STROKE: return near_segment(p.g[0], p.g[1], p.g[2], p.g[3], X, Y, p.g[4]);
    default: {   // a map object: even-odd over the edges of all its rings, or on one of them
      bool in = false;
      for (int s = p.s0; s < p.s1; ++s) {
        const float4 e = S.seg[s];
        if (near_segment(e.x, e.y, e.z, e.w, X, Y, 0.0)) return true;
        in ^= ray_crosses(e.x, e.y, e.z, e.w, X, Y);
      }
      return in;
    }
  }
}

struct Smem {
  Scene S;
  int count;
  uint32_t key[MAX_PRIMS];
  uint16_t order[MAX_PRIMS];    // rank (0 = top-most) -> staged slot
  uint32_t mask[BINS_X][WORDS]; // this band's bins: bit r = the primitive of rank r may cover a centre of the bin
  Prim prim[MAX_PRIMS];
  const float* goal;            // ROWS: the row's goal rectangle (cx, cy, heading, half_len, half_wid), or nullptr
};

__device__ __forceinline__ void store_run(const Args& A, long long row, long long off, int len, const uint8_t (&cls)[16]) {
  if (!A.rgb) {
    uint8_t* dst = A.out + row * (long long)A.W * A.H + off;
    if (len == 16 && ((uintptr_t)dst & 15) == 0) {
      uint4 v;
      memcpy(&v, cls, 16);
      *reinterpret_cast<uint4*>(dst) = v;
    } else {
      for (int k = 0; k < len; ++k) dst[k] = cls[k];
    }
    return;
  }
  uint8_t* dst = A.out + (row * (long long)A.W * A.H + off) * 3;
  uint8_t px[48];
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    px[3 * k] = A.style_rgb[cls[k]][0];
    px[3 * k + 1] = A.style_rgb[cls[k]][1];
    px[3 * k + 2] = A.style_rgb[cls[k]][2];
  }
  if (len == 16 && ((uintptr_t)dst & 15) == 0) {
    uint4 v[3];
    memcpy(v, px, 48);
    uint4* d = reinterpret_cast<uint4*>(dst);
    d[0] = v[0]; d[1] = v[1]; d[2] = v[2];
  } else {
    for (int k = 0; k < 3 * len; ++k) dst[k] = px[k];
  }
}

// View centred on slot pj (a global slot index), +x along its heading
__device__ __forceinline__ View slot_view(const Args& A, long long pj) {
  View v;
  v.ex = A.x[pj]; v.ey = A.y[pj];
  sincos((double)A.h[pj], &v.sn, &v.cs);
  return v;
}

// ROWS = false: the ego's view (t2d_bev_render), one CTA per scenario.  ROWS = true: one CTA per observer row n·Q + q
// (t2d_bev_render_agents); with Q = 1 and no list that is slot 0's view, except that a scenario without slot 0 gives an
// absent row instead of the no-ego view.
template <bool ROWS>
__global__ void __launch_bounds__(CTA) t2d_bev_kernel(const __grid_constant__ Args A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  Scene& S = sm.S;
  const long long row = blockIdx.x;
  const long long n = ROWS ? row / A.Q : row;
  const int tid = threadIdx.x;
  if (tid == 0) {
    const unsigned char* blob = tile_blob(A.map, n);
    const MapHeader* mh = reinterpret_cast<const MapHeader*>(blob);
    S.blob = blob;
    S.n_seg = blob ? mh->n_seg : 0;
    S.n_poly = blob ? mh->n_poly : 0;
    S.seg = blob ? reinterpret_cast<const float4*>(blob + mh->off_seg) : nullptr;
    S.pstart = blob ? reinterpret_cast<const int32_t*>(blob + mh->off_poly) : nullptr;
    S.pbox = blob ? reinterpret_cast<const float4*>(blob + mh->off_pbox) : nullptr;
    S.ring_lo = S.n_poly > 0 ? S.pstart[0] : 0;
    S.ring_hi = S.n_poly > 0 ? S.pstart[S.n_poly] : 0;
    S.sstyle = A.seg_style ? A.seg_style + A.seg_base[A.map.tile_id ? A.map.tile_id[n] : 0] : nullptr;
    S.n_cand = 1 + S.n_poly + S.n_seg + 2 * A.M;
    View v;
    if (ROWS) {
      const int q = (int)(row - n * A.Q);
      const int j = A.observers ? (int)A.observers[row] : q;   // the observing slot
      v = View{0.0, 0.0, 1.0, 0.0};
      if (j >= 0 && j < A.M && A.type_id[n * A.M + j] < A.n_types) v = slot_view(A, n * A.M + j);
      else S.n_cand = 0;   // not a slot, an empty or a retired one: an absent row, all background
      // the goal (observe_agents' rule): the row's own (NaN cx: none), or without goals the target for slot 0 only
      if (A.goals) sm.goal = isnan(A.goals[row * 5]) ? nullptr : A.goals + row * 5;
      else sm.goal = j == 0 && A.target ? A.target + n * 5 : nullptr;
    } else if (A.type_id[n * A.M] < A.n_types) {   // the ego: centred, +x along its heading
      v = slot_view(A, n * A.M);
    } else {   // no ego (sensor_base.py:185-191): the tile's bounds box centre, or the origin; yaw 0
      v.ex = v.ey = 0.0;
      if (blob && mh->has_bounds) {
        v.ex = mul(add((double)mh->bxmin, (double)mh->bxmax), 0.5);
        v.ey = mul(add((double)mh->bymin, (double)mh->bymax), 0.5);
      }
      v.cs = 1.0; v.sn = 0.0;
    }
    S.view = v;
    sm.count = 0;
  }
  __syncthreads();
  // ---- stage the visible primitives
  const float* goal = ROWS ? sm.goal : nullptr;
  for (int i = tid; i < S.n_cand; i += CTA) {
    Prim p;
    if (make_prim<ROWS>(A, S, goal, n, i, p)) {
      const int slot = atomicAdd(&sm.count, 1);
      if (slot < MAX_PRIMS) { sm.prim[slot] = p; sm.key[slot] = p.key; }
    }
  }
  __syncthreads();
  const int P = sm.count;
  const bool staged = P <= MAX_PRIMS;
  if (staged) {   // rank by key, largest first (keys are distinct: the draw index is unique)
    for (int i = tid; i < P; i += CTA) {
      const uint32_t k = sm.key[i];
      int r = 0;
      for (int j = 0; j < P; ++j) r += sm.key[j] > k;
      sm.order[r] = (uint16_t)i;
    }
  }
  const int nw = (P + 31) >> 5, nbx = (A.W + BIN - 1) / BIN;
  for (int band = 0; band * BIN < A.H; ++band) {
    const int row0 = band * BIN, row1 = min(A.H, row0 + BIN);
    if (staged) {
      __syncthreads();   // the previous band's pixels are done with the masks
      for (int k = tid; k < nbx * WORDS; k += CTA) sm.mask[k / WORDS][k % WORDS] = 0u;
      __syncthreads();
      for (int r = tid; r < P; r += CTA) {
        const Prim& p = sm.prim[sm.order[r]];
        if (p.r1 < row0 || p.r0 >= row1) continue;
        for (int b = p.c0 / BIN; b <= p.c1 / BIN; ++b) atomicOr(&sm.mask[b][r >> 5], 1u << (r & 31));
      }
      __syncthreads();
    }
    // ---- pixels: a thread owns a run of 16 consecutive pixels in flat order
    const int f0 = row0 * A.W, f1 = row1 * A.W;
    for (int off = f0 + 16 * tid; off < f1; off += 16 * CTA) {
      const int len = min(16, f1 - off);
      uint8_t cls[16];
#pragma unroll 1
      for (int k = 0; k < 16; ++k) {
        cls[k] = 0;
        if (k >= len) continue;
        const int r = (off + k) / A.W, c = (off + k) - r * A.W;
        double X = 0.0, Y = 0.0;
        if (staged) {   // the pixel centre's world coordinates are computed once a primitive's box holds the pixel
          const uint32_t* m = sm.mask[c / BIN];
          bool hit = false, placed = false;
          for (int w = 0; w < nw && !hit; ++w) {
            uint32_t bits = m[w];
            while (bits) {
              const int rank = (w << 5) + __ffs(bits) - 1;
              bits &= bits - 1;
              const Prim& p = sm.prim[sm.order[rank]];
              if (r < p.r0 || r > p.r1 || c < p.c0 || c > p.c1) continue;
              if (!placed) { pixel_world(S.view, A.win, r, c, X, Y); placed = true; }
              if (covers(p, S, A, X, Y)) { cls[k] = p.style; hit = true; break; }
            }
          }
        } else {   // more visible primitives than shared memory holds: every candidate, top-most by key
          pixel_world(S.view, A.win, r, c, X, Y);
          uint32_t best = 0;
          for (int i = 0; i < S.n_cand; ++i) {
            Prim p;
            if (!make_prim<ROWS>(A, S, goal, n, i, p) || p.key <= best) continue;
            if (r < p.r0 || r > p.r1 || c < p.c0 || c > p.c1) continue;
            if (covers(p, S, A, X, Y)) { best = p.key; cls[k] = p.style; }
          }
        }
      }
      store_run(A, row, off, len, cls);
    }
  }
}

}  // namespace bev
#endif

}  // namespace t2d
