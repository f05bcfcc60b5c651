// t2d_obs.cuh - K8: the vector observation of every scenario's ego - its own motion, the goal, the nearest participants and
// the nearest map segments, in the ego frame, packed into one fp32 row per scenario.
//
// Contract: DESIGN.md section 1, "Vector observation" (an extension: the reference has no counterpart).  Every value is fp64
// with one round-to-nearest per operation (__dadd_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn, no FMA contraction) in the order
// the float64 oracle (tests/vector_obs_oracle.py) evaluates it, then rounded once to fp32.  The selection is decided by the
// squared distances alone, which involve no trigonometry: selection, order and indices are bit-exact against the oracle.
//
// One warp per scenario.  Agents: the in-range candidates are compacted in slot order and ranked by (d2, slot).  Segments:
// the lanes take the tile's segments 32 at a time; each chunk's in-range candidates are sorted by (d2, index) and merged into a
// running best-S list in shared memory.  Ties in d2 go to the lower index everywhere, so the result does not depend on the
// chunking or on lane order.  The row is assembled in shared memory 32 entries at a time and stored by consecutive lanes.
//
// K9 (t2d_obs_agents_kernel, DESIGN.md section 1 "Per-agent vector observation") is the same row seen from any slot: one warp
// per (scenario, observer) row runs the row routine K8 runs, so a row observed by slot 0 without per-row goals is K8's row.
#pragma once

#include <stdint.h>

#include "t2d_world.cuh"

namespace t2d {
namespace obs {

constexpr int WARPS = 4;              // scenarios per CTA
constexpr int MAX_K = 127;            // agents per row (the other slots of a 128-slot scenario)
constexpr int MAX_S = 256;            // segments per row
constexpr int EGO_F = 8, GOAL_F = 8, AGENT_F = 11, SEG_F = 9;
constexpr unsigned long long NO_KEY = ~0ull;

struct Args : WorldArgs {
  int max_step;
  MapArgs map;
  const float* target;             // [N][5] goal rectangles, or nullptr
  int K, S, F;
  double ra2, rs2;                 // squared ranges
  float* out;                      // [N][F]
  int16_t* agent_index;            // [N][K] or nullptr
  int16_t* segment_index;          // [N][S] or nullptr
};

struct Smem {   // per warp
  unsigned long long bkey[2][MAX_S];   // best-S segments, ascending (d2 bits, index); double-buffered for the merge
  int16_t bidx[2][MAX_S];
  unsigned long long ckey[32];         // this chunk's in-range segments, sorted
  int16_t cidx[32];
  unsigned long long akey[128];        // in-range agents in slot order
  int16_t aslot[128];
  int16_t asel[128];                   // row -> slot
  float stage[32 * AGENT_F];           // 32 rows of the block being written
};

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float f32(double a) { return __double2float_rn(a); }

// A non-negative double's bits order like the double: the key of a squared distance (NaN never becomes a key).
__device__ __forceinline__ unsigned long long key_of(double d2) { return (unsigned long long)__double_as_longlong(d2); }

// v modulo 2, exactly: 0.5 v, its rint and twice that are exact, and so is the difference (|v - 2k| <= 1 is a multiple of
// v's ulp; for |v| >= 2^53 v is itself even and the result is 0).
__device__ __forceinline__ double mod2(double v) { return __dsub_rn(v, 2.0 * rint(0.5 * v)); }

// fp64 (sin a, cos a) for |a| < 2^129 (an fp32 heading or the difference of two) without the library's Payne-Hanek slow path,
// whose local array would be the kernel's only stack.  a / pi = sum_k a P_k with 1 / pi = P_0 + ... + P_4 (265 bits, the
// rest below 2^-272): every product is split exactly into hi + lo by an FMA and each part reduced modulo 2 exactly, so the
// sum q is a / pi modulo 2 up to the rounding of a few additions of numbers below 1 (a few 1e-16), and sincospi(q) finishes
// without any further reduction error.  The result can differ from a correctly rounded sin / cos in the last bits only,
// which the contract's tolerance on the rotated values allows for (DESIGN.md section 1).
__device__ __forceinline__ void sincos_angle(double a, double* s, double* c) {
  const double P[5] = {0x1.45f306dc9c883p-2, -0x1.6b01ec5417056p-56, -0x1.6447e493ad4cep-110, 0x1.e21c820ff28b2p-164,
                       -0x1.508510ea79237p-219};
  double q = 0.0;
#pragma unroll
  for (int k = 4; k >= 0; --k) {   // smallest terms first
    const double hi = __dmul_rn(a, P[k]);
    const double lo = __fma_rn(a, P[k], -hi);
    q = mod2(__dadd_rn(q, __dadd_rn(mod2(lo), mod2(hi))));
  }
  sincospi(q, s, c);
}

struct Frame {   // the ego: origin and (cos, sin) of its heading
  double x0, y0, c, s;
  __device__ __forceinline__ double ex(double dx, double dy) const { return dadd(dmul(c, dx), dmul(s, dy)); }
  __device__ __forceinline__ double ey(double dx, double dy) const { return dadd(dmul(-s, dx), dmul(c, dy)); }
};

// Fields 1..6 of an agent row - ex, ey, cos dh, sin dh, v_x, v_y - of the participant at index p of the arrays (x, y, h, vx,
// vy), in the frame f of an observer whose heading is h0: frame_vals computes them in fp64 ((dx, dy) is the participant's
// offset from the observer's centre), frame_put rounds them into o[0..5].  K8 / K9's agent rows and K16's history rows
// (t2d_history.cuh) both run them, so a history row of the current state is an agent row bit for bit.
struct FrameVals {
  double dx, dy, vx, vy, sd, cd;
};
__device__ __forceinline__ FrameVals frame_vals(const Frame& f, double h0, const float* x, const float* y, const float* h,
                                                const float* vx, const float* vy, long long p) {
  FrameVals r;
  r.dx = dsub(x[p], f.x0); r.dy = dsub(y[p], f.y0);
  r.vx = vx[p]; r.vy = vy[p];
  sincos_angle(dsub(h[p], h0), &r.sd, &r.cd);
  return r;
}
__device__ __forceinline__ void frame_put(const Frame& f, const FrameVals& r, float* o) {
  o[0] = f32(f.ex(r.dx, r.dy)); o[1] = f32(f.ey(r.dx, r.dy)); o[2] = f32(r.cd); o[3] = f32(r.sd);
  o[4] = f32(f.ex(r.vx, r.vy)); o[5] = f32(f.ey(r.vx, r.vy));
}

__device__ __forceinline__ void extents(const Params& p, float& hl, float& hw, float& disc) {
  const int sh = p.shape();
  if (sh == SHAPE_CIRCLE) { hl = hw = p.radius; disc = 1.0f; }
  else if (sh == SHAPE_OBB) { hl = p.half_len; hw = p.half_wid; disc = 0.0f; }
  else { hl = hw = 0.0f; disc = 0.0f; }
}

// Closest point of the segment to the ego centre, relative to it: (px, py) and its squared distance.
__device__ __forceinline__ double seg_closest(const float4 e, const Frame& f, double& px, double& py) {
  const double ax = dsub(e.x, f.x0), ay = dsub(e.y, f.y0);
  const double ux = dsub(e.z, e.x), uy = dsub(e.w, e.y);
  const double uu = dadd(dmul(ux, ux), dmul(uy, uy));
  double t = 0.0;
  if (uu > 0.0) t = fmin(fmax(__ddiv_rn(-dadd(dmul(ax, ux), dmul(ay, uy)), uu), 0.0), 1.0);
  px = dadd(ax, dmul(t, ux));
  py = dadd(ay, dmul(t, uy));
  return dadd(dmul(px, px), dmul(py, py));
}

// Stores n floats of the warp's stage to dst, consecutive lanes on consecutive addresses.
__device__ __forceinline__ void flush(float* dst, const float* stage, int n, int lane) {
  __syncwarp();
  for (int i = lane; i < n; i += 32) dst[i] = stage[i];
  __syncwarp();
}

// An absent row (no observer): F zeros, every index -1.  rid: the row's number in out / agent_index / segment_index.
__device__ __forceinline__ void absent_row(const Args& A, float* row, long long rid, int K, int S, int lane) {
  for (int i = lane; i < A.F; i += 32) row[i] = 0.0f;
  if (A.agent_index) for (int i = lane; i < K; i += 32) A.agent_index[rid * K + i] = -1;
  if (A.segment_index) for (int i = lane; i < S; i += 32) A.segment_index[rid * S + i] = -1;
}

// The row of scenario n seen from its slot jo (0 <= jo < M), written by one warp to row rid of out / agent_index /
// segment_index; the goal rectangle (cx, cy, heading, half_len, half_wid) is row grow of gtab, gtab == nullptr gives the zero
// block.  K8 and K9 both run it; EGO (K8) fixes jo = 0, which keeps K8's candidate test as the slots j >= 1, and takes row n
// of the t2d_set_goal target whatever gtab says.
template <bool EGO>
__device__ __forceinline__ void observe_row(const Args& A, Smem& sm, int lane, long long n, long long rid, int jo,
                                            const float* gtab, long long grow) {
  const long long base = n * A.M;
  const long long po = base + jo;
  float* row = A.out + rid * (long long)A.F;
  const int K = A.K, S = A.S;
  const int t0 = A.type_id[po];
  if (t0 >= A.n_types) {   // no observer: the whole row is zeros, every index -1
    absent_row(A, row, rid, K, S, lane);
    return;
  }
  Frame f;
  f.x0 = A.x[po]; f.y0 = A.y[po];
  const double h0 = A.h[po];
  sincos_angle(h0, &f.s, &f.c);

  // ---- the tile (as K4 finds it)
  const unsigned char* blob = tile_blob(A.map, n);
  const MapHeader* mh = reinterpret_cast<const MapHeader*>(blob);
  const int n_seg = blob ? mh->n_seg : 0;
  const float4* seg = n_seg > 0 ? reinterpret_cast<const float4*>(blob + mh->off_seg) : nullptr;
  int ring_lo = 0, ring_hi = 0;
  if (n_seg > 0 && mh->n_poly > 0) {
    const int32_t* ps = reinterpret_cast<const int32_t*>(blob + mh->off_poly);
    ring_lo = ps[0]; ring_hi = ps[mh->n_poly];
  }

  // ---- agents: compact the in-range candidates in slot order, then rank them by (d2, slot)
  int na = 0;
  if (K > 0) {
    for (int j0 = 0; j0 < A.M; j0 += 32) {
      const int j = j0 + lane;
      bool in = false;
      unsigned long long key = NO_KEY;
      if ((EGO ? j >= 1 : j != jo) && j < A.M) {
        const int t = A.type_id[base + j];
        if (t < A.n_types && A.table[t].shape() != SHAPE_NONE) {
          const double dx = dsub(A.x[base + j], f.x0), dy = dsub(A.y[base + j], f.y0);
          const double d2 = dadd(dmul(dx, dx), dmul(dy, dy));
          in = d2 <= A.ra2;   // NaN fails
          key = key_of(d2);
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, in);
      if (in) {
        const int p = na + __popc(m & ((1u << lane) - 1u));
        sm.akey[p] = key; sm.aslot[p] = (int16_t)j;
      }
      na += __popc(m);
    }
    __syncwarp();
    for (int i = lane; i < na; i += 32) {
      const unsigned long long k = sm.akey[i];
      int r = 0;
      for (int q = 0; q < na; ++q) {
        const unsigned long long kq = sm.akey[q];
        r += (kq < k) || (kq == k && q < i);   // compacted order is slot order
      }
      if (r < K) sm.asel[r] = sm.aslot[i];
    }
    na = min(na, K);
  }

  // ---- segments: a running best-S list, merged with every chunk of 32
  int ns = 0, cur = 0;
  if (S > 0) {
    for (int s0 = 0; s0 < n_seg; s0 += 32) {
      const int si = s0 + lane;
      bool in = false;
      unsigned long long key = NO_KEY;
      if (si < n_seg) {
        double px, py;
        const double d2 = seg_closest(seg[si], f, px, py);
        in = d2 <= A.rs2;
        key = key_of(d2);
        // a full list keeps its own entries on a tie: they have the lower index
        if (in && ns == S) in = key < sm.bkey[cur][S - 1];
      }
      const unsigned m = __ballot_sync(0xffffffffu, in);
      if (m == 0u) continue;
      const int nc = __popc(m);
      int rc = 0;   // rank inside the chunk by (key, lane)
      for (int q = 0; q < 32; ++q) {
        const unsigned long long kq = __shfl_sync(0xffffffffu, key, q);
        rc += ((m >> q) & 1u) && (kq < key || (kq == key && q < lane));
      }
      if (in) { sm.ckey[rc] = key; sm.cidx[rc] = (int16_t)si; }
      __syncwarp();
      const unsigned long long* bk = sm.bkey[cur];
      const int16_t* bi = sm.bidx[cur];
      unsigned long long* nk = sm.bkey[cur ^ 1];
      int16_t* ni = sm.bidx[cur ^ 1];
      if (in) {   // position = best entries with key <= this one (lower index on a tie) + rank in the chunk
        int lo = 0, hi = ns;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (bk[mid] <= key) lo = mid + 1;
          else hi = mid;
        }
        const int p = lo + rc;
        if (p < S) { nk[p] = key; ni[p] = (int16_t)si; }
      }
      for (int i = lane; i < ns; i += 32) {   // position = i + chunk entries with a strictly smaller key
        const unsigned long long k = bk[i];
        int lo = 0, hi = nc;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (sm.ckey[mid] < k) lo = mid + 1;
          else hi = mid;
        }
        const int p = i + lo;
        if (p < S) { nk[p] = k; ni[p] = bi[i]; }
      }
      ns = min(S, ns + nc);
      cur ^= 1;
      __syncwarp();
    }
  }

  // ---- ego and goal: 16 values
  if (lane == 0) {
    float* o = sm.stage;
    const Params& pe = A.table[t0];
    float hl, hw, disc;
    extents(pe, hl, hw, disc);
    const double vx = A.vx[po], vy = A.vy[po];
    o[0] = 1.0f; o[1] = A.v[po];
    o[2] = f32(f.ex(vx, vy)); o[3] = f32(f.ey(vx, vy));
    o[4] = hl; o[5] = hw; o[6] = disc;
    o[7] = A.max_step > 0 ? f32(__ddiv_rn((double)A.step_count[n], (double)A.max_step)) : 0.0f;
    const float* gt = EGO ? A.target : gtab;   // K8: the t2d_set_goal target of the scenario
    if (gt) {
      const float* g = gt + (EGO ? n : grow) * 5;
      const double dx = dsub(g[0], f.x0), dy = dsub(g[1], f.y0);
      double sd, cd;
      sincos_angle(dsub(g[2], h0), &sd, &cd);
      o[8] = 1.0f; o[9] = f32(f.ex(dx, dy)); o[10] = f32(f.ey(dx, dy));
      o[11] = f32(cd); o[12] = f32(sd); o[13] = g[3]; o[14] = g[4];
      o[15] = f32(__dsqrt_rn(dadd(dmul(dx, dx), dmul(dy, dy))));
    } else {
      for (int k = 8; k < 16; ++k) o[k] = 0.0f;
    }
  }
  flush(row, sm.stage, EGO_F + GOAL_F, lane);

  // ---- agent rows, 32 at a time
  for (int r0 = 0; r0 < K; r0 += 32) {
    const int r = r0 + lane, nrow = min(32, K - r0);
    float* o = sm.stage + lane * AGENT_F;
    int j = -1;
    if (r < na) {
      j = sm.asel[r];
      const long long pj = base + j;
      const FrameVals fv = frame_vals(f, h0, A.x, A.y, A.h, A.vx, A.vy, pj);
      float hl, hw, disc;
      extents(A.table[A.type_id[pj]], hl, hw, disc);
      o[0] = 1.0f; frame_put(f, fv, o + 1);
      o[7] = hl; o[8] = hw; o[9] = disc;
      o[10] = f32(__dsqrt_rn(dadd(dmul(fv.dx, fv.dx), dmul(fv.dy, fv.dy))));
    } else if (r < K) {
      for (int k = 0; k < AGENT_F; ++k) o[k] = 0.0f;
    }
    if (A.agent_index && r < K) A.agent_index[rid * K + r] = (int16_t)j;
    flush(row + EGO_F + GOAL_F + r0 * AGENT_F, sm.stage, nrow * AGENT_F, lane);
  }

  // ---- segment rows, 32 at a time
  const int16_t* best = sm.bidx[cur];
  float* srow = row + EGO_F + GOAL_F + K * AGENT_F;
  for (int r0 = 0; r0 < S; r0 += 32) {
    const int r = r0 + lane, nrow = min(32, S - r0);
    float* o = sm.stage + lane * SEG_F;
    int si = -1;
    if (r < ns) {
      si = best[r];
      const float4 e = seg[si];
      double px, py;
      const double d2 = seg_closest(e, f, px, py);
      const double ax = dsub(e.x, f.x0), ay = dsub(e.y, f.y0), bx = dsub(e.z, f.x0), by = dsub(e.w, f.y0);
      o[0] = 1.0f; o[1] = f32(f.ex(ax, ay)); o[2] = f32(f.ey(ax, ay)); o[3] = f32(f.ex(bx, by)); o[4] = f32(f.ey(bx, by));
      o[5] = f32(f.ex(px, py)); o[6] = f32(f.ey(px, py)); o[7] = f32(__dsqrt_rn(d2));
      o[8] = (si >= ring_lo && si < ring_hi) ? 1.0f : 0.0f;
    } else if (r < S) {
      for (int k = 0; k < SEG_F; ++k) o[k] = 0.0f;
    }
    if (A.segment_index && r < S) A.segment_index[rid * S + r] = (int16_t)si;
    flush(srow + r0 * SEG_F, sm.stage, nrow * SEG_F, lane);
  }
}

// K8: the row of every scenario's ego (participant 0), one warp per scenario.
__global__ void __launch_bounds__(WARPS * 32) t2d_obs_kernel(const __grid_constant__ Args A) {
  __shared__ Smem s_all[WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n = (long long)blockIdx.x * WARPS + warp;
  if (n >= A.N) return;
  observe_row<true>(A, s_all[warp], lane, n, n, 0, nullptr, 0);
}

// K9: the rows of a list of observers per scenario, one warp per (scenario, observer) row.  The rows of one scenario are
// consecutive, so the warps of a CTA share its slots and its tile's segments through L1.
struct AgentArgs {
  Args a;                     // out / agent_index / segment_index are indexed by the row n·Q + q
  const int16_t* observers;   // [N][Q], or nullptr: observer q is slot q
  const float* goals;         // [N][Q][5], or nullptr: slot 0's rows take the t2d_set_goal target, the others none
  int Q;
};

__global__ void __launch_bounds__(WARPS * 32) t2d_obs_agents_kernel(const __grid_constant__ AgentArgs G) {
  __shared__ Smem s_all[WARPS];
  const Args& A = G.a;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long rows = (long long)A.N * G.Q;
  for (long long rid = (long long)blockIdx.x * WARPS + warp; rid < rows; rid += (long long)gridDim.x * WARPS) {
    const long long n = rid / G.Q;
    const int q = (int)(rid - n * G.Q);
    const int jo = G.observers ? G.observers[rid] : q;
    if (jo < 0 || jo >= A.M) {   // not a slot: an absent row
      absent_row(A, A.out + rid * (long long)A.F, rid, A.K, A.S, lane);
      continue;
    }
    const float* gtab = nullptr;   // the goal: row grow of gtab
    long long grow = 0;
    if (G.goals) {
      if (!isnan(G.goals[rid * 5])) { gtab = G.goals; grow = rid; }
    } else if (jo == 0) {
      gtab = A.target; grow = n;
    }
    observe_row<false>(A, s_all[warp], lane, n, rid, jo, gtab, grow);
  }
}

}  // namespace obs
}  // namespace t2d
