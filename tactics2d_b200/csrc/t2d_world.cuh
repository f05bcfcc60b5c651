// t2d_world.cuh - what more than one kernel family reads: the launch-shape constants, the map tile header, the
// bound world, map and goal detectors as the kernels take them, the PTX and vector helpers, the collision primitives
// K1 and K14 share and the Arrival / NoAction detectors K1 and K10 share.
#pragma once

#include <stddef.h>
#include <stdint.h>

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

}  // namespace t2d
