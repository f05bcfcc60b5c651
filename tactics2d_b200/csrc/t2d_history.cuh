// t2d_history.cuh - the trajectory history of every participant slot: a per-scenario ring of its recent states (K15) and
// their past poses in each observer's current frame (K16).
//
// Contract: DESIGN.md section 1, "Trajectory history" (Trajectory.add_state / reset / history_states,
// participant/trajectory/trajectory.py:115-149,170-188).  The ring holds, for each of x, y, heading, speed, vx, vy, an fp32
// [N][H][M] array, the type ids uint8 [N][H][M] and, while a log schedule with a track output is bound, the shown track
// int32 [N][H][M]; count[n] (int64) is the number of entries since scenario n's episode began, and entry e lives at ring
// index e % H.  Entry e of slot m counts for the slot's current occupant iff it is one of the last min(count, H) entries,
// its type is < n_types and equals the slot's current type id, and (with a track ring) its track equals the slot's current
// track: a history is never spliced across an empty slot, a retired one or a schedule's change of track.
//
// K15 appends the state of every scenario after a tick, or restarts the history of the masked scenarios after a reset (entry 0
// = the state, count = 1): one warp per scenario, M contiguous values per field.  K16 writes, per observer row, HIST_F values
// per lag for the observer itself and for K agent slots: one warp per row, lanes over lags, through a shared-memory stage
// flushed by consecutive lanes, as K8.  The values go through obs::frame_vals / frame_put, the routine of K8 / K9's agent
// rows.
#pragma once

#include <stdint.h>

#include "t2d_obs.cuh"
#include "t2d_world.cuh"

namespace t2d {
namespace hist {

constexpr int MAX_H = 64;
constexpr int HIST_F = 7;       // valid, ex, ey, cos dh, sin dh, v_x, v_y
constexpr int K15_WARPS = 8;    // scenarios per CTA of K15
constexpr int K16_WARPS = 4;    // rows per CTA of K16

struct Ring {   // the world's ring (t2d_set_history)
  float *x, *y, *h, *v, *vx, *vy;   // [N][H][M]
  uint8_t* type;                    // [N][H][M]
  int32_t* track;                   // [N][H][M], or nullptr: no schedule with a track output bound
  long long* count;                 // [N]
  int H;
};

struct AppendArgs : WorldArgs {
  Ring ring;
  const int32_t* track_now;   // [N][M] the track each slot shows (the schedule's track output) when ring.track is set
  const uint8_t* mask;        // [N]: restart the masked scenarios; nullptr: append to every scenario
};

// K15: one warp per scenario.  Lane 0 reads the count and broadcasts it; the warp then owns the scenario's ring entries and
// its count, so nothing races.  Launched without the programmatic-serialization attribute, it starts after the tick (or the
// reset) has completed; it lets the next tick's grid launch at once, whose griddepcontrol.wait then waits for this grid.
__global__ void __launch_bounds__(K15_WARPS * 32) t2d_history_append_kernel(const __grid_constant__ AppendArgs A) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int lane = threadIdx.x & 31;
  const long long n = (long long)blockIdx.x * K15_WARPS + (threadIdx.x >> 5);
  if (n >= A.N) return;   // (warp-uniform, as is the mask below)
  long long e = 0;
  if (A.mask) {
    if (!A.mask[n]) return;
  } else {
    e = __shfl_sync(0xffffffffu, lane == 0 ? A.ring.count[n] : 0ll, 0);
  }
  const Ring& R = A.ring;
  const long long src = n * A.M, dst = (n * R.H + e % R.H) * A.M;
  for (int m = lane; m < A.M; m += 32) {
    R.x[dst + m] = A.x[src + m]; R.y[dst + m] = A.y[src + m]; R.h[dst + m] = A.h[src + m];
    R.v[dst + m] = A.v[src + m]; R.vx[dst + m] = A.vx[src + m]; R.vy[dst + m] = A.vy[src + m];
    R.type[dst + m] = A.type_id[src + m];
    if (R.track) R.track[dst + m] = A.track_now[src + m];
  }
  if (lane == 0) R.count[n] = e + 1;
}

struct ObsArgs : WorldArgs {
  Ring ring;
  const int32_t* track_now;       // as AppendArgs
  const int16_t* observers;       // [N][Q] or nullptr: observer q is slot q (Q > 0)
  int Q;                          // 0: one row per scenario, observed by slot 0 (K8's rows); else Q rows per scenario (K9's)
  const int16_t* agent_index;     // [rows][K] the agent slots of every row, -1 for none (nullptr when K == 0)
  int K;
  float* out;                     // [rows][1 + K][H][HIST_F]
};

struct Smem {   // per warp
  float stage[MAX_H * HIST_F];
};

// The H lags of slot j's history (j outside [0, M) or ok == false: zeros) in the frame (f, h0), into the warp's stage
__device__ __forceinline__ void history_block(const ObsArgs& A, float* stage, int lane, long long n, int j, bool ok,
                                              const obs::Frame& f, double h0, long long n_valid) {
  const Ring& R = A.ring;
  const int H = R.H;
  int t_now = 0, k_now = 0;
  if (ok && j >= 0 && j < A.M) {
    t_now = A.type_id[n * A.M + j];
    if (R.track) k_now = A.track_now[n * A.M + j];
  } else {
    ok = false;
  }
  ok = ok && t_now < A.n_types;
  for (int l = lane; l < H; l += 32) {
    float* o = stage + l * HIST_F;
    bool valid = false;
    long long p = 0;
    if (ok && l < n_valid) {
      const long long e = R.count[n] - 1 - l;
      p = (n * H + e % H) * A.M + j;
      valid = R.type[p] == t_now && (R.track == nullptr || R.track[p] == k_now);
    }
    if (valid) {
      const obs::FrameVals fv = obs::frame_vals(f, h0, R.x, R.y, R.h, R.vx, R.vy, p);
      o[0] = 1.0f;
      obs::frame_put(f, fv, o + 1);
    } else {
      for (int k = 0; k < HIST_F; ++k) o[k] = 0.0f;
    }
  }
}

// K16: one warp per observer row; rows of one scenario are consecutive, so the warps of a CTA share its ring lines in L1.
__global__ void __launch_bounds__(K16_WARPS * 32) t2d_history_obs_kernel(const __grid_constant__ ObsArgs A) {
  __shared__ Smem s_all[K16_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int Q = A.Q > 0 ? A.Q : 1, H = A.ring.H;
  const long long rows = (long long)A.N * Q;
  const long long block_f = (long long)H * HIST_F;
  float* stage = s_all[warp].stage;
  for (long long rid = (long long)blockIdx.x * K16_WARPS + warp; rid < rows; rid += (long long)gridDim.x * K16_WARPS) {
    const long long n = rid / Q;
    const int q = (int)(rid - n * Q);
    const int jo = A.Q == 0 ? 0 : (A.observers ? A.observers[rid] : q);
    bool ok = jo >= 0 && jo < A.M;
    const long long po = n * A.M + (ok ? jo : 0);
    ok = ok && A.type_id[po] < A.n_types;
    obs::Frame f{};
    double h0 = 0.0;
    if (ok) {   // the observer's current frame, as observe_row builds it
      f.x0 = A.x[po]; f.y0 = A.y[po];
      h0 = A.h[po];
      obs::sincos_angle(h0, &f.s, &f.c);
    }
    const long long cnt = A.ring.count[n];
    const long long n_valid = cnt < H ? cnt : H;
    float* row = A.out + rid * (1 + A.K) * block_f;
    for (int b = 0; b <= A.K; ++b) {
      const int j = b == 0 ? jo : A.agent_index[rid * A.K + (b - 1)];
      history_block(A, stage, lane, n, j, ok, f, h0, n_valid);
      obs::flush(row + b * block_f, stage, (int)block_f, lane);
    }
  }
}

}  // namespace hist
}  // namespace t2d
