// t2d_replay.cuh - K7 t2d_replay_kernel: recorded tracks pose the replayed slots before K1 / after K2.
#pragma once

#include "t2d_world.cuh"

namespace t2d {

// ---------------------------------------------------------------------------- K7
// Log replay (t2d_set_log): every replayed slot takes its track's state at the time the next tick produces (or, in
// reset mode, at the row's t0), before K1, which then only builds the pose of these static-model slots.  One thread
// per (scenario, slot), consecutive threads on consecutive slots: the [N, M] slot offset reads and the state / type_id
// stores coalesce; the schedule entries, the track entry and its two frame records are gathers.  A slot's schedule is
// a run of entries with strictly increasing, disjoint presence intervals; the thread takes the first entry whose last
// stamp is >= t (the slot's final entry if none is), so a schedule of L entries costs ceil(log2 L) dependent probes.
// When no schedule of the log holds more than one entry (t2d_set_log's row_track, and any such schedule), the host
// uploads the slots' tracks as one [n_rows][M] array instead and the offsets and the entry gather drop out of the
// dependent chain.  Whether the chosen track is present at t is then decided exactly as for a single track.  Interpolation in fp64 with explicit round-to-nearest operations (no FMA
// contraction), in the order oracle/replay.py states.
struct ReplayTrack { int32_t first_ms, period_ms, n_frames, rec_off; };
struct ReplayEntry { int32_t last_ms, track; };   // one 8-byte load per probe

struct ReplayArgs {
  float *x, *y, *h, *v, *vx, *vy;
  uint8_t* type_id;
  const int32_t* step_count;       // [N]
  const int32_t* log_row;          // [N] the row each scenario runs (tick mode)
  const uint8_t* mask;             // reset mode: [N] the scenarios being reset; nullptr in tick mode
  const int32_t* pool_index;       // reset mode: the new row of each masked scenario, nullptr = row n
  int32_t* log_row_out;            // reset mode: log_row, written for the masked scenarios
  const ReplayTrack* tracks;       // [n_tracks]
  const uint8_t* track_type;       // [n_tracks]
  const float* rec;                // [sum n_frames][5] x, y, heading, vx, vy
  const int32_t* t0;               // [n_rows] ms
  const int32_t* slot_off;         // [n_rows * M + 1] schedule of (row, m): entries [slot_off[row M + m], slot_off[row M + m + 1])
  const ReplayEntry* entries;      // [E]
  const int32_t* slot_track1;      // when no schedule has more than one entry: [n_rows * M] its track, -1 for none
                                   // (slot_off / entries then unused); nullptr otherwise
  int32_t* track_out;              // [N][M] the track each slot shows, -1 for none; nullptr: not written
  int N, M, n_rows, offset, interval_ms;
};

__device__ __forceinline__ float replay_lerp(float a, float b, double w) {   // a + w (b - a)
  return __double2float_rn(__dadd_rn((double)a, __dmul_rn(w, __dsub_rn((double)b, (double)a))));
}

// Reactive replay (t2d_set_log_reactive): the per-track tables and the per-slot arrays a handover writes.  The base part
// is the plain kernel's; pid_state / last_accel address the first scenario of the launch like the state does.
struct ReactiveReplayArgs : ReplayArgs {
  const int16_t* track_path;       // [n_tracks] the path of a reactive track, -1: plain replay
  const uint8_t* drive_row;        // [n_tracks] the non-static row that drives a reactive track after its handover
  const float* desired_speed;      // [n_tracks] its IDM desired speed
  int16_t* drive_path;             // [N][M] the path K17 and K5 read, -1 unless the slot shows a reactive track
  float* slot_desired_speed;       // [N][M]
  double* pid_state;               // [N][M][6] or nullptr: the lateral half is zeroed on handover
  float* last_accel;               // [N][M] or nullptr: zeroed on handover
};

// REACTIVE: the reactive instance (t2d_reactive_replay_kernel).  A slot that shows a reactive track k is posed from the
// log only at its handover - reset mode, or the first sample with first_k <= t, i.e. t - first_k < interval_ms - where
// it also takes the track's path and desired speed and a cleared controller state; at every later sample it keeps its
// state and takes the driving row drive_row[k], which the tick integrates.  Every other slot the launch visits gets
// drive_path = -1 and is replayed exactly as by the plain instance.
template <bool REACTIVE, class Args>
__device__ __forceinline__ void replay_body(const Args& A) {
  constexpr double PI_D = 3.141592653589793, TWO_PI_D = 6.283185307179586;
  const long long total = (long long)A.N * A.M;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(i / A.M), m = (int)(i - (long long)n * A.M);
    int row;
    if (A.mask != nullptr) {
      if (!A.mask[n]) continue;
      row = A.pool_index ? A.pool_index[n] : n;
      row = min(max(row, 0), A.n_rows - 1);   // as K2 clamps its pool row (n_pool == n_rows)
      if (m == 0) A.log_row_out[n] = row;
    } else {
      row = min(max(A.log_row[n], 0), A.n_rows - 1);
    }
    const long long s = (long long)row * A.M + m;
    int k;
    long long t;
    if (A.slot_track1 != nullptr) {   // at most one entry per slot: the track itself, no offsets
      k = __ldg(A.slot_track1 + s);
      if (k < 0) {
        if (A.track_out) A.track_out[i] = -1;
        if constexpr (REACTIVE) A.drive_path[i] = -1;
        continue;
      }
      t = (long long)A.t0[row] + ((long long)A.step_count[n] + A.offset) * A.interval_ms;
    } else {
      int lo = __ldg(A.slot_off + s), hi = __ldg(A.slot_off + s + 1) - 1;
      if (hi < lo) {   // an empty schedule: the slot is not replayed
        if (A.track_out) A.track_out[i] = -1;
        if constexpr (REACTIVE) A.drive_path[i] = -1;
        continue;
      }
      t = (long long)A.t0[row] + ((long long)A.step_count[n] + A.offset) * A.interval_ms;
      while (lo < hi) {   // the first entry with last_ms >= t; the final one stands for "after every entry"
        const int mid = (lo + hi) >> 1;
        if ((long long)__ldg(&A.entries[mid].last_ms) >= t) hi = mid;
        else lo = mid + 1;
      }
      k = __ldg(&A.entries[lo].track);
    }
    const int4 tr4 = __ldg(reinterpret_cast<const int4*>(A.tracks) + k);
    const int first = tr4.x, period = tr4.y, n_frames = tr4.z, rec_off = tr4.w;
    const long long d = t - first;
    if (d < 0 || d > (long long)(n_frames - 1) * period) {   // the track is not in the scene at t
      A.type_id[i] = T2D_TYPE_INACTIVE;
      if (A.track_out) A.track_out[i] = -1;
      if constexpr (REACTIVE) A.drive_path[i] = -1;
      continue;
    }
    if (A.track_out) A.track_out[i] = k;
    if constexpr (REACTIVE) {
      const int16_t path = __ldg(A.track_path + k);
      A.drive_path[i] = path;
      if (path >= 0) {
        A.slot_desired_speed[i] = __ldg(A.desired_speed + k);
        if (A.mask == nullptr && d >= (long long)A.interval_ms) {   // simulated: K5 drives it, K1 integrates it
          A.type_id[i] = __ldg(A.drive_row + k);
          continue;
        }
        if (A.pid_state) {   // handover: a fresh controller on the log's state
          double* st = A.pid_state + 6 * i;
          st[0] = 0.0; st[1] = 0.0; st[2] = 0.0;
        }
        if (A.last_accel) A.last_accel[i] = 0.0f;
      }
    }
    const long long j = d / period;
    const int r = (int)(d - j * period);
    const float* a = A.rec + 5 * ((long long)rec_off + j);
    float x, y, h, vx, vy;
    if (r == 0) {   // on a frame: the record, bit for bit
      x = a[0]; y = a[1]; h = a[2]; vx = a[3]; vy = a[4];
    } else {        // between frames j and j + 1 (an extension: the reference has no state there)
      const float* b = a + 5;
      const double w = __ddiv_rn((double)r, (double)period);
      x = replay_lerp(a[0], b[0], w);
      y = replay_lerp(a[1], b[1], w);
      vx = replay_lerp(a[3], b[3], w);
      vy = replay_lerp(a[4], b[4], w);
      const double ha = (double)a[2];
      double dh = __dsub_rn((double)b[2], ha);   // the shorter arc: fold once into [-pi, pi]
      if (dh > PI_D) dh = __dsub_rn(dh, TWO_PI_D);
      else if (dh < -PI_D) dh = __dadd_rn(dh, TWO_PI_D);
      double hh = __dadd_rn(ha, __dmul_rn(w, dh));
      if (hh < 0.0) hh = __dadd_rn(hh, TWO_PI_D);   // wrap once into [0, 2 pi)
      else if (hh >= TWO_PI_D) hh = __dsub_rn(hh, TWO_PI_D);
      h = __double2float_rn(hh);
      if (h == (float)TWO_PI_D) h = 0.0f;   // just below 2 pi, rounded up to fp32(2 pi): the same direction as 0
    }
    // State.speed (state.py:143-146) from the fp32 velocity
    const float v = __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn((double)vx, (double)vx), __dmul_rn((double)vy, (double)vy))));
    A.x[i] = x; A.y[i] = y; A.h[i] = h; A.v[i] = v; A.vx[i] = vx; A.vy[i] = vy;
    A.type_id[i] = A.track_type[k];
  }
}

__global__ void __launch_bounds__(256) t2d_replay_kernel(const __grid_constant__ ReplayArgs A) { replay_body<false>(A); }

__global__ void __launch_bounds__(256) t2d_reactive_replay_kernel(const __grid_constant__ ReactiveReplayArgs A) {
  replay_body<true>(A);
}

}  // namespace t2d
