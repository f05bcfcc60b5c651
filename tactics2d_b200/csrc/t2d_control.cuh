// t2d_control.cuh - K5 t2d_control_kernel: the NPC controllers (IDM, cruise / adaptive cruise, pure pursuit, PID).
#pragma once

#include "t2d_route.cuh"
#include "t2d_world.cuh"

namespace t2d {

// ============================================================================ K5: NPC controllers
// One warp per scenario; lane l owns participants l, l + 32, ... .  fp64 on the fp32 state (a few dozen flops per
// participant: the kernel is bound by its ~30 B / participant of HBM traffic).  All reads of last_accel (own and the
// leader's, previous tick) happen before the warp barrier, all writes (this tick) after it.

// The leading fields of t2d_controller_params, the only ones the IDM / cruise / pure-pursuit laws read.  The row also
// holds doubles (the PID part), so it is 8-byte aligned; read through this 4-byte-aligned view, those laws load their
// fields one by one as they did before the row grew.
struct CtrlLawRow {
  int32_t kind;
  float desired_speed, time_headway, min_spacing, max_acceleration, comfortable_deceleration, delta;
  float target_speed, kp, accel_change_rate, delta_t, max_accel, min_accel, interval;
  float min_pre_aiming_distance, pp_interval, wheel_base;
};
static_assert(alignof(CtrlLawRow) == 4 && offsetof(CtrlLawRow, wheel_base) == offsetof(t2d_controller_params, wheel_base),
              "CtrlLawRow is the float prefix of t2d_controller_params");

struct CtrlArgs : WorldArgs {
  const t2d_controller_params* ctab;
  int n_ctrl;
  const uint8_t* ctrl_id;
  const int16_t* lead;
  const int16_t* path_id;
  PathTable paths;
  float* last_accel;
  float* action;
  const float* ego_action;   // [N][2] or nullptr: participant 0's action (written into its row of `action` as well)
  int steer_first;
  const float* pid_target;   // [N][M][2] (target_speed, lateral target) or nullptr; read by the HAS_PID instance only
  double* pid_state;         // [N][M][6] or nullptr; read and written by the HAS_PID instance only
  const float* slot_desired_speed;   // [N][M]: the reactive instance's IDM desired speed of every slot with a path
  const float* stop_gap;             // [N][M]: the yielding instance's K19 output, +inf where the slot does not yield
  const double2* stop_xy;            // [N][M]: ... and the stop point where it does
};

__device__ __forceinline__ double clip_np(double v, double lo, double hi) {   // np.clip: NaN propagates
  return v != v ? v : fmin(fmax(v, lo), hi);
}

// acceleration_controller.py:82-130: cruise, or adaptive cruise when a leader is given
__device__ double longitudinal_law(const CtrlLawRow& p, double v, double x, double y, double a_last, bool has_lead,
                                   double vl, double xl, double yl, double al) {
  const double kp = (double)p.kp;
  double a;
  if (has_lead) {
    const double d_front = sqrt((x - xl) * (x - xl) + (y - yl) * (y - yl));                  // :114
    const double d_target = clip_np(v * (double)p.interval + 5.0, 7.0, 80.0);                // :115-118, :42-45
    const double rel_speed = vl - v;                                                         // :120
    const double rel_target_speed = (d_target - d_front) / kp;                               // :121
    const double rel_accel = (rel_target_speed - rel_speed) / kp;                            // :122
    a = al - rel_accel;                                                                      // :124
  } else {
    a = ((double)p.target_speed - v) / kp;                                                   // :94
  }
  const double w = (double)p.accel_change_rate * (double)p.delta_t;
  a = clip_np(a, a_last - w, a_last + w);                                                    // :95-99, :126-130
  return clip_np(a, (double)p.min_accel, (double)p.max_accel);
}

// (v / v_des) ** delta: the IDM exponent is 4 by default - two multiplications instead of the general pow()
__device__ __forceinline__ double idm_pow(double r, double delta) {
  if (delta == 4.0) { const double r2 = r * r; return r2 * r2; }
  if (delta == 2.0) return r * r;
  return pow(r, delta);
}

// idm_controller.py:59-141
__device__ double idm_law(const CtrlLawRow& p, double v, double x, double y, bool has_lead, double vl, double xl,
                          double yl) {
  const double vd = (double)p.desired_speed, am = (double)p.max_acceleration, b = (double)p.comfortable_deceleration;
  double a;
  if (!has_lead) {
    a = vd > 0.0 ? am * (1.0 - idm_pow(v / vd, (double)p.delta)) : (v > 0.0 ? -b : 0.0);     // :74-82
  } else {
    const double dist = sqrt((xl - x) * (xl - x) + (yl - y) * (yl - y));                     // :107-109 (np.hypot, no overflow concern at map scale)
    const double dv = vl - v;                                                                // :112
    double s_star = (double)p.min_spacing + v * (double)p.time_headway + (v * dv) / (2.0 * sqrt(am * b));   // :116-120
    s_star = fmax(s_star, (double)p.min_spacing);                                            // :121
    if (dist > 0.0) {
      const double ratio = vd > 0.0 ? idm_pow(v / vd, (double)p.delta) : (v > 0.0 ? 1.0 : 0.0);  // :127-130
      const double q = s_star / dist;
      a = am * (1.0 - ratio - q * q);                                                        // :132-134
    } else {
      a = -b;                                                                                // :137
    }
  }
  return clip_np(a, -b, am);                                                                 // :89
}

// pure_pursuit_controller.py:51-74,90-92; LineString.interpolate = arc-length walk from the first vertex
__device__ double pure_pursuit_law(const CtrlLawRow& p, const PathVertex* pv, int n_vert, double v, double x, double y,
                                   double heading) {
  const double d = fmax(v * (double)p.pp_interval, (double)p.min_pre_aiming_distance);     // :90-91
  double px = pv[n_vert - 1].x, py = pv[n_vert - 1].y;
  for (int i = 0; i + 1 < n_vert; ++i) {
    const PathVertex q = pv[i];
    if (d <= q.cum + q.len && q.len > 0.0) {
      const double t = (d - q.cum) / q.len;
      px = q.x + t * (pv[i + 1].x - q.x);
      py = q.y + t * (pv[i + 1].y - q.y);
      break;
    }
  }
  const double ang = atan2(py - y, px - x);                                                 // :62-64
  const double dist = hypot(py - y, px - x);                                                // :65-67
  return atan(2.0 * (double)p.wheel_base * sin(ang - heading) / dist);                      // :68-70
}

// pid_controller.py:159-234, one channel.  s = (integral, prev_error, prev_derivative) is rewritten in place.  Every
// operation rounds once (no FMA contraction) in the reference's order; `limited` selects the output_limits branch.
__device__ double pid_channel(const t2d_controller_params& p, double e, double s[3], double kp, double ki, double kd,
                              bool limited, double lo, double hi) {
  const double alpha = p.derivative_filter_alpha;
  const double p_term = __dmul_rn(kp, e);                                                     // :191
  const double raw = __ddiv_rn(__dsub_rn(e, s[1]), p.dt);                                     // :194
  const double d = __dadd_rn(__dmul_rn(alpha, raw), __dmul_rn(__dsub_rn(1.0, alpha), s[2]));   // :195-198
  double out = __dadd_rn(p_term, __dmul_rn(kd, d));                                          // :199-202
  bool saturated = false;
  if (limited) {                                                                             // :205-214
    if (out > hi) { saturated = true; out = hi; }
    else if (out < lo) { saturated = true; out = lo; }
  }
  s[0] = saturated ? __dmul_rn(s[0], 0.99) : __dadd_rn(s[0], __dmul_rn(e, p.dt));            // :217-222
  out = __dadd_rn(out, __dmul_rn(ki, s[0]));                                                 // :224-227
  if (limited) out = clip_np(out, lo, hi);                                                   // :230-232
  s[1] = e;
  s[2] = d;
  return out;
}

// The lateral error of a PATH_* source (no reference counterpart), from the closest point c and its tangent u:
// PATH_CROSS_TRACK: e = u.x (c.y - y) - u.y (c.x - x), positive when the path lies to the left; PATH_HEADING:
// target_heading = atan2(u.y, u.x).  false: no segment.
__device__ bool path_lateral_error(const PathVertex* pv, int n_vert, double x, double y, double heading, bool cross,
                                   double& e) {
  PathPoint c;
  if (!closest_on_path<false>(pv, n_vert, x, y, c)) return false;
  if (cross) {
    e = __dsub_rn(__dmul_rn(c.ux, __dsub_rn(c.cy, y)), __dmul_rn(c.uy, __dsub_rn(c.cx, x)));
  } else {
    const double err = __dsub_rn(atan2(c.uy, c.ux), heading);
    e = atan2(sin(err), cos(err));
  }
  return true;
}

// The lateral channel of pid_controller.py:309-406 for slot i: the steering, 0 when the source is NONE or its error is
// missing (a PATH source without a usable path: the combined mode's missing keyword); the lateral half of the slot's state
// row is rewritten when the channel runs.  PID rows and IDM rows with a lateral channel (lane keeping) share it.
__device__ __forceinline__ double pid_lateral_law(const t2d_controller_params& p, const CtrlArgs& A, size_t i, double x,
                                                  double y, double heading) {
  double* st = A.pid_state + 6 * i;
  double steer = 0.0;
  const int lat = p.pid_lateral;
  if (lat != T2D_PID_LAT_NONE) {
    double e = 0.0;
    bool have = true;
    if (lat == T2D_PID_LAT_HEADING) {                                                       // :267-274
      const double err = __dsub_rn((double)A.pid_target[2 * i + 1], heading);
      e = atan2(sin(err), cos(err));
    } else if (lat == T2D_PID_LAT_CROSS_TRACK) {                                             // :275-279
      e = (double)A.pid_target[2 * i + 1];
    } else {
      const PathVertex* pv;
      int nv;
      have = A.paths.vertices(A.path_id ? (int)A.path_id[i] : -1, pv, nv) &&
             path_lateral_error(pv, nv, x, y, heading, lat == T2D_PID_LAT_PATH_CROSS_TRACK, e);
    }
    if (have) {
      double s[3] = {st[0], st[1], st[2]};
      const double out = pid_channel(p, e, s, p.kp_lat, p.ki_lat, p.kd_lat, false, 0.0, 0.0);   // :338-348
      const bool cross = lat == T2D_PID_LAT_CROSS_TRACK || lat == T2D_PID_LAT_PATH_CROSS_TRACK;
      steer = cross ? __dmul_rn(out, __ddiv_rn(2.0, (double)p.wheel_base)) : out;            // :355-365
      steer = clip_np(steer, -p.max_steering, p.max_steering);                               // :368
      st[0] = s[0]; st[1] = s[1]; st[2] = s[2];
    }
  }
  return steer;
}

// pid_controller.py:309-406 for slot i: (steering, acceleration) into steer / acc; the slot's state row is rewritten
// for each channel that runs.  A channel whose source is NONE, or whose error is missing, gives 0 and leaves its half of
// the row alone.
__device__ void pid_law(const t2d_controller_params& p, const CtrlArgs& A, size_t i, double x, double y, double v,
                        double heading, double& steer, double& acc) {
  double* st = A.pid_state + 6 * i;
  steer = pid_lateral_law(p, A, i, x, y, heading);
  acc = 0.0;
  if (p.pid_longitudinal == T2D_PID_LON_TARGET) {
    const double e = __dsub_rn((double)A.pid_target[2 * i], v);                              // :306-307
    double s[3] = {st[3], st[4], st[5]};
    const double lo = (double)p.min_accel, hi = (double)p.max_accel;
    acc = clip_np(pid_channel(p, e, s, p.kp_lon, p.ki_lon, p.kd_lon, true, lo, hi), lo, hi);   // :383-397
    st[3] = s[0]; st[4] = s[1]; st[5] = s[2];
  }
}

// The yielding IDM law of slot i: min(a on the leader, a on the stop point standing at speed 0) while K19 found a stop
__device__ __forceinline__ double yield_law(const CtrlArgs& A, size_t i, const CtrlLawRow& p, double v, double x, double y,
                                            double acc) {
  if (!(A.stop_gap[i] < __int_as_float(0x7f800000))) return acc;   // +inf: no stop
  const double2 s = A.stop_xy[i];
  return fmin(acc, idm_law(p, v, x, y, true, 0.0, s.x, s.y));
}

__device__ __forceinline__ const CtrlLawRow& law_row(const t2d_controller_params* ctab, int cid) {
  return *reinterpret_cast<const CtrlLawRow*>(reinterpret_cast<const char*>(ctab) + (size_t)cid * sizeof(t2d_controller_params));
}

// HAS_PID: the instance with the PID law, launched when the bound table holds a PID row or an IDM row with a lateral
// channel; the other one is the plain K5.  SLOT_SPEED: the reactive-replay instance (t2d_reactive_control_kernel, with
// the PID law), whose IDM rows take slot_desired_speed in place of the row's desired_speed on every slot whose path_id
// (there: the replay's drive_path) is >= 0.  YIELD: the instance launched while yielding is bound (t2d_yield_control_kernel,
// with the PID law, and the slot desired speeds when slot_desired_speed is not nullptr): an IDM row with a finite stop_gap
// takes the smaller of its law on the leader and its law on the stop point as a leader standing at speed 0.
template <bool HAS_PID, bool SLOT_SPEED, bool YIELD = false>
__device__ __forceinline__ void control_body(const CtrlArgs& A) {
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; n < A.N; n += warps) {
    const size_t base = (size_t)n * A.M;
    float2 out[4];
    float mag[4];
    bool ctl[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = lane + 32 * j;
      ctl[j] = false;
      mag[j] = 0.0f;
      out[j] = make_float2(0.0f, 0.0f);
      if (m >= A.M) continue;
      const int tid = A.type_id[base + m];
      if (tid >= A.n_types) continue;                  // inactive slot
      const Params& tp = A.table[tid];
      out[j] = reinterpret_cast<const float2*>(A.action)[base + m];
      if (m == 0 && A.ego_action != nullptr) { out[j] = reinterpret_cast<const float2*>(A.ego_action)[n]; ctl[j] = true; }   // row 0 <- the ego's action
      const int cid = A.ctrl_id[base + m];
      if (cid < A.n_ctrl && law_row(A.ctab, cid).kind != T2D_CTRL_EXTERNAL) {
        const CtrlLawRow& p = law_row(A.ctab, cid);
        const double x = A.x[base + m], y = A.y[base + m], v = A.v[base + m];
        const int li = A.lead ? (int)A.lead[base + m] : -1;
        const bool has = li >= 0 && li < A.M && li != m && A.type_id[base + li] < A.n_types;
        double xl = 0.0, yl = 0.0, vl = 0.0, al = 0.0;
        if (has) {
          xl = A.x[base + li]; yl = A.y[base + li]; vl = A.v[base + li]; al = A.last_accel[base + li];
        }
        double acc, steer = 0.0;
        if (HAS_PID && p.kind == T2D_CTRL_PID) {
          pid_law(A.ctab[cid], A, base + m, x, y, v, (double)A.h[base + m], steer, acc);
        } else if (p.kind == T2D_CTRL_IDM) {
          if (SLOT_SPEED && (!YIELD || A.slot_desired_speed) && A.path_id[base + m] >= 0) {   // a reactive slot: its track's desired speed
            CtrlLawRow q = p;
            q.desired_speed = A.slot_desired_speed[base + m];
            acc = idm_law(q, v, x, y, has, vl, xl, yl);
            if constexpr (YIELD) acc = yield_law(A, base + m, q, v, x, y, acc);
          } else {
            acc = idm_law(p, v, x, y, has, vl, xl, yl);
            if constexpr (YIELD) acc = yield_law(A, base + m, p, v, x, y, acc);
          }
          // lane keeping: an IDM row with a lateral channel (only a PATH source passes t2d_set_controllers)
          if (HAS_PID && A.ctab[cid].pid_lateral != T2D_PID_LAT_NONE)
            steer = pid_lateral_law(A.ctab[cid], A, base + m, x, y, (double)A.h[base + m]);
        } else {
          acc = longitudinal_law(p, v, x, y, (double)A.last_accel[base + m], has, vl, xl, yl, al);
          if (p.kind == T2D_CTRL_PURE_PURSUIT) {
            const PathVertex* pv;
            int nv;
            if (A.paths.vertices(A.path_id ? (int)A.path_id[base + m] : -1, pv, nv))
              steer = pure_pursuit_law(p, pv, nv, v, x, y, (double)A.h[base + m]);
          }
        }
        out[j] = A.steer_first ? make_float2((float)steer, (float)acc) : make_float2((float)acc, (float)steer);
        ctl[j] = true;
      }
      // |a| the physics will apply: single_track_kinematics.py:192 clips to the accel range; point_mass.py takes (ax, ay) as is
      if (tp.model() <= T2D_MODEL_DYNAMICS || tp.model() == T2D_MODEL_DRIFT)
        mag[j] = fabsf(clampf(A.steer_first ? out[j].y : out[j].x, tp.accel_lo, tp.accel_hi));
      else if (tp.model() <= T2D_MODEL_POINTMASS_EULER)
        mag[j] = (float)hypot((double)out[j].x, (double)out[j].y);
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = lane + 32 * j;
      if (m >= A.M) continue;
      if (ctl[j]) reinterpret_cast<float2*>(A.action)[base + m] = out[j];
      A.last_accel[base + m] = mag[j];
    }
  }
}

template <bool HAS_PID>
__global__ void __launch_bounds__(128) t2d_control_kernel(const __grid_constant__ CtrlArgs A) {
  control_body<HAS_PID, false>(A);
}

__global__ void __launch_bounds__(128) t2d_reactive_control_kernel(const __grid_constant__ CtrlArgs A) {
  control_body<true, true>(A);
}

__global__ void __launch_bounds__(128) t2d_yield_control_kernel(const __grid_constant__ CtrlArgs A) {
  control_body<true, true, true>(A);
}

}  // namespace t2d
