// hostsim.cpp - TEST HARNESS ONLY (never shipped, never used by tactics2d_b200).
//
// Compiles the device arithmetic of tactics2d_b200/csrc/t2d_math.cuh with g++ so that the
// fp32 / filtered-predicate numerics can be unit-tested against the float64 oracle on a
// machine without a GPU (`pytest -m "not gpu"`).  The CUDA kernels inline the very same header.
#include <cstdint>
#include <cstring>

#include "../../tactics2d_b200/csrc/t2d_math.cuh"

using namespace t2d;

extern "C" {

// state arrays in/out; action [n,2] in, applied [n,2] out; ptab: one Params per element
void hs_physics(int n, const AbiParams* atab, const int32_t* type_id, int n_steps, double dt, double dt_rem, double interval,
                float* x, float* y, float* h, float* v, float* vx, float* vy, const float* action, float* applied) {
  for (int i = 0; i < n; ++i) {
    const Params p = derive_params(atab[type_id[i]]);
    if (p.model() == MODEL_KINEMATICS) {
      KinIO<1> io;
      io.x[0] = x[i]; io.y[0] = y[i]; io.h[0] = h[i]; io.v[0] = v[i];
      io.acc[0] = action[2 * i]; io.steer[0] = action[2 * i + 1];
      const Params* const p1[1] = {&p};
      kinematics_step<1>(io, p1, n_steps, (float)dt, (float)dt_rem);
      x[i] = io.x[0]; y[i] = io.y[0]; h[i] = io.h[0]; v[i] = io.v[0]; vx[i] = io.vx[0]; vy[i] = io.vy[0];
      applied[2 * i] = io.acc[0]; applied[2 * i + 1] = io.steer[0];
    } else {
      OneIO io;
      io.x = x[i]; io.y = y[i]; io.h = h[i]; io.v = v[i]; io.vx = vx[i]; io.vy = vy[i];
      io.a0 = action[2 * i]; io.a1 = action[2 * i + 1]; io.ch = 1.0f; io.sh = 0.0f;
      if (p.model() == MODEL_DYNAMICS) dynamics_step(io, p, n_steps, dt);
      else if (p.model() == MODEL_POINTMASS_NEWTON) pointmass_newton_step(io, p, interval);
      else if (p.model() == MODEL_POINTMASS_EULER) pointmass_euler_step(io, p, n_steps, dt, dt_rem);
      x[i] = io.x; y[i] = io.y; h[i] = io.h; v[i] = io.v; vx[i] = io.vx; vy[i] = io.vy;
      applied[2 * i] = io.a0; applied[2 * i + 1] = io.a1;
    }
  }
}

// 4-wide kinematics (the kernel's fast path): n must be a multiple of 4
void hs_kinematics4(int n, const AbiParams* ap, int n_steps, double dt, double dt_rem, float* x, float* y, float* h, float* v,
                    float* vx, float* vy, const float* action) {
  const Params pd = derive_params(*ap);
  const Params* p = &pd;
  for (int b = 0; b + 4 <= n; b += 4) {
    KinIO<4> io;
    const Params* pp[4] = {p, p, p, p};
    for (int i = 0; i < 4; ++i) {
      io.x[i] = x[b + i]; io.y[i] = y[b + i]; io.h[i] = h[b + i]; io.v[i] = v[b + i];
      io.acc[i] = action[2 * (b + i)]; io.steer[i] = action[2 * (b + i) + 1];
    }
    kinematics_step<4>(io, pp, n_steps, (float)dt, (float)dt_rem);
    for (int i = 0; i < 4; ++i) {
      x[b + i] = io.x[i]; y[b + i] = io.y[i]; h[b + i] = io.h[i]; v[b + i] = io.v[i]; vx[b + i] = io.vx[i]; vy[b + i] = io.vy[i];
    }
  }
}

// pose rows: x, y, heading, l, w  (w < 0: disc of radius l).  out_f32: -1/0/1 filter verdict; out_exact: 0/1.
// The filters take (cos, sin) of the heading from sincos_fast, as K1's poses do.
void hs_pairs(int n, const float* a, const float* b, int32_t* out_f32, int32_t* out_exact) {
  for (int i = 0; i < n; ++i) {
    const float* pa = a + 5 * i; const float* pb = b + 5 * i;
    float sa, ca, sb, cb;
    sincos_fast(pa[2], &sa, &ca); sincos_fast(pb[2], &sb, &cb);
    const bool ka = pa[4] < 0, kb = pb[4] < 0;
    int r; bool e;
    if (!ka && !kb) { r = obb_obb_f32(pa[0], pa[1], ca, sa, pa[3], pa[4], pb[0], pb[1], cb, sb, pb[3], pb[4]);
                      e = obb_obb_f64(pa[0], pa[1], pa[2], pa[3], pa[4], pb[0], pb[1], pb[2], pb[3], pb[4]); }
    else if (!ka && kb) { r = obb_circle_f32(pa[0], pa[1], ca, sa, pa[3], pa[4], pb[0], pb[1], pb[3]);
                          e = obb_circle_f64(pa[0], pa[1], pa[2], pa[3], pa[4], pb[0], pb[1], pb[3]); }
    else if (ka && !kb) { r = obb_circle_f32(pb[0], pb[1], cb, sb, pb[3], pb[4], pa[0], pa[1], pa[3]);
                          e = obb_circle_f64(pb[0], pb[1], pb[2], pb[3], pb[4], pa[0], pa[1], pa[3]); }
    else { r = circle_circle_f32(pa[0], pa[1], pa[3], pb[0], pb[1], pb[3]);
           e = circle_circle_f64(pa[0], pa[1], pa[3], pb[0], pb[1], pb[3]); }
    out_f32[i] = r; out_exact[i] = e ? 1 : 0;
  }
}

void hs_segments(int n, const float* a, const float* seg, int32_t* out_f32, int32_t* out_exact) {
  for (int i = 0; i < n; ++i) {
    const float* pa = a + 5 * i; const float* s = seg + 4 * i;
    float sa, ca;
    sincos_fast(pa[2], &sa, &ca);
    if (pa[4] < 0) { out_f32[i] = circle_segment_f32(pa[0], pa[1], pa[3], s[0], s[1], s[2], s[3]);
                     out_exact[i] = circle_segment_f64(pa[0], pa[1], pa[3], s[0], s[1], s[2], s[3]); }
    else { out_f32[i] = obb_segment_f32(pa[0], pa[1], ca, sa, pa[3], pa[4], s[0], s[1], s[2], s[3]);
           out_exact[i] = obb_segment_f64(pa[0], pa[1], pa[2], pa[3], pa[4], s[0], s[1], s[2], s[3]); }
  }
}

void hs_outbound(int n, const float* a, const float* bounds, int32_t* out_f32, int32_t* out_exact) {
  for (int i = 0; i < n; ++i) {
    const float* pa = a + 5 * i;
    float sa, ca;
    sincos_fast(pa[2], &sa, &ca);
    out_f32[i] = out_of_bound_f32(pa[0], pa[1], ca, sa, pa[3], pa[4], pa[4] < 0, bounds[0], bounds[1], bounds[2], bounds[3]);
    out_exact[i] = out_of_bound_f64(pa[0], pa[1], pa[2], pa[3], pa[4], pa[4] < 0, bounds[0], bounds[1], bounds[2], bounds[3]);
  }
}

// SingleTrackDrift: wheel speeds in / out next to the state
void hs_drift(int n, const AbiParams* ap, int n_steps, double dt, double dt_rem, float* x, float* y, float* h, float* v,
              float* wf, float* wr, const float* action, float* applied) {
  const Params p = derive_params(*ap);
  for (int i = 0; i < n; ++i) {
    OneIO io;
    io.x = x[i]; io.y = y[i]; io.h = h[i]; io.v = v[i]; io.vx = 0.0f; io.vy = 0.0f; io.w0 = wf[i]; io.w1 = wr[i];
    io.a0 = action[2 * i]; io.a1 = action[2 * i + 1]; io.ch = 1.0f; io.sh = 0.0f;
    drift_step(io, p, n_steps, dt, dt_rem);
    x[i] = io.x; y[i] = io.y; h[i] = io.h; v[i] = io.v; wf[i] = io.w0; wr[i] = io.w1;
    applied[2 * i] = io.a0; applied[2 * i + 1] = io.a1;
  }
}

// lidar beam windows: edges (x1, y1, x2, y2) in the ego frame, distance^2 of the edge to the origin -> (first, count)
void hs_beam_window(int n, const double* edge, const double* dist2, int n_beams, int32_t* out) {
  for (int i = 0; i < n; ++i) {
    const BeamWindow w = beam_window(edge[4 * i], edge[4 * i + 1], edge[4 * i + 2], edge[4 * i + 3], dist2[i], n_beams);
    out[2 * i] = w.x; out[2 * i + 1] = w.y;
  }
}

float hs_wrap(float phi) { return wrap_two_pi(phi); }

// rows: x, y, heading, l, w (fp32, as the kernel sees them)
void hs_rect_iou(int n, const float* a, const float* b, double* out) {
  for (int i = 0; i < n; ++i) {
    const float* p = a + 5 * i; const float* q = b + 5 * i;
    out[i] = rect_iou_f64(p[0], p[1], p[2], p[3], p[4], q[0], q[1], q[2], q[3], q[4]);
  }
}
}
