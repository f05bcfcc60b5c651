// devsim.cu - TEST HARNESS ONLY (never shipped, never used by tactics2d_b200).
//
// The device twin of tests/hostsim/hostsim.cpp: the same extern "C" entry points with the same signatures, but every
// one of them runs the arithmetic of tactics2d_b200/csrc/t2d_math.cuh on the GPU, compiled with the library's own nvcc
// flags.  So the numerics batteries of tests/test_hostsim_math.py see what the sm_90a kernels compute - FMA contraction,
// rsqrtf / __fdividef, CUDA's sincosf and sincos, and the warp vote of the fast kinematics loop - instead of the g++
// build.  Each entry point takes host pointers: it copies the inputs to the device, launches one element per thread
// (hs_kinematics4: four participants per thread, in full warps), synchronises and copies the results back.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include <cuda_runtime.h>

#include "../../tactics2d_b200/csrc/t2d_math.cuh"

using namespace t2d;

namespace {

constexpr int BLOCK = 128;

void check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) {
    fprintf(stderr, "devsim: %s: %s\n", what, cudaGetErrorString(e));
    abort();
  }
}

int blocks(int n) { return (n + BLOCK - 1) / BLOCK; }

// A device copy of a host array; `back` copies it home when the buffer goes out of scope.
template <typename T>
struct Dev {
  T* d = nullptr;
  T* host;
  size_t n;
  bool back;
  Dev(const T* h, size_t count, bool copy_back) : host(const_cast<T*>(h)), n(count), back(copy_back) {
    check(cudaMalloc(&d, (n > 0 ? n : 1) * sizeof(T)), "cudaMalloc");
    if (n > 0) check(cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice), "copy in");
  }
  ~Dev() {
    if (back && n > 0) check(cudaMemcpy(host, d, n * sizeof(T), cudaMemcpyDeviceToHost), "copy out");
    cudaFree(d);
  }
};

void finish(const char* what) {
  check(cudaGetLastError(), what);
  check(cudaDeviceSynchronize(), what);
}

// ------------------------------------------------------------------------------------------ kernels
__global__ void k_physics(int n, const Params* ptab, const int32_t* type_id, int n_steps, double dt, double dt_rem, double interval,
                          float* x, float* y, float* h, float* v, float* vx, float* vy, const float* action, float* applied) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Params p = ptab[type_id[i]];
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

// Four participants per thread, like K1's lanes: thread t owns participants 4t .. 4t + 3, so a warp holds 128 of them
// and the fast loop is taken only when all 128 can (the vote in kinematics_step).
__global__ void k_kinematics4(int n4, const Params* p, int n_steps, float dt, float dt_rem, float* x, float* y, float* h, float* v,
                              float* vx, float* vy, const float* action) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n4) return;
  const Params pd = *p;
  const Params* pp[4] = {&pd, &pd, &pd, &pd};
  KinIO<4> io;
  const int b = 4 * t;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    io.x[i] = x[b + i]; io.y[i] = y[b + i]; io.h[i] = h[b + i]; io.v[i] = v[b + i];
    io.acc[i] = action[2 * (b + i)]; io.steer[i] = action[2 * (b + i) + 1];
  }
  kinematics_step<4>(io, pp, n_steps, dt, dt_rem);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    x[b + i] = io.x[i]; y[b + i] = io.y[i]; h[b + i] = io.h[i]; v[b + i] = io.v[i]; vx[b + i] = io.vx[i]; vy[b + i] = io.vy[i];
  }
}

__global__ void k_pairs(int n, const float* a, const float* b, int32_t* out_f32, int32_t* out_exact) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
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

__global__ void k_segments(int n, const float* a, const float* seg, int32_t* out_f32, int32_t* out_exact) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* pa = a + 5 * i; const float* s = seg + 4 * i;
  float sa, ca;
  sincos_fast(pa[2], &sa, &ca);
  if (pa[4] < 0) { out_f32[i] = circle_segment_f32(pa[0], pa[1], pa[3], s[0], s[1], s[2], s[3]);
                   out_exact[i] = circle_segment_f64(pa[0], pa[1], pa[3], s[0], s[1], s[2], s[3]); }
  else { out_f32[i] = obb_segment_f32(pa[0], pa[1], ca, sa, pa[3], pa[4], s[0], s[1], s[2], s[3]);
         out_exact[i] = obb_segment_f64(pa[0], pa[1], pa[2], pa[3], pa[4], s[0], s[1], s[2], s[3]); }
}

__global__ void k_outbound(int n, const float* a, const float* bounds, int32_t* out_f32, int32_t* out_exact) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* pa = a + 5 * i;
  float sa, ca;
  sincos_fast(pa[2], &sa, &ca);
  out_f32[i] = out_of_bound_f32(pa[0], pa[1], ca, sa, pa[3], pa[4], pa[4] < 0, bounds[0], bounds[1], bounds[2], bounds[3]);
  out_exact[i] = out_of_bound_f64(pa[0], pa[1], pa[2], pa[3], pa[4], pa[4] < 0, bounds[0], bounds[1], bounds[2], bounds[3]);
}

__global__ void k_drift(int n, const Params* p, int n_steps, double dt, double dt_rem, float* x, float* y, float* h, float* v,
                        float* wf, float* wr, const float* action, float* applied) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  OneIO io;
  io.x = x[i]; io.y = y[i]; io.h = h[i]; io.v = v[i]; io.vx = 0.0f; io.vy = 0.0f; io.w0 = wf[i]; io.w1 = wr[i];
  io.a0 = action[2 * i]; io.a1 = action[2 * i + 1]; io.ch = 1.0f; io.sh = 0.0f;
  drift_step(io, *p, n_steps, dt, dt_rem);
  x[i] = io.x; y[i] = io.y; h[i] = io.h; v[i] = io.v; wf[i] = io.w0; wr[i] = io.w1;
  applied[2 * i] = io.a0; applied[2 * i + 1] = io.a1;
}

__global__ void k_beam_window(int n, const double* edge, const double* dist2, int n_beams, int32_t* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const BeamWindow w = beam_window(edge[4 * i], edge[4 * i + 1], edge[4 * i + 2], edge[4 * i + 3], dist2[i], n_beams);
  out[2 * i] = w.x; out[2 * i + 1] = w.y;
}

__global__ void k_wrap(float phi, float* out) { *out = wrap_two_pi(phi); }

__global__ void k_rect_iou(int n, const float* a, const float* b, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = a + 5 * i; const float* q = b + 5 * i;
  out[i] = rect_iou_f64(p[0], p[1], p[2], p[3], p[4], q[0], q[1], q[2], q[3], q[4]);
}

}  // namespace

extern "C" {

void hs_physics(int n, const AbiParams* atab, const int32_t* type_id, int n_steps, double dt, double dt_rem, double interval,
                float* x, float* y, float* h, float* v, float* vx, float* vy, const float* action, float* applied) {
  if (n <= 0) return;
  int n_types = 0;
  for (int i = 0; i < n; ++i) n_types = type_id[i] + 1 > n_types ? type_id[i] + 1 : n_types;
  std::vector<Params> ptab(n_types);
  for (int t = 0; t < n_types; ++t) ptab[t] = derive_params(atab[t]);
  Dev<Params> dp(ptab.data(), ptab.size(), false);
  Dev<int32_t> dt_id(type_id, n, false);
  Dev<float> dx(x, n, true), dy(y, n, true), dh(h, n, true), dv(v, n, true), dvx(vx, n, true), dvy(vy, n, true);
  Dev<float> da(action, 2 * (size_t)n, false), dap(applied, 2 * (size_t)n, true);
  k_physics<<<blocks(n), BLOCK>>>(n, dp.d, dt_id.d, n_steps, dt, dt_rem, interval, dx.d, dy.d, dh.d, dv.d, dvx.d, dvy.d, da.d, dap.d);
  finish("hs_physics");
}

void hs_kinematics4(int n, const AbiParams* ap, int n_steps, double dt, double dt_rem, float* x, float* y, float* h, float* v,
                    float* vx, float* vy, const float* action) {
  const int n4 = n / 4;
  if (n4 <= 0) return;
  const Params pd = derive_params(*ap);
  Dev<Params> dp(&pd, 1, false);
  Dev<float> dx(x, n, true), dy(y, n, true), dh(h, n, true), dv(v, n, true), dvx(vx, n, true), dvy(vy, n, true);
  Dev<float> da(action, 2 * (size_t)n, false);
  k_kinematics4<<<blocks(n4), BLOCK>>>(n4, dp.d, n_steps, (float)dt, (float)dt_rem, dx.d, dy.d, dh.d, dv.d, dvx.d, dvy.d, da.d);
  finish("hs_kinematics4");
}

void hs_pairs(int n, const float* a, const float* b, int32_t* out_f32, int32_t* out_exact) {
  if (n <= 0) return;
  Dev<float> da(a, 5 * (size_t)n, false), db(b, 5 * (size_t)n, false);
  Dev<int32_t> df(out_f32, n, true), de(out_exact, n, true);
  k_pairs<<<blocks(n), BLOCK>>>(n, da.d, db.d, df.d, de.d);
  finish("hs_pairs");
}

void hs_segments(int n, const float* a, const float* seg, int32_t* out_f32, int32_t* out_exact) {
  if (n <= 0) return;
  Dev<float> da(a, 5 * (size_t)n, false), ds(seg, 4 * (size_t)n, false);
  Dev<int32_t> df(out_f32, n, true), de(out_exact, n, true);
  k_segments<<<blocks(n), BLOCK>>>(n, da.d, ds.d, df.d, de.d);
  finish("hs_segments");
}

void hs_outbound(int n, const float* a, const float* bounds, int32_t* out_f32, int32_t* out_exact) {
  if (n <= 0) return;
  Dev<float> da(a, 5 * (size_t)n, false), db(bounds, 4, false);
  Dev<int32_t> df(out_f32, n, true), de(out_exact, n, true);
  k_outbound<<<blocks(n), BLOCK>>>(n, da.d, db.d, df.d, de.d);
  finish("hs_outbound");
}

void hs_drift(int n, const AbiParams* ap, int n_steps, double dt, double dt_rem, float* x, float* y, float* h, float* v,
              float* wf, float* wr, const float* action, float* applied) {
  if (n <= 0) return;
  const Params pd = derive_params(*ap);
  Dev<Params> dp(&pd, 1, false);
  Dev<float> dx(x, n, true), dy(y, n, true), dh(h, n, true), dv(v, n, true), dwf(wf, n, true), dwr(wr, n, true);
  Dev<float> da(action, 2 * (size_t)n, false), dap(applied, 2 * (size_t)n, true);
  k_drift<<<blocks(n), BLOCK>>>(n, dp.d, n_steps, dt, dt_rem, dx.d, dy.d, dh.d, dv.d, dwf.d, dwr.d, da.d, dap.d);
  finish("hs_drift");
}

void hs_beam_window(int n, const double* edge, const double* dist2, int n_beams, int32_t* out) {
  if (n <= 0) return;
  Dev<double> de(edge, 4 * (size_t)n, false), dd(dist2, n, false);
  Dev<int32_t> dout(out, 2 * (size_t)n, true);
  k_beam_window<<<blocks(n), BLOCK>>>(n, de.d, dd.d, n_beams, dout.d);
  finish("hs_beam_window");
}

float hs_wrap(float phi) {
  float r = 0.0f;
  {
    Dev<float> dr(&r, 1, true);
    k_wrap<<<1, 1>>>(phi, dr.d);
    finish("hs_wrap");
  }
  return r;
}

void hs_rect_iou(int n, const float* a, const float* b, double* out) {
  if (n <= 0) return;
  Dev<float> da(a, 5 * (size_t)n, false), db(b, 5 * (size_t)n, false);
  Dev<double> dout(out, n, true);
  k_rect_iou<<<blocks(n), BLOCK>>>(n, da.d, db.d, dout.d);
  finish("hs_rect_iou");
}
}
