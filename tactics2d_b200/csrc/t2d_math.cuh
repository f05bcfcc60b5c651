// t2d_math.cuh - per-participant physics and per-pair predicates of the batched tick.
//
// Everything here is a pure function of its arguments so that the same source is
//   * inlined into the sm_90a kernels (t2d_kernels.cu), and
//   * compiled by g++ into tests/hostsim (a unit-test harness that checks this arithmetic
//     against the float64 oracle without a GPU; it is NOT a product fallback).
//
// Arithmetic policy (DESIGN.md "numerics"):
//   * SingleTrackKinematics: fp32.  The reference's n Euler sub-steps are reproduced as the
//     same discrete sums, but (cos, sin)(phi+beta) is advanced by an angle-addition rotation
//     with a short polynomial for the small increment, and the position / heading sums are
//     accumulated separately and added to the state once (one rounding at |x| scale).
//   * SingleTrackDynamics: fp64 (the yaw/slip ODE is stiff below ~0.4 m/s, explicit Euler
//     amplifies rounding by up to (0.745/v - 1)^20 there; H100 issues DFMA at half FFMA rate).
//   * PointMass: fp64 arithmetic on the fp32 state (a few dozen flops).
//   * Collision predicates: fp32 with a forward error bound ("filtered predicate"); a pair
//     whose margin is inside the bound is re-evaluated exactly as the float64 oracle does
//     (double trig of the fp32 heading), so flags are bit-exact against the oracle.
#pragma once

#include <math.h>
#include <string.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define T2D_HD __host__ __device__ __forceinline__
#define T2D_HD_NOINLINE __host__ __device__ __noinline__
#else
#define T2D_HD inline
#define T2D_HD_NOINLINE
#endif

#if defined(__CUDA_ARCH__)
#define T2D_RSQRTF(x) rsqrtf(x)
#else
#define T2D_RSQRTF(x) (1.0f / sqrtf(x))
#endif

namespace t2d {

constexpr int MODEL_KINEMATICS = 0;
constexpr int MODEL_DYNAMICS = 1;
constexpr int MODEL_POINTMASS_NEWTON = 2;
constexpr int MODEL_POINTMASS_EULER = 3;
constexpr int MODEL_STATIC = 4;
constexpr int MODEL_DRIFT = 5;
constexpr int SHAPE_OBB = 0;
constexpr int SHAPE_CIRCLE = 1;
constexpr int SHAPE_NONE = 2;

constexpr float TWO_PI_HI = 6.2831854820251465f;   // fp32(2*pi)  ( > 2*pi )
constexpr float TWO_PI_LO = -1.7484555e-7f;        // 2*pi - TWO_PI_HI
constexpr float INV_TWO_PI = 0.15915494309189535f;
constexpr double TWO_PI_D = 6.283185307179586476925286766559;
constexpr double G_ACC = 9.81;                     // physics_model_base.py:25

// Mirror of t2d_type_params (include/t2d_b200.h); 23 words.
struct AbiParams {
  float half_len, half_wid, radius, lf, lr;
  float steer_lo, steer_hi, speed_lo, speed_hi, accel_lo, accel_hi;
  float mass, mass_height, mu, I_z, cf, cr;
  int32_t model, shape;
  float wheel_radius, T_sb, T_se, I_yw;   // SingleTrackDrift only
};

// The row the kernels read (28 words = 112 B): the ABI values regrouped so that everything a kinematic participant
// needs sits in THREE 16-byte groups (one 128-bit shared-memory load each instead of a dozen scalar ones; with the
// 112-byte row stride eight consecutive rows land on distinct bank groups), plus constants derived once on the host.
struct alignas(16) Vec4 { float x, y, z, w; };

struct alignas(16) Params {
  // group 0: action ranges
  float accel_lo, accel_hi, steer_lo, steer_hi;
  // group 1: speed range and the wheel-base constants  1 / (lf + lr), lr / (lf + lr)
  float speed_lo, speed_hi, lr_over_L, inv_L;
  // group 2: the collision shape as the pose tile stores it - (half_len, half_wid) of a box, (radius, -1) of a disc -
  // its bounding-circle radius (rounded up), and model | shape << 8 as an integer
  float pose_l, pose_w, rbound;
  int32_t model_shape;
  // the rest (fp64 models, controllers, lidar)
  float half_len, half_wid, radius, lf, lr;
  float mass, mass_height, mu, I_z, cf, cr;
  float wheel_radius, T_sb, T_se, I_yw;
  float pad0;
  T2D_HD int model() const { return model_shape & 0xff; }
  T2D_HD int shape() const { return model_shape >> 8; }
};
static_assert(sizeof(Params) == 112, "device type row");

inline Params derive_params(const AbiParams& a) {
  Params p;
  const float L = a.lf + a.lr;
  p.accel_lo = a.accel_lo; p.accel_hi = a.accel_hi; p.steer_lo = a.steer_lo; p.steer_hi = a.steer_hi;
  p.speed_lo = a.speed_lo; p.speed_hi = a.speed_hi;
  p.inv_L = 1.0f / L;
  p.lr_over_L = a.lr / L;
  p.rbound = a.shape == SHAPE_CIRCLE ? a.radius : sqrtf(a.half_len * a.half_len + a.half_wid * a.half_wid) * 1.000002f;
  p.pose_l = a.shape == SHAPE_CIRCLE ? a.radius : a.half_len;
  p.pose_w = a.shape == SHAPE_CIRCLE ? -1.0f : a.half_wid;
  p.model_shape = a.model | (a.shape << 8);
  p.half_len = a.half_len; p.half_wid = a.half_wid; p.radius = a.radius; p.lf = a.lf; p.lr = a.lr;
  p.mass = a.mass; p.mass_height = a.mass_height; p.mu = a.mu; p.I_z = a.I_z; p.cf = a.cf; p.cr = a.cr;
  p.wheel_radius = a.wheel_radius; p.T_sb = a.T_sb; p.T_se = a.T_se; p.I_yw = a.I_yw;
  p.pad0 = 0.0f;
  return p;
}

// One 16-byte group of a row (group g starts at word 4 g).
T2D_HD Vec4 params_group(const Params* p, int g) { return reinterpret_cast<const Vec4*>(p)[g]; }

T2D_HD float clampf(float v, float lo, float hi) { return fminf(fmaxf(v, lo), hi); }  // np.clip
T2D_HD double clampd(double v, double lo, double hi) { return fmin(fmax(v, lo), hi); }

// Bits of a float (device: a register move; host: memcpy).
T2D_HD int float_bits(float f) {
#if defined(__CUDA_ARCH__)
  return __float_as_int(f);
#else
  int i;
  memcpy(&i, &f, sizeof(i));
  return i;
#endif
}

#if defined(__CUDA_ARCH__)
#define T2D_FDIV(a, b) __fdividef((a), (b))   // reciprocal + multiply (2 ulp), no slow-path branch
#else
#define T2D_FDIV(a, b) ((a) / (b))
#endif

// Round-to-nearest-integer without the conversion unit: adding 1.5 * 2^23 leaves rint(u) in the low mantissa bits
// (|u| < 2^22): FRND / F2I would run on the quarter-rate conversion pipe.
constexpr float RINT_MAGIC = 12582912.0f;

// np.mod(phi, 2*pi) for an fp32 angle: result in [0, 2*pi) (Cody-Waite two-term reduction).  q = rint(phi / 2 pi - 1/2)
// is floor(phi / 2 pi) or its neighbour (at ties); the two corrections below absorb either.
T2D_HD float wrap_two_pi(float phi) {
  const float q = (fmaf(phi, INV_TWO_PI, -0.5f) + RINT_MAGIC) - RINT_MAGIC;
  float r = fmaf(-q, TWO_PI_HI, phi);
  r = fmaf(-q, TWO_PI_LO, r);
  if (r < 0.0f) r += TWO_PI_HI;
  if (r >= TWO_PI_HI) r -= TWO_PI_HI;
  if (r < 0.0f) r = 0.0f;
  return r;
}

// sincos without the library's large-argument (Payne-Hanek) path inlined at every call site: Cody-Waite
// reduction to [-pi/4, pi/4] (three-term pi/2, exact for |x| <= 512) + degree-7/8 polynomials; abs error < 1e-7.
// Larger arguments go to one out-of-line copy of the library routine.
// (The slow path returns its results BY VALUE: handing it the callers' output pointers would force both results of
//  every inlined sincos_fast through local memory, also on the fast path.)
struct SinCos { float s, c; };
#if defined(__CUDACC__)
__host__ __device__ __noinline__ SinCos sincosf_slow(float x) { SinCos r; sincosf(x, &r.s, &r.c); return r; }
#else
inline SinCos sincosf_slow(float x) { SinCos r; sincosf(x, &r.s, &r.c); return r; }
#endif

// The two polynomials on the reduced argument r in [-pi/4, pi/4].
T2D_HD void sincos_poly(float r, float& s, float& c) {
  const float z = r * r;
  s = fmaf(r * z, fmaf(z, fmaf(z, -1.9515295891e-4f, 8.3321608736e-3f), -1.6666654611e-1f), r);
  c = fmaf(z * z, fmaf(z, fmaf(z, 2.443315711809948e-5f, -1.388731625493765e-3f), 4.166664568298827e-2f),
           fmaf(-0.5f, z, 1.0f));
}

// The branch-free part: correct for |x| <= 512 (NaN / inf give NaN).  Callers that cannot rule out larger arguments
// check that themselves, ONCE for a whole group of evaluations, so that the evaluations of independent participants
// stay in one basic block and interleave (a slow-path CALL after every evaluation serialises them).
T2D_HD void sincos_core(float x, float& so, float& co) {
  const float t = fmaf(x, 0.636619772f, RINT_MAGIC);   // the quadrant k = rint(x * 2 / pi) sits in t's low mantissa bits
  const float k = t - RINT_MAGIC;
  float r = fmaf(-k, 1.570556640625f, x);
  r = fmaf(-k, 2.396702766418457e-4f, r);
  r = fmaf(-k, 1.5893254712295857e-8f, r);
  float s, c;
  sincos_poly(r, s, c);
  const int q = float_bits(t);
  const float a = (q & 1) ? c : s, b = (q & 1) ? s : c;
  so = (q & 2) ? -a : a;
  co = ((q + 1) & 2) ? -b : b;
}

T2D_HD void sincos_fast(float x, float* sn, float* cs) {
  float so, co;
  if (!(fabsf(x) <= 512.0f)) {
    const SinCos r = sincosf_slow(x);
    so = r.s; co = r.c;
  } else {
    sincos_core(x, so, co);
  }
  *sn = so;
  *cs = co;
}

// Small-angle rotation, |d| <= 0.25 (Taylor: |err| < 2e-9 on cos, 1.3e-8 relative on sin).
constexpr float SIN_C3 = -1.6666667e-1f, SIN_C5 = 8.3333333e-3f;
constexpr float COS_C2 = -0.5f, COS_C4 = 4.1666667e-2f, COS_C6 = -1.3888889e-3f;

// (c, s) <- (c, s) rotated by d, given d and nd = -d.
T2D_HD void rotate_small(float& c, float& s, float d, float nd) {
  const float dd = d * d;
  const float ts = fmaf(dd, fmaf(dd, SIN_C5, SIN_C3), 1.0f);
  const float sn = d * ts, nsn = nd * ts;
  const float nhv = dd * fmaf(dd, fmaf(dd, COS_C6, COS_C4), COS_C2);   // cos(d) - 1
  const float cn = fmaf(s, nsn, fmaf(c, nhv, c));
  const float sm = fmaf(c, sn, fmaf(s, nhv, s));
  c = cn;
  s = sm;
}

// ------------------------------------------------------------------------------------------
// SingleTrackKinematics.step/_step  (single_track_kinematics.py:178-198,126-176), W lanes of
// independent participants advanced together (instruction-level parallelism for the serial
// Euler chain).
// ------------------------------------------------------------------------------------------
template <int W>
struct KinIO {
  float x[W], y[W], h[W], v[W];   // in: state; out: new state (heading wrapped to [0, 2pi))
  float vx[W], vy[W];             // out: v*(cos, sin)(phi)                         :170-171
  float ch[W], sh[W];             // out: (cos, sin)(new heading) for the pose
  float acc[W], steer[W];         // in: raw action; out: clipped action            :192-193
};

// Tail of kinematics_step: position / heading from the sub-step sums, the remainder sub-step, wrap, velocity.
template <int W>
T2D_HD void kinematics_finish(KinIO<W>& io, const Params* const (&p)[W], const float (&c)[W], const float (&s)[W], float (&v)[W],
                              const float (&Sx)[W], const float (&Sy)[W], const float (&Sv)[W], const float (&kdt)[W],
                              const float (&k)[W], const float (&a)[W], const float (&vlo)[W], const float (&vhi)[W], float dt,
                              float dt_rem) {
#pragma unroll
  for (int i = 0; i < W; ++i) {
    float x = fmaf(dt, Sx[i], io.x[i]);
    float y = fmaf(dt, Sy[i], io.y[i]);
    float dphi = kdt[i] * Sv[i];
    if (dt_rem > 0.0f) {  // remainder sub-step :151-163
      x = fmaf(dt_rem * v[i], c[i], x);
      y = fmaf(dt_rem * v[i], s[i], y);
      dphi = fmaf(k[i] * dt_rem, v[i], dphi);
      v[i] = clampf(fmaf(a[i], dt_rem, v[i]), vlo[i], vhi[i]);
    }
    float hn = wrap_two_pi(io.h[i] + dphi);     // np.mod(phi, 2 pi)                        :169
    float sh, ch;
    sincos_core(hn, sh, ch);                    // hn is in [0, 2 pi] (or NaN): no large-argument path needed
    io.x[i] = x; io.y[i] = y; io.h[i] = hn; io.v[i] = v[i];
    io.vx[i] = v[i] * ch;                        // v cos(phi), no beta                    :170
    io.vy[i] = v[i] * sh;                        //                                        :171
    io.ch[i] = ch; io.sh[i] = sh;
  }
}

template <int W>
T2D_HD void kinematics_step(KinIO<W>& io, const Params* const (&p)[W], int n_steps, float dt, float dt_rem) {
  // Speed recurrence in closed form.  The reference iterates w_{i+1} = clip(w_i + a dt) (:147-148).  With
  // w_1 = clip(w_0 + a dt) inside [lo, hi], the sequence is monotone and saturates at most once, hence
  // w_i = clip(w_1 + (i-1) a dt) for i >= 1 (w_0 itself may lie outside the range).  One rounding per
  // term instead of an accumulated sum.
  float c[W], s[W], w1[W], Sx[W], Sy[W], Sv[W], kdt[W], adt[W], vlo[W], vhi[W], k[W], a[W];
  bool small = true;
  // fast loop: no participant of this group touches a speed bound during the tick, and the tick has at most 24
  // sub-steps - the carried rotation accumulates rounding quadratically in the sub-step count (measured against float64
  // at v <= 69 m/s: 4e-6 at 20 sub-steps, 9e-6 at 100, 2e-5 at 40 sub-steps of a 200 ms tick; the general loop stays
  // below 7e-6 there), so longer ticks keep the general loop
  bool lin = n_steps >= 2 && n_steps <= 24;
  // Trigonometry of the steering angle and the heading first, for all W participants in one basic block; the arguments
  // the short forms cannot take (a steering range beyond +-pi/4, a heading beyond +-512) are re-done afterwards, once.
  float sd[W], cd[W], sp[W], cp[W];
  bool rare = false;
#pragma unroll
  for (int i = 0; i < W; ++i) {
    const Vec4 g0 = params_group(p[i], 0);      // accel lo hi, steer lo hi
    a[i] = clampf(io.acc[i], g0.x, g0.y);       // :192
    const float d = clampf(io.steer[i], g0.z, g0.w);  // :193
    io.acc[i] = a[i];
    io.steer[i] = d;
    sincos_poly(d, sd[i], cd[i]);               // = sincos_fast for |d| <= pi/4 (its reduction is the identity there)
    sincos_core(io.h[i], sp[i], cp[i]);
    rare = rare || !(fabsf(d) <= 0.78f) || !(fabsf(io.h[i]) <= 512.0f);
  }
  if (rare) {
#pragma unroll
    for (int i = 0; i < W; ++i) {
      if (!(fabsf(io.steer[i]) <= 0.78f)) sincos_fast(io.steer[i], &sd[i], &cd[i]);
      if (!(fabsf(io.h[i]) <= 512.0f)) sincos_fast(io.h[i], &sp[i], &cp[i]);
    }
  }
#pragma unroll
  for (int i = 0; i < W; ++i) {
    const Vec4 g1 = params_group(p[i], 1);      // speed lo hi, lr / L, 1 / L
    const float tan_d = T2D_FDIV(sd[i], cd[i]);
    const float tb = g1.z * tan_d;              // tan(beta), beta = atan(lr/L tan delta)  :127  (L = lf + lr, :85)
    const float cb = T2D_RSQRTF(fmaf(tb, tb, 1.0f));  // cos(beta)
    const float sb = tb * cb;                    // sin(beta)
    k[i] = tan_d * cb * g1.w;                    // dphi = v * k                           :141
    kdt[i] = k[i] * dt;
    adt[i] = a[i] * dt;
    c[i] = cp[i] * cb - sp[i] * sb;              // cos(phi + beta)
    s[i] = sp[i] * cb + cp[i] * sb;              // sin(phi + beta)
    vlo[i] = g1.x;
    vhi[i] = g1.y;
    const float w1u = fmaf(a[i], dt, io.v[i]);
    w1[i] = clampf(w1u, vlo[i], vhi[i]);
    const float wlu = fmaf((float)(n_steps - 1), adt[i], w1[i]);   // one step past the last speed the loop uses
    const float wl = clampf(fmaf((float)(n_steps - 2), adt[i], w1[i]), vlo[i], vhi[i]);
    lin = lin && (w1u == w1[i]) && (wlu >= vlo[i]) && (wlu <= vhi[i]) && (fabsf(kdt[i] * adt[i]) <= 1e-4f);
    const float wmax = fmaxf(fabsf(io.v[i]), fmaxf(fabsf(w1[i]), fabsf(wl)));
    small = small && (fabsf(kdt[i]) * wmax <= 0.25f);   // every sub-step rotation stays in the polynomial's range
    Sx[i] = 0.0f; Sy[i] = 0.0f; Sv[i] = 0.0f;
  }
  // Fast loop: with no speed bound touched, v_i = w_1 + (i - 1) a dt exactly as above and the per-sub-step rotation
  // angles d_i = k dt v_i form an arithmetic sequence with the tiny step e = k dt a dt (<= 1e-4).  Instead of
  // evaluating the sin / cos polynomials of d_i every sub-step, carry (cos d_i - 1, -sin d_i) along by rotating them
  // by e (two adds + two fmas; sin e = e and cos e - 1 = -e^2 / 2 to fp32 precision, products with e^2 dropped),
  // and drop the speed clamp and the running speed sum (closed form).  12 operations per participant and sub-step
  // instead of 19.
  // One loop per warp: lanes that could take the fast loop next to lanes that cannot would make the warp run both, so
  // the warp takes it only when every lane that is executing this function can (the general loop is valid for all).
#if defined(__CUDA_ARCH__)
  const bool fast = __all_sync(__activemask(), lin && small);
#else
  const bool fast = lin && small;
#endif
  if (fast) {
    float h[W], nsn[W], se[W], nse[W], he[W];
#pragma unroll
    for (int i = 0; i < W; ++i) {
      const float d0 = kdt[i] * io.v[i], dd = d0 * d0;
      const float ts = fmaf(dd, fmaf(dd, SIN_C5, SIN_C3), 1.0f);
      nsn[i] = (-d0) * ts;                                           // -sin d_0
      h[i] = dd * fmaf(dd, fmaf(dd, COS_C6, COS_C4), COS_C2);        // cos d_0 - 1
      se[i] = kdt[i] * adt[i];
      nse[i] = -se[i];
      he[i] = -0.5f * se[i] * se[i];
    }
    float v[W];
#pragma unroll
    for (int i = 0; i < W; ++i) v[i] = io.v[i];
    {
      float fi = -1.0f;
      for (int it = 0; it < n_steps; ++it) {
        fi += 1.0f;
#pragma unroll
        for (int i = 0; i < W; ++i) {
          Sx[i] = fmaf(v[i], c[i], Sx[i]);
          Sy[i] = fmaf(v[i], s[i], Sy[i]);
          const float sn = -nsn[i];
          const float cn = fmaf(s[i], nsn[i], fmaf(c[i], h[i], c[i]));
          const float sm = fmaf(c[i], sn, fmaf(s[i], h[i], s[i]));
          const float hn = fmaf(nsn[i], se[i], h[i] + he[i]);
          const float nn = fmaf(h[i], nse[i], nsn[i] + nse[i]);
          c[i] = cn; s[i] = sm; h[i] = hn; nsn[i] = nn;
          v[i] = fmaf(fi, adt[i], w1[i]);
        }
      }
    }
    // sum of the speeds the loop used: v_0 + sum_{i=1}^{n-1} (w_1 + (i - 1) a dt)
    const float nm1 = (float)(n_steps - 1), tri = 0.5f * (float)(n_steps - 1) * (float)(n_steps - 2);
#pragma unroll
    for (int i = 0; i < W; ++i) Sv[i] = fmaf(tri, adt[i], fmaf(nm1, w1[i], io.v[i]));
    kinematics_finish<W>(io, p, c, s, v, Sx, Sy, Sv, kdt, k, a, vlo, vhi, dt, dt_rem);
    return;
  }
  float v[W];
#pragma unroll
  for (int i = 0; i < W; ++i) v[i] = io.v[i];
  // main sub-steps :137-148 ; derivatives from the OLD (phi, v), then v clipped
  if (small) {
    float fi = -1.0f;
    for (int it = 0; it < n_steps; ++it) {
      fi += 1.0f;
#pragma unroll
      for (int i = 0; i < W; ++i) {
        Sx[i] = fmaf(v[i], c[i], Sx[i]);
        Sy[i] = fmaf(v[i], s[i], Sy[i]);
        Sv[i] += v[i];
        rotate_small(c[i], s[i], kdt[i] * v[i], -kdt[i] * v[i]);
        v[i] = clampf(fmaf(fi, adt[i], w1[i]), vlo[i], vhi[i]);   // w_{it+1}
      }
    }
  } else {  // unconstrained speed ranges only: exact trig per sub-step
    float fi = -1.0f;
    for (int it = 0; it < n_steps; ++it) {
      fi += 1.0f;
#pragma unroll
      for (int i = 0; i < W; ++i) {
        Sx[i] = fmaf(v[i], c[i], Sx[i]);
        Sy[i] = fmaf(v[i], s[i], Sy[i]);
        Sv[i] += v[i];
        float sn, cs;
        sincos_fast(kdt[i] * v[i], &sn, &cs);
        const float c2 = c[i] * cs - s[i] * sn;
        const float s2 = s[i] * cs + c[i] * sn;
        c[i] = c2;
        s[i] = s2;
        v[i] = clampf(fmaf(fi, adt[i], w1[i]), vlo[i], vhi[i]);
      }
    }
  }
  kinematics_finish<W>(io, p, c, s, v, Sx, Sy, Sv, kdt, k, a, vlo, vhi, dt, dt_rem);
}

// ------------------------------------------------------------------------------------------
// SingleTrackDynamics.step/_step  (single_track_dynamics.py:231-251,140-229), fp64.
// No remainder sub-step (the reference computes `remainder` at :143 and never uses it).
// ------------------------------------------------------------------------------------------
struct OneIO {
  float x, y, h, v, vx, vy;  // state in / out
  float ch, sh;              // out: (cos, sin)(new heading)
  float a0, a1;              // in: raw action; out: applied action
  float w0, w1;              // SingleTrackDrift only: front / rear wheel angular speed in / out
};

// Written over W participants side by side; the kernels use W = 1 (a second fp64 chain per call enlarges the call's
// register footprint, which bounds the occupancy of K1).
template <int W>
T2D_HD void dynamics_step_n(OneIO* const (&io)[W], const Params* const (&pp)[W], int n_steps, double dt) {
  double x[W], y[W], phi[W], v[W], d_phi[W], beta[W], sn[W], cs[W];
  double accel[W], delta[W], tan_d[W], L[W], vlo[W], vhi[W], d_beta_slow[W], mu[W];
  double k_a[W], k_sum[W], k_dif[W], k_cc[W], lf_cf_f[W], cf_f[W];
#pragma unroll
  for (int i = 0; i < W; ++i) {
    const Params& p = *pp[i];
    const double lf = p.lf, lr = p.lr;
    L[i] = (double)p.lf + (double)p.lr;
    accel[i] = clampd(io[i]->a0, p.accel_lo, p.accel_hi);   // :245
    delta[i] = clampd(io[i]->a1, p.steer_lo, p.steer_hi);   // :246
    io[i]->a0 = (float)accel[i];
    io[i]->a1 = (float)delta[i];
    const double mass = p.mass, h = p.mass_height, Iz = p.I_z, cf = p.cf, cr = p.cr;
    mu[i] = p.mu;
    const double factor_f = (G_ACC * lr - accel[i] * h) / L[i];          // :145
    const double factor_r = (G_ACC * lf + accel[i] * h) / L[i];          // :146
    lf_cf_f[i] = lf * cf * factor_f;                                     // :149-150
    const double lr_cr_r = lr * cr * factor_r;
    const double lf2_cf_f = lf * lf * cf * factor_f, lr2_cr_r = lr * lr * cr * factor_r;
    cf_f[i] = cf * factor_f;
    const double cr_r = cr * factor_r;
    tan_d[i] = tan(delta[i]);
    const double cos_d = cos(delta[i]);
    x[i] = io[i]->x; y[i] = io[i]->y; phi[i] = io[i]->h; v[i] = io[i]->v;
    d_phi[i] = v[i] / L[i] * tan_d[i];                                    // :159
    beta[i] = atan(lr / lf * tan_d[i]);                                   // :160 (lr/lf, not lr/L)
    vlo[i] = p.speed_lo; vhi[i] = p.speed_hi;
    d_beta_slow[i] = lr / ((1.0 + tan_d[i] * lr / L[i]) * (1.0 + tan_d[i] * lr / L[i])) / L[i] / (cos_d * cos_d) * delta[i];  // :194-200
    k_a[i] = mu[i] * mass / Iz; k_sum[i] = lf2_cf_f + lr2_cr_r; k_dif[i] = lr_cr_r - lf_cf_f[i]; k_cc[i] = cr_r + cf_f[i];
    // (cos, sin)(phi + beta) is carried from sub-step to sub-step by a rotation through the sub-step's change of phi + beta
    // (a degree-9/10 Taylor pair, exact to 1e-18 for |d| <= 0.1) instead of a double-precision sincos per sub-step; a larger
    // change (only in the unstable low-speed band) re-evaluates it.  One division per sub-step serves the three quotients
    // by v_safe.  Both differ from the reference's evaluation order in the last bit only - immaterial outside the band that
    // is ill-conditioned for ANY float64 implementation (tests/test_oracle_c.py).
    sincos(phi[i] + beta[i], &sn[i], &cs[i]);
  }
  for (int it = 0; it < n_steps; ++it) {                          // :163-218
#pragma unroll
    for (int i = 0; i < W; ++i) {
      const double dx = v[i] * cs[i], dy = v[i] * sn[i];
      const double v_safe = fabs(v[i]) > 1e-6 ? v[i] : (v[i] >= 0.0 ? 1e-6 : -1e-6);  // :169
      double d_beta;
      if (fabs(v[i]) >= 0.1) {                                    // :171
        const double inv_v = 1.0 / v_safe;
        const double w = d_phi[i] * inv_v;
        const double dd_phi = k_a[i] * (lf_cf_f[i] * delta[i] + k_dif[i] * beta[i] - k_sum[i] * w);
        d_beta = mu[i] * inv_v * (cf_f[i] * delta[i] - k_cc[i] * beta[i] + k_dif[i] * w) - d_phi[i];
        d_phi[i] += dd_phi * dt;                                  // :192
      } else {
        d_beta = d_beta_slow[i];
        d_phi[i] += v[i] * cos(beta[i]) / L[i] * tan_d[i] * dt;   // :210
      }
      x[i] += dx * dt;                                            // :212-216
      y[i] += dy * dt;
      v[i] += accel[i] * dt;
      const double dphi_step = d_phi[i] * dt, dbeta_step = d_beta * dt;
      phi[i] += dphi_step;
      beta[i] += dbeta_step;
      v[i] = clampd(v[i], vlo[i], vhi[i]);                        // :218
      const double d = dphi_step + dbeta_step;
      if (fabs(d) <= 0.1) {
        const double dd = d * d;
        const double sd = d * (1.0 + dd * (-1.0 / 6 + dd * (1.0 / 120 + dd * (-1.0 / 5040 + dd * (1.0 / 362880)))));
        const double hd_ = dd * (-0.5 + dd * (1.0 / 24 + dd * (-1.0 / 720 + dd * (1.0 / 40320 + dd * (-1.0 / 3628800)))));   // cos d - 1
        const double c2 = cs[i] + (cs[i] * hd_ - sn[i] * sd), s2 = sn[i] + (sn[i] * hd_ + cs[i] * sd);
        cs[i] = c2; sn[i] = s2;
      } else {
        sincos(phi[i] + beta[i], &sn[i], &cs[i]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < W; ++i) {
    double hd = fmod(phi[i], TWO_PI_D);                          // np.mod(phi, 2 pi) :224
    if (hd < 0.0) hd += TWO_PI_D;
    float hn = (float)hd;
    if (hn >= TWO_PI_HI) hn = 0.0f;
    float sh, ch;
    sincos_fast(hn, &sh, &ch);
    io[i]->x = (float)x[i]; io[i]->y = (float)y[i]; io[i]->h = hn; io[i]->v = (float)v[i];
    io[i]->vx = io[i]->v * ch; io[i]->vy = io[i]->v * sh;      // State.velocity of a State without vx, vy (state.py:160-165)
    io[i]->ch = ch; io[i]->sh = sh;
  }
}

T2D_HD void dynamics_step(OneIO& io, const Params& p, int n_steps, double dt) {
  OneIO* const ios[1] = {&io};
  const Params* const ps[1] = {&p};
  dynamics_step_n<1>(ios, ps, n_steps, dt);
}

// ------------------------------------------------------------------------------------------
// SingleTrackDrift.step/_step  (single_track_drift.py:467-499,340-465) with the built-in tyre
// (class Tire, :14-49; the reference evaluates every force at camber gamma = 0), fp64.
// This model DOES take the remainder sub-step (:352-355).  Wheel speeds travel in io.w0 / io.w1.
// ------------------------------------------------------------------------------------------
namespace tire {
constexpr double p_cx1 = 1.6411, p_dx1 = 1.1739, p_ex1 = 0.4640, p_kx1 = 22.303, p_hx1 = 1.2297e-3, p_vx1 = -8.8098e-6;
constexpr double r_bx1 = 13.276, r_bx2 = -13.778, r_ex1 = 1.2568, r_cx1 = 0.6522, r_hx1 = 5.0722e-3;
constexpr double p_cy1 = 1.3507, p_dy1 = 1.0489, p_ey1 = -7.4722e-3, p_ky1 = -21.920;
constexpr double r_by1 = 7.1433, r_by2 = 9.1917, r_by3 = -2.7856e-2, r_cy1 = 1.0719, r_ey1 = -0.2757, r_hy1 = 5.7448e-6;
constexpr double r_vy1 = -2.7825e-2, r_vy4 = 12.120, r_vy5 = 1.9, r_vy6 = -10.704;
}  // namespace tire

T2D_HD double safe_div(double u) { return fabs(u) > 1e-6 ? u : (u >= 0.0 ? 1e-6 : -1e-6); }   // :287,289,308-309,345
T2D_HD double magic(double B, double C, double E, double arg) {                                 // C atan(B a - E (B a - atan(B a)))
  const double ba = B * arg;
  return C * atan(ba - E * (ba - atan(ba)));
}

struct TireForces { double F_xf, F_xr, F_yf, F_yr; };

// _tire_forces :282-338 and the four Pacejka helpers :185-280 (gamma = 0: S_hy = S_vy = 0, mu_y = p_dy1, mu_x = p_dx1)
T2D_HD TireForces drift_tire_forces(double v_safe, double delta, double d_phi, double beta, double om_f, double om_r, double lf,
                                    double lr, double mass, double radius) {
  using namespace tire;
  double sb, cb, sd, cd;
  sincos(beta, &sb, &cb);
  sincos(delta, &sd, &cd);
  const double vs = safe_div(v_safe);                                                        // :287
  const double cbs = safe_div(cb);                                                           // :288-289
  const double alpha_f = atan((vs * sb + d_phi * lf) / (vs * cbs)) - delta;                  // :292-294
  const double alpha_r = atan((vs * sb - d_phi * lr) / (vs * cbs));                          // :295
  const double L = lf + lr;
  const double F_zf = (mass * G_ACC * lr) / L, F_zr = (mass * G_ACC * lf) / L;               // :298-299
  const double u_wf = vs * cbs * cd + (vs * sb + lf * d_phi) * sd;                           // :302-304
  const double u_wr = vs * cbs;                                                              // :305
  const double s_f = 1.0 - radius * om_f / safe_div(u_wf);                                   // :308-313
  const double s_r = 1.0 - radius * om_r / safe_div(u_wr);
  TireForces out;
  for (int axle = 0; axle < 2; ++axle) {
    const double kappa = axle ? s_r : s_f, alpha = axle ? alpha_r : alpha_f, F_z = axle ? F_zr : F_zf;
    // pure slip, longitudinal :185-203
    const double D_x = p_dx1 * F_z;
    const double B_x = (p_kx1 * F_z) / (p_cx1 * D_x + 1e-6);
    const double F0_x = D_x * sin(magic(B_x, p_cx1, p_ex1, -kappa + p_hx1) + p_vx1 * F_z);
    // pure slip, lateral :205-224
    const double D_y = p_dy1 * F_z;
    const double B_y = (p_ky1 * F_z) / (p_cy1 * D_y + 1e-6);
    const double F0_y = D_y * sin(magic(B_y, p_cy1, p_ey1, alpha));
    // combined slip, longitudinal :226-250
    const double B_xa = r_bx1 * cos(atan(r_bx2 * kappa));
    const double D_xa = F0_x / cos(magic(B_xa, r_cx1, r_ex1, r_hx1));
    const double F_x = D_xa * cos(magic(B_xa, r_cx1, r_ex1, alpha + r_hx1));
    // combined slip, lateral :252-280
    const double B_yk = r_by1 * cos(atan(r_by2 * (alpha - r_by3)));
    const double D_yk = F0_y / cos(magic(B_yk, r_cy1, r_ey1, r_hy1));
    const double D_vyk = p_dy1 * F_z * r_vy1 * cos(atan(r_vy4 * alpha));
    const double S_vyk = D_vyk * sin(r_vy5 * atan(r_vy6 * kappa));
    const double F_y = D_yk * cos(magic(B_yk, r_cy1, r_ey1, kappa + r_hy1)) + S_vyk;
    if (axle) { out.F_xr = F_x; out.F_yr = F_y; } else { out.F_xf = F_x; out.F_yf = F_y; }
  }
  return out;
}

T2D_HD void drift_step(OneIO& io, const Params& p, int n_steps, double dt_main, double dt_rem) {
  const double lf = p.lf, lr = p.lr, L = (double)p.lf + (double)p.lr;
  const double accel = clampd(io.a0, p.accel_lo, p.accel_hi);    // :490
  const double delta = clampd(io.a1, p.steer_lo, p.steer_hi);    // :491
  io.a0 = (float)accel;
  io.a1 = (float)delta;
  const double mass = p.mass, radius = p.wheel_radius, T_sb = p.T_sb, T_se = p.T_se, Iz = p.I_z, Iyw = p.I_yw;
  const double tan_d = tan(delta), cos_d = cos(delta), sin_d = sin(delta);
  double x = io.x, y = io.y, phi = io.h, v = io.v, om_f = io.w0, om_r = io.w1;
  double d_phi = v / L * tan_d;                                   // :360
  double beta = atan(lr / lf * tan_d);                            // :361
  const double T_B = accel > 0.0 ? 0.0 : mass * radius * accel;   // :363-368
  const double T_E = accel > 0.0 ? mass * radius * accel : 0.0;
  const double vlo = p.speed_lo, vhi = p.speed_hi;
  const int total = n_steps + (dt_rem > 0.0 ? 1 : 0);
  for (int it = 0; it < total; ++it) {                            // :370-455
    const double dt = it < n_steps ? dt_main : dt_rem;
    const double v_safe = safe_div(v);
    const TireForces F = drift_tire_forces(v_safe, delta, d_phi, beta, om_f, om_r, lf, lr, mass, radius);
    double sn, cs, sb, cb;
    sincos(phi + beta, &sn, &cs);
    sincos(beta, &sb, &cb);
    const double dx = v * cs, dy = v * sn;
    double dv, d_beta, d_om_f, d_om_r;
    if (fabs(v) >= 0.1) {                                         // :381
      double sdb, cdb;
      sincos(delta - beta, &sdb, &cdb);
      dv = 1.0 / mass * (-F.F_yf * sdb + F.F_yr * sb + F.F_xr * cb + F.F_xf * cdb);                    // :382-391
      d_beta = -d_phi + 1.0 / (mass * v_safe) * (F.F_yf * cdb + F.F_yr * cb - F.F_xr * sb + F.F_xf * sdb);   // :392-397
      const double dd_phi = 1.0 / Iz * (F.F_yf * cos_d * lf - F.F_yr * lr + F.F_xf * sin_d * lf);      // :398-406
      d_phi += dd_phi * dt;                                                                            // :407
      d_om_f = 1.0 / Iyw * (-radius * F.F_xf + T_sb * T_B + T_se * T_E);                               // :408-410
      d_om_r = 1.0 / Iyw * (-radius * F.F_xr + (1.0 - T_sb) * T_B + (1.0 - T_se) * T_E);               // :411-415
    } else {
      dv = accel;                                                                                      // :417
      d_beta = lr / ((1.0 + tan_d * lr / L) * (1.0 + tan_d * lr / L)) / L / (cos_d * cos_d) * delta;   // :418-424
      d_phi += v * cb / L * tan_d * dt;                                                                // :434
      d_om_f = 1.0 / (cos_d * radius) * (accel * cb - v * sb * d_beta + v * cb * tan_d * delta);       // :435-443
      d_om_r = 1.0 / radius * (accel * cb - v * sb * d_beta);                                          // :444
    }
    x += dx * dt;                                                 // :446-453
    y += dy * dt;
    v += dv * dt;
    phi += d_phi * dt;
    beta += d_beta * dt;
    om_f += d_om_f * dt;
    om_r += d_om_r * dt;
    v = clampd(v, vlo, vhi);                                      // :455
  }
  double hd = fmod(phi, TWO_PI_D);                               // np.mod(phi, 2 pi) :461
  if (hd < 0.0) hd += TWO_PI_D;
  float hn = (float)hd;
  if (hn >= TWO_PI_HI) hn = 0.0f;
  float sh, ch;
  sincos_fast(hn, &sh, &ch);
  io.x = (float)x; io.y = (float)y; io.h = hn; io.v = (float)v;
  io.vx = io.v * ch; io.vy = io.v * sh;      // State.velocity of a State without vx, vy (state.py:160-165)
  io.ch = ch; io.sh = sh;
  io.w0 = (float)om_f; io.w1 = (float)om_r;
}

// ------------------------------------------------------------------------------------------
// PointMass.step  (point_mass.py:209-232).  The acceleration is NOT clipped (:222-225 computes
// a clipped magnitude and drops it).  Input velocity = (vx, vy); heading = atan2(new velocity).
// ------------------------------------------------------------------------------------------
T2D_HD double pm_t1(double ax, double ay, double vx, double vy, double lim, double sign, double dt) {
  const double a_ = ax * ax + ay * ay;                    // :106-108 / :141-143
  const double b_ = 2.0 * (ax * vx + ay * vy);
  const double c_ = vx * vx + vy * vy - lim * lim;
  double t1;
  if (fabs(a_) < 1e-12) {
    t1 = fabs(b_) < 1e-12 ? 0.0 : -c_ / b_;               // :111-118
  } else {
    const double disc = fmax(0.0, b_ * b_ - 4.0 * a_ * c_);
    t1 = (-b_ + sign * sqrt(disc)) / (2.0 * a_);          // :124 (-) / :159 (+)
  }
  return clampd(t1, 0.0, dt);                             // :127
}

T2D_HD void pointmass_newton_step(OneIO& io, const Params& p, double dt) {
  const double ax = io.a0, ay = io.a1, vx = io.vx, vy = io.vy;
  const double nvx = vx + ax * dt, nvy = vy + ay * dt;    // :88-89
  const double nsp = sqrt(nvx * nvx + nvy * nvy);
  const double slo = p.speed_lo, shi = p.speed_hi;
  double x, y, ovx, ovy;
  if (slo <= nsp && nsp <= shi) {                          // :93-101
    x = (double)io.x + vx * dt + 0.5 * ax * dt * dt;
    y = (double)io.y + vy * dt + 0.5 * ay * dt * dt;
    ovx = nvx; ovy = nvy;
  } else {
    const bool low = nsp < slo;                            // :105 else :140
    const double t1 = pm_t1(ax, ay, vx, vy, low ? slo : shi, low ? -1.0 : 1.0, dt);
    const double t2 = dt - t1;
    ovx = vx + ax * t1; ovy = vy + ay * t1;
    x = (double)io.x + vx * t1 + 0.5 * ax * t1 * t1 + ovx * t2;
    y = (double)io.y + vy * t1 + 0.5 * ay * t1 * t1 + ovy * t2;
  }
  io.x = (float)x; io.y = (float)y;
  io.vx = (float)ovx; io.vy = (float)ovy;
  io.h = (float)atan2(ovy, ovx);
  io.v = (float)sqrt(ovx * ovx + ovy * ovy);               // State.speed (state.py:143-146)
  sincos_fast(io.h, &io.sh, &io.ch);
}

T2D_HD void pointmass_euler_step(OneIO& io, const Params& p, int n_steps, double dt, double dt_rem) {
  const double ax = io.a0, ay = io.a1;                     // point_mass.py:177-207
  double vx = io.vx, vy = io.vy, x = io.x, y = io.y, heading = io.h;
  const double slo = p.speed_lo, shi = p.speed_hi;
  const int total = n_steps + (dt_rem > 0.0 ? 1 : 0);
  for (int it = 0; it < total; ++it) {
    const double h = it < n_steps ? dt : dt_rem;
    vx += ax * h;
    vy += ay * h;
    const double sp = sqrt(vx * vx + vy * vy);
    const double cl = clampd(sp, slo, shi);
    if (fabs(sp - cl) > 1e-12) {                           // :195
      vx = cl * cos(heading);
      vy = cl * sin(heading);
    }
    x += vx * h;
    y += vy * h;
    heading = atan2(vy, vx);
  }
  io.x = (float)x; io.y = (float)y; io.h = (float)heading;
  io.vx = (float)vx; io.vy = (float)vy;
  io.v = (float)sqrt(vx * vx + vy * vy);
  sincos_fast(io.h, &io.sh, &io.ch);
}

// ------------------------------------------------------------------------------------------
// Sampled resets (K13 / K14; DESIGN.md section 1 "Sampled resets")
// ------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11): stateless and counter-based, so
// every thread that needs a draw recomputes it from (key, counter).  Counter 0 with key 0 gives 6627e8d5 e169c58d
// bc57ac4c 9b00dbd8 (Random123's known-answer vector; cuRAND's Philox4_32_10 at seed 0, offset 0 gives the same words).
struct U4 { uint32_t x, y, z, w; };

T2D_HD uint32_t mulhi32(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __umulhi(a, b);
#else
  return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

T2D_HD U4 philox4x32_10(U4 c, uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = mulhi32(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = mulhi32(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = U4{hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0};
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c;
}

// Draw d of scenario n in its episode e under a 64-bit seed: key (seed low, seed high), counter (d, n, e, 0).
T2D_HD U4 episode_draw(uint64_t seed, uint32_t d, uint32_t n, uint32_t e) {
  return philox4x32_10(U4{d, n, e, 0u}, (uint32_t)seed, (uint32_t)(seed >> 32));
}

// The pool row of a draw word over P rows: multiply-high, bias below P / 2^32.
T2D_HD int draw_row(uint32_t u, int P) { return (int)(((uint64_t)u * (uint32_t)P) >> 32); }

// (u >> 8) 2^-24: exact in fp32, in [0, 1).  Then lo + f (hi - lo), each operation rounded on its own (no FMA), in [lo, hi].
T2D_HD float draw_unit(uint32_t u) { return (float)(u >> 8) * 5.9604644775390625e-8f; }
#if defined(__CUDA_ARCH__)
#define T2D_FADD_RN(a, b) __fadd_rn((a), (b))
#define T2D_FSUB_RN(a, b) __fsub_rn((a), (b))
#define T2D_FMUL_RN(a, b) __fmul_rn((a), (b))
#else
#define T2D_FADD_RN(a, b) ((a) + (b))   // (host builds use -ffp-contract=off)
#define T2D_FSUB_RN(a, b) ((a) - (b))
#define T2D_FMUL_RN(a, b) ((a) * (b))
#endif
T2D_HD float draw_range(uint32_t u, float lo, float hi) {
  return T2D_FADD_RN(lo, T2D_FMUL_RN(draw_unit(u), T2D_FSUB_RN(hi, lo)));
}

// Try t of a slot: the candidate (x, y, heading, speed) from the four words of its draw and the slot's jitter row
// jit[8] = (lo, hi) of dx, dy, dheading, dspeed.
struct Cand { float x, y, h, v; };
T2D_HD Cand jitter_candidate(U4 u, const float* jit, float x, float y, float h, float v) {
  Cand c;
  c.x = T2D_FADD_RN(x, draw_range(u.x, jit[0], jit[1]));
  c.y = T2D_FADD_RN(y, draw_range(u.y, jit[2], jit[3]));
  c.h = wrap_two_pi(T2D_FADD_RN(h, draw_range(u.z, jit[4], jit[5])));
  c.v = T2D_FADD_RN(v, draw_range(u.w, jit[6], jit[7]));
  return c;
}

// ------------------------------------------------------------------------------------------
// Lidar (K4)
// ------------------------------------------------------------------------------------------
struct BeamWindow { int x, y; };   // first beam, number of beams (wraps modulo n_beams)

// Beam window of an edge.  The reference tests every (beam, edge) pair, but its filters (:201-209) keep an
// intersection only if it lies on the edge (within 1e-8) AND on the beam's forward ray (within 2e-8 of the origin
// side): a beam can score on an edge only if its direction falls inside the angle the edge subtends at the ego.  The
// window is that angular interval widened by a whole beam on either side (the 1e-8 slacks are < 1e-5 rad beyond 1 cm
// from the ego, atan2f is good to 1e-6 rad, beams are >= 1.7e-3 rad apart); edges that come within 1 cm of the ego, or
// subtend nearly pi, get every beam.  Beams are uniformly spaced, theta_b = 2 pi b / n_beams (lidar.py:160).
T2D_HD BeamWindow beam_window(double x1, double y1, double x2, double y2, double dist2, int n_beams) {
  if (dist2 < 1e-4) return BeamWindow{0, n_beams};
  const float a1 = atan2f((float)y1, (float)x1), a2 = atan2f((float)y2, (float)x2);
  float diff = a2 - a1;
  if (diff > 3.14159265f) diff -= 6.28318531f;
  if (diff < -3.14159265f) diff += 6.28318531f;
  if (fabsf(diff) > 3.0f) return BeamWindow{0, n_beams};
  float start = diff >= 0.0f ? a1 : a2;
  if (start < 0.0f) start += 6.28318531f;
  const float inv = (float)n_beams * 0.159154943f;      // beams per radian
  const int lo = (int)floorf(start * inv) - 1;
  const int hi = (int)ceilf((start + fabsf(diff)) * inv) + 1;
  const int cnt = hi - lo + 1 < n_beams ? hi - lo + 1 : n_beams;
  return BeamWindow{((lo % n_beams) + n_beams) % n_beams, cnt};
}


// ==========================================================================================
// Closed-set predicates.  *_f32 return 1 (intersects), 0 (disjoint) or -1 (inside the fp32
// error bound: caller must ask the *_f64 twin).  *_f64 evaluate exactly the float64 formulas
// of oracle/geometry.py on the fp32 inputs.
// Pose of an OBB: centre (x, y), (c, s) = (cos, sin) heading, half extents (l, w).
// ==========================================================================================
constexpr float EPS_LIN = 2e-6f;  // >= 4x the forward error of the fp32 evaluation, relative to the magnitudes summed

T2D_HD int obb_obb_f32(float xa, float ya, float ca, float sa, float la, float wa,
                       float xb, float yb, float cb, float sb, float lb, float wb) {
  const float tx = xb - xa, ty = yb - ya;
  const float c = fmaf(ca, cb, sa * sb), s = fmaf(ca, sb, -sa * cb);
  const float ac = fabsf(c), as = fabsf(s);
  const float m0 = fabsf(fmaf(tx, ca, ty * sa)) - (la + fmaf(lb, ac, wb * as));
  const float m1 = fabsf(fmaf(ty, ca, -tx * sa)) - (wa + fmaf(lb, as, wb * ac));
  const float m2 = fabsf(fmaf(tx, cb, ty * sb)) - (lb + fmaf(la, ac, wa * as));
  const float m3 = fabsf(fmaf(ty, cb, -tx * sb)) - (wb + fmaf(la, as, wa * ac));
  const float e = EPS_LIN * (fabsf(tx) + fabsf(ty) + la + wa + lb + wb);
  const float mx = fmaxf(fmaxf(m0, m1), fmaxf(m2, m3));
  if (mx > e) return 0;
  if (mx < -e) return 1;
  return -1;
}

T2D_HD bool obb_obb_f64(double xa, double ya, double ha, double la, double wa,
                        double xb, double yb, double hb, double lb, double wb) {
  double sa, ca, sb, cb;
  sincos(ha, &sa, &ca);
  sincos(hb, &sb, &cb);
  const double tx = xb - xa, ty = yb - ya;
  const double c = ca * cb + sa * sb, s = ca * sb - sa * cb;
  const double ac = fabs(c), as = fabs(s);
  return fabs(tx * ca + ty * sa) <= la + (lb * ac + wb * as) &&
         fabs(ty * ca - tx * sa) <= wa + (lb * as + wb * ac) &&
         fabs(tx * cb + ty * sb) <= lb + (la * ac + wa * as) &&
         fabs(ty * cb - tx * sb) <= wb + (la * as + wa * ac);
}

T2D_HD int obb_circle_f32(float xa, float ya, float ca, float sa, float la, float wa,
                          float xc, float yc, float r) {
  const float tx = xc - xa, ty = yc - ya;
  const float qx = fabsf(fmaf(tx, ca, ty * sa)) - la;
  const float qy = fabsf(fmaf(ty, ca, -tx * sa)) - wa;
  const float dx = fmaxf(qx, 0.0f), dy = fmaxf(qy, 0.0f);
  const float m = fmaf(dx, dx, dy * dy) - r * r;
  const float e1 = EPS_LIN * (fabsf(tx) + fabsf(ty) + la + wa + r);
  const float e = fmaf(2.0f * e1, dx + dy + r, e1 * e1);
  if (m > e) return 0;
  if (m < -e) return 1;
  return -1;
}

T2D_HD bool obb_circle_f64(double xa, double ya, double ha, double la, double wa,
                           double xc, double yc, double r) {
  double sa, ca;
  sincos(ha, &sa, &ca);
  const double tx = xc - xa, ty = yc - ya;
  const double qx = fabs(tx * ca + ty * sa) - la;
  const double qy = fabs(ty * ca - tx * sa) - wa;
  const double dx = fmax(qx, 0.0), dy = fmax(qy, 0.0);
  return dx * dx + dy * dy <= r * r;
}

T2D_HD int circle_circle_f32(float xa, float ya, float ra, float xb, float yb, float rb) {
  const float tx = xb - xa, ty = yb - ya;
  const float d2 = fmaf(tx, tx, ty * ty), rr = (ra + rb) * (ra + rb);
  const float e = 4.0f * EPS_LIN * (d2 + rr);
  const float m = d2 - rr;
  if (m > e) return 0;
  if (m < -e) return 1;
  return -1;
}

T2D_HD bool circle_circle_f64(double xa, double ya, double ra, double xb, double yb, double rb) {
  const double tx = xb - xa, ty = yb - ya;
  return tx * tx + ty * ty <= (ra + rb) * (ra + rb);
}

T2D_HD int obb_segment_f32(float xa, float ya, float ca, float sa, float la, float wa,
                           float x1, float y1, float x2, float y2) {
  const float ux = x1 - xa, uy = y1 - ya, vx = x2 - xa, vy = y2 - ya;
  const float p1x = fmaf(ux, ca, uy * sa), p1y = fmaf(uy, ca, -ux * sa);
  const float p2x = fmaf(vx, ca, vy * sa), p2y = fmaf(vy, ca, -vx * sa);
  const float dx = p2x - p1x, dy = p2y - p1y;
  const float e1 = EPS_LIN * (fabsf(ux) + fabsf(uy) + fabsf(vx) + fabsf(vy) + la + wa);
  const float m0 = -la - fmaxf(p1x, p2x);
  const float m1 = fminf(p1x, p2x) - la;
  const float m2 = -wa - fmaxf(p1y, p2y);
  const float m3 = fminf(p1y, p2y) - wa;
  const float mb = fmaxf(fmaxf(m0, m1), fmaxf(m2, m3));
  const float m4 = fabsf(fmaf(p1x, dy, -p1y * dx)) - fmaf(la, fabsf(dy), wa * fabsf(dx));
  const float e4 = 2.0f * e1 * (fabsf(dx) + fabsf(dy) + fabsf(p1x) + fabsf(p1y) + la + wa);
  if (mb > e1 || m4 > e4) return 0;
  if (mb < -e1 && m4 < -e4) return 1;
  return -1;
}

T2D_HD bool obb_segment_f64(double xa, double ya, double ha, double la, double wa,
                            double x1, double y1, double x2, double y2) {
  double sa, ca;
  sincos(ha, &sa, &ca);
  const double ux = x1 - xa, uy = y1 - ya, vx = x2 - xa, vy = y2 - ya;
  const double p1x = ux * ca + uy * sa, p1y = uy * ca - ux * sa;
  const double p2x = vx * ca + vy * sa, p2y = vy * ca - vx * sa;
  const double dx = p2x - p1x, dy = p2y - p1y;
  return fmax(p1x, p2x) >= -la && fmin(p1x, p2x) <= la && fmax(p1y, p2y) >= -wa && fmin(p1y, p2y) <= wa &&
         fabs(p1x * dy - p1y * dx) <= la * fabs(dy) + wa * fabs(dx);
}

T2D_HD int circle_segment_f32(float xc, float yc, float r, float x1, float y1, float x2, float y2) {
  const float dx = x2 - x1, dy = y2 - y1, ux = xc - x1, uy = yc - y1;
  const float dd = fmaf(dx, dx, dy * dy);
  float t = dd > 0.0f ? fmaf(ux, dx, uy * dy) / dd : 0.0f;
  t = fminf(fmaxf(t, 0.0f), 1.0f);
  const float ex = fmaf(-t, dx, ux), ey = fmaf(-t, dy, uy);
  const float d2 = fmaf(ex, ex, ey * ey);
  const float m = d2 - r * r;
  const float e1 = 2.0f * EPS_LIN * (fabsf(ux) + fabsf(uy) + fabsf(dx) + fabsf(dy) + r);
  const float e = fmaf(2.0f * e1, sqrtf(d2) + r, e1 * e1);
  if (m > e) return 0;
  if (m < -e) return 1;
  return -1;
}

T2D_HD bool circle_segment_f64(double xc, double yc, double r, double x1, double y1, double x2, double y2) {
  const double dx = x2 - x1, dy = y2 - y1, ux = xc - x1, uy = yc - y1;
  const double dd = dx * dx + dy * dy;
  double t = dd > 0.0 ? (ux * dx + uy * dy) / dd : 0.0;
  t = fmin(fmax(t, 0.0), 1.0);
  const double ex = ux - t * dx, ey = uy - t * dy;
  return ex * ex + ey * ey <= r * r;
}

// OutBound.update (out_bound.py:37-48): pose not inside the closed box <=> some corner strictly
// outside.  (ex, ey) = half sizes of the pose's axis-aligned box.  bounds = xmin, xmax, ymin, ymax.
T2D_HD int out_of_bound_f32(float x, float y, float c, float s, float l, float w, bool circle,
                            float xmin, float xmax, float ymin, float ymax) {
  const float ex = circle ? l : fmaf(l, fabsf(c), w * fabsf(s));
  const float ey = circle ? l : fmaf(l, fabsf(s), w * fabsf(c));
  const float a0 = x - xmin, a1 = xmax - x, a2 = y - ymin, a3 = ymax - y;
  const float m = fmaxf(fmaxf(ex - a0, ex - a1), fmaxf(ey - a2, ey - a3));  // > 0 <=> out
  const float e = EPS_LIN * (fmaxf(fmaxf(fabsf(a0), fabsf(a1)), fmaxf(fabsf(a2), fabsf(a3))) + l + w);
  if (m > e) return 1;
  if (m < -e) return 0;
  return -1;
}

T2D_HD bool out_of_bound_f64(double x, double y, double h, double l, double w, bool circle,
                             double xmin, double xmax, double ymin, double ymax) {
  double ex = l, ey = l;
  if (!circle) {
    double s, c;
    sincos(h, &s, &c);
    ex = l * fabs(c) + w * fabs(s);
    ey = l * fabs(s) + w * fabs(c);
  }
  return (x - ex < xmin) || (x + ex > xmax) || (y - ey < ymin) || (y + ey > ymax);
}

// ------------------------------------------------------------------------------------------
// IoU of two rotated rectangles in fp64 (Arrival.update, arrival.py:42-46 and NoAction.update,
// no_action.py:43-46: intersection.area / union.area of two shapely polygons).  The intersection of two convex
// polygons is computed by Sutherland-Hodgman clipping of A against the four half planes of B (both rings are
// counter-clockwise in the reference's corner order), areas by the shoelace formula; union = |A| + |B| - |A n B|.
// Run by one lane per scenario (the ego only), so fp64 costs nothing measurable and keeps the thresholds
// (>= 0.95, > 0.999) within 1e-12 of the float64 oracle.
// ------------------------------------------------------------------------------------------
T2D_HD void rect_corners_f64(double x, double y, double h, double l, double w, double (&cx)[4], double (&cy)[4]) {
  double s, c;
  sincos(h, &s, &c);
  const double lx[4] = {l, l, -l, -l}, ly[4] = {-w, w, w, -w};   // vehicle.py:133-140
  for (int i = 0; i < 4; ++i) {
    cx[i] = x + lx[i] * c - ly[i] * s;                             // vehicle.py:272-281
    cy[i] = y + lx[i] * s + ly[i] * c;
  }
}

T2D_HD double rect_iou_f64(double xa, double ya, double ha, double la, double wa, double xb, double yb, double hb, double lb,
                           double wb) {
  double ax[4], ay[4], bx[4], by[4];
  rect_corners_f64(xa, ya, ha, la, wa, ax, ay);
  rect_corners_f64(xb, yb, hb, lb, wb, bx, by);
  double px[10], py[10], qx[10], qy[10];
  int n = 4;
  for (int i = 0; i < 4; ++i) { px[i] = ax[i]; py[i] = ay[i]; }
  for (int e = 0; e < 4 && n > 0; ++e) {           // clip against edge b[e] -> b[e+1]; inside = left of it
    const double ex = bx[(e + 1) & 3] - bx[e], ey = by[(e + 1) & 3] - by[e];
    int m = 0;
    for (int i = 0; i < n; ++i) {
      const int j = i + 1 == n ? 0 : i + 1;
      const double di = ex * (py[i] - by[e]) - ey * (px[i] - bx[e]);
      const double dj = ex * (py[j] - by[e]) - ey * (px[j] - bx[e]);
      if (di >= 0.0) { qx[m] = px[i]; qy[m] = py[i]; ++m; }
      if ((di >= 0.0) != (dj >= 0.0)) {
        const double t = di / (di - dj);
        qx[m] = px[i] + t * (px[j] - px[i]);
        qy[m] = py[i] + t * (py[j] - py[i]);
        ++m;
      }
    }
    n = m;
    for (int i = 0; i < n; ++i) { px[i] = qx[i]; py[i] = qy[i]; }
  }
  double inter = 0.0;
  for (int i = 0; i < n; ++i) {
    const int j = i + 1 == n ? 0 : i + 1;
    inter += px[i] * py[j] - px[j] * py[i];
  }
  inter = 0.5 * fabs(inter);
  const double uni = 4.0 * la * wa + 4.0 * lb * wb - inter;
  return uni > 0.0 ? inter / uni : 0.0;
}

}  // namespace t2d
