// samplersim.cpp - TEST HARNESS ONLY (never shipped, never used by tactics2d_b200).
//
// Compiles the sampled-reset arithmetic of tactics2d_b200/csrc/t2d_math.cuh (Philox4x32-10, the row draw and the jitter
// candidate) with g++ so that tests/test_reset_sampler_host.py can hold it to the Python restatement without a GPU.
#include <cstdint>

#include "../../tactics2d_b200/csrc/t2d_math.cuh"

using namespace t2d;

extern "C" {

// out [n][4]: the words of draw d[i] of scenario s[i] in episode e[i]
void ss_draw(int n, uint64_t seed, const uint32_t* d, const uint32_t* s, const uint32_t* e, uint32_t* out) {
  for (int i = 0; i < n; ++i) {
    const U4 u = episode_draw(seed, d[i], s[i], e[i]);
    out[4 * i] = u.x; out[4 * i + 1] = u.y; out[4 * i + 2] = u.z; out[4 * i + 3] = u.w;
  }
}

void ss_row(int n, const uint32_t* u, int P, int32_t* out) {
  for (int i = 0; i < n; ++i) out[i] = draw_row(u[i], P);
}

void ss_range(int n, const uint32_t* u, const float* lo, const float* hi, float* out) {
  for (int i = 0; i < n; ++i) out[i] = draw_range(u[i], lo[i], hi[i]);
}

// state [n][4] (x, y, heading, speed), u [n][4], jit [n][8] -> out [n][4]
void ss_candidate(int n, const float* state, const uint32_t* u, const float* jit, float* out) {
  for (int i = 0; i < n; ++i) {
    const Cand c = jitter_candidate(U4{u[4 * i], u[4 * i + 1], u[4 * i + 2], u[4 * i + 3]}, jit + 8 * i, state[4 * i],
                                    state[4 * i + 1], state[4 * i + 2], state[4 * i + 3]);
    out[4 * i] = c.x; out[4 * i + 1] = c.y; out[4 * i + 2] = c.h; out[4 * i + 3] = c.v;
  }
}
}
