// t2d_exchange.cuh - t2d_exchange_allgather_kernel: all-gather of the done masks over NVLink peer memory.
#pragma once

#include "t2d_world.cuh"

namespace t2d {

// ============================================================================ done exchange over peer memory
// All-gather of the per-rank done masks as ONE small kernel per rank and step, over NVLink / NVSwitch peer memory:
//   put     warp w serves the peers w, w + warps, ...: its lanes store 16-byte pieces of this rank's mask into slot
//           (step % slots), row `rank`, of that peer's gather ring (the own ring included);
//   signal  every lane fences its stores to system scope, the warp synchronises and lane 0 writes step + 1 into word
//           `rank` of the peer's flag array (a strong relaxed store behind the fence = a release): ONE fence round
//           trip per peer, all peers in parallel - not a chain of release stores issued by one thread;
//   wait    lanes 0 .. world-1 of warp 0 poll the OWN flag array (acquire, system scope) until every rank has signalled
//           step - lag; bounded (`timeout` SM cycles): on expiry the sticky error word is set and dst is filled with 0xFF;
//   copy    the slot of step - lag (all ranks' masks in rank order) goes to the caller's array.
// lag = 0 is the synchronous all-gather (the kernel cannot retire before the slowest rank's tick of this step has
// signalled).  lag >= 1 delivers the masks `lag` steps late: by then every signal has long arrived, the wait never spins
// and the kernel is a few microseconds of posted stores - the exchange leaves the critical path (the consumer of the
// gathered masks, a learner or reset scheduler, is behind the simulation anyway).  The kernels of one rank run in
// stream order and kernel k only completes after every rank has signalled step k - lag, i.e. after every rank's kernel
// k - lag - 1 has copied step k - 2 lag - 1 out: a ring of 2 lag + 2 slots is never overwritten before it was read.
struct AllGatherArgs {
  unsigned char* peer[T2D_MAX_RANKS];   // every rank's exchange allocation (own included)
  unsigned char* base;                  // = peer[rank]
  const unsigned char* local;           // this rank's done mask [n_real]
  unsigned char* dst;                   // [world * n_local]
  int world, rank, n_local, n_real, slots, lag;
  long long timeout;                    // SM cycles the wait may spin
};

__global__ void __launch_bounds__(512) t2d_exchange_allgather_kernel(const __grid_constant__ AllGatherArgs A) {
  __shared__ int s_ok;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
  const size_t flag_off = (size_t)A.slots * A.world * A.n_local;
  unsigned* words = reinterpret_cast<unsigned*>(A.base + flag_off);      // [0, MAX_RANKS): flags; then step, -, -, error
  const unsigned step = words[T2D_MAX_RANKS];
  const size_t row = (size_t)(step % (unsigned)A.slots) * A.world * A.n_local + (size_t)A.rank * A.n_local;
  if (threadIdx.x == 0) s_ok = 1;
  // ---- put + signal, one warp per peer
  const int n16 = A.n_local / 16;   // n_local is a multiple of 16; the tail beyond n_real is zero
  for (int p = warp; p < A.world; p += warps) {
    uint4* out = reinterpret_cast<uint4*>(A.peer[p] + row);
    for (int i = lane; i < n16; i += 32) {
      uint4 v;
      if (16 * i + 16 <= A.n_real && (reinterpret_cast<uintptr_t>(A.local) & 15) == 0) {
        v = __ldcg(reinterpret_cast<const uint4*>(A.local) + i);
      } else {
        unsigned char b[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) b[k] = (16 * i + k < A.n_real) ? A.local[16 * i + k] : (unsigned char)0;
        memcpy(&v, b, 16);
      }
      out[i] = v;
    }
    __threadfence_system();
    __syncwarp();
    if (lane == 0) {
      unsigned* f = reinterpret_cast<unsigned*>(A.peer[p] + flag_off) + A.rank;
      asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(f), "r"(step + 1u) : "memory");
    }
  }
  // ---- wait for step - lag
  const bool deliver = step >= (unsigned)A.lag;
  const unsigned target = step - (unsigned)A.lag;     // the step whose masks this call delivers
  if (deliver && threadIdx.x < (unsigned)A.world) {
    const unsigned* f = words + threadIdx.x;
    const long long t0 = clock64();
    unsigned v;
    for (;;) {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(f) : "memory");
      if (v >= target + 1u) break;
      if (clock64() - t0 > A.timeout) { s_ok = 0; break; }
      __nanosleep(20);
    }
  }
  __syncthreads();
  const size_t bytes = (size_t)A.world * A.n_local;
  if (deliver) {
    if (s_ok) {
      // ---- copy
      const unsigned char* src = A.base + (size_t)(target % (unsigned)A.slots) * bytes;
      if ((reinterpret_cast<uintptr_t>(A.dst) & 15) == 0) {
        for (size_t i = threadIdx.x; i < bytes / 16; i += blockDim.x)
          reinterpret_cast<uint4*>(A.dst)[i] = __ldcg(reinterpret_cast<const uint4*>(src) + i);
      } else {
        for (size_t i = threadIdx.x; i < bytes; i += blockDim.x) A.dst[i] = __ldcg(src + i);
      }
    } else {
      // a rank never showed up: the caller must not mistake stale masks for this step's - 0xFF is no done value
      for (size_t i = threadIdx.x; i < bytes; i += blockDim.x) A.dst[i] = (unsigned char)0xFF;
      if (threadIdx.x == 0) words[T2D_MAX_RANKS + 3] = 1u;
    }
  }
  if (threadIdx.x == 0) words[T2D_MAX_RANKS] = step + 1u;
}

}  // namespace t2d
