// common.cuh -- shared helpers for libb2rl.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/b2rl.h"

namespace b2rl {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return B2RL_ERR_CUDA;
  }
  count_launch();
  return B2RL_OK;
}

// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  Kernels on the per-update chain are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization: the next kernel's CTAs are scheduled, and run their prologue
// (barrier init, tensor-map prefetch), while the previous kernel is still executing; they then block in
// pdl_wait() until the previous kernel has completed and its memory is visible.  Contract for every kernel launched
// through launch_pdl(): (1) pdl_wait() is executed on EVERY path before the first global-memory access of any kind and
// before any early return; (2) pdl_trigger() comes after pdl_wait(), so that the kernel after this one can only start once
// the kernel before this one has completed (no kernel ever overlaps its grand-predecessor).
// Without the launch attribute both instructions are no-ops.  b2rl_set_pdl(0) / B2RL_PDL=0 turns the attribute off.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_sync() { pdl_wait(); pdl_trigger(); }

bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline void launch_ordered(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  // plain stream order (no programmatic overlap) for kernels measured to be faster without it
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

#define B2RL_REQUIRE(cond, msg)                     \
  do {                                              \
    if (!(cond)) {                                  \
      b2rl::set_error("%s: %s", __func__, msg);     \
      return B2RL_ERR_ARG;                          \
    }                                               \
  } while (0)

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11): counter-based, one call = 4 x 32 random bits.
// ---------------------------------------------------------------------------------------------
struct Philox {
  __device__ static inline uint4 gen(uint64_t seed, uint64_t ctr_lo, uint64_t ctr_hi) {
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    uint32_t c0 = (uint32_t)ctr_lo, c1 = (uint32_t)(ctr_lo >> 32), c2 = (uint32_t)ctr_hi, c3 = (uint32_t)(ctr_hi >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
      uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
      uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
      uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
      c0 = n0; c1 = n1; c2 = n2; c3 = n3;
      k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
  }
  // uniform double in [0,1) with 53 random bits (the resolution of CPython's random.random())
  __device__ static inline double u53(uint64_t seed, uint64_t ctr, uint64_t stream) {
    uint4 r = gen(seed, ctr, stream);
    uint64_t a = r.x >> 5, b = r.y >> 6;
    return (double)(a * 67108864ull + b) * (1.0 / 9007199254740992.0);
  }
  // integer in [0, n): multiply-high of a 64-bit draw (bias < 2^-40 for n <= 2^24)
  __device__ static inline uint64_t below(uint64_t seed, uint64_t ctr, uint64_t stream, uint64_t n) {
    uint4 r = gen(seed, ctr, stream);
    uint64_t x = ((uint64_t)r.x << 32) | r.y;
    return __umul64hi(x, n);
  }
  // uniform float in [0, 1) with 24 random bits
  __device__ static inline float u24(uint64_t seed, uint64_t ctr, uint64_t stream) {
    return (gen(seed, ctr, stream).x >> 8) * (1.0f / 16777216.0f);
  }
  // standard normal: Box-Muller on two 24-bit uniforms of one draw (u1 in (0, 1], so the log is finite)
  __device__ static inline float normal(uint64_t seed, uint64_t ctr, uint64_t stream) {
    const uint4 r = gen(seed, ctr, stream);
    const float u1 = ((r.x >> 8) + 1) * (1.0f / 16777216.0f), u2 = (r.y >> 8) * (1.0f / 16777216.0f);
    return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
  }
};

// ---------------------------------------------------------------------------------------------
// block-wide reductions (blockDim.x multiple of 32, <= 1024)
// ---------------------------------------------------------------------------------------------
template <typename T, typename Op>
__device__ inline T warp_reduce(T v, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <typename T, typename Op>
__device__ inline T block_reduce(T v, Op op, T identity, T* smem /* >= 32 */) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_reduce(v, op);
  __syncthreads();
  if (lane == 0) smem[w] = v;
  __syncthreads();
  T r = (threadIdx.x < nw) ? smem[threadIdx.x] : identity;
  if (w == 0) {
    r = warp_reduce(r, op);
    if (lane == 0) smem[0] = r;
  }
  __syncthreads();
  r = smem[0];
  __syncthreads();
  return r;
}

struct OpAdd { template <typename T> __device__ T operator()(T a, T b) const { return a + b; } };
struct OpMax { template <typename T> __device__ T operator()(T a, T b) const { return a > b ? a : b; } };

}  // namespace b2rl
