// dense.cu -- epilogues of the dense path (NatureConvBody / FCBody layers, network_bodies.py:27-33,70-73):
//   forward   y = relu(conv_or_linear(x) + bias)          -> b2rl_bias_act_bf16 (in place on the bf16 GEMM output)
//   backward  g = gy * (y > 0);  dbias = sum_rows g       -> b2rl_act_bwd_bias_grad_bf16 (one pass, block partials + atomics)
// Activations are bf16 [rows][C] (NHWC flattened: rows = batch x spatial), bias / dbias are fp32.
// Both kernels are pure streaming passes (L2 / HBM bound): 16-byte vector loads, 8 channels per thread.  sm_90a only.
#include "common.cuh"

namespace b2rl {

__device__ __forceinline__ void unpack8(const int4& v, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    float2 t = __bfloat1622float2(h[k]);
    f[2 * k] = t.x;
    f[2 * k + 1] = t.y;
  }
}
__device__ __forceinline__ int4 pack8(const float* f) {
  int4 v;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&v);
#pragma unroll
  for (int k = 0; k < 4; ++k) h[k] = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
  return v;
}

__global__ void __launch_bounds__(256) bias_act_kernel(__nv_bfloat16* __restrict__ y, const float* __restrict__ bias,
                                                       int64_t n8, int C8, int relu) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  // n8 = rows*C/8 vectors; vector e covers channels (e % C8)*8 .. +7
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n8; e += (int64_t)gridDim.x * blockDim.x) {
    const int c0 = (int)(e % C8) * 8;
    int4 v = reinterpret_cast<const int4*>(y)[e];
    float f[8];
    unpack8(v, f);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      f[k] += __ldg(bias + c0 + k);
      if (relu) f[k] = fmaxf(f[k], 0.0f);
    }
    reinterpret_cast<int4*>(y)[e] = pack8(f);
  }
}

// split-K GEMM results (fp32) -> bf16 activations with bias + ReLU
__global__ void __launch_bounds__(256) bias_act_f32_kernel(const float* __restrict__ x, const float* __restrict__ bias,
                                                           __nv_bfloat16* __restrict__ y, int64_t n8, int C8, int relu) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n8; e += (int64_t)gridDim.x * blockDim.x) {
    const int c0 = (int)(e % C8) * 8;
    const float4 a = reinterpret_cast<const float4*>(x)[2 * e], b = reinterpret_cast<const float4*>(x)[2 * e + 1];
    float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      f[k] += __ldg(bias + c0 + k);
      if (relu) f[k] = fmaxf(f[k], 0.0f);
    }
    reinterpret_cast<int4*>(y)[e] = pack8(f);
  }
}

// Layout changes between the layers of the grid-GEMM convolution stack.  With a map the kernel walks the DESTINATION rows
// (a G x G grid per image) and returns the source row that feeds each, or -1 for a padding row (written as zeros):
//   map 0: identity
//   map 1: G x G grid rows <- compact V x V positions per image             (fc4's input gradient -> conv3's output grid)
//   map 2: G x G grid rows (oy, ox) <- space-to-depth(2) rows [b][oy/2][ox/2], channel group (oy%2, ox%2); the source is
//          addressed as rows*4 "virtual rows" of C channels                 (conv2's input gradient -> conv1's output grid)
__device__ __forceinline__ int64_t src_row(int64_t r, int map, int G, int V) {
  if (map == 0) return r;
  const int64_t b = r / (G * G);
  const int rem = (int)(r - b * G * G);
  const int oy = rem / G, ox = rem - oy * G;
  if (oy >= V || ox >= V) return -1;
  if (map == 1) return b * V * V + oy * V + ox;
  const int h = V >> 1;
  return ((b * h * h + (oy >> 1) * h + (ox >> 1)) << 2) | (((oy & 1) << 1) | (ox & 1));
}

// each thread owns one 8-channel group and walks rows with stride (threads per block / C8) * gridDim
__global__ void __launch_bounds__(256) act_bwd_kernel(const __nv_bfloat16* __restrict__ gy,
                                                      const __nv_bfloat16* __restrict__ y, int64_t rows, int C8, int relu,
                                                      __nv_bfloat16* __restrict__ gx, float* __restrict__ dbias,
                                                      int map, int G, int V) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ float sred[];          // [rows_per_block][C] partial sums
  const int C = C8 * 8;
  const int rpb = blockDim.x / C8;         // rows handled per block per iteration
  const int lr = threadIdx.x / C8, cg = threadIdx.x % C8;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (lr < rpb) {
    for (int64_t r = (int64_t)blockIdx.x * rpb + lr; r < rows; r += (int64_t)gridDim.x * rpb) {
      const int64_t sr = src_row(r, map, G, V);
      if (sr < 0) {                                        // padding row of the destination grid
        reinterpret_cast<int4*>(gx)[r * C8 + cg] = make_int4(0, 0, 0, 0);
        continue;
      }
      const int64_t e = sr * C8 + cg;
      int4 g4 = reinterpret_cast<const int4*>(gy)[e];
      float g[8];
      unpack8(g4, g);
      if (relu) {
        int4 y4 = reinterpret_cast<const int4*>(y)[e];
        float yv[8];
        unpack8(y4, yv);
#pragma unroll
        for (int k = 0; k < 8; ++k) g[k] = yv[k] > 0.0f ? g[k] : 0.0f;
        if (gx) reinterpret_cast<int4*>(gx)[r * C8 + cg] = pack8(g);
      } else if (gx && (gx != gy || map != 0)) {
        reinterpret_cast<int4*>(gx)[r * C8 + cg] = g4;
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += g[k];
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) sred[lr * C + cg * 8 + k] = acc[k];
  }
  __syncthreads();
  // block partial -> dbias with fp32 atomics (dbias is zeroed by the caller; the summation order over blocks is not
  // fixed, which perturbs the last bits of a bias gradient -- the deterministic single-block reduction it replaces was
  // latency-bound)
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.0f;
    for (int q = 0; q < rpb; ++q) s += sred[q * C + c];
    atomicAdd(dbias + c, s);
  }
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_bias_act_bf16(uint16_t* y, const float* bias, int64_t rows, int32_t C, int32_t relu, void* stream) {
  B2RL_REQUIRE(y && bias, "null pointer");
  B2RL_REQUIRE(rows > 0 && C > 0 && C % 8 == 0, "C must be a positive multiple of 8");
  B2RL_REQUIRE(reinterpret_cast<uintptr_t>(y) % 16 == 0, "y must be 16-byte aligned");
  const int64_t n8 = rows * C / 8;
  int blocks = (int)((n8 + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  launch_pdl(bias_act_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, reinterpret_cast<__nv_bfloat16*>(y), bias, n8, C / 8, relu);
  return check_launch("b2rl_bias_act_bf16");
}

extern "C" int b2rl_act_bwd_bias_grad_bf16(const uint16_t* gy, const uint16_t* y, int64_t rows, int32_t C, int32_t relu,
                                           uint16_t* gx, float* dbias, float* partial, int32_t* counter, int32_t row_map,
                                           int32_t G, int32_t V, void* stream) {
  B2RL_REQUIRE(row_map >= 0 && row_map <= 2 && (row_map == 0 || (G > 0 && V > 0 && V <= G)), "bad row map");
  B2RL_REQUIRE(row_map == 0 || gx != gy, "a row-mapped gradient cannot be written in place");
  B2RL_REQUIRE(gy && dbias && (y || !relu), "null pointer");
  (void)partial; (void)counter;
  cudaMemsetAsync(dbias, 0, sizeof(float) * C, (cudaStream_t)stream);
  B2RL_REQUIRE(rows > 0 && C > 0 && C % 8 == 0 && C <= 2048, "C must be a multiple of 8, <= 2048");
  const int C8 = C / 8;
  const int rpb = 256 / C8 > 0 ? 256 / C8 : 1;
  B2RL_REQUIRE(C8 <= 256, "C too large");
  int64_t want = (rows + rpb - 1) / rpb;
  int64_t by_work = rows * C / 4096 + 1;               // >= 4K elements per block: few partials for small layers
  if (want > by_work) want = by_work;
  int blocks = (int)(want < 592 ? want : 592);         // 4 CTAs per SM keep enough 16-byte loads in flight
  size_t smem = (size_t)rpb * C * sizeof(float);
  launch_pdl(act_bwd_kernel, dim3(blocks), dim3(256), smem, (cudaStream_t)stream, 
      reinterpret_cast<const __nv_bfloat16*>(gy), reinterpret_cast<const __nv_bfloat16*>(y), rows, C8, relu,
      reinterpret_cast<__nv_bfloat16*>(gx), dbias, row_map, G, V);
  return check_launch("b2rl_act_bwd_bias_grad_bf16");
}

extern "C" int b2rl_bias_act_f32_to_bf16(const float* x, const float* bias, uint16_t* y, int64_t rows, int32_t C,
                                         int32_t relu, void* stream) {
  B2RL_REQUIRE(x && bias && y, "null pointer");
  B2RL_REQUIRE(rows > 0 && C > 0 && C % 8 == 0, "C must be a positive multiple of 8");
  B2RL_REQUIRE(reinterpret_cast<uintptr_t>(x) % 16 == 0 && reinterpret_cast<uintptr_t>(y) % 16 == 0, "16-byte alignment");
  const int64_t n8 = rows * C / 8;
  int blocks = (int)((n8 + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  launch_pdl(bias_act_f32_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, x, bias, reinterpret_cast<__nv_bfloat16*>(y), n8, C / 8, relu);
  return check_launch("b2rl_bias_act_f32_to_bf16");
}
