// disthead.cu -- the element-wise halves of the distributional heads (CategoricalNet / QuantileNet, network_heads.py:40-55, 89-102)
// around the wgmma GEMMs of csrc/gemm.cu, so that the C51 / QR-DQN update runs no cuBLAS / ATen kernel:
//
//   forward   logits [B][A*N] = phi W^T + b        b2rl_gemm_bf16 (bias in the epilogue, fp32 out)
//             prob, log_prob = softmax / log_softmax over the N atoms of every (b, a)      dist_softmax_kernel   (C51)
//   backward  dlogits = dlog_prob - prob * sum_n dlog_prob   (log_softmax backward; QR: dlogits = dquantile)
//             -> bf16 GEMM operand g [B][ld] + bias gradient (column sums)                 dist_bwd_prep_kernel
//             dW = g^T phi, dphi = relu_mask(g W)  b2rl_gemm_bf16 (MN-major operands) / b2rl_gemm_bwd_bf16
// sm_90a only.
#include "common.cuh"

namespace b2rl {

// one warp per (b, a) row of N atoms
__global__ void __launch_bounds__(256) dist_softmax_kernel(const float* __restrict__ logits, int rows, int N,
                                                           float* __restrict__ prob, float* __restrict__ logp) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  const int lane = threadIdx.x & 31, r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* x = logits + (int64_t)r * N;
  float m = -INFINITY;
  for (int i = lane; i < N; i += 32) m = fmaxf(m, x[i]);
  m = warp_reduce(m, OpMax());
  float s = 0.0f;
  for (int i = lane; i < N; i += 32) s += expf(x[i] - m);
  s = warp_reduce(s, OpAdd());
  const float ls = logf(s);
  for (int i = lane; i < N; i += 32) {
    const float lp = (x[i] - m) - ls;                       // torch.log_softmax: x - max - log(sum exp(x - max))
    if (logp) logp[(int64_t)r * N + i] = lp;
    if (prob) prob[(int64_t)r * N + i] = expf(x[i] - m) / s;
  }
}

// CTA = DB_ROWS batch rows.  Phase 1 (one warp per (b, a) row): dlogit; bf16 store; fp32 copy to shared memory.  Phase 2: column
// sums over the CTA's batch rows, one atomicAdd per column per CTA (B / DB_ROWS per address).
constexpr int DB_ROWS = 8;
__global__ void __launch_bounds__(256) dist_bwd_prep_kernel(const float* __restrict__ dout, const float* __restrict__ prob,
                                                            int B, int A, int N, __nv_bfloat16* __restrict__ g, int ld,
                                                            float* __restrict__ dbias) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ float tile[];                           // [DB_ROWS][A*N]
  const int AN = A * N, b0 = blockIdx.x * DB_ROWS;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int rr = warp; rr < DB_ROWS * A; rr += nw) {
    const int bl = rr / A, a = rr - bl * A, b = b0 + bl;
    float* t = tile + bl * AN + a * N;
    if (b >= B) {
      for (int i = lane; i < N; i += 32) t[i] = 0.0f;
      continue;
    }
    const float* d = dout + ((int64_t)b * A + a) * N;
    float s = 0.0f;
    if (prob) {
      for (int i = lane; i < N; i += 32) s += d[i];
      s = warp_reduce(s, OpAdd());
    }
    const float* p = prob ? prob + ((int64_t)b * A + a) * N : nullptr;
    __nv_bfloat16* go = g + (int64_t)b * ld + a * N;
    for (int i = lane; i < N; i += 32) {
      const float v = p ? d[i] - p[i] * s : d[i];
      t[i] = v;
      go[i] = __float2bfloat16_rn(v);
    }
  }
  // padding columns of the operand row (ld > A*N) are zero
  for (int e = threadIdx.x; e < DB_ROWS * (ld - AN); e += blockDim.x) {
    const int bl = e / (ld - AN), c = AN + e - bl * (ld - AN);
    if (b0 + bl < B) g[(int64_t)(b0 + bl) * ld + c] = __float2bfloat16_rn(0.0f);
  }
  __syncthreads();
  if (dbias) {
    for (int c = threadIdx.x; c < AN; c += blockDim.x) {
      float s = 0.0f;
#pragma unroll
      for (int bl = 0; bl < DB_ROWS; ++bl) s += tile[bl * AN + c];
      atomicAdd(dbias + c, s);
    }
  }
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_dist_softmax(const float* logits, int32_t rows, int32_t N, float* prob, float* log_prob, void* stream) {
  B2RL_REQUIRE(logits && (prob || log_prob), "null pointer");
  B2RL_REQUIRE(rows > 0 && N > 0, "bad shape");
  launch_pdl(dist_softmax_kernel, dim3((rows + 7) / 8), dim3(256), 0, (cudaStream_t)stream, logits, rows, N, prob, log_prob);
  return check_launch("b2rl_dist_softmax");
}

extern "C" int b2rl_dist_head_bwd_prep(const float* dout, const float* prob, int32_t B, int32_t A, int32_t N, uint16_t* g,
                                       int32_t ld, float* dbias, void* stream) {
  B2RL_REQUIRE(dout && g, "null pointer");
  B2RL_REQUIRE(B > 0 && A > 0 && N > 0 && ld >= A * N && ld % 8 == 0, "bad shape (ld >= A*N, multiple of 8)");
  const size_t smem = (size_t)DB_ROWS * A * N * sizeof(float);
  B2RL_REQUIRE(smem <= 200 * 1024, "A * N too large");
  static size_t attr = 0;
  if (smem > attr) {
    cudaFuncSetAttribute(dist_bwd_prep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = smem;
  }
  launch_pdl(dist_bwd_prep_kernel, dim3((B + DB_ROWS - 1) / DB_ROWS), dim3(256), smem, (cudaStream_t)stream, dout, prob, B, A, N,
             reinterpret_cast<__nv_bfloat16*>(g), ld, dbias);
  return check_launch("b2rl_dist_head_bwd_prep");
}
