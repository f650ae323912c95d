// losses.cu -- fused target / loss / gradient kernels of the DQN family.
// Reference: deep_rl/agent/DQN_agent.py:78-127, CategoricalDQN_agent.py:60-89,
// QuantileRegressionDQN_agent.py:55-77, utils/torch_utils.py:47-48.  sm_90a only.
//
// Each entry point replaces ~15-20 eager ATen launches with one kernel that produces the per-sample
// loss tensor the reference's compute_loss returns, the PER priorities / importance weights
// (DQN_agent.py:120-127), the reduced scalar and dLoss/d(network output).  Arithmetic follows the
// reference's operation order in fp32 with explicit _rn intrinsics where FMA contraction would change bits.
#include "common.cuh"

namespace b2rl {

__device__ __forceinline__ float pow_like_torch(float x, float e) {
  // at::pow(Tensor, Scalar) special-cases (aten/native/cpu/PowKernel.cpp): 0.5 -> sqrt, 2 -> x*x, ...
  if (e == 0.5f) return sqrtf(x);
  if (e == 1.0f) return x;
  if (e == 2.0f) return x * x;
  if (e == -0.5f) return 1.0f / sqrtf(x);
  if (e == -1.0f) return 1.0f / x;
  return powf(x, e);
}

// PER importance weight before max-normalisation: (P*B + 1e-6)^(-beta)   (DQN_agent.py:125)
__device__ __forceinline__ float per_raw_weight(float prob, int B, float beta) {
  return pow_like_torch(__fadd_rn(__fmul_rn(prob, (float)B), 1e-6f), -beta);
}

// --------------------------------------------------------------------------------------------- DQN
__global__ void __launch_bounds__(1024) dqn_loss_kernel(const float* __restrict__ q, const float* __restrict__ qn_t,
                                                        const float* __restrict__ qn_o,
                                                        const int64_t* __restrict__ action,
                                                        const float* __restrict__ reward,
                                                        const float* __restrict__ mask, float gamma_n, int B, int A,
                                                        const float* __restrict__ is_prob, float beta, float eps,
                                                        float alpha, float* __restrict__ delta_out,
                                                        float* __restrict__ prio_out, float* __restrict__ loss_out,
                                                        float* __restrict__ dq_out, const float* __restrict__ beta_dev) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ float red[32];
  if (beta_dev) beta = *beta_dev;
  float wmax = 1.0f;
  if (is_prob) {
    float m = 0.0f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) m = fmaxf(m, per_raw_weight(is_prob[b], B, beta));
    wmax = block_reduce(m, OpMax(), 0.0f, red);
  }
  float acc = 0.0f;
  const float invB = 1.0f / (float)B;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const float* qt = qn_t + (int64_t)b * A;
    float qnext;
    if (qn_o) {                                   // DQN_agent.py:88-90: argmax (first max) of the ONLINE net
      const float* qo = qn_o + (int64_t)b * A;
      int best = 0;
      float bv = qo[0];
      for (int a = 1; a < A; ++a)
        if (qo[a] > bv) { bv = qo[a]; best = a; }
      qnext = qt[best];
    } else {                                      // :92
      qnext = qt[0];
      for (int a = 1; a < A; ++a) qnext = fmaxf(qnext, qt[a]);
    }
    const int a_b = (int)action[b];
    const float target = __fadd_rn(reward[b], __fmul_rn(__fmul_rn(gamma_n, qnext), mask[b]));   // :95
    const float delta = __fsub_rn(target, q[(int64_t)b * A + a_b]);                            // :99
    float w = 1.0f;
    if (is_prob) {
      if (prio_out) prio_out[b] = pow_like_torch(__fadd_rn(fabsf(delta), eps), alpha);         // :121
      w = __fdiv_rn(per_raw_weight(is_prob[b], B, beta), wmax);                                // :125-126
    }
    const float wl = __fmul_rn(delta, w);                                                      // :127
    if (delta_out) delta_out[b] = delta;
    acc += __fmul_rn(__fmul_rn(wl, wl), 0.5f);                                                 // :79
    if (dq_out) {
      for (int a = 0; a < A; ++a) dq_out[(int64_t)b * A + a] = 0.0f;
      dq_out[(int64_t)b * A + a_b] = -wl * w * invB;        // d/dq of mean(0.5*(w*(y-q))^2)
    }
  }
  float tot = block_reduce(acc, OpAdd(), 0.0f, red);
  if (threadIdx.x == 0 && loss_out) loss_out[0] = tot * invB;
}

// --------------------------------------------------------------------------------------------- C51
// one CTA (64 threads) per sample
__global__ void __launch_bounds__(64) c51_loss_kernel(const float* __restrict__ log_prob,
                                                      const float* __restrict__ pn_t, const float* __restrict__ pn_o,
                                                      const int64_t* __restrict__ action,
                                                      const float* __restrict__ reward,
                                                      const float* __restrict__ mask, float gamma_n, float v_min,
                                                      float v_max, double lin_start, double lin_step, float delta_atom,
                                                      int B, int A, int N, const float* __restrict__ is_prob, float beta,
                                                      float eps, float alpha, float* __restrict__ kl_out,
                                                      float* __restrict__ prio_out, float* __restrict__ loss_out,
                                                      float* __restrict__ dlogp_out, float* __restrict__ tp_out,
                                                      int32_t* __restrict__ counter, const float* __restrict__ beta_dev) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ float sm[];
  if (beta_dev) beta = *beta_dev;
  float* z = sm;            // [N] atoms
  float* tz = sm + N;       // [N] projected atom positions
  float* pn = sm + 2 * N;   // [N] next-state probabilities of the greedy action
  float* qa = sm + 3 * N;   // [A]
  __shared__ float red[32];
  __shared__ int a_star;
  __shared__ bool is_last;
  const int b = blockIdx.x, t = threadIdx.x;
  for (int k = t; k < N; k += blockDim.x)       // np.linspace(v_min, v_max, N) in float64, then tensor() -> float32
    z[k] = (k == N - 1) ? v_max : (float)__dadd_rn(__dmul_rn((double)k, lin_step), lin_start);
  __syncthreads();
  const float* sel = (pn_o ? pn_o : pn_t) + (int64_t)b * A * N;     // CategoricalDQN_agent.py:66-70
  for (int a = t; a < A; a += blockDim.x) {
    float s = 0.0f;
    for (int k = 0; k < N; ++k) s += __fmul_rn(sel[a * N + k], z[k]);
    qa[a] = s;
  }
  __syncthreads();
  if (t == 0) {
    int best = 0;
    for (int a = 1; a < A; ++a)
      if (qa[a] > qa[best]) best = a;
    a_star = best;
  }
  __syncthreads();
  const float r = reward[b], gm = __fmul_rn(gamma_n, mask[b]);
  for (int k = t; k < N; k += blockDim.x) {
    pn[k] = pn_t[((int64_t)b * A + a_star) * N + k];                                     // :71
    tz[k] = fminf(fmaxf(__fadd_rn(r, __fmul_rn(gm, z[k])), v_min), v_max);               // :75-76
  }
  __syncthreads();
  float w = 1.0f;
  if (is_prob) {
    float m = 0.0f;
    for (int i = t; i < B; i += blockDim.x) m = fmaxf(m, per_raw_weight(is_prob[i], B, beta));
    float wmax = block_reduce(m, OpMax(), 0.0f, red);
    w = __fdiv_rn(per_raw_weight(is_prob[b], B, beta), wmax);
  }
  const int a_b = (int)action[b];
  const float* lp = log_prob + ((int64_t)b * A + a_b) * N;
  const float scale = w / (float)B;
  float kl = 0.0f;
  for (int j = t; j < N; j += blockDim.x) {
    float mj = 0.0f;
    for (int k = 0; k < N; ++k) {                                                        // :78-80
      float c = __fsub_rn(1.0f, __fdiv_rn(fabsf(__fsub_rn(tz[k], z[j])), delta_atom));
      c = fminf(fmaxf(c, 0.0f), 1.0f);
      mj += __fmul_rn(c, pn[k]);
    }
    kl += __fsub_rn(__fmul_rn(mj, logf(__fadd_rn(mj, 1e-5f))), __fmul_rn(mj, lp[j]));   // :85
    if (tp_out) tp_out[(int64_t)b * N + j] = mj;
    if (dlogp_out) {
      for (int a = 0; a < A; ++a) dlogp_out[((int64_t)b * A + a) * N + j] = (a == a_b) ? -mj * scale : 0.0f;
    }
  }
  kl = block_reduce(kl, OpAdd(), 0.0f, red);
  if (t == 0) {
    kl_out[b] = kl;
    if (prio_out && is_prob) prio_out[b] = pow_like_torch(__fadd_rn(fabsf(kl), eps), alpha);
    // weighted per-sample loss parked in dedicated storage for the last CTA: reuse tz? no -> use kl_out + weights again
    __threadfence();
    is_last = (atomicAdd(counter, 1) == B - 1);
  }
  __syncthreads();
  if (is_last) {                                   // deterministic final reduction in index order
    __threadfence();
    float wmax = 1.0f;
    if (is_prob) {
      float m = 0.0f;
      for (int i = t; i < B; i += blockDim.x) m = fmaxf(m, per_raw_weight(is_prob[i], B, beta));
      wmax = block_reduce(m, OpMax(), 0.0f, red);
    }
    float s = 0.0f;
    for (int i = t; i < B; i += blockDim.x) {
      float wi = is_prob ? __fdiv_rn(per_raw_weight(is_prob[i], B, beta), wmax) : 1.0f;
      s += __fmul_rn(__ldcg(kl_out + i), wi);
    }
    s = block_reduce(s, OpAdd(), 0.0f, red);
    if (t == 0) {
      if (loss_out) loss_out[0] = s / (float)B;    // reduce_loss: mean (:88-89)
      *counter = 0;
    }
  }
}

// --------------------------------------------------------------------------------------------- QR-DQN
__device__ __forceinline__ float huber_f(float x, float k) {                 // utils/torch_utils.py:47-48
  float ax = fabsf(x);
  return ax < k ? __fmul_rn(0.5f, __fmul_rn(x, x)) : __fmul_rn(k, __fsub_rn(ax, __fmul_rn(0.5f, k)));
}

// one CTA (256 threads) per sample
__global__ void __launch_bounds__(256) qr_loss_kernel(const float* __restrict__ quant, const float* __restrict__ qnext,
                                                      const int64_t* __restrict__ action,
                                                      const float* __restrict__ reward,
                                                      const float* __restrict__ mask, float gamma_n, float kappa, int B,
                                                      int A, int N, float* __restrict__ vec_out,
                                                      float* __restrict__ loss_out, float* __restrict__ dq_out,
                                                      float* __restrict__ partial, int32_t* __restrict__ counter,
                                                      const float* __restrict__ gw) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ float sm[];
  float* T = sm;           // [N] target quantiles  r + gamma^n * m * theta'(s', a*)
  float* th = sm + N;      // [N] theta(s, a)
  float* tau = sm + 2 * N; // [N]
  float* qsum = sm + 3 * N;  // [A]
  __shared__ float red[32];
  __shared__ int a_star;
  __shared__ bool is_last;
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5, nw = blockDim.x >> 5;
  const float* qn = qnext + (int64_t)b * A * N;
  for (int a = w; a < A; a += nw) {                                  // :60  argmax_a sum_k theta'
    float s = 0.0f;
    for (int k = lane; k < N; k += 32) s += qn[a * N + k];
    s = warp_reduce(s, OpAdd());
    if (lane == 0) qsum[a] = s;
  }
  __syncthreads();
  if (t == 0) {
    int best = 0;
    for (int a = 1; a < A; ++a)
      if (qsum[a] > qsum[best]) best = a;
    a_star = best;
  }
  __syncthreads();
  const int a_b = (int)action[b];
  const float r = reward[b], gm = __fmul_rn(gamma_n, mask[b]);
  for (int k = t; k < N; k += blockDim.x) {
    T[k] = __fadd_rn(r, __fmul_rn(gm, qn[a_star * N + k]));                               // :65
    th[k] = quant[((int64_t)b * A + a_b) * N + k];                                        // :67-69
    tau[k] = (float)((2.0 * k + 1.0) / (2.0 * N));                                        // :44-45
  }
  __syncthreads();
  const float gscale = 1.0f / ((float)B * (float)N);
  // pass 1: gradient wrt theta_i  (sum over target quantiles j)
  for (int i = t; i < N && dq_out; i += blockDim.x) {
    float g = 0.0f;
    const float thi = th[i], taui = tau[i];
    for (int j = 0; j < N; ++j) {
      float u = __fsub_rn(T[j], thi);
      float wq = fabsf(__fsub_rn(taui, u < 0.0f ? 1.0f : 0.0f));
      float hp = fabsf(u) < kappa ? u : (u > 0.0f ? kappa : -kappa);
      g -= (gw ? gw[j] : gscale) * hp * wq;     // gw[j] = dLoss/dvec[j] / B (custom upstream gradient)
    }
    dq_out[((int64_t)b * A + a_b) * N + i] = g;
  }
  if (dq_out) {
    for (int e = t; e < A * N; e += blockDim.x)
      if (e / N != a_b) dq_out[(int64_t)b * A * N + e] = 0.0f;
  }
  if (!partial) return;                      // gradient-only call (autograd backward)
  // pass 2: row sums over i for every target quantile j   (loss.sum(-1), :74)
  for (int j = t; j < N; j += blockDim.x) {
    float s = 0.0f;
    const float Tj = T[j];
    for (int i = 0; i < N; ++i) {
      float u = __fsub_rn(Tj, th[i]);
      float wq = fabsf(__fsub_rn(tau[i], u < 0.0f ? 1.0f : 0.0f));
      s += __fmul_rn(huber_f(u, kappa), wq);                                              // :73
    }
    partial[(int64_t)b * N + j] = s;
  }
  __threadfence();
  __syncthreads();
  if (t == 0) is_last = (atomicAdd(counter, 1) == B - 1);
  __syncthreads();
  if (is_last) {
    __threadfence();
    float tot = 0.0f;
    for (int j = t; j < N; j += blockDim.x) {
      // 8 interleaved partial sums (a fixed order: deterministic): 8 independent loads in flight instead of a chain of B
      float p8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      int i = 0;
      for (; i + 8 <= B; i += 8) {
#pragma unroll
        for (int k = 0; k < 8; ++k) p8[k] += __ldcg(partial + (int64_t)(i + k) * N + j);
      }
      for (; i < B; ++i) p8[0] += __ldcg(partial + (int64_t)i * N + j);
      float s = ((p8[0] + p8[1]) + (p8[2] + p8[3])) + ((p8[4] + p8[5]) + (p8[6] + p8[7]));
      s /= (float)B;                                                                     // .mean(1)
      if (vec_out) vec_out[j] = s;
      tot += s;
    }
    tot = block_reduce(tot, OpAdd(), 0.0f, red);
    if (t == 0) {
      if (loss_out) loss_out[0] = tot / (float)N;                                         // reduce_loss: mean (:76-77)
      *counter = 0;
    }
  }
}

// --------------------------------------------------------------------------------------------- n-step Q-learning
// NStepDQN_agent.py:56-63 for a rollout of T env steps x N workers, q rows t-major (row i = t N + n): bootstrap
// max_a q_T[n] (:56-57), the backward scan ret_t = r_t + discount * m_t * ret_{t+1} (:58-60, the reference's operation
// order), delta = ret - q[a], loss = 0.5 * mean(delta^2) over the T N rows (:63) and gq = dloss/dq = -delta / (T N) at the
// taken action, 0 elsewhere.  One thread per worker column (its scan is sequential in t), NSTEP_THREADS columns per CTA; each
// CTA's sum of delta^2 is parked in partial[cta] and the last CTA to arrive adds the partials in CTA order, so the loss does
// not depend on which CTA finishes when.
constexpr int NSTEP_THREADS = 128;
constexpr int NSTEP_MAX_A = 32;                 // the narrow heads' action limit (csrc/head.cu)
constexpr int NSTEP_MAX_ROWS = 1 << 24;         // T N converts to float exactly

__global__ void __launch_bounds__(NSTEP_THREADS) nstep_q_loss_kernel(const float* __restrict__ q,
                                                                    const float* __restrict__ q_boot,
                                                                    const int64_t* __restrict__ action,
                                                                    const float* __restrict__ reward,
                                                                    const float* __restrict__ mask, float discount, int T,
                                                                    int N, int A, float* __restrict__ ret_out,
                                                                    float* __restrict__ delta_out,
                                                                    float* __restrict__ loss_out, float* __restrict__ gq_out,
                                                                    float* __restrict__ partial,
                                                                    int32_t* __restrict__ counter) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ float red[32];
  __shared__ bool is_last;
  const int n = blockIdx.x * NSTEP_THREADS + threadIdx.x;
  const float rows = (float)(T * N);
  float acc = 0.0f;
  if (n < N) {
    const float* qb = q_boot + (int64_t)n * A;
    float ret = qb[0];
    for (int a = 1; a < A; ++a) ret = fmaxf(ret, qb[a]);
    for (int t = T - 1; t >= 0; --t) {
      const int64_t i = (int64_t)t * N + n;
      ret = __fadd_rn(reward[i], __fmul_rn(__fmul_rn(discount, mask[i]), ret));
      const int a_i = (int)action[i];
      const float delta = __fsub_rn(ret, q[i * A + a_i]);
      if (ret_out) ret_out[i] = ret;
      if (delta_out) delta_out[i] = delta;
      acc = __fadd_rn(acc, __fmul_rn(delta, delta));
      if (gq_out) {
        float* g = gq_out + i * A;
        for (int a = 0; a < A; ++a) g[a] = a == a_i ? __fdiv_rn(-delta, rows) : 0.0f;
      }
    }
  }
  const float s = block_reduce(acc, OpAdd(), 0.0f, red);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = s;
    __threadfence();
    is_last = atomicAdd(counter, 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (is_last && threadIdx.x == 0) {              // deterministic final reduction in CTA order
    __threadfence();
    float tot = 0.0f;
    for (int c = 0; c < (int)gridDim.x; ++c) tot = __fadd_rn(tot, __ldcg(partial + c));
    if (loss_out) loss_out[0] = __fmul_rn(0.5f, __fdiv_rn(tot, rows));
    *counter = 0;
  }
}

// Shape limits of the C51 / QR entry points.  Their dynamic shared memory is (3N + A) floats: 64 KiB at the limits, past the
// 48 KiB a launch gets by default and well inside the 227 KiB per block of sm_90.  A request over 48 KiB raises the kernel's
// limit to the largest accepted request (always the same value, so no call lowers it under a launch a captured graph holds).
constexpr int DIST_MAX_N = 4096, DIST_MAX_A = 4096;
constexpr size_t DIST_MAX_SMEM = (size_t)(3 * DIST_MAX_N + DIST_MAX_A) * sizeof(float);
static_assert(DIST_MAX_SMEM + 1024 <= 227 * 1024, "C51 / QR shared memory at the shape limits exceeds sm_90's per-block limit");

template <typename K>
static int raise_dyn_smem(K kernel, size_t smem, const char* what) {
  if (smem <= 48 * 1024) return B2RL_OK;
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DIST_MAX_SMEM) != cudaSuccess) {
    set_error("%s: cannot raise the dynamic shared-memory limit to %zu bytes", what, DIST_MAX_SMEM);
    return B2RL_ERR_CUDA;
  }
  return B2RL_OK;
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_dqn_loss(const float* q, const float* q_next_target, const float* q_next_online,
                             const int64_t* action, const float* reward, const float* mask, float gamma_n, int32_t B,
                             int32_t A, const float* is_prob, float beta, float eps, float alpha, float* delta_out,
                             float* priority_out, float* loss_out, float* dq_out, const float* beta_dev, void* stream) {
  B2RL_REQUIRE(q && q_next_target && action && reward && mask, "null pointer");
  B2RL_REQUIRE(B > 0 && A > 0, "bad shape");
  int threads = B >= 1024 ? 1024 : ((B + 31) / 32) * 32;
  launch_pdl(dqn_loss_kernel, dim3(1), dim3(threads), 0, (cudaStream_t)stream, q, q_next_target, q_next_online, action, reward, mask,
                                                           gamma_n, B, A, is_prob, beta, eps, alpha, delta_out,
                                                           priority_out, loss_out, dq_out, beta_dev);
  return check_launch("b2rl_dqn_loss");
}

extern "C" int b2rl_c51_loss(const float* log_prob, const float* prob_next_target, const float* prob_next_online,
                             const int64_t* action, const float* reward, const float* mask, float gamma_n, float v_min,
                             float v_max, int32_t B, int32_t A, int32_t N, const float* is_prob, float beta, float eps,
                             float alpha, float* kl_out, float* priority_out, float* loss_out, float* dlogp_out,
                             float* target_prob_out, int32_t* counter, const float* beta_dev, void* stream) {
  B2RL_REQUIRE(log_prob && prob_next_target && action && reward && mask && kl_out && counter, "null pointer");
  B2RL_REQUIRE(B > 0 && A > 0 && N >= 2 && N <= DIST_MAX_N && A <= DIST_MAX_A, "bad shape");
  const double start = (double)v_min, step = ((double)v_max - (double)v_min) / (double)(N - 1);
  const float delta_atom = (float)(((double)v_max - (double)v_min) / (double)(N - 1));   // CategoricalDQN_agent.py:46
  const size_t smem = (size_t)(3 * N + A) * sizeof(float);
  if (int rc = raise_dyn_smem(c51_loss_kernel, smem, "b2rl_c51_loss")) return rc;
  launch_pdl(c51_loss_kernel, dim3(B), dim3(64), smem, (cudaStream_t)stream, log_prob, prob_next_target, prob_next_online, action, reward,
                                                         mask, gamma_n, v_min, v_max, start, step, delta_atom, B, A, N,
                                                         is_prob, beta, eps, alpha, kl_out, priority_out, loss_out,
                                                         dlogp_out, target_prob_out, counter, beta_dev);
  return check_launch("b2rl_c51_loss");
}

extern "C" int b2rl_qr_loss(const float* quantile, const float* quantile_next, const int64_t* action,
                            const float* reward, const float* mask, float gamma_n, float kappa, int32_t B, int32_t A,
                            int32_t N, float* vec_out, float* loss_out, float* dquant_out, float* partial,
                            int32_t* counter, const float* grad_weight, void* stream) {
  B2RL_REQUIRE(quantile && quantile_next && action && reward && mask, "null pointer");
  B2RL_REQUIRE((partial && counter) || dquant_out, "nothing to compute");
  B2RL_REQUIRE(B > 0 && A > 0 && N > 0 && N <= DIST_MAX_N && A <= DIST_MAX_A, "bad shape");
  const size_t smem = (size_t)(3 * N + A) * sizeof(float);
  if (int rc = raise_dyn_smem(qr_loss_kernel, smem, "b2rl_qr_loss")) return rc;
  launch_pdl(qr_loss_kernel, dim3(B), dim3(256), smem, (cudaStream_t)stream, quantile, quantile_next, action, reward, mask, gamma_n, kappa,
                                                         B, A, N, vec_out, loss_out, dquant_out, partial, counter,
                                                         grad_weight);
  return check_launch("b2rl_qr_loss");
}

extern "C" int b2rl_nstep_q_loss_ctas(int32_t N) { return N > 0 ? (N + NSTEP_THREADS - 1) / NSTEP_THREADS : 0; }

extern "C" int b2rl_nstep_q_loss(const float* q, const float* q_boot, const int64_t* action, const float* reward,
                                 const float* mask, float discount, int32_t T, int32_t N, int32_t A, float* ret_out,
                                 float* delta_out, float* loss_out, float* gq_out, float* partial, int32_t* counter,
                                 void* stream) {
  B2RL_REQUIRE(q && q_boot && action && reward && mask && partial && counter, "null pointer");
  B2RL_REQUIRE(T >= 1 && N >= 1 && A >= 1 && A <= NSTEP_MAX_A, "bad shape: needs T >= 1, N >= 1 and 1 <= A <= 32");
  B2RL_REQUIRE((int64_t)T * N <= NSTEP_MAX_ROWS, "T * N must not exceed 2^24 rows");
  launch_pdl(nstep_q_loss_kernel, dim3(b2rl_nstep_q_loss_ctas(N)), dim3(NSTEP_THREADS), 0, (cudaStream_t)stream, q, q_boot,
             action, reward, mask, discount, T, N, A, ret_out, delta_out, loss_out, gq_out, partial, counter);
  return check_launch("b2rl_nstep_q_loss");
}
