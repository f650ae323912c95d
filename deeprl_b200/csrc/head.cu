// head.cu -- value heads with a handful of outputs (VanillaNet / DuelingNet, network_heads.py:11-37) on CUDA cores:
// the contraction is [B x 512] x [512 x A] with A = number of actions (4..18): far too narrow for a tensor-core tile,
// and in eager form it costs ~12 launches per update (weight / bias casts, GEMM, float cast, dueling combine, and their
// backward counterparts).  Forward: q = phi W_a^T + b_a, or the dueling combine q = v + adv - mean(adv) with
// v = phi W_v^T + b_v.  Backward: dphi = geff W, dW += geff^T phi, db += sum geff, where geff is dq mapped through the
// dueling combine.  phi is the bf16 feature vector of the fused body; weights and gradients are fp32 (master).
// sm_90a only.
#include "common.cuh"

namespace b2rl {

constexpr int HEAD_MAX_OUT = 32;       // A (+1 for the dueling value row)

// one warp per batch row; the row of phi is read once (16-byte loads, 8 features per lane per 256-feature chunk) and
// every output accumulates against it, so all weight loads of a chunk are independent and in flight together
// dot products of one bf16 feature row against every output row of a head (A advantage / action rows + the dueling value
// row): the row of phi is read once (16-byte loads, 8 features per lane per 256-feature chunk) and every output
// accumulates against it, so all weight loads of a chunk are independent and in flight together.  On return every lane
// holds, for n < n_out, the full dot product plus bias in acc[n].
template <int NB>
__device__ __forceinline__ void head_row_dots(const __nv_bfloat16* __restrict__ x, const float* __restrict__ Wa,
                                              const float* __restrict__ ba, const float* __restrict__ Wv,
                                              const float* __restrict__ bv, int K, int A, int lane, float (&acc)[NB]) {
  const int n_out = A + (Wv ? 1 : 0);
#pragma unroll
  for (int n = 0; n < NB; ++n) acc[n] = 0.0f;
  for (int k0 = lane * 8; k0 < K; k0 += 256) {
    const int4 xr = *reinterpret_cast<const int4*>(x + k0);
    const __nv_bfloat162* xp = reinterpret_cast<const __nv_bfloat162*>(&xr);
    float xf[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __bfloat1622float2(xp[j]);
      xf[2 * j] = f.x, xf[2 * j + 1] = f.y;
    }
#pragma unroll
    for (int n = 0; n < NB; ++n) {
      if (n < n_out) {
        const float* w = ((n < A) ? Wa + (int64_t)n * K : Wv) + k0;
        const float4 w0 = __ldg(reinterpret_cast<const float4*>(w)), w1 = __ldg(reinterpret_cast<const float4*>(w) + 1);
        float s = acc[n];
        s = fmaf(xf[0], w0.x, s), s = fmaf(xf[1], w0.y, s), s = fmaf(xf[2], w0.z, s), s = fmaf(xf[3], w0.w, s);
        s = fmaf(xf[4], w1.x, s), s = fmaf(xf[5], w1.y, s), s = fmaf(xf[6], w1.z, s), s = fmaf(xf[7], w1.w, s);
        acc[n] = s;
      }
    }
  }
#pragma unroll
  for (int n = 0; n < NB; ++n) {
    if (n < n_out) {
      const float s = warp_reduce(acc[n], OpAdd());
      acc[n] = s + ((n < A) ? ba[n] : bv[0]);
    }
  }
}

// q values of one row from the dot products: plain head q = acc, dueling q = value + (adv - mean(adv)) (network_heads.py:34-36)
template <int NB>
__device__ __forceinline__ void head_combine(float (&acc)[NB], int A, bool dueling) {
  if (!dueling) return;
  float mean = 0.0f, value = 0.0f;
#pragma unroll
  for (int n = 0; n < NB; ++n) {
    if (n < A) mean += acc[n];
    if (n == A) value = acc[n];
  }
  mean /= (float)A;
#pragma unroll
  for (int n = 0; n < NB; ++n)
    if (n < A) acc[n] = value + (acc[n] - mean);
}

// one warp per batch row
template <int NB>
__global__ void __launch_bounds__(128) head_fwd_kernel(const __nv_bfloat16* __restrict__ phi, const float* __restrict__ Wa,
                                                       const float* __restrict__ ba, const float* __restrict__ Wv,
                                                       const float* __restrict__ bv, int B, int K, int A,
                                                       float* __restrict__ q) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  const int lane = threadIdx.x & 31, b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  float acc[NB];
  head_row_dots<NB>(phi + (int64_t)b * K, Wa, ba, Wv, bv, K, A, lane, acc);
  head_combine<NB>(acc, A, Wv != nullptr);
  if (lane == 0) {
#pragma unroll
    for (int n = 0; n < NB; ++n)
      if (n < A) q[(int64_t)b * A + n] = acc[n];
  }
}

// Actor-critic head (CategoricalActorCriticNet with DummyBody actor / critic bodies, network_heads.py:184-194): the A fc_action
// rows and the fc_critic row of one bf16 feature row, written as out[b] = (logits[0..A-1], v) -- no combine.  With a counter,
// the same warp draws the action as a2c_actor_kernel does (csrc/a2c.cu): the inverse CDF of softmax(logits) on
// Philox::u24(seed, ctr0 + b, AC_PHILOX_STREAM), written as int64 to action_out[b].  The counter advances by B; every CTA reads
// it first and the last CTA to arrive (ticket) writes it, so no CTA can see the advanced value.
constexpr uint64_t AC_PHILOX_STREAM = 13;      // csrc/a2c.cu A2C_PHILOX_STREAM: one categorical stream for both actors

template <int NB>
__global__ void __launch_bounds__(128) ac_head_fwd_kernel(const __nv_bfloat16* __restrict__ phi, const float* __restrict__ Wa,
                                                          const float* __restrict__ ba, const float* __restrict__ Wv,
                                                          const float* __restrict__ bv, int B, int K, int A,
                                                          float* __restrict__ out, uint64_t seed, int64_t* __restrict__ counter,
                                                          int64_t* __restrict__ action_out, int* __restrict__ ticket) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ int64_t s_ctr0;
  const int lane = threadIdx.x & 31, b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (counter) {
    if (threadIdx.x == 0) s_ctr0 = *counter;
    __syncthreads();
  }
  if (b < B) {
    float acc[NB];
    head_row_dots<NB>(phi + (int64_t)b * K, Wa, ba, Wv, bv, K, A, lane, acc);
    if (lane == 0) {
#pragma unroll
      for (int n = 0; n < NB; ++n)
        if (n <= A) out[(int64_t)b * (A + 1) + n] = acc[n];
      if (counter) {
        float mx = acc[0];
#pragma unroll
        for (int j = 1; j < NB; ++j)
          if (j < A) mx = fmaxf(mx, acc[j]);
        float s = 0.0f;
#pragma unroll
        for (int j = 0; j < NB; ++j)
          if (j < A) s += expf(acc[j] - mx);
        const float target = Philox::u24(seed, (uint64_t)(s_ctr0 + b), AC_PHILOX_STREAM) * s;
        int pick = A - 1;                         // (rounding may leave the target above the last partial sum)
        float c = 0.0f;
        bool found = false;
#pragma unroll
        for (int j = 0; j < NB; ++j) {
          if (j < A && !found) {
            c += expf(acc[j] - mx);
            if (target < c) { pick = j; found = true; }
          }
        }
        action_out[b] = pick;
      }
    }
  }
  if (counter) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      if (atomicAdd(ticket, 1) == (int)gridDim.x - 1) {   // every CTA has read the counter
        *counter = s_ctr0 + B;
        *ticket = 0;
      }
    }
  }
}

// grid (K/64, ceil(B/HB_ROWS)); block 256 = 64 columns x 4 row groups of HB_ROWS/4 rows (many small CTAs: the kernel is
// latency-bound, 16 rows per CTA puts 256 CTAs in flight at B = 512)
constexpr int HB_ROWS = 16;

struct HeadBwdShared {
  float geff[HB_ROWS][HEAD_MAX_OUT + 1];       // [row][a], last used column = value gradient (dueling)
  float red[4][64][HEAD_MAX_OUT + 1];
};

// effective output gradients of one row: dq mapped through the dueling combine (identity for a plain head)
__device__ __forceinline__ float head_geff(const float* gr, int n, int A, bool dueling) {
  if (!dueling) return gr[n];
  float sum = 0.0f;
  for (int a = 0; a < A; ++a) sum += gr[a];
  return (n < A) ? gr[n] - sum / (float)A : sum;      // d/d adv_n and d/d value of q = v + adv - mean(adv)
}

// with sh.geff filled for the HB_ROWS rows of this CTA: dphi = geff W (masked by phi > 0 when relu_colsum is given), dW += geff^T
// phi, db += sum geff, relu_colsum += column sums of the masked dphi.  grid (K/64, ceil(B/HB_ROWS)), 256 threads = 64 columns x
// 4 row groups.
__device__ __forceinline__ void head_bwd_body(HeadBwdShared& sh, const __nv_bfloat16* __restrict__ phi,
                                              const float* __restrict__ Wa, const float* __restrict__ Wv, int B, int K, int A,
                                              __nv_bfloat16* __restrict__ gphi, float* __restrict__ gWa,
                                              float* __restrict__ gba, float* __restrict__ gWv, float* __restrict__ gbv,
                                              float* __restrict__ relu_colsum) {
  const int k = blockIdx.x * 64 + (threadIdx.x & 63), rg = threadIdx.x >> 6;
  const int r0 = blockIdx.y * HB_ROWS;
  const int n_out = A + (Wv ? 1 : 0);
  float w[HEAD_MAX_OUT + 1], acc[HEAD_MAX_OUT + 1];
#pragma unroll
  for (int n = 0; n < HEAD_MAX_OUT + 1; ++n) {
    acc[n] = 0.0f;
    w[n] = (n < n_out && k < K) ? ((n < A) ? Wa[(int64_t)n * K + k] : Wv[k]) : 0.0f;
  }
  float colsum = 0.0f;
  if (k < K) {
    float xs[HB_ROWS / 4];
#pragma unroll
    for (int rr = 0; rr < HB_ROWS / 4; ++rr) {         // all loads in flight before the FMAs
      const int r = r0 + rg * (HB_ROWS / 4) + rr;
      xs[rr] = r < B ? __bfloat162float(phi[(int64_t)r * K + k]) : 0.0f;
    }
#pragma unroll
    for (int rr = 0; rr < HB_ROWS / 4; ++rr) {
      const int r = rg * (HB_ROWS / 4) + rr;
      if (r0 + r >= B) break;
      const float x = xs[rr];
      float g = 0.0f;
#pragma unroll
      for (int n = 0; n < HEAD_MAX_OUT + 1; ++n) {
        if (n < n_out) {
          const float ge = sh.geff[r][n];
          g = fmaf(ge, w[n], g);
          acc[n] = fmaf(ge, x, acc[n]);
        }
      }
      if (relu_colsum && !(x > 0.0f)) g = 0.0f;
      const __nv_bfloat16 gb = __float2bfloat16_rn(g);
      colsum += __bfloat162float(gb);                  // the sum of the stored (bf16) values, as the separate pass computes it
      gphi[(int64_t)(r0 + r) * K + k] = gb;
    }
  }
  sh.red[rg][threadIdx.x & 63][HEAD_MAX_OUT] = colsum;     // slot HEAD_MAX_OUT is free: n_out <= HEAD_MAX_OUT
#pragma unroll
  for (int n = 0; n < HEAD_MAX_OUT + 1; ++n)
    if (n < n_out) sh.red[rg][threadIdx.x & 63][n] = acc[n];
  __syncthreads();
  for (int e = threadIdx.x; e < 64 * n_out; e += blockDim.x) {
    const int c = e % 64, n = e / 64;
    const int kk = blockIdx.x * 64 + c;
    if (kk < K) {
      const float s = sh.red[0][c][n] + sh.red[1][c][n] + sh.red[2][c][n] + sh.red[3][c][n];
      atomicAdd((n < A) ? gWa + (int64_t)n * K + kk : gWv + kk, s);
    }
  }
  if (relu_colsum && threadIdx.x < 64) {
    const int kk = blockIdx.x * 64 + threadIdx.x;
    if (kk < K)
      atomicAdd(relu_colsum + kk, sh.red[0][threadIdx.x][HEAD_MAX_OUT] + sh.red[1][threadIdx.x][HEAD_MAX_OUT] +
                                      sh.red[2][threadIdx.x][HEAD_MAX_OUT] + sh.red[3][threadIdx.x][HEAD_MAX_OUT]);
  }
  if (blockIdx.x == 0 && threadIdx.x < n_out) {      // bias gradients: sum of geff over this block's rows
    float s = 0.0f;
    for (int r = 0; r < HB_ROWS; ++r) s += sh.geff[r][threadIdx.x];
    atomicAdd((threadIdx.x < A) ? gba + threadIdx.x : gbv, s);
  }
}

// many small CTAs: the kernel is latency-bound, 16 rows per CTA puts 256 CTAs in flight at B = 512
__global__ void __launch_bounds__(256) head_bwd_kernel(const float* __restrict__ gq, const __nv_bfloat16* __restrict__ phi,
                                                       const float* __restrict__ Wa, const float* __restrict__ Wv, int B,
                                                       int K, int A, __nv_bfloat16* __restrict__ gphi,
                                                       float* __restrict__ gWa, float* __restrict__ gba,
                                                       float* __restrict__ gWv, float* __restrict__ gbv,
                                                       float* __restrict__ relu_colsum, const float* __restrict__ geff_in) {
  // geff_in != NULL: the effective output gradients [B][HEAD_MAX_OUT + 1] were already computed (dqn_head_loss_kernel).
  // relu_colsum != NULL: phi is the output of a ReLU layer (NatureConvBody's fc4): the gradient is masked here (gphi = 0 where
  // phi <= 0) and its column sums -- that layer's bias gradient -- are accumulated into relu_colsum[K] (zeroed by the caller),
  // which replaces the separate mask / bias-gradient pass over gphi.
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ HeadBwdShared sh;
  const int r0 = blockIdx.y * HB_ROWS;
  const int n_out = A + (Wv ? 1 : 0);
  for (int e = threadIdx.x; e < HB_ROWS * n_out; e += blockDim.x) {
    const int r = e / n_out, n = e - r * n_out;
    if (r0 + r >= B) sh.geff[r][n] = 0.0f;
    else sh.geff[r][n] = geff_in ? geff_in[(int64_t)(r0 + r) * (HEAD_MAX_OUT + 1) + n] : head_geff(gq + (int64_t)(r0 + r) * A, n, A, Wv != nullptr);
  }
  __syncthreads();
  head_bwd_body(sh, phi, Wa, Wv, B, K, A, gphi, gWa, gba, gWv, gbv, relu_colsum);
}

// ---------------------------------------------------------------------------------------------------------------
// DQN update, head part, in ONE launch (DQN_agent.py:81-99 compute_loss, :120-127 PER block, :78-79 reduce_loss, and the
// backward of the head): q = head(phi) for the online network on s, q_next = head_target(phi_t) on s' [, argmax from
// head(phi_o) on s' for double-Q], delta / priorities / importance weights / loss exactly as csrc/losses.cu dqn_loss_kernel
// computes them, dL/dq mapped through the dueling combine, then head_bwd_body: dphi (masked by the ReLU of fc4), head weight
// and bias gradients and fc4's bias gradient.  Replaces 2-3 head_fwd launches + dqn_loss + head_bwd (+ a zero fill).
// The 16 rows of a CTA are evaluated by its 8 warps (2 rows each); the K/64 CTAs of a row block repeat those few dot
// products (16 x 3 x (A+1) rows of 512: negligible) instead of exchanging them.
// ---------------------------------------------------------------------------------------------------------------
struct DqnHeadArgs {
  const __nv_bfloat16* phi; const __nv_bfloat16* phi_t; const __nv_bfloat16* phi_o;
  const float* Wa; const float* ba; const float* Wv; const float* bv;
  const float* Wa_t; const float* ba_t; const float* Wv_t; const float* bv_t;
  const int64_t* action; const float* reward; const float* mask;
  float gamma_n;
  int B, K, A;
  const float* is_prob; float beta; const float* beta_dev; float eps, alpha;
  __nv_bfloat16* gphi; float* gWa; float* gba; float* gWv; float* gbv; float* relu_colsum;
  float* q_out; float* delta_out; float* prio_out; float* loss_out; float* loss_partial; int* counter;
};

__device__ __forceinline__ float head_pow_like_torch(float x, float e) {      // csrc/losses.cu pow_like_torch
  if (e == 0.5f) return sqrtf(x);
  if (e == 1.0f) return x;
  if (e == 2.0f) return x * x;
  if (e == -0.5f) return 1.0f / sqrtf(x);
  if (e == -1.0f) return 1.0f / x;
  return powf(x, e);
}
__device__ __forceinline__ float head_per_raw_weight(float prob, int B, float beta) {
  return head_pow_like_torch(__fadd_rn(__fmul_rn(prob, (float)B), 1e-6f), -beta);
}

// Two-launch form of the DQN head (the default): dqn_head_loss_kernel -- ONE WARP PER BATCH ROW (128 CTAs at B = 512) evaluates
// the online head on s, the target head on s' [, the online head on s' for double-Q], the target / loss / PER block, and leaves
// the effective output gradient of the row (through the dueling combine) in geff_out [B][HEAD_MAX_OUT + 1]; head_bwd_kernel then
// reads geff directly.  The single-launch form below repeats the row dot products in every 64-column CTA of the backward grid,
// which puts 4 dependent L2 round trips in front of the backward part of all 256 CTAs.
template <int NB>
__global__ void __launch_bounds__(128) dqn_head_loss_kernel(const DqnHeadArgs a, float* __restrict__ geff_out) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ float s_red[32];
  __shared__ float s_loss[4];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int A = a.A, K = a.K, B = a.B;
  const bool dueling = a.Wv != nullptr;
  const int n_out = A + (dueling ? 1 : 0);
  float beta = a.beta;
  if (a.beta_dev) beta = *a.beta_dev;
  float wmax = 1.0f;
  if (a.is_prob) {
    float m = 0.0f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) m = fmaxf(m, head_per_raw_weight(a.is_prob[b], B, beta));
    wmax = block_reduce(m, OpMax(), 0.0f, s_red);
  }
  const float invB = 1.0f / (float)B;
  const int b = blockIdx.x * 4 + warp;
  float loss_r = 0.0f;
  if (b < B) {
    float q[NB], qt[NB];
    head_row_dots<NB>(a.phi + (int64_t)b * K, a.Wa, a.ba, a.Wv, a.bv, K, A, lane, q);
    head_row_dots<NB>(a.phi_t + (int64_t)b * K, a.Wa_t, a.ba_t, a.Wv_t, a.bv_t, K, A, lane, qt);
    head_combine<NB>(q, A, dueling);
    head_combine<NB>(qt, A, a.Wv_t != nullptr);
    float qnext;
    if (a.phi_o) {                                   // DQN_agent.py:88-90: argmax (first max) of the ONLINE net on s'
      float qo[NB];
      head_row_dots<NB>(a.phi_o + (int64_t)b * K, a.Wa, a.ba, a.Wv, a.bv, K, A, lane, qo);
      head_combine<NB>(qo, A, dueling);
      int best = 0;
      float bv = qo[0];
#pragma unroll
      for (int n = 1; n < NB; ++n)
        if (n < A && qo[n] > bv) { bv = qo[n]; best = n; }
      qnext = 0.0f;
#pragma unroll
      for (int n = 0; n < NB; ++n)
        if (n == best) qnext = qt[n];
    } else {                                         // :92
      qnext = qt[0];
#pragma unroll
      for (int n = 1; n < NB; ++n)
        if (n < A) qnext = fmaxf(qnext, qt[n]);
    }
    const int a_b = (int)a.action[b];
    float q_ab = 0.0f;
#pragma unroll
    for (int n = 0; n < NB; ++n)
      if (n == a_b) q_ab = q[n];
    const float target = __fadd_rn(a.reward[b], __fmul_rn(__fmul_rn(a.gamma_n, qnext), a.mask[b]));   // :95
    const float delta = __fsub_rn(target, q_ab);                                                    // :99
    float w = 1.0f;
    if (a.is_prob) w = __fdiv_rn(head_per_raw_weight(a.is_prob[b], B, beta), wmax);                 // :125-126
    const float wl = __fmul_rn(delta, w);                                                           // :127
    loss_r = __fmul_rn(__fmul_rn(wl, wl), 0.5f);                                                    // :79
    const float g_ab = -wl * w * invB;               // d/dq[a_b] of mean(0.5 * (w * (y - q))^2)
    if (lane == 0) {
      if (a.delta_out) a.delta_out[b] = delta;
      if (a.prio_out && a.is_prob) a.prio_out[b] = head_pow_like_torch(__fadd_rn(fabsf(delta), a.eps), a.alpha);   // :121
      if (a.q_out) {
#pragma unroll
        for (int n = 0; n < NB; ++n)
          if (n < A) a.q_out[(int64_t)b * A + n] = q[n];
      }
    }
    if (lane < n_out) {
      float g;
      if (!dueling) g = (lane == a_b) ? g_ab : 0.0f;
      else g = (lane < A) ? ((lane == a_b ? g_ab : 0.0f) - g_ab / (float)A) : g_ab;
      geff_out[(int64_t)b * (HEAD_MAX_OUT + 1) + lane] = g;
    }
  }
  if (lane == 0) s_loss[warp] = loss_r;
  __syncthreads();
  __shared__ bool s_last;
  if (threadIdx.x == 0) {
    s_last = false;
    if (a.loss_out) {
      a.loss_partial[blockIdx.x] = (s_loss[0] + s_loss[1]) + (s_loss[2] + s_loss[3]);
      __threadfence();
      s_last = atomicAdd(a.counter, 1) == (int)gridDim.x - 1;
    }
  }
  __syncthreads();
  if (s_last) {            // the last CTA adds the partials: every thread loads a few (all in flight), fixed reduction tree
    __threadfence();
    float t = 0.0f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) t += __ldcg(a.loss_partial + i);
    t = block_reduce(t, OpAdd(), 0.0f, s_red);
    if (threadIdx.x == 0) {
      a.loss_out[0] = t * invB;
      *a.counter = 0;
    }
  }
}

template <int NB>
__global__ void __launch_bounds__(256) dqn_head_fused_kernel(const DqnHeadArgs a) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ HeadBwdShared sh;
  __shared__ float s_red[32];
  __shared__ float s_loss[HB_ROWS];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r0 = blockIdx.y * HB_ROWS;
  const int A = a.A, K = a.K, B = a.B;
  const bool dueling = a.Wv != nullptr;
  const int n_out = A + (dueling ? 1 : 0);
  float beta = a.beta;
  if (a.beta_dev) beta = *a.beta_dev;
  float wmax = 1.0f;
  if (a.is_prob) {
    float m = 0.0f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) m = fmaxf(m, head_per_raw_weight(a.is_prob[b], B, beta));
    wmax = block_reduce(m, OpMax(), 0.0f, s_red);
  }
  const float invB = 1.0f / (float)B;
#pragma unroll
  for (int rr = 0; rr < HB_ROWS / 8; ++rr) {
    const int r = warp * (HB_ROWS / 8) + rr, b = r0 + r;
    float loss_r = 0.0f;
    float g_ab = 0.0f;
    int a_b = -1;
    if (b < B) {
      float q[NB], qt[NB];
      head_row_dots<NB>(a.phi + (int64_t)b * K, a.Wa, a.ba, a.Wv, a.bv, K, A, lane, q);
      head_combine<NB>(q, A, dueling);
      head_row_dots<NB>(a.phi_t + (int64_t)b * K, a.Wa_t, a.ba_t, a.Wv_t, a.bv_t, K, A, lane, qt);
      head_combine<NB>(qt, A, a.Wv_t != nullptr);
      float qnext;
      if (a.phi_o) {                                   // DQN_agent.py:88-90: argmax (first max) of the ONLINE net on s'
        float qo[NB];
        head_row_dots<NB>(a.phi_o + (int64_t)b * K, a.Wa, a.ba, a.Wv, a.bv, K, A, lane, qo);
        head_combine<NB>(qo, A, dueling);
        int best = 0;
        float bv = qo[0];
#pragma unroll
        for (int n = 1; n < NB; ++n)
          if (n < A && qo[n] > bv) { bv = qo[n]; best = n; }
        qnext = 0.0f;
#pragma unroll
        for (int n = 0; n < NB; ++n)
          if (n == best) qnext = qt[n];
      } else {                                         // :92
        qnext = qt[0];
#pragma unroll
        for (int n = 1; n < NB; ++n)
          if (n < A) qnext = fmaxf(qnext, qt[n]);
      }
      a_b = (int)a.action[b];
      float q_ab = 0.0f;
#pragma unroll
      for (int n = 0; n < NB; ++n)
        if (n == a_b) q_ab = q[n];
      const float target = __fadd_rn(a.reward[b], __fmul_rn(__fmul_rn(a.gamma_n, qnext), a.mask[b]));   // :95
      const float delta = __fsub_rn(target, q_ab);                                                    // :99
      float w = 1.0f;
      if (a.is_prob) w = __fdiv_rn(head_per_raw_weight(a.is_prob[b], B, beta), wmax);                 // :125-126
      const float wl = __fmul_rn(delta, w);                                                           // :127
      loss_r = __fmul_rn(__fmul_rn(wl, wl), 0.5f);                                                    // :79
      g_ab = -wl * w * invB;                            // d/dq[a_b] of mean(0.5 * (w * (y - q))^2)
      if (blockIdx.x == 0 && lane == 0) {
        if (a.delta_out) a.delta_out[b] = delta;
        if (a.prio_out && a.is_prob) a.prio_out[b] = head_pow_like_torch(__fadd_rn(fabsf(delta), a.eps), a.alpha);   // :121
        if (a.q_out) {
#pragma unroll
          for (int n = 0; n < NB; ++n)
            if (n < A) a.q_out[(int64_t)b * A + n] = q[n];
        }
      }
    }
    // geff of this row: dq has one non-zero entry (the taken action); the dueling combine spreads it
    if (lane < n_out) {
      float g;
      if (!dueling) g = (lane == a_b) ? g_ab : 0.0f;
      else g = (lane < A) ? ((lane == a_b ? g_ab : 0.0f) - g_ab / (float)A) : g_ab;
      sh.geff[r][lane] = (b < B) ? g : 0.0f;
    }
    if (lane == 0) s_loss[r] = loss_r;
  }
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0 && a.loss_out) {
    float t = 0.0f;
    for (int r = 0; r < HB_ROWS; ++r) t += s_loss[r];
    a.loss_partial[blockIdx.y] = t;
    __threadfence();
    s_last = atomicAdd(a.counter, 1) == (int)gridDim.y - 1;
    if (s_last) {                                       // the last row block adds the partials in a fixed order
      __threadfence();
      float tot = 0.0f;
      for (int i = 0; i < (int)gridDim.y; ++i) tot += __ldcg(a.loss_partial + i);
      a.loss_out[0] = tot * invB;
      *a.counter = 0;
    }
  }
  head_bwd_body(sh, a.phi, a.Wa, a.Wv, B, K, A, a.gphi, a.gWa, a.gba, a.gWv, a.gbv, a.relu_colsum);
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_head_fwd(const uint16_t* phi, const float* Wa, const float* ba, const float* Wv, const float* bv,
                             int32_t B, int32_t K, int32_t A, float* q, void* stream) {
  B2RL_REQUIRE(phi && Wa && ba && q && ((Wv == nullptr) == (bv == nullptr)), "null pointer");
  B2RL_REQUIRE(B > 0 && K > 0 && K % 8 == 0 && A > 0 && A < HEAD_MAX_OUT, "need K % 8 == 0 and 0 < A < 32");
  B2RL_REQUIRE(reinterpret_cast<uintptr_t>(phi) % 16 == 0 && (reinterpret_cast<uintptr_t>(Wa) | reinterpret_cast<uintptr_t>(Wv)) % 16 == 0,
               "phi and the weights must be 16-byte aligned");
  const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(phi);
  const int n_out = A + (Wv ? 1 : 0);
  const dim3 grid((B + 3) / 4);
  cudaStream_t st = (cudaStream_t)stream;
  if (n_out <= 8) launch_pdl(head_fwd_kernel<8>, dim3(grid), dim3(128), 0, st, x, Wa, ba, Wv, bv, B, K, A, q);
  else if (n_out <= 19) launch_pdl(head_fwd_kernel<19>, dim3(grid), dim3(128), 0, st, x, Wa, ba, Wv, bv, B, K, A, q);
  else launch_pdl(head_fwd_kernel<HEAD_MAX_OUT>, dim3(grid), dim3(128), 0, st, x, Wa, ba, Wv, bv, B, K, A, q);
  return check_launch("b2rl_head_fwd");
}

static int head_bwd_impl(const float* gq, const uint16_t* phi, const float* Wa, const float* Wv, int32_t B, int32_t K,
                         int32_t A, uint16_t* gphi, float* gWa, float* gba, float* gWv, float* gbv, float* relu_colsum,
                         void* stream, const float* geff_in = nullptr) {
  B2RL_REQUIRE((gq || geff_in) && phi && Wa && gphi && gWa && gba && ((Wv == nullptr) == (gWv == nullptr)) && ((Wv == nullptr) == (gbv == nullptr)),
               "null pointer");
  B2RL_REQUIRE(B > 0 && K > 0 && A > 0 && A < HEAD_MAX_OUT, "need 0 < A < 32");
  dim3 grid((K + 63) / 64, (B + HB_ROWS - 1) / HB_ROWS);
  launch_pdl(head_bwd_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, gq, reinterpret_cast<const __nv_bfloat16*>(phi), Wa, Wv, B, K, A,
                                                          reinterpret_cast<__nv_bfloat16*>(gphi), gWa, gba, gWv, gbv, relu_colsum, geff_in);
  return check_launch("b2rl_head_bwd");
}

extern "C" int b2rl_head_bwd(const float* gq, const uint16_t* phi, const float* Wa, const float* Wv, int32_t B, int32_t K,
                             int32_t A, uint16_t* gphi, float* gWa, float* gba, float* gWv, float* gbv, void* stream) {
  return head_bwd_impl(gq, phi, Wa, Wv, B, K, A, gphi, gWa, gba, gWv, gbv, nullptr, stream);
}

// b2rl_head_bwd for features phi = relu(layer(.)): gphi is masked (0 where phi <= 0) and relu_colsum[K] += column sums of the
// masked gphi (the bias gradient of that layer; zero it first) -- the ReLU backward of the body's last layer in the same pass
extern "C" int b2rl_head_bwd_relu(const float* gq, const uint16_t* phi, const float* Wa, const float* Wv, int32_t B, int32_t K,
                                  int32_t A, uint16_t* gphi, float* gWa, float* gba, float* gWv, float* gbv,
                                  float* relu_colsum, void* stream) {
  B2RL_REQUIRE(relu_colsum, "null relu_colsum");
  return head_bwd_impl(gq, phi, Wa, Wv, B, K, A, gphi, gWa, gba, gWv, gbv, relu_colsum, stream);
}

// Actor-critic head forward (ac_head_fwd_kernel): out [B][A + 1] = (fc_action logits, fc_critic value).  counter != NULL: also
// draw the actions into action_out [B] (int64) from Philox(seed, *counter + b) and advance *counter by B; ticket: int32,
// zero-initialised once (the kernel re-arms it).
extern "C" int b2rl_ac_head_fwd(const uint16_t* phi, const float* Wa, const float* ba, const float* Wv, const float* bv,
                                int32_t B, int32_t K, int32_t A, float* out, uint64_t seed, int64_t* counter,
                                int64_t* action_out, int32_t* ticket, void* stream) {
  B2RL_REQUIRE(phi && Wa && ba && Wv && bv && out, "null pointer");
  B2RL_REQUIRE(!counter || (action_out && ticket), "a draw needs action_out and ticket");
  B2RL_REQUIRE(B > 0 && K > 0 && K % 8 == 0 && A > 0 && A + 1 <= HEAD_MAX_OUT, "need K % 8 == 0 and 0 < A <= 31");
  B2RL_REQUIRE(reinterpret_cast<uintptr_t>(phi) % 16 == 0 && (reinterpret_cast<uintptr_t>(Wa) | reinterpret_cast<uintptr_t>(Wv)) % 16 == 0,
               "phi and the weights must be 16-byte aligned");
  const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(phi);
  const dim3 grid((B + 3) / 4);
  cudaStream_t st = (cudaStream_t)stream;
  if (A + 1 <= 8) launch_pdl(ac_head_fwd_kernel<8>, grid, dim3(128), 0, st, x, Wa, ba, Wv, bv, B, K, A, out, seed, counter, action_out, ticket);
  else if (A + 1 <= 19) launch_pdl(ac_head_fwd_kernel<19>, grid, dim3(128), 0, st, x, Wa, ba, Wv, bv, B, K, A, out, seed, counter, action_out, ticket);
  else launch_pdl(ac_head_fwd_kernel<HEAD_MAX_OUT>, grid, dim3(128), 0, st, x, Wa, ba, Wv, bv, B, K, A, out, seed, counter, action_out, ticket);
  return check_launch("b2rl_ac_head_fwd");
}

// b2rl_head_bwd_relu on effective output gradients already computed: geff [B][HEAD_MAX_OUT + 1], column n < A the gradient of
// Wa's output n, column A that of Wv's (the actor-critic head: dL/dlogit, then dL/dv; b2rl_a2c_rollout_loss writes this layout)
extern "C" int b2rl_head_bwd_geff_relu(const float* geff, const uint16_t* phi, const float* Wa, const float* Wv, int32_t B,
                                       int32_t K, int32_t A, uint16_t* gphi, float* gWa, float* gba, float* gWv, float* gbv,
                                       float* relu_colsum, void* stream) {
  B2RL_REQUIRE(geff && relu_colsum, "null pointer");
  return head_bwd_impl(nullptr, phi, Wa, Wv, B, K, A, gphi, gWa, gba, gWv, gbv, relu_colsum, stream, geff);
}


// DQN head forward (online on s, target on s', optional online on s' for double-Q) + target / loss / PER block + head
// backward in one launch; see dqn_head_fused_kernel.  phi* are bf16 [B][K] outputs of a ReLU layer; *_t = target network's
// head.  relu_colsum [K] (zeroed by the caller) receives fc4's bias gradient.  scratch: one int32 counter (zero-initialised once; the
// kernel re-arms it), 12 bytes of padding, then float [>= ceil(B/16)].  q_out / delta_out / prio_out / loss_out may be NULL.
extern "C" int b2rl_dqn_head_fused(const uint16_t* phi, const uint16_t* phi_t, const uint16_t* phi_o, const float* Wa,
                                   const float* ba, const float* Wv, const float* bv, const float* Wa_t, const float* ba_t,
                                   const float* Wv_t, const float* bv_t, const int64_t* action, const float* reward,
                                   const float* mask, float gamma_n, int32_t B, int32_t K, int32_t A, const float* is_prob,
                                   float beta, const float* beta_dev, float eps, float alpha, uint16_t* gphi, float* gWa,
                                   float* gba, float* gWv, float* gbv, float* relu_colsum, float* q_out, float* delta_out,
                                   float* prio_out, float* loss_out, float* scratch, void* stream) {
  B2RL_REQUIRE(phi && phi_t && Wa && ba && Wa_t && ba_t && action && reward && mask && gphi && gWa && gba && relu_colsum && scratch,
               "null pointer");
  B2RL_REQUIRE(((Wv == nullptr) == (bv == nullptr)) && ((Wv == nullptr) == (gWv == nullptr)) && ((Wv == nullptr) == (gbv == nullptr)) &&
               ((Wv_t == nullptr) == (bv_t == nullptr)) && ((Wv == nullptr) == (Wv_t == nullptr)), "inconsistent dueling arguments");
  B2RL_REQUIRE(B > 0 && K > 0 && K % 8 == 0 && A > 0 && A < HEAD_MAX_OUT, "need K % 8 == 0 and 0 < A < 32");
  B2RL_REQUIRE((reinterpret_cast<uintptr_t>(phi) | reinterpret_cast<uintptr_t>(phi_t) | reinterpret_cast<uintptr_t>(phi_o) |
                reinterpret_cast<uintptr_t>(Wa) | reinterpret_cast<uintptr_t>(Wv) | reinterpret_cast<uintptr_t>(Wa_t) |
                reinterpret_cast<uintptr_t>(Wv_t)) % 16 == 0, "features and weights must be 16-byte aligned");
  DqnHeadArgs a;
  a.phi = reinterpret_cast<const __nv_bfloat16*>(phi); a.phi_t = reinterpret_cast<const __nv_bfloat16*>(phi_t);
  a.phi_o = reinterpret_cast<const __nv_bfloat16*>(phi_o);
  a.Wa = Wa; a.ba = ba; a.Wv = Wv; a.bv = bv; a.Wa_t = Wa_t; a.ba_t = ba_t; a.Wv_t = Wv_t; a.bv_t = bv_t;
  a.action = action; a.reward = reward; a.mask = mask; a.gamma_n = gamma_n; a.B = B; a.K = K; a.A = A;
  a.is_prob = is_prob; a.beta = beta; a.beta_dev = beta_dev; a.eps = eps; a.alpha = alpha;
  a.gphi = reinterpret_cast<__nv_bfloat16*>(gphi); a.gWa = gWa; a.gba = gba; a.gWv = gWv; a.gbv = gbv; a.relu_colsum = relu_colsum;
  a.q_out = q_out; a.delta_out = delta_out; a.prio_out = prio_out; a.loss_out = loss_out;
  const int row_blocks = (B + HB_ROWS - 1) / HB_ROWS;
  a.counter = reinterpret_cast<int*>(scratch); a.loss_partial = scratch + 4;      // counter first: its place does not depend on B
  const dim3 grid((K + 63) / 64, row_blocks);
  const int n_out = A + (Wv ? 1 : 0);
  cudaStream_t st = (cudaStream_t)stream;
  if (n_out <= 8) launch_pdl(dqn_head_fused_kernel<8>, dim3(grid), dim3(256), 0, st, a);
  else if (n_out <= 19) launch_pdl(dqn_head_fused_kernel<19>, dim3(grid), dim3(256), 0, st, a);
  else launch_pdl(dqn_head_fused_kernel<HEAD_MAX_OUT>, dim3(grid), dim3(256), 0, st, a);
  return check_launch("b2rl_dqn_head_fused");
}


// The same update as b2rl_dqn_head_fused in TWO launches (the default of the learner): a row kernel (one warp per batch row:
// heads forward, target / loss / PER block, effective output gradient) and the head backward reading that gradient.
// geff: float scratch [B][33].  scratch: int32 counter + 12 bytes + float [ceil(B/4)], zero-initialised once.
extern "C" int b2rl_dqn_head_two(const uint16_t* phi, const uint16_t* phi_t, const uint16_t* phi_o, const float* Wa,
                                 const float* ba, const float* Wv, const float* bv, const float* Wa_t, const float* ba_t,
                                 const float* Wv_t, const float* bv_t, const int64_t* action, const float* reward,
                                 const float* mask, float gamma_n, int32_t B, int32_t K, int32_t A, const float* is_prob,
                                 float beta, const float* beta_dev, float eps, float alpha, uint16_t* gphi, float* gWa,
                                 float* gba, float* gWv, float* gbv, float* relu_colsum, float* q_out, float* delta_out,
                                 float* prio_out, float* loss_out, float* scratch, float* geff, void* stream) {
  B2RL_REQUIRE(phi && phi_t && Wa && ba && Wa_t && ba_t && action && reward && mask && gphi && gWa && gba && relu_colsum && scratch && geff,
               "null pointer");
  B2RL_REQUIRE(((Wv == nullptr) == (bv == nullptr)) && ((Wv == nullptr) == (gWv == nullptr)) && ((Wv == nullptr) == (gbv == nullptr)) &&
               ((Wv_t == nullptr) == (bv_t == nullptr)) && ((Wv == nullptr) == (Wv_t == nullptr)), "inconsistent dueling arguments");
  B2RL_REQUIRE(B > 0 && K > 0 && K % 8 == 0 && A > 0 && A < HEAD_MAX_OUT, "need K % 8 == 0 and 0 < A < 32");
  B2RL_REQUIRE((reinterpret_cast<uintptr_t>(phi) | reinterpret_cast<uintptr_t>(phi_t) | reinterpret_cast<uintptr_t>(phi_o) |
                reinterpret_cast<uintptr_t>(Wa) | reinterpret_cast<uintptr_t>(Wv) | reinterpret_cast<uintptr_t>(Wa_t) |
                reinterpret_cast<uintptr_t>(Wv_t)) % 16 == 0, "features and weights must be 16-byte aligned");
  DqnHeadArgs a;
  a.phi = reinterpret_cast<const __nv_bfloat16*>(phi); a.phi_t = reinterpret_cast<const __nv_bfloat16*>(phi_t);
  a.phi_o = reinterpret_cast<const __nv_bfloat16*>(phi_o);
  a.Wa = Wa; a.ba = ba; a.Wv = Wv; a.bv = bv; a.Wa_t = Wa_t; a.ba_t = ba_t; a.Wv_t = Wv_t; a.bv_t = bv_t;
  a.action = action; a.reward = reward; a.mask = mask; a.gamma_n = gamma_n; a.B = B; a.K = K; a.A = A;
  a.is_prob = is_prob; a.beta = beta; a.beta_dev = beta_dev; a.eps = eps; a.alpha = alpha;
  a.gphi = reinterpret_cast<__nv_bfloat16*>(gphi); a.gWa = gWa; a.gba = gba; a.gWv = gWv; a.gbv = gbv; a.relu_colsum = relu_colsum;
  a.q_out = q_out; a.delta_out = delta_out; a.prio_out = prio_out; a.loss_out = loss_out;
  a.counter = reinterpret_cast<int*>(scratch); a.loss_partial = scratch + 4;
  const int n_out = A + (Wv ? 1 : 0);
  const dim3 grid((B + 3) / 4);
  cudaStream_t st = (cudaStream_t)stream;
  if (n_out <= 8) launch_pdl(dqn_head_loss_kernel<8>, dim3(grid), dim3(128), 0, st, a, geff);
  else if (n_out <= 19) launch_pdl(dqn_head_loss_kernel<19>, dim3(grid), dim3(128), 0, st, a, geff);
  else launch_pdl(dqn_head_loss_kernel<HEAD_MAX_OUT>, dim3(grid), dim3(128), 0, st, a, geff);
  int rc = check_launch("b2rl_dqn_head_two(loss)");
  if (rc) return rc;
  return head_bwd_impl(nullptr, phi, Wa, Wv, B, K, A, gphi, gWa, gba, gWv, gbv, relu_colsum, stream, geff);
}
