// onpolicy.cu -- GAE backward recurrence, advantage normalisation, PPO clipped surrogate, A2C objective, and the rollout
// launches of the captured pixel learners (A2C rollout loss, PPO rollout prep and categorical minibatch loss).
// Reference: deep_rl/agent/A2C_agent.py:43-64, deep_rl/agent/PPO_agent.py:51-86.  sm_90a only.
#include "common.cuh"

namespace b2rl {

// mode 0: one thread per env, time loop in the reference's order and association (bit-identical):
//   returns    = r + (gamma*m) * returns
//   td         = r + (gamma*m) * v[t+1] - v[t]
//   advantages = ((advantages*tau)*gamma)*m + td
__global__ void __launch_bounds__(128) gae_seq_kernel(const float* __restrict__ reward, const float* __restrict__ mask,
                                                      const float* __restrict__ value, float discount, float tau, int T,
                                                      int N, int use_gae, float* __restrict__ adv_out,
                                                      float* __restrict__ ret_out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float ret = value[(int64_t)T * N + n];
  float adv = 0.0f;
  float vnext = ret;
  for (int t = T - 1; t >= 0; --t) {
    const int64_t o = (int64_t)t * N + n;
    const float r = reward[o], m = mask[o], v = value[o];
    const float gm = __fmul_rn(discount, m);
    ret = __fadd_rn(r, __fmul_rn(gm, ret));
    if (use_gae) {
      const float td = __fsub_rn(__fadd_rn(r, __fmul_rn(gm, vnext)), v);
      adv = __fadd_rn(__fmul_rn(__fmul_rn(__fmul_rn(adv, tau), discount), m), td);
    } else {
      adv = __fsub_rn(ret, v);
    }
    adv_out[o] = adv;
    ret_out[o] = ret;
    vnext = v;
  }
}

// mode 1: one warp per env, segmented backward scan.  Both recurrences are x_t = a_t * x_{t+1} + b_t.
// Lane l owns the contiguous time chunk [l*C, (l+1)*C); pass 1 composes its chunk into (a, b), a warp
// suffix-scan over lanes gives every lane its carry-in x_{(l+1)*C}, pass 2 replays the chunk with it.
struct Affine { float a, b; };
__device__ __forceinline__ Affine compose(Affine outer, Affine inner) {   // outer(inner(x))
  return Affine{outer.a * inner.a, fmaf(outer.a, inner.b, outer.b)};
}

__global__ void __launch_bounds__(128) gae_scan_kernel(const float* __restrict__ reward, const float* __restrict__ mask,
                                                       const float* __restrict__ value, float discount, float tau,
                                                       int T, int N, int use_gae, float* __restrict__ adv_out,
                                                       float* __restrict__ ret_out) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  const int C = (T + 31) / 32;
  const int t0 = lane * C, t1 = min(T, t0 + C);
  Affine fr{1.0f, 0.0f}, fa{1.0f, 0.0f};                 // composite of the chunk, applied to x_{t1}
  for (int t = t1 - 1; t >= t0; --t) {
    const int64_t o = (int64_t)t * N + n;
    const float r = reward[o], m = mask[o], gm = discount * m;
    const float td = r + gm * value[o + N] - value[o];
    fr = compose(Affine{gm, r}, fr);
    fa = compose(Affine{tau * gm, td}, fa);
  }
  // suffix scan over lanes: carry-in of lane l = composite of lanes l+1..31 applied to the terminal values
  Affine sr = fr, sa = fa;                                // inclusive suffix composite (lanes l..31)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    Affine or_{__shfl_down_sync(0xffffffffu, sr.a, o), __shfl_down_sync(0xffffffffu, sr.b, o)};
    Affine oa_{__shfl_down_sync(0xffffffffu, sa.a, o), __shfl_down_sync(0xffffffffu, sa.b, o)};
    if (lane + o < 32) { sr = compose(sr, or_); sa = compose(sa, oa_); }
  }
  const float vT = value[(int64_t)T * N + n];
  // exclusive: take the inclusive composite of lane+1
  float ea_r = __shfl_down_sync(0xffffffffu, sr.a, 1), eb_r = __shfl_down_sync(0xffffffffu, sr.b, 1);
  float ea_a = __shfl_down_sync(0xffffffffu, sa.a, 1), eb_a = __shfl_down_sync(0xffffffffu, sa.b, 1);
  float ret = (lane == 31) ? vT : fmaf(ea_r, vT, eb_r);
  float adv = (lane == 31) ? 0.0f : eb_a;                 // terminal advantage is 0
  (void)ea_a;
  for (int t = t1 - 1; t >= t0; --t) {
    const int64_t o = (int64_t)t * N + n;
    const float r = reward[o], m = mask[o], gm = discount * m, v = value[o];
    ret = fmaf(gm, ret, r);
    if (use_gae) adv = fmaf(tau * gm, adv, r + gm * value[o + N] - v);
    else adv = ret - v;
    adv_out[o] = adv;
    ret_out[o] = ret;
  }
}

// (adv - mean) / std, unbiased std, no epsilon (PPO_agent.py:66); accumulation in float64, one CTA
__global__ void __launch_bounds__(1024) normalize_adv_kernel(float* __restrict__ adv, int M) {
  __shared__ double red[32];
  double s = 0.0;
  for (int i = threadIdx.x; i < M; i += blockDim.x) s += (double)adv[i];
  const double mean = block_reduce(s, OpAdd(), 0.0, red) / (double)M;
  const float meanf = (float)mean;
  double q = 0.0;
  for (int i = threadIdx.x; i < M; i += blockDim.x) {
    double d = (double)adv[i] - mean;
    q += d * d;
  }
  const float stdf = (float)sqrt(block_reduce(q, OpAdd(), 0.0, red) / (double)(M - 1));
  for (int i = threadIdx.x; i < M; i += blockDim.x) adv[i] = __fdiv_rn(__fsub_rn(adv[i], meanf), stdf);
}

// PPO_agent.py:77-86 for one minibatch, one CTA
__global__ void __launch_bounds__(1024) ppo_loss_kernel(const float* __restrict__ logp, const float* __restrict__ ent,
                                                        const float* __restrict__ v, const float* __restrict__ old_logp,
                                                        const float* __restrict__ adv, const float* __restrict__ ret,
                                                        float clip, float ew, int M, float* __restrict__ out,
                                                        float* __restrict__ dlogp, float* __restrict__ dent,
                                                        float* __restrict__ dv) {
  __shared__ float red[32];
  float s_obj = 0.0f, s_ent = 0.0f, s_v = 0.0f, s_kl = 0.0f;
  const float invM = 1.0f / (float)M;
  for (int i = threadIdx.x; i < M; i += blockDim.x) {
    const float d = __fsub_rn(logp[i], old_logp[i]);
    const float ratio = expf(d);
    const float a = adv[i];
    const float obj = __fmul_rn(ratio, a);
    const float rc = fminf(fmaxf(ratio, 1.0f - clip), 1.0f + clip);
    const float objc = __fmul_rn(rc, a);
    s_obj += fminf(obj, objc);
    s_ent += ent[i];
    const float e = __fsub_rn(ret[i], v[i]);
    s_v += __fmul_rn(e, e);
    s_kl += __fsub_rn(old_logp[i], logp[i]);
    // torch.min picks `obj` when obj <= objc (ties -> first argument gets the gradient in torch.min backward
    // only when strictly smaller... torch splits ties evenly); clamp passes gradient only inside the interval
    float g;
    const bool inside = ratio >= 1.0f - clip && ratio <= 1.0f + clip;
    if (obj < objc) g = a * ratio;
    else if (obj > objc) g = inside ? a * ratio : 0.0f;
    else g = 0.5f * a * ratio + (inside ? 0.5f * a * ratio : 0.0f);
    if (dlogp) dlogp[i] = -g * invM;
    if (dent) dent[i] = -ew * invM;
    if (dv) dv[i] = -e * invM;
  }
  s_obj = block_reduce(s_obj, OpAdd(), 0.0f, red);
  s_ent = block_reduce(s_ent, OpAdd(), 0.0f, red);
  s_v = block_reduce(s_v, OpAdd(), 0.0f, red);
  s_kl = block_reduce(s_kl, OpAdd(), 0.0f, red);
  if (threadIdx.x == 0) {
    out[0] = -(s_obj * invM) - ew * (s_ent * invM);
    out[1] = 0.5f * (s_v * invM);
    out[2] = s_kl * invM;
  }
}

// A2C_agent.py:55-62, one CTA
__global__ void __launch_bounds__(1024) a2c_loss_kernel(const float* __restrict__ logp, const float* __restrict__ ent,
                                                        const float* __restrict__ v, const float* __restrict__ adv,
                                                        const float* __restrict__ ret, float ew, float vw, int M,
                                                        float* __restrict__ out, float* __restrict__ dlogp,
                                                        float* __restrict__ dent, float* __restrict__ dv) {
  __shared__ float red[32];
  float s_p = 0.0f, s_e = 0.0f, s_v = 0.0f;
  const float invM = 1.0f / (float)M;
  for (int i = threadIdx.x; i < M; i += blockDim.x) {
    s_p += __fmul_rn(logp[i], adv[i]);
    s_e += ent[i];
    const float e = __fsub_rn(ret[i], v[i]);
    s_v += __fmul_rn(e, e);
    if (dlogp) dlogp[i] = -adv[i] * invM;
    if (dent) dent[i] = -ew * invM;
    if (dv) dv[i] = -vw * e * invM;
  }
  s_p = block_reduce(s_p, OpAdd(), 0.0f, red);
  s_e = block_reduce(s_e, OpAdd(), 0.0f, red);
  s_v = block_reduce(s_v, OpAdd(), 0.0f, red);
  if (threadIdx.x == 0) {
    const float pl = -(s_p * invM), el = s_e * invM, vl = 0.5f * (s_v * invM);
    out[0] = pl - ew * el + vw * vl;
    out[1] = pl;
    out[2] = vl;
    out[3] = el;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// A2C_agent.py:43-62 for a rollout whose forward is ONE actor-critic head launch over the (T + 1) N rows (b2rl_ac_head_fwd):
// head [(T+1) N][A + 1] (logits, then v; rows t-major, slot T the final states).  One warp per env column: every lane runs
// the column's backward GAE scan in gae_seq_kernel's order (mode 0, the same bits as ops.gae(exact=True)) -- the operands are
// warp-uniform -- and lane j < A then owns logit j of the row: p = softmax(z), lp = log_softmax(z), H = -sum p lp,
//   geff[i][j] = -(adv / R)(1[j = a] - p_j) + (ew / R) p_j (lp_j + H),   geff[i][A] = (vw / R)(v_i - ret_i)
// with R = T N, the gradient of  loss = -mean(lp_a adv) - ew mean(H) + vw 0.5 mean((ret - v)^2)  (adv, ret detached) with
// respect to the head's outputs; the final rows get zero (the reference detaches their values).  geff has the head
// backward's row stride (HEAD_MAX_OUT + 1 = 33, csrc/head.cu).  Each CTA parks its three sums (lp_a adv, H, (ret - v)^2; per
// warp in t order, then in warp order) in partial[3 cta ..] and the last CTA adds them in CTA order: two launches on the same
// inputs give the same loss bits.
constexpr int A2CR_WARPS = 4;
constexpr int A2CR_LD = 33;                    // csrc/head.cu HEAD_MAX_OUT + 1
constexpr int A2CR_MAX_ROWS = 1 << 24;         // (T + 1) N converts to float exactly

__device__ __forceinline__ float a2cr_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(A2CR_WARPS * 32) a2c_rollout_loss_kernel(
    const float* __restrict__ head, const int64_t* __restrict__ action, const float* __restrict__ reward,
    const float* __restrict__ mask, float discount, float tau, int use_gae, float ew, float vw, int T, int N, int A,
    float* __restrict__ adv_out, float* __restrict__ ret_out, float* __restrict__ loss_out, float* __restrict__ geff,
    float* __restrict__ partial, int32_t* __restrict__ counter) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ float s_sum[3][A2CR_WARPS];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * A2CR_WARPS + warp;
  const int ld = A + 1;
  const float R = (float)(T * N);
  float s_pol = 0.0f, s_ent = 0.0f, s_val = 0.0f;
  if (n < N) {
    const int64_t fin = (int64_t)T * N + n;
    if (lane <= A) geff[fin * A2CR_LD + lane] = 0.0f;
    float ret = head[fin * ld + A];
    float adv = 0.0f;
    float vnext = ret;
    for (int t = T - 1; t >= 0; --t) {
      const int64_t i = (int64_t)t * N + n;
      const float r = reward[i], m = mask[i], v = head[i * ld + A];
      const float gm = __fmul_rn(discount, m);
      ret = __fadd_rn(r, __fmul_rn(gm, ret));
      if (use_gae) {
        const float td = __fsub_rn(__fadd_rn(r, __fmul_rn(gm, vnext)), v);
        adv = __fadd_rn(__fmul_rn(__fmul_rn(__fmul_rn(adv, tau), discount), m), td);
      } else {
        adv = __fsub_rn(ret, v);
      }
      vnext = v;
      // the row's softmax: lane j < A holds logit j
      const int a_i = (int)action[i];
      const float z = lane < A ? head[i * ld + lane] : -INFINITY;
      float mx = z;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float e = lane < A ? expf(z - mx) : 0.0f;
      const float s = a2cr_warp_sum(e);
      const float lp = lane < A ? (z - mx) - logf(s) : 0.0f;
      const float p = e / s;
      const float H = -a2cr_warp_sum(p * lp);
      const float lp_a = __shfl_sync(0xffffffffu, lp, a_i & 31);
      if (lane < A) {
        const float pol = (lane == a_i ? 1.0f : 0.0f) - p;
        geff[i * A2CR_LD + lane] = -(adv / R) * pol + (ew / R) * (p * (lp + H));
      } else if (lane == A) {
        geff[i * A2CR_LD + A] = (vw / R) * (v - ret);
      }
      if (lane == 0) {
        if (adv_out) adv_out[i] = adv;
        if (ret_out) ret_out[i] = ret;
      }
      s_pol = __fadd_rn(s_pol, __fmul_rn(lp_a, adv));
      s_ent = __fadd_rn(s_ent, H);
      const float d = __fsub_rn(ret, v);
      s_val = __fadd_rn(s_val, __fmul_rn(d, d));
    }
  }
  if (lane == 0) s_sum[0][warp] = s_pol, s_sum[1][warp] = s_ent, s_sum[2][warp] = s_val;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 0; q < 3; ++q) {
      float c = 0.0f;
      for (int w = 0; w < A2CR_WARPS; ++w) c = __fadd_rn(c, s_sum[q][w]);
      partial[3 * blockIdx.x + q] = c;
    }
    __threadfence();
    is_last = atomicAdd(counter, 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (is_last && threadIdx.x == 0) {              // deterministic final reduction in CTA order
    __threadfence();
    float tot[3] = {0.0f, 0.0f, 0.0f};
    for (int c = 0; c < (int)gridDim.x; ++c)
      for (int q = 0; q < 3; ++q) tot[q] = __fadd_rn(tot[q], __ldcg(partial + 3 * c + q));
    const float pl = -__fdiv_rn(tot[0], R), el = __fdiv_rn(tot[1], R), vl = __fmul_rn(0.5f, __fdiv_rn(tot[2], R));
    if (loss_out) loss_out[0] = __fadd_rn(__fsub_rn(pl, __fmul_rn(ew, el)), __fmul_rn(vw, vl));
    *counter = 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// PPO_agent.py:44-66 (shared_repr) for a rollout whose (logits, v) rows the actor's head launches stored: head
// [(T+1) N][A + 1] (rows t-major, slot T the final states).  One warp per env column: every lane runs the column's backward
// GAE scan in gae_seq_kernel's order (the bits of ops.gae(exact=True)) and the warp takes the log-softmax of each row at its
// action (Categorical.log_prob: the pre-update log pi(a|s) the ratio needs).  adv_out is normalised afterwards by
// b2rl_normalize_advantage.
__global__ void __launch_bounds__(A2CR_WARPS * 32) ppo_rollout_prep_kernel(
    const float* __restrict__ head, const int64_t* __restrict__ action, const float* __restrict__ reward,
    const float* __restrict__ mask, float discount, float tau, int use_gae, int T, int N, int A,
    float* __restrict__ logp_out, float* __restrict__ adv_out, float* __restrict__ ret_out) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = blockIdx.x * A2CR_WARPS + warp;
  if (n >= N) return;
  const int ld = A + 1;
  float ret = head[((int64_t)T * N + n) * ld + A];
  float adv = 0.0f;
  float vnext = ret;
  for (int t = T - 1; t >= 0; --t) {
    const int64_t i = (int64_t)t * N + n;
    const float r = reward[i], m = mask[i], v = head[i * ld + A];
    const float gm = __fmul_rn(discount, m);
    ret = __fadd_rn(r, __fmul_rn(gm, ret));
    if (use_gae) {
      const float td = __fsub_rn(__fadd_rn(r, __fmul_rn(gm, vnext)), v);
      adv = __fadd_rn(__fmul_rn(__fmul_rn(__fmul_rn(adv, tau), discount), m), td);
    } else {
      adv = __fsub_rn(ret, v);
    }
    vnext = v;
    const float z = lane < A ? head[i * ld + lane] : -INFINITY;
    float mx = z;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float s = a2cr_warp_sum(lane < A ? expf(z - mx) : 0.0f);
    const float lp = (z - mx) - logf(s);
    const float lp_a = __shfl_sync(0xffffffffu, lp, (int)action[i] & 31);
    if (lane == 0) {
      logp_out[i] = lp_a;
      adv_out[i] = adv;
      ret_out[i] = ret;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// PPO_agent.py:77-92 (shared_repr) for one minibatch of a categorical actor-critic head: head [B][A + 1] = (logits, v) of the
// minibatch's rows, idx [B] their rows in the rollout, through which action / old_logp / adv (normalised) / ret are read.
// One warp per row, lane j < A owning logit j: p = softmax(z), lp = log_softmax(z), H = -sum p lp, r = exp(lp_a - old_lp_a),
//   policy_loss = -mean(min(r A, clamp(r, 1 - c, 1 + c) A)) - ew mean(H),   value_loss = 0.5 mean((ret - v)^2)
//   geff[b][j] = g_b (1[j = a] - p_j) + (ew / B) p_j (lp_j + H),   geff[b][A] = (v - ret) / B
// with g_b = d policy_loss / d lp_a under ppo_loss_kernel's tie and boundary rules (torch.min splits a tie evenly; clamp
// passes the gradient on the closed interval).  Each CTA parks its four sums (min-objective, H, (ret - v)^2, old_lp - lp_a;
// per warp in row order, then in warp order) in partial[4 cta ..] and the last CTA adds them in CTA order: two launches on
// the same inputs give the same bits of stats = [policy_loss, value_loss, approx_kl].
constexpr int PPOC_WARPS = 8;

__global__ void __launch_bounds__(PPOC_WARPS * 32) ppo_cat_loss_kernel(
    const float* __restrict__ head, const int64_t* __restrict__ idx, const int64_t* __restrict__ action,
    const float* __restrict__ old_logp, const float* __restrict__ adv, const float* __restrict__ ret, float clip, float ew,
    int B, int A, float* __restrict__ geff, float* __restrict__ stats, float* __restrict__ partial,
    int32_t* __restrict__ counter) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ float s_sum[4][PPOC_WARPS];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x * PPOC_WARPS + warp;
  const float invB = 1.0f / (float)B;
  float s_obj = 0.0f, s_ent = 0.0f, s_val = 0.0f, s_kl = 0.0f;
  if (b < B) {
    const int ld = A + 1;
    const int64_t i = idx[b];
    const int a_i = (int)action[i];
    const float z = lane < A ? head[(int64_t)b * ld + lane] : -INFINITY;
    const float v = head[(int64_t)b * ld + A];
    float mx = z;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float e = lane < A ? expf(z - mx) : 0.0f;
    const float s = a2cr_warp_sum(e);
    const float lp = lane < A ? (z - mx) - logf(s) : 0.0f;
    const float p = e / s;
    const float H = -a2cr_warp_sum(p * lp);
    const float lp_a = __shfl_sync(0xffffffffu, lp, a_i & 31);
    const float olp = old_logp[i], A_i = adv[i], R_i = ret[i];
    // ppo_loss_kernel's statements for this row
    const float ratio = expf(__fsub_rn(lp_a, olp));
    const float obj = __fmul_rn(ratio, A_i);
    const float rc = fminf(fmaxf(ratio, 1.0f - clip), 1.0f + clip);
    const float objc = __fmul_rn(rc, A_i);
    const bool inside = ratio >= 1.0f - clip && ratio <= 1.0f + clip;
    float g;
    if (obj < objc) g = A_i * ratio;
    else if (obj > objc) g = inside ? A_i * ratio : 0.0f;
    else g = 0.5f * A_i * ratio + (inside ? 0.5f * A_i * ratio : 0.0f);
    const float dlogp = -g * invB;
    const float d = __fsub_rn(R_i, v);
    if (lane < A) {
      geff[(int64_t)b * A2CR_LD + lane] = dlogp * ((lane == a_i ? 1.0f : 0.0f) - p) + (ew * invB) * (p * (lp + H));
    } else if (lane == A) {
      geff[(int64_t)b * A2CR_LD + A] = -d * invB;
    }
    s_obj = fminf(obj, objc);
    s_ent = H;
    s_val = __fmul_rn(d, d);
    s_kl = __fsub_rn(olp, lp_a);
  }
  if (lane == 0) s_sum[0][warp] = s_obj, s_sum[1][warp] = s_ent, s_sum[2][warp] = s_val, s_sum[3][warp] = s_kl;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 0; q < 4; ++q) {
      float c = 0.0f;
      for (int w = 0; w < PPOC_WARPS; ++w) c = __fadd_rn(c, s_sum[q][w]);
      partial[4 * blockIdx.x + q] = c;
    }
    __threadfence();
    is_last = atomicAdd(counter, 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (is_last && threadIdx.x == 0) {              // deterministic final reduction in CTA order
    __threadfence();
    float tot[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int c = 0; c < (int)gridDim.x; ++c)
      for (int q = 0; q < 4; ++q) tot[q] = __fadd_rn(tot[q], __ldcg(partial + 4 * c + q));
    const float Bf = (float)B;
    stats[0] = __fsub_rn(-__fdiv_rn(tot[0], Bf), __fmul_rn(ew, __fdiv_rn(tot[1], Bf)));
    stats[1] = __fmul_rn(0.5f, __fdiv_rn(tot[2], Bf));
    stats[2] = __fdiv_rn(tot[3], Bf);
    *counter = 0;
  }
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_gae(const float* reward, const float* mask, const float* value, float discount, float tau,
                        int32_t T, int32_t N, int32_t use_gae, int32_t mode, float* adv_out, float* ret_out,
                        void* stream) {
  B2RL_REQUIRE(reward && mask && value && adv_out && ret_out, "null pointer");
  B2RL_REQUIRE(T > 0 && N > 0, "bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  if (mode == 0) {
    gae_seq_kernel<<<(N + 127) / 128, 128, 0, st>>>(reward, mask, value, discount, tau, T, N, use_gae, adv_out, ret_out);
  } else {
    gae_scan_kernel<<<(N + 3) / 4, 128, 0, st>>>(reward, mask, value, discount, tau, T, N, use_gae, adv_out, ret_out);
  }
  return check_launch("b2rl_gae");
}

extern "C" int b2rl_normalize_advantage(float* adv, int32_t M, void* stream) {
  B2RL_REQUIRE(adv && M > 1, "need at least two elements");
  normalize_adv_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(adv, M);
  return check_launch("b2rl_normalize_advantage");
}

static int threads_for(int M) { return M >= 1024 ? 1024 : ((M + 31) / 32) * 32; }

extern "C" int b2rl_ppo_loss(const float* log_pi_a, const float* entropy, const float* v, const float* old_log_pi_a,
                             const float* advantage, const float* ret, float clip, float entropy_weight, int32_t M,
                             float* out, float* dlogp_out, float* dent_out, float* dv_out, void* stream) {
  B2RL_REQUIRE(log_pi_a && entropy && v && old_log_pi_a && advantage && ret && out, "null pointer");
  B2RL_REQUIRE(M > 0, "bad shape");
  ppo_loss_kernel<<<1, threads_for(M), 0, (cudaStream_t)stream>>>(log_pi_a, entropy, v, old_log_pi_a, advantage, ret,
                                                                  clip, entropy_weight, M, out, dlogp_out, dent_out,
                                                                  dv_out);
  return check_launch("b2rl_ppo_loss");
}

extern "C" int b2rl_a2c_loss(const float* log_pi_a, const float* entropy, const float* v, const float* advantage,
                             const float* ret, float entropy_weight, float value_loss_weight, int32_t M, float* out,
                             float* dlogp_out, float* dent_out, float* dv_out, void* stream) {
  B2RL_REQUIRE(log_pi_a && entropy && v && advantage && ret && out, "null pointer");
  B2RL_REQUIRE(M > 0, "bad shape");
  a2c_loss_kernel<<<1, threads_for(M), 0, (cudaStream_t)stream>>>(log_pi_a, entropy, v, advantage, ret, entropy_weight,
                                                                  value_loss_weight, M, out, dlogp_out, dent_out,
                                                                  dv_out);
  return check_launch("b2rl_a2c_loss");
}

extern "C" int b2rl_a2c_rollout_loss_ctas(int32_t N) { return N > 0 ? (N + A2CR_WARPS - 1) / A2CR_WARPS : 0; }

extern "C" int b2rl_a2c_rollout_loss(const float* head, const int64_t* action, const float* reward, const float* mask,
                                     float discount, float gae_tau, int32_t use_gae, float entropy_weight,
                                     float value_loss_weight, int32_t T, int32_t N, int32_t A, float* adv_out, float* ret_out,
                                     float* loss_out, float* geff_out, float* partial, int32_t* counter, void* stream) {
  B2RL_REQUIRE(head && action && reward && mask && geff_out && partial && counter, "null pointer");
  B2RL_REQUIRE(T >= 1 && N >= 1 && A >= 1 && A + 1 <= A2CR_LD - 1, "bad shape: needs T >= 1, N >= 1 and 1 <= A <= 31");
  B2RL_REQUIRE((int64_t)(T + 1) * N <= A2CR_MAX_ROWS, "(T + 1) * N must not exceed 2^24 rows");
  launch_pdl(a2c_rollout_loss_kernel, dim3(b2rl_a2c_rollout_loss_ctas(N)), dim3(A2CR_WARPS * 32), 0, (cudaStream_t)stream,
             head, action, reward, mask, discount, gae_tau, (int)use_gae, entropy_weight, value_loss_weight, (int)T, (int)N,
             (int)A, adv_out, ret_out, loss_out, geff_out, partial, counter);
  return check_launch("b2rl_a2c_rollout_loss");
}

extern "C" int b2rl_ppo_rollout_prep(const float* head, const int64_t* action, const float* reward, const float* mask,
                                     float discount, float gae_tau, int32_t use_gae, int32_t T, int32_t N, int32_t A,
                                     float* logp_out, float* adv_out, float* ret_out, void* stream) {
  B2RL_REQUIRE(head && action && reward && mask && logp_out && adv_out && ret_out, "null pointer");
  B2RL_REQUIRE(T >= 1 && N >= 1 && A >= 1 && A + 1 <= A2CR_LD - 1, "bad shape: needs T >= 1, N >= 1 and 1 <= A <= 31");
  B2RL_REQUIRE((int64_t)(T + 1) * N <= A2CR_MAX_ROWS, "(T + 1) * N must not exceed 2^24 rows");
  launch_pdl(ppo_rollout_prep_kernel, dim3((N + A2CR_WARPS - 1) / A2CR_WARPS), dim3(A2CR_WARPS * 32), 0,
             (cudaStream_t)stream, head, action, reward, mask, discount, gae_tau, (int)use_gae, (int)T, (int)N, (int)A,
             logp_out, adv_out, ret_out);
  return check_launch("b2rl_ppo_rollout_prep");
}

extern "C" int b2rl_ppo_cat_loss_ctas(int32_t B) { return B > 0 ? (B + PPOC_WARPS - 1) / PPOC_WARPS : 0; }

extern "C" int b2rl_ppo_cat_loss(const float* head, const int64_t* idx, const int64_t* action, const float* old_logp,
                                 const float* adv, const float* ret, float clip, float entropy_weight, int32_t B, int32_t A,
                                 float* geff_out, float* stats_out, float* partial, int32_t* counter, void* stream) {
  B2RL_REQUIRE(head && idx && action && old_logp && adv && ret && geff_out && stats_out && partial && counter, "null pointer");
  B2RL_REQUIRE(B >= 1 && B <= A2CR_MAX_ROWS && A >= 1 && A + 1 <= A2CR_LD - 1, "bad shape: needs 1 <= B <= 2^24 and 1 <= A <= 31");
  launch_pdl(ppo_cat_loss_kernel, dim3(b2rl_ppo_cat_loss_ctas(B)), dim3(PPOC_WARPS * 32), 0, (cudaStream_t)stream, head, idx,
             action, old_logp, adv, ret, clip, entropy_weight, (int)B, (int)A, geff_out, stats_out, partial, counter);
  return check_launch("b2rl_ppo_cat_loss");
}
