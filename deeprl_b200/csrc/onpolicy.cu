// onpolicy.cu -- GAE backward recurrence, advantage normalisation, PPO clipped surrogate, A2C objective.
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
