// actor.cu -- device-side actor step for the on-policy agents (SURVEY 8f-3): what PPOAgent / A2CAgent do per env step between
// two task.step() calls (PPO_agent.py:45-50) as ONE launch instead of ~25 host / eager operations:
//
//   MeanStdNormalizer.__call__ (normalizer.py:36-51 on baselines' RunningMeanStd): batch mean / population variance of the raw
//       observations, Chan parallel-variance merge into the running moments (float64, count starts at 1e-4), then
//       clip((x - mean) / sqrt(var + eps), -clip, clip) in float64, rounded once to float32 (tensor(), torch_utils.py:20-25)
//   GaussianActorCriticNet.forward (network_heads.py:173-214) with FCBody(tanh) actor / critic bodies and DummyBody phi:
//       mean = tanh(fc_action(actor_body(x))), v = fc_critic(critic_body(x)), std = softplus(std_param),
//       action = mean + std * z (z ~ N(0,1): Philox4x32-10 + Box-Muller, or supplied normals in parity mode),
//       log_pi_a = sum_a Normal(mean, std).log_prob(action), entropy = sum_a Normal.entropy()
//
// One CTA (the batch is num_workers <= 64 rows; the MLPs are 17 -> 64 -> 64 -> 6 | 1): latency, not throughput.  sm_90a only.
#include "common.cuh"

namespace b2rl {

constexpr int ACT_MAX_N = 64, ACT_MAX_D = 128, ACT_MAX_H = 128, ACT_MAX_A = 32;

struct ActorArgs {
  const float* obs;          // raw observations [N][D]
  double* rm_mean; double* rm_var; double* rm_count;      // running moments [D], [D], [1] (device); null: no normalisation
  int update_stats;          // 0: read-only normaliser
  double clip, eps;
  const float* aw1; const float* ab1; const float* aw2; const float* ab2;       // actor body  [H1][D], [H2][H1]
  const float* faw; const float* fab;                                           // fc_action   [A][H2]
  const float* cw1; const float* cb1; const float* cw2; const float* cb2;       // critic body
  const float* fcw; const float* fcb;                                           // fc_critic   [1][H2]
  const float* std_param;    // [A]
  int N, D, H1, H2, A;
  const float* z;            // supplied standard normals [N][A] (parity mode) or null
  uint64_t seed; int64_t* counter;      // Philox stream position (device, advanced by N*A)
  const float* given_action; // null: sample; else evaluate log_prob of these actions
  float* state_out; float* action; float* log_pi_a; float* entropy; float* mean; float* v;
};

__device__ __forceinline__ float softplus_f(float x) {            // torch.nn.functional.softplus (beta 1, threshold 20)
  return x > 20.0f ? x : log1pf(expf(x));
}

// y[n][j] = act(sum_k x[n][k] * W[j][k] + b[j]) for a [N][K] tile in shared memory; (n, j) pairs over the CTA
__device__ __forceinline__ void dense_tile(const float* x, int ldx, const float* __restrict__ W, const float* __restrict__ b,
                                           int N, int K, int J, float* y, int ldy, bool use_tanh) {
  for (int e = threadIdx.x; e < N * J; e += blockDim.x) {
    const int n = e / J, j = e - n * J;
    const float* w = W + (int64_t)j * K;
    const float* xr = x + n * ldx;
    float s = 0.0f;
    for (int k = 0; k < K; ++k) s = fmaf(xr[k], __ldg(w + k), s);
    s += __ldg(b + j);
    y[n * ldy + j] = use_tanh ? tanhf(s) : s;
  }
}

__global__ void __launch_bounds__(256) gaussian_actor_step_kernel(const ActorArgs a) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ float sm[];
  const int N = a.N, D = a.D, H1 = a.H1, H2 = a.H2, A = a.A;
  float* xs = sm;                          // [N][D]  normalised observations
  float* h1 = xs + N * D;                  // [N][Hmax]
  float* h2 = h1 + N * max(H1, H2);        // [N][Hmax]
  float* mu = h2 + N * max(H1, H2);        // [N][A]
  // ---- running moments + normalisation
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    double mean = 0.0, var = 1.0;
    if (a.rm_mean) {
      mean = a.rm_mean[d]; var = a.rm_var[d];
      if (a.update_stats) {
        // batch.mean(axis=0), batch.var(axis=0) of a float32 array: numpy accumulates row after row in float32
        float s = 0.0f;
        for (int n = 0; n < N; ++n) s += a.obs[n * D + d];
        const float mb = s / (float)N;
        float q = 0.0f;
        for (int n = 0; n < N; ++n) { const float t = a.obs[n * D + d] - mb; q += t * t; }
        const float vb = q / (float)N;
        const double na = *a.rm_count, nb = (double)N, nt = na + nb;
        const double delta = (double)mb - mean;
        const double m2 = var * na + (double)vb * nb + delta * delta * na * nb / nt;
        mean = mean + delta * nb / nt;
        var = m2 / nt;
        a.rm_mean[d] = mean; a.rm_var[d] = var;
      }
    }
    for (int n = 0; n < N; ++n) {
      float xn = a.obs[n * D + d];
      if (a.rm_mean) {
        double t = ((double)xn - mean) / sqrt(var + a.eps);
        t = fmin(fmax(t, -a.clip), a.clip);
        xn = (float)t;
      }
      xs[n * D + d] = xn;
      if (a.state_out) a.state_out[n * D + d] = xn;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0 && a.rm_mean && a.update_stats) *a.rm_count += (double)N;
  const int Hm = max(H1, H2);
  // ---- critic: v = fc_critic(tanh(W2 tanh(W1 x)))
  dense_tile(xs, D, a.cw1, a.cb1, N, D, H1, h1, Hm, true);
  __syncthreads();
  dense_tile(h1, Hm, a.cw2, a.cb2, N, H1, H2, h2, Hm, true);
  __syncthreads();
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float s = 0.0f;
    for (int k = 0; k < H2; ++k) s = fmaf(h2[n * Hm + k], __ldg(a.fcw + k), s);
    a.v[n] = s + a.fcb[0];
  }
  __syncthreads();
  // ---- actor: mean = tanh(fc_action(tanh(W2 tanh(W1 x))))
  dense_tile(xs, D, a.aw1, a.ab1, N, D, H1, h1, Hm, true);
  __syncthreads();
  dense_tile(h1, Hm, a.aw2, a.ab2, N, H1, H2, h2, Hm, true);
  __syncthreads();
  dense_tile(h2, Hm, a.faw, a.fab, N, H2, A, mu, A, true);
  __syncthreads();
  // ---- Normal(mean, softplus(std)): sample / log_prob / entropy, summed over the action dimension (one thread per row)
  const int64_t ctr0 = a.counter ? *a.counter : 0;
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float lp = 0.0f, ent = 0.0f;
    for (int j = 0; j < A; ++j) {
      const float m = mu[n * A + j], sd = softplus_f(a.std_param[j]);
      float act;
      if (a.given_action) {
        act = a.given_action[n * A + j];
      } else {
        float zz;
        if (a.z) {
          zz = a.z[n * A + j];
        } else {                                           // Box-Muller on two 24-bit uniforms of one Philox draw
          zz = Philox::normal(a.seed, (uint64_t)(ctr0 + n * A + j), 7);
        }
        act = m + sd * zz;
      }
      const float lsd = logf(sd), t = act - m;
      lp += -(t * t) / (2.0f * sd * sd) - lsd - 0.91893853320467274178f;      // Normal.log_prob: -((x-mu)^2)/(2 var) - log sd - log sqrt(2 pi)
      ent += 0.5f + 0.91893853320467274178f + lsd;                             // Normal.entropy: 0.5 + 0.5 log(2 pi) + log sd
      a.action[n * A + j] = act;
      if (a.mean) a.mean[n * A + j] = m;
    }
    a.log_pi_a[n] = lp;
    a.entropy[n] = ent;
  }
  if (threadIdx.x == 0 && a.counter && !a.given_action && !a.z) *a.counter = ctr0 + (int64_t)N * A;
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_gaussian_actor_step(const float* obs, double* rm_mean, double* rm_var, double* rm_count, int32_t update_stats,
                                        double clip, double eps, const float* aw1, const float* ab1, const float* aw2,
                                        const float* ab2, const float* faw, const float* fab, const float* cw1, const float* cb1,
                                        const float* cw2, const float* cb2, const float* fcw, const float* fcb,
                                        const float* std_param, int32_t N, int32_t D, int32_t H1, int32_t H2, int32_t A,
                                        const float* z, uint64_t seed, int64_t* counter, const float* given_action,
                                        float* state_out, float* action, float* log_pi_a, float* entropy, float* mean, float* v,
                                        void* stream) {
  B2RL_REQUIRE(obs && aw1 && ab1 && aw2 && ab2 && faw && fab && cw1 && cb1 && cw2 && cb2 && fcw && fcb && std_param && action &&
               log_pi_a && entropy && v, "null pointer");
  B2RL_REQUIRE((rm_mean == nullptr) == (rm_var == nullptr) && (rm_mean == nullptr) == (rm_count == nullptr), "all running moments or none");
  B2RL_REQUIRE(N > 0 && N <= ACT_MAX_N && D > 0 && D <= ACT_MAX_D && H1 > 0 && H1 <= ACT_MAX_H && H2 > 0 && H2 <= ACT_MAX_H &&
               A > 0 && A <= ACT_MAX_A, "shape limits: N <= 64, D <= 128, hidden <= 128, A <= 32");
  B2RL_REQUIRE(z || counter || given_action, "need a Philox counter, supplied normals or given actions");
  ActorArgs a;
  a.obs = obs; a.rm_mean = rm_mean; a.rm_var = rm_var; a.rm_count = rm_count; a.update_stats = update_stats; a.clip = clip; a.eps = eps;
  a.aw1 = aw1; a.ab1 = ab1; a.aw2 = aw2; a.ab2 = ab2; a.faw = faw; a.fab = fab;
  a.cw1 = cw1; a.cb1 = cb1; a.cw2 = cw2; a.cb2 = cb2; a.fcw = fcw; a.fcb = fcb; a.std_param = std_param;
  a.N = N; a.D = D; a.H1 = H1; a.H2 = H2; a.A = A; a.z = z; a.seed = seed; a.counter = counter; a.given_action = given_action;
  a.state_out = state_out; a.action = action; a.log_pi_a = log_pi_a; a.entropy = entropy; a.mean = mean; a.v = v;
  const int Hm = H1 > H2 ? H1 : H2;
  const size_t smem = (size_t)(N * D + 2 * N * Hm + N * A) * sizeof(float);
  static size_t attr = 0;
  if (smem > attr) {
    cudaFuncSetAttribute(gaussian_actor_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = smem;
  }
  launch_pdl(gaussian_actor_step_kernel, dim3(1), dim3(256), smem, (cudaStream_t)stream, a);
  return check_launch("b2rl_gaussian_actor_step");
}
