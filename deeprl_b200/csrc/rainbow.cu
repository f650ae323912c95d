// rainbow.cu -- CategoricalDQNAgent.step() on the device for a RainbowNet on a two-layer FCBody (rainbow_feature): all four
// layers NoisyLinear with their factorised noise drawn in the kernels, or all four nn.Linear; a dueling categorical head.
//
//   b2rl_rainbow_actor_step     ONE launch per env step: a fresh noise vector for the online network, RescaleNormalizer of the raw
//                               observations, the forward on the effective weights, the dueling combination, sum_k softmax z_k per
//                               action and the action.  NoisyLinear: the argmax (epsilon is 0, DQN_agent.py:34-35); nn.Linear:
//                               dist_dqn.cu dist_actor_kernel's epsilon-greedy on the same Philox stream.
//   b2rl_rainbow_replay_update  the gradient update on a sampled batch as ONE launch of one block (rainbow_sequence.inc): fresh
//                               noise for the target and then the online network, the forwards, C51's projection + KL + PER,
//                               the backward through the dueling head and the noisy layers, clip_grad_norm_ and RMSprop on
//                               DQNAgent._flat's arena.
//
// sm_90a only.
#include "common.cuh"
#include "rainbow_phases.h"

namespace b2rl {

constexpr int RB_NT = 512, RB_ACT_NT = 256;
constexpr uint64_t RB_EPS_STREAM = 17;      // the stream of dist_dqn.cu's epsilon-greedy actor steps
constexpr uint64_t RB_NOISE_STREAM = 29;    // NoisyLinear noise: element i of a noise vector is the normal at counter + i

struct RbDraw {
  uint64_t seed;
  __device__ __forceinline__ float operator()(int64_t c) const { return Philox::normal(seed, (uint64_t)c, RB_NOISE_STREAM); }
};

struct RbActorArgs {
  b2rl_a2c::A2cNet eff;         // the effective network: A = (A + 1) K (flat and off unused)
  b2rl_rainbow::RbNet net;
  double v_min, v_max;
  const double* obs;            // raw observations [N][D]
  double scale;                 // RescaleNormalizer coefficient
  int N;
  float* action_out;            // [N]
  const float* given;           // these actions are written through, no uniform is drawn
  uint64_t seed;
  int64_t* counter;             // epsilon-greedy Philox position, advanced by 2 N (nn.Linear layers only)
  const float* given_noise;     // [noise_len]: this noise vector is used, no normal is drawn
  float* noise_out;             // optional [noise_len]: the noise vector used
  float noise_std;
  int64_t* noise_counter;       // noise Philox position, advanced by noise_len (NoisyLinear layers, noise drawn)
};

template <bool NOISY, int GATE>
__global__ void __launch_bounds__(RB_ACT_NT, 1) rainbow_actor_kernel(const __grid_constant__ RbActorArgs a, float epsilon) {
  using namespace b2rl_a2c;
  using namespace b2rl_rainbow;
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ __align__(16) float rb_smem[];
  A2cShared S;
  const int A = a.net.A, K = a.net.K, D = a.net.D, nz = rb_noise_len(a.net);
  const size_t used = a2c_carve<Q, true>(S, rb_smem, D, a.net.H1, a.net.H2, a.eff.A, a.N, 0);
  float* atoms = rb_smem + used;                  // [K]
  float* q = atoms + (K + 3) / 4 * 4;             // [N][A]
  float* f = q + (a.N * A + 3) / 4 * 4;           // [noise_len]
  const int tid = threadIdx.x, NT = RB_ACT_NT;
  const int64_t ctr0 = *a.counter, nctr0 = *a.noise_counter;   // read by every thread before the barriers
  const RbDraw draw = {a.seed};
  ph_rb_noise<NOISY>(a.net, f, a.given_noise, a.noise_out, a.noise_std, draw, nctr0, tid, NT);
  for (int e = tid; e < a.N * D; e += NT) {
    const int n = e / D, k = e - n * D;
    S.x[n * S.ldx + k] = (float)(a.scale * a.obs[e]);
  }
  for (int k = tid; k < K; k += NT) atoms[k] = b2rl_dist::dist_atom(k, K, a.v_min, a.v_max);
  __syncthreads();
  ph_rb_load_weights<NOISY>(S, a.net, f, nullptr, tid, NT);
  __syncthreads();
  ph_fwd1<Q, true, GATE>(S, a.eff, true, tid, NT);
  __syncthreads();
  ph_fwd2<Q, true, GATE>(S, a.eff, true, tid, NT);
  __syncthreads();
  ph_heads<Q, true>(S, a.eff, true, tid, NT);
  __syncthreads();
  ph_rb_duel(S, A, K, 0, a.N, tid, NT);
  __syncthreads();
  for (int e = tid; e < a.N * A; e += NT) {       // per (row, action): sum_k softmax(z)_k atom_k, as dist_actor_kernel
    const int n = e / A, j = e - n * A;
    const float* z = S.z + n * S.lda + j * K;
    float mx = z[0];
    for (int k = 1; k < K; ++k) mx = fmaxf(mx, z[k]);
    float s = 0.0f, v = 0.0f;
    for (int k = 0; k < K; ++k) s += expf(z[k] - mx);
    for (int k = 0; k < K; ++k) v += __fmul_rn(__fdiv_rn(expf(z[k] - mx), s), atoms[k]);
    q[e] = v;
  }
  __syncthreads();
  for (int n = tid; n < a.N; n += NT) {
    if (a.given) {
      a.action_out[n] = a.given[n];
      continue;
    }
    const uint64_t c = (uint64_t)(ctr0 + 2 * (int64_t)n);
    int pick;
    if (!NOISY && Philox::u24(a.seed, c, RB_EPS_STREAM) < epsilon) {
      pick = min((int)(Philox::u24(a.seed, c + 1, RB_EPS_STREAM) * (float)A), A - 1);
    } else {
      const float* qr = q + n * A;
      pick = 0;
      for (int j = 1; j < A; ++j)
        if (qr[j] > qr[pick]) pick = j;
    }
    a.action_out[n] = (float)pick;
  }
  if (tid == 0) {
    if (!NOISY && !a.given) *a.counter = ctr0 + 2 * (int64_t)a.N;
    if (NOISY && !a.given_noise) *a.noise_counter = nctr0 + nz;
  }
}

struct RbUpdateArgs {
  b2rl_rainbow::RbArgs r;
  uint64_t seed;
  int64_t* noise_counter;       // advanced by 2 noise_len (NoisyLinear layers, noise drawn)
};

// one Rainbow gradient update on a sampled batch as ONE launch of one block (rainbow_sequence.inc)
template <bool NOISY, int GATE>
__global__ void __launch_bounds__(RB_NT, 1) rainbow_replay_update_kernel(const __grid_constant__ RbUpdateArgs u) {
  pdl_sync();
  extern __shared__ __align__(16) float rb_smem[];
  const b2rl_rainbow::RbArgs& r = u.r;
  const b2rl_dist::DistArgs& g = r.g;
  const b2rl_a2c::DqnArgs& d = g.d;
  b2rl_rainbow::RbShared RS;
  b2rl_rainbow::rb_carve<NOISY>(RS, rb_smem, r.net, d.a.N);
  b2rl_dist::DistShared& T = RS.t;
  b2rl_a2c::A2cShared& S = T.ds.s;
  b2rl_a2c::A2cShared SO = b2rl_rainbow::rb_online_rows(S, d.double_q);
  const int NT = RB_NT;
  const int64_t ctr0 = *u.noise_counter;          // read by every thread before the barriers; thread 0 writes it at the end
  const RbDraw draw = {u.seed};
#define A2C_PHASE(...) { const int tid = threadIdx.x; __VA_ARGS__; } __syncthreads();
#include "rainbow_sequence.inc"
#undef A2C_PHASE
  if (NOISY && !r.given && threadIdx.x == 0) *u.noise_counter = ctr0 + 2 * (int64_t)b2rl_rainbow::rb_noise_len(r.net);
}

template <bool NOISY, int GATE> struct RbActorLaunch {
  static void run(const RbActorArgs& a, float epsilon, size_t smem, cudaStream_t st) {
    static size_t attr = 0;
    if (smem > attr) {
      cudaFuncSetAttribute(rainbow_actor_kernel<NOISY, GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      attr = smem;
    }
    launch_pdl(rainbow_actor_kernel<NOISY, GATE>, dim3(1), dim3(RB_ACT_NT), smem, st, a, epsilon);
  }
};

template <bool NOISY, int GATE> struct RbUpdateLaunch {
  static void run(const RbUpdateArgs& u, size_t smem, cudaStream_t st) {
    static size_t attr = 0;
    if (smem > attr) {
      cudaFuncSetAttribute(rainbow_replay_update_kernel<NOISY, GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      attr = smem;
    }
    launch_pdl(rainbow_replay_update_kernel<NOISY, GATE>, dim3(1), dim3(RB_NT), smem, st, u);
  }
};

// the instantiated configurations: NoisyLinear / nn.Linear x tanh / ReLU
template <template <bool, int> class F, typename... Args>
static void rb_dispatch(int noisy, int gate, Args&&... args) {
  using b2rl_a2c::RELU;
  using b2rl_a2c::TANH;
  if (noisy) {
    if (gate == TANH) F<true, TANH>::run(args...);
    else F<true, RELU>::run(args...);
  } else {
    if (gate == TANH) F<false, TANH>::run(args...);
    else F<false, RELU>::run(args...);
  }
}

static b2rl_rainbow::RbNet rb_net(float* flat, const int32_t* off, int noisy, int D, int H1, int H2, int A, int K) {
  b2rl_rainbow::RbNet n;
  n.flat = flat;
  for (int i = 0; i < b2rl_rainbow::RB_MAX_TENSORS; ++i) n.off[i] = off && i < (noisy ? 16 : 8) ? off[i] : 0;
  n.D = D; n.H1 = H1; n.H2 = H2; n.A = A; n.K = K;
  return n;
}

static b2rl_a2c::A2cNet rb_eff_net(const b2rl_rainbow::RbNet& n) {
  b2rl_a2c::A2cNet e = {};
  e.D = n.D; e.H1 = n.H1; e.H2 = n.H2; e.A = (n.A + 1) * n.K;
  return e;
}

static bool rb_shape_ok(int noisy, int D, int H1, int H2, int A, int K) {
  return (noisy == 0 || noisy == 1) && D > 0 && D <= 256 && H1 > 0 && H1 <= 128 && H2 > 0 && H2 <= 128 && A >= 2 && A <= 32 &&
         K >= 2 && K <= 256;
}

}  // namespace b2rl

using namespace b2rl;

#define RB_CHECK_NET()                                                                                                       \
  B2RL_REQUIRE(flat && off, "null pointer");                                                                                 \
  B2RL_REQUIRE(noisy == 0 || noisy == 1, "noisy must be 0 (nn.Linear) or 1 (NoisyLinear)");                                  \
  B2RL_REQUIRE(gate == 0 || gate == 1, "gate must be 0 (tanh) or 1 (relu)");                                                 \
  B2RL_REQUIRE(rb_shape_ok(noisy, D, H1, H2, A, K),                                                                          \
               "shape limits: D <= 256, hidden <= 128, 2 <= A <= 32, 2 <= K <= 256");                                        \
  B2RL_REQUIRE(v_max > v_min, "the support needs v_min < v_max")

// dynamic shared memory of the update for these sizes (0: invalid input; the caller checks it against the 227 KB of one SM).
// double_q does not change it.
extern "C" int64_t b2rl_rainbow_smem_bytes(int32_t noisy, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, int32_t B,
                                           int32_t double_q) {
  (void)double_q;
  if (!rb_shape_ok(noisy, D, H1, H2, A, K) || B <= 0) return 0;
  const b2rl_rainbow::RbNet n = rb_net(nullptr, nullptr, noisy, D, H1, H2, A, K);
  b2rl_rainbow::RbShared probe;
  float* dummy = reinterpret_cast<float*>(uintptr_t(4096));
  return (int64_t)((noisy ? b2rl_rainbow::rb_carve<true>(probe, dummy, n, B) : b2rl_rainbow::rb_carve<false>(probe, dummy, n, B)) *
                   sizeof(float));
}

extern "C" int b2rl_rainbow_actor_step(int32_t noisy, int32_t gate, const double* obs, double obs_scale, const float* flat,
                                       const int32_t* off, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, int32_t N,
                                       double v_min, double v_max, float epsilon, float* action_out, const float* given_action,
                                       uint64_t seed, int64_t* counter, float noise_std, const float* given_noise,
                                       float* noise_out, int64_t* noise_counter, void* stream) {
  RB_CHECK_NET();
  B2RL_REQUIRE(obs && action_out && counter && noise_counter, "null pointer");
  B2RL_REQUIRE(N > 0 && N <= 1024, "N must be in [1, 1024]");
  RbActorArgs a;
  a.net = rb_net(const_cast<float*>(flat), off, noisy, D, H1, H2, A, K);
  a.eff = rb_eff_net(a.net);
  a.v_min = v_min; a.v_max = v_max;
  a.obs = obs; a.scale = obs_scale; a.N = N; a.action_out = action_out; a.given = given_action;
  a.seed = seed; a.counter = counter;
  a.given_noise = given_noise; a.noise_out = noise_out; a.noise_std = noise_std; a.noise_counter = noise_counter;
  b2rl_a2c::A2cShared probe;
  const size_t smem = (b2rl_a2c::a2c_carve<b2rl_a2c::Q, true>(probe, reinterpret_cast<float*>(uintptr_t(4096)), D, H1, H2,
                                                              a.eff.A, N, 0) +
                       (size_t)(K + 3) / 4 * 4 + ((size_t)N * A + 3) / 4 * 4 + (size_t)b2rl_rainbow::rb_noise_len(a.net)) *
                      sizeof(float);
  B2RL_REQUIRE(smem <= 227 * 1024, "network / worker count too large for the shared memory of one SM");
  rb_dispatch<RbActorLaunch>(noisy, gate, a, epsilon, smem, (cudaStream_t)stream);
  return check_launch("b2rl_rainbow_actor_step");
}

extern "C" int b2rl_rainbow_replay_update(int32_t noisy, int32_t gate, const void* state, const void* next_state,
                                          int32_t state_f64, double state_scale, const int64_t* action, const float* reward,
                                          const float* mask, int32_t B, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K,
                                          float* flat, const float* target, float* square_avg, float* grad_avg, int64_t* step,
                                          const int32_t* off, float lr, float alpha, float eps, int32_t centered,
                                          float discount_n, int32_t double_q, double v_min, double v_max, float max_norm,
                                          const float* sampling_prob, float beta, float replay_eps, float replay_alpha,
                                          float* priority_out, float* loss_vec_out, float* loss, uint64_t seed, float noise_std,
                                          const float* given_noise, float* noise_out, float* target_noise_out,
                                          int64_t* noise_counter, void* stream) {
  RB_CHECK_NET();
  B2RL_REQUIRE(state && next_state && action && reward && mask && target && square_avg && step && loss && noise_counter &&
                   (grad_avg || !centered) && (priority_out || !sampling_prob),
               "null pointer");
  B2RL_REQUIRE(B > 0, "bad batch size");
  RbUpdateArgs u = {};
  b2rl_rainbow::RbArgs& r = u.r;
  b2rl_dist::DistArgs& g = r.g;
  b2rl_a2c::DqnArgs& d = g.d;
  b2rl_a2c::A2cArgs& a = d.a;
  r.net = rb_net(flat, off, noisy, D, H1, H2, A, K);
  a.net = rb_eff_net(r.net);
  a.N = B; a.T = 1;
  a.sq = square_avg; a.ga = grad_avg; a.step = step;
  a.lr = lr; a.alpha = alpha; a.eps = eps; a.centered = centered;
  a.discount = discount_n; a.max_norm = max_norm; a.loss = loss;
  d.state = state; d.next_state = next_state; d.f64 = state_f64 != 0; d.scale = state_scale;
  d.action = action; d.reward = reward; d.mask = mask; d.target = target;
  d.double_q = double_q != 0;
  d.prob = sampling_prob; d.beta = beta; d.per_eps = replay_eps; d.per_alpha = replay_alpha;
  d.priority = priority_out; d.delta = nullptr;
  g.A = A; g.K = K; g.v_min = v_min; g.v_max = v_max; g.loss_vec = loss_vec_out;
  r.given = given_noise; r.noise_out = noise_out; r.target_noise_out = target_noise_out; r.noise_std = noise_std;
  u.seed = seed; u.noise_counter = noise_counter;
  const size_t smem = (size_t)b2rl_rainbow_smem_bytes(noisy, D, H1, H2, A, K, B, double_q);
  B2RL_REQUIRE(smem > 0 && smem <= 227 * 1024,
               "batch / network too large for the shared memory of one SM (b2rl_rainbow_smem_bytes)");
  rb_dispatch<RbUpdateLaunch>(noisy, gate, u, smem, (cudaStream_t)stream);
  return check_launch("b2rl_rainbow_replay_update");
}
