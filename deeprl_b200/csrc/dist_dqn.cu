// dist_dqn.cu -- the distributional DQN agents' step() on the device for the feature launchers (categorical_dqn_feature,
// quantile_regression_dqn_feature): a CategoricalNet (C51) or QuantileNet (QR-DQN) on a two-layer FCBody.
//
//   b2rl_dist_dqn_actor_step     ONE launch per env step: RescaleNormalizer of the raw observations, the forward, the action
//                                values (C51: sum_k softmax z_k, CategoricalDQN_agent.py:23; QR: the mean over the quantiles,
//                                QuantileRegressionDQN_agent.py:19) and a2c.cu dqn_actor_kernel's epsilon-greedy on the same
//                                Philox stream.
//   b2rl_dist_dqn_replay_update  the gradient update on a sampled batch as ONE launch of one block (dist_sequence.inc): the
//                                online and target forwards, the C51 projection + KL or the QR quantile-Huber loss, PER
//                                (C51), the backward, clip_grad_norm_ and RMSprop on DQNAgent._flat's arena.
//
// sm_90a only.
#include "common.cuh"
#include "dist_phases.h"

namespace b2rl {

constexpr int DIST_NT = 512, DIST_ACT_NT = 256;
constexpr uint64_t DIST_PHILOX_STREAM = 17;     // the stream of a2c.cu's epsilon-greedy actor steps

struct DistActorArgs {
  b2rl_a2c::A2cNet net;         // net.A = A K
  int A, K;
  double v_min, v_max;          // C51 support
  const double* obs;            // raw observations [N][D]
  double scale;                 // RescaleNormalizer coefficient
  int N;
  float* action_out;            // [N]
  const float* given;           // these actions are written through, nothing is drawn
  uint64_t seed;
  int64_t* counter;             // Philox position, advanced by 2 N
};

template <int KIND, int GATE>
__global__ void __launch_bounds__(DIST_ACT_NT, 1) dist_actor_kernel(const __grid_constant__ DistActorArgs a, float epsilon) {
  using namespace b2rl_a2c;
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ __align__(16) float dist_smem[];
  A2cShared S;
  const size_t used = a2c_carve<Q, true>(S, dist_smem, a.net.D, a.net.H1, a.net.H2, a.net.A, a.N, 0);
  float* atoms = dist_smem + used;                // [K]
  float* q = atoms + (a.K + 3) / 4 * 4;           // [N][A]
  const int tid = threadIdx.x, NT = DIST_ACT_NT, D = a.net.D, A = a.A, K = a.K;
  const int64_t ctr0 = *a.counter;                // read by every thread before the barriers; thread 0 writes it at the end
  // the forward of a2c.cu's actor kernels (not shared through a helper, as there)
  ph_load_weights<Q, true>(S, a.net, true, tid, NT);
  for (int e = tid; e < a.N * D; e += NT) {
    const int n = e / D, k = e - n * D;
    S.x[n * S.ldx + k] = (float)(a.scale * a.obs[e]);
  }
  if (KIND == b2rl_dist::C51)
    for (int k = tid; k < K; k += NT) atoms[k] = b2rl_dist::dist_atom(k, K, a.v_min, a.v_max);
  __syncthreads();
  ph_fwd1<Q, true, GATE>(S, a.net, true, tid, NT);
  __syncthreads();
  ph_fwd2<Q, true, GATE>(S, a.net, true, tid, NT);
  __syncthreads();
  ph_heads<Q, true>(S, a.net, true, tid, NT);
  __syncthreads();
  for (int e = tid; e < a.N * A; e += NT) {       // per (row, action): the action value
    const int n = e / A, j = e - n * A;
    const float* z = S.z + n * S.lda + j * K;
    float v = 0.0f;
    if (KIND == b2rl_dist::C51) {
      float mx = z[0];
      for (int k = 1; k < K; ++k) mx = fmaxf(mx, z[k]);
      float s = 0.0f;
      for (int k = 0; k < K; ++k) s += expf(z[k] - mx);
      for (int k = 0; k < K; ++k) v += __fmul_rn(__fdiv_rn(expf(z[k] - mx), s), atoms[k]);
    } else {
      for (int k = 0; k < K; ++k) v += z[k];
      v = __fdiv_rn(v, (float)K);
    }
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
    if (Philox::u24(a.seed, c, DIST_PHILOX_STREAM) < epsilon) {
      pick = min((int)(Philox::u24(a.seed, c + 1, DIST_PHILOX_STREAM) * (float)A), A - 1);
    } else {
      const float* qr = q + n * A;
      pick = 0;
      for (int j = 1; j < A; ++j)
        if (qr[j] > qr[pick]) pick = j;
    }
    a.action_out[n] = (float)pick;
  }
  if (tid == 0 && !a.given) *a.counter = ctr0 + 2 * (int64_t)a.N;
}

// one C51 / QR-DQN gradient update on a sampled batch as ONE launch of one block (dist_sequence.inc)
template <int KIND, int GATE>
__global__ void __launch_bounds__(DIST_NT, 1) dist_replay_update_kernel(const __grid_constant__ b2rl_dist::DistArgs g) {
  using namespace b2rl_a2c;
  pdl_sync();
  extern __shared__ __align__(16) float dist_smem[];
  const DqnArgs& d = g.d;
  b2rl_dist::DistShared T;
  b2rl_dist::dist_carve<KIND>(T, dist_smem, d.a.net.D, d.a.net.H1, d.a.net.H2, g.A, g.K, d.a.N, d.double_q);
  DqnShared& DS = T.ds;
  A2cShared& S = DS.s;
  const int NT = DIST_NT;
#define A2C_PHASE(...) { const int tid = threadIdx.x; __VA_ARGS__; } __syncthreads();
#include "dist_sequence.inc"
#undef A2C_PHASE
}

template <int KIND, int GATE> struct DistActorLaunch {
  static void run(const DistActorArgs& a, float epsilon, size_t smem, cudaStream_t st) {
    static size_t attr = 0;
    if (smem > attr) {
      cudaFuncSetAttribute(dist_actor_kernel<KIND, GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      attr = smem;
    }
    launch_pdl(dist_actor_kernel<KIND, GATE>, dim3(1), dim3(DIST_ACT_NT), smem, st, a, epsilon);
  }
};

template <int KIND, int GATE> struct DistUpdateLaunch {
  static void run(const b2rl_dist::DistArgs& g, size_t smem, cudaStream_t st) {
    static size_t attr = 0;
    if (smem > attr) {
      cudaFuncSetAttribute(dist_replay_update_kernel<KIND, GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      attr = smem;
    }
    launch_pdl(dist_replay_update_kernel<KIND, GATE>, dim3(1), dim3(DIST_NT), smem, st, g);
  }
};

// the instantiated configurations: C51 / QR x tanh / ReLU
template <template <int, int> class F, typename... Args>
static void dist_dispatch(int kind, int gate, Args&&... args) {
  using b2rl_a2c::RELU;
  using b2rl_a2c::TANH;
  if (kind == b2rl_dist::C51) {
    if (gate == TANH) F<b2rl_dist::C51, TANH>::run(args...);
    else F<b2rl_dist::C51, RELU>::run(args...);
  } else {
    if (gate == TANH) F<b2rl_dist::QR, TANH>::run(args...);
    else F<b2rl_dist::QR, RELU>::run(args...);
  }
}

static b2rl_a2c::A2cNet dist_net(float* flat, const int32_t* off, int D, int H1, int H2, int A, int K) {
  b2rl_a2c::A2cNet net;
  net.flat = flat;
  const int nt = b2rl_a2c::A2cKind<b2rl_a2c::Q, true>::ntensors;
  for (int i = 0; i < b2rl_a2c::A2C_MAX_TENSORS; ++i) net.off[i] = i < nt ? off[i] : 0;
  net.D = D; net.H1 = H1; net.H2 = H2; net.A = A * K;
  return net;
}

static bool dist_shape_ok(int kind, int D, int H1, int H2, int A, int K) {
  return (kind == b2rl_dist::C51 || kind == b2rl_dist::QR) && D > 0 && D <= 256 && H1 > 0 && H1 <= 128 && H2 > 0 &&
         H2 <= 128 && A >= 2 && A <= 32 && K >= 2 && K <= 256;
}

static size_t dist_bytes(int kind, int D, int H1, int H2, int A, int K, int B, int double_q) {
  b2rl_dist::DistShared probe;
  float* dummy = reinterpret_cast<float*>(uintptr_t(4096));
  return (kind == b2rl_dist::C51 ? b2rl_dist::dist_carve<b2rl_dist::C51>(probe, dummy, D, H1, H2, A, K, B, double_q)
                                 : b2rl_dist::dist_carve<b2rl_dist::QR>(probe, dummy, D, H1, H2, A, K, B, double_q)) *
         sizeof(float);
}

}  // namespace b2rl

using namespace b2rl;

#define DIST_CHECK_NET()                                                                                                     \
  B2RL_REQUIRE(flat && off, "null pointer");                                                                                 \
  B2RL_REQUIRE(kind == 0 || kind == 1, "kind must be 0 (C51) or 1 (QR-DQN)");                                                \
  B2RL_REQUIRE(gate == 0 || gate == 1, "gate must be 0 (tanh) or 1 (relu)");                                                 \
  B2RL_REQUIRE(dist_shape_ok(kind, D, H1, H2, A, K),                                                                         \
               "shape limits: D <= 256, hidden <= 128, 2 <= A <= 32, 2 <= K <= 256")

// dynamic shared memory of the update for these sizes (0: invalid input; the caller checks it against the 227 KB of one SM).
// QR ignores double_q.
extern "C" int64_t b2rl_dist_dqn_smem_bytes(int32_t kind, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, int32_t B,
                                            int32_t double_q) {
  if (!dist_shape_ok(kind, D, H1, H2, A, K) || B <= 0) return 0;
  return (int64_t)dist_bytes(kind, D, H1, H2, A, K, B, double_q != 0);
}

extern "C" int b2rl_dist_dqn_actor_step(int32_t kind, int32_t gate, const double* obs, double obs_scale, const float* flat,
                                        const int32_t* off, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, int32_t N,
                                        double v_min, double v_max, float epsilon, float* action_out, const float* given_action,
                                        uint64_t seed, int64_t* counter, void* stream) {
  DIST_CHECK_NET();
  B2RL_REQUIRE(obs && action_out && counter, "null pointer");
  B2RL_REQUIRE(N > 0 && N <= 1024, "N must be in [1, 1024]");
  B2RL_REQUIRE(kind == 1 || v_max > v_min, "C51 needs v_min < v_max");
  DistActorArgs a;
  a.net = dist_net(const_cast<float*>(flat), off, D, H1, H2, A, K);
  a.A = A; a.K = K; a.v_min = v_min; a.v_max = v_max;
  a.obs = obs; a.scale = obs_scale; a.N = N; a.action_out = action_out; a.given = given_action;
  a.seed = seed; a.counter = counter;
  b2rl_a2c::A2cShared probe;
  const size_t smem = (b2rl_a2c::a2c_carve<b2rl_a2c::Q, true>(probe, reinterpret_cast<float*>(uintptr_t(4096)), D, H1, H2,
                                                              A * K, N, 0) +
                       (size_t)(K + 3) / 4 * 4 + (size_t)N * A) * sizeof(float);
  B2RL_REQUIRE(smem <= 227 * 1024, "network / worker count too large for the shared memory of one SM");
  dist_dispatch<DistActorLaunch>(kind, gate, a, epsilon, smem, (cudaStream_t)stream);
  return check_launch("b2rl_dist_dqn_actor_step");
}

extern "C" int b2rl_dist_dqn_replay_update(int32_t kind, int32_t gate, const void* state, const void* next_state,
                                           int32_t state_f64, double state_scale, const int64_t* action, const float* reward,
                                           const float* mask, int32_t B, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K,
                                           float* flat, const float* target, float* square_avg, float* grad_avg, int64_t* step,
                                           const int32_t* off, float lr, float alpha, float eps, int32_t centered,
                                           float discount_n, int32_t double_q, double v_min, double v_max, float max_norm,
                                           const float* sampling_prob, float beta, float replay_eps, float replay_alpha,
                                           float* priority_out, float* loss_vec_out, float* loss, void* stream) {
  DIST_CHECK_NET();
  B2RL_REQUIRE(state && next_state && action && reward && mask && target && square_avg && step && loss &&
                   (grad_avg || !centered) && (priority_out || !sampling_prob),
               "null pointer");
  B2RL_REQUIRE(B > 0, "bad batch size");
  B2RL_REQUIRE(kind == 0 || !sampling_prob, "QR-DQN with prioritized replay is undefined: its loss is per target quantile");
  B2RL_REQUIRE(kind == 1 || v_max > v_min, "C51 needs v_min < v_max");
  b2rl_dist::DistArgs g = {};
  b2rl_a2c::DqnArgs& d = g.d;
  b2rl_a2c::A2cArgs& a = d.a;
  a.net = dist_net(flat, off, D, H1, H2, A, K);
  a.N = B; a.T = 1;
  a.sq = square_avg; a.ga = grad_avg; a.step = step;
  a.lr = lr; a.alpha = alpha; a.eps = eps; a.centered = centered;
  a.discount = discount_n; a.max_norm = max_norm; a.loss = loss;
  d.state = state; d.next_state = next_state; d.f64 = state_f64 != 0; d.scale = state_scale;
  d.action = action; d.reward = reward; d.mask = mask; d.target = target;
  d.double_q = kind == b2rl_dist::C51 && double_q != 0;
  d.prob = sampling_prob; d.beta = beta; d.per_eps = replay_eps; d.per_alpha = replay_alpha;
  d.priority = priority_out; d.delta = nullptr;
  g.A = A; g.K = K; g.v_min = v_min; g.v_max = v_max; g.loss_vec = loss_vec_out;
  const size_t smem = (size_t)b2rl_dist_dqn_smem_bytes(kind, D, H1, H2, A, K, B, double_q);
  B2RL_REQUIRE(smem > 0 && smem <= 227 * 1024,
               "batch / network too large for the shared memory of one SM (b2rl_dist_dqn_smem_bytes)");
  dist_dispatch<DistUpdateLaunch>(kind, gate, g, smem, (cudaStream_t)stream);
  return check_launch("b2rl_dist_dqn_replay_update");
}
