// a2c.cu -- A2CAgent.step() (A2C_agent.py:22-64) on the device for the feature launchers (a2c_feature, a2c_continuous):
//
//   b2rl_a2c_actor_step   ONE launch per env step: RescaleNormalizer of the raw observations (float64 product, rounded once to
//                         float32 like tensor()), the actor's forward (a2c_phases.h) and the action draw -- categorical: inverse
//                         CDF of the softmax on one Philox uniform; Gaussian: mean + softplus(std) z with Box-Muller normals.
//                         The state goes to row t of the rollout arena, the action to row t of the action arena.  No log-prob,
//                         entropy or value: the parameters do not change during a rollout, so the update recomputes them from
//                         the same weights.
//   b2rl_a2c_update       the rest of step() as ONE launch of one block: forward of all (T + 1) N rows, GAE, the objective,
//                         backward, clip_grad_norm_, RMSprop on the FlatOptimizer arena (a2c_sequence.inc).  The network is
//                         5-12 k parameters over 25-100 rows: the eager form is several hundred launches of a few microseconds.
//   b2rl_nstep_dqn_*      NStepDQNAgent.step() (NStepDQN_agent.py:26-67) for a VanillaNet on a two-layer FCBody the same way: an
//                         actor step with epsilon-greedy on Philox uniforms, and one update launch (nstep_sequence.inc) that also
//                         does the rollout's target sync.
//   b2rl_dqn_replay_*     DQNAgent's gradient update (DQN_agent.py:81-134) for a VanillaNet or DuelingNet on a two-layer FCBody:
//                         one launch on the sampled batch (dqn_sequence.inc); its actor step is b2rl_nstep_dqn_actor_step's
//                         dqn_actor_kernel (DuelingNet head, no state row).
//
// sm_90a only.
#include "common.cuh"
#include "a2c_phases.h"

namespace b2rl {

constexpr int A2C_NT = 512, A2C_ACT_NT = 256;
constexpr uint64_t A2C_PHILOX_STREAM = 13;

template <int HEAD, bool SHARED, int GATE>
__global__ void __launch_bounds__(A2C_NT, 1) a2c_update_kernel(const __grid_constant__ b2rl_a2c::A2cArgs a) {
  using namespace b2rl_a2c;
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ __align__(16) float a2c_smem[];
  A2cShared S;
  a2c_carve<HEAD, SHARED>(S, a2c_smem, a.net.D, a.net.H1, a.net.H2, a.net.A, (a.T + 1) * a.N, a.T * a.N);
  const int NT = A2C_NT;
#define A2C_PHASE(...) { const int tid = threadIdx.x; __VA_ARGS__; } __syncthreads();
#include "a2c_sequence.inc"
#undef A2C_PHASE
}

struct A2cActorArgs {
  b2rl_a2c::A2cNet net;
  const double* obs;          // raw observations [N][D]
  double scale;               // RescaleNormalizer coefficient
  int N;
  float* state_out;           // row t of the rollout arena [N][D]
  float* action_out;          // row t of the action arena [N][acols]
  const float* given;         // parity mode: these actions are written through, nothing is drawn
  uint64_t seed;
  int64_t* counter;           // Philox position, advanced by the number of draws
};

template <int HEAD, bool SHARED, int GATE>
__global__ void __launch_bounds__(A2C_ACT_NT, 1) a2c_actor_kernel(const __grid_constant__ A2cActorArgs a) {
  using namespace b2rl_a2c;
  pdl_sync();
  extern __shared__ __align__(16) float a2c_smem[];
  A2cShared S;
  a2c_carve<HEAD, SHARED>(S, a2c_smem, a.net.D, a.net.H1, a.net.H2, a.net.A, a.N, 0);
  const int tid = threadIdx.x, NT = A2C_ACT_NT, D = a.net.D, A = a.net.A;
  const int64_t ctr0 = *a.counter;               // read by every thread before the barriers; thread 0 writes it at the end
  ph_load_weights<HEAD, SHARED>(S, a.net, true, tid, NT);
  for (int e = tid; e < a.N * D; e += NT) {
    const int n = e / D, k = e - n * D;
    const float x = (float)(a.scale * a.obs[e]);
    S.x[n * S.ldx + k] = x;
    a.state_out[e] = x;
  }
  __syncthreads();
  ph_fwd1<HEAD, SHARED, GATE>(S, a.net, true, tid, NT);
  __syncthreads();
  ph_fwd2<HEAD, SHARED, GATE>(S, a.net, true, tid, NT);
  __syncthreads();
  ph_heads<HEAD, SHARED>(S, a.net, true, tid, NT);
  __syncthreads();
  if (HEAD == CAT) {
    for (int n = tid; n < a.N; n += NT) {
      if (a.given) {
        a.action_out[n] = a.given[n];
        continue;
      }
      const float* z = S.z + n * S.lda;
      float mx = z[0];
      for (int j = 1; j < A; ++j) mx = fmaxf(mx, z[j]);
      float s = 0.0f;
      for (int j = 0; j < A; ++j) s += expf(z[j] - mx);
      const float target = Philox::u24(a.seed, (uint64_t)(ctr0 + n), A2C_PHILOX_STREAM) * s;
      int pick = A - 1;                           // (rounding may leave the target above the last partial sum)
      float c = 0.0f;
      for (int j = 0; j < A; ++j) {
        c += expf(z[j] - mx);
        if (target < c) { pick = j; break; }
      }
      a.action_out[n] = (float)pick;
    }
  } else {
    for (int e = tid; e < a.N * A; e += NT) {
      const int n = e / A, j = e - n * A;
      a.action_out[e] = a.given ? a.given[e]
                                : S.z[n * S.lda + j] + S.sdv[j] * Philox::normal(a.seed, (uint64_t)(ctr0 + e), A2C_PHILOX_STREAM);
    }
  }
  if (tid == 0 && !a.given) *a.counter = ctr0 + (int64_t)a.N * (HEAD == CAT ? 1 : A);
}

// ------------------------------------------------------------------------------------------------ n-step Q (NStepDQN_agent.py)
constexpr uint64_t NSTEP_PHILOX_STREAM = 17;

template <int GATE>
__global__ void __launch_bounds__(A2C_NT, 1) nstep_dqn_update_kernel(const __grid_constant__ b2rl_a2c::NStepArgs q) {
  using namespace b2rl_a2c;
  pdl_sync();
  extern __shared__ __align__(16) float a2c_smem[];
  const A2cArgs& a = q.a;
  A2cShared S;
  a2c_carve<Q, true>(S, a2c_smem, a.net.D, a.net.H1, a.net.H2, a.net.A, (a.T + 1) * a.N, a.T * a.N);
  const int NT = A2C_NT;
#define A2C_PHASE(...) { const int tid = threadIdx.x; __VA_ARGS__; } __syncthreads();
#include "nstep_sequence.inc"
#undef A2C_PHASE
}

// epsilon-greedy on the actor step's q (torch_utils.py:51-58 with the device's Philox stream): per row two uniforms, the dice
// u0 < epsilon and the random action min(floor(u1 A), A - 1); otherwise the first index of the maximum, as np.argmax
template <int GATE>
__global__ void __launch_bounds__(A2C_ACT_NT, 1) nstep_dqn_actor_kernel(const __grid_constant__ A2cActorArgs a, float epsilon) {
  using namespace b2rl_a2c;
  pdl_sync();
  extern __shared__ __align__(16) float a2c_smem[];
  A2cShared S;
  a2c_carve<Q, true>(S, a2c_smem, a.net.D, a.net.H1, a.net.H2, a.net.A, a.N, 0);
  const int tid = threadIdx.x, NT = A2C_ACT_NT, D = a.net.D, A = a.net.A;
  const int64_t ctr0 = *a.counter;
  // the forward of a2c_actor_kernel (not shared through a helper: that changes the A2C kernels' instruction schedule)
  ph_load_weights<Q, true>(S, a.net, true, tid, NT);
  for (int e = tid; e < a.N * D; e += NT) {
    const int n = e / D, k = e - n * D;
    const float x = (float)(a.scale * a.obs[e]);
    S.x[n * S.ldx + k] = x;
    a.state_out[e] = x;
  }
  __syncthreads();
  ph_fwd1<Q, true, GATE>(S, a.net, true, tid, NT);
  __syncthreads();
  ph_fwd2<Q, true, GATE>(S, a.net, true, tid, NT);
  __syncthreads();
  ph_heads<Q, true>(S, a.net, true, tid, NT);
  __syncthreads();
  for (int n = tid; n < a.N; n += NT) {
    if (a.given) {
      a.action_out[n] = a.given[n];
      continue;
    }
    const uint64_t c = (uint64_t)(ctr0 + 2 * (int64_t)n);
    int pick;
    if (Philox::u24(a.seed, c, NSTEP_PHILOX_STREAM) < epsilon) {
      pick = min((int)(Philox::u24(a.seed, c + 1, NSTEP_PHILOX_STREAM) * (float)A), A - 1);
    } else {
      const float* z = S.z + n * S.lda;
      pick = 0;
      for (int j = 1; j < A; ++j)
        if (z[j] > z[pick]) pick = j;
    }
    a.action_out[n] = (float)pick;
  }
  if (tid == 0 && !a.given) *a.counter = ctr0 + 2 * (int64_t)a.N;
}

// ------------------------------------------------------------------------------------------------ replay Q (DQN_agent.py)
// the actor step of the replay DQN agent: the forward of nstep_dqn_actor_kernel for a VanillaNet (HEAD = Q) or a DuelingNet
// (HEAD = DUEL, which also needs fc_value and the q = v + (adv - mean(adv)) phase) and the same epsilon-greedy on the same
// Philox stream; the state row is optional (the replay agent keeps no rollout arena).  A kernel of its own, so that the n-step
// instantiations above keep their code.
template <int HEAD, int GATE>
__global__ void __launch_bounds__(A2C_ACT_NT, 1) dqn_actor_kernel(const __grid_constant__ A2cActorArgs a, float epsilon) {
  using namespace b2rl_a2c;
  pdl_sync();
  extern __shared__ __align__(16) float a2c_smem[];
  A2cShared S;
  a2c_carve<HEAD, true>(S, a2c_smem, a.net.D, a.net.H1, a.net.H2, a.net.A, a.N, 0);
  const int tid = threadIdx.x, NT = A2C_ACT_NT, D = a.net.D, A = a.net.A;
  const int64_t ctr0 = *a.counter;
  constexpr bool actor_only = HEAD == Q;
  ph_load_weights<HEAD, true>(S, a.net, actor_only, tid, NT);
  for (int e = tid; e < a.N * D; e += NT) {
    const int n = e / D, k = e - n * D;
    const float x = (float)(a.scale * a.obs[e]);
    S.x[n * S.ldx + k] = x;
    if (a.state_out) a.state_out[e] = x;
  }
  __syncthreads();
  ph_fwd1<HEAD, true, GATE>(S, a.net, actor_only, tid, NT);
  __syncthreads();
  ph_fwd2<HEAD, true, GATE>(S, a.net, actor_only, tid, NT);
  __syncthreads();
  ph_heads<HEAD, true>(S, a.net, actor_only, tid, NT);
  __syncthreads();
  if (HEAD == DUEL) {
    ph_duel_q(S, a.N, A, tid, NT);
    __syncthreads();
  }
  for (int n = tid; n < a.N; n += NT) {
    if (a.given) {
      a.action_out[n] = a.given[n];
      continue;
    }
    const uint64_t c = (uint64_t)(ctr0 + 2 * (int64_t)n);
    int pick;
    if (Philox::u24(a.seed, c, NSTEP_PHILOX_STREAM) < epsilon) {
      pick = min((int)(Philox::u24(a.seed, c + 1, NSTEP_PHILOX_STREAM) * (float)A), A - 1);
    } else {
      const float* z = S.z + n * S.lda;
      pick = 0;
      for (int j = 1; j < A; ++j)
        if (z[j] > z[pick]) pick = j;
    }
    a.action_out[n] = (float)pick;
  }
  if (tid == 0 && !a.given) *a.counter = ctr0 + 2 * (int64_t)a.N;
}

// DQNAgent's update for one sampled batch as ONE launch of one block (dqn_sequence.inc)
template <int HEAD, int GATE>
__global__ void __launch_bounds__(A2C_NT, 1) dqn_replay_update_kernel(const __grid_constant__ b2rl_a2c::DqnArgs d) {
  using namespace b2rl_a2c;
  pdl_sync();
  extern __shared__ __align__(16) float a2c_smem[];
  DqnShared DS;
  dqn_carve<HEAD>(DS, a2c_smem, d.a.net.D, d.a.net.H1, d.a.net.H2, d.a.net.A, d.a.N, d.double_q);
  A2cShared& S = DS.s;
  const int NT = A2C_NT;
#define A2C_PHASE(...) { const int tid = threadIdx.x; __VA_ARGS__; } __syncthreads();
#include "dqn_sequence.inc"
#undef A2C_PHASE
}

template <int HEAD, int GATE> struct DqnActorLaunch {
  static void run(const A2cActorArgs& a, float epsilon, size_t smem, cudaStream_t st) {
    static size_t attr = 0;
    if (smem > attr) {
      cudaFuncSetAttribute(dqn_actor_kernel<HEAD, GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      attr = smem;
    }
    launch_pdl(dqn_actor_kernel<HEAD, GATE>, dim3(1), dim3(A2C_ACT_NT), smem, st, a, epsilon);
  }
};

template <int HEAD, int GATE> struct DqnUpdateLaunch {
  static void run(const b2rl_a2c::DqnArgs& d, size_t smem, cudaStream_t st) {
    static size_t attr = 0;
    if (smem > attr) {
      cudaFuncSetAttribute(dqn_replay_update_kernel<HEAD, GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      attr = smem;
    }
    launch_pdl(dqn_replay_update_kernel<HEAD, GATE>, dim3(1), dim3(A2C_NT), smem, st, d);
  }
};

// the instantiated replay Q configurations: VanillaNet / DuelingNet (head 0 / 1) x tanh / ReLU
template <template <int, int> class F, typename... Args>
static void dqn_dispatch(int head, int gate, Args&&... args) {
  using namespace b2rl_a2c;
  if (head == 0) {
    if (gate == TANH) F<Q, TANH>::run(args...);
    else F<Q, RELU>::run(args...);
  } else {
    if (gate == TANH) F<DUEL, TANH>::run(args...);
    else F<DUEL, RELU>::run(args...);
  }
}

template <int GATE>
static void nstep_update_launch(const b2rl_a2c::NStepArgs& q, size_t smem, cudaStream_t st) {
  static size_t attr = 0;
  if (smem > attr) {
    cudaFuncSetAttribute(nstep_dqn_update_kernel<GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = smem;
  }
  launch_pdl(nstep_dqn_update_kernel<GATE>, dim3(1), dim3(A2C_NT), smem, st, q);
}

template <int GATE>
static void nstep_actor_launch(const A2cActorArgs& a, float epsilon, size_t smem, cudaStream_t st) {
  static size_t attr = 0;
  if (smem > attr) {
    cudaFuncSetAttribute(nstep_dqn_actor_kernel<GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = smem;
  }
  launch_pdl(nstep_dqn_actor_kernel<GATE>, dim3(1), dim3(A2C_ACT_NT), smem, st, a, epsilon);
}

// the instantiated configurations: (CAT, shared trunk) and (GAUSS, separate trunks), each with a tanh or ReLU gate
template <template <int, bool, int> class F, typename... Args>
static bool a2c_dispatch(int head, int shared, int gate, Args&&... args) {
  using namespace b2rl_a2c;
  if (head == CAT && shared && gate == TANH) return F<CAT, true, TANH>::run(args...), true;
  if (head == CAT && shared && gate == RELU) return F<CAT, true, RELU>::run(args...), true;
  if (head == GAUSS && !shared && gate == TANH) return F<GAUSS, false, TANH>::run(args...), true;
  if (head == GAUSS && !shared && gate == RELU) return F<GAUSS, false, RELU>::run(args...), true;
  return false;
}

template <int HEAD, bool SHARED, int GATE> struct UpdateLaunch {
  static void run(const b2rl_a2c::A2cArgs& a, size_t smem, cudaStream_t st) {
    static size_t attr = 0;
    if (smem > attr) {
      cudaFuncSetAttribute(a2c_update_kernel<HEAD, SHARED, GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      attr = smem;
    }
    launch_pdl(a2c_update_kernel<HEAD, SHARED, GATE>, dim3(1), dim3(A2C_NT), smem, st, a);
  }
};

template <int HEAD, bool SHARED, int GATE> struct ActorLaunch {
  static void run(const A2cActorArgs& a, size_t smem, cudaStream_t st) {
    static size_t attr = 0;
    if (smem > attr) {
      cudaFuncSetAttribute(a2c_actor_kernel<HEAD, SHARED, GATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      attr = smem;
    }
    launch_pdl(a2c_actor_kernel<HEAD, SHARED, GATE>, dim3(1), dim3(A2C_ACT_NT), smem, st, a);
  }
};

static size_t a2c_bytes(int head, int shared, int D, int H1, int H2, int A, int R, int M) {
  using namespace b2rl_a2c;
  A2cShared probe;
  float* dummy = reinterpret_cast<float*>(uintptr_t(4096));
  if (head == CAT && shared) return a2c_carve<CAT, true>(probe, dummy, D, H1, H2, A, R, M) * sizeof(float);
  if (head == GAUSS && !shared) return a2c_carve<GAUSS, false>(probe, dummy, D, H1, H2, A, R, M) * sizeof(float);
  return 0;
}

}  // namespace b2rl

using namespace b2rl;

#define A2C_CHECK_NET()                                                                                                      \
  B2RL_REQUIRE(flat && off, "null pointer");                                                                                 \
  B2RL_REQUIRE((head == 0 && shared == 1) || (head == 1 && shared == 0),                                                     \
               "instantiated: categorical head on a shared trunk, Gaussian head on separate trunks");                        \
  B2RL_REQUIRE(gate == 0 || gate == 1, "gate must be 0 (tanh) or 1 (relu)");                                                 \
  B2RL_REQUIRE(D > 0 && D <= 256 && H1 > 0 && H1 <= 128 && H2 > 0 && H2 <= 128 && A > 0 && A <= 32,                          \
               "shape limits: D <= 256, hidden <= 128, A <= 32");                                                            \
  B2RL_REQUIRE(head == 1 || A >= 2, "a categorical head needs at least two actions")

static b2rl_a2c::A2cNet a2c_net(float* flat, const int32_t* off, int head, int shared, int D, int H1, int H2, int A) {
  b2rl_a2c::A2cNet net;
  net.flat = flat;
  const int nt = head == b2rl_a2c::Q ? b2rl_a2c::A2cKind<b2rl_a2c::Q, true>::ntensors : 4 * (shared ? 1 : 2) + 4 + (head == 1 ? 1 : 0);
  for (int i = 0; i < b2rl_a2c::A2C_MAX_TENSORS; ++i) net.off[i] = i < nt ? off[i] : 0;
  net.D = D; net.H1 = H1; net.H2 = H2; net.A = A;
  return net;
}

// dynamic shared memory of the update kernel for these sizes (the caller checks it against the 227 KB of one SM)
extern "C" int64_t b2rl_a2c_smem_bytes(int32_t head, int32_t shared, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t N,
                                       int32_t T) {
  if (D <= 0 || H1 <= 0 || H2 <= 0 || A <= 0 || N <= 0 || T <= 0) return 0;
  return (int64_t)a2c_bytes(head, shared, D, H1, H2, A, (T + 1) * N, T * N);
}

extern "C" int b2rl_a2c_actor_step(int32_t head, int32_t shared, int32_t gate, const double* obs, double obs_scale,
                                   const float* flat, const int32_t* off, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t N,
                                   float* state_out, float* action_out, const float* given_action, uint64_t seed,
                                   int64_t* counter, void* stream) {
  A2C_CHECK_NET();
  B2RL_REQUIRE(obs && state_out && action_out && counter, "null pointer");
  B2RL_REQUIRE(N > 0 && N <= 1024, "N must be in [1, 1024]");
  A2cActorArgs a;
  a.net = a2c_net(const_cast<float*>(flat), off, head, shared, D, H1, H2, A);
  a.obs = obs; a.scale = obs_scale; a.N = N; a.state_out = state_out; a.action_out = action_out; a.given = given_action;
  a.seed = seed; a.counter = counter;
  const size_t smem = a2c_bytes(head, shared, D, H1, H2, A, N, 0);
  B2RL_REQUIRE(smem <= 227 * 1024, "network / worker count too large for the shared memory of one SM");
  a2c_dispatch<ActorLaunch>(head, shared, gate, a, smem, (cudaStream_t)stream);
  return check_launch("b2rl_a2c_actor_step");
}

extern "C" int b2rl_a2c_update(int32_t head, int32_t shared, int32_t gate, const float* states, const float* actions,
                               const float* reward, const float* mask, int32_t T, int32_t N, int32_t D, int32_t H1, int32_t H2,
                               int32_t A, float* flat, float* square_avg, float* grad_avg, int64_t* step, const int32_t* off,
                               float lr, float alpha, float eps, int32_t centered, float discount, float tau, int32_t use_gae,
                               float entropy_weight, float value_loss_weight, float max_norm, float* loss, void* stream) {
  A2C_CHECK_NET();
  B2RL_REQUIRE(states && actions && reward && mask && square_avg && step && loss && (grad_avg || !centered), "null pointer");
  B2RL_REQUIRE(T > 0 && N > 0, "bad T / N");
  b2rl_a2c::A2cArgs a;
  a.net = a2c_net(flat, off, head, shared, D, H1, H2, A);
  a.state = states; a.action = actions; a.reward = reward; a.mask = mask; a.T = T; a.N = N;
  a.sq = square_avg; a.ga = grad_avg; a.step = step;
  a.lr = lr; a.alpha = alpha; a.eps = eps; a.centered = centered;
  a.discount = discount; a.tau = tau; a.use_gae = use_gae;
  a.ent_w = entropy_weight; a.vw = value_loss_weight; a.max_norm = max_norm; a.loss = loss;
  const size_t smem = (size_t)b2rl_a2c_smem_bytes(head, shared, D, H1, H2, A, N, T);
  B2RL_REQUIRE(smem > 0 && smem <= 227 * 1024, "rollout / network too large for the shared memory of one SM (b2rl_a2c_smem_bytes)");
  a2c_dispatch<UpdateLaunch>(head, shared, gate, a, smem, (cudaStream_t)stream);
  return check_launch("b2rl_a2c_update");
}

// ------------------------------------------------------------------------------------------------ n-step Q entry points
#define NSTEP_CHECK_NET()                                                                                                    \
  B2RL_REQUIRE(flat && off, "null pointer");                                                                                 \
  B2RL_REQUIRE(gate == 0 || gate == 1, "gate must be 0 (tanh) or 1 (relu)");                                                 \
  B2RL_REQUIRE(D > 0 && D <= 256 && H1 > 0 && H1 <= 128 && H2 > 0 && H2 <= 128 && A >= 2 && A <= 32,                         \
               "shape limits: D <= 256, hidden <= 128, 2 <= A <= 32")

static size_t nstep_bytes(int D, int H1, int H2, int A, int R, int M) {
  b2rl_a2c::A2cShared probe;
  return b2rl_a2c::a2c_carve<b2rl_a2c::Q, true>(probe, reinterpret_cast<float*>(uintptr_t(4096)), D, H1, H2, A, R, M) *
         sizeof(float);
}

// dynamic shared memory of the n-step Q update for these sizes (the caller checks it against the 227 KB of one SM)
extern "C" int64_t b2rl_nstep_dqn_smem_bytes(int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t N, int32_t T) {
  if (D <= 0 || H1 <= 0 || H2 <= 0 || A <= 0 || N <= 0 || T <= 0) return 0;
  return (int64_t)nstep_bytes(D, H1, H2, A, (T + 1) * N, T * N);
}

// net_kind = gate + 2 * head: gate 0 tanh / 1 ReLU, head 0 VanillaNet / 1 DuelingNet.  state_out may be NULL.
extern "C" int b2rl_nstep_dqn_actor_step(int32_t net_kind, const double* obs, double obs_scale, const float* flat,
                                         const int32_t* off, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t N,
                                         float epsilon, float* state_out, float* action_out, const float* given_action,
                                         uint64_t seed, int64_t* counter, void* stream) {
  B2RL_REQUIRE(net_kind >= 0 && net_kind <= 3, "net_kind must be gate (0 tanh, 1 relu) + 2 x head (0 VanillaNet, 1 DuelingNet)");
  const int32_t gate = net_kind & 1, head = net_kind >> 1;
  NSTEP_CHECK_NET();
  B2RL_REQUIRE(obs && action_out && counter, "null pointer");
  B2RL_REQUIRE(N > 0 && N <= 1024, "N must be in [1, 1024]");
  A2cActorArgs a;
  a.net = a2c_net(const_cast<float*>(flat), off, head ? b2rl_a2c::DUEL : b2rl_a2c::Q, 1, D, H1, H2, A);
  a.obs = obs; a.scale = obs_scale; a.N = N; a.state_out = state_out; a.action_out = action_out; a.given = given_action;
  a.seed = seed; a.counter = counter;
  b2rl_a2c::A2cShared probe;
  const size_t smem = head ? b2rl_a2c::a2c_carve<b2rl_a2c::DUEL, true>(probe, reinterpret_cast<float*>(uintptr_t(4096)), D, H1,
                                                                        H2, A, N, 0) * sizeof(float)
                           : nstep_bytes(D, H1, H2, A, N, 0);
  B2RL_REQUIRE(smem <= 227 * 1024, "network / worker count too large for the shared memory of one SM");
  if (head == 0 && state_out) {                  // the n-step agent's form: the state row goes to its rollout arena
    if (gate == b2rl_a2c::TANH) nstep_actor_launch<b2rl_a2c::TANH>(a, epsilon, smem, (cudaStream_t)stream);
    else nstep_actor_launch<b2rl_a2c::RELU>(a, epsilon, smem, (cudaStream_t)stream);
  } else {
    dqn_dispatch<DqnActorLaunch>(head, gate, a, epsilon, smem, (cudaStream_t)stream);
  }
  return check_launch("b2rl_nstep_dqn_actor_step");
}

// ------------------------------------------------------------------------------------------------ replay Q entry points
static size_t dqn_bytes(int head, int D, int H1, int H2, int A, int B, int double_q) {
  b2rl_a2c::DqnShared probe;
  float* dummy = reinterpret_cast<float*>(uintptr_t(4096));
  return (head ? b2rl_a2c::dqn_carve<b2rl_a2c::DUEL>(probe, dummy, D, H1, H2, A, B, double_q)
               : b2rl_a2c::dqn_carve<b2rl_a2c::Q>(probe, dummy, D, H1, H2, A, B, double_q)) * sizeof(float);
}

// dynamic shared memory of the replay Q update for these sizes (the caller checks it against the 227 KB of one SM)
extern "C" int64_t b2rl_dqn_replay_smem_bytes(int32_t head, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t B,
                                              int32_t double_q) {
  if (D <= 0 || H1 <= 0 || H2 <= 0 || A <= 0 || B <= 0 || (head != 0 && head != 1)) return 0;
  return (int64_t)dqn_bytes(head, D, H1, H2, A, B, double_q != 0);
}

extern "C" int b2rl_dqn_replay_update(int32_t head, int32_t gate, const void* state, const void* next_state, int32_t state_f64,
                                      double state_scale, const int64_t* action, const float* reward, const float* mask,
                                      int32_t B, int32_t D, int32_t H1, int32_t H2, int32_t A, float* flat, const float* target,
                                      float* square_avg, float* grad_avg, int64_t* step, const int32_t* off, float lr,
                                      float alpha, float eps, int32_t centered, float discount_n, int32_t double_q,
                                      float max_norm, const float* sampling_prob, float beta, float replay_eps,
                                      float replay_alpha, float* priority_out, float* delta_out, float* loss, void* stream) {
  NSTEP_CHECK_NET();
  B2RL_REQUIRE(head == 0 || head == 1, "head must be 0 (VanillaNet) or 1 (DuelingNet)");
  B2RL_REQUIRE(state && next_state && action && reward && mask && target && square_avg && step && loss &&
                   (grad_avg || !centered) && (priority_out || !sampling_prob),
               "null pointer");
  B2RL_REQUIRE(B > 0, "bad batch size");
  b2rl_a2c::DqnArgs d = {};
  b2rl_a2c::A2cArgs& a = d.a;
  a.net = a2c_net(flat, off, head ? b2rl_a2c::DUEL : b2rl_a2c::Q, 1, D, H1, H2, A);
  a.N = B; a.T = 1;
  a.sq = square_avg; a.ga = grad_avg; a.step = step;
  a.lr = lr; a.alpha = alpha; a.eps = eps; a.centered = centered;
  a.discount = discount_n; a.max_norm = max_norm; a.loss = loss;
  d.state = state; d.next_state = next_state; d.f64 = state_f64 != 0; d.scale = state_scale;
  d.action = action; d.reward = reward; d.mask = mask; d.target = target; d.double_q = double_q != 0;
  d.prob = sampling_prob; d.beta = beta; d.per_eps = replay_eps; d.per_alpha = replay_alpha;
  d.priority = priority_out; d.delta = delta_out;
  const size_t smem = (size_t)b2rl_dqn_replay_smem_bytes(head, D, H1, H2, A, B, double_q);
  B2RL_REQUIRE(smem > 0 && smem <= 227 * 1024,
               "batch / network too large for the shared memory of one SM (b2rl_dqn_replay_smem_bytes)");
  dqn_dispatch<DqnUpdateLaunch>(head, gate, d, smem, (cudaStream_t)stream);
  return check_launch("b2rl_dqn_replay_update");
}

extern "C" int b2rl_nstep_dqn_update(int32_t gate, const float* states, const float* actions, const float* reward,
                                     const float* mask, int32_t T, int32_t N, int32_t D, int32_t H1, int32_t H2, int32_t A,
                                     float* flat, float* target, int32_t sync_target, float* square_avg, float* grad_avg,
                                     int64_t* step, const int32_t* off, float lr, float alpha, float eps, int32_t centered,
                                     float discount, float max_norm, float* loss, void* stream) {
  NSTEP_CHECK_NET();
  B2RL_REQUIRE(states && actions && reward && mask && target && square_avg && step && loss && (grad_avg || !centered),
               "null pointer");
  B2RL_REQUIRE(T > 0 && N > 0, "bad T / N");
  b2rl_a2c::NStepArgs q = {};
  b2rl_a2c::A2cArgs& a = q.a;
  a.net = a2c_net(flat, off, b2rl_a2c::Q, 1, D, H1, H2, A);
  a.state = states; a.action = actions; a.reward = reward; a.mask = mask; a.T = T; a.N = N;
  a.sq = square_avg; a.ga = grad_avg; a.step = step;
  a.lr = lr; a.alpha = alpha; a.eps = eps; a.centered = centered;
  a.discount = discount; a.max_norm = max_norm; a.loss = loss;
  q.target = target; q.sync = sync_target != 0;
  const size_t smem = (size_t)b2rl_nstep_dqn_smem_bytes(D, H1, H2, A, N, T);
  B2RL_REQUIRE(smem > 0 && smem <= 227 * 1024,
               "rollout / network too large for the shared memory of one SM (b2rl_nstep_dqn_smem_bytes)");
  if (gate == b2rl_a2c::TANH) nstep_update_launch<b2rl_a2c::TANH>(q, smem, (cudaStream_t)stream);
  else nstep_update_launch<b2rl_a2c::RELU>(q, smem, (cudaStream_t)stream);
  return check_launch("b2rl_nstep_dqn_update");
}
