// TEST INFRASTRUCTURE: the phase functions of the one-launch C51 / QR-DQN update (deeprl_b200/csrc/dist_phases.h on
// a2c_phases.h, dist_sequence.inc) compiled for the host, the threads of a phase run one after another as in dqn_emul.cpp.
// tests/test_dist_dqn_device.py builds this with g++ and checks it against oracle/agents.py DQNFamilyOracle and the
// reference's recorded C51 / QR losses without a GPU.  Arguments are those of b2rl_dist_dqn_replay_update, plus the thread
// count and the thread order of every phase.
#include <cstdint>
#include <vector>

#include "../../deeprl_b200/csrc/dist_phases.h"

template <int KIND, int GATE>
static void run(const b2rl_dist::DistArgs& g, int NT, bool reversed) {
  using namespace b2rl_a2c;
  const DqnArgs& d = g.d;
  b2rl_dist::DistShared T;
  float dummy[4];
  const A2cNet& net = d.a.net;
  const size_t n = b2rl_dist::dist_carve<KIND>(T, dummy, net.D, net.H1, net.H2, g.A, g.K, d.a.N, d.double_q);
  std::vector<float> block(n, -12345.0f);                 // (poisoned: a phase that reads before anybody wrote shows up)
  b2rl_dist::dist_carve<KIND>(T, block.data(), net.D, net.H1, net.H2, g.A, g.K, d.a.N, d.double_q);
  DqnShared& DS = T.ds;
  A2cShared& S = DS.s;
#define A2C_PHASE(...)                                                  \
  if (reversed) {                                                       \
    for (int tid = NT - 1; tid >= 0; --tid) { __VA_ARGS__; }            \
  } else {                                                              \
    for (int tid = 0; tid < NT; ++tid) { __VA_ARGS__; }                 \
  }
#include "../../deeprl_b200/csrc/dist_sequence.inc"
#undef A2C_PHASE
}

extern "C" int dist_emul_update(int32_t kind, int32_t gate, const void* state, const void* next_state, int32_t state_f64,
                                double state_scale, const int64_t* action, const float* reward, const float* mask, int32_t B,
                                int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, float* flat, const float* target,
                                float* square_avg, float* grad_avg, int64_t* step, const int32_t* off, float lr, float alpha,
                                float eps, int32_t centered, float discount_n, int32_t double_q, double v_min, double v_max,
                                float max_norm, const float* sampling_prob, float beta, float replay_eps, float replay_alpha,
                                float* priority_out, float* loss_vec_out, float* loss, int32_t n_threads, int32_t reversed) {
  using namespace b2rl_a2c;
  b2rl_dist::DistArgs g = {};
  DqnArgs& d = g.d;
  A2cArgs& a = d.a;
  a.net.flat = flat;
  for (int i = 0; i < A2C_MAX_TENSORS; ++i) a.net.off[i] = i < A2cKind<Q, true>::ntensors ? off[i] : 0;
  a.net.D = D; a.net.H1 = H1; a.net.H2 = H2; a.net.A = A * K;
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
  const bool rev = reversed != 0;
  if (kind == b2rl_dist::C51 && gate == TANH) run<b2rl_dist::C51, TANH>(g, n_threads, rev);
  else if (kind == b2rl_dist::C51 && gate == RELU) run<b2rl_dist::C51, RELU>(g, n_threads, rev);
  else if (kind == b2rl_dist::QR && gate == TANH) run<b2rl_dist::QR, TANH>(g, n_threads, rev);
  else if (kind == b2rl_dist::QR && gate == RELU) run<b2rl_dist::QR, RELU>(g, n_threads, rev);
  else return 1;
  return 0;
}
