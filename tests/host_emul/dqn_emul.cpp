// TEST INFRASTRUCTURE: the phase functions of the one-launch replay Q update (deeprl_b200/csrc/a2c_phases.h with HEAD = Q or
// DUEL, dqn_sequence.inc) compiled for the host, the threads of a phase run one after another as in nstep_emul.cpp.
// tests/test_dqn_device.py builds this with g++ and checks it against oracle/agents.py DQNFamilyOracle and the reference's
// recorded DQN updates without a GPU.  Arguments are those of b2rl_dqn_replay_update, plus the thread count and the thread
// order of every phase.
#include <cstdint>
#include <vector>

#include "../../deeprl_b200/csrc/a2c_phases.h"

template <int HEAD, int GATE>
static void run(const b2rl_a2c::DqnArgs& d, int NT, bool reversed) {
  using namespace b2rl_a2c;
  DqnShared DS;
  float dummy[4];
  const A2cNet& net = d.a.net;
  const size_t n = dqn_carve<HEAD>(DS, dummy, net.D, net.H1, net.H2, net.A, d.a.N, d.double_q);
  std::vector<float> block(n, -12345.0f);                 // (poisoned: a phase that reads before anybody wrote shows up)
  dqn_carve<HEAD>(DS, block.data(), net.D, net.H1, net.H2, net.A, d.a.N, d.double_q);
  A2cShared& S = DS.s;
#define A2C_PHASE(...)                                                  \
  if (reversed) {                                                       \
    for (int tid = NT - 1; tid >= 0; --tid) { __VA_ARGS__; }            \
  } else {                                                              \
    for (int tid = 0; tid < NT; ++tid) { __VA_ARGS__; }                 \
  }
#include "../../deeprl_b200/csrc/dqn_sequence.inc"
#undef A2C_PHASE
}

extern "C" int dqn_emul_update(int32_t head, int32_t gate, const void* state, const void* next_state, int32_t state_f64,
                               double state_scale, const int64_t* action, const float* reward, const float* mask, int32_t B,
                               int32_t D, int32_t H1, int32_t H2, int32_t A, float* flat, const float* target, float* square_avg,
                               float* grad_avg, int64_t* step, const int32_t* off, float lr, float alpha, float eps,
                               int32_t centered, float discount_n, int32_t double_q, float max_norm, const float* sampling_prob,
                               float beta, float replay_eps, float replay_alpha, float* priority_out, float* delta_out,
                               float* loss, int32_t n_threads, int32_t reversed) {
  using namespace b2rl_a2c;
  DqnArgs d = {};
  A2cArgs& a = d.a;
  a.net.flat = flat;
  const int nt = head ? A2cKind<DUEL, true>::ntensors : A2cKind<Q, true>::ntensors;
  for (int i = 0; i < A2C_MAX_TENSORS; ++i) a.net.off[i] = i < nt ? off[i] : 0;
  a.net.D = D; a.net.H1 = H1; a.net.H2 = H2; a.net.A = A;
  a.N = B; a.T = 1;
  a.sq = square_avg; a.ga = grad_avg; a.step = step;
  a.lr = lr; a.alpha = alpha; a.eps = eps; a.centered = centered;
  a.discount = discount_n; a.max_norm = max_norm; a.loss = loss;
  d.state = state; d.next_state = next_state; d.f64 = state_f64 != 0; d.scale = state_scale;
  d.action = action; d.reward = reward; d.mask = mask; d.target = target; d.double_q = double_q != 0;
  d.prob = sampling_prob; d.beta = beta; d.per_eps = replay_eps; d.per_alpha = replay_alpha;
  d.priority = priority_out; d.delta = delta_out;
  const bool rev = reversed != 0;
  if (head == 0 && gate == TANH) run<Q, TANH>(d, n_threads, rev);
  else if (head == 0 && gate == RELU) run<Q, RELU>(d, n_threads, rev);
  else if (head == 1 && gate == TANH) run<DUEL, TANH>(d, n_threads, rev);
  else if (head == 1 && gate == RELU) run<DUEL, RELU>(d, n_threads, rev);
  else return 1;
  return 0;
}
