// TEST INFRASTRUCTURE: the phase functions of the one-launch n-step Q update (deeprl_b200/csrc/a2c_phases.h with HEAD = Q,
// nstep_sequence.inc) compiled for the host, the threads of a phase run one after another as in a2c_emul.cpp.
// tests/test_nstep_dqn_device.py builds this with g++ and checks it against oracle/agents.py nstep_dqn_update and the
// reference's recorded trajectory without a GPU.  Arguments are those of b2rl_nstep_dqn_update, plus the thread count and the
// thread order of every phase.
#include <cstdint>
#include <vector>

#include "../../deeprl_b200/csrc/a2c_phases.h"

template <int GATE>
static void run(const b2rl_a2c::NStepArgs& q, int NT, bool reversed) {
  using namespace b2rl_a2c;
  const A2cArgs& a = q.a;
  A2cShared S;
  float dummy[4];
  const int R = (a.T + 1) * a.N, M = a.T * a.N;
  const size_t n = a2c_carve<Q, true>(S, dummy, a.net.D, a.net.H1, a.net.H2, a.net.A, R, M);
  std::vector<float> block(n, -12345.0f);                 // (poisoned: a phase that reads before anybody wrote shows up)
  a2c_carve<Q, true>(S, block.data(), a.net.D, a.net.H1, a.net.H2, a.net.A, R, M);
#define A2C_PHASE(...)                                                  \
  if (reversed) {                                                       \
    for (int tid = NT - 1; tid >= 0; --tid) { __VA_ARGS__; }            \
  } else {                                                              \
    for (int tid = 0; tid < NT; ++tid) { __VA_ARGS__; }                 \
  }
#include "../../deeprl_b200/csrc/nstep_sequence.inc"
#undef A2C_PHASE
}

extern "C" int nstep_emul_update(int32_t gate, const float* states, const float* actions, const float* reward, const float* mask,
                                 int32_t T, int32_t N, int32_t D, int32_t H1, int32_t H2, int32_t A, float* flat, float* target,
                                 int32_t sync_target, float* square_avg, float* grad_avg, int64_t* step, const int32_t* off,
                                 float lr, float alpha, float eps, int32_t centered, float discount, float max_norm, float* loss,
                                 int32_t n_threads, int32_t reversed) {
  using namespace b2rl_a2c;
  NStepArgs q = {};
  A2cArgs& a = q.a;
  a.net.flat = flat;
  for (int i = 0; i < A2C_MAX_TENSORS; ++i) a.net.off[i] = i < A2cKind<Q, true>::ntensors ? off[i] : 0;
  a.net.D = D; a.net.H1 = H1; a.net.H2 = H2; a.net.A = A;
  a.state = states; a.action = actions; a.reward = reward; a.mask = mask; a.T = T; a.N = N;
  a.sq = square_avg; a.ga = grad_avg; a.step = step;
  a.lr = lr; a.alpha = alpha; a.eps = eps; a.centered = centered;
  a.discount = discount; a.max_norm = max_norm; a.loss = loss;
  q.target = target; q.sync = sync_target != 0;
  const bool rev = reversed != 0;
  if (gate == TANH) run<TANH>(q, n_threads, rev);
  else if (gate == RELU) run<RELU>(q, n_threads, rev);
  else return 1;
  return 0;
}
