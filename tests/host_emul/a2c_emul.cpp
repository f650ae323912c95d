// TEST INFRASTRUCTURE: the phase functions of the one-launch A2C update (deeprl_b200/csrc/a2c_phases.h, a2c_sequence.inc)
// compiled for the host.  A "block" is emulated by running the NT threads of a phase one after another and the barrier by the
// end of that loop -- valid because no phase lets a thread read what another thread of the SAME phase writes (which is also what
// makes the CUDA version race-free).  tests/test_a2c_device.py builds this with g++ and checks it against the oracle's A2C
// updates (oracle/agents.py) and the reference's recorded trajectory without a GPU; the CUDA build of the same source is checked
// on the device.  Arguments are those of b2rl_a2c_update, plus the thread count and the thread order of every phase.
#include <cstdint>
#include <vector>

#include "../../deeprl_b200/csrc/a2c_phases.h"

template <int HEAD, bool SHARED, int GATE>
static void run(const b2rl_a2c::A2cArgs& a, int NT, bool reversed) {
  using namespace b2rl_a2c;
  A2cShared S;
  float dummy[4];
  const int R = (a.T + 1) * a.N, M = a.T * a.N;
  const size_t n = a2c_carve<HEAD, SHARED>(S, dummy, a.net.D, a.net.H1, a.net.H2, a.net.A, R, M);
  std::vector<float> block(n, -12345.0f);                 // (poisoned: a phase that reads before anybody wrote shows up)
  a2c_carve<HEAD, SHARED>(S, block.data(), a.net.D, a.net.H1, a.net.H2, a.net.A, R, M);
#define A2C_PHASE(...)                                                  \
  if (reversed) {                                                       \
    for (int tid = NT - 1; tid >= 0; --tid) { __VA_ARGS__; }            \
  } else {                                                              \
    for (int tid = 0; tid < NT; ++tid) { __VA_ARGS__; }                 \
  }
#include "../../deeprl_b200/csrc/a2c_sequence.inc"
#undef A2C_PHASE
}

extern "C" int a2c_emul_update(int32_t head, int32_t shared, int32_t gate, const float* states, const float* actions,
                               const float* reward, const float* mask, int32_t T, int32_t N, int32_t D, int32_t H1, int32_t H2,
                               int32_t A, float* flat, float* square_avg, float* grad_avg, int64_t* step, const int32_t* off,
                               float lr, float alpha, float eps, int32_t centered, float discount, float tau, int32_t use_gae,
                               float entropy_weight, float value_loss_weight, float max_norm, float* loss, int32_t n_threads,
                               int32_t reversed) {
  using namespace b2rl_a2c;
  A2cArgs a;
  a.net.flat = flat;
  const int nt = 4 * (shared ? 1 : 2) + 4 + (head == GAUSS ? 1 : 0);
  for (int i = 0; i < A2C_MAX_TENSORS; ++i) a.net.off[i] = i < nt ? off[i] : 0;
  a.net.D = D; a.net.H1 = H1; a.net.H2 = H2; a.net.A = A;
  a.state = states; a.action = actions; a.reward = reward; a.mask = mask; a.T = T; a.N = N;
  a.sq = square_avg; a.ga = grad_avg; a.step = step;
  a.lr = lr; a.alpha = alpha; a.eps = eps; a.centered = centered;
  a.discount = discount; a.tau = tau; a.use_gae = use_gae;
  a.ent_w = entropy_weight; a.vw = value_loss_weight; a.max_norm = max_norm; a.loss = loss;
  const bool rev = reversed != 0;
  if (head == CAT && shared && gate == TANH) run<CAT, true, TANH>(a, n_threads, rev);
  else if (head == CAT && shared && gate == RELU) run<CAT, true, RELU>(a, n_threads, rev);
  else if (head == GAUSS && !shared && gate == TANH) run<GAUSS, false, TANH>(a, n_threads, rev);
  else if (head == GAUSS && !shared && gate == RELU) run<GAUSS, false, RELU>(a, n_threads, rev);
  else return 1;
  return 0;
}
