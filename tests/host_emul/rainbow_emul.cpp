// TEST INFRASTRUCTURE: the phase functions of the one-launch Rainbow update (deeprl_b200/csrc/rainbow_phases.h on dist_phases.h
// and a2c_phases.h, rainbow_sequence.inc) compiled for the host, the threads of a phase run one after another as in
// dist_emul.cpp.  tests/test_rainbow_device.py builds this with g++ and checks it against oracle/rainbow.py RainbowOracle
// and the reference's recorded Rainbow updates without a GPU.  Arguments are those of
// b2rl_rainbow_replay_update without the Philox key and counter (the host draws nothing: with NoisyLinear layers the noise
// vectors are given), plus the thread count and the thread order of every phase.
#include <cstdint>
#include <vector>

#include "../../deeprl_b200/csrc/rainbow_phases.h"

struct NoDraw {
  float operator()(int64_t) const { return 0.0f; }
};

template <bool NOISY, int GATE>
static void run(const b2rl_rainbow::RbArgs& r, int NT, bool reversed) {
  const b2rl_dist::DistArgs& g = r.g;
  const b2rl_a2c::DqnArgs& d = g.d;
  b2rl_rainbow::RbShared RS;
  float dummy[4];
  const size_t n = b2rl_rainbow::rb_carve<NOISY>(RS, dummy, r.net, d.a.N);
  std::vector<float> block(n, -12345.0f);                 // (poisoned: a phase that reads before anybody wrote shows up)
  b2rl_rainbow::rb_carve<NOISY>(RS, block.data(), r.net, d.a.N);
  b2rl_dist::DistShared& T = RS.t;
  b2rl_a2c::A2cShared& S = T.ds.s;
  b2rl_a2c::A2cShared SO = b2rl_rainbow::rb_online_rows(S, d.double_q);
  const NoDraw draw;
  const int64_t ctr0 = 0;
#define A2C_PHASE(...)                                                  \
  if (reversed) {                                                       \
    for (int tid = NT - 1; tid >= 0; --tid) { __VA_ARGS__; }            \
  } else {                                                              \
    for (int tid = 0; tid < NT; ++tid) { __VA_ARGS__; }                 \
  }
#include "../../deeprl_b200/csrc/rainbow_sequence.inc"
#undef A2C_PHASE
}

extern "C" int rainbow_emul_noise_len(int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, int32_t arena) {
  b2rl_rainbow::RbNet n = {};
  n.D = D; n.H1 = H1; n.H2 = H2; n.A = A; n.K = K;
  return arena ? b2rl_rainbow::rb_noise_arena_len(n) : b2rl_rainbow::rb_noise_len(n);
}

extern "C" int rainbow_emul_update(int32_t noisy, int32_t gate, const void* state, const void* next_state, int32_t state_f64,
                                   double state_scale, const int64_t* action, const float* reward, const float* mask, int32_t B,
                                   int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, float* flat, const float* target,
                                   float* square_avg, float* grad_avg, int64_t* step, const int32_t* off, float lr, float alpha,
                                   float eps, int32_t centered, float discount_n, int32_t double_q, double v_min, double v_max,
                                   float max_norm, const float* sampling_prob, float beta, float replay_eps, float replay_alpha,
                                   float* priority_out, float* loss_vec_out, float* loss, const float* given_noise,
                                   float* noise_out, float* target_noise_out, int32_t n_threads, int32_t reversed) {
  using namespace b2rl_a2c;
  if (noisy && !given_noise) return 2;
  b2rl_rainbow::RbArgs r = {};
  b2rl_dist::DistArgs& g = r.g;
  DqnArgs& d = g.d;
  A2cArgs& a = d.a;
  r.net.flat = flat;
  for (int i = 0; i < b2rl_rainbow::RB_MAX_TENSORS; ++i) r.net.off[i] = i < (noisy ? 16 : 8) ? off[i] : 0;
  r.net.D = D; r.net.H1 = H1; r.net.H2 = H2; r.net.A = A; r.net.K = K;
  a.net.D = D; a.net.H1 = H1; a.net.H2 = H2; a.net.A = (A + 1) * K;
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
  r.given = given_noise; r.noise_out = noise_out; r.target_noise_out = target_noise_out; r.noise_std = 0.0f;
  const bool rev = reversed != 0;
  if (noisy && gate == TANH) run<true, TANH>(r, n_threads, rev);
  else if (noisy && gate == RELU) run<true, RELU>(r, n_threads, rev);
  else if (!noisy && gate == TANH) run<false, TANH>(r, n_threads, rev);
  else if (!noisy && gate == RELU) run<false, RELU>(r, n_threads, rev);
  else return 1;
  return 0;
}
