// TEST INFRASTRUCTURE: the data-parallel phase sequence of the persistent PPO kernel (deeprl_b200/csrc/ppo_phases.h,
// ppo_dp_sequence.inc) compiled for the host, in the manner of ppo_emul.cpp (the threads of a phase run one after another,
// the barrier is the end of that loop).  tests/test_ppo_data_parallel.py builds it together with ppo_emul.cpp and checks it
// against a union-minibatch oracle without a GPU; the CUDA build of the same source is checked on the device.
#include <cstdint>
#include <vector>

#include "../../deeprl_b200/csrc/ppo_phases.h"

// The data-parallel sequence (ppo_dp_sequence.inc) for W ranks in lockstep: every phase runs rank after rank (each with its own
// block of shared memory and arguments), and inside a rank thread after thread.  The exchange is then a phase boundary: when
// any rank runs its wait phase, every rank has run its publish phase.  Per-rank arrays hold W consecutive copies (the
// one-device layout of b2rl_ppo_minibatch_updates_dp); `regions` is one zero-filled buffer of W exchange regions of
// `region_floats` floats.  reverse_ranks / reverse_threads: run ranks / threads in the opposite order.
extern "C" int ppo_emul_minibatch_updates_dp(const float* state, const float* action, const float* old_log_pi_a, const float* ret,
                                             const float* advantage, int32_t D, int32_t A, int32_t H1, int32_t H2, int32_t mb,
                                             const int64_t* perm, int32_t n_batches, float* a_flat, float* a_exp_avg,
                                             float* a_exp_avg_sq, int64_t* a_step, const int32_t* a_off, float* c_flat,
                                             float* c_exp_avg, float* c_exp_avg_sq, int64_t* c_step, const int32_t* c_off,
                                             float a_lr, float a_beta1, float a_beta2, float a_eps, float c_lr, float c_beta1,
                                             float c_beta2, float c_eps, float ratio_clip, float entropy_weight, float kl_gate,
                                             float* stats, int32_t rows, int32_t a_n, int32_t c_n, int32_t world, float* regions,
                                             int64_t region_floats, int64_t seq_base, int64_t* status, int32_t n_threads,
                                             int32_t reverse_ranks, int32_t reverse_threads) {
  using namespace b2rl_ppo;
  if (world < 1 || world > PPO_DP_MAX_WORLD) return -1;
  std::vector<PpoArgs> as(world);
  std::vector<PpoDp> ds(world);
  std::vector<PpoShared> Ss(world);
  std::vector<std::vector<float>> blocks(world);
  int c_base = 0, stat_at = 0;
  const int slot_floats = ppo_dp_slot_floats(a_n, c_n, &c_base, &stat_at);
  if (PPO_DP_HEADER_FLOATS + 2 * (int64_t)slot_floats > region_floats) return -1;
  for (int r = 0; r < world; ++r) {
    PpoArgs& a = as[r];
    const int64_t R = rows;
    a.state = state + r * R * D; a.action = action + r * R * A; a.old_logp = old_log_pi_a + r * R; a.ret = ret + r * R;
    a.adv = advantage + r * R;
    a.D = D; a.A = A; a.H1 = H1; a.H2 = H2; a.mb = mb; a.perm = perm + (int64_t)r * n_batches * mb; a.n_batches = n_batches;
    a.a_flat = a_flat + (int64_t)r * a_n; a.a_m = a_exp_avg + (int64_t)r * a_n; a.a_v = a_exp_avg_sq + (int64_t)r * a_n;
    a.a_step = a_step + r;
    a.c_flat = c_flat + (int64_t)r * c_n; a.c_m = c_exp_avg + (int64_t)r * c_n; a.c_v = c_exp_avg_sq + (int64_t)r * c_n;
    a.c_step = c_step + r;
    for (int i = 0; i < 7; ++i) a.a_off[i] = a_off[i];
    for (int i = 0; i < 6; ++i) a.c_off[i] = c_off[i];
    a.a_lr = a_lr; a.a_b1 = a_beta1; a.a_b2 = a_beta2; a.a_eps = a_eps;
    a.c_lr = c_lr; a.c_b1 = c_beta1; a.c_b2 = c_beta2; a.c_eps = c_eps;
    a.clip = ratio_clip; a.ent_w = entropy_weight; a.gate_max = kl_gate; a.stats = stats + 4 * r; a.clk = nullptr;
    PpoDp& d = ds[r];
    d = PpoDp{};
    for (int p = 0; p < world; ++p) d.region[p] = regions + p * region_floats;
    d.world = world; d.rank = r;
    d.slot_floats = slot_floats; d.c_base = c_base; d.stat_at = stat_at;
    d.seq_base = seq_base;
    d.timeout_ns = 1000000000LL;
    d.status = reinterpret_cast<long long*>(status) + r;
    float dummy[4];
    const size_t n = ppo_carve(Ss[r], dummy, D, A, H1, H2, mb);
    blocks[r].assign(n, -12345.0f);
    ppo_carve(Ss[r], blocks[r].data(), D, A, H1, H2, mb);
  }
  const int NT = n_threads;
  const PpoArgs& a = as[0];                               // (the loop bound outside the phases: n_batches, the same on every rank)
#define PPO_PHASE(stmt)                                                                   \
  for (int ri = 0; ri < world; ++ri) {                                                    \
    const int rr = reverse_ranks ? world - 1 - ri : ri;                                   \
    PpoShared& S = Ss[rr];                                                                \
    const PpoArgs& a = as[rr];                                                            \
    const PpoDp& d = ds[rr];                                                              \
    for (int ti = 0; ti < NT; ++ti) {                                                     \
      const int tid = reverse_threads ? NT - 1 - ti : ti;                                 \
      stmt;                                                                               \
    }                                                                                     \
  }
  bool aborted = false;
#define PPO_DP_ABORTED (aborted = aborted || [&] { for (int r = 0; r < world; ++r) if (Ss[r].flag[6] != 0.0f) return true; return false; }())
#include "../../deeprl_b200/csrc/ppo_dp_sequence.inc"
#undef PPO_DP_ABORTED
#undef PPO_PHASE
  return aborted ? 1 : 0;
}
