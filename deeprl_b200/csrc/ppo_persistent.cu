// ppo_persistent.cu -- ALL minibatch updates of one PPO iteration (PPO_agent.py:68-99: optimization_epochs x rows/mini_batch_size
// updates, 5 120 in examples.py:496-522) as ONE launch of one persistent thread block.
//
// Why one block: an update is 2 M FMAs on an 11 k-parameter pair of MLPs over 64 rows -- a few microseconds of one SM -- and
// every update depends on the parameters written by the one before it.  As separate launches (the CUDA-graph form,
// learner.GraphedPPOLearner) it is bound by the launch / dependency latency of ~45 tiny kernels.  Here the
// weights live in shared memory for the whole iteration, the Adam moments in L2, the minibatch rows are fetched one update
// ahead by the idle half of the block, and the only synchronisation is the block barrier between the nine phases of an
// update (ppo_phases.h, ppo_sequence.inc: the same source is compiled for the host by tests/host_emul to check the arithmetic).
// The actor and the critic are independent networks (non-shared representation): they run side by side on the two halves
// of the block.  sm_90a only.
#include "common.cuh"
#include "ppo_phases.h"

namespace b2rl {

constexpr int PPO_NT = 512;

__global__ void __launch_bounds__(PPO_NT, 1) ppo_minibatch_persistent_kernel(const b2rl_ppo::PpoArgs a) {
  using namespace b2rl_ppo;
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ __align__(16) float ppo_smem[];
  PpoShared S;
  ppo_carve(S, ppo_smem, a.D, a.A, a.H1, a.H2, a.mb);
  const int NT = PPO_NT;
  int clk_i = 0;                  // (profiling hook: thread 0 stamps the end of every phase when a clock buffer is installed)
#define PPO_PHASE(stmt) { const int tid = threadIdx.x; stmt; } __syncthreads(); \
  if (a.clk && threadIdx.x == 0) a.clk[clk_i++] = clock64();
#include "ppo_sequence.inc"
#undef PPO_PHASE
}

}  // namespace b2rl

using namespace b2rl;

static long long* g_ppo_clocks = nullptr;

// Profiling hook: install (or with NULL remove) a device buffer of int64 [2 + 9 * n_batches] that the next launches fill with
// clock64() of thread 0 after every phase barrier (scripts/ppo_phase_clocks.py turns it into cycles per phase).
extern "C" int b2rl_ppo_set_phase_clocks(int64_t* clocks) {
  g_ppo_clocks = reinterpret_cast<long long*>(clocks);
  return 0;
}

// dynamic shared memory the persistent kernel needs for these sizes (the caller checks it against the 227 KB of one SM)
extern "C" int64_t b2rl_ppo_minibatch_smem_bytes(int32_t D, int32_t A, int32_t H1, int32_t H2, int32_t mb) {
  b2rl_ppo::PpoShared probe;
  return (int64_t)(b2rl_ppo::ppo_carve(probe, reinterpret_cast<float*>(uintptr_t(4096)), D, A, H1, H2, mb) * sizeof(float));
}

extern "C" int b2rl_ppo_minibatch_updates(const float* state, const float* action, const float* old_log_pi_a, const float* ret,
                                          const float* advantage, int32_t D, int32_t A, int32_t H1, int32_t H2, int32_t mb,
                                          const int64_t* perm, int32_t n_batches,
                                          float* a_flat, float* a_exp_avg, float* a_exp_avg_sq, int64_t* a_step, const int32_t* a_off,
                                          float* c_flat, float* c_exp_avg, float* c_exp_avg_sq, int64_t* c_step, const int32_t* c_off,
                                          float a_lr, float a_beta1, float a_beta2, float a_eps, float c_lr, float c_beta1,
                                          float c_beta2, float c_eps, float ratio_clip, float entropy_weight, float kl_gate,
                                          float* stats, void* stream) {
  B2RL_REQUIRE(state && action && old_log_pi_a && ret && advantage && perm && a_flat && a_exp_avg && a_exp_avg_sq && a_step &&
               a_off && c_flat && c_exp_avg && c_exp_avg_sq && c_step && c_off && stats, "null pointer");
  B2RL_REQUIRE(D > 0 && D <= 256 && A > 0 && A <= 32 && H1 > 0 && H1 <= 128 && H2 > 0 && H2 <= 128, "shape limits: D <= 256, A <= 32, hidden <= 128");
  B2RL_REQUIRE(mb >= 4 && mb <= 128 && mb % 4 == 0, "mini_batch_size must be a multiple of 4, at most 128");
  B2RL_REQUIRE(n_batches >= 0, "bad n_batches");
  b2rl_ppo::PpoArgs a;
  a.state = state; a.action = action; a.old_logp = old_log_pi_a; a.ret = ret; a.adv = advantage;
  a.D = D; a.A = A; a.H1 = H1; a.H2 = H2; a.mb = mb; a.perm = perm; a.n_batches = n_batches;
  a.a_flat = a_flat; a.a_m = a_exp_avg; a.a_v = a_exp_avg_sq; a.a_step = a_step;
  a.c_flat = c_flat; a.c_m = c_exp_avg; a.c_v = c_exp_avg_sq; a.c_step = c_step;
  for (int i = 0; i < 7; ++i) a.a_off[i] = a_off[i];
  for (int i = 0; i < 6; ++i) a.c_off[i] = c_off[i];
  a.a_lr = a_lr; a.a_b1 = a_beta1; a.a_b2 = a_beta2; a.a_eps = a_eps;
  a.c_lr = c_lr; a.c_b1 = c_beta1; a.c_b2 = c_beta2; a.c_eps = c_eps;
  a.clip = ratio_clip; a.ent_w = entropy_weight; a.gate_max = kl_gate; a.stats = stats; a.clk = g_ppo_clocks;
  const size_t smem = (size_t)b2rl_ppo_minibatch_smem_bytes(D, A, H1, H2, mb);
  B2RL_REQUIRE(smem <= 227 * 1024, "networks / minibatch too large for the shared memory of one SM");
  static size_t attr = 0;
  if (smem > attr) {
    cudaFuncSetAttribute(ppo_minibatch_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = smem;
  }
  launch_pdl(ppo_minibatch_persistent_kernel, dim3(1), dim3(PPO_NT), smem, (cudaStream_t)stream, a);
  return check_launch("b2rl_ppo_minibatch_updates");
}
