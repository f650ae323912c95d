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

#include <cstring>

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

// The data-parallel form (ppo_dp_sequence.inc): one block per rank.  Across GPUs every process launches one block
// (ranks_in_launch = 1); on one device the W ranks are the W blocks of ONE cooperative launch (co-resident by construction, so a
// block never waits on one that is not scheduled) and block b runs as rank b.  The per-rank arguments and peer tables live in
// the parameter space (__grid_constant__: read in place, never copied to local memory) and are selected by blockIdx.x -- the
// only code the one-device form adds.
struct PpoDpLaunch {
  b2rl_ppo::PpoArgs a[b2rl_ppo::PPO_DP_MAX_WORLD];
  b2rl_ppo::PpoDp d[b2rl_ppo::PPO_DP_MAX_WORLD];
  int ranks_in_launch;
};

__global__ void __launch_bounds__(PPO_NT, 1) ppo_dp_persistent_kernel(const __grid_constant__ PpoDpLaunch L) {
  using namespace b2rl_ppo;
  pdl_sync();
  extern __shared__ __align__(16) float ppo_smem[];
  const int r = L.ranks_in_launch > 1 ? (int)blockIdx.x : 0;
  const PpoArgs& a = L.a[r];
  const PpoDp& d = L.d[r];
  PpoShared S;
  ppo_carve(S, ppo_smem, a.D, a.A, a.H1, a.H2, a.mb);
  const int NT = PPO_NT;
  int clk_i = 0;
#define PPO_PHASE(stmt) { const int tid = threadIdx.x; stmt; } __syncthreads(); \
  if (a.clk && threadIdx.x == 0) a.clk[clk_i++] = clock64();
#define PPO_DP_ABORTED (S.flag[6] != 0.0f)
#include "ppo_dp_sequence.inc"
#undef PPO_DP_ABORTED
#undef PPO_PHASE
}

}  // namespace b2rl

using namespace b2rl;

static long long* g_ppo_clocks = nullptr;

// Profiling hook: install (or with NULL remove) a device buffer of int64 [2 + 9 * n_batches] (data-parallel kernel:
// [2 + 12 * n_batches], rank 0 / block 0 only) that the next launches fill with clock64() of thread 0 after every phase
// barrier (scripts/ppo_phase_clocks.py, scripts/ppo_dp_scaling.py turn it into cycles per phase).
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

// ------------------------------------------------------------------------------------------------ data parallel
// bytes of one rank's exchange region for arenas of a_n / c_n elements (flag header + two gradient slots)
extern "C" int64_t b2rl_ppo_dp_region_bytes(int32_t a_n, int32_t c_n) {
  if (a_n <= 0 || c_n <= 0) return 0;
  return (int64_t)(b2rl_ppo::PPO_DP_HEADER_FLOATS + 2 * (int64_t)b2rl_ppo::ppo_dp_slot_floats(a_n, c_n, nullptr, nullptr)) * 4;
}

extern "C" int b2rl_ppo_minibatch_updates_dp(const float* state, const float* action, const float* old_log_pi_a, const float* ret,
                                             const float* advantage, int32_t D, int32_t A, int32_t H1, int32_t H2, int32_t mb,
                                             const int64_t* perm, int32_t n_batches,
                                             float* a_flat, float* a_exp_avg, float* a_exp_avg_sq, int64_t* a_step, const int32_t* a_off,
                                             float* c_flat, float* c_exp_avg, float* c_exp_avg_sq, int64_t* c_step, const int32_t* c_off,
                                             float a_lr, float a_beta1, float a_beta2, float a_eps, float c_lr, float c_beta1,
                                             float c_beta2, float c_eps, float ratio_clip, float entropy_weight, float kl_gate,
                                             float* stats, int32_t rows, int32_t a_n, int32_t c_n, int32_t world, int32_t rank,
                                             void* const* regions, int64_t seq_base, int64_t timeout_ns, int64_t* status,
                                             int32_t ranks_in_launch, void* stream) {
  B2RL_REQUIRE(state && action && old_log_pi_a && ret && advantage && perm && a_flat && a_exp_avg && a_exp_avg_sq && a_step &&
               a_off && c_flat && c_exp_avg && c_exp_avg_sq && c_step && c_off && stats && regions && status, "null pointer");
  B2RL_REQUIRE(D > 0 && D <= 256 && A > 0 && A <= 32 && H1 > 0 && H1 <= 128 && H2 > 0 && H2 <= 128, "shape limits: D <= 256, A <= 32, hidden <= 128");
  B2RL_REQUIRE(mb >= 4 && mb <= 128 && mb % 4 == 0, "mini_batch_size must be a multiple of 4, at most 128");
  B2RL_REQUIRE(n_batches >= 0 && rows > 0, "bad n_batches / rows");
  B2RL_REQUIRE(world >= 1 && world <= b2rl_ppo::PPO_DP_MAX_WORLD, "world must be in [1, 8]");
  B2RL_REQUIRE(rank >= 0 && rank < world, "rank must be < world");
  B2RL_REQUIRE(ranks_in_launch == 1 || ranks_in_launch == world, "ranks_in_launch must be 1 (one process per GPU) or world (one device)");
  B2RL_REQUIRE(ranks_in_launch == 1 || rank == 0, "ranks_in_launch == world: block b is rank b, pass rank 0");
  B2RL_REQUIRE(seq_base >= 0 && timeout_ns > 0, "bad seq_base / timeout");
  for (int p = 0; p < world; ++p) B2RL_REQUIRE(regions[p] != nullptr, "null exchange region");
  const int64_t a_sz[7] = {(int64_t)H1 * D, H1, (int64_t)H2 * H1, H2, (int64_t)A * H2, A, A};
  const int64_t c_sz[6] = {(int64_t)H1 * D, H1, (int64_t)H2 * H1, H2, H2, 1};
  for (int i = 0; i < 7; ++i) B2RL_REQUIRE(a_off[i] >= 0 && a_off[i] + a_sz[i] <= a_n, "actor offsets outside the arena of a_n elements");
  for (int i = 0; i < 6; ++i) B2RL_REQUIRE(c_off[i] >= 0 && c_off[i] + c_sz[i] <= c_n, "critic offsets outside the arena of c_n elements");
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
  // one argument set per rank of the launch: in the one-device form rank r's copy of every per-rank array starts r copies in
  PpoDpLaunch L = {};
  L.ranks_in_launch = ranks_in_launch;
  int c_base = 0, stat_at = 0;
  const int slot_floats = b2rl_ppo::ppo_dp_slot_floats(a_n, c_n, &c_base, &stat_at);
  for (int r = 0; r < ranks_in_launch; ++r) {
    b2rl_ppo::PpoArgs& x = L.a[r];
    x = a;
    const int64_t R = rows;
    x.state += r * R * D; x.action += r * R * A; x.old_logp += r * R; x.ret += r * R; x.adv += r * R;
    x.perm += (int64_t)r * n_batches * mb;
    x.a_flat += (int64_t)r * a_n; x.a_m += (int64_t)r * a_n; x.a_v += (int64_t)r * a_n; x.a_step += r;
    x.c_flat += (int64_t)r * c_n; x.c_m += (int64_t)r * c_n; x.c_v += (int64_t)r * c_n; x.c_step += r;
    x.stats += 4 * r;
    if (r != 0) x.clk = nullptr;
    b2rl_ppo::PpoDp& d = L.d[r];
    d = {};
    for (int p = 0; p < world; ++p) d.region[p] = reinterpret_cast<float*>(regions[p]);
    d.world = world;
    d.rank = ranks_in_launch > 1 ? r : rank;
    d.slot_floats = slot_floats;
    d.c_base = c_base;
    d.stat_at = stat_at;
    d.seq_base = seq_base;
    d.timeout_ns = timeout_ns;
    d.status = reinterpret_cast<long long*>(status) + r;
  }
  const size_t smem = (size_t)b2rl_ppo_minibatch_smem_bytes(D, A, H1, H2, mb);
  B2RL_REQUIRE(smem <= 227 * 1024, "networks / minibatch too large for the shared memory of one SM");
  static size_t attr = 0;
  if (smem > attr) {
    cudaFuncSetAttribute(ppo_dp_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = smem;
  }
  // cooperative: the ranks_in_launch blocks are co-resident or the launch fails (never a spin on an unscheduled block)
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(ranks_in_launch);
  cfg.blockDim = dim3(PPO_NT);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr_c[1];
  attr_c[0].id = cudaLaunchAttributeCooperative;
  attr_c[0].val.cooperative = 1;
  cfg.attrs = attr_c;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, ppo_dp_persistent_kernel, L);
  return check_launch("b2rl_ppo_minibatch_updates_dp");
}

// Exchange memory shared between processes (CUDA IPC, plain runtime calls).  Allocated and zero-filled once at setup; the
// update path allocates nothing.
extern "C" int b2rl_ipc_alloc(int64_t bytes, void** out) {
  B2RL_REQUIRE(out && bytes > 0, "bad arguments");
  void* p = nullptr;
  cudaError_t e = cudaMalloc(&p, (size_t)bytes);
  if (e == cudaSuccess) e = cudaMemset(p, 0, (size_t)bytes);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    if (p) cudaFree(p);
    set_error("b2rl_ipc_alloc: %s", cudaGetErrorString(e));
    return B2RL_ERR_CUDA;
  }
  *out = p;
  return B2RL_OK;
}

extern "C" int b2rl_ipc_get_handle(void* ptr, void* handle_out) {
  B2RL_REQUIRE(ptr && handle_out, "null pointer");
  cudaIpcMemHandle_t h;
  const cudaError_t e = cudaIpcGetMemHandle(&h, ptr);
  if (e != cudaSuccess) {
    set_error("b2rl_ipc_get_handle: %s", cudaGetErrorString(e));
    return B2RL_ERR_CUDA;
  }
  memcpy(handle_out, &h, sizeof(h));
  return B2RL_OK;
}

extern "C" int b2rl_ipc_open_handle(const void* handle, void** out) {
  B2RL_REQUIRE(handle && out, "null pointer");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  const cudaError_t e = cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    set_error("b2rl_ipc_open_handle: %s", cudaGetErrorString(e));
    return B2RL_ERR_CUDA;
  }
  return B2RL_OK;
}

extern "C" int b2rl_ipc_close(void* ptr) {
  B2RL_REQUIRE(ptr, "null pointer");
  const cudaError_t e = cudaIpcCloseMemHandle(ptr);
  if (e != cudaSuccess) {
    set_error("b2rl_ipc_close: %s", cudaGetErrorString(e));
    return B2RL_ERR_CUDA;
  }
  return B2RL_OK;
}

extern "C" int b2rl_ipc_free(void* ptr) {
  B2RL_REQUIRE(ptr, "null pointer");
  const cudaError_t e = cudaFree(ptr);
  if (e != cudaSuccess) {
    set_error("b2rl_ipc_free: %s", cudaGetErrorString(e));
    return B2RL_ERR_CUDA;
  }
  return B2RL_OK;
}

// *ok = 1 when device dev_a can access device dev_b's memory directly (or they are the same device)
extern "C" int b2rl_peer_access_ok(int32_t dev_a, int32_t dev_b, int32_t* ok) {
  B2RL_REQUIRE(ok, "null pointer");
  int v = 1;
  if (dev_a != dev_b) {
    const cudaError_t e = cudaDeviceCanAccessPeer(&v, dev_a, dev_b);
    if (e != cudaSuccess) {
      set_error("b2rl_peer_access_ok: %s", cudaGetErrorString(e));
      return B2RL_ERR_CUDA;
    }
  }
  *ok = v;
  return B2RL_OK;
}
