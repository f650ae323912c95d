/* b2rl.h -- C ABI of libb2rl.so: the sm_90a hot path behind the DeepRL (ShangtongZhang/DeepRL) API.
 *
 * The reference has NO FFI / plugin layer: its seams are duck-typed Python factories on Config
 * (SURVEY.md 8b).  This header is the boundary a maintainer binds with ctypes (INTEGRATION.md)
 * from the reference-side classes named beside each entry point.  Citations are file:line under
 * /root/reference/deep_rl.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; the caller (PyTorch caching
 *     allocator in our host mirror) owns every buffer; the library allocates nothing on the hot path
 *   - every call enqueues work on `stream` (a cudaStream_t passed as void*) and returns at once;
 *     all calls are CUDA-graph capturable (no host sync, no allocation)
 *   - return value: 0 on success, negative b2rl_status on error; b2rl_last_error() gives the message
 *     (thread-local).  Nothing throws across the boundary.
 *   - "ring state" is a device int64[8]: [0]=pos [1]=size [2]=capacity [3]=tree write cursor
 *     [4]=philox counter [5..7] reserved; device-resident so that feed/sample/update can be captured
 *     in one CUDA graph
 */
#ifndef B2RL_H
#define B2RL_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  B2RL_OK = 0,
  B2RL_ERR_ARG = -1,      /* bad argument (null pointer, size out of range, unsupported shape) */
  B2RL_ERR_CUDA = -2,     /* a CUDA runtime call / kernel launch failed */
  B2RL_ERR_UNSUPPORTED = -3
} b2rl_status;

typedef enum { B2RL_U8 = 0, B2RL_F16 = 1, B2RL_BF16 = 2, B2RL_F32 = 3 } b2rl_dtype;

int b2rl_version(void);
const char* b2rl_last_error(void);
/* number of kernels this library has launched since load / since the last reset (bench.py "gpu_launches") */
int64_t b2rl_launch_count(void);
void b2rl_reset_launch_count(void);
/* Programmatic dependent launch of the per-update kernels (each kernel's prologue overlaps the tail of the one before it;
 * csrc/common.cuh).  On by default; 0 launches every kernel with plain stream order (also: environment B2RL_PDL=0). */
void b2rl_set_pdl(int32_t on);

/* ---------------------------------------------------------------------------------------------
 * Replay ring -- UniformReplay.feed / valid_index / construct_transition / sample
 * (component/replay.py:75-90, 105-110, 112-140, 92-103)
 * frames: uint8 [capacity][row_bytes]  (row_bytes = 84*84 for Atari frames, 4*state_dim for f32 features)
 * action: int32 [capacity]; reward: float64 [capacity] (the reference keeps python floats); mask: int32
 * ------------------------------------------------------------------------------------------- */

/* feed n items (staged on the device in new_*) at the ring cursor; updates ring_state[0..1].
 * reference_quirk != 0 reproduces replay.py:87 (a multi-item feed into a FULL ring writes every item to
 * the slot the call started at); 0 writes each item to its own slot. */
int b2rl_replay_feed(uint8_t* frames, int32_t* action, double* reward, int32_t* mask, int64_t* ring_state,
                     int64_t row_bytes, const uint8_t* new_frames, const int32_t* new_action,
                     const double* new_reward, const int32_t* new_mask, int32_t n, int32_t reference_quirk,
                     void* stream);

/* choose B valid ring indices in candidate-stream order (replay.py:96-100).  candidates: int64 [n_cand] drawn
 * like np.random.randint(0,size) (parity mode) or NULL -> Philox4x32-10 (seed, ring_state[4]) draws n_cand
 * candidates on the device and advances the counter.  idx_out: int64 [B].  status_out: int32 [2] =
 * {accepted (== B on success, < B if the stream ran dry), candidates consumed}. */
int b2rl_replay_select_uniform(int64_t* ring_state, const int64_t* candidates, int32_t n_cand, uint64_t seed,
                               int32_t history, int32_t n_step, int32_t B, int64_t* idx_out, int32_t* status_out,
                               void* stream);

/* b2rl_replay_select_uniform + the action / n-step reward / mask of the chosen indices in the same launch (exactly the
 * scalar outputs of b2rl_replay_gather, same rounding): the sample of a consumer that reads the frame stacks from the
 * ring itself (K1).  At least one *_out must be non-NULL; a NULL one is skipped. */
int b2rl_replay_select_uniform_scalars(int64_t* ring_state, const int64_t* candidates, int32_t n_cand, uint64_t seed,
                                       int32_t history, int32_t n_step, int32_t B, int64_t* idx_out, int32_t* status_out,
                                       const int32_t* action, const double* reward, const int32_t* mask, double discount,
                                       int64_t* action_out, float* reward_out, float* mask_out, void* stream);

/* construct_transition for B indices (replay.py:112-140): frame-stack gather + n-step return.
 * out_dtype B2RL_U8: raw stacks [B][history][row_bytes] (lut must be NULL, layout 0).
 * converted dtypes (F16/BF16/F32): value = lut[v] (float32 [256] table, e.g. float32(float64(v)/255) = the reference's
 * ImageNormalizer + tensor() rounding) or, with lut == NULL, the integer v itself (exact; the consumer folds the scale
 * into its weights).  layout 0 = [B][history][row_bytes] (NCHW), 1 = [B][row_bytes][history] (NHWC),
 * 2 = space-to-depth by 4 over frames of width frame_w: [B][H/4][W/4][history*16], channel = f*16 + dy*4 + dx.
 * action_out int64 [B]; reward_out float32 [B] (float64 n-step sum rounded once, as tensor() does,
 * utils/torch_utils.py:23); mask_out float32 [B].  Any *_out may be NULL to skip it. */
int b2rl_replay_gather(const uint8_t* frames, const int32_t* action, const double* reward, const int32_t* mask,
                       int64_t capacity, int64_t row_bytes, const int64_t* idx, int32_t B, int32_t history,
                       int32_t n_step, double discount, const float* lut, int32_t out_dtype, int32_t layout,
                       int32_t frame_w, void* state_out, void* next_out, int64_t* action_out, float* reward_out,
                       float* mask_out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Sum tree in HBM -- SumTree (utils/sum_tree.py:6-67) + PrioritizedReplay (component/replay.py:152-196)
 * tree: float64 [2*capacity-1] array heap, leaves at [capacity-1, 2*capacity-2]; pending: uint8 [capacity]
 * (the reference's pending_idx set, indexed by data index); max_priority: float64 [1] on the device.
 * All arithmetic is sequential-order float64, bit-identical to the reference.
 * ------------------------------------------------------------------------------------------- */

/* n x SumTree.add(max_priority) at the tree write cursor ring_state[3] (replay.py:160-162, sum_tree.py:39-51). */
int b2rl_sumtree_add(double* tree, uint8_t* pending, int64_t capacity, int64_t* ring_state, const double* max_priority,
                     int32_t n, double* scratch /* 16*n bytes */, void* stream);

/* PrioritizedReplay.sample index part (replay.py:167-186): stratified descents with s_i = seg*i +
 * (seg*(i+1) - seg*i) * u_i (CPython random.uniform), sum_tree.py:23-33 descent rule, validity filter in batch
 * order, back-fill.  uniforms: float64 [B] in [0,1) or NULL (Philox, 53-bit).  fills: int64 [B] positions for
 * the back-fill draws (used modulo the current list length) or NULL (Philox).
 * Philox draws: u_i = u53 at ring_state[4] + i (stream 2), back-fill k = below(len) at ring_state[4] + B + k (stream 3);
 * ring_state[4] advances by 2B unless both uniforms and fills are given.  history must be in [1, capacity].
 * Outputs: tree_idx int64 [B], data_idx int64 [B], sampling_prob float64 [B] (= p / total), status int32[2] =
 * {valid before back-fill, 0}.  With no valid draw (status[0] == 0, where the reference's random.choice raises) every
 * row gets data index history - 1, its leaf and that leaf's p / total, so that consumers reading frames through the
 * outputs without a host check stay inside the ring. */
int b2rl_sumtree_sample(const double* tree, uint8_t* pending, int64_t capacity, int64_t* ring_state,
                        const double* uniforms, const int64_t* fills, uint64_t seed, int32_t history, int32_t n_step,
                        int32_t B, int64_t* tree_idx_out, int64_t* data_idx_out, double* sampling_prob_out,
                        int32_t* status_out, void* stream);

/* SumTree.get(s) for B explicit prefix values (sum_tree.py:63-67): tree_idx_out int64 [B], priority_out float64 [B];
 * marks the leaves pending. */
int b2rl_sumtree_get(const double* tree, uint8_t* pending, int64_t capacity, const double* prefix, int32_t B,
                     int64_t* tree_idx_out, double* priority_out, void* stream);

/* PrioritizedReplay.update_priorities (replay.py:193-196): for i in batch order: max_priority = max(.., p_i);
 * SumTree.update(tree_idx_i, p_i) honouring the pending guard (sum_tree.py:54-60).  priority: float32 [B]
 * (to_np of an fp32 tensor, DQN_agent.py:121-123).  scratch: 16*B bytes. */
int b2rl_sumtree_update(double* tree, uint8_t* pending, int64_t capacity, const int64_t* tree_idx,
                        const float* priority, int32_t B, double* max_priority, void* scratch, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused target/loss kernels.  Each computes the reference's per-sample loss tensor, the reduced scalar and
 * dLoss/d(network output) in ONE launch.  is_prob (float32 [B], tensor(sampling_prob)) != NULL switches on
 * the PER block of DQN_agent.py:120-127: priority = (|loss|+eps)^alpha ; w = (B*P+1e-6)^-beta / max ;
 * loss *= w before reduce_loss.  priority_out float32 [B] may be NULL when is_prob is NULL.
 * ------------------------------------------------------------------------------------------- */

/* DQNAgent.compute_loss + reduce_loss (DQN_agent.py:78-99): delta = r + gamma_n*q_next*mask - q[a];
 * loss = mean(0.5*(delta*w)^2).  q_next_online != NULL selects double-Q.  dq_out [B][A] receives dLoss/dq. */
int b2rl_dqn_loss(const float* q, const float* q_next_target, const float* q_next_online, const int64_t* action,
                  const float* reward, const float* mask, float gamma_n, int32_t B, int32_t A,
                  const float* is_prob, float beta, float eps, float alpha,
                  float* delta_out, float* priority_out, float* loss_out, float* dq_out,
                  const float* beta_dev /* optional device scalar overriding beta (CUDA-graph replays) */, void* stream);

/* NStepDQNAgent's target and loss (NStepDQN_agent.py:56-63) in one launch, for a rollout of T env steps x N workers with
 * rows t-major (row i = t*N + n): q [T*N][A] (online, s_0..s_{T-1}), q_boot [N][A] (target, s_T), action [T*N] int64 in
 * [0, A), reward / mask [T*N].  ret_t = r_t + discount*m_t*ret_{t+1} from ret_T = max_a q_boot; delta = ret - q[a];
 * loss_out[0] = 0.5*mean(delta^2); gq_out [T*N][A] = dloss/dq (-delta/(T*N) at the taken action, 0 elsewhere).  ret_out,
 * delta_out [T*N], loss_out and gq_out may each be NULL.  Limits: T >= 1, N >= 1, 1 <= A <= 32, T*N <= 2^24.  partial:
 * float [b2rl_nstep_q_loss_ctas(N)] scratch; counter: int32, zero-initialised once (the kernel re-arms it).  The loss is
 * reduced in a fixed order: the same inputs give the same bits. */
int b2rl_nstep_q_loss_ctas(int32_t N);
int b2rl_nstep_q_loss(const float* q, const float* q_boot, const int64_t* action, const float* reward, const float* mask,
                      float discount, int32_t T, int32_t N, int32_t A, float* ret_out, float* delta_out, float* loss_out,
                      float* gq_out, float* partial, int32_t* counter, void* stream);

/* CategoricalDQNAgent.compute_loss + reduce_loss (CategoricalDQN_agent.py:60-89).  log_prob [B][A][N] (online, s),
 * prob_next_target / prob_next_online [B][A][N] (online NULL -> not double).  kl_out [B], loss_out [1] = mean,
 * dlogp_out [B][A][N] = dLoss/dlog_prob.  target_prob_out [B][N] optional (NULL to skip). */
int b2rl_c51_loss(const float* log_prob, const float* prob_next_target, const float* prob_next_online,
                  const int64_t* action, const float* reward, const float* mask, float gamma_n, float v_min,
                  float v_max, int32_t B, int32_t A, int32_t N, const float* is_prob, float beta, float eps,
                  float alpha, float* kl_out, float* priority_out, float* loss_out, float* dlogp_out,
                  float* target_prob_out, int32_t* counter /* int32 scratch [1], zero on first use */,
                  const float* beta_dev /* optional device scalar overriding beta */, void* stream);

/* QuantileRegressionDQNAgent.compute_loss + reduce_loss (QuantileRegressionDQN_agent.py:55-77).
 * quantile / quantile_next [B][A][N].  vec_out [N] = the reference's per-TARGET-quantile vector, loss_out = its
 * mean, dquant_out [B][A][N].  partial: float32 scratch [B][N]; counter: int32 scratch [1], zero on first use. */
int b2rl_qr_loss(const float* quantile, const float* quantile_next, const int64_t* action, const float* reward,
                 const float* mask, float gamma_n, float kappa, int32_t B, int32_t A, int32_t N, float* vec_out,
                 float* loss_out, float* dquant_out, float* partial, int32_t* counter,
                 const float* grad_weight /* float32 [N] = dLoss/dvec / B, or NULL for the mean (1/(B*N)); with
                 partial == NULL only the gradient is computed */, void* stream);

/* ---------------------------------------------------------------------------------------------
 * On-policy: GAE backward recurrence (A2C_agent.py:43-53 == PPO_agent.py:51-61) and the losses.
 * reward, mask: [T][N]; value: [T+1][N]; adv_out, ret_out: [T][N].
 * mode 0 = sequential per env (bit-identical to the reference loop); mode 1 = warp segmented scan
 * (same recurrence re-associated; <= 1e-5 relative).  use_gae == 0 gives adv = ret - v (A2C_agent.py:46-47).
 * ------------------------------------------------------------------------------------------- */
int b2rl_gae(const float* reward, const float* mask, const float* value, float discount, float tau, int32_t T,
             int32_t N, int32_t use_gae, int32_t mode, float* adv_out, float* ret_out, void* stream);

/* advantage normalisation of PPO_agent.py:66: (adv - mean) / std, unbiased std, no epsilon; in place, M elements. */
int b2rl_normalize_advantage(float* adv, int32_t M, void* stream);

/* PPO clipped surrogate for one minibatch of M rows (PPO_agent.py:77-86).  Inputs [M]: log_pi_a (new), entropy,
 * v, old_log_pi_a, advantage, ret.  out[0]=policy_loss out[1]=value_loss out[2]=approx_kl.
 * Gradients: dlogp_out, dent_out = d policy_loss / d(log_pi_a, entropy); dv_out = d value_loss / dv. */
int b2rl_ppo_loss(const float* log_pi_a, const float* entropy, const float* v, const float* old_log_pi_a,
                  const float* advantage, const float* ret, float clip, float entropy_weight, int32_t M, float* out,
                  float* dlogp_out, float* dent_out, float* dv_out, void* stream);

/* A2C objective (A2C_agent.py:55-62): -mean(logp*adv) - ew*mean(ent) + vw*0.5*mean((ret-v)^2) over M rows.
 * out (float32 [4]) = {objective, policy_loss, value_loss, entropy_loss}. */
int b2rl_a2c_loss(const float* log_pi_a, const float* entropy, const float* v, const float* advantage,
                  const float* ret, float entropy_weight, float value_loss_weight, int32_t M, float* out,
                  float* dlogp_out, float* dent_out, float* dv_out, void* stream);

/* A2CAgent's GAE and objective (A2C_agent.py:43-62) with the gradient to the actor-critic head, in one launch, for a rollout of
 * T env steps x N workers: head [(T+1)*N][A+1] = (logits, v) rows t-major (b2rl_ac_head_fwd; rows T*N.. the final states),
 * action [T*N] int64 in [0, A), reward / mask [T*N].  adv_out / ret_out [T*N] (may be NULL) are the bits of b2rl_gae mode 0.
 * loss_out[0] = -mean(lp_a*adv) - ew*mean(H) + vw*0.5*mean((ret-v)^2) (may be NULL).  geff_out [(T+1)*N][33] = the loss's
 * gradient with respect to the head's outputs in b2rl_head_bwd_geff_relu's layout (columns 0..A; the final rows zero).
 * Limits: T >= 1, N >= 1, 1 <= A <= 31, (T+1)*N <= 2^24.  partial: float [3 * b2rl_a2c_rollout_loss_ctas(N)] scratch; counter:
 * int32, zero-initialised once (the kernel re-arms it).  The loss is reduced in a fixed order: the same inputs give the same
 * bits. */
int b2rl_a2c_rollout_loss_ctas(int32_t N);
int b2rl_a2c_rollout_loss(const float* head, const int64_t* action, const float* reward, const float* mask, float discount,
                          float gae_tau, int32_t use_gae, float entropy_weight, float value_loss_weight, int32_t T, int32_t N,
                          int32_t A, float* adv_out, float* ret_out, float* loss_out, float* geff_out, float* partial,
                          int32_t* counter, void* stream);

/* PPOAgent's rollout statistics (PPO_agent.py:44-61, shared_repr) from the (logits, v) rows the actor's head launches stored:
 * head [(T+1)*N][A+1] rows t-major (rows T*N.. the final states), action [T*N] int64, reward / mask [T*N].  logp_out [T*N] =
 * log_softmax(logits)[action] (the old log-probabilities), adv_out / ret_out [T*N] the bits of b2rl_gae mode 0 (before
 * b2rl_normalize_advantage).  Limits: T >= 1, N >= 1, 1 <= A <= 31, (T+1)*N <= 2^24. */
int b2rl_ppo_rollout_prep(const float* head, const int64_t* action, const float* reward, const float* mask, float discount,
                          float gae_tau, int32_t use_gae, int32_t T, int32_t N, int32_t A, float* logp_out, float* adv_out,
                          float* ret_out, void* stream);

/* PPO's clipped surrogate for one minibatch of a categorical actor-critic head (PPO_agent.py:77-92, shared_repr): head [B][A+1]
 * = (logits, v) of the minibatch, idx [B] int64 its rows of the rollout arrays action (int64) / old_logp / adv / ret.
 * geff_out [B][33] = d(policy_loss + value_loss) / d(head outputs) in b2rl_head_bwd_geff_relu's layout (columns 0..A), with
 * b2rl_ppo_loss's tie and boundary rules; stats_out[0..2] = policy_loss, value_loss, approx_kl.  partial: float
 * [4 * b2rl_ppo_cat_loss_ctas(B)] scratch; counter: int32, zero-initialised once (the kernel re-arms it).  The statistics are
 * reduced in a fixed order: the same inputs give the same bits.  Limits: 1 <= B <= 2^24, 1 <= A <= 31. */
int b2rl_ppo_cat_loss_ctas(int32_t B);
int b2rl_ppo_cat_loss(const float* head, const int64_t* idx, const int64_t* action, const float* old_logp, const float* adv,
                      const float* ret, float clip, float entropy_weight, int32_t B, int32_t A, float* geff_out,
                      float* stats_out, float* partial, int32_t* counter, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Multi-tensor optimizer step with global-norm clip (DQN_agent.py:132-134; examples.py:67-68,139,204):
 * flat float32 views of all parameters / gradients (one contiguous arena, n elements).
 * clip_grad_norm_(max_norm) then RMSprop(centered) or Adam, torch semantics.  norm_scratch: 2048 bytes, zero on first
 * use; after the call float32 norm_scratch[0] = total gradient norm (what clip_grad_norm_ returns).
 * bf16_shadow (optional, uint16 [n]): refreshed copy of the updated parameters in bf16.
 * ------------------------------------------------------------------------------------------- */
int b2rl_clip_rmsprop(float* param, const float* grad, float* square_avg, float* grad_avg, int64_t n,
                      float max_norm, float lr, float alpha, float eps, int32_t centered, float grad_scale,
                      void* norm_scratch, uint16_t* bf16_shadow, void* stream);
int b2rl_clip_adam(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float max_norm,
                   float lr, float beta1, float beta2, float eps, int64_t* step_dev, float grad_scale,
                   void* norm_scratch, uint16_t* bf16_shadow, void* stream);
/* b2rl_clip_adam taken only if the DEVICE scalar *gate <= gate_max (nothing is touched otherwise): the KL gate of the PPO
 * actor step, `if approx_kl <= 1.5 * target_kl:` PPO_agent.py:94, decided on the device so the update can be graph-captured */
int b2rl_clip_adam_gated(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float max_norm,
                         float lr, float beta1, float beta2, float eps, int64_t* step_dev, float grad_scale,
                         void* norm_scratch, uint16_t* bf16_shadow, const float* gate, float gate_max, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Dense-layer epilogues (network_bodies.py:27-33,70-73: y = relu(layer(x))), bf16 activations [rows][C] (NHWC
 * flattened), fp32 bias.  Forward: y = act(y + bias) in place.  Backward: gx = gy * (y > 0) (gx may alias gy or be
 * NULL) and dbias[c] = sum over rows of gx (block partials + fp32 atomics; dbias is zeroed by the call).  partial /
 * counter: unused (kept for ABI stability), may be NULL.
 * ------------------------------------------------------------------------------------------- */
int b2rl_bias_act_bf16(uint16_t* y, const float* bias, int64_t rows, int32_t C, int32_t relu, void* stream);
/* same epilogue for a split-K GEMM result: y(bf16) = act(x(fp32) + bias) */
int b2rl_bias_act_f32_to_bf16(const float* x, const float* bias, uint16_t* y, int64_t rows, int32_t C, int32_t relu,
                              void* stream);
/* row_map re-lays the gradient out for the next GEMM of the grid-convolution stack (csrc/gemm.cu): 0 identity;
 * 1: compact V x V rows per image -> G x G grid rows; 2: space-to-depth(2) rows (4 groups of C channels per row) ->
 * G x G grid rows.  With a map, `rows` counts the DESTINATION rows (batch*G*G) and gx is [rows][C]; padding rows of the
 * grid are written as zeros. */
int b2rl_act_bwd_bias_grad_bf16(const uint16_t* gy, const uint16_t* y, int64_t rows, int32_t C, int32_t relu,
                                uint16_t* gx, float* dbias, float* partial, int32_t* counter, int32_t row_map, int32_t G,
                                int32_t V, void* stream);

/* ---------------------------------------------------------------------------------------------
 * wgmma GEMM for the dense contractions (network_bodies.py:27-33, network_heads.py:18-21):
 *   D[M,N] (+)= A[M,K] * B[N,K]^T, bf16 operands, fp32 accumulation in registers, TMA-fed.
 * a_mn / b_mn = 0: operand stored row-major [rows][K] (K-major); 1: stored row-major [K][rows] (MN-major) -- weight
 * gradients dW = g^T x read both operands as stored, nothing is transposed in memory.  lda/ldb/ldd: row strides in
 * elements (operands: multiples of 8).  out_mode 0: bf16 store, 1: fp32 store, 2: fp32 atomicAdd into D (required for
 * splits > 1; D must be pre-zeroed or hold the value to accumulate into).  bias (fp32 [N]) and relu are fused into the
 * epilogue.  block_n in {32, 64, 128} = output tile width (tile height is 128).
 * ------------------------------------------------------------------------------------------- */
int b2rl_gemm_bf16(const uint16_t* A, int32_t a_mn, int64_t lda, const uint16_t* B, int32_t b_mn, int64_t ldb, void* D,
                   int64_t ldd, int32_t M, int32_t N, int32_t K, const float* bias, int32_t relu, int32_t out_mode,
                   int32_t splits, int32_t block_n, void* stream);

/* Convolution over a G x G position grid as a shifted-row GEMM, no im2col (csrc/gemm.cu header).
 * mode 0 (forward / dgrad): D[r,:] = sum_taps X[r + shift(tap), :] * W[:, tap*C .. tap*C + C]^T, X bf16 [rows][C] (C % 64
 *   == 0), W bf16 [n_out][taps*C]; shift(tap) = shift_sign * ((tap / taps_x) * grid_w + tap % taps_x); rows off the grid
 *   read zeros.  out_map 1 writes the valid V x V positions of the G grid in space-to-depth(2) layout
 *   ([batch*(V/2)^2][4*n_out], ldd = 4*n_out), out_map 2 compacts them to [batch*V*V][n_out].
 * mode 1 (wgrad): D[n, tap*C + c] += sum_r Gr[r, n] * X[r + shift(tap), c], Gr bf16 [rows][n_out] passed as W_or_G,
 *   D fp32 [n_out][taps*C] (out_mode 2, atomic accumulation over `splits` K slices). */
/* forward / dgrad calls use the slab kernel (one activation slab per tile, resident weights) unless switched off */
void b2rl_set_conv_slab(int32_t on);
/* CTA budget of the following launches of the slab convolution kernel (forward / dgrad), the plain GEMM (b2rl_gemm_bf16,
 * b2rl_gemm_bwd_bf16, b2rl_gemm_splitk_bf16) and the convolution weight gradient (b2rl_conv_wgrad_partials): each sizes its
 * grid to at most `ctas` CTAs (the persistent kernels loop over more tiles per CTA, the weight gradient writes fewer split-K
 * partials, the plain GEMM launches without clusters; a weight gradient keeps at least one CTA per 128-column group) instead
 * of up to one per SM, so that kernels on two parallel graph branches hold disjoint SMs.  0 (the default): up to one CTA per
 * SM.  The setting is read on the host at launch time; per-tile arithmetic does not depend on it.
 * b2rl_last_grid_ctas: the CTAs of the last launch of those launchers (summed over the kernels of one call). */
int b2rl_set_cta_budget(int32_t ctas);
int b2rl_last_grid_ctas(int32_t* ctas);
int b2rl_conv_gemm_bf16(int32_t mode, const uint16_t* X, int64_t rows, int32_t C, const uint16_t* W_or_G, int32_t n_out,
                        int32_t taps, int32_t taps_x, int32_t grid_w, int32_t shift_sign, void* D, int64_t ldd,
                        const float* bias, int32_t relu, int32_t out_mode, int32_t out_map, int32_t G, int32_t V,
                        int32_t splits, int32_t block_n, void* stream);

/* Dual launches: the same GEMM / convolution for TWO independent operand sets of identical shape (online network on the
 * sampled states, target network on the next states -- DQN_agent.py:84-99 evaluates both every update) in ONE grid;
 * half of the CTAs work on each set, so the per-kernel fixed cost (launch, prologue, weight load, drain) is paid once. */
int b2rl_conv_gemm_dual_bf16(const uint16_t* X, const uint16_t* X2, int64_t rows, int32_t C, const uint16_t* W,
                             const uint16_t* W2, int32_t n_out, int32_t taps, int32_t taps_x, int32_t grid_w,
                             int32_t shift_sign, void* D, void* D2, int64_t ldd, const float* bias, const float* bias2,
                             int32_t relu, int32_t out_mode, int32_t out_map, int32_t G, int32_t V, int32_t block_n,
                             void* stream);
int b2rl_gemm_dual_bf16(const uint16_t* A, const uint16_t* A2, int64_t lda, const uint16_t* B, const uint16_t* B2,
                        int64_t ldb, void* D, void* D2, int64_t ldd, int32_t M, int32_t N, int32_t K, const float* bias,
                        const float* bias2, int32_t relu, int32_t out_mode, int32_t block_n, void* stream);

/* Backward GEMMs with the element-wise backward pass fused into the epilogue (replaces b2rl_act_bwd_bias_grad_bf16 between the
 * dgrad GEMMs of NatureConvBody).  mask: the saved forward activation (bf16) in the GEMM's own output coordinates,
 * [M][mask_ld] -- the ReLU gradient D = mask > 0 ? D : 0; dbias: fp32 [dbias_mod], receives (atomically, zero it first) the
 * column sums of the masked output, index = column % dbias_mod (dbias_mod 0: index = column, dbias is [N]) = the bias gradient
 * of the layer below; sub_c: channels per
 * position for the scatter maps.  out_map 3: rows are space-to-depth(2) positions of a (V/2)^2 grid with 4 x sub_c columns ->
 * rows of the G x G grid; out_map 4: rows are images with V*V x sub_c columns -> rows of the G x G grid.  Grid rows that no
 * tile covers are left untouched (keep the destination zeroed). */
typedef struct {
  const uint16_t* mask;
  int64_t mask_ld;
  float* dbias;
  int32_t dbias_mod;
  int32_t sub_c;
} b2rl_bwd_epilogue;
int b2rl_conv_gemm_bwd_bf16(const uint16_t* G_rows, int64_t rows, int32_t C, const uint16_t* W, int32_t n_out, int32_t taps,
                            int32_t taps_x, int32_t grid_w, void* D, int64_t ldd, int32_t out_map, int32_t G, int32_t V,
                            const b2rl_bwd_epilogue* ext, int32_t block_n, void* stream);
int b2rl_gemm_bwd_bf16(const uint16_t* A, int64_t lda, const uint16_t* B, int32_t b_mn, int64_t ldb, void* D, int64_t ldd,
                       int32_t M, int32_t N, int32_t K, int32_t out_map, int32_t G, int32_t V,
                       const b2rl_bwd_epilogue* ext, int32_t block_n, void* stream);

/* NatureConvBody weights (network_bodies.py:13-20) between the reference's parameter layouts and the tap-major bf16
 * operands of the grid-GEMM stack: w1 [32,c1,8,8] -> w1f [32][4 taps][16*c1] (times `scale` = ImageNormalizer's 1/255);
 * w2 [64,32,4,4] -> w2f [64][4][128], w2d [128][4][64]; w3 [64,64,3,3] -> w3f [64][9][64], w3d [64][9][64];
 * w4 [n4, 64*7*7 in (c,h,w) order] -> w4p [n4][(h,w,c)].  unpack maps fp32 gradients in the GEMM layouts back and ADDS
 * them (and the four bias gradients) into the reference-layout .grad buffers. */
int b2rl_nature_pack_weights(const float* w1, const float* w2, const float* w3, const float* w4, int32_t c1, int32_t n4,
                             float scale, uint16_t* w1f, uint16_t* w2f, uint16_t* w2d, uint16_t* w3f, uint16_t* w3d,
                             uint16_t* w4p, void* stream);
int b2rl_nature_unpack_grads(const float* g1f, const float* g2f, const float* g3f, const float* g4p, const float* db1,
                             const float* db2, const float* db3, const float* db4, int32_t c1, int32_t n4, float scale,
                             float* gw1, float* gw2, float* gw3, float* gw4, float* gb1, float* gb2, float* gb3,
                             float* gb4, int32_t p1, int32_t p2, int32_t p3 /* split-K partial counts of g1f/g2f/g3f, stored
                             n_out*K floats apart (b2rl_conv_wgrad_partials); 1 = plain */, void* stream);

/* Narrow value heads (VanillaNet / DuelingNet, network_heads.py:11-37) on the bf16 features phi [B][K] of the fused body:
 * forward q [B][A] (fp32) = phi Wa^T + ba, or with Wv/bv != NULL the dueling combine q = v + adv - mean(adv);
 * backward from gq [B][A]: gphi [B][K] (bf16), and gWa [A][K], gba [A], gWv [K], gbv [1] ACCUMULATED (atomics) into the
 * given fp32 buffers.  0 < A < 32. */
int b2rl_head_fwd(const uint16_t* phi, const float* Wa, const float* ba, const float* Wv, const float* bv, int32_t B,
                  int32_t K, int32_t A, float* q, void* stream);
int b2rl_head_bwd(const float* gq, const uint16_t* phi, const float* Wa, const float* Wv, int32_t B, int32_t K, int32_t A,
                  uint16_t* gphi, float* gWa, float* gba, float* gWv, float* gbv, void* stream);
/* b2rl_head_bwd when phi = relu(layer(.)) (NatureConvBody's fc4 output): gphi is masked (0 where phi <= 0) and
 * relu_colsum[K] (fp32, zero it first) receives the column sums of the masked gphi = that layer's bias gradient. */
int b2rl_head_bwd_relu(const float* gq, const uint16_t* phi, const float* Wa, const float* Wv, int32_t B, int32_t K, int32_t A,
                       uint16_t* gphi, float* gWa, float* gba, float* gWv, float* gbv, float* relu_colsum, void* stream);
/* Actor-critic head (CategoricalActorCriticNet with DummyBody actor / critic bodies): out [B][A+1] (fp32) = (phi Wa^T + ba,
 * phi Wv^T + bv), Wa = fc_action [A][K], Wv = fc_critic [1][K].  counter != NULL: the action of row b is also drawn into
 * action_out[b] (int64) -- the inverse CDF of softmax(logits) on Philox u24(seed, *counter + b, stream 13), as
 * b2rl_a2c_actor_step draws it -- and *counter advances by B once every CTA has read it (ticket: int32, zero-initialised once;
 * the kernel re-arms it).  0 < A <= 31, K % 8 == 0, phi and the weights 16-byte aligned. */
int b2rl_ac_head_fwd(const uint16_t* phi, const float* Wa, const float* ba, const float* Wv, const float* bv, int32_t B,
                     int32_t K, int32_t A, float* out, uint64_t seed, int64_t* counter, int64_t* action_out, int32_t* ticket,
                     void* stream);
/* b2rl_head_bwd_relu from effective output gradients geff [B][33] (column n < A: output n of Wa; column A: Wv's output when
 * Wv != NULL) instead of gq -- the actor-critic head's backward from b2rl_a2c_rollout_loss's geff_out. */
int b2rl_head_bwd_geff_relu(const float* geff, const uint16_t* phi, const float* Wa, const float* Wv, int32_t B, int32_t K,
                            int32_t A, uint16_t* gphi, float* gWa, float* gba, float* gWv, float* gbv, float* relu_colsum,
                            void* stream);

/* Convolution weight gradient as split-K partials (no atomics): partial i of *n_partials_host (<= one per SM, written on the
 * HOST, deterministic for given shapes) is stored at partials + i * n_out*taps*C floats. */
int b2rl_conv_wgrad_partials(const uint16_t* X, int64_t rows, int32_t C, const uint16_t* G, int32_t n_out, int32_t taps,
                             int32_t taps_x, int32_t grid_w, float* partials, int32_t* n_partials_host, void* stream);
/* The same partials for conv2 (C 128, 2 x 2 taps) and conv3 (C 64, 3 x 3 taps), n_out 64: one CTA computes every tap of its
 * 128-row k-blocks from one load of each operand.  One partial per CTA: at most one per SM, or the CTA budget. */
int b2rl_conv_taps_wgrad_partials(const uint16_t* X, int64_t rows, int32_t C, const uint16_t* G, int32_t n_out, int32_t taps,
                                  int32_t taps_x, int32_t grid_w, float* partials, int32_t* n_partials_host, void* stream);

/* K1 -- conv1 of NatureConvBody straight from the uint8 replay ring: the fused gather -> normalize -> conv1 of the
 * reference chain replay.py:124-134 (frame-stack gather) -> normalizer.py:58-61 -> network_bodies.py:27, with no
 * materialised batch.  frames: ring [capacity][row_bytes] uint8 (16-byte aligned rows); idx: int64 [batch] sampled ring indices; first: ring row of
 * the oldest stacked frame relative to idx[b] (-(history-1) for the state, n_step-(history-1) for the next state);
 * history must be 4 (4 frames x 16 pixels = the 64 channels of one space-to-depth(4) position).  The pixels enter as
 * exact integers 0..255; ImageNormalizer's 1/255 is folded into W [n_out][4 taps * 64] (b2rl_nature_pack_weights).
 * fwd: D = relu(conv1 + bias) over rows (b, gy, gx) of the (frame_w/4)^2 grid, bf16, output row maps of
 * b2rl_conv_gemm_bf16; relu must be 1, n_out a multiple of 8, D 16-byte aligned and ldd a multiple of 8 (the slab
 * kernel's one store form: whole 16-byte column groups).  wgrad_partials: split-K partials of dW[n][tap*64+c] = sum_r G[r][n] * x[r + shift(tap)][c],
 * contract of b2rl_conv_wgrad_partials; n_out must be 32. */
int b2rl_conv1_u8_fwd(const uint8_t* frames, int64_t capacity, const int64_t* idx, int32_t first, int64_t row_bytes,
                      int32_t frame_w, int32_t batch, int32_t history, const uint16_t* W, int32_t n_out, void* D, int64_t ldd,
                      const float* bias, int32_t relu, int32_t out_map, int32_t V, void* stream);
int b2rl_conv1_u8_wgrad_partials(const uint8_t* frames, int64_t capacity, const int64_t* idx, int32_t first, int64_t row_bytes,
                                 int32_t frame_w, int32_t batch, int32_t history, const uint16_t* G_rows, int32_t n_out, float* partials,
                                 int32_t* n_partials_host, void* stream);
/* conv1's weight-gradient partials from the materialised bf16 stacks X [rows][64] (the space-to-depth(4) grid matrix,
 * grid_w x grid_w positions per image), G_rows [rows][32]: the same partition, partials and bits as
 * b2rl_conv1_u8_wgrad_partials on the ring the stacks came from.  n_out must be 32. */
int b2rl_conv1_wgrad_partials(const uint16_t* X, int64_t rows, int32_t grid_w, const uint16_t* G_rows, int32_t n_out,
                              float* partials, int32_t* n_partials_host, void* stream);
/* The online forward on the state and the target forward on the next state (n_step 1) in ONE launch: D = act(conv1_W(s) +
 * bias) and D2 = act(conv1_W2(s') + bias2), s the stacks idx[b] + first .. + history - 1 and s' the stacks one ring row
 * later, read together from the history + 1 ring rows they span.  W, W2 [32][4 taps * 64]; D, D2 as D of b2rl_conv1_u8_fwd
 * with n_out 32 (row stride ldd); relu must be 1.  Bit-identical to b2rl_conv1_u8_fwd(first, W, D, bias) and (first + 1, W2, D2, bias2).
 * history 4 and 84 x 84 frames only. */
int b2rl_conv1_u8_fwd_pair(const uint8_t* frames, int64_t capacity, const int64_t* idx, int32_t first, int64_t row_bytes,
                           int32_t frame_w, int32_t batch, int32_t history, const uint16_t* W, const uint16_t* W2, void* D,
                           void* D2, int64_t ldd, const float* bias, const float* bias2, int32_t relu, int32_t out_map, int32_t V,
                           void* stream);
/* Profiling hook of every convolution slab launch (the two conv1 forwards above, the conv_gemm forwards and dgrads) and of
 * conv1's weight gradient: while `clocks` (device, 12 int64, zeroed by the caller) is set, every launch adds per-role clock64()
 * cycle sums to it -- CTA run, producer waits, converter waits (slab, pixels) and conversion, MMA waits for the slab, MMA
 * chain, MMA waits for a free staging tile, accumulator staging, epilogue waits for a staged half, epilogue work, tiles
 * (csrc/gemm.cu K1_CLK_*).  NULL (the default) turns it off. */
int b2rl_conv1_set_phase_clocks(int64_t* clocks);

/* D = act(A B^T + bias) (bf16 out) in one launch: K split over the `splits` CTAs (1, 2, 4 or 8; 0: chosen from the shape) of
 * a thread-block cluster per output tile, the partials summed in distributed shared memory in a fixed order (deterministic),
 * bias / ReLU in the same epilogue (fc4 of NatureConvBody, network_bodies.py:33).  A [M][K], B [N][K] bf16 K-major. */
int b2rl_gemm_splitk_bf16(const uint16_t* A, int64_t lda, const uint16_t* B, int64_t ldb, void* D, int64_t ldd, int32_t M,
                          int32_t N, int32_t K, const float* bias, int32_t relu, int32_t splits, int32_t block_n, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Tail of one gradient update for a NatureConvBody network on the wgmma path (csrc/tail.cu):
 * loss.backward()'s last step + clip_grad_norm_ + optimizer.step (DQN_agent.py:131-134) in two launches.
 * Work is described by unit tables (int32 x 4 per unit: arena offset, length, kind, row | segment << 16;
 * kinds 0 plain, 1-4 one output row (or 256-element segment of it) of conv1 / conv2 / conv3 / fc4 weights,
 * 5-8 their biases), built once by the host (deeprl_b200/network/tail.py).
 *
 * grad_reduce: sums the split-K partials of the conv weight gradients (g1p/g2p/g3p: [p][n_out][taps*C] fp32),
 *   maps all four weight gradients from the GEMM layouts to the reference layouts and WRITES them into the flat
 *   gradient arena, moves the bias gradients there (db1..db4 are re-zeroed), and leaves the sum of squares of the
 *   gradient elements of unit i in unit_sumsq[i] (plain units: whatever the arena already holds, e.g. the head's
 *   gradients).  step_dev (Adam) is incremented by one if not NULL.  norm_scratch != NULL: the CTA that finishes last adds the
 *   unit partials (fixed order) and leaves clip_grad_norm_'s total norm and coefficient there, as b2rl_grad_norm does.
 * fused_opt: clip coefficient from the unit partials (NULL: from norm_scratch, see b2rl_grad_norm), RMSprop
 *   (opt 0 plain, 1 centered; a_ = alpha) or Adam (opt 2; a_, b_ = betas) exactly as b2rl_clip_rmsprop / b2rl_clip_adam,
 *   gradient re-zeroed when zero_grad != 0, and the updated conv / fc4 weights written to the bf16 tap-major GEMM
 *   operands of b2rl_nature_pack_weights (all six pointers, or all NULL); bf16_shadow != NULL: a bf16 copy of every updated
 *   parameter at the same arena offset (the GEMM operands of the distributional heads).
 * ------------------------------------------------------------------------------------------- */
int b2rl_nature_grad_reduce(const int32_t* units, int32_t n_units, const float* g1p, int32_t p1, const float* g2p, int32_t p2,
                            const float* g3p, int32_t p3, const float* g4p, float* db1, float* db2, float* db3, float* db4,
                            int32_t c1, int32_t n4, float scale, float* grad, float* unit_sumsq, int64_t* step_dev,
                            void* norm_scratch, float max_norm, float grad_scale, void* stream);
int b2rl_nature_fused_opt(const int32_t* units, int32_t n_units, float* param, float* grad, float* s1, float* s2, int32_t opt,
                          float lr, float a_, float b_, float eps, float max_norm, float grad_scale, const float* unit_sumsq,
                          int32_t n_sumsq, void* norm_scratch, const int64_t* step_dev, int32_t c1, int32_t n4, float scale,
                          uint16_t* w1f, uint16_t* w2f, uint16_t* w2d, uint16_t* w3f, uint16_t* w3d, uint16_t* w4p,
                          int32_t zero_grad, uint16_t* bf16_shadow, void* stream);
/* b2rl_nature_fused_opt with the learning rate on the device: lr_dev (float32) != NULL replaces lr, so a captured graph
 * follows a schedule the host writes between replays; lr_dev == NULL is b2rl_nature_fused_opt. */
int b2rl_nature_fused_opt_lr(const int32_t* units, int32_t n_units, float* param, float* grad, float* s1, float* s2, int32_t opt,
                             float lr, const float* lr_dev, float a_, float b_, float eps, float max_norm, float grad_scale,
                             const float* unit_sumsq, int32_t n_sumsq, void* norm_scratch, const int64_t* step_dev, int32_t c1,
                             int32_t n4, float scale, uint16_t* w1f, uint16_t* w2f, uint16_t* w2d, uint16_t* w3f, uint16_t* w3d,
                             uint16_t* w4p, int32_t zero_grad, uint16_t* bf16_shadow, void* stream);
/* clip_grad_norm_'s coefficient alone (torch.nn.utils.clip_grad_norm_): norm_scratch[0] = ||grad * grad_scale||,
 * norm_scratch[1] = min(max_norm / (norm + 1e-6), 1) * grad_scale. */
int b2rl_grad_norm(const float* grad, int64_t n, float grad_scale, float max_norm, void* norm_scratch, void* stream);

/* b2rl_dqn_head_fused in two launches (row kernel: one warp per batch row; then the head backward): same arguments plus
 * geff = float scratch [B][33]; scratch: int32 counter + 12 bytes padding + float [ceil(B/4)], zero-initialised once. */
int b2rl_dqn_head_two(const uint16_t* phi, const uint16_t* phi_t, const uint16_t* phi_o, const float* Wa, const float* ba,
                      const float* Wv, const float* bv, const float* Wa_t, const float* ba_t, const float* Wv_t,
                      const float* bv_t, const int64_t* action, const float* reward, const float* mask, float gamma_n, int32_t B,
                      int32_t K, int32_t A, const float* is_prob, float beta, const float* beta_dev, float eps, float alpha,
                      uint16_t* gphi, float* gWa, float* gba, float* gWv, float* gbv, float* relu_colsum, float* q_out,
                      float* delta_out, float* prio_out, float* loss_out, float* scratch, float* geff, void* stream);

/* Device-side actor step of the on-policy agents (SURVEY 8f-3; PPO_agent.py:45-50 between two task.step() calls) in one
 * launch: MeanStdNormalizer (normalizer.py:36-51 over baselines' RunningMeanStd: float64 Chan merge of the batch moments into
 * rm_mean / rm_var / rm_count -- all three NULL: no normalisation; update_stats 0: read-only -- then clip((x - mean) /
 * sqrt(var + eps), +-clip) rounded once to float32), GaussianActorCriticNet.forward (network_heads.py:173-214) with two-layer
 * tanh FCBody actor / critic bodies, and the Normal sample / log_prob / entropy.  obs [N][D]; weights in the reference's
 * nn.Linear layouts ([out][in]); z: supplied standard normals [N][A] (parity mode) or NULL -> Philox4x32-10 (seed, *counter)
 * with Box-Muller; given_action != NULL: log_prob of those actions instead of sampling.  Outputs: state_out [N][D] (normalised,
 * may be NULL), action / mean [N][A] (mean may be NULL), log_pi_a / entropy / v [N].  Limits: N <= 64, D, hidden <= 128, A <= 32. */
int b2rl_gaussian_actor_step(const float* obs, double* rm_mean, double* rm_var, double* rm_count, int32_t update_stats, double clip,
                             double eps, const float* aw1, const float* ab1, const float* aw2, const float* ab2, const float* faw,
                             const float* fab, const float* cw1, const float* cb1, const float* cw2, const float* cb2,
                             const float* fcw, const float* fcb, const float* std_param, int32_t N, int32_t D, int32_t H1,
                             int32_t H2, int32_t A, const float* z, uint64_t seed, int64_t* counter, const float* given_action,
                             float* state_out, float* action, float* log_pi_a, float* entropy, float* mean, float* v,
                             void* stream);

/* Every minibatch update of one PPO iteration (PPO_agent.py:68-99, non-shared representation; optimization_epochs x
 * rows / mini_batch_size updates) in ONE launch of one persistent thread block: per minibatch b the rows perm[b][0..mb) of the
 * rollout (state [R][D], action [R][A], old_log_pi_a / ret / advantage [R], advantage already normalised, PPO_agent.py:66) go
 * through GaussianActorCriticNet (network_heads.py:198-214: DummyBody phi, two-layer tanh FCBody actor / critic bodies,
 * mean = tanh(fc_action), std = softplus(std)), the clipped-surrogate / entropy / value losses (PPO_agent.py:79-88), the
 * backward pass, the actor Adam step iff approx_kl <= kl_gate (= 1.5 * target_kl, PPO_agent.py:94) and the critic Adam step
 * (torch.optim.Adam arithmetic).  a_* / c_*: flat arenas holding the actor's / critic's parameters, exp_avg, exp_avg_sq
 * (float32) and step count (int64 [1], device); a_off int32 [7] = element offsets of actor_body.layers.0.weight, .bias,
 * layers.1.weight, .bias, fc_action.weight, fc_action.bias, std inside the actor arenas (host array); c_off int32 [6] likewise
 * for critic_body.* and fc_critic.*.  stats float32 [4] = policy loss, value loss, approx_kl of the LAST minibatch and the
 * number of actor steps taken.  Limits: D <= 256, A <= 32, hidden <= 128, mini batch <= 128 and a multiple of 4. */
/* Profiling hook of b2rl_ppo_minibatch_updates: install (NULL: remove) a device buffer int64 [2 + 9 * n_batches] that the next
 * launches fill with clock64() of thread 0 after every phase barrier (scripts/ppo_phase_clocks.py).  The data-parallel form
 * fills [2 + 12 * n_batches] (rank 0 of the launch; scripts/ppo_dp_scaling.py). */
int b2rl_ppo_set_phase_clocks(int64_t* clocks);

/* Dynamic shared memory (bytes) b2rl_ppo_minibatch_updates needs for these sizes; it must fit the 227 KB of one SM. */
int64_t b2rl_ppo_minibatch_smem_bytes(int32_t D, int32_t A, int32_t H1, int32_t H2, int32_t mb);

int b2rl_ppo_minibatch_updates(const float* state, const float* action, const float* old_log_pi_a, const float* ret,
                               const float* advantage, int32_t D, int32_t A, int32_t H1, int32_t H2, int32_t mb,
                               const int64_t* perm, int32_t n_batches, float* a_flat, float* a_exp_avg, float* a_exp_avg_sq,
                               int64_t* a_step, const int32_t* a_off, float* c_flat, float* c_exp_avg, float* c_exp_avg_sq,
                               int64_t* c_step, const int32_t* c_off, float a_lr, float a_beta1, float a_beta2, float a_eps,
                               float c_lr, float c_beta1, float c_beta2, float c_eps, float ratio_clip, float entropy_weight,
                               float kl_gate, float* stats, void* stream);

/* Data-parallel form of b2rl_ppo_minibatch_updates: `world` ranks, each with its own rollout rows, advantage normalisation and
 * minibatch permutation; update k of every rank is ONE step on the union of the ranks' k-th minibatches.  Each rank writes
 * its gradients and loss values into its exchange region, pushes the update's sequence number into every peer's flags, waits
 * for every peer, sums the gradients over ranks 0..world-1 in order, scales them by 1/world and applies Adam (critic always,
 * actor iff the MEAN approx_kl over ranks <= kl_gate): parameters, moments and step counts stay bit-identical on every rank.
 * regions: host array [world] of device pointers to every rank's exchange region of b2rl_ppo_dp_region_bytes(a_n, c_n) bytes,
 * zero-filled once (regions[rank] is this rank's own).  a_n / c_n: arena lengths (elements).  seq_base: updates exchanged
 * before this launch (monotonic across launches; the flags are never reset).  timeout_ns: bound on the wait for one update's
 * peers; on expiry status (int64, device) gets 1 + peer + 16 * update and the launch skips its remaining updates.
 * ranks_in_launch: 1 = one process per GPU (regions mapped by b2rl_ipc_open_handle); world = all ranks as the blocks of ONE
 * cooperative launch on one device (pass rank 0): every per-rank array then holds world consecutive copies (rows rows each
 * for the rollout arrays, n_batches x mb for perm, a_n / c_n for the arenas, 1 per step count and status word, 4 per stats). */
int64_t b2rl_ppo_dp_region_bytes(int32_t a_n, int32_t c_n);
int b2rl_ppo_minibatch_updates_dp(const float* state, const float* action, const float* old_log_pi_a, const float* ret,
                                  const float* advantage, int32_t D, int32_t A, int32_t H1, int32_t H2, int32_t mb,
                                  const int64_t* perm, int32_t n_batches, float* a_flat, float* a_exp_avg, float* a_exp_avg_sq,
                                  int64_t* a_step, const int32_t* a_off, float* c_flat, float* c_exp_avg, float* c_exp_avg_sq,
                                  int64_t* c_step, const int32_t* c_off, float a_lr, float a_beta1, float a_beta2, float a_eps,
                                  float c_lr, float c_beta1, float c_beta2, float c_eps, float ratio_clip, float entropy_weight,
                                  float kl_gate, float* stats, int32_t rows, int32_t a_n, int32_t c_n, int32_t world,
                                  int32_t rank, void* const* regions, int64_t seq_base, int64_t timeout_ns, int64_t* status,
                                  int32_t ranks_in_launch, void* stream);

/* Device memory shared between processes (CUDA IPC; setup only, never on the update path): allocate + zero-fill, export a
 * 64-byte handle, map a peer's handle (peer access enabled lazily), unmap, free; peer_access_ok: *ok = 1 when device dev_a can
 * address device dev_b's memory (or dev_a == dev_b). */
/* A2CAgent.step() (A2C_agent.py:22-64) on the device for FCBody actor-critic networks: head 0 = CategoricalActorCriticNet on a
 * shared two-layer phi_body (shared 1), head 1 = GaussianActorCriticNet on separate two-layer actor / critic bodies (shared 0);
 * gate 0 = tanh, 1 = ReLU.  flat: the FlatOptimizer arena; off (host, int32): arena offset of every tensor in the order
 * trunk 0 (w1 b1 w2 b2), [trunk 1 (w1 b1 w2 b2)], fc_action (w b), fc_critic (w b), [std].
 * smem_bytes: dynamic shared memory of the update for a rollout of T steps of N workers (0: not an instantiated configuration);
 *   it must fit the 227 KB of one SM.
 * actor_step: one env step in one launch -- state_out[n][d] = (float)(obs_scale * obs[n][d]) (RescaleNormalizer; obs is the
 *   float64 raw observation [N][D]), the actor's forward and the draw: categorical inverse CDF of the softmax on one Philox
 *   uniform, Gaussian mean + softplus(std) * N(0, 1) (Box-Muller); action_out [N][1] (the category as a float) or [N][A].
 *   *counter (device) advances by the number of draws (N or N * A).  given_action != NULL: written through, nothing drawn.
 * update: forward of states [T + 1][N][D], GAE (discount, tau, use_gae; the reference's order and association), objective
 *   -mean(log pi(a) adv) - entropy_weight mean(entropy) + value_loss_weight 0.5 mean((ret - v)^2) into *loss (device), its
 *   gradient, clip_grad_norm_(max_norm) and RMSprop (lr, alpha, eps, centered) on flat / square_avg / grad_avg; *step += 1. */
int64_t b2rl_a2c_smem_bytes(int32_t head, int32_t shared, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t N, int32_t T);
int b2rl_a2c_actor_step(int32_t head, int32_t shared, int32_t gate, const double* obs, double obs_scale, const float* flat,
                        const int32_t* off, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t N, float* state_out,
                        float* action_out, const float* given_action, uint64_t seed, int64_t* counter, void* stream);
int b2rl_a2c_update(int32_t head, int32_t shared, int32_t gate, const float* states, const float* actions, const float* reward,
                    const float* mask, int32_t T, int32_t N, int32_t D, int32_t H1, int32_t H2, int32_t A, float* flat,
                    float* square_avg, float* grad_avg, int64_t* step, const int32_t* off, float lr, float alpha, float eps,
                    int32_t centered, float discount, float tau, int32_t use_gae, float entropy_weight,
                    float value_loss_weight, float max_norm, float* loss, void* stream);

/* NStepDQNAgent.step() (NStepDQN_agent.py:26-67) on the device for a VanillaNet on a two-layer FCBody (gate 0 = tanh, 1 = ReLU).
 * flat: the FlatOptimizer arena; off (host, int32): arena offset of w1 b1 w2 b2 fc_head.w fc_head.b.
 * smem_bytes: dynamic shared memory of the update for a rollout of T steps of N workers; it must fit the 227 KB of one SM.
 * actor_step: state_out = (float)(obs_scale * obs) (RescaleNormalizer), q = net(state) and per row epsilon-greedy on two Philox
 *   uniforms: u0 < epsilon draws min(floor(u1 * A), A - 1), otherwise the first index of the largest q; action_out [N] (as a
 *   float).  *counter (device) advances by 2 N.  given_action != NULL: written through, nothing drawn, counter unchanged.
 * update: forward of states [T][N][D], bootstrap max_a q_target(states[T]), ret = r + discount * mask * ret backwards over T,
 *   0.5 mean((q[a] - ret)^2) into *loss (device), its gradient, clip_grad_norm_(max_norm) and RMSprop on flat / square_avg /
 *   grad_avg; *step += 1.  target: the target network's arena (same offsets).  sync_target != 0: target = flat (before the
 *   RMSprop step) first, and the bootstrap uses those weights.
 * actor_step also serves DQNAgent (b2rl_dqn_replay_*): net_kind = gate + 2 * head, head 0 = VanillaNet, 1 = DuelingNet (off:
 *   w1 b1 w2 b2 fc_advantage.w fc_advantage.b fc_value.w fc_value.b; q = v + (adv - mean(adv))).  state_out may be NULL. */
int64_t b2rl_nstep_dqn_smem_bytes(int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t N, int32_t T);
int b2rl_nstep_dqn_actor_step(int32_t net_kind, const double* obs, double obs_scale, const float* flat, const int32_t* off,
                              int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t N, float epsilon, float* state_out,
                              float* action_out, const float* given_action, uint64_t seed, int64_t* counter, void* stream);
int b2rl_nstep_dqn_update(int32_t gate, const float* states, const float* actions, const float* reward, const float* mask,
                          int32_t T, int32_t N, int32_t D, int32_t H1, int32_t H2, int32_t A, float* flat, float* target,
                          int32_t sync_target, float* square_avg, float* grad_avg, int64_t* step, const int32_t* off, float lr,
                          float alpha, float eps, int32_t centered, float discount, float max_norm, float* loss, void* stream);

/* DQNAgent's gradient update (DQN_agent.py:81-134) for one sampled batch on the device, as ONE launch of one block: head 0 =
 * VanillaNet, 1 = DuelingNet on a two-layer FCBody (gate 0 = tanh, 1 = ReLU); flat / off / target as for b2rl_nstep_dqn_*.
 * state / next_state [B][D]: float64 (state_f64) or float32 rows, rescaled as float32(state_scale * double(x)).  action int64,
 * reward / mask float32 [B].  y = reward + discount_n * q_next * mask with q_next = max_a q_target(s') or, double_q, q_target(s')
 * at the online argmax; delta = y - q[a] (delta_out, optional).  sampling_prob != NULL (PER): priority_out = (|delta| +
 * replay_eps)^replay_alpha, w = (P B + 1e-6)^-beta / max; the objective 0.5 mean((w delta)^2) into *loss, its gradient,
 * clip_grad_norm_(max_norm) and RMSprop on flat / square_avg / grad_avg; *step += 1.  The target arena is only read.
 * smem_bytes: dynamic shared memory for a batch of B; it must fit the 227 KB of one SM. */
int64_t b2rl_dqn_replay_smem_bytes(int32_t head, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t B, int32_t double_q);
int b2rl_dqn_replay_update(int32_t head, int32_t gate, const void* state, const void* next_state, int32_t state_f64,
                           double state_scale, const int64_t* action, const float* reward, const float* mask, int32_t B, int32_t D,
                           int32_t H1, int32_t H2, int32_t A, float* flat, const float* target, float* square_avg, float* grad_avg,
                           int64_t* step, const int32_t* off, float lr, float alpha, float eps, int32_t centered,
                           float discount_n, int32_t double_q, float max_norm, const float* sampling_prob, float beta,
                           float replay_eps, float replay_alpha, float* priority_out, float* delta_out, float* loss,
                           void* stream);

/* C51 / QR-DQN on the device (csrc/dist_dqn.cu): CategoricalDQNAgent / QuantileRegressionDQNAgent for a CategoricalNet /
 * QuantileNet on a two-layer FCBody.  kind 0 = C51, 1 = QR-DQN; gate 0 tanh / 1 ReLU.  The parameters: flat at off[6] in the
 * order w1 b1 w2 b2 fc.weight [A K][H2] fc.bias [A K] (fc_categorical / fc_quantiles).  Limits: D <= 256, H1, H2 <= 128,
 * 2 <= A <= 32, 2 <= K <= 256.  C51's support is np.linspace(v_min, v_max, K) in float64, rounded to float32.
 *
 * actor_step: rescale + forward + the action values (C51: sum_k softmax z_k; QR: the mean of the quantiles) + epsilon-greedy
 * on Philox stream 17 as b2rl_nstep_dqn_actor_step (two uniforms per row; the counter advances by 2 N; given_action != NULL:
 * written through, nothing drawn).
 *
 * replay_update: one launch on a sampled batch (the layout of b2rl_dqn_replay_update's arguments).  C51: the projection of the
 * target's p(a*) (a* the first maximum of sum_k p z_k of the target, or with double_q of the online network), KL = sum m log(m +
 * 1e-5) - m log p[a] (loss_vec_out [B], optional), PER when sampling_prob != NULL (priority_out = (|KL| + replay_eps)^alpha),
 * the objective mean(w KL).  QR (double_q ignored, no PER): T_j = r + discount_n mask theta'_j(a*), the quantile-Huber loss
 * vector indexed by target quantile (loss_vec_out [K], optional) and its mean.  Then the backward, clip_grad_norm_(max_norm)
 * and RMSprop as b2rl_dqn_replay_update.  smem_bytes: 0 for invalid input; the result must fit the 227 KB of one SM. */
int64_t b2rl_dist_dqn_smem_bytes(int32_t kind, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, int32_t B,
                                 int32_t double_q);
int b2rl_dist_dqn_actor_step(int32_t kind, int32_t gate, const double* obs, double obs_scale, const float* flat,
                             const int32_t* off, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, int32_t N, double v_min,
                             double v_max, float epsilon, float* action_out, const float* given_action, uint64_t seed,
                             int64_t* counter, void* stream);
int b2rl_dist_dqn_replay_update(int32_t kind, int32_t gate, const void* state, const void* next_state, int32_t state_f64,
                                double state_scale, const int64_t* action, const float* reward, const float* mask, int32_t B,
                                int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, float* flat, const float* target,
                                float* square_avg, float* grad_avg, int64_t* step, const int32_t* off, float lr, float alpha,
                                float eps, int32_t centered, float discount_n, int32_t double_q, double v_min, double v_max,
                                float max_norm, const float* sampling_prob, float beta, float replay_eps, float replay_alpha,
                                float* priority_out, float* loss_vec_out, float* loss, void* stream);

/* Rainbow on the device (csrc/rainbow.cu): CategoricalDQNAgent for a RainbowNet on a two-layer FCBody.  noisy 1: all four
 * layers (body.layers.0, body.layers.1, fc_advantage [A K][H2], fc_value [K][H2], the kernels' layer order) are NoisyLinear and
 * flat holds weight_mu weight_sigma bias_mu bias_sigma of layer l at off[4 l .. 4 l + 3]; noisy 0: all four are nn.Linear,
 * weight bias at off[2 l], off[2 l + 1].  gate 0 tanh / 1 ReLU.  Limits and the support as b2rl_dist_dqn_*.
 *
 * A network's noise vector is, layer after layer, noise_in [in], noise_out_weight [out], noise_out_bias [out]: noise_len =
 * sum (in + 2 out) floats.  Element i of a drawn vector is noise_std times the standard normal of Philox stream 29 under
 * `seed` at position *noise_counter + i.  f(x) = sign(x) sqrt|x|; the effective parameters mu + sigma (f(out_w) (x) f(in)),
 * mu_b + sigma_b f(out_b) are formed as the weights are read.  With noisy 0 nothing is drawn and the noise arguments are ignored.
 *
 * actor_step: one noise vector for the online network (given_noise != NULL: that vector [noise_len], nothing drawn, the
 * counter stays; else *noise_counter advances by noise_len), rescale + forward + q[a][k] = v[k] + adv[a][k] - mean_a adv[.][k]
 * + sum_k softmax(q[a])_k z_k + the action.  noisy 1: the argmax, epsilon is not read and *counter stays (DQN_agent.py:34-35);
 * noisy 0: b2rl_dist_dqn_actor_step's epsilon-greedy on stream 17 (*counter advances by 2 N).  given_action != NULL: written
 * through.  noise_out (optional) [noise_len]: the vector used.
 *
 * replay_update: one launch on a sampled batch (the arguments of b2rl_dist_dqn_replay_update with kind C51, then the noise).
 * Noise for the target network, then for the online network (given_noise != NULL: [2][noise_len] in that order, nothing drawn;
 * else *noise_counter advances by 2 noise_len).  The forwards, C51's projection, KL (loss_vec_out [B], optional), PER and logit
 * gradient, the backward through the dueling combination and the effective weights; d mu = dW, d sigma = dW eps_w, d mu_b = db,
 * d sigma_b = db eps_b; clip_grad_norm_(max_norm) over all tensors and RMSprop.  noise_out (optional): the online module's
 * noise arena -- the online vector [noise_len], then every layer's bias_epsilon [out], then every layer's weight_epsilon
 * [out][in].  target_noise_out (optional) [noise_len].  smem_bytes: 0 for invalid input; double_q does not change it (the
 * online forward of the next states uses the rows the target's forward takes afterwards); it must fit the 227 KB of one SM. */
int64_t b2rl_rainbow_smem_bytes(int32_t noisy, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, int32_t B,
                                int32_t double_q);
int b2rl_rainbow_actor_step(int32_t noisy, int32_t gate, const double* obs, double obs_scale, const float* flat,
                            const int32_t* off, int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, int32_t N, double v_min,
                            double v_max, float epsilon, float* action_out, const float* given_action, uint64_t seed,
                            int64_t* counter, float noise_std, const float* given_noise, float* noise_out,
                            int64_t* noise_counter, void* stream);
int b2rl_rainbow_replay_update(int32_t noisy, int32_t gate, const void* state, const void* next_state, int32_t state_f64,
                               double state_scale, const int64_t* action, const float* reward, const float* mask, int32_t B,
                               int32_t D, int32_t H1, int32_t H2, int32_t A, int32_t K, float* flat, const float* target,
                               float* square_avg, float* grad_avg, int64_t* step, const int32_t* off, float lr, float alpha,
                               float eps, int32_t centered, float discount_n, int32_t double_q, double v_min, double v_max,
                               float max_norm, const float* sampling_prob, float beta, float replay_eps, float replay_alpha,
                               float* priority_out, float* loss_vec_out, float* loss, uint64_t seed, float noise_std,
                               const float* given_noise, float* noise_out, float* target_noise_out, int64_t* noise_counter,
                               void* stream);

int b2rl_ipc_alloc(int64_t bytes, void** out);
int b2rl_ipc_get_handle(void* ptr, void* handle_out);
int b2rl_ipc_open_handle(const void* handle, void** out);
int b2rl_ipc_close(void* ptr);
int b2rl_ipc_free(void* ptr);
int b2rl_peer_access_ok(int32_t dev_a, int32_t dev_b, int32_t* ok);

/* Element-wise halves of the distributional heads (CategoricalNet / QuantileNet, network_heads.py:40-55, 89-102) around the
 * wgmma GEMMs: softmax + log_softmax over the N atoms of every (b, a) row (either output may be NULL), and the backward
 * preparation dlogits = dout - prob * sum_n dout (prob == NULL: dlogits = dout, QR-DQN) written as the bf16 GEMM operand
 * g [B][ld] (ld >= A*N, multiple of 8; padding zeroed) with its column sums ADDED to dbias [A*N] (the bias gradient). */
int b2rl_dist_softmax(const float* logits, int32_t rows, int32_t N, float* prob, float* log_prob, void* stream);
int b2rl_dist_head_bwd_prep(const float* dout, const float* prob, int32_t B, int32_t A, int32_t N, uint16_t* g, int32_t ld,
                            float* dbias, void* stream);

/* DQN update, head part, in one launch (DQN_agent.py:78-99, 120-127 and the head's backward): q = head(phi) on s,
 * q_next = target_head(phi_t) on s' [argmax from head(phi_o) for double-Q], delta / priorities / IS weights / loss as
 * b2rl_dqn_loss, then the gradients of the head (accumulated into gWa / gba / gWv / gbv), dphi masked by phi > 0 and
 * its column sums (fc4's bias gradient) accumulated into relu_colsum.  Heads: VanillaNet (Wv == NULL) or DuelingNet
 * (network_heads.py:11-37).  scratch: int32 counter (zero-initialised once, self re-arming) + 12 bytes
 * padding + float [ceil(B/16)]. */
int b2rl_dqn_head_fused(const uint16_t* phi, const uint16_t* phi_t, const uint16_t* phi_o, const float* Wa, const float* ba,
                        const float* Wv, const float* bv, const float* Wa_t, const float* ba_t, const float* Wv_t,
                        const float* bv_t, const int64_t* action, const float* reward, const float* mask, float gamma_n,
                        int32_t B, int32_t K, int32_t A, const float* is_prob, float beta, const float* beta_dev, float eps,
                        float alpha, uint16_t* gphi, float* gWa, float* gba, float* gWv, float* gbv, float* relu_colsum,
                        float* q_out, float* delta_out, float* prio_out, float* loss_out, float* scratch, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B2RL_H */
