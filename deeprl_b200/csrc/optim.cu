// optim.cu -- multi-tensor global-norm clip + optimizer step over one flat parameter arena.
// Reference call sites: deep_rl/agent/DQN_agent.py:132-134 (clip_grad_norm_ then optimizer.step),
// examples.py:67-68 (RMSprop lr 2.5e-4, alpha .95, eps .01, centered), :139,:204 (Adam).
// Update rules are torch.optim's (RMSprop: _single_tensor_rmsprop, Adam: _single_tensor_adam),
// clip rule is torch.nn.utils.clip_grad_norm_ (coef = max_norm / (total_norm + 1e-6), clamped to 1).
// One arena => 2 launches instead of ~10 tensors x (norm + mul + ~8 optimizer ops).  sm_90a only.
#include "common.cuh"
#include "optim_elem.h"

namespace b2rl {

struct NormScratch { float sumsq; float coef; int32_t counter; int32_t pad; };

// grid-stride sum of squares; last CTA turns it into the clip coefficient
__global__ void __launch_bounds__(512) sumsq_kernel(const float* __restrict__ g, int64_t n, float grad_scale,
                                                    float max_norm, float* __restrict__ partial,
                                                    NormScratch* __restrict__ sc) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ float red[32];
  __shared__ bool is_last;
  float s = 0.0f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
    if (i + 3 < n) {
      float4 v = *reinterpret_cast<const float4*>(g + i);
      v.x *= grad_scale; v.y *= grad_scale; v.z *= grad_scale; v.w *= grad_scale;
      s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    } else {
      for (int64_t k = i; k < n; ++k) { float x = g[k] * grad_scale; s += x * x; }
    }
  }
  s = block_reduce(s, OpAdd(), 0.0f, red);
  if (threadIdx.x == 0) {
    partial[blockIdx.x] = s;
    __threadfence();
    is_last = atomicAdd(&sc->counter, 1) == (int)gridDim.x - 1;
  }
  __syncthreads();
  if (is_last) {
    __threadfence();
    float t = 0.0f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) t += __ldcg(partial + i);
    t = block_reduce(t, OpAdd(), 0.0f, red);
    if (threadIdx.x == 0) {
      float norm = sqrtf(t);
      sc->sumsq = norm;                               // total_norm (what clip_grad_norm_ returns)
      float c = max_norm > 0.0f ? max_norm / (norm + 1e-6f) : 1.0f;
      sc->coef = fminf(c, 1.0f) * grad_scale;
      sc->counter = 0;
    }
  }
}

__global__ void __launch_bounds__(256) rmsprop_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                      float* __restrict__ sq, float* __restrict__ ga, int64_t n,
                                                      float lr, float alpha, float eps, int centered,
                                                      const NormScratch* __restrict__ sc,
                                                      __nv_bfloat16* __restrict__ shadow) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  const float coef = sc->coef;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gr = g[i] * coef;
    const float np_ = b2rl_elem::rmsprop_elem(p[i], gr, sq, ga, i, lr, alpha, eps, centered);
    p[i] = np_;
    if (shadow) shadow[i] = __float2bfloat16_rn(np_);
  }
}

__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                   float* __restrict__ m, float* __restrict__ v, int64_t n, float lr,
                                                   float b1, float b2, float eps, const int64_t* __restrict__ step_dev,
                                                   const NormScratch* __restrict__ sc,
                                                   __nv_bfloat16* __restrict__ shadow, const float* __restrict__ gate,
                                                   float gate_max) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  if (gate && !(*gate <= gate_max)) return;        // device-side `if approx_kl <= 1.5 * target_kl:` (PPO_agent.py:94)
  const float coef = sc->coef;
  const float t = (float)(*step_dev);
  const float bc1 = 1.0f - powf(b1, t), bc2 = 1.0f - powf(b2, t);
  const float step_size = lr / bc1, bc2s = sqrtf(bc2);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gr = g[i] * coef;
    float mi = m[i];
    mi = mi + (1.0f - b1) * (gr - mi);                            // exp_avg.lerp_(grad, 1 - beta1)
    float vi = b2 * v[i] + (1.0f - b2) * gr * gr;                 // exp_avg_sq.mul_(beta2).addcmul_(g, g, 1-beta2)
    m[i] = mi; v[i] = vi;
    const float denom = sqrtf(vi) / bc2s + eps;
    const float np_ = p[i] - step_size * (mi / denom);
    p[i] = np_;
    if (shadow) shadow[i] = __float2bfloat16_rn(np_);
  }
}

__global__ void bump_step_kernel(int64_t* step, const float* gate, float gate_max) {
  pdl_sync();
  if (gate && !(*gate <= gate_max)) return;
  *step += 1;
}

}  // namespace b2rl

using namespace b2rl;

static int norm_pass(const float* grad, int64_t n, float grad_scale, float max_norm, void* norm_scratch,
                     cudaStream_t st) {
  // scratch layout: NormScratch (16 B) then float partial[296]
  NormScratch* sc = reinterpret_cast<NormScratch*>(norm_scratch);
  float* partial = reinterpret_cast<float*>(sc + 1);
  int blocks = (int)((n + 512 * 4 - 1) / (512 * 4));
  if (blocks > 296) blocks = 296;
  if (blocks < 1) blocks = 1;
  launch_pdl(sumsq_kernel, dim3(blocks), dim3(512), 0, st, grad, n, grad_scale, max_norm, partial, sc);
  return check_launch("clip/sumsq");
}

// clip_grad_norm_'s coefficient on its own: norm_scratch[0] = total norm of grad * grad_scale, norm_scratch[1] = the factor
// min(max_norm / (norm + 1e-6), 1) * grad_scale every gradient element is multiplied by (max_norm <= 0: grad_scale).  Used
// after a gradient all-reduce, before b2rl_nature_fused_opt without unit partials.
extern "C" int b2rl_grad_norm(const float* grad, int64_t n, float grad_scale, float max_norm, void* norm_scratch, void* stream) {
  B2RL_REQUIRE(grad && norm_scratch, "null pointer");
  B2RL_REQUIRE(n > 0 && (reinterpret_cast<uintptr_t>(grad) % 16 == 0), "bad size / gradient arena must be 16B aligned");
  return norm_pass(grad, n, grad_scale, max_norm, norm_scratch, (cudaStream_t)stream);
}

extern "C" int b2rl_clip_rmsprop(float* param, const float* grad, float* square_avg, float* grad_avg, int64_t n,
                                 float max_norm, float lr, float alpha, float eps, int32_t centered, float grad_scale,
                                 void* norm_scratch, uint16_t* bf16_shadow, void* stream) {
  B2RL_REQUIRE(param && grad && square_avg && norm_scratch && (grad_avg || !centered), "null pointer");
  B2RL_REQUIRE(n > 0 && (reinterpret_cast<uintptr_t>(grad) % 16 == 0), "bad size / gradient arena must be 16B aligned");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = norm_pass(grad, n, grad_scale, max_norm, norm_scratch, st);
  if (rc) return rc;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  launch_pdl(rmsprop_kernel, dim3(blocks), dim3(256), 0, st, param, grad, square_avg, grad_avg, n, lr, alpha, eps, centered,
                                         reinterpret_cast<NormScratch*>(norm_scratch),
                                         reinterpret_cast<__nv_bfloat16*>(bf16_shadow));
  return check_launch("b2rl_clip_rmsprop");
}

static int clip_adam_impl(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n, float max_norm,
                          float lr, float beta1, float beta2, float eps, int64_t* step_dev, float grad_scale,
                          void* norm_scratch, uint16_t* bf16_shadow, const float* gate, float gate_max, void* stream) {
  B2RL_REQUIRE(param && grad && exp_avg && exp_avg_sq && step_dev && norm_scratch, "null pointer");
  B2RL_REQUIRE(n > 0 && (reinterpret_cast<uintptr_t>(grad) % 16 == 0), "bad size / gradient arena must be 16B aligned");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = norm_pass(grad, n, grad_scale, max_norm, norm_scratch, st);
  if (rc) return rc;
  launch_pdl(bump_step_kernel, dim3(1), dim3(1), 0, st, step_dev, gate, gate_max);
  rc = check_launch("adam/step");
  if (rc) return rc;
  int blocks = (int)((n + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;
  launch_pdl(adam_kernel, dim3(blocks), dim3(256), 0, st, param, grad, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps, step_dev,
             reinterpret_cast<NormScratch*>(norm_scratch), reinterpret_cast<__nv_bfloat16*>(bf16_shadow), gate, gate_max);
  return check_launch("b2rl_clip_adam");
}

extern "C" int b2rl_clip_adam(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                              float max_norm, float lr, float beta1, float beta2, float eps, int64_t* step_dev,
                              float grad_scale, void* norm_scratch, uint16_t* bf16_shadow, void* stream) {
  return clip_adam_impl(param, grad, exp_avg, exp_avg_sq, n, max_norm, lr, beta1, beta2, eps, step_dev, grad_scale,
                        norm_scratch, bf16_shadow, nullptr, 0.0f, stream);
}

// The same step, taken only if the DEVICE scalar *gate <= gate_max (moments, step count and parameters untouched otherwise):
// the KL gate of the PPO actor update (`if approx_kl <= 1.5 * target_kl:` PPO_agent.py:94) without a host round trip, so the
// minibatch update can live in a CUDA graph.
extern "C" int b2rl_clip_adam_gated(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                                    float max_norm, float lr, float beta1, float beta2, float eps, int64_t* step_dev,
                                    float grad_scale, void* norm_scratch, uint16_t* bf16_shadow, const float* gate,
                                    float gate_max, void* stream) {
  B2RL_REQUIRE(gate, "null gate");
  return clip_adam_impl(param, grad, exp_avg, exp_avg_sq, n, max_norm, lr, beta1, beta2, eps, step_dev, grad_scale,
                        norm_scratch, bf16_shadow, gate, gate_max, stream);
}
