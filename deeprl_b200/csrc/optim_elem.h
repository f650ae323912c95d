// optim_elem.h -- the element arithmetic of torch.optim.RMSprop (_single_tensor_rmsprop, no momentum / weight decay), ONE copy
// shared by rmsprop_kernel (optim.cu) and the one-launch A2C update (a2c_phases.h, which tests/host_emul also compiles for the
// host).  `gr` is the gradient element after clip_grad_norm_'s coefficient.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define B2RL_ELEM_FN __host__ __device__ __forceinline__
#else
#define B2RL_ELEM_FN static inline
#endif

namespace b2rl_elem {

// returns the new parameter; square_avg[i] (and grad_avg[i] when centered) are updated in place
B2RL_ELEM_FN float rmsprop_elem(float p, float gr, float* sq, float* ga, int64_t i, float lr, float alpha, float eps,
                                int centered) {
  const float s = alpha * sq[i] + (1.0f - alpha) * gr * gr;      // square_avg.mul_(alpha).addcmul_(g, g, 1-alpha)
  sq[i] = s;
  float avg;
  if (centered) {
    float a = ga[i];
    a = a + (1.0f - alpha) * (gr - a);                            // grad_avg.lerp_(grad, 1 - alpha)
    ga[i] = a;
    avg = sqrtf(s - a * a) + eps;                                 // addcmul(grad_avg, grad_avg, -1).sqrt_().add_(eps)
  } else {
    avg = sqrtf(s) + eps;
  }
  return p - lr * (gr / avg);                                     // param.addcdiv_(grad, avg, value=-lr)
}

}  // namespace b2rl_elem
