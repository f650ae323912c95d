// tail.cu -- the tail of one gradient update (DQN_agent.py:131-134: backward's last step, clip_grad_norm_, optimizer.step)
// for a NatureConvBody network on the wgmma path, as TWO launches instead of five:
//
//   A  nature_grad_reduce_kernel : split-K partials of the three convolution weight gradients summed (deterministic order),
//                                  all four weight gradients mapped from the GEMM layouts to the reference's parameter
//                                  layouts and WRITTEN (not accumulated) into the flat .grad arena, bias gradients moved
//                                  there too (and their atomic accumulators re-zeroed), and the sum of squares of every
//                                  gradient element -- including the head's, which head_bwd already put in the arena --
//                                  left as one partial per work unit.
//   B  nature_fused_opt_kernel   : takes the clip coefficient of torch.nn.utils.clip_grad_norm_ from the norm scratch
//                                  (what NatureTail.step does: kernel A's last CTA left it there, or b2rl_grad_norm after
//                                  a multi-GPU all-reduce) or, given the unit partials, has every CTA add them in the same
//                                  fixed order and derive it itself (the same bits in every CTA and as kernel A's: no grid
//                                  barrier, no second launch), applies RMSprop (plain / centered) or Adam exactly as
//                                  csrc/optim.cu does, re-zeroes the gradient it consumed, and writes the updated weights
//                                  straight into the bf16 tap-major GEMM operands (forward + dgrad orientations) that the next
//                                  update's wgmma kernels read -- the separate pack launch disappears as well.
//
// Replaces unpack_grads (it walked the split-K partials with strided gathers) + sumsq + rmsprop + pack_weights
// + the memset of the gradient arena.  Work is described by unit tables built once on the host (network/tail.py):
// int32 x 4 per unit = {arena offset, length, kind, row | segment << 16}.
// sm_90a only.
#include "common.cuh"

namespace b2rl {

constexpr int TAIL_THREADS = 256;
enum { U_PLAIN = 0, U_W1 = 1, U_W2 = 2, U_W3 = 3, U_W4 = 4, U_B1 = 5, U_B2 = 6, U_B3 = 7, U_B4 = 8 };

struct NormScratch { float sumsq; float coef; int32_t counter; int32_t pad; };     // same layout as csrc/optim.cu

// index of GEMM-layout element k of one output row in the reference's parameter layout of that row (the inverse of the
// maps in csrc/pack.cu): w1 [f][ky][kx] <- [tap=(ty,tx)][f][dy][dx], w2 [c][ky][kx] <- [tap][(py,px,c)],
// w3 [c][ky*3+kx] <- [tap][c], w4 [c*49+hw] <- [hw][c]
__device__ __forceinline__ int ref_index(int kind, int k, int c1) {
  if (kind == U_W1) {
    const int per = 16 * c1, tap = k / per, c = k - tap * per;
    const int f = c >> 4, dy = (c & 15) >> 2, dx = c & 3, ty = tap >> 1, tx = tap & 1;
    return (f * 8 + 4 * ty + dy) * 8 + 4 * tx + dx;
  }
  if (kind == U_W2) {
    const int tap = k >> 7, r = k & 127, ty = tap >> 1, tx = tap & 1, py = r >> 6, px = (r >> 5) & 1, c = r & 31;
    return (c * 4 + 2 * ty + py) * 4 + 2 * tx + px;
  }
  if (kind == U_W3) return (k & 63) * 9 + (k >> 6);
  return (k & 63) * 49 + (k >> 6);
}

__device__ __forceinline__ int row_len(int kind, int c1) {
  return kind == U_W1 ? 64 * c1 : kind == U_W2 ? 512 : kind == U_W3 ? 576 : 3136;
}

struct ReduceArgs {
  const int4* units;
  const float* g1p; const float* g2p; const float* g3p; const float* g4p;   // GEMM-layout gradients (conv: split-K partials)
  int p1, p2, p3;
  float* db1; float* db2; float* db3; float* db4;                            // bias-gradient accumulators (re-zeroed here)
  int c1, n4;
  float scale;
  float* grad;                                                               // flat .grad arena
  float* unit_sumsq;                                                         // [gridDim.x]
  int64_t* step_dev;                                                         // Adam step counter (bumped by unit 0) or null
  NormScratch* sc;                                                           // non-null: the CTA that finishes last turns the unit
  float max_norm, grad_scale;                                                // partials into clip_grad_norm_'s coefficient
};

__device__ __forceinline__ void add4(float4& a, const float4 b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }

__global__ void __launch_bounds__(TAIL_THREADS) nature_grad_reduce_kernel(const ReduceArgs a) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ float sbuf[49 * 65 + 7];
  __shared__ float red[32];
  const int tid = threadIdx.x;
  const int4 u = __ldg(a.units + blockIdx.x);
  const int off = u.x, len = u.y, kind = u.z, row = u.w & 0xFFFF, seg = u.w >> 16;
  float ss = 0.0f;
  if (kind == U_W4) {
    // one fc4 row: [hw][c] -> [c][hw] through shared memory (row pitch 65: conflict-free both ways)
    const float4* src = reinterpret_cast<const float4*>(a.g4p + (int64_t)row * 3136);
    float4 x[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {                             // 784 float4 = 3.06 per thread: all requested before any is used
      const int v = tid + t * TAIL_THREADS;
      if (v < 784) x[t] = __ldg(src + v);
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int v = tid + t * TAIL_THREADS;
      if (v < 784) {
        const int k = 4 * v, hw = k >> 6, c = k & 63;
        float* d = sbuf + hw * 65 + c;
        d[0] = x[t].x; d[1] = x[t].y; d[2] = x[t].z; d[3] = x[t].w;
      }
    }
    __syncthreads();
    float4* dst = reinterpret_cast<float4*>(a.grad + off);
    for (int v = tid; v < 784; v += TAIL_THREADS) {
      float g[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int i = 4 * v + j, c = i / 49, hw = i - c * 49;
        g[j] = sbuf[hw * 65 + c];
        ss += g[j] * g[j];
      }
      dst[v] = make_float4(g[0], g[1], g[2], g[3]);
    }
  } else if (kind >= U_W1 && kind <= U_W3) {
    // one 256-element segment of one output row of a convolution weight gradient: 4 thread groups x 64 float4 columns,
    // group g adds partials g, g+4, ... (8 independent 16-byte loads in flight per thread), then the groups are added
    const int L = row_len(kind, a.c1);
    const float* gp = kind == U_W1 ? a.g1p : kind == U_W2 ? a.g2p : a.g3p;
    const int P = kind == U_W1 ? a.p1 : kind == U_W2 ? a.p2 : a.p3;
    const int n_out = kind == U_W1 ? 32 : 64;
    const int64_t pstride = (int64_t)n_out * L;
    const int seg0 = seg * 256, seglen = len;
    const int vec = tid & 63, grp = tid >> 6;
    float4 acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (4 * vec < seglen) {
      const float* base = gp + (int64_t)row * L + seg0 + 4 * vec;
      int p = grp;
      for (; p + 28 < P; p += 32) {
#pragma unroll
        for (int j = 0; j < 8; ++j) add4(acc[j], __ldg(reinterpret_cast<const float4*>(base + (int64_t)(p + 4 * j) * pstride)));
      }
      for (; p < P; p += 4) add4(acc[0], __ldg(reinterpret_cast<const float4*>(base + (int64_t)p * pstride)));
#pragma unroll
      for (int j = 1; j < 8; ++j) add4(acc[0], acc[j]);
    }
    float* r = sbuf + grp * 256 + 4 * vec;
    r[0] = acc[0].x; r[1] = acc[0].y; r[2] = acc[0].z; r[3] = acc[0].w;
    __syncthreads();
    if (tid < seglen) {
      float s = (sbuf[tid] + sbuf[256 + tid]) + (sbuf[512 + tid] + sbuf[768 + tid]);
      if (kind == U_W1) s *= a.scale;                      // w1f = w1 * scale  =>  dL/dw1 = dL/dw1f * scale
      a.grad[off + ref_index(kind, seg0 + tid, a.c1)] = s;
      ss = s * s;
    }
  } else if (kind >= U_B1) {
    float* db = kind == U_B1 ? a.db1 : kind == U_B2 ? a.db2 : kind == U_B3 ? a.db3 : a.db4;
    for (int i = tid; i < len; i += TAIL_THREADS) {
      const float g = db[i];
      db[i] = 0.0f;                                        // the dgrad epilogues accumulate into it with atomics
      a.grad[off + i] = g;
      ss += g * g;
    }
  } else {
    const float4* g4 = reinterpret_cast<const float4*>(a.grad + off);
    for (int v = tid; v < (len >> 2); v += TAIL_THREADS) {
      const float4 x = g4[v];
      ss += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
    }
  }
  ss = block_reduce(ss, OpAdd(), 0.0f, red);
  __shared__ bool is_last;
  if (tid == 0) {
    a.unit_sumsq[blockIdx.x] = ss;
    if (blockIdx.x == 0 && a.step_dev) *a.step_dev += 1;
    is_last = false;
    if (a.sc) {
      __threadfence();
      is_last = atomicAdd(&a.sc->counter, 1) == (int)gridDim.x - 1;
    }
  }
  __syncthreads();
  if (is_last) {                                          // fixed summation order: the result does not depend on which CTA is last
    __threadfence();
    float t = 0.0f;
    for (int i = tid; i < (int)gridDim.x; i += TAIL_THREADS) t += __ldcg(a.unit_sumsq + i);
    t = block_reduce(t, OpAdd(), 0.0f, red);
    if (tid == 0) {
      const float norm = sqrtf(t) * a.grad_scale;
      const float c = a.max_norm > 0.0f ? a.max_norm / (norm + 1e-6f) : 1.0f;
      a.sc->sumsq = norm;                                 // total_norm (what clip_grad_norm_ returns)
      a.sc->coef = fminf(c, 1.0f) * a.grad_scale;
      a.sc->counter = 0;
    }
  }
}

struct OptArgs {
  const int4* units;
  float* param; float* grad; float* s1; float* s2;
  int opt;                      // 0 RMSprop, 1 RMSprop centered, 2 Adam
  float lr, a, b, eps;          // RMSprop: a = alpha; Adam: a = beta1, b = beta2
  float max_norm, grad_scale;
  const float* unit_sumsq; int n_sumsq;           // null: the clip coefficient comes from norm_scratch (b2rl_grad_norm)
  NormScratch* sc;
  const int64_t* step_dev;
  int c1, n4;
  float scale;
  __nv_bfloat16* w1f; __nv_bfloat16* w2f; __nv_bfloat16* w2d; __nv_bfloat16* w3f; __nv_bfloat16* w3d; __nv_bfloat16* w4p;
  int zero_grad;
  __nv_bfloat16* shadow;        // bf16 copy of the whole arena at the same offsets, or null (the GEMM operands of the heads)
  const float* lr_dev;          // the learning rate on the device (a schedule stepped between graph replays), or null: lr
};

__global__ void __launch_bounds__(TAIL_THREADS) nature_fused_opt_kernel(const OptArgs a) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ float sbuf[3136];
  __shared__ float red[32];
  const int tid = threadIdx.x;
  const int4 u = __ldg(a.units + blockIdx.x);
  const int off = u.x, len = u.y, kind = u.z, row = u.w & 0xFFFF;
  float coef;
  if (a.unit_sumsq) {
    float t = 0.0f;
    for (int i = tid; i < a.n_sumsq; i += TAIL_THREADS) t += __ldcg(a.unit_sumsq + i);
    t = block_reduce(t, OpAdd(), 0.0f, red);              // same order, same bits in every CTA
    const float norm = sqrtf(t) * a.grad_scale;
    const float c = a.max_norm > 0.0f ? a.max_norm / (norm + 1e-6f) : 1.0f;
    coef = fminf(c, 1.0f) * a.grad_scale;
    if (blockIdx.x == 0 && tid == 0) { a.sc->sumsq = norm; a.sc->coef = coef; }
  } else {
    coef = a.sc->coef;
  }
  const float lr = a.lr_dev ? *a.lr_dev : a.lr;
  float step_size = lr, bc2s = 1.0f;
  if (a.opt == 2) {
    const float t = (float)(*a.step_dev);
    const float bc1 = 1.0f - powf(a.a, t), bc2 = 1.0f - powf(a.b, t);
    step_size = lr / bc1;
    bc2s = sqrtf(bc2);
  }
  const bool packs = kind >= U_W1 && kind <= U_W4 && a.w4p != nullptr;
  float4* p4 = reinterpret_cast<float4*>(a.param + off);
  float4* g4 = reinterpret_cast<float4*>(a.grad + off);
  float4* s14 = reinterpret_cast<float4*>(a.s1 + off);
  float4* s24 = reinterpret_cast<float4*>(a.s2 + off);
  constexpr int MAXV = 4;                                      // a unit has at most 3136 / 4 = 784 float4 = 3.06 per thread
  float4 gq[MAXV], pq[MAXV], s1q[MAXV], s2q[MAXV];
#pragma unroll
  for (int t = 0; t < MAXV; ++t) {                            // one round trip: every load of the unit is in flight together
    const int v = tid + t * TAIL_THREADS;
    if (v < (len >> 2)) {
      gq[t] = g4[v]; pq[t] = p4[v]; s1q[t] = s14[v];
      s2q[t] = a.opt != 0 ? s24[v] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
#pragma unroll
  for (int t = 0; t < MAXV; ++t) {
    const int v = tid + t * TAIL_THREADS;
    if (v >= (len >> 2)) continue;
    const float4 gv = gq[t], pv = pq[t], s1v = s1q[t], s2v = s2q[t];
    const float g[4] = {gv.x * coef, gv.y * coef, gv.z * coef, gv.w * coef};
    float p[4] = {pv.x, pv.y, pv.z, pv.w}, s1[4] = {s1v.x, s1v.y, s1v.z, s1v.w}, s2[4] = {s2v.x, s2v.y, s2v.z, s2v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gr = g[j];
      if (a.opt == 2) {                                              // torch.optim.Adam (_single_tensor_adam)
        float mi = s1[j];
        mi = mi + (1.0f - a.a) * (gr - mi);
        const float vi = a.b * s2[j] + (1.0f - a.b) * gr * gr;
        s1[j] = mi; s2[j] = vi;
        const float denom = sqrtf(vi) / bc2s + a.eps;
        p[j] = p[j] - step_size * (mi / denom);
      } else {                                                       // torch.optim.RMSprop (_single_tensor_rmsprop)
        const float s = a.a * s1[j] + (1.0f - a.a) * gr * gr;
        s1[j] = s;
        float avg;
        if (a.opt == 1) {
          float ga = s2[j];
          ga = ga + (1.0f - a.a) * (gr - ga);
          s2[j] = ga;
          avg = sqrtf(s - ga * ga) + a.eps;
        } else {
          avg = sqrtf(s) + a.eps;
        }
        p[j] = p[j] - lr * (gr / avg);
      }
    }
    p4[v] = make_float4(p[0], p[1], p[2], p[3]);
    s14[v] = make_float4(s1[0], s1[1], s1[2], s1[3]);
    if (a.opt != 0) s24[v] = make_float4(s2[0], s2[1], s2[2], s2[3]);
    if (a.zero_grad) g4[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.shadow) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(p[0], p[1]), hi = __floats2bfloat162_rn(p[2], p[3]);
      uint2 o;
      o.x = *reinterpret_cast<uint32_t*>(&lo); o.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(a.shadow + off + 4 * v) = o;
    }
    if (packs) {
      float* d = sbuf + 4 * v;
      d[0] = p[0]; d[1] = p[1]; d[2] = p[2]; d[3] = p[3];
    }
  }
  if (!packs) return;
  __syncthreads();
  // the updated row in the bf16 GEMM layouts (coalesced over the destination index k; shared-memory reads are permuted)
  if (kind == U_W4) {
    __nv_bfloat16* d = a.w4p + (int64_t)row * 3136;
    for (int k2 = tid; k2 < 1568; k2 += TAIL_THREADS) {
      const int k = 2 * k2;
      const int i0 = ref_index(U_W4, k, a.c1), i1 = ref_index(U_W4, k + 1, a.c1);
      *reinterpret_cast<__nv_bfloat162*>(d + k) = __floats2bfloat162_rn(sbuf[i0], sbuf[i1]);
    }
  } else if (kind == U_W1) {
    const int L = 64 * a.c1;
    for (int k = tid; k < L; k += TAIL_THREADS)
      a.w1f[(int64_t)row * L + k] = __float2bfloat16_rn(sbuf[ref_index(U_W1, k, a.c1)] * a.scale);
  } else if (kind == U_W2) {
    for (int k = tid; k < 512; k += TAIL_THREADS) {
      const __nv_bfloat16 v = __float2bfloat16_rn(sbuf[ref_index(U_W2, k, a.c1)]);
      a.w2f[row * 512 + k] = v;
      a.w2d[(k & 127) * 256 + (k >> 7) * 64 + row] = v;
    }
  } else {
    for (int k = tid; k < 576; k += TAIL_THREADS) {
      const __nv_bfloat16 v = __float2bfloat16_rn(sbuf[ref_index(U_W3, k, a.c1)]);
      a.w3f[row * 576 + k] = v;
      a.w3d[(k & 63) * 576 + (k >> 6) * 64 + row] = v;
    }
  }
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_nature_grad_reduce(const int32_t* units, int32_t n_units, const float* g1p, int32_t p1, const float* g2p,
                                       int32_t p2, const float* g3p, int32_t p3, const float* g4p, float* db1, float* db2,
                                       float* db3, float* db4, int32_t c1, int32_t n4, float scale, float* grad,
                                       float* unit_sumsq, int64_t* step_dev, void* norm_scratch, float max_norm,
                                       float grad_scale, void* stream) {
  B2RL_REQUIRE(units && g1p && g2p && g3p && g4p && db1 && db2 && db3 && db4 && grad && unit_sumsq, "null pointer");
  B2RL_REQUIRE(n_units > 0 && p1 > 0 && p2 > 0 && p3 > 0, "bad counts");
  B2RL_REQUIRE(c1 > 0 && c1 <= 16 && c1 % 4 == 0 && n4 > 0, "conv1 input channels must be a multiple of 4, at most 16");
  B2RL_REQUIRE((reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(g1p) | reinterpret_cast<uintptr_t>(g2p) |
                reinterpret_cast<uintptr_t>(g3p) | reinterpret_cast<uintptr_t>(g4p) | reinterpret_cast<uintptr_t>(units)) % 16 == 0,
               "buffers must be 16-byte aligned");
  ReduceArgs a;
  a.units = reinterpret_cast<const int4*>(units);
  a.g1p = g1p; a.g2p = g2p; a.g3p = g3p; a.g4p = g4p; a.p1 = p1; a.p2 = p2; a.p3 = p3;
  a.db1 = db1; a.db2 = db2; a.db3 = db3; a.db4 = db4; a.c1 = c1; a.n4 = n4; a.scale = scale;
  a.grad = grad; a.unit_sumsq = unit_sumsq; a.step_dev = step_dev;
  a.sc = reinterpret_cast<NormScratch*>(norm_scratch); a.max_norm = max_norm; a.grad_scale = grad_scale;
  launch_pdl(nature_grad_reduce_kernel, dim3(n_units), dim3(TAIL_THREADS), 0, (cudaStream_t)stream, a);
  return check_launch("b2rl_nature_grad_reduce");
}

// b2rl_nature_fused_opt with the learning rate read from the device: lr_dev != NULL replaces lr (a float32 the host writes
// between replays of a captured graph, e.g. a decaying schedule); lr_dev == NULL is b2rl_nature_fused_opt.
extern "C" int b2rl_nature_fused_opt_lr(const int32_t* units, int32_t n_units, float* param, float* grad, float* s1, float* s2,
                                        int32_t opt, float lr, const float* lr_dev, float a_, float b_, float eps,
                                        float max_norm, float grad_scale, const float* unit_sumsq, int32_t n_sumsq,
                                        void* norm_scratch, const int64_t* step_dev, int32_t c1, int32_t n4, float scale,
                                        uint16_t* w1f, uint16_t* w2f, uint16_t* w2d, uint16_t* w3f, uint16_t* w3d, uint16_t* w4p,
                                        int32_t zero_grad, uint16_t* bf16_shadow, void* stream) {
  B2RL_REQUIRE(units && param && grad && s1 && norm_scratch, "null pointer");
  B2RL_REQUIRE(opt >= 0 && opt <= 2 && (opt == 0 || s2) && (opt != 2 || step_dev), "bad optimizer description");
  B2RL_REQUIRE(n_units > 0 && (!unit_sumsq || n_sumsq > 0), "bad counts");
  B2RL_REQUIRE((w4p == nullptr) == (w1f == nullptr) && (!w4p || (w2f && w2d && w3f && w3d)), "all packed operands or none");
  B2RL_REQUIRE(c1 > 0 && c1 <= 16 && c1 % 4 == 0 && n4 > 0, "conv1 input channels must be a multiple of 4, at most 16");
  B2RL_REQUIRE((reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(s1) |
                reinterpret_cast<uintptr_t>(s2) | reinterpret_cast<uintptr_t>(units)) % 16 == 0, "arenas must be 16-byte aligned");
  OptArgs a;
  a.units = reinterpret_cast<const int4*>(units);
  a.param = param; a.grad = grad; a.s1 = s1; a.s2 = s2; a.opt = opt; a.lr = lr; a.a = a_; a.b = b_; a.eps = eps;
  a.max_norm = max_norm; a.grad_scale = grad_scale; a.unit_sumsq = unit_sumsq; a.n_sumsq = n_sumsq;
  a.sc = reinterpret_cast<NormScratch*>(norm_scratch); a.step_dev = step_dev; a.c1 = c1; a.n4 = n4; a.scale = scale;
  a.w1f = reinterpret_cast<__nv_bfloat16*>(w1f); a.w2f = reinterpret_cast<__nv_bfloat16*>(w2f);
  a.w2d = reinterpret_cast<__nv_bfloat16*>(w2d); a.w3f = reinterpret_cast<__nv_bfloat16*>(w3f);
  a.w3d = reinterpret_cast<__nv_bfloat16*>(w3d); a.w4p = reinterpret_cast<__nv_bfloat16*>(w4p);
  a.zero_grad = zero_grad;
  a.shadow = reinterpret_cast<__nv_bfloat16*>(bf16_shadow);
  a.lr_dev = lr_dev;
  launch_pdl(nature_fused_opt_kernel, dim3(n_units), dim3(TAIL_THREADS), 0, (cudaStream_t)stream, a);
  return check_launch("b2rl_nature_fused_opt");
}

extern "C" int b2rl_nature_fused_opt(const int32_t* units, int32_t n_units, float* param, float* grad, float* s1, float* s2,
                                     int32_t opt, float lr, float a_, float b_, float eps, float max_norm, float grad_scale,
                                     const float* unit_sumsq, int32_t n_sumsq, void* norm_scratch, const int64_t* step_dev,
                                     int32_t c1, int32_t n4, float scale, uint16_t* w1f, uint16_t* w2f, uint16_t* w2d,
                                     uint16_t* w3f, uint16_t* w3d, uint16_t* w4p, int32_t zero_grad, uint16_t* bf16_shadow,
                                     void* stream) {
  return b2rl_nature_fused_opt_lr(units, n_units, param, grad, s1, s2, opt, lr, nullptr, a_, b_, eps, max_norm, grad_scale,
                                  unit_sumsq, n_sumsq, norm_scratch, step_dev, c1, n4, scale, w1f, w2f, w2d, w3f, w3d, w4p,
                                  zero_grad, bf16_shadow, stream);
}
