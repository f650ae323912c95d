// pack.cu -- weight / gradient re-layout between the reference's parameter layouts (network_bodies.py:13-20:
// conv [Cout,Cin,kh,kw], fc4 [512, (c,h,w)]) and the tap-major bf16 operands of the grid-GEMM convolution stack
// (csrc/gemm.cu, network/nature_tc.py).  One launch packs all four layers (forward and dgrad orientations), one launch
// maps the four fp32 weight gradients back and ACCUMULATES them (and the bias gradients) into the .grad arena.
// sm_90a only.
#include "common.cuh"

namespace b2rl {

struct PackArgs {
  const float* w1; const float* w2; const float* w3; const float* w4;   // master parameters (reference layouts)
  __nv_bfloat16* w1f; __nv_bfloat16* w2f; __nv_bfloat16* w2d; __nv_bfloat16* w3f; __nv_bfloat16* w3d; __nv_bfloat16* w4p;
  int c1;          // conv1 input channels (frames)
  int n4;          // fc4 output features
  float scale;     // ImageNormalizer coefficient folded into conv1
};

// segment sizes: w1f 32*64*c1 | w2f 64*512 | w2d 128*256 | w3f 64*576 | w3d 64*576 | w4p n4*3136
__global__ void __launch_bounds__(256) pack_weights_kernel(PackArgs a) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  const int64_t s1 = 32LL * 64 * a.c1, s2 = 64 * 512, s3 = 128 * 256, s4 = 64 * 576, s5 = 64 * 576,
                s6 = (int64_t)a.n4 * 3136;
  const int64_t total = s1 + s2 + s3 + s4 + s5 + s6;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = e;
    if (i < s1) {   // w1f[n][tap=(ty,tx)][f][dy][dx] = w1[n][f][4ty+dy][4tx+dx] * scale
      const int K = 64 * a.c1;
      const int n = (int)(i / K), k = (int)(i % K);
      const int tap = k / (16 * a.c1), c = k % (16 * a.c1);
      const int f = c / 16, dy = (c % 16) / 4, dx = c % 4, ty = tap / 2, tx = tap % 2;
      a.w1f[i] = __float2bfloat16_rn(a.w1[((n * a.c1 + f) * 8 + 4 * ty + dy) * 8 + 4 * tx + dx] * a.scale);
      continue;
    }
    i -= s1;
    if (i < s2) {   // w2f[n][(ty,tx)][(py,px,c)] = w2[n][c][2ty+py][2tx+px]
      const int n = (int)(i / 512), k = (int)(i % 512);
      const int tap = k / 128, r = k % 128, ty = tap / 2, tx = tap % 2, py = r / 64, px = (r / 32) % 2, c = r % 32;
      a.w2f[i] = __float2bfloat16_rn(a.w2[((n * 32 + c) * 4 + 2 * ty + py) * 4 + 2 * tx + px]);
      continue;
    }
    i -= s2;
    if (i < s3) {   // w2d[(py,px,c)][(ty,tx)][n]
      const int row = (int)(i / 256), k = (int)(i % 256);
      const int py = row / 64, px = (row / 32) % 2, c = row % 32, tap = k / 64, n = k % 64, ty = tap / 2, tx = tap % 2;
      a.w2d[i] = __float2bfloat16_rn(a.w2[((n * 32 + c) * 4 + 2 * ty + py) * 4 + 2 * tx + px]);
      continue;
    }
    i -= s3;
    if (i < s4) {   // w3f[n][(ky,kx)][c] = w3[n][c][ky][kx]
      const int n = (int)(i / 576), k = (int)(i % 576), tap = k / 64, c = k % 64;
      a.w3f[i] = __float2bfloat16_rn(a.w3[(n * 64 + c) * 9 + tap]);
      continue;
    }
    i -= s4;
    if (i < s5) {   // w3d[c][(ky,kx)][n]
      const int c = (int)(i / 576), k = (int)(i % 576), tap = k / 64, n = k % 64;
      a.w3d[i] = __float2bfloat16_rn(a.w3[(n * 64 + c) * 9 + tap]);
      continue;
    }
    i -= s5;
    {               // w4p[n][(h,w)][c] = w4[n][c*49 + hw]
      const int64_t n = i / 3136;
      const int k = (int)(i % 3136), hw = k / 64, c = k % 64;
      a.w4p[i] = __float2bfloat16_rn(a.w4[n * 3136 + c * 49 + hw]);
    }
  }
}

struct UnpackArgs {
  const float* g1f; const float* g2f; const float* g3f; const float* g4p;   // GEMM-layout fp32 gradients
  const float* db1; const float* db2; const float* db3; const float* db4;   // bias gradients
  float* gw1; float* gw2; float* gw3; float* gw4;                            // .grad in reference layouts (accumulated)
  float* gb1; float* gb2; float* gb3; float* gb4;
  int c1, n4;
  float scale;
  int p1, p2, p3;      // number of split-K partials of g1f / g2f / g3f (1 = already reduced)
};

// sum over split-K partials; consecutive threads read consecutive elements of the same partial (coalesced), 16
// independent loads in flight per thread hide the L2 latency
__device__ __forceinline__ float sum_partials(const float* __restrict__ g, int64_t idx, int parts, int64_t stride) {
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.0f;
  int p = 0;
  for (; p + 15 < parts; p += 16) {
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] += __ldg(g + idx + (int64_t)(p + j) * stride);
  }
  for (; p < parts; ++p) acc[0] += __ldg(g + idx + (int64_t)p * stride);
  float s = 0.0f;
#pragma unroll
  for (int j = 0; j < 16; ++j) s += acc[j];
  return s;
}

__global__ void __launch_bounds__(256) unpack_grads_kernel(UnpackArgs a) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  const int64_t s1 = 32LL * a.c1 * 64, s2 = 64 * 512, s3 = 64 * 576, s4 = (int64_t)a.n4 * 3136;
  const int64_t sb = 32 + 64 + 64 + a.n4;
  const int64_t total = s1 + s2 + s3 + s4 + sb;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    int64_t i = e;      // i indexes the REFERENCE-layout destination (coalesced writes)
    if (i < s1) {       // gw1[n][f][ky][kx]
      const int kx = (int)(i % 8), ky = (int)((i / 8) % 8), f = (int)((i / 64) % a.c1), n = (int)(i / (64 * a.c1));
      const int tap = (ky / 4) * 2 + kx / 4, c = f * 16 + (ky % 4) * 4 + kx % 4;
      a.gw1[i] += sum_partials(a.g1f, (int64_t)n * 64 * a.c1 + tap * 16 * a.c1 + c, a.p1, s1) * a.scale;
      continue;
    }
    i -= s1;
    if (i < s2) {       // gw2[n][c][ky][kx]
      const int kx = (int)(i % 4), ky = (int)((i / 4) % 4), c = (int)((i / 16) % 32), n = (int)(i / 512);
      const int tap = (ky / 2) * 2 + kx / 2, r = ((ky % 2) * 2 + kx % 2) * 32 + c;
      a.gw2[i] += sum_partials(a.g2f, n * 512 + tap * 128 + r, a.p2, s2);
      continue;
    }
    i -= s2;
    if (i < s3) {       // gw3[n][c][ky][kx]
      const int tap = (int)(i % 9), c = (int)((i / 9) % 64), n = (int)(i / 576);
      a.gw3[i] += sum_partials(a.g3f, n * 576 + tap * 64 + c, a.p3, s3);
      continue;
    }
    i -= s3;
    if (i < s4) {       // gw4[n][c*49 + hw]
      const int64_t n = i / 3136;
      const int k = (int)(i % 3136), c = k / 49, hw = k % 49;
      a.gw4[i] += a.g4p[n * 3136 + hw * 64 + c];
      continue;
    }
    i -= s4;
    if (i < 32) { a.gb1[i] += a.db1[i]; continue; }
    i -= 32;
    if (i < 64) { a.gb2[i] += a.db2[i]; continue; }
    i -= 64;
    if (i < 64) { a.gb3[i] += a.db3[i]; continue; }
    i -= 64;
    a.gb4[i] += a.db4[i];
  }
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_nature_pack_weights(const float* w1, const float* w2, const float* w3, const float* w4, int32_t c1,
                                        int32_t n4, float scale, uint16_t* w1f, uint16_t* w2f, uint16_t* w2d,
                                        uint16_t* w3f, uint16_t* w3d, uint16_t* w4p, void* stream) {
  B2RL_REQUIRE(w1 && w2 && w3 && w4 && w1f && w2f && w2d && w3f && w3d && w4p, "null pointer");
  B2RL_REQUIRE(c1 > 0 && n4 > 0, "bad shape");
  PackArgs a;
  a.w1 = w1; a.w2 = w2; a.w3 = w3; a.w4 = w4;
  a.w1f = reinterpret_cast<__nv_bfloat16*>(w1f); a.w2f = reinterpret_cast<__nv_bfloat16*>(w2f);
  a.w2d = reinterpret_cast<__nv_bfloat16*>(w2d); a.w3f = reinterpret_cast<__nv_bfloat16*>(w3f);
  a.w3d = reinterpret_cast<__nv_bfloat16*>(w3d); a.w4p = reinterpret_cast<__nv_bfloat16*>(w4p);
  a.c1 = c1; a.n4 = n4; a.scale = scale;
  launch_pdl(pack_weights_kernel, dim3(132 * 8), dim3(256), 0, (cudaStream_t)stream, a);
  return check_launch("b2rl_nature_pack_weights");
}

extern "C" int b2rl_nature_unpack_grads(const float* g1f, const float* g2f, const float* g3f, const float* g4p,
                                        const float* db1, const float* db2, const float* db3, const float* db4,
                                        int32_t c1, int32_t n4, float scale, float* gw1, float* gw2, float* gw3,
                                        float* gw4, float* gb1, float* gb2, float* gb3, float* gb4, int32_t p1,
                                        int32_t p2, int32_t p3, void* stream) {
  B2RL_REQUIRE(g1f && g2f && g3f && g4p && db1 && db2 && db3 && db4 && gw1 && gw2 && gw3 && gw4 && gb1 && gb2 && gb3 && gb4,
               "null pointer");
  UnpackArgs a;
  a.g1f = g1f; a.g2f = g2f; a.g3f = g3f; a.g4p = g4p; a.db1 = db1; a.db2 = db2; a.db3 = db3; a.db4 = db4;
  a.gw1 = gw1; a.gw2 = gw2; a.gw3 = gw3; a.gw4 = gw4; a.gb1 = gb1; a.gb2 = gb2; a.gb3 = gb3; a.gb4 = gb4;
  a.c1 = c1; a.n4 = n4; a.scale = scale;
  a.p1 = p1 < 1 ? 1 : p1; a.p2 = p2 < 1 ? 1 : p2; a.p3 = p3 < 1 ? 1 : p3;
  launch_pdl(unpack_grads_kernel, dim3(132 * 8), dim3(256), 0, (cudaStream_t)stream, a);
  return check_launch("b2rl_nature_unpack_grads");
}
