// replay.cu -- HBM-resident replay ring: feed, uniform index selection, frame-stack gather.
// Reference semantics: deep_rl/component/replay.py:75-140 (UniformReplay).  sm_90a only.
//
// Data layout (all in HBM, allocated by the caller):
//   frames  uint8  [capacity][row_bytes]   one row per env step (newest 84x84 frame, DQN_agent.py:108)
//   action  int32  [capacity]
//   reward  float64[capacity]              the reference keeps python floats; n-step sums are float64
//   mask    int32  [capacity]
//   ring_state int64[8]                    {pos, size, capacity, tree write cursor, philox counter, ...}
//
// The gather is the HBM-bound kernel of the path: per sampled transition it reads history+n_step
// contiguous rows ONCE (valid indices never straddle the ring seam, replay.py:105-110) with one TMA
// bulk copy into shared memory and writes the two overlapping stacks (state, next_state) from there.
#include <cstdlib>
#include "common.cuh"

namespace b2rl {

// --------------------------------------------------------------------------------------------- feed
__global__ void __launch_bounds__(512) feed_kernel(uint8_t* __restrict__ frames, int32_t* __restrict__ action,
                                                   double* __restrict__ reward, int32_t* __restrict__ mask,
                                                   int64_t* __restrict__ ring_state, int64_t row_bytes,
                                                   const uint8_t* __restrict__ nf, const int32_t* __restrict__ na,
                                                   const double* __restrict__ nr, const int32_t* __restrict__ nm,
                                                   int n, int quirk) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ int64_t slot[1024];
  __shared__ int64_t fin[2];
  if (threadIdx.x == 0) {
    // replay.py:80-90, statement by statement
    int64_t pos0 = ring_state[0], len = ring_state[1], cap = ring_state[2];
    int64_t pos = pos0;
    for (int j = 0; j < n; ++j) {
      if (pos >= len) { slot[j] = len; ++len; }       // storage.append(v)
      else slot[j] = quirk ? pos0 : pos;              // storage[self.pos] = v   (sic, replay.py:87)
      pos = (pos + 1) % cap;
    }
    fin[0] = pos; fin[1] = len;
  }
  __syncthreads();
  const bool vec = (row_bytes % 16 == 0) && ((reinterpret_cast<uintptr_t>(frames) | reinterpret_cast<uintptr_t>(nf)) % 16 == 0);
  for (int j = 0; j < n; ++j) {   // in order: with the quirk several items hit the same slot, last one wins
    uint8_t* dst = frames + slot[j] * row_bytes;
    const uint8_t* src = nf + (int64_t)j * row_bytes;
    if (vec) {
      const int4* s4 = reinterpret_cast<const int4*>(src);
      int4* d4 = reinterpret_cast<int4*>(dst);
      for (int64_t k = threadIdx.x; k < row_bytes / 16; k += blockDim.x) d4[k] = s4[k];
    } else {
      for (int64_t k = threadIdx.x; k < row_bytes; k += blockDim.x) dst[k] = src[k];
    }
    if (threadIdx.x == 0) {
      action[slot[j]] = na[j];
      reward[slot[j]] = nr[j];
      mask[slot[j]] = nm[j];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { ring_state[0] = fin[0]; ring_state[1] = fin[1]; }
}

// --------------------------------------------------------------------------------------------- select
__device__ __forceinline__ bool valid_index(int64_t i, int64_t pos, int64_t size, int hl, int n) {
  // replay.py:105-110
  if (i - hl + 1 >= 0 && i + n < pos) return true;
  if (i - hl + 1 >= pos && i + n < size) return true;
  return false;
}

__device__ __forceinline__ void gather_scalars(const int32_t* action, const double* reward, const int32_t* mask,
                                               int64_t i, int n, double discount, int64_t* a_out, float* r_out,
                                               float* m_out, int b) {
  // replay.py:128-140: cum_r = reward[k] + mask[k]*discount*cum_r for k reversed (float64); cum_mask = AND
  double cum_r = 0.0;
  int cum_m = 1;
  for (int k = n - 1; k >= 0; --k) {
    double mk = (double)mask[i + k];
    cum_r = __dadd_rn(reward[i + k], __dmul_rn(__dmul_rn(mk, discount), cum_r));
    cum_m = (cum_m && mask[i + k]) ? 1 : 0;
  }
  if (a_out) a_out[b] = (int64_t)action[i];
  if (r_out) r_out[b] = (float)cum_r;          // one rounding float64 -> float32, as np.asarray(x, float32)
  if (m_out) m_out[b] = (float)cum_m;
}

constexpr int SEL_THREADS = 1024;
constexpr int SEL_PER_THREAD = 8;

__global__ void __launch_bounds__(SEL_THREADS) select_uniform_kernel(int64_t* __restrict__ ring_state,
                                                                     const int64_t* __restrict__ cand, int n_cand,
                                                                     uint64_t seed, int hl, int n, int B,
                                                                     int64_t* __restrict__ idx_out,
                                                                     int32_t* __restrict__ status, const int32_t* action,
                                                                     const double* reward, const int32_t* mask,
                                                                     double discount, int64_t* a_out, float* r_out,
                                                                     float* m_out) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  __shared__ int warp_tot[32];
  __shared__ int last_used;
  const int64_t pos = ring_state[0], size = ring_state[1];
  const uint64_t ctr = (uint64_t)ring_state[4];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  int64_t c[SEL_PER_THREAD];
  int cnt = 0;
  unsigned vmask = 0;
#pragma unroll
  for (int k = 0; k < SEL_PER_THREAD; ++k) {
    int g = t * SEL_PER_THREAD + k;
    if (g < n_cand) {
      c[k] = cand ? cand[g] : (int64_t)Philox::below(seed, ctr + g, 1, (uint64_t)size);
      bool v = c[k] >= 0 && c[k] < size && valid_index(c[k], pos, size, hl, n);
      vmask |= (unsigned)v << k;
      cnt += v;
    }
  }
  // exclusive scan of cnt over the block (thread order == candidate-stream order)
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_tot[w] = incl;
  if (t == 0) last_used = 0;
  __syncthreads();
  if (w == 0) {
    int x = warp_tot[lane], s = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    warp_tot[lane] = s - x;   // exclusive warp offsets
    if (lane == 31) status[0] = s < B ? s : B;
  }
  __syncthreads();
  int rank = warp_tot[w] + incl - cnt;
#pragma unroll
  for (int k = 0; k < SEL_PER_THREAD; ++k) {
    if ((vmask >> k) & 1) {
      if (rank < B) {
        idx_out[rank] = c[k];
        if (rank == B - 1) last_used = t * SEL_PER_THREAD + k + 1;
      }
      ++rank;
    }
  }
  __syncthreads();
  // The candidate stream is finite; the reference keeps drawing (replay.py:97-100).  If it ran dry (status[0] < B: a tiny ring,
  // or B close to the stream length) the unfilled tail must still hold VALID indices -- the consumers (gather, conv1's ring
  // producer) read frames through them without a host check inside a captured graph -- so the accepted indices are cycled;
  // with none at all every slot gets the smallest index that cannot read below the ring (hl - 1).  status[0] keeps the count.
  {
    __shared__ int s_total;
    if (t == SEL_THREADS - 1) s_total = min(warp_tot[w] + incl, B);     // accepted = inclusive count of the last thread
    __syncthreads();
    const int total = s_total;
    for (int j = total + t; j < B; j += SEL_THREADS) idx_out[j] = total > 0 ? idx_out[j % total] : (int64_t)(hl - 1);
  }
  // action / n-step reward / mask of the chosen indices (K1: the frame stacks stay in the ring), in the same launch: the
  // separate gather_scalars_kernel would be one more dependent launch between the draw and the forward pass
  if (a_out || r_out || m_out) {
    __syncthreads();                                  // idx_out complete, including the cycled tail
    for (int j = t; j < B; j += SEL_THREADS) gather_scalars(action, reward, mask, idx_out[j], n, discount, a_out, r_out, m_out, j);
  }
  if (t == 0) {
    status[1] = last_used ? last_used : n_cand;       // candidates consumed (all of them if the stream ran dry)
    if (!cand) ring_state[4] = (int64_t)(ctr + (uint64_t)n_cand);
  }
}

// --------------------------------------------------------------------------------------------- gather
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra WAIT_DONE;\n"
      "bra WAIT_LOOP;\n"
      "WAIT_DONE:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(phase)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_wait_read() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

template <typename T> struct Cvt;
template <> struct Cvt<float> { __device__ static float f(float x) { return x; } };
template <> struct Cvt<__half> { __device__ static __half f(float x) { return __float2half_rn(x); } };
template <> struct Cvt<__nv_bfloat16> { __device__ static __nv_bfloat16 f(float x) { return __float2bfloat16_rn(x); } };

// scalars only (action, n-step reward, mask): the frame stacks stay in the ring and are read by conv1 itself (K1, csrc/gemm.cu)
__global__ void __launch_bounds__(128) gather_scalars_kernel(const int32_t* __restrict__ action, const double* __restrict__ reward,
                                                             const int32_t* __restrict__ mask, const int64_t* __restrict__ idx,
                                                             int B, int n, double discount, int64_t* a_out, float* r_out,
                                                             float* m_out) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) gather_scalars(action, reward, mask, idx[b], n, discount, a_out, r_out, m_out, b);
}

// raw uint8 stacks, [B][hl][row_bytes]: pure TMA bulk copies, issued by one thread per CTA.
__global__ void __launch_bounds__(32) gather_raw_tma_kernel(const uint8_t* __restrict__ frames,
                                                            const int32_t* __restrict__ action,
                                                            const double* __restrict__ reward,
                                                            const int32_t* __restrict__ mask, int64_t row_bytes,
                                                            const int64_t* __restrict__ idx, int hl, int n,
                                                            double discount, uint8_t* __restrict__ state_out,
                                                            uint8_t* __restrict__ next_out, int64_t* a_out,
                                                            float* r_out, float* m_out) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar;
  const int b = blockIdx.x;
  const int64_t i = idx[b];
  const uint32_t span = (uint32_t)((hl + n) * row_bytes), stack = (uint32_t)(hl * row_bytes);
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    mbar_expect_tx(&bar, span);
    bulk_g2s(smem, frames + (i - hl + 1) * row_bytes, span, &bar);
  }
  if (threadIdx.x == 1) gather_scalars(action, reward, mask, i, n, discount, a_out, r_out, m_out, b);
  if (threadIdx.x == 0) {
    mbar_wait(&bar, 0);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    if (state_out) bulk_s2g(state_out + (int64_t)b * stack, smem, stack);
    if (next_out) bulk_s2g(next_out + (int64_t)b * stack, smem + (int64_t)n * row_bytes, stack);
    bulk_commit_wait_read();
  }
}

// converted stacks: TMA bulk load, then vectorised convert + store.
// LAYOUT 0: [B][hl][row_bytes] (NCHW)   1: [B][row_bytes][hl] (NHWC)
//        2: space-to-depth by 4: [B][H/4][W/4][hl*16], channel = f*16 + dy*4 + dx  (an 8x8/stride-4 convolution over
//           the frames becomes a 2x2/stride-1 convolution over 16*hl channels: conv1 turns into a plain implicit GEMM)
// lut != NULL: value = lut[v] rounded to T (exact ImageNormalizer semantics in float32);
// lut == NULL: value = (T)v, the integer 0..255 exactly (the 1/255 scale is folded into the consumer's weights).
template <typename T>
__device__ __forceinline__ void cvt_word(uint32_t w, const T* __restrict__ slut, bool use_lut, T* out4) {
  if (use_lut) {
#pragma unroll
    for (int k = 0; k < 4; ++k) out4[k] = slut[(w >> (8 * k)) & 255];
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) out4[k] = Cvt<T>::f((float)((w >> (8 * k)) & 255));
  }
}
template <>
__device__ __forceinline__ void cvt_word<__nv_bfloat16>(uint32_t w, const __nv_bfloat16* __restrict__ slut, bool use_lut,
                                                        __nv_bfloat16* out4) {
  if (use_lut) {
#pragma unroll
    for (int k = 0; k < 4; ++k) out4[k] = slut[(w >> (8 * k)) & 255];
  } else {
    // exact u8 -> bf16 without I2F: 0x4B0000vv is the float 2^23 + v; subtract 2^23; the top 16 bits are the bf16
    const float m = 8388608.0f;
    uint32_t f0 = __float_as_uint(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540)) - m);
    uint32_t f1 = __float_as_uint(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7541)) - m);
    uint32_t f2 = __float_as_uint(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7542)) - m);
    uint32_t f3 = __float_as_uint(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7543)) - m);
    uint32_t* o = reinterpret_cast<uint32_t*>(out4);
    o[0] = __byte_perm(f0, f1, 0x7632);
    o[1] = __byte_perm(f2, f3, 0x7632);
  }
}

template <typename T, int LAYOUT>
__global__ void __launch_bounds__(256) gather_cvt_kernel(const uint8_t* __restrict__ frames,
                                                         const int32_t* __restrict__ action,
                                                         const double* __restrict__ reward,
                                                         const int32_t* __restrict__ mask, int64_t row_bytes,
                                                         const int64_t* __restrict__ idx, int hl, int n,
                                                         double discount, const float* __restrict__ lut,
                                                         T* __restrict__ state_out, T* __restrict__ next_out,
                                                         int64_t* a_out, float* r_out, float* m_out, int use_tma,
                                                         int frame_w) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ T slut[256];
  const int b = blockIdx.x;
  const int64_t i = idx[b];
  const int64_t span = (int64_t)(hl + n) * row_bytes, stack = (int64_t)hl * row_bytes;
  const uint8_t* src = frames + (i - hl + 1) * row_bytes;
  const bool use_lut = lut != nullptr;
  if (use_tma) {
    if (threadIdx.x == 0) {
      mbar_init(&bar, 1);
      mbar_expect_tx(&bar, (uint32_t)span);
      bulk_g2s(smem, src, (uint32_t)span, &bar);
    }
  } else {
    for (int64_t k = threadIdx.x; k < span; k += blockDim.x) smem[k] = src[k];
  }
  if (use_lut) slut[threadIdx.x] = Cvt<T>::f(lut[threadIdx.x]);
  if (threadIdx.x == 32) gather_scalars(action, reward, mask, i, n, discount, a_out, r_out, m_out, b);
  __syncthreads();                       // barrier init + lut visible
  if (use_tma) mbar_wait(&bar, 0);       // every thread observes the completed phase
  __syncthreads();

  constexpr int VEC = 16 / sizeof(T);    // output elements per 16-byte store
  for (int which = 0; which < 2; ++which) {
    T* out = which ? next_out : state_out;
    if (!out) continue;
    out += (int64_t)b * stack;
    const uint8_t* s = smem + (which ? (int64_t)n * row_bytes : 0);
    // Every fast path below gives one thread exactly one 16-byte store per iteration, consecutive lanes writing
    // consecutive 16-byte pieces: a warp store fills whole 32-byte sectors (two stores of a 32-byte-per-thread unit would
    // each fill half of 32 sectors and double the L1->L2 write traffic).
    constexpr int SUBS = 16 / VEC;         // 16-byte pieces per 16-element unit (bf16/fp16: 2, fp32: 4)
    if (LAYOUT == 2) {
      // unit = (position (Y,X), frame f): rows 4Y..4Y+3, cols 4X..4X+3 -> 16 contiguous outputs; piece = ROWS rows of it
      constexpr int ROWS = 4 / SUBS;
      const int Wq = frame_w / 4, Hq = (int)(row_bytes / frame_w) / 4;
      const int pieces = Hq * Wq * hl * SUBS;
      for (int h = threadIdx.x; h < pieces; h += blockDim.x) {
        const int u = h / SUBS, sub = h - u * SUBS;
        const int pos = u / hl, f = u - pos * hl;
        const int Y = pos / Wq, X = pos - Y * Wq;
        const uint8_t* base = s + (int64_t)f * row_bytes + (4 * Y + sub * ROWS) * frame_w + 4 * X;
        __align__(16) T v[VEC];
#pragma unroll
        for (int dy = 0; dy < ROWS; ++dy)
          cvt_word<T>(*reinterpret_cast<const uint32_t*>(base + dy * frame_w), slut, use_lut, v + 4 * dy);
        *reinterpret_cast<int4*>(out + (int64_t)h * VEC) = *reinterpret_cast<const int4*>(v);
      }
    } else if (LAYOUT == 1 && hl == 4 && row_bytes % 4 == 0) {
      // piece = PX pixels x 4 frames: one LDS.32 per frame (the word holding the pixels), shifted to the piece
      constexpr int PX = VEC / 4;
      const int pieces = (int)(row_bytes / 4) * SUBS;
      for (int h = threadIdx.x; h < pieces; h += blockDim.x) {
        const int p4 = h / SUBS, sub = h - p4 * SUBS;
        __align__(16) T c[4][4];
#pragma unroll
        for (int f = 0; f < 4; ++f)
          cvt_word<T>(*reinterpret_cast<const uint32_t*>(s + f * row_bytes + p4 * 4) >> (8 * PX * sub), slut, use_lut, c[f]);
        __align__(16) T v[VEC];
#pragma unroll
        for (int px = 0; px < PX; ++px)
#pragma unroll
          for (int f = 0; f < 4; ++f) v[px * 4 + f] = c[f][px];
        *reinterpret_cast<int4*>(out + (int64_t)h * VEC) = *reinterpret_cast<const int4*>(v);
      }
    } else if (LAYOUT == 1) {
      for (int64_t e = threadIdx.x; e < stack; e += blockDim.x) {
        int64_t p = e / hl;
        int c = (int)(e - p * hl);
        uint8_t v = s[(int64_t)c * row_bytes + p];
        out[e] = use_lut ? slut[v] : Cvt<T>::f((float)v);
      }
    } else if (row_bytes % 16 == 0) {
      // NCHW: VEC input bytes -> one 16-byte store
      for (int64_t e = threadIdx.x; e < stack / VEC; e += blockDim.x) {
        __align__(16) T v[VEC];
#pragma unroll
        for (int k = 0; k < VEC / 4; ++k)
          cvt_word<T>(*reinterpret_cast<const uint32_t*>(s + e * VEC + 4 * k), slut, use_lut, v + 4 * k);
        *reinterpret_cast<int4*>(out + e * VEC) = *reinterpret_cast<const int4*>(v);
      }
    } else {
      for (int64_t e = threadIdx.x; e < stack; e += blockDim.x) out[e] = use_lut ? slut[s[e]] : Cvt<T>::f((float)s[e]);
    }
  }
}

// Space-to-depth gather with BULK stores (16-bit outputs): the converted stack of a sample is one contiguous range of
// (H/4)*(W/4)*hl*16 elements, so instead of 16-byte stores from every thread (the L1->L2 store path is what holds the kernel
// above at 0.60 of the copy peak while the raw uint8 variant, all bulk copies, reaches 0.76) the threads convert a third of
// the positions at a time into a shared staging tile laid out exactly like the output and ONE thread hands the tile to the
// copy engine (cp.async.bulk shared -> global); two tiles alternate so that conversion overlaps the previous tile's store.
// NOT YET VERIFIED ON A GPU (selected with B2RL_GATHER_BULK=1).
template <typename T>
__global__ void __launch_bounds__(256) gather_s2d_bulk_kernel(const uint8_t* __restrict__ frames,
                                                              const int32_t* __restrict__ action,
                                                              const double* __restrict__ reward,
                                                              const int32_t* __restrict__ mask, int64_t row_bytes,
                                                              const int64_t* __restrict__ idx, int hl, int n,
                                                              double discount, T* __restrict__ state_out,
                                                              T* __restrict__ next_out, int64_t* a_out, float* r_out,
                                                              float* m_out, int frame_w, int tile_pos) {
  static_assert(sizeof(T) == 2, "16-bit outputs: one 16-byte piece = 2 image rows x 4 pixels of one frame");
  pdl_sync();
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar;
  const int b = blockIdx.x;
  const int64_t i = idx[b];
  const int64_t span = (int64_t)(hl + n) * row_bytes, stack = (int64_t)hl * row_bytes;
  const uint32_t span_al = ((uint32_t)span + 127u) & ~127u;
  const uint32_t tile_bytes = (uint32_t)tile_pos * hl * 16 * sizeof(T);
  uint8_t* stage0 = smem + span_al;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    mbar_expect_tx(&bar, (uint32_t)span);
    bulk_g2s(smem, frames + (i - hl + 1) * row_bytes, (uint32_t)span, &bar);
  }
  if (threadIdx.x == 32) gather_scalars(action, reward, mask, i, n, discount, a_out, r_out, m_out, b);
  __syncthreads();
  mbar_wait(&bar, 0);
  __syncthreads();
  const int Wq = frame_w / 4, Hq = (int)(row_bytes / frame_w) / 4;
  const int positions = Hq * Wq;
  const int tiles = (positions + tile_pos - 1) / tile_pos;
  int t_global = 0;
  for (int which = 0; which < 2; ++which) {
    T* out = which ? next_out : state_out;
    if (!out) continue;
    out += (int64_t)b * stack;
    const uint8_t* src = smem + (which ? (int64_t)n * row_bytes : 0);
    for (int t = 0; t < tiles; ++t, ++t_global) {
      uint8_t* stage = stage0 + (size_t)(t_global & 1) * tile_bytes;
      // the tile that used this staging buffer two rounds ago must have been read by the copy engine
      if (t_global >= 2) {
        if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
        __syncthreads();
      }
      const int p0 = t * tile_pos, np = min(tile_pos, positions - p0);
      const int pieces = np * hl * 2;                                   // 16-byte pieces: (position, frame, half)
      for (int h = threadIdx.x; h < pieces; h += blockDim.x) {
        const int u = h >> 1, half = h & 1;
        const int pos = p0 + u / hl, f = u % hl;
        const int Y = pos / Wq, X = pos - Y * Wq;
        const uint8_t* base = src + (int64_t)f * row_bytes + (4 * Y + 2 * half) * frame_w + 4 * X;
        __align__(16) T v[8];
        cvt_word<T>(*reinterpret_cast<const uint32_t*>(base), nullptr, false, v);
        cvt_word<T>(*reinterpret_cast<const uint32_t*>(base + frame_w), nullptr, false, v + 4);
        *reinterpret_cast<int4*>(stage + (size_t)h * 16) = *reinterpret_cast<const int4*>(v);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> visible to the copy engine
      __syncthreads();
      if (threadIdx.x == 0) {
        bulk_s2g(out + (int64_t)p0 * hl * 16, stage, (uint32_t)np * hl * 16 * sizeof(T));
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    }
  }
  if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// raw uint8 fallback when rows are not 16-byte multiples (feature vectors)
__global__ void __launch_bounds__(128) gather_raw_generic_kernel(const uint8_t* __restrict__ frames,
                                                                 const int32_t* __restrict__ action,
                                                                 const double* __restrict__ reward,
                                                                 const int32_t* __restrict__ mask, int64_t row_bytes,
                                                                 const int64_t* __restrict__ idx, int hl, int n,
                                                                 double discount, uint8_t* __restrict__ state_out,
                                                                 uint8_t* __restrict__ next_out, int64_t* a_out,
                                                                 float* r_out, float* m_out) {
  pdl_sync();   // PDL contract (common.cuh): before any global-memory access or return
  const int b = blockIdx.x;
  const int64_t i = idx[b];
  const int64_t stack = (int64_t)hl * row_bytes;
  const uint8_t* src = frames + (i - hl + 1) * row_bytes;
  if (threadIdx.x == 0) gather_scalars(action, reward, mask, i, n, discount, a_out, r_out, m_out, b);
  for (int64_t k = threadIdx.x; k < stack; k += blockDim.x) {
    if (state_out) state_out[(int64_t)b * stack + k] = src[k];
    if (next_out) next_out[(int64_t)b * stack + k] = src[(int64_t)n * row_bytes + k];
  }
}

template <typename T, int LAYOUT>
static int launch_cvt1(dim3 grid, size_t smem, cudaStream_t st, const uint8_t* frames, const int32_t* action,
                       const double* reward, const int32_t* mask, int64_t row_bytes, const int64_t* idx, int hl, int n,
                       double discount, const float* lut, void* so, void* no, int64_t* a, float* r, float* m, int use_tma,
                       int frame_w) {
  auto k = gather_cvt_kernel<T, LAYOUT>;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  // plain stream order: with programmatic overlap the CTAs of back-to-back gathers are placed while the previous launch still
  // holds its slots, the placement is skewed and the launch gets slower
  launch_ordered(k, dim3(grid), dim3(256), smem, st, frames, action, reward, mask, row_bytes, idx, hl, n, discount, lut, (T*)so, (T*)no, a, r, m,
                             use_tma, frame_w);
  return check_launch("b2rl_replay_gather");
}

template <typename T>
static int launch_s2d_bulk(dim3 grid, cudaStream_t st, const uint8_t* frames, const int32_t* action, const double* reward,
                           const int32_t* mask, int64_t row_bytes, const int64_t* idx, int hl, int n, double discount,
                           void* so, void* no, int64_t* a, float* r, float* m, int frame_w) {
  const int positions = (frame_w / 4) * ((int)(row_bytes / frame_w) / 4);
  const int tile_pos = (positions + 2) / 3;
  const size_t span_al = ((size_t)(hl + n) * row_bytes + 127) & ~(size_t)127;
  const size_t smem = span_al + 2 * (size_t)tile_pos * hl * 16 * sizeof(T);
  if (smem > 200 * 1024) return 1;
  auto k = gather_s2d_bulk_kernel<T>;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  launch_ordered(k, dim3(grid), dim3(256), smem, st, frames, action, reward, mask, row_bytes, idx, hl, n, discount, (T*)so,
                 (T*)no, a, r, m, frame_w, tile_pos);
  return check_launch("b2rl_replay_gather(s2d bulk)");
}

template <typename T>
static int launch_cvt(int layout, dim3 grid, size_t smem, cudaStream_t st, const uint8_t* frames, const int32_t* action,
                      const double* reward, const int32_t* mask, int64_t row_bytes, const int64_t* idx, int hl, int n,
                      double discount, const float* lut, void* so, void* no, int64_t* a, float* r, float* m,
                      int use_tma, int frame_w) {
  if constexpr (sizeof(T) == 2) {
    static int bulk = -1;                                            // B2RL_GATHER_BULK=1: bulk-store variant (unverified)
    if (bulk < 0) {
      const char* e = getenv("B2RL_GATHER_BULK");
      bulk = (e && atoi(e) == 1) ? 1 : 0;
    }
    if (layout == 2 && bulk && use_tma && lut == nullptr) {
      int rc = launch_s2d_bulk<T>(grid, st, frames, action, reward, mask, row_bytes, idx, hl, n, discount, so, no, a, r, m,
                                  frame_w);
      if (rc <= 0) return rc;
    }
  }
  if (layout == 2)
    return launch_cvt1<T, 2>(grid, smem, st, frames, action, reward, mask, row_bytes, idx, hl, n, discount, lut, so, no,
                             a, r, m, use_tma, frame_w);
  if (layout == 1)
    return launch_cvt1<T, 1>(grid, smem, st, frames, action, reward, mask, row_bytes, idx, hl, n, discount, lut, so, no,
                             a, r, m, use_tma, frame_w);
  return launch_cvt1<T, 0>(grid, smem, st, frames, action, reward, mask, row_bytes, idx, hl, n, discount, lut, so, no, a,
                           r, m, use_tma, frame_w);
}

}  // namespace b2rl

using namespace b2rl;

extern "C" int b2rl_replay_feed(uint8_t* frames, int32_t* action, double* reward, int32_t* mask, int64_t* ring_state,
                                int64_t row_bytes, const uint8_t* new_frames, const int32_t* new_action,
                                const double* new_reward, const int32_t* new_mask, int32_t n, int32_t reference_quirk,
                                void* stream) {
  B2RL_REQUIRE(frames && action && reward && mask && ring_state && new_frames && new_action && new_reward && new_mask,
               "null pointer");
  B2RL_REQUIRE(n >= 0 && n <= 1024, "n must be in [0, 1024]");
  B2RL_REQUIRE(row_bytes > 0, "row_bytes must be positive");
  if (n == 0) return B2RL_OK;
  launch_pdl(feed_kernel, dim3(1), dim3(512), 0, (cudaStream_t)stream, frames, action, reward, mask, ring_state, row_bytes, new_frames,
                                                   new_action, new_reward, new_mask, n, reference_quirk);
  return check_launch("b2rl_replay_feed");
}

extern "C" int b2rl_replay_select_uniform(int64_t* ring_state, const int64_t* candidates, int32_t n_cand,
                                          uint64_t seed, int32_t history, int32_t n_step, int32_t B, int64_t* idx_out,
                                          int32_t* status_out, void* stream) {
  B2RL_REQUIRE(ring_state && idx_out && status_out, "null pointer");
  B2RL_REQUIRE(B > 0 && n_cand >= B && n_cand <= SEL_THREADS * SEL_PER_THREAD, "need B <= n_cand <= 8192");
  B2RL_REQUIRE(history >= 1 && n_step >= 1, "history and n_step must be >= 1");
  launch_pdl(select_uniform_kernel, dim3(1), dim3(SEL_THREADS), 0, (cudaStream_t)stream, ring_state, candidates, n_cand, seed, history,
                                                                      n_step, B, idx_out, status_out, (const int32_t*)nullptr,
             (const double*)nullptr, (const int32_t*)nullptr, 0.0, (int64_t*)nullptr, (float*)nullptr, (float*)nullptr);
  return check_launch("b2rl_replay_select_uniform");
}

extern "C" int b2rl_replay_select_uniform_scalars(int64_t* ring_state, const int64_t* candidates, int32_t n_cand,
                                                  uint64_t seed, int32_t history, int32_t n_step, int32_t B,
                                                  int64_t* idx_out, int32_t* status_out, const int32_t* action,
                                                  const double* reward, const int32_t* mask, double discount,
                                                  int64_t* action_out, float* reward_out, float* mask_out, void* stream) {
  B2RL_REQUIRE(ring_state && idx_out && status_out && action && reward && mask, "null pointer");
  B2RL_REQUIRE(action_out || reward_out || mask_out, "no scalar output: use b2rl_replay_select_uniform");
  B2RL_REQUIRE(B > 0 && n_cand >= B && n_cand <= SEL_THREADS * SEL_PER_THREAD, "need B <= n_cand <= 8192");
  B2RL_REQUIRE(history >= 1 && n_step >= 1, "history and n_step must be >= 1");
  launch_pdl(select_uniform_kernel, dim3(1), dim3(SEL_THREADS), 0, (cudaStream_t)stream, ring_state, candidates, n_cand, seed, history,
             n_step, B, idx_out, status_out, action, reward, mask, discount, action_out, reward_out, mask_out);
  return check_launch("b2rl_replay_select_uniform_scalars");
}

extern "C" int b2rl_replay_gather(const uint8_t* frames, const int32_t* action, const double* reward,
                                  const int32_t* mask, int64_t capacity, int64_t row_bytes, const int64_t* idx,
                                  int32_t B, int32_t history, int32_t n_step, double discount, const float* lut,
                                  int32_t out_dtype, int32_t layout, int32_t frame_w, void* state_out, void* next_out,
                                  int64_t* action_out, float* reward_out, float* mask_out, void* stream) {
  B2RL_REQUIRE(frames && action && reward && mask && idx, "null pointer");
  B2RL_REQUIRE(B > 0 && history >= 1 && n_step >= 1 && row_bytes > 0 && capacity > 0, "bad shape");
  B2RL_REQUIRE(out_dtype >= B2RL_U8 && out_dtype <= B2RL_F32, "bad out_dtype");
  B2RL_REQUIRE(!(out_dtype == B2RL_U8 && lut != nullptr), "a lut needs a converted (non-uint8) output dtype");
  B2RL_REQUIRE(layout >= 0 && layout <= 2, "layout must be 0 (NCHW), 1 (NHWC) or 2 (space-to-depth 4)");
  B2RL_REQUIRE(!(out_dtype == B2RL_U8 && layout != 0), "NHWC / space-to-depth need a converted dtype");
  B2RL_REQUIRE(layout != 2 || (frame_w > 0 && frame_w % 4 == 0 && row_bytes % frame_w == 0 && (row_bytes / frame_w) % 4 == 0),
               "space-to-depth needs frame_w and frame height multiples of 4");
  cudaStream_t st = (cudaStream_t)stream;
  if (!state_out && !next_out) {                                     // scalars only: the consumer reads the frames from the ring
    launch_pdl(gather_scalars_kernel, dim3((B + 127) / 128), dim3(128), 0, st, action, reward, mask, idx, B, n_step, discount,
               action_out, reward_out, mask_out);
    return check_launch("b2rl_replay_gather(scalars)");
  }
  const size_t span = (size_t)(history + n_step) * row_bytes;
  B2RL_REQUIRE(span <= 200 * 1024, "history+n_step rows do not fit in shared memory");
  const bool aligned = row_bytes % 16 == 0 && reinterpret_cast<uintptr_t>(frames) % 16 == 0;
  if (out_dtype == B2RL_U8) {
    const bool out_aligned = (reinterpret_cast<uintptr_t>(state_out) | reinterpret_cast<uintptr_t>(next_out)) % 16 == 0;
    if (aligned && out_aligned) {
      cudaFuncSetAttribute(gather_raw_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)span);
      launch_ordered(gather_raw_tma_kernel, dim3(B), dim3(32), span, st, frames, action, reward, mask, row_bytes, idx, history, n_step,
                                                 discount, (uint8_t*)state_out, (uint8_t*)next_out, action_out,
                                                 reward_out, mask_out);
    } else {
      launch_ordered(gather_raw_generic_kernel, dim3(B), dim3(128), 0, st, frames, action, reward, mask, row_bytes, idx, history, n_step,
                                                   discount, (uint8_t*)state_out, (uint8_t*)next_out, action_out,
                                                   reward_out, mask_out);
    }
    return check_launch("b2rl_replay_gather");
  }
  const size_t smem = (span + 15) / 16 * 16;
  const int use_tma = aligned ? 1 : 0;
  switch (out_dtype) {
    case B2RL_F16:
      return launch_cvt<__half>(layout, B, smem, st, frames, action, reward, mask, row_bytes, idx, history, n_step,
                                discount, lut, state_out, next_out, action_out, reward_out, mask_out, use_tma, frame_w);
    case B2RL_BF16:
      return launch_cvt<__nv_bfloat16>(layout, B, smem, st, frames, action, reward, mask, row_bytes, idx, history,
                                       n_step, discount, lut, state_out, next_out, action_out, reward_out, mask_out,
                                       use_tma, frame_w);
    default:
      return launch_cvt<float>(layout, B, smem, st, frames, action, reward, mask, row_bytes, idx, history, n_step,
                               discount, lut, state_out, next_out, action_out, reward_out, mask_out, use_tma, frame_w);
  }
}
