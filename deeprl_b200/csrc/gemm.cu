// gemm.cu -- persistent wgmma / TMA GEMM for the dense layers of the path: NatureConvBody convolutions as shifted-row
// implicit GEMMs, fc4, heads (network_bodies.py:27-33, network_heads.py:18-21), forward, dgrad and wgrad.
//
//   D[M,N] (+)= A[M,K] * B[N,K]^T        bf16 operands, fp32 accumulation in registers
//
// Operand storage is described per operand:
//   K-major  (major = 0): row-major [rows = M or N][K], K contiguous            (activations x weights: y = x W^T)
//   MN-major (major = 1): row-major [K][rows = M or N], M/N contiguous          (weight gradients: dW = g^T x)
// so no operand is ever transposed in memory.
//
// Convolutions without im2col ("tap addressing").  Activations live as [batch * G * G][C] matrices over a G x G grid
// per image.  A k x k / stride-1 convolution over that grid is  y[r] = sum_taps x[r + dy*G + dx] W_tap^T : the A operand
// of k-tile `kt` is the SAME matrix read at a row offset that depends on the tap the k-tile belongs to (rows that run
// off the grid produce garbage output rows, which the epilogue drops or the next layer never reads).  Stride-s
// convolutions are first turned into stride-1 ones by a space-to-depth(s) layout of their input, which the PRODUCING
// kernel writes directly (the replay gather for conv1, conv1's epilogue for conv2).  dgrad is the same with negative
// shifts; wgrad reads both operands MN-major with the tap shift applied to the B operand per output column block.
//
// One persistent CTA per SM loops over output tiles (128 x BN), in three warpgroups:
//   warpgroup 0      TMA producer: one ELECTED thread of warp 0 (elect.sync, see elect_one) issues cp.async.bulk.tensor
//                    into a STAGES-deep 128B-swizzled smem ring (mbarrier full/empty); warps 1-3 idle
//   warpgroups 1, 2  rows 0-63 / 64-127 of the tile: wgmma.mma_async m64nBNk16 (fp32 accumulators in registers), then the
//                    epilogue: accumulators -> shared staging tile -> 8 columns x BN/16 rows per thread, whole rows
//                    per warp instruction (epi_col / epi_row) -> bias / ReLU -> bf16 | fp32 | atomic fp32
// (the convolution slab kernel instead gives the MMAs to one warpgroup and the two halves' epilogues to two more: see
// conv_slab_body)
// Every kernel runs its prologue (barrier init, tensor-map prefetch) before pdl_sync(): under programmatic dependent launch
// that part overlaps the tail of the previous kernel (common.cuh).
// sm_90a only.
#include <cuda.h>
#include "common.cuh"
#include "wgmma.cuh"

namespace b2rl {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;           // 64 bf16 = 128 bytes = one swizzle-128B atom row
constexpr int GEMM_THREADS = 384;     // warpgroup 0: TMA producer, warpgroups 1 / 2: MMA + epilogue of rows 0-63 / 64-127
constexpr int MMA_WARPS = 8;          // a shared-memory stage is free again once every MMA warp has arrived on its barrier

__device__ __forceinline__ uint32_t s2u(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mb_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s2u(bar)), "r"(count));
}
__device__ __forceinline__ void mb_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s2u(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s2u(bar)) : "memory");
}
// try_wait with a suspend-time hint: the waiting thread sleeps in hardware until the phase completes instead of polling
// the barrier word
__device__ __forceinline__ void mb_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
      "@p bra LAB_DONE;\n"
      "bra LAB_WAIT;\n"
      "LAB_DONE:\n"
      "}\n" ::"r"(s2u(bar)), "r"(parity), "r"(0x989680u)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          s2u(smem_dst)),
      "l"(map), "r"(s2u(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// bulk prefetch of `bytes` (a multiple of 16, 16-byte aligned start) from global memory into L2
__device__ __forceinline__ void prefetch_l2_bulk(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
// One elected lane of a fully active warp: the single-thread producer role is entered through elect.sync rather than a
// plain `lane == 0` test, so that the compiler issues the TMA instructions without an ELECT / BRA.U.ANY loop around them.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "elect.sync _|p, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}
// named barriers: 0 = __syncthreads, 1 = the 256 MMA threads, 2 / 3 = MMA warpgroup 1 / 2, 4 = uint8 converters,
// 5 / 6 = half 0 / 1 of the slab kernel's staging tile written, 7 / 8 = half 0 / 1 read (SLAB_BAR_STAGED / SLAB_BAR_FREE)
__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// wgmma shared-memory matrix descriptor, 128B swizzle (layout type 1 in bits 62-63):
//   K-major : 8-row groups 1024 B apart (SBO), LBO unused
//   MN-major: 64-element MN groups `lbo` bytes apart, 8-K-row groups 1024 B apart (SBO)
// base_offset (bits 49-51) = (start address >> 7) & 7 for a start that is not aligned to the 1024-byte swizzle pattern;
// 0 when the swizzle is taken from the address itself (see the slab kernel).
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t base_offset = 0) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)(base_offset & 7) << 49) | ((uint64_t)1 << 62);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wg_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void acc_zero(float* d) {
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.0f;
}
// keeps the compiler from moving accumulator reads above wgmma.wait_group
template <int N>
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
  for (int i = 0; i < N / 2; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// the four k16 steps of one 64-wide k-tile; a step advances K-major operands 32 bytes along the swizzled row, MN-major ones
// 16 rows (2048 bytes) -- in 16-byte descriptor units 2 / 128
template <int N, int TA, int TB>
__device__ __forceinline__ void mma_ktile(float* d, uint64_t a, uint64_t b) {
#pragma unroll
  for (int k = 0; k < GEMM_BK / 16; ++k) {
    if constexpr (N == 32) wgmma_n32<TA, TB>(d, a + k * (TA ? 128 : 2), b + k * (TB ? 128 : 2));
    else if constexpr (N == 64) wgmma_n64<TA, TB>(d, a + k * (TA ? 128 : 2), b + k * (TB ? 128 : 2));
    else wgmma_n128<TA, TB>(d, a + k * (TA ? 128 : 2), b + k * (TB ? 128 : 2));
  }
}
// wgmma accumulator fragment of one warp (rows 16 wl .. 16 wl + 15 of the warpgroup's 64) -> rows of the staging tile `s`
template <int N>
__device__ __forceinline__ void stage_acc(const float* d, float* s, int ld, int wl, int lane) {
  const int r = 16 * wl + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    *reinterpret_cast<float2*>(s + r * ld + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(s + (r + 8) * ld + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}

struct GemmParams {
  int M, N, K;
  int ldd;                 // row stride of D in elements
  int k_tiles_per_split;   // K tiles (of 64) handled by one blockIdx.z
  int a_mn, b_mn;          // operand majors (0 = K-major, 1 = MN-major)
  int relu, out_mode;      // out_mode 0: bf16 store, 1: fp32 store, 2: fp32 atomicAdd (split-K / accumulate)
  const float* bias;       // [N] or null (added by split 0 only)
  void* D;
  // tap addressing (0 = plain GEMM)
  int a_tap_tiles;         // K-major A: k-tiles per tap (= channels / 64); the A matrix is [rows][a_tap_tiles*64]
  int b_tap_tiles;         // MN-major B (wgrad): output column tiles per tap (= channels / BN); B is [rows][b_tap_tiles*BN]
  int taps_x, grid_w, shift_sign;   // row shift of tap t = sign * ((t / taps_x) * grid_w + t % taps_x)
  // output row mapping (rows of the GEMM are positions of a G x G grid per image)
  int out_map;             // 0: identity; 1: G-grid -> space-to-depth(2) rows, valid V x V; 2: G-grid -> compact V x V
  int G, V;
  // dual launch: the same GEMM for two independent operand sets (online / target network) in ONE grid -- the first half of
  // the CTAs works on (tmA, tmB, D, bias), the second half on (tmA2, tmB2, D2, bias2); halves the per-kernel fixed cost
  int dual;
  void* D2;
  const float* bias2;
  // backward extras (see epilogue_half): ReLU-gradient mask, bias-gradient accumulation, grid scatter maps 3 / 4
  const __nv_bfloat16* mask;
  int64_t mask_ld;
  float* dbias;
  int dbias_mod, sub_c;
};

__device__ __forceinline__ int tap_shift(const GemmParams& p, int tap) {
  return p.shift_sign * ((tap / p.taps_x) * p.grid_w + tap % p.taps_x);
}

// accumulator staging tile of the epilogue: 128 rows x (BN + 8) fp32.  The 8-float pad puts consecutive rows 32 bytes apart
// in the bank pattern: the float2 writes of stage_acc (4 rows x 32 bytes per half-warp) and the float4 reads of
// epilogue_half (see there) are free of bank conflicts.
__host__ __device__ constexpr int acc_ld(int bn) { return bn + 8; }
__host__ __device__ constexpr size_t acc_stage_bytes(int bn) { return (size_t)GEMM_BM * acc_ld(bn) * 4; }

// Epilogue thread mapping: in a 64-row half of a 128 x BN tile, thread t (0..127 of the warpgroup) owns the 8 columns
// epi_col(t) .. + 7 of the rows epi_row(t, k), k = 0 .. BN/16 - 1.  BN/8 consecutive lanes cover one row, so one warp
// instruction covers 32 / (BN/8) whole consecutive rows: every 16-byte store or mask load of a warp is part of a contiguous
// run of BN * 2 bytes (bf16) per row -- or, for the scatter maps 3 / 4, of sub_c channels -- and a thread visits the same
// columns in every row, which lets it keep the bias-gradient column sums of a half in registers (dbias_flush).
template <int BN>
__device__ __forceinline__ int epi_col(int t) { return 8 * (t % (BN / 8)); }
template <int BN>
__device__ __forceinline__ int epi_row(int t, int k) { return t / (BN / 8) + k * (1024 / BN); }

// Backward extras (dgrad GEMMs): `mask` is the saved forward activation in the GEMM's own output coordinates -- the ReLU
// gradient is applied in the epilogue (v = mask > 0 ? v : 0); `dbias` receives the column sums of the masked tile (the bias
// gradient of the layer below), index = column % dbias_mod (dbias_mod 0: the column).  Output row maps 3 / 4 scatter the
// tile into the G x G grid matrix the next backward GEMMs read:
//   map 3: rows are space-to-depth(2) positions [b][oy][ox] of an (V/2)^2 grid, columns are 4 sub-positions x sub_c channels
//          -> grid row b*G*G + (2*oy + dy)*G + 2*ox + dx, column = channel           (conv2's input gradient -> conv1's grid)
//   map 4: rows are images b, columns are V*V positions x sub_c channels
//          -> grid row b*G*G + (pos / V)*G + pos % V, column = channel               (fc4's input gradient -> conv3's grid)
// Grid rows that no tile covers keep whatever the destination holds: the caller keeps it zeroed (persistent buffer).
//
// The ReLU-gradient mask of one 64-row half (rows row0 ..), requested into registers ahead of its use so that its round
// trip overlaps other work; the slab kernel's producer has prefetched it into L2 several tiles earlier.  A TMA ring of
// 64-row mask boxes in shared memory fits beside the dgrad slab kernels only by giving up slab stages (conv2, BN 128: two
// 16 KB boxes leave three of its five; conv3, BN 64: four 8 KB boxes leave four of six).  Built and measured that way, against the
// old epilogue in the same session, it took conv2's dgrad from 59.5 to 52.7 us per update where these register loads take
// it to 44.7 (from 60.1), and conv3's to 31.7 as these do to 31.1: the mask stays in global memory (DESIGN section 9).  fc4's dgrad, dense_gemm_kernel, has one tile per CTA.
// 16-byte shared-memory load through an explicit shared-space address (a generic pointer would go through the L1 path
// and hold a 64-bit address)
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
// 16-byte read-only global load issued exactly where it is written: an asm volatile statement keeps its order with the
// kernel's other asm volatile statements (barrier waits, wgmma), so the compiler cannot hoist it and its destination
// registers above the MMAs
__device__ __forceinline__ int4 ldg_v4_here(const void* ptr) {
  int4 v;
  asm volatile("ld.global.nc.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(ptr));
  return v;
}
// 8 floats rounded to bf16 (round to nearest even, as __floats2bfloat162_rn) and stored as one 16-byte group
__device__ __forceinline__ void stg_bf16x8(__nv_bfloat16* ptr, const float (&v)[8]) {
  asm volatile(
      "{\n"
      ".reg .b32 h<4>;\n"
      "cvt.rn.bf16x2.f32 h0, %2, %1;\n"
      "cvt.rn.bf16x2.f32 h1, %4, %3;\n"
      "cvt.rn.bf16x2.f32 h2, %6, %5;\n"
      "cvt.rn.bf16x2.f32 h3, %8, %7;\n"
      "st.global.v4.b32 [%0], {h0, h1, h2, h3};\n"
      "}\n" ::"l"(ptr), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7])
      : "memory");
}
template <int BN, bool EXT>
__device__ __forceinline__ void epi_mask_load(const GemmParams& p, int row0, int n0, int t, int4 (&m)[BN / 16]) {
  if constexpr (EXT) {
    const int n = n0 + epi_col<BN>(t);
#pragma unroll
    for (int k = 0; k < BN / 16; ++k) {
      const int row = row0 + epi_row<BN>(t, k);
      m[k] = make_int4(0, 0, 0, 0);
      if (p.mask && row < p.M && n < p.N) m[k] = ldg_v4_here(p.mask + (int64_t)row * p.mask_ld + n);
    }
  }
}

// The bias-gradient sums a thread has kept for its 8 columns n0 + epi_col(t) .. + 7 -> added up over the lanes of the warp
// that share those columns, then one shared-memory atomic per column and warp (BN / 32 instructions) into the per-CTA
// accumulator s_dbias (index column % dbias_mod, or the column itself for dbias_mod 0), which the kernel adds to global
// memory once at its end (dbias_slots).  dbias_mod 0 columns past 128 (plain GEMMs only) go to global memory directly.
// All 32 lanes take part.
template <int BN>
__device__ __forceinline__ void dbias_flush(const GemmParams& p, int n0, int t, float (&dsum)[8], float* s_dbias) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int s = BN / 8; s < 32; s <<= 1) dsum[j] += __shfl_xor_sync(0xffffffffu, dsum[j], s);
  }
  // lanes 0 .. BN/8 - 1 now hold the warp's sums of columns 8 lane .. + 7; spread them one column per lane, so that each
  // shared-memory atomic instruction covers 32 distinct columns
  const int lane = t & 31;
#pragma unroll
  for (int r = 0; r < BN / 32; ++r) {
    const int v = 32 * r + lane;
    float x = 0.0f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float y = __shfl_sync(0xffffffffu, dsum[j], v >> 3);
      if (j == (v & 7)) x = y;
    }
    const int col = n0 + v;
    if (col < p.N) {
      const int i = p.dbias_mod > 0 ? col % p.dbias_mod : col;
      if (i < 128) atomicAdd(s_dbias + i, x);
      else atomicAdd(p.dbias + col, x);
    }
  }
}
// entries of s_dbias a CTA adds to global memory at its end
__device__ __forceinline__ int dbias_slots(const GemmParams& p) { return p.dbias_mod > 0 ? p.dbias_mod : min(p.N, 128); }

// Row part of a destination offset (element index of the row's column 0 in D), or -1 for a row that is not stored: rows
// past M, grid positions outside the valid V x V (maps 1 / 2)
template <bool EXT>
__device__ __forceinline__ int64_t epi_row_base(const GemmParams& p, int row) {
  if (row >= p.M) return -1;
  if (p.out_map == 1 || p.out_map == 2) {
    const int gg = p.G * p.G;
    const int bi = row / gg, rem = row - bi * gg;
    const int oy = rem / p.G, ox = rem - oy * p.G;
    if (oy >= p.V || ox >= p.V) return -1;
    if (p.out_map == 2) return ((int64_t)bi * p.V * p.V + oy * p.V + ox) * p.ldd;
    const int h = p.V >> 1;
    return ((int64_t)bi * h * h + (oy >> 1) * h + (ox >> 1)) * p.ldd + (((oy & 1) << 1) | (ox & 1)) * p.N;
  }
  if (EXT && p.out_map == 3) {
    const int h = p.V >> 1, hh = h * h;
    const int img = row / hh, rem = row - img * hh;
    const int sy = rem / h, sx = rem - sy * h;
    return ((int64_t)img * p.G * p.G + 2 * sy * p.G + 2 * sx) * p.ldd;
  }
  if (EXT && p.out_map == 4) return (int64_t)row * p.G * p.G * p.ldd;
  return (int64_t)row * p.ldd;
}
// Column part of a destination offset for column n (maps 3 / 4: sub_c is a multiple of 32, so 8 columns share one sub-position)
template <bool EXT>
__device__ __forceinline__ int64_t epi_col_off(const GemmParams& p, int n) {
  if (EXT && p.out_map == 3) {
    const int sub = n / p.sub_c, cc = n - sub * p.sub_c;
    return (int64_t)((sub >> 1) * p.G + (sub & 1)) * p.ldd + cc;
  }
  if (EXT && p.out_map == 4) {
    const int pos = n / p.sub_c, cc = n - pos * p.sub_c;
    return (int64_t)((pos / p.V) * p.G + pos % p.V) * p.ldd + cc;
  }
  return n;
}

// Epilogue of one 64-row half of a 128 x BN tile (first row row0, first column n0) for warpgroup thread t: `s` is the
// half's fp32 staging tile, `m` its mask (epi_mask_load).  The bias-gradient column sums of the half stay in registers
// (dsum: the thread's 8 columns over its BN/16 rows) until one dbias_flush at the end.  The general form of the plain and
// tap-addressing GEMMs (every output mode and column count); the convolution slab kernels use slab_epilogue_half.
template <int BN, bool EXT>
__device__ __forceinline__ void epilogue_half(const GemmParams& p, int row0, int n0, int t, const float* s,
                                              const int4 (&m)[BN / 16], float* s_dbias) {
  constexpr int ACC_LD = acc_ld(BN);
  float dsum[8] = {};
  const int c = epi_col<BN>(t);
  const int n = n0 + c;
  const float* bias = p.bias;
  void* D = p.D;
  const bool cols = n < p.N, full = n + 8 <= p.N;
  const bool add_bias = bias && blockIdx.z == 0 && cols;
  float b[8];
  if (add_bias) {
    const float* bp = bias + n;
    if (full && (reinterpret_cast<uintptr_t>(bp) & 15) == 0) {
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(bp)), b1 = __ldg(reinterpret_cast<const float4*>(bp + 4));
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = n + j < p.N ? __ldg(bp + j) : 0.0f;
    }
  }
  // the 8 lanes of a 128-bit shared-memory access phase read distinct banks when the half of the 8 columns a lane reads
  // first alternates with column group (BN 64 / 128: 8 lanes on one row) and with the row (BN 32: 4 lanes on each of two
  // rows 32 bytes apart in the bank pattern); the rows of one thread all have the same parity
  const int h0 = ((c >> 5) ^ epi_row<BN>(t, 0)) & 1;
  const uint32_t s_base = s2u(s);
  // destination offset = row part + column part: the column part is the same in every row of the thread; the row part
  // (integer divisions for the maps) is computed once per row of the warp, by lane q for the warp's q-th row (pass
  // q / (32 / (BN/8)), row q % (32 / (BN/8)) of the pass), and handed to the lanes of that row by a shuffle
  const int64_t coff = epi_col_off<EXT>(p, n);
  int64_t rbase = -1;
  if ((t & 31) < 16) {
    constexpr int RPW = 256 / BN;                                     // rows per warp instruction
    const int q = t & 31;
    rbase = epi_row_base<EXT>(p, row0 + (t >> 5) * RPW + q % RPW + (q / RPW) * 4 * RPW);
  }
#pragma unroll
  for (int k = 0; k < BN / 16; ++k) {
    const int rl = epi_row<BN>(t, k);
    const uint32_t sp = s_base + (uint32_t)(rl * ACC_LD + c) * 4;
    const float4 x = lds128(sp + 16 * h0), y = lds128(sp + 16 * (h0 ^ 1));
    const float4 lo = h0 ? y : x, hi = h0 ? x : y;
    float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    const int64_t base = __shfl_sync(0xffffffffu, rbase, k * (256 / BN) + (t & 31) / (BN / 8));
    const int64_t off = base + coff;
    if (!(base >= 0 && cols)) continue;
    if (add_bias) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (full || n + j < p.N) v[j] += b[j];
    }
    if (p.relu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.0f);
    }
    if constexpr (EXT) {
      if (p.mask) {                                                     // ReLU gradient: zero where the forward output was <= 0
        const __nv_bfloat162* mh = reinterpret_cast<const __nv_bfloat162*>(&m[k]);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 mf = __bfloat1622float2(mh[q]);
          if (!(mf.x > 0.0f)) v[2 * q] = 0.0f;
          if (!(mf.y > 0.0f)) v[2 * q + 1] = 0.0f;
        }
      }
      if (p.dbias) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (full || n + j < p.N) dsum[j] += v[j];
      }
    }
    if (p.out_mode == 0) {
      __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(D) + off;
      if (full && off % 8 == 0) {
        int4 o;
        __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
        for (int q = 0; q < 4; ++q) h[q] = __floats2bfloat162_rn(v[2 * q], v[2 * q + 1]);
        *reinterpret_cast<int4*>(d) = o;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (n + j < p.N) d[j] = __float2bfloat16_rn(v[j]);
      }
    } else if (p.out_mode == 1) {
      float* d = reinterpret_cast<float*>(D) + off;
      if (full && off % 4 == 0) {
        *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(d + 4) = make_float4(v[4], v[5], v[6], v[7]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (n + j < p.N) d[j] = v[j];
      }
    } else {
      float* d = reinterpret_cast<float*>(D) + off;
      if (full && (reinterpret_cast<uintptr_t>(d) & 15) == 0) {
        atomicAdd(reinterpret_cast<float4*>(d), make_float4(v[0], v[1], v[2], v[3]));
        atomicAdd(reinterpret_cast<float4*>(d + 4), make_float4(v[4], v[5], v[6], v[7]));
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (n + j < p.N) atomicAdd(d + j, v[j]);
      }
    }
  }
  if (EXT && p.dbias) dbias_flush<BN>(p, n0, t, dsum, s_dbias);
}

// Rows of one pass of slab_epilogue_half: all of a thread's BN/16 rows, except where their staged values and masks do
// not fit beside the rest in the epilogue warpgroup's registers (BN 128 with the mask: 32 registers of mask) -- two passes
template <int BN, bool EXT>
__host__ __device__ constexpr int slab_epi_pass_rows() { return EXT && BN == 128 ? BN / 32 : BN / 16; }

// The epilogue of the convolution slab kernels (conv_slab_body), on the same thread mapping as epilogue_half.  The launchers
// give these kernels one output form (conv_gemm_impl, b2rl_conv1_u8_fwd / _pair): bf16 in whole 16-byte column groups (N and
// ldd multiples of 8, D and D2 16-byte aligned, columns 0 .. N - 1 from n0 = 0), forwards with ReLU (bias optional) and no
// extras, EXT dgrads with mask and bias gradient, no bias, no ReLU.  So each row is one 16-byte store and the per-row tests
// of epilogue_half are gone.  Every staged value of a pass (two 16-byte loads per row) and every row base is requested
// before the first is used: a pass waits for one shared-memory round trip, not one per row.  The arithmetic of each element
// and the order of the dsum additions (rows k = 0, 1, ...) are those of epilogue_half, so every output has the same bits.
// PAIR (paired conv1 forward): tile columns 0 .. BN/2 - 1 are columns of (D, bias), BN/2 .. BN - 1 those of (D2, bias2);
// p.N = BN / 2.
template <int BN, bool EXT, bool PAIR>
__device__ __forceinline__ void slab_epilogue_half(const GemmParams& p, int row0, int t, const float* s,
                                                   const int4 (&m)[BN / 16], float* s_dbias) {
  constexpr int ACC_LD = acc_ld(BN);
  constexpr int ROWS = BN / 16, PASS = slab_epi_pass_rows<BN, EXT>();
  float dsum[8] = {};
  const int c = epi_col<BN>(t);
  const bool second = PAIR && c >= BN / 2;                    // the thread's 8 columns all lie in one half
  const int n = c - (second ? BN / 2 : 0);
  __nv_bfloat16* D = reinterpret_cast<__nv_bfloat16*>(second ? p.D2 : p.D);
  const bool cols = n < p.N;
  const float* bias = second ? p.bias2 : p.bias;
  const bool add_bias = !EXT && bias && cols;
  float b[8];
  if (add_bias) {
    const float* bp = bias + n;
    if ((reinterpret_cast<uintptr_t>(bp) & 15) == 0) {
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(bp)), b1 = __ldg(reinterpret_cast<const float4*>(bp + 4));
      b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = __ldg(bp + j);
    }
  }
  // bank-conflict-free order of the two 16-byte reads and the row bases handed over by lane: as in epilogue_half
  const int h0 = ((c >> 5) ^ epi_row<BN>(t, 0)) & 1;
  const uint32_t s_base = s2u(s);
  const int64_t coff = epi_col_off<EXT>(p, n);
  int64_t rbase = -1;
  if ((t & 31) < 16) {
    constexpr int RPW = 256 / BN;
    const int q = t & 31;
    rbase = epi_row_base<EXT>(p, row0 + (t >> 5) * RPW + q % RPW + (q / RPW) * 4 * RPW);
  }
#pragma unroll
  for (int k0 = 0; k0 < ROWS; k0 += PASS) {
    float4 x[PASS], y[PASS];
    int64_t base[PASS];
#pragma unroll
    for (int i = 0; i < PASS; ++i) {
      const uint32_t sp = s_base + (uint32_t)(epi_row<BN>(t, k0 + i) * ACC_LD + c) * 4;
      x[i] = lds128(sp + 16 * h0);
      y[i] = lds128(sp + 16 * (h0 ^ 1));
    }
#pragma unroll
    for (int i = 0; i < PASS; ++i) base[i] = __shfl_sync(0xffffffffu, rbase, (k0 + i) * (256 / BN) + (t & 31) / (BN / 8));
    // a warp barrier between the requests and their first use: without it the compiler hoists a row's stores above the
    // loads of the rows after it (forward kernels), and the pass waits for the shared-memory round trip more than once
    __syncwarp();
#pragma unroll
    for (int i = 0; i < PASS; ++i) {
      const int k = k0 + i;
      const float4 lo = h0 ? y[i] : x[i], hi = h0 ? x[i] : y[i];
      float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
      // rows that are not stored are computed too and only their store and sum are dropped: a branch around the row would
      // let the compiler sink its shared-memory loads into it, back behind the previous row's store
      const bool store = base[i] >= 0 && cols;
      if constexpr (EXT) {
        const __nv_bfloat162* mh = reinterpret_cast<const __nv_bfloat162*>(&m[k]);   // ReLU gradient
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 mf = __bfloat1622float2(mh[q]);
          if (!(mf.x > 0.0f)) v[2 * q] = 0.0f;
          if (!(mf.y > 0.0f)) v[2 * q + 1] = 0.0f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) dsum[j] = store ? dsum[j] + v[j] : dsum[j];
      } else {
        if (add_bias) {
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] += b[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.0f);
      }
      if (store) stg_bf16x8(D + base[i] + coff, v);
    }
  }
  if constexpr (EXT) dbias_flush<BN>(p, 0, t, dsum, s_dbias);
}

template <int BN, int STAGES, bool EXT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                     const __grid_constant__ CUtensorMap tmB,
                                                                     const __grid_constant__ CUtensorMap tmA2,
                                                                     const __grid_constant__ CUtensorMap tmB2,
                                                                     const GemmParams p0) {
  const int n_cta = p0.dual ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  const bool second = p0.dual && (int)blockIdx.x >= n_cta;
  const int cta = second ? (int)blockIdx.x - n_cta : (int)blockIdx.x;
  const CUtensorMap* mA = second ? &tmA2 : &tmA;
  const CUtensorMap* mB = second ? &tmB2 : &tmB;
  GemmParams p = p0;
  if (second) { p.D = p0.D2; p.bias = p0.bias2; }
  constexpr uint32_t A_BYTES = GEMM_BM * GEMM_BK * 2, B_BYTES = BN * GEMM_BK * 2;
  constexpr int ACC_LD = acc_ld(BN);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  float* sAcc = reinterpret_cast<float*>(sB + STAGES * B_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(sAcc + GEMM_BM * ACC_LD);
  uint64_t* empty = full + STAGES;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
  const int m_tiles = (p.M + GEMM_BM - 1) / GEMM_BM, n_tiles = (p.N + BN - 1) / BN;
  const int tiles = m_tiles * n_tiles;
  const int kt_total = (p.K + GEMM_BK - 1) / GEMM_BK;
  const int kt_begin = blockIdx.z * p.k_tiles_per_split;
  const int kt_end = min(kt_total, kt_begin + p.k_tiles_per_split);
  const int n_kt = max(kt_end - kt_begin, 0);

  __shared__ float s_dbias[128];                    // per-CTA bias-gradient accumulator (backward extras)
  if (threadIdx.x < 128) s_dbias[threadIdx.x] = 0.0f;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mb_init(&full[s], 1); mb_init(&empty[s], MMA_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(mA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(mB) : "memory");
  }
  __syncthreads();
  pdl_sync();   // everything above (barriers, tensor-map prefetch) overlaps the previous kernel's tail

  if (warp == 0 && n_kt > 0 && elect_one()) {
    // ---------------------------------------------------------------------- TMA producer
    uint32_t it = 0;                                         // global k-iteration counter across tiles
    for (int tile = cta; tile < tiles; tile += n_cta) {
      const int mt = tile / n_tiles, nt = tile - mt * n_tiles;
      const int m0 = mt * GEMM_BM, n0 = nt * BN;
      int b_shift = 0, b_col = n0;
      if (p.b_tap_tiles > 0) {                               // wgrad: the tap is selected by the output column block
        const int tap = nt / p.b_tap_tiles;
        b_shift = tap_shift(p, tap);
        b_col = (nt - tap * p.b_tap_tiles) * BN;
      }
      for (int i = 0; i < n_kt; ++i, ++it) {
        const int s = it % STAGES;
        mb_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
        mb_expect_tx(&full[s], A_BYTES + B_BYTES);
        const int g = kt_begin + i;
        uint8_t* a = sA + s * A_BYTES;
        uint8_t* b = sB + s * B_BYTES;
        if (!p.a_mn) {
          int ak = g * GEMM_BK, arow = m0;
          if (p.a_tap_tiles > 0) {
            const int tap = g / p.a_tap_tiles;
            ak = (g - tap * p.a_tap_tiles) * GEMM_BK;
            arow = m0 + tap_shift(p, tap);
          }
          tma_load_2d(a, mA, &full[s], ak, arow);                       // box [128 rows][64 k]
        } else {
          tma_load_2d(a, mA, &full[s], m0, g * GEMM_BK);                // 2 boxes [64 k][64 m]
          tma_load_2d(a + 8192, mA, &full[s], m0 + 64, g * GEMM_BK);
        }
        if (!p.b_mn) {
          tma_load_2d(b, mB, &full[s], g * GEMM_BK, n0);                // box [BN rows][64 k]
        } else {
#pragma unroll
          for (int q = 0; q < (BN + 63) / 64; ++q)
            tma_load_2d(b + q * 8192, mB, &full[s], b_col + q * 64, g * GEMM_BK + b_shift);
        }
      }
    }
  } else if (warp >= 4) {
    // ---------------------------------------------------------------------- MMA + epilogue, warpgroup g: rows 64 g .. 64 g + 63
    // (K-major A: rows 64.. start 64 x 128 bytes into the stage; MN-major A: the second [64 k][64 m] box)
    const int cw = warp - 4, g = cw >> 2, wl = cw & 3;
    const int t = wl * 32 + lane;                                          // epilogue_half's thread index in the warpgroup
    float* sAcc_g = sAcc + g * 64 * ACC_LD;
    const uint64_t a0 = make_desc(s2u(sA) + g * 8192, 8192), b0 = make_desc(s2u(sB), 8192);
    uint32_t it = 0;
    for (int tile = cta; tile < tiles; tile += n_cta) {
      const int mt = tile / n_tiles, nt = tile - mt * n_tiles;
      const int m0 = mt * GEMM_BM, n0 = nt * BN;
      float d[BN / 2];
      acc_zero<BN>(d);
      for (int i = 0; i < n_kt; ++i, ++it) {
        const int s = it % STAGES;
        mb_wait(&full[s], (it / STAGES) & 1);
        const uint64_t a = a0 + (uint64_t)s * (A_BYTES >> 4), b = b0 + (uint64_t)s * (B_BYTES >> 4);
        wg_fence();
        if (!p.a_mn) {
          if (!p.b_mn) mma_ktile<BN, 0, 0>(d, a, b);
          else mma_ktile<BN, 0, 1>(d, a, b);
        } else {
          if (!p.b_mn) mma_ktile<BN, 1, 0>(d, a, b);
          else mma_ktile<BN, 1, 1>(d, a, b);
        }
        wg_commit();
        wg_wait0();
        acc_fence<BN>(d);
        if (lane == 0) mb_arrive(&empty[s]);
      }
      int4 mk[BN / 16];
      epi_mask_load<BN, EXT>(p, m0 + 64 * g, n0, t, mk);     // in flight during the staging (fc4 dgrad: one tile per CTA)
      stage_acc<BN>(d, sAcc_g, ACC_LD, wl, lane);
      named_sync(2 + g, 128);
      epilogue_half<BN, EXT>(p, m0 + 64 * g, n0, t, sAcc_g, mk, s_dbias);
      named_sync(2 + g, 128);                        // staging tile read: the next tile may overwrite it
    }
  }
  __syncthreads();
  if (EXT && p0.dbias && (int)threadIdx.x < dbias_slots(p0)) atomicAdd(p0.dbias + threadIdx.x, s_dbias[threadIdx.x]);
}

// ---------------------------------------------------------------------------------------------------------------
// Plain GEMM (no tap addressing): fc4 forward / dgrad / weight gradient and the distributional heads.  Same roles, ring and
// epilogue as gemm_wgmma_kernel, with two differences:
//  * the operand majors TA / TB are template parameters, so a tile's k-tiles form one chain of wgmmas of one shape.  Each
//    k-tile is one commit group: after issuing k-tile i a warpgroup waits for k-tile i - 1 only (wgmma.wait_group 1) and
//    releases its stage, and it drains once per tile, so its MMAs overlap the next k-tile's barrier wait and issue.
//  * cluster split-K: launched with clusters of S > 1 CTAs (one output tile per cluster), CTA rank r computes the tile over
//    k-tiles [r kps, (r + 1) kps) and stages its partial accumulators in its own shared memory.  After a cluster barrier
//    each CTA adds, for its 128 / S rows of the tile, the S partials in rank order through distributed shared memory (the
//    sum is the same in every launch), and a second barrier ends all remote reads.  The CTA then runs the epilogue on its
//    rows only: one launch, no global workspace, no atomics.  Without a cluster (S = 1) the CTAs are persistent over the
//    tiles, and blockIdx.z selects the k range of an atomic split-K (out_mode 2).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_size() {
  uint32_t n;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(n));
  return n;
}
// every thread of every CTA of the cluster arrives (release: its shared-memory writes become visible to the cluster) and
// waits for all others (acquire)
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// 16 bytes at shared-memory address `addr` of cluster CTA `rank`
__device__ __forceinline__ float4 ld_dsmem128(uint32_t addr, uint32_t rank) {
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(addr), "r"(rank));
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(ra) : "memory");
  return v;
}

constexpr int DENSE_MAX_CLUSTER = 8;

template <int BN, int STAGES, int TA, int TB, bool EXT>
__global__ void __launch_bounds__(GEMM_THREADS, 1) dense_gemm_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                     const __grid_constant__ CUtensorMap tmB,
                                                                     const GemmParams p) {
  constexpr uint32_t A_BYTES = GEMM_BM * GEMM_BK * 2, B_BYTES = BN * GEMM_BK * 2;
  constexpr int ACC_LD = acc_ld(BN);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_BYTES;
  float* sAcc = reinterpret_cast<float*>(sB + STAGES * B_BYTES);
  uint64_t* full = reinterpret_cast<uint64_t*>(sAcc + GEMM_BM * ACC_LD);
  uint64_t* empty = full + STAGES;

  const int S = (int)cluster_size(), rank = (int)cluster_rank();   // 1 / 0 without a cluster launch
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int n_tiles = (p.N + BN - 1) / BN, tiles = ((p.M + GEMM_BM - 1) / GEMM_BM) * n_tiles;
  const int n_cta = (int)gridDim.x / S, cta = (int)blockIdx.x / S;
  const int kt_total = (p.K + GEMM_BK - 1) / GEMM_BK;
  const int kt_begin = (S > 1 ? rank : (int)blockIdx.z) * p.k_tiles_per_split;
  const int n_kt = max(min(kt_total, kt_begin + p.k_tiles_per_split) - kt_begin, 0);

  __shared__ float s_dbias[128];
  if (threadIdx.x < 128) s_dbias[threadIdx.x] = 0.0f;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mb_init(&full[s], 1); mb_init(&empty[s], MMA_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  __syncthreads();
  pdl_sync();

  if (warp == 0 && n_kt > 0 && elect_one()) {
    // ---------------------------------------------------------------------- TMA producer
    uint32_t it = 0;
    for (int tile = cta; tile < tiles; tile += n_cta) {
      const int mt = tile / n_tiles;
      const int m0 = mt * GEMM_BM, n0 = (tile - mt * n_tiles) * BN;
      for (int i = 0; i < n_kt; ++i, ++it) {
        const int s = it % STAGES;
        mb_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
        mb_expect_tx(&full[s], A_BYTES + B_BYTES);
        const int k0 = (kt_begin + i) * GEMM_BK;
        uint8_t* a = sA + s * A_BYTES;
        uint8_t* b = sB + s * B_BYTES;
        if constexpr (!TA) {
          tma_load_2d(a, &tmA, &full[s], k0, m0);                        // box [128 rows][64 k]
        } else {
          tma_load_2d(a, &tmA, &full[s], m0, k0);                        // 2 boxes [64 k][64 m]
          tma_load_2d(a + 8192, &tmA, &full[s], m0 + 64, k0);
        }
        if constexpr (!TB) {
          tma_load_2d(b, &tmB, &full[s], k0, n0);                        // box [BN rows][64 k]
        } else {
#pragma unroll
          for (int q = 0; q < BN / 64; ++q) tma_load_2d(b + q * 8192, &tmB, &full[s], n0 + q * 64, k0);
        }
      }
    }
  } else if (warp >= 4) {
    // ---------------------------------------------------------------------- MMA + epilogue, warpgroup g: rows 64 g .. 64 g + 63
    const int cw = warp - 4, g = cw >> 2, wl = cw & 3;
    const int t = wl * 32 + lane;
    const uint64_t a0 = make_desc(s2u(sA) + g * 8192, 8192), b0 = make_desc(s2u(sB), 8192);
    uint32_t it = 0;
    for (int tile = cta; tile < tiles; tile += n_cta) {
      const int mt = tile / n_tiles;
      const int m0 = mt * GEMM_BM, n0 = (tile - mt * n_tiles) * BN;
      float d[BN / 2];
      acc_zero<BN>(d);
      for (int i = 0; i < n_kt; ++i, ++it) {
        const int s = it % STAGES;
        mb_wait(&full[s], (it / STAGES) & 1);
        wg_fence();
        mma_ktile<BN, TA, TB>(d, a0 + (uint64_t)s * (A_BYTES >> 4), b0 + (uint64_t)s * (B_BYTES >> 4));
        wg_commit();
        wg_wait1();                                          // k-tile i - 1 has retired: release its stage
        if (i > 0 && lane == 0) mb_arrive(&empty[(it - 1) % STAGES]);
      }
      wg_wait0();
      acc_fence<BN>(d);
      if (n_kt > 0 && lane == 0) mb_arrive(&empty[(it - 1) % STAGES]);
      float* sAcc_g = sAcc + g * 64 * ACC_LD;
      if (S > 1) {                                           // partial tile: reduced across the cluster below
        stage_acc<BN>(d, sAcc_g, ACC_LD, wl, lane);
        continue;
      }
      int4 mk[BN / 16];
      epi_mask_load<BN, EXT>(p, m0 + 64 * g, n0, t, mk);
      stage_acc<BN>(d, sAcc_g, ACC_LD, wl, lane);
      named_sync(2 + g, 128);
      epilogue_half<BN, EXT>(p, m0 + 64 * g, n0, t, sAcc_g, mk, s_dbias);
      named_sync(2 + g, 128);                                // staging tile read: the next tile may overwrite it
    }
  }
  if (S > 1) {
    // one tile per cluster (the launcher sizes the grid so): every thread of the CTA takes part in both cluster barriers
    const int R = GEMM_BM / S;                               // rows of the tile this CTA reduces and stores
    const int mt = cta / n_tiles;
    const int m0 = mt * GEMM_BM, n0 = (cta - mt * n_tiles) * BN;
    const int g = (warp - 4) >> 2, t = (warp & 3) * 32 + lane, tid = (int)threadIdx.x - 128;
    // warpgroup g stores rows R/2 g .. R/2 g + R/2 - 1 of the CTA's rows: the half-tile epilogue with the rows past them cut off
    GemmParams pe = p;
    const int row0 = m0 + rank * R + g * (R / 2);
    pe.M = min(p.M, row0 + R / 2);
    int4 mk[BN / 16];
    if (warp >= 4) epi_mask_load<BN, EXT>(pe, row0, n0, t, mk);
    cluster_sync();                                          // every CTA's partial tile is staged
    // An MMA thread owns BN / (8 S) float4s of the CTA's R x BN rows (e = tid + 256 j; at BN 32, S 8 half the threads own one)
    // and loads each from all S ranks: slot f = S j + q, all issued before the first add so that their remote latencies
    // overlap.  Then each slot adds its predecessor's sum (rank order: the same sum in every launch); slot S j + S - 1 ends
    // with float4 j.
    constexpr int NL = BN / 8 > DENSE_MAX_CLUSTER ? BN / 8 : DENSE_MAX_CLUSTER;
    const int ls = __ffs(S) - 1;
    float4 x[NL];
    const uint32_t base = s2u(sAcc);
    if (warp >= 4) {
#pragma unroll
      for (int f = 0; f < NL; ++f) {
        const int e = tid + 256 * (f >> ls), r = e / (BN / 4), c = 4 * (e % (BN / 4));
        x[f] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (r < R) x[f] = ld_dsmem128(base + (uint32_t)(((rank * R + r) * ACC_LD + c) * 4), (uint32_t)(f & (S - 1)));
      }
#pragma unroll
      for (int f = 1; f < NL; ++f) {
        if (f & (S - 1)) { x[f].x += x[f - 1].x; x[f].y += x[f - 1].y; x[f].z += x[f - 1].z; x[f].w += x[f - 1].w; }
      }
    }
    cluster_sync();                                          // no CTA reads another's staging tile any more
    if (warp >= 4) {
#pragma unroll
      for (int f = 0; f < NL; ++f) {
        const int e = tid + 256 * (f >> ls), r = e / (BN / 4), c = 4 * (e % (BN / 4));
        if ((f & (S - 1)) == S - 1 && r < R) *reinterpret_cast<float4*>(sAcc + r * ACC_LD + c) = x[f];   // compacted: rows 0 .. R-1
      }
      named_sync(1, 256);
      epilogue_half<BN, EXT>(pe, row0, n0, t, sAcc + g * (R / 2) * ACC_LD, mk, s_dbias);
    }
  }
  __syncthreads();
  if (EXT && p.dbias && (int)threadIdx.x < dbias_slots(p)) atomicAdd(p.dbias + threadIdx.x, s_dbias[threadIdx.x]);
}


// ---------------------------------------------------------------------------------------------------------------
// Slab variant of the forward / dgrad convolution GEMM: the taps of a tile read overlapping row windows of the same
// activation matrix, so the CTA loads ONE slab of 128 + max_shift rows per tile and issues every tap's MMAs on windows
// that start `shift` rows (x 128 bytes) into that swizzled slab.  The 128-byte swizzle is a pure function of the shared
// memory ADDRESS (bits 4-6 ^= bits 7-9), for TMA writes and wgmma reads alike, so a window may start at any row of a
// 1024-byte-aligned slab with descriptor base_offset = 0 (base_offset_mode 2; mode 1 sets (start >> 7) & 7 instead).  The
// weights (all taps) are loaded once per CTA and stay resident.  Activation traffic drops by the number of taps (4x
// conv1/conv2, 9x conv3) and the weight traffic per tile to zero.
// ---------------------------------------------------------------------------------------------------------------
// K1: fused replay gather -> exact u8->bf16 -> conv1 operand.  Instead of reading a materialised bf16 space-to-depth matrix
// (57.8 MB per batch-512 stack, written by the gather kernel and re-read here), conv1's forward and weight-gradient kernels
// build their activation slabs themselves from the uint8 frame ring: four converter warps read, for every slab row
// (b, gy, gx) and 16-byte chunk j (8 channels = frame j/2, pixel rows 4gy + 2(j&1) + {0,1}, pixel columns 4gx..4gx+3), two
// aligned 32-bit words of the ring, convert the eight pixels exactly (integers 0..255 are representable in bf16; the 1/255
// of ImageNormalizer is folded into conv1's weights) and store one 16-byte chunk at the 128-byte-swizzled position
// (chunk ^ (row & 7)) the TMA would have written.  Reference chain replaced: replay.py:124-134 (frame-stack gather),
// normalizer.py:58-61, network_bodies.py:27.
// ---------------------------------------------------------------------------------------------------------------
struct U8Src {
  const uint8_t* frames;     // ring [capacity][row_bytes]
  const int64_t* idx;        // sampled ring indices [batch]
  int64_t row_bytes;         // bytes per ring row (84 * 84)
  int first;                 // ring row of channel-frame 0 relative to idx[b]: -(history-1) for s, n_step-(history-1) for s'
  int frame_w;               // pixels per frame row (84)
  int G;                     // grid width = frame_w / 4 (21); slab rows are (b, gy, gx) over G x G positions per image
  int rows;                  // batch * G * G
  int stages;                // uint8 staging tiles in flight (set by the launcher, <= U8_MAX_STAGES)
  int nf;                    // frames per image box: history (4), or 5 for the paired forward's window of s and s'
};

__device__ __forceinline__ int4 cvt8_u8_bf16(uint32_t w0, uint32_t w1) {
  // exact u8 -> bf16 without I2F: 0x4B0000vv is the float 2^23 + v; subtract 2^23; the top 16 bits are the bf16
  const float m = 8388608.0f;
  uint32_t f[8];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    f[k] = __float_as_uint(__uint_as_float(__byte_perm(w0, 0x4B000000u, 0x7540 + k)) - m);
    f[4 + k] = __float_as_uint(__uint_as_float(__byte_perm(w1, 0x4B000000u, 0x7540 + k)) - m);
  }
  int4 o;
  o.x = (int)__byte_perm(f[0], f[1], 0x7632);
  o.y = (int)__byte_perm(f[2], f[3], 0x7632);
  o.z = (int)__byte_perm(f[4], f[5], 0x7632);
  o.w = (int)__byte_perm(f[6], f[7], 0x7632);
  return o;
}

// The uint8 pixels travel ring -> shared memory by TMA, several tiles ahead of the converters, so that no thread ever waits on a
// global load.  The ring is described to the TMA as a 3-D tensor of 32-bit words [capacity rows][G grid rows][frame_w words]
// (the 4 pixel rows of one grid row of one frame are 4 * frame_w contiguous bytes = frame_w words): the pixels a slab needs from
// ONE image are the box [4 frames][slots grid rows][frame_w words] at (word 0, grid row q0 - b*G, ring row idx[b] + first) --
// one tensor load per image the slab touches (at most two), instead of one bulk copy per (image, frame) whose fixed cost
// is serialised per SM.  Grid rows past the end of the image are
// zero-filled by the TMA and never read.  The paired forward (b2rl_conv1_u8_fwd_pair) loads nf = 5 frames per image: the
// window idx-3 .. idx+1 that holds both s (frames 0-3) and s' (frames 1-4).
//   staging layout of one tile: [image segment 0 | 1][frame f < nf][slot = grid-row index q - qseg][4 * frame_w bytes]
constexpr int U8_MAX_STAGES = 8;
__host__ __device__ inline int u8_slots(int slab_rows, int G) { return (slab_rows + G - 2) / G + 1; }
__host__ __device__ inline int u8_box_bytes(int slab_rows, int G, int frame_w, int nf) {
  return (nf * u8_slots(slab_rows, G) * 4 * frame_w + 127) & ~127;
}
__host__ __device__ inline int u8_stage_bytes(int slab_rows, int G, int frame_w, int nf) {
  return 2 * u8_box_bytes(slab_rows, G, frame_w, nf);
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          s2u(smem_dst)),
      "l"(map), "r"(s2u(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// images a slab starting at grid-matrix row R0 touches: b0 (always, if any row is inside the batch) and b1 = b0 + 1 (n1 > 0)
struct U8Plan { int b0, n0, n1, q0; };
__device__ __forceinline__ U8Plan u8_plan(const U8Src& u, int R0, int slab_rows) {
  U8Plan pl;
  const int totalq = u.rows / u.G;
  pl.q0 = R0 / u.G;
  int q1 = (R0 + slab_rows - 1) / u.G;
  if (q1 > totalq - 1) q1 = totalq - 1;
  pl.b0 = 0; pl.n0 = 0; pl.n1 = 0;
  if (q1 >= pl.q0) {
    pl.b0 = pl.q0 / u.G;
    const int b1 = q1 / u.G;
    pl.n0 = min(q1, pl.b0 * u.G + u.G - 1) - pl.q0 + 1;
    pl.n1 = b1 > pl.b0 ? q1 - b1 * u.G + 1 : 0;
  }
  return pl;
}
// ONE thread: arm `bar` with the tile's byte count and issue its one or two tensor loads; i0 / i1 = idx[b0] / idx[b0 + 1]
__device__ __forceinline__ void u8_issue(const U8Src& u, const CUtensorMap* map, const U8Plan& pl, long long i0, long long i1,
                                         uint8_t* stage, uint64_t* bar, int slots) {
  const uint32_t box = (uint32_t)(u.nf * slots * 4 * u.frame_w);       // bytes the TMA reports per box (zero fill included)
  const int nb = (pl.n0 > 0) + (pl.n1 > 0);
  if (nb == 0) { mb_arrive(bar); return; }
  mb_expect_tx(bar, box * nb);
  tma_load_3d(stage, map, bar, 0, pl.q0 - pl.b0 * u.G, (int)(i0 + u.first));
  if (pl.n1 > 0) tma_load_3d(stage + ((box + 127) & ~127u), map, bar, 0, 0, (int)(i1 + u.first));
}

// explicit shared-space accesses: the staging / slab pointers are carved out of the dynamic shared memory through integer
// arithmetic, so the compiler only sees GENERIC pointers -- generic loads of shared memory go through the L1 path with ~10x the
// latency of LDS
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const int4 v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// shared-memory address of chunk j (16 bytes = 8 channels) of slab row rl: chunks 0-7 (frames 0-3) lie in the 128B-swizzled
// 64-channel block `slab`; chunks 8-9 (frame 4, paired forward only) in block `slab_b` of 32-byte rows with the 32-byte swizzle
// (address bit 4 ^= bit 7; slab_b is 256-byte aligned, so bit 7 is bit 2 of the row)
__device__ __forceinline__ uint32_t slab_chunk(uint32_t slab, uint32_t slab_b, int rl, int j) {
  return j < 8 ? slab + (uint32_t)(rl * 128 + ((j ^ (rl & 7)) << 4)) : slab_b + (uint32_t)(rl * 32 + (((j - 8) ^ ((rl >> 2) & 1)) << 4));
}

template <int J0, int NJ>
__device__ __forceinline__ void u8_store_chunks(uint32_t stage, uint32_t slab, uint32_t slab_b, int rl, int so, int fstride,
                                                int frame_w) {
  // chunks J0 .. J0+NJ-1 of slab row rl; so = staging offset of pixel (4gy, 4gx) of frame 0, or -1: zeros
  uint32_t w0[NJ], w1[NJ];
#pragma unroll
  for (int jj = 0; jj < NJ; ++jj) {                       // all loads first, then the conversions
    const int j = J0 + jj;
    w0[jj] = w1[jj] = 0;
    if (so >= 0) {
      const uint32_t src = stage + (uint32_t)((j >> 1) * fstride + so + (2 * (j & 1)) * frame_w);
      w0[jj] = lds32(src);
      w1[jj] = lds32(src + frame_w);
    }
  }
#pragma unroll
  for (int jj = 0; jj < NJ; ++jj) sts128(slab_chunk(slab, slab_b, rl, J0 + jj), cvt8_u8_bf16(w0[jj], w1[jj]));
}

// NT = 128 or 256 threads (tid 0..NT-1, named barrier `bar_id`) convert one staged tile into the swizzled bf16 slab of
// `slab_rows` rows x 8 NCH channels whose first row is grid-matrix row R0 (NCH = 8: one 64-channel block; 10: the paired
// forward's block A of frames 0-3 and block B of frame 4, see slab_chunk); rows >= u.rows are zero (what the TMA's
// out-of-bounds fill gave).  Thread t owns slab row t & 127 (consecutive threads -> consecutive pixels of the staging rows and
// the 8 distinct swizzle positions of a 128-byte window: conflict-free both ways) and, with 256 threads, one half of its NCH
// chunks; rows beyond 128 are shared out chunk-wise.  On return every thread's stores are fenced towards the async proxy
// (wgmma reads shared memory through it) and all NT threads have arrived.
template <int NT, int NCH>
__device__ __forceinline__ void u8_convert(const U8Src& u, const uint8_t* stage_p, uint8_t* slab_p, uint8_t* slab_b_p, int R0,
                                           int slab_rows, int slots, int tid, int bar_id) {
  const uint32_t stage = s2u(stage_p), slab = s2u(slab_p), slab_b = NCH > 8 ? s2u(slab_b_p) : 0u;
  const int rowb = 4 * u.frame_w, fstride = slots * rowb;
  const int q0 = R0 / u.G;
  const int qb1 = (q0 / u.G + 1) * u.G;                   // first grid row of the second image the slab may touch
  const int seg1 = (u.nf * fstride + 127) & ~127;         // its box sits behind the first image's
  const int rl0 = tid & 127;
  if (rl0 < slab_rows) {
    const int r = R0 + rl0;
    int so = -1;
    if (r < u.rows) {
      const int q = r / u.G;
      so = (q >= qb1 ? seg1 + (q - qb1) * rowb : (q - q0) * rowb) + 4 * (r - q * u.G);
    }
    if (NT == 128) {
      u8_store_chunks<0, NCH>(stage, slab, slab_b, rl0, so, fstride, u.frame_w);
    } else if (tid < 128) {
      u8_store_chunks<0, NCH / 2>(stage, slab, slab_b, rl0, so, fstride, u.frame_w);
    } else {
      u8_store_chunks<NCH / 2, NCH / 2>(stage, slab, slab_b, rl0, so, fstride, u.frame_w);
    }
  }
  for (int e = tid; e < (slab_rows - 128) * NCH; e += NT) {
    const int rl = 128 + e / NCH, j = e % NCH, r = R0 + rl;
    uint32_t w0 = 0, w1 = 0;
    if (r < u.rows) {
      const int q = r / u.G;
      const uint32_t src = stage + (uint32_t)((j >> 1) * fstride + (q >= qb1 ? seg1 + (q - qb1) * rowb : (q - q0) * rowb) +
                                              4 * (r - q * u.G) + (2 * (j & 1)) * u.frame_w);
      w0 = lds32(src);
      w1 = lds32(src + u.frame_w);
    }
    sts128(slab_chunk(slab, slab_b, rl, j), cvt8_u8_bf16(w0, w1));
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "n"(NT) : "memory");
}

struct SlabParams {
  GemmParams g;            // M, N, ldd, relu, out_mode, bias, D, taps_x, grid_w, shift_sign, out_map, G, V
  int taps, col_blocks;    // taps, channels / 64
  int slab_rows;           // multiple of 8, >= 128 + max_shift
  int min_shift;           // row offset of the slab start relative to m0 (0 for forward, -max_shift for dgrad)
  int stages;
  int base_offset_mode;    // 1: descriptor base_offset = (window start >> 7) & 7; 2: base_offset = 0 (address-based swizzle)
  U8Src u8;                // U8 kernels: the activation slabs are built from the uint8 frame ring (K1), tmA is unused
  unsigned long long* clk; // profiling hook (normally null): cycles per role summed over the CTAs, K1_CLK_*
};

// slots of the phase probe of the slab and K1 kernels (b2rl_conv1_set_phase_clocks): clock64() cycles summed over all CTAs,
// each role timed by its thread 0 -- the CTA's whole run (thread 0), the producer's waits for a free stage, the converters'
// waits for a free slab and for the pixels and their conversion; the MMA warpgroup's waits for the slab, its chain from the
// first issue to its retirement, its waits for the epilogue warpgroups to free the staging tile and its accumulator staging;
// the epilogue warpgroups' (both summed) waits for a staged half and their work on it; the tiles the MMA warpgroup took.
enum { K1_CLK_CTA, K1_CLK_PRODUCER_WAIT, K1_CLK_CONVERT_WAIT_SLAB, K1_CLK_CONVERT_WAIT_PIXELS, K1_CLK_CONVERT, K1_CLK_MMA_WAIT,
       K1_CLK_MMA, K1_CLK_MMA_WAIT_FREE, K1_CLK_MMA_STAGE, K1_CLK_EPILOGUE_WAIT, K1_CLK_EPILOGUE, K1_CLK_TILES, K1_CLK_SLOTS };
__device__ __forceinline__ long long clk_now(const unsigned long long* clk) { return clk ? clock64() : 0; }

constexpr int SLAB_U8_THREADS = GEMM_THREADS + 128;   // K1 weight gradient: a fourth warpgroup (warps 12-15) converts the pixels
// The slab kernel: warpgroup 0 TMA producer, 1 MMA, 2 / 3 epilogue of rows 0-63 / 64-127 of each tile; K1: warpgroup 4
// converts the uint8 pixels
constexpr int SLAB_THREADS = 512;
constexpr int SLAB_K1_THREADS = SLAB_THREADS + 128;
constexpr int SLAB_BAR_STAGED = 5, SLAB_BAR_FREE = 7;  // + half: named barriers of the staging-tile hand-off (256 threads)
// register split (setmaxnreg, per thread) per role: the launch gives every thread 65536 / threads (128 at 512 threads, 96 at
// 640), and the roles' shares add up to at most that sum.  The MMA warpgroup holds both m64 x BN accumulator halves (BN 128:
// 128 registers); an epilogue warpgroup one half's mask (BN 128: 32 registers) and its per-row work.
template <bool U8> struct SlabRegs;
template <> struct SlabRegs<false> { static constexpr int producer = 40, mma = 232, epilogue = 120, convert = 0; };   // 512
template <> struct SlabRegs<true> { static constexpr int producer = 64, mma = 136, epilogue = 88, convert = 104; };    // 480
template <int R> __device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// Paired conv1 forward (PAIR: U8, BN 64, 2 x 2 taps, one column block): x1 = conv1_online(s) and z1 = conv1_target(s') in ONE
// launch from the five-frame ring window idx-3 .. idx+1 shared by s (frames 0-3) and s' (frames 1-4, n_step 1).
//   slab:    block A = window frames 0-3, the 128B-swizzled 64-channel slab of s as above; block B = window frame 4, 16
//            channels, rows of 32 bytes with the 32-byte swizzle (slab_chunk), pair_block_b_bytes behind block A
//   weights: N = 64 stacked, per tap a 128B-swizzled [64 n][64 k] tile (k16 step j reads window frame j) and a 32B-swizzled
//            [64 n][16 k] tile for frame 4.  Rows 0-31 = online: frames 0-3 as stored, zero at frame 4 (set in the prologue);
//            rows 32-63 = target: zero at frame 0 (the TMA's out-of-bounds fill of a box that starts at channel -16), its
//            frames 0-3 at window frames 1-4.
// Per tap and accumulator half the chain is the four k16 steps over block A, then one over block B: every output column sees
// the products of today's separate launch in the same k16 groups and tap order, plus exact zeros -- the same bits.
__host__ __device__ inline uint32_t pair_block_b_bytes(int slab_rows) { return ((uint32_t)slab_rows * 32 + 1023) & ~1023u; }
// wgmma descriptor of a K-major operand with 32-byte rows and the 32-byte swizzle (layout type 3): 8-row groups 256 B apart
__device__ __forceinline__ uint64_t make_desc_sw32(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(256 >> 4) << 32) | ((uint64_t)3 << 62);
}
// The tap grid (TX x TY taps) and the column blocks (CB = channels / 64) are template parameters: a tile's 2 x TX x TY x CB
// k-tiles are then one unrolled chain of wgmmas in ONE commit group (a chain carried through runtime loops makes ptxas
// serialize every wgmma).  One MMA warpgroup issues every tile of the CTA, whole 128-row tiles as two m64 accumulator
// halves, and stages them into the fp32 staging tile; two epilogue warpgroups finish one 64-row half each, side by side.
// Per half, named barriers hand the staging tile over (SLAB_BAR_STAGED: written, SLAB_BAR_FREE: read): the MMAs of the
// next tile run during the epilogue of this one, so the CTA's period per tile is about the longest of MMA chain + staging,
// one half's epilogue and (K1) one slab's conversion, not MMA chain + both halves' epilogue over two warpgroups.
// The body of conv_slab_wgmma_kernel and of its paired conv1 instantiation conv1_pair_wgmma_kernel (below); the tensor maps
// are the kernels' __grid_constant__ parameters.  PAIR: tmA = ring, tmB = online weights (box [32 n][1 tap][64 k]),
// tmA2 / tmB2 = target weights (boxes [32][1][64] / [32][1][16]).
template <int BN, bool EXT, bool U8, int TX, int TY, int CB, bool PAIR>
__device__ __forceinline__ void conv_slab_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmA2,
                                               const CUtensorMap& tmB2, const SlabParams& sp) {
  static_assert(!PAIR || (U8 && !EXT && BN == 64 && TX == 2 && TY == 2 && CB == 1), "the paired forward is conv1's K1 shape");
  const int n_cta = sp.g.dual ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  const bool second = sp.g.dual && (int)blockIdx.x >= n_cta;
  const int cta = second ? (int)blockIdx.x - n_cta : (int)blockIdx.x;
  const CUtensorMap* mA = second ? &tmA2 : &tmA;
  const CUtensorMap* mB = second ? &tmB2 : &tmB;
  GemmParams p = sp.g;
  if (second) { p.D = sp.g.D2; p.bias = sp.g.bias2; }
  constexpr uint32_t W_TILE = BN * 128;                               // one 64-wide k-tile of the weights
  constexpr uint32_t WB_TILE = BN * 32;                               // PAIR: one tap's frame-4 weights
  constexpr int ACC_LD = acc_ld(BN);
  constexpr int MAX_STAGES = 6;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int k_tiles = TX * TY * CB;
  const uint32_t slab_block = (uint32_t)sp.slab_rows * 128;          // one 64-channel column block of a slab
  const uint32_t slab_bytes = slab_block * CB + (PAIR ? pair_block_b_bytes(sp.slab_rows) : 0u);
  uint8_t* sW = smem;
  uint8_t* sWB = smem + (size_t)k_tiles * W_TILE;                     // PAIR: frame-4 weight tiles
  uint8_t* sS = sWB + (PAIR ? (size_t)k_tiles * WB_TILE : 0);
  float* sAcc = reinterpret_cast<float*>(sS + (size_t)sp.stages * slab_bytes);
  uint64_t* full = reinterpret_cast<uint64_t*>(sAcc + GEMM_BM * ACC_LD);
  uint64_t* empty = full + MAX_STAGES;
  uint64_t* w_full = empty + MAX_STAGES;
  // U8 (K1): uint8 staging tiles + their full / empty barriers live behind the barriers (launch_slab_t sizes the allocation)
  const int u8_slots_ = U8 ? u8_slots(sp.slab_rows, sp.u8.G) : 0;
  const int u8_bytes = U8 ? u8_stage_bytes(sp.slab_rows, sp.u8.G, sp.u8.frame_w, sp.u8.nf) : 0;
  uint8_t* sU = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(w_full + 2) + 127) & ~uintptr_t(127));
  const int U8_STAGES = U8 ? sp.u8.stages : 1;
  uint64_t* u8_full = reinterpret_cast<uint64_t*>(sU + (size_t)U8_STAGES * u8_bytes);
  uint64_t* u8_empty = u8_full + U8_MAX_STAGES;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
  const int tiles = (p.M + GEMM_BM - 1) / GEMM_BM;

  __shared__ float s_dbias[128];                    // per-CTA bias-gradient accumulator (backward extras)
  if (threadIdx.x < 128) s_dbias[threadIdx.x] = 0.0f;
  if (threadIdx.x == 0) {
    for (int s = 0; s < MAX_STAGES; ++s) { mb_init(&full[s], 1); mb_init(&empty[s], MMA_WARPS / 2); }   // the MMA warpgroup
    mb_init(w_full, 1);
    if (U8) {
      for (int s = 0; s < U8_STAGES; ++s) { mb_init(&u8_full[s], 1); mb_init(&u8_empty[s], 1); }
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(mA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(mB) : "memory");
    if (PAIR) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA2) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB2) : "memory");
    }
  }
  if constexpr (PAIR) {
    // the online rows (0-31) of every tap's frame-4 weights are zero; the wgmmas read them through the async proxy
    for (int i = threadIdx.x; i < k_tiles * (int)WB_TILE / 32; i += blockDim.x)
      sts128(s2u(sWB) + (uint32_t)((i / 64) * WB_TILE + (i % 64) * 16), make_int4(0, 0, 0, 0));
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_sync();   // everything above (barriers, tensor-map prefetch) overlaps the previous kernel's tail
  unsigned long long* const clk = sp.clk;
  const long long t_start = clk_now(clk);
  long long c_wait = 0, c_wait2 = 0, c_work = 0, c_stage = 0;   // per-role sums of the probe (thread 0 of its role)
  using R = SlabRegs<U8>;
  constexpr int launch_regs = 65536 / (U8 ? SLAB_K1_THREADS : SLAB_THREADS) / 8 * 8;   // per thread
  static_assert(R::producer + R::mma + 2 * R::epilogue + R::convert <= (U8 ? 5 : 4) * launch_regs,
                "the roles' register shares exceed what the launch allocates");
  if (warp < 4) {
    reg_dec<R::producer>();
    if (warp == 0 && elect_one()) {
    if constexpr (PAIR) {
      mb_expect_tx(w_full, (uint32_t)k_tiles * (W_TILE + WB_TILE / 2));
      for (int kt = 0; kt < k_tiles; ++kt) {
        tma_load_3d(sW + (size_t)kt * W_TILE, mB, w_full, 0, kt, 0);                           // online, frames 0-3
        tma_load_3d(sW + (size_t)kt * W_TILE + W_TILE / 2, &tmA2, w_full, -16, kt, 0);         // target: zero, frames 0-2
        tma_load_3d(sWB + (size_t)kt * WB_TILE + WB_TILE / 2, &tmB2, w_full, 48, kt, 0);       // target: frame 3
      }
    } else {
      mb_expect_tx(w_full, (uint32_t)k_tiles * W_TILE);
      for (int kt = 0; kt < k_tiles; ++kt) tma_load_2d(sW + (size_t)kt * W_TILE, mB, w_full, kt * GEMM_BK, 0);
    }
    if constexpr (U8) {
      // -------------------------------------------------------------------- K1 producer: the uint8 pixels of every tile (one
      // tensor load per image the slab touches), up to sp.u8.stages tiles ahead; idx[] is requested one tile early
      const int nimg = sp.u8.rows / (sp.u8.G * sp.u8.G);
      U8Plan pl = u8_plan(sp.u8, cta * GEMM_BM + sp.min_shift, sp.slab_rows);
      long long i0 = 0, i1 = 0;
      if (cta < tiles && pl.n0 > 0) { i0 = __ldg(sp.u8.idx + pl.b0); i1 = __ldg(sp.u8.idx + min(pl.b0 + 1, nimg - 1)); }
      uint32_t it = 0;
      for (int tile = cta; tile < tiles; tile += n_cta, ++it) {
        const U8Plan cur = pl;
        const long long c0 = i0, c1 = i1;
        if (tile + n_cta < tiles) {
          pl = u8_plan(sp.u8, (tile + n_cta) * GEMM_BM + sp.min_shift, sp.slab_rows);
          if (pl.n0 > 0) { i0 = __ldg(sp.u8.idx + pl.b0); i1 = __ldg(sp.u8.idx + min(pl.b0 + 1, nimg - 1)); }
        }
        const int us = it % U8_STAGES;
        const long long t0 = clk_now(clk);
        mb_wait(&u8_empty[us], ((it / U8_STAGES) & 1) ^ 1);
        c_wait += clk_now(clk) - t0;
        u8_issue(sp.u8, mA, cur, c0, c1, sU + (size_t)us * u8_bytes, &u8_full[us], u8_slots_);
      }
      if (clk) atomicAdd(clk + K1_CLK_PRODUCER_WAIT, (unsigned long long)c_wait);
    } else {
      // -------------------------------------------------------------------- TMA producer: one slab per tile
      uint32_t it = 0;
      for (int tile = cta; tile < tiles; tile += n_cta, ++it) {
        const int s = it % sp.stages;
        const long long t0 = clk_now(clk);
        mb_wait(&empty[s], ((it / sp.stages) & 1) ^ 1);
        c_wait += clk_now(clk) - t0;
        mb_expect_tx(&full[s], slab_bytes);
        for (int cb = 0; cb < CB; ++cb)
          tma_load_2d(sS + (size_t)s * slab_bytes + (size_t)cb * slab_block, mA, &full[s], cb * GEMM_BK,
                      tile * GEMM_BM + sp.min_shift);
        if (EXT && p.mask) {
          // the tile's ReLU-gradient mask rows into L2, as many tiles ahead as the slab ring: the epilogue's register loads
          // of them (epi_mask_load) then wait for an L2 hit, not for HBM
          const int r0 = tile * GEMM_BM, nr = min(GEMM_BM, p.M - r0);
          prefetch_l2_bulk(p.mask + (int64_t)r0 * p.mask_ld, (uint32_t)(((int64_t)(nr - 1) * p.mask_ld + p.N) * 2));
        }
      }
      if (clk) atomicAdd(clk + K1_CLK_PRODUCER_WAIT, (unsigned long long)c_wait);
    }
    }
  } else if (U8 && warp >= 16) {
    // ---------------------------------------------------------------------- K1 converters (warps 16-19): staged uint8 -> slab
    reg_inc<R::convert>();
    const int tid = (int)threadIdx.x - SLAB_THREADS;
    uint32_t it = 0;
    for (int tile = cta; tile < tiles; tile += n_cta, ++it) {
      const int s = it % sp.stages, us = it % U8_STAGES;
      const long long t0 = clk_now(clk);
      mb_wait(&empty[s], ((it / sp.stages) & 1) ^ 1);
      const long long t1 = clk_now(clk);
      mb_wait(&u8_full[us], (it / U8_STAGES) & 1);
      const long long t2 = clk_now(clk);
      u8_convert<128, PAIR ? 10 : 8>(sp.u8, sU + (size_t)us * u8_bytes, sS + (size_t)s * slab_bytes,
                                     sS + (size_t)s * slab_bytes + slab_block, tile * GEMM_BM + sp.min_shift, sp.slab_rows,
                                     u8_slots_, tid, 4);
      if (tid == 0) { mb_arrive(&full[s]); mb_arrive(&u8_empty[us]); }
      c_wait += t1 - t0, c_wait2 += t2 - t1, c_work += clk_now(clk) - t2;
    }
    if (clk && tid == 0) {
      atomicAdd(clk + K1_CLK_CONVERT_WAIT_SLAB, (unsigned long long)c_wait);
      atomicAdd(clk + K1_CLK_CONVERT_WAIT_PIXELS, (unsigned long long)c_wait2);
      atomicAdd(clk + K1_CLK_CONVERT, (unsigned long long)c_work);
    }
  } else if (warp < 8) {
    // ---------------------------------------------------------------------- MMA (warps 4-7): every tile of this CTA, rows
    // 0-63 / 64-127 in accumulator halves d[0] / d[1], each staged into its half of sAcc once its epilogue warpgroup has
    // read the previous tile's
    reg_inc<R::mma>();
    const int wl = warp - 4;
    const uint32_t w0 = s2u(sW), wb0 = s2u(sWB);
    mb_wait(w_full, 0);
    long long c_free = 0;
    uint32_t it = 0;
    for (int tile = cta; tile < tiles; tile += n_cta, ++it) {
      const int s = it % sp.stages;
      const long long t0 = clk_now(clk);
      mb_wait(&full[s], (it / sp.stages) & 1);
      const long long t1 = clk_now(clk);
      float d[2][BN / 2];
      acc_zero<BN>(d[0]);
      acc_zero<BN>(d[1]);
      acc_fence<BN>(d[0]);                                          // both halves zeroed before the chain: no wait inside it
      acc_fence<BN>(d[1]);
      const uint32_t slab = s2u(sS) + (uint32_t)s * slab_bytes;
      wg_fence();
      // taps in (dy, dx) order; the window of tap (dy, dx) of half h starts sign*(dy*grid_w + dx) - min_shift + 64 h rows
      // into the slab
#pragma unroll
      for (int dy = 0; dy < TY; ++dy) {
#pragma unroll
        for (int dx = 0; dx < TX; ++dx) {
#pragma unroll
          for (int cb = 0; cb < CB; ++cb) {
            const uint64_t b = make_desc(w0 + ((dy * TX + dx) * CB + cb) * W_TILE, 16);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = 64 * h - sp.min_shift + p.shift_sign * (dy * p.grid_w + dx);
              const uint32_t a_addr = slab + cb * slab_block + (uint32_t)row * 128;
              mma_ktile<BN, 0, 0>(d[h], make_desc(a_addr, 16, sp.base_offset_mode == 1 ? (a_addr >> 7) & 7 : 0), b);
              if constexpr (PAIR)                                     // window frame 4: block B
                wgmma_n64<0, 0>(d[h], make_desc_sw32(slab + slab_block + (uint32_t)row * 32),
                                make_desc_sw32(wb0 + (dy * TX + dx) * WB_TILE));
            }
          }
        }
      }
      wg_commit();
      wg_wait0();
      acc_fence<BN>(d[0]);
      acc_fence<BN>(d[1]);
      if (lane == 0) mb_arrive(&empty[s]);
      const long long t2 = clk_now(clk);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long t3 = clk_now(clk);
        if (it > 0) named_sync(SLAB_BAR_FREE + h, 256);              // epilogue warpgroup h has read the previous tile's half
        const long long t4 = clk_now(clk);
        stage_acc<BN>(d[h], sAcc + h * 64 * ACC_LD, ACC_LD, wl, lane);
        named_arrive(SLAB_BAR_STAGED + h, 256);
        c_free += t4 - t3, c_stage += clk_now(clk) - t4;
      }
      c_wait += t1 - t0, c_work += t2 - t1;
    }
    if (clk && wl == 0 && lane == 0) {
      atomicAdd(clk + K1_CLK_MMA_WAIT, (unsigned long long)c_wait);
      atomicAdd(clk + K1_CLK_MMA, (unsigned long long)c_work);
      atomicAdd(clk + K1_CLK_MMA_WAIT_FREE, (unsigned long long)c_free);
      atomicAdd(clk + K1_CLK_MMA_STAGE, (unsigned long long)c_stage);
      atomicAdd(clk + K1_CLK_TILES, (unsigned long long)it);
    }
  } else {
    // ---------------------------------------------------------------------- epilogue, warpgroup 2 + e (warps 8-15): rows
    // 64 e .. 64 e + 63 of every tile of this CTA; the tile's mask is requested before the wait for its staged half, so that
    // it is in flight during the tile's MMAs
    reg_dec<R::epilogue>();
    const int e = (warp - 8) >> 2, wl = (warp - 8) & 3;
    const int t = wl * 32 + lane;                                   // epilogue_half's thread index in the warpgroup
    const float* sAcc_e = sAcc + e * 64 * ACC_LD;
    for (int tile = cta; tile < tiles; tile += n_cta) {
      int4 mk[BN / 16];
      epi_mask_load<BN, EXT>(p, tile * GEMM_BM + 64 * e, 0, t, mk);
      const long long t0 = clk_now(clk);
      named_sync(SLAB_BAR_STAGED + e, 256);
      const long long t1 = clk_now(clk);
      slab_epilogue_half<BN, EXT, PAIR>(p, tile * GEMM_BM + 64 * e, t, sAcc_e, mk, s_dbias);
      if (tile + n_cta < tiles) named_arrive(SLAB_BAR_FREE + e, 256);   // the MMA warpgroup waits only for a next tile
      c_wait += t1 - t0, c_work += clk_now(clk) - t1;
    }
    if (clk && t == 0) {
      atomicAdd(clk + K1_CLK_EPILOGUE_WAIT, (unsigned long long)c_wait);
      atomicAdd(clk + K1_CLK_EPILOGUE, (unsigned long long)c_work);
    }
  }
  __syncthreads();
  if (clk && threadIdx.x == 0) atomicAdd(clk + K1_CLK_CTA, (unsigned long long)(clock64() - t_start));
  if (EXT && sp.g.dbias && (int)threadIdx.x < dbias_slots(sp.g)) atomicAdd(sp.g.dbias + threadIdx.x, s_dbias[threadIdx.x]);
}

template <int BN, bool EXT, bool U8, int TX, int TY, int CB>
__global__ void __launch_bounds__(U8 ? SLAB_K1_THREADS : SLAB_THREADS, 1) conv_slab_wgmma_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                          const __grid_constant__ CUtensorMap tmB,
                                                                          const __grid_constant__ CUtensorMap tmA2,
                                                                          const __grid_constant__ CUtensorMap tmB2,
                                                                          const SlabParams sp) {
  conv_slab_body<BN, EXT, U8, TX, TY, CB, false>(tmA, tmB, tmA2, tmB2, sp);
}
// conv1's K1 instantiation with the PAIR flag: b2rl_conv1_u8_fwd_pair
__global__ void __launch_bounds__(SLAB_K1_THREADS, 1) conv1_pair_wgmma_kernel(const __grid_constant__ CUtensorMap tmA,
                                                                             const __grid_constant__ CUtensorMap tmB,
                                                                             const __grid_constant__ CUtensorMap tmA2,
                                                                             const __grid_constant__ CUtensorMap tmB2,
                                                                             const SlabParams sp) {
  conv_slab_body<64, false, true, 2, 2, 1, true>(tmA, tmB, tmA2, tmB2, sp);
}


// ---------------------------------------------------------------------------------------------------------------
// conv1's weight gradient with the taps in the MMA rows.  conv1 has n_out = 32 channels and 2 x 2 taps at row shifts
// s_t = 0, 1, G, G + 1 of the G x G grid.  The sum is written with the activations unshifted and the gradient rows carrying
// the shift:
//   dW[n][t*64 + c] = sum_r G[r][n] x[r + s_t][c] = sum_r' G[r' - s_t][n] x[r'][c]
// (r' - s_t < 0: the TMA's out-of-bounds zero fill; r' >= rows: x is zero there -- the same products as the first sum).
// Each MMA warpgroup g holds ONE m64n64 accumulator over two taps: rows 0-31 are tap 2g + 1, rows 32-63 tap 2g, so every
// accumulator row is a result.  The A operand (MN-major, K = rows r') is one TMA box of the gradient rows [k0 - G - 1,
// k0 + BK) stored with the 64-byte swizzle (one 64-byte row per grid row = 32 channels = one swizzle atom column): the
// descriptor of warpgroup g starts at the row of its larger shift and reaches the smaller one through the MN-direction
// atom stride (LBO) of one row, 64 bytes.  The 64-byte swizzle, like the 128-byte one of the slab kernels, is a function of
// the shared-memory address (bits 4-5 ^= bits 7-8), so a descriptor may start at any 64-byte row with base_offset 0.  The
// B operand is the 64-channel activation block of rows [k0, k0 + BK) with no halo, 128B-swizzled MN-major.
// A CTA takes a contiguous range of 128-row k-blocks (at most one CTA per SM, equal ranges) and stores its [32][256] fp32
// partial block at D + blockIdx.x * 8192.  Two producers of the activation block give bit-identical partials: U8 builds it
// from the uint8 frame ring (K1: u8_issue / u8_convert with a 128-row slab), the bf16 form loads it by TMA from x0m.
// ---------------------------------------------------------------------------------------------------------------
constexpr int C1W_BK = 128;                           // rows of one k-block
constexpr uint32_t C1W_X_BYTES = C1W_BK * 128;        // activation block: 128 rows x 64 channels bf16
struct Conv1WgradParams {
  int rows, grid_w;             // batch * G * G rows of the G x G grid; G
  int blocks, blocks_per_cta;   // 128-row k-blocks in all / per CTA
  int stages;                   // operand stages (G box + activation block)
  float* D;                     // partials: CTA i at D + i * 32 * 256
  U8Src u8;                     // U8: the activation blocks come from the uint8 frame ring (K1)
  unsigned long long* clk;      // profiling hook (normally null), K1_CLK_* slots: see conv1_wgrad_body
};
// bytes of one gradient box: rows [k0 - G - 1, k0 + BK) of 64 bytes, padded to the 1024-byte alignment of the stage ring
__host__ __device__ inline uint32_t c1w_g_bytes(int grid_w) { return ((uint32_t)(C1W_BK + grid_w + 1) * 64 + 1023) & ~1023u; }
// wgmma descriptor of an MN-major operand with the 64-byte swizzle (layout type 2): 32-element MN atoms `lbo` bytes apart,
// 8-K-row groups 512 bytes apart
__device__ __forceinline__ uint64_t make_desc_sw64(uint32_t smem_addr, uint32_t lbo_bytes) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)(512 >> 4) << 32) |
         ((uint64_t)2 << 62);
}

// Phase probe (b2rl_conv1_set_phase_clocks) slots used here: K1_CLK_CTA (thread 0's run), K1_CLK_PRODUCER_WAIT (the
// producer's waits for a free uint8 stage and a free operand stage), K1_CLK_CONVERT_WAIT_SLAB / _PIXELS / K1_CLK_CONVERT
// (U8 converters), K1_CLK_MMA_WAIT (MMA warpgroups' waits for a full stage), K1_CLK_MMA (their issue, retire-one wait and
// release), K1_CLK_TILES (k-blocks, counted by the MMA warpgroups).
template <bool U8>
__global__ void __launch_bounds__(U8 ? SLAB_U8_THREADS : GEMM_THREADS, 1) conv1_taps_conv_wgrad_wgmma_kernel(
    const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmX, const Conv1WgradParams w) {
  constexpr int MAX_STAGES = 6;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int halo = w.grid_w + 1;
  const uint32_t g_bytes = c1w_g_bytes(w.grid_w), stage_bytes = g_bytes + C1W_X_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)w.stages * stage_bytes);
  uint64_t* empty = full + MAX_STAGES;
  // U8: uint8 staging tiles + their full / empty barriers behind the operand ring (launch_conv1_wgrad sizes the allocation)
  const int u8_slots_ = U8 ? u8_slots(C1W_BK, w.u8.G) : 0;
  const int u8_bytes = U8 ? u8_stage_bytes(C1W_BK, w.u8.G, w.u8.frame_w, w.u8.nf) : 0;
  uint8_t* sU = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(empty + MAX_STAGES) + 127) & ~uintptr_t(127));
  const int U8_STAGES = U8 ? w.u8.stages : 1;
  uint64_t* u8_full = reinterpret_cast<uint64_t*>(sU + (size_t)U8_STAGES * u8_bytes);
  uint64_t* u8_empty = u8_full + U8_MAX_STAGES;
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
  const int blk0 = (int)blockIdx.x * w.blocks_per_cta;
  const int n_blk = max(min(w.blocks, blk0 + w.blocks_per_cta) - blk0, 0);

  if (threadIdx.x == 0) {
    for (int s = 0; s < MAX_STAGES; ++s) { mb_init(&full[s], U8 ? 2 : 1); mb_init(&empty[s], MMA_WARPS); }   // U8: TMA + converters
    if (U8) {
      for (int s = 0; s < U8_STAGES; ++s) { mb_init(&u8_full[s], 1); mb_init(&u8_empty[s], 1); }
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmG) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX) : "memory");
  }
  __syncthreads();
  pdl_sync();   // everything above (barriers, tensor-map prefetch) overlaps the previous kernel's tail
  unsigned long long* const clk = w.clk;
  const long long t_start = clk_now(clk);
  long long c_wait = 0, c_wait2 = 0, c_work = 0;                 // per-role sums of the probe (one thread per role)

  if (warp == 0 && elect_one()) {
    // ------------------------------------------------------------------------ producer: per k-block the gradient box and
    // (bf16) the activation block, or (U8) the uint8 pixels of the block, up to w.u8.stages blocks ahead, idx[] one block early
    U8Plan pl = {};
    long long i0 = 0, i1 = 0;
    int nimg = 1;
    if constexpr (U8) {
      nimg = w.u8.rows / (w.u8.G * w.u8.G);
      pl = u8_plan(w.u8, blk0 * C1W_BK, C1W_BK);
      if (n_blk > 0 && pl.n0 > 0) { i0 = __ldg(w.u8.idx + pl.b0); i1 = __ldg(w.u8.idx + min(pl.b0 + 1, nimg - 1)); }
    }
    for (int i = 0; i < n_blk; ++i) {
      const int s = i % w.stages, k0 = (blk0 + i) * C1W_BK;
      uint8_t* st = smem + (size_t)s * stage_bytes;
      const long long t0 = clk_now(clk);
      if constexpr (U8) {
        const U8Plan cur = pl;
        const long long c0 = i0, c1 = i1;
        if (i + 1 < n_blk) {
          pl = u8_plan(w.u8, k0 + C1W_BK, C1W_BK);
          if (pl.n0 > 0) { i0 = __ldg(w.u8.idx + pl.b0); i1 = __ldg(w.u8.idx + min(pl.b0 + 1, nimg - 1)); }
        }
        const int us = i % U8_STAGES;
        mb_wait(&u8_empty[us], ((i / U8_STAGES) & 1) ^ 1);
        u8_issue(w.u8, &tmX, cur, c0, c1, sU + (size_t)us * u8_bytes, &u8_full[us], u8_slots_);
        mb_wait(&empty[s], ((i / w.stages) & 1) ^ 1);
        mb_expect_tx(&full[s], (uint32_t)(C1W_BK + halo) * 64);
      } else {
        mb_wait(&empty[s], ((i / w.stages) & 1) ^ 1);
        mb_expect_tx(&full[s], (uint32_t)(C1W_BK + halo) * 64 + C1W_X_BYTES);
        tma_load_2d(st + g_bytes, &tmX, &full[s], 0, k0);                                // [128 rows][64 c]
      }
      c_wait += clk_now(clk) - t0;
      tma_load_2d(st, &tmG, &full[s], 0, k0 - halo);                                     // [BK + halo rows][32 n]
    }
    if (clk) atomicAdd(clk + K1_CLK_PRODUCER_WAIT, (unsigned long long)c_wait);
  } else if (U8 && warp >= 12) {
    // ------------------------------------------------------------------------ K1 converters (warps 12-15): the activation
    // block of every k-block from the staged uint8 pixels, one block row per thread
    const int tid = (int)threadIdx.x - GEMM_THREADS;
    for (int i = 0; i < n_blk; ++i) {
      const int s = i % w.stages, us = i % U8_STAGES;
      const long long t0 = clk_now(clk);
      mb_wait(&empty[s], ((i / w.stages) & 1) ^ 1);
      const long long t1 = clk_now(clk);
      mb_wait(&u8_full[us], (i / U8_STAGES) & 1);
      const long long t2 = clk_now(clk);
      u8_convert<128, 8>(w.u8, sU + (size_t)us * u8_bytes, smem + (size_t)s * stage_bytes + g_bytes, nullptr,
                         (blk0 + i) * C1W_BK, C1W_BK, u8_slots_, tid, 4);
      if (tid == 0) { mb_arrive(&full[s]); mb_arrive(&u8_empty[us]); }
      c_wait += t1 - t0, c_wait2 += t2 - t1, c_work += clk_now(clk) - t2;
    }
    if (clk && tid == 0) {
      atomicAdd(clk + K1_CLK_CONVERT_WAIT_SLAB, (unsigned long long)c_wait);
      atomicAdd(clk + K1_CLK_CONVERT_WAIT_PIXELS, (unsigned long long)c_wait2);
      atomicAdd(clk + K1_CLK_CONVERT, (unsigned long long)c_work);
    }
  } else if (warp >= 4 && warp < 12 && n_blk > 0) {
    // ------------------------------------------------------------------------ MMA, warpgroup g: taps 2g + 1 (rows 0-31) and
    // 2g (rows 32-63); shift of the larger tap: 1 (g = 0) or G + 1 (g = 1), its rows start halo - shift rows into the box
    const int cw = warp - 4, g = cw >> 2, wl = cw & 3;
    const uint32_t a0 = s2u(smem) + (uint32_t)(g ? 0 : halo - 1) * 64, b0 = s2u(smem) + g_bytes;
    float d[32];
    acc_zero<64>(d);
#pragma unroll 2
    for (int i = 0; i < n_blk; ++i) {
      const int s = i % w.stages;
      const long long t0 = clk_now(clk);
      mb_wait(&full[s], (i / w.stages) & 1);
      const long long t1 = clk_now(clk);
      const uint32_t st = (uint32_t)s * stage_bytes;
      wg_fence();
#pragma unroll
      for (int k = 0; k < C1W_BK / 16; ++k)                         // k16 step: 16 rows = 1024 bytes of A, 2048 of B
        wgmma_n64<1, 1>(d, make_desc_sw64(a0 + st + k * 1024, 64), make_desc(b0 + st + k * 2048, 8192));
      wg_commit();
      wg_wait1();                                                    // k-block i - 1 has retired: release its stage
      if (i > 0 && lane == 0) mb_arrive(&empty[(i - 1) % w.stages]);
      c_wait += t1 - t0, c_work += clk_now(clk) - t1;
    }
    wg_wait0();
    acc_fence<64>(d);
    if (lane == 0) mb_arrive(&empty[(n_blk - 1) % w.stages]);
    // accumulator element d[4 jj + 2 h + e]: row m = 16 wl + lane / 4 + 8 h (channel m & 31, tap 2g + 1 - m / 32), column
    // c = 8 jj + 2 (lane % 4) + e
    float* base = w.D + (int64_t)blockIdx.x * (32 * 256) + 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = 16 * wl + (lane >> 2) + 8 * h;
      float* dst = base + (m & 31) * 256 + (2 * g + 1 - (m >> 5)) * 64;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) *reinterpret_cast<float2*>(dst + 8 * jj) = make_float2(d[4 * jj + 2 * h], d[4 * jj + 2 * h + 1]);
    }
    if (clk && (threadIdx.x & 127) == 0) {
      atomicAdd(clk + K1_CLK_MMA_WAIT, (unsigned long long)c_wait);
      atomicAdd(clk + K1_CLK_MMA, (unsigned long long)c_work);
      if (g == 0) atomicAdd(clk + K1_CLK_TILES, (unsigned long long)n_blk);
    }
  }
  __syncthreads();
  if (clk && threadIdx.x == 0) atomicAdd(clk + K1_CLK_CTA, (unsigned long long)(clock64() - t_start));
}

// ---------------------------------------------------------------------------------------------------------------
// conv2's and conv3's weight gradients with every tap of a k-block in one CTA.  n_out = 64 output channels, C input channels
// and TAPS_X x TAPS_X taps on the G x G grid, tap t = (dy, dx) at row shift s_t = dy G + dx: conv3 C 64, 3 x 3 taps; conv2
// C 128 (its space-to-depth(2) input), 2 x 2 taps.  As in conv1's kernel the gradient rows carry the shift:
//   dW[n][t*C + c] = sum_r' G[r' - s_t][n] x[r'][c]
// Per 128-row k-block the producer loads ONE gradient box, rows [k0 - halo, k0 + BK) with halo = s_max = (TAPS_X - 1)(G + 1),
// 64 channels = one 128-byte row each, 128B-swizzled MN-major, and ONE activation block, rows [k0, k0 + BK) of C channels
// (C / 64 boxes of [128 rows][64 c], no halo).  Every tap's MMAs read these two: the A descriptor of tap t starts halo - s_t
// rows into the gradient box (a 128-byte step; the swizzle is a function of the address, as in the slab kernels), B is the
// activation block for all taps.  Tap t has its own m64 x C accumulator (output channels x input channels), so each
// accumulator row is a result; MMA warpgroup g holds taps g*TPW .. g*TPW + TPW - 1: conv3 3 warpgroups x 3 taps of m64n64
// (96 registers), conv2 2 x 2 taps of m64n128 (128 registers).  Loads per k-block: (BK + halo) * 128 + BK * 2C bytes for
// 2 * BK * 64 * taps * C FLOP: every operand is loaded once, whatever the number of taps.
// A CTA takes a contiguous range of k-blocks (equal ranges, at most one CTA per SM or per CTA of the budget) and stores its
// [64][taps * C] fp32 partial block at D + blockIdx.x * 64 * taps * C; the consumer sums the partials (deterministic).
// Each k-block is one commit group per warpgroup, retired (its stage released) after the next one has been issued.
// Phase probe slots: K1_CLK_CTA, K1_CLK_PRODUCER_WAIT (waits for a free stage), K1_CLK_MMA_WAIT (MMA warpgroups' waits for a
// full stage, summed over them), K1_CLK_MMA (their issue, retire-one wait and release), K1_CLK_TILES (k-blocks).
// ---------------------------------------------------------------------------------------------------------------
constexpr int CTW_BK = 128;                           // rows of one k-block
struct TapsWgradParams {
  int rows, grid_w;             // batch * G * G rows of the G x G grid; G
  int blocks, blocks_per_cta;   // 128-row k-blocks in all / per CTA
  int stages;                   // operand stages (gradient box + activation block)
  float* D;                     // partials: CTA i at D + i * 64 * taps * C
  unsigned long long* clk;      // profiling hook (normally null), K1_CLK_* slots
};
// bytes of one gradient box: rows [k0 - halo, k0 + BK) of 128 bytes, padded to the 1024-byte alignment of the stage ring
__host__ __device__ inline uint32_t ctw_g_bytes(int halo) { return ((uint32_t)(CTW_BK + halo) * 128 + 1023) & ~1023u; }
template <int WGS> __host__ __device__ constexpr int ctw_threads() { return 128 * (WGS + 1); }

template <int C, int TAPS_X, int WGS>
__global__ void __launch_bounds__(ctw_threads<WGS>(), 1) conv_taps_wgrad_wgmma_kernel(const __grid_constant__ CUtensorMap tmG,
                                                                                     const __grid_constant__ CUtensorMap tmX,
                                                                                     const TapsWgradParams w) {
  constexpr int MAX_STAGES = 6, TAPS = TAPS_X * TAPS_X, TPW = TAPS / WGS, CB = C / 64;
  constexpr uint32_t X_BOX = CTW_BK * 128, X_BYTES = X_BOX * CB;
  static_assert(TPW * WGS == TAPS && (C == 64 || C == 128), "taps split evenly over the MMA warpgroups; C 64 or 128");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int halo = (TAPS_X - 1) * (w.grid_w + 1);
  const uint32_t g_bytes = ctw_g_bytes(halo), stage_bytes = g_bytes + X_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)w.stages * stage_bytes);
  uint64_t* empty = full + MAX_STAGES;
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform role index
  const int blk0 = (int)blockIdx.x * w.blocks_per_cta;
  const int n_blk = max(min(w.blocks, blk0 + w.blocks_per_cta) - blk0, 0);

  if (threadIdx.x == 0) {
    for (int s = 0; s < MAX_STAGES; ++s) { mb_init(&full[s], 1); mb_init(&empty[s], 4 * WGS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmG) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX) : "memory");
  }
  __syncthreads();
  pdl_sync();   // everything above (barriers, tensor-map prefetch) overlaps the previous kernel's tail
  unsigned long long* const clk = w.clk;
  const long long t_start = clk_now(clk);
  long long c_wait = 0, c_work = 0;                              // per-role sums of the probe (one thread per role)
  // register split (setmaxnreg): the producer warpgroup gives its share to the MMA warpgroups (conv3: 96 accumulator
  // registers of 128 per thread at 512 threads)
  constexpr int launch_regs = 65536 / ctw_threads<WGS>() / 8 * 8, producer_regs = 40;
  constexpr int mma_regs = ((WGS + 1) * launch_regs - producer_regs) / WGS / 8 * 8;

  if (warp < 4) {
    reg_dec<producer_regs>();
    if (warp == 0 && elect_one()) {
    // ------------------------------------------------------------------------ producer: per k-block the gradient box and the
    // activation block
    for (int i = 0; i < n_blk; ++i) {
      const int s = i % w.stages, k0 = (blk0 + i) * CTW_BK;
      uint8_t* st = smem + (size_t)s * stage_bytes;
      const long long t0 = clk_now(clk);
      mb_wait(&empty[s], ((i / w.stages) & 1) ^ 1);
      c_wait += clk_now(clk) - t0;
      mb_expect_tx(&full[s], (uint32_t)(CTW_BK + halo) * 128 + X_BYTES);
      tma_load_2d(st, &tmG, &full[s], 0, k0 - halo);                                     // [BK + halo rows][64 n]
#pragma unroll
      for (int cb = 0; cb < CB; ++cb) tma_load_2d(st + g_bytes + cb * X_BOX, &tmX, &full[s], cb * 64, k0);   // [BK][64 c]
    }
    if (clk) atomicAdd(clk + K1_CLK_PRODUCER_WAIT, (unsigned long long)c_wait);
    }
  } else {
    reg_inc<mma_regs>();
    if (n_blk > 0) {
    // ------------------------------------------------------------------------ MMA, warpgroup g: taps g*TPW + j
    const int cw = warp - 4, g = cw >> 2, wl = cw & 3;
    uint32_t a0[TPW];
#pragma unroll
    for (int j = 0; j < TPW; ++j) {
      const int t = g * TPW + j;
      a0[j] = s2u(smem) + (uint32_t)(halo - (t / TAPS_X) * w.grid_w - t % TAPS_X) * 128;
    }
    const uint32_t b0 = s2u(smem) + g_bytes;
    float d[TPW][C / 2];
#pragma unroll
    for (int j = 0; j < TPW; ++j) acc_zero<C>(d[j]);
    for (int i = 0; i < n_blk; ++i) {
      const int s = i % w.stages;
      const long long t0 = clk_now(clk);
      mb_wait(&full[s], (i / w.stages) & 1);
      const long long t1 = clk_now(clk);
      const uint32_t st = (uint32_t)s * stage_bytes;
      wg_fence();
#pragma unroll
      for (int k = 0; k < CTW_BK / 16; ++k) {                       // k16 step: 16 rows = 2048 bytes of every operand
        const uint64_t b = make_desc(b0 + st + k * 2048, X_BOX);     // C 128: the second 64-channel box X_BOX bytes on
#pragma unroll
        for (int j = 0; j < TPW; ++j) {
          const uint64_t a = make_desc(a0[j] + st + k * 2048, 8192);
          if constexpr (C == 64) wgmma_n64<1, 1>(d[j], a, b);
          else wgmma_n128<1, 1>(d[j], a, b);
        }
      }
      wg_commit();
      wg_wait1();                                                    // k-block i - 1 has retired: release its stage
      if (i > 0 && lane == 0) mb_arrive(&empty[(i - 1) % w.stages]);
      c_wait += t1 - t0, c_work += clk_now(clk) - t1;
    }
    wg_wait0();
#pragma unroll
    for (int j = 0; j < TPW; ++j) acc_fence<C>(d[j]);
    if (lane == 0) mb_arrive(&empty[(n_blk - 1) % w.stages]);
    // accumulator element d[j][4 jj + 2 h + e]: output channel 16 wl + lane / 4 + 8 h, input channel 8 jj + 2 (lane % 4) + e
    float* base = w.D + (int64_t)blockIdx.x * (64 * TAPS * C) + 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = 16 * wl + (lane >> 2) + 8 * h;
#pragma unroll
      for (int j = 0; j < TPW; ++j) {
        float* dst = base + n * (TAPS * C) + (g * TPW + j) * C;
#pragma unroll
        for (int jj = 0; jj < C / 8; ++jj)
          *reinterpret_cast<float2*>(dst + 8 * jj) = make_float2(d[j][4 * jj + 2 * h], d[j][4 * jj + 2 * h + 1]);
      }
    }
    if (clk && (threadIdx.x & 127) == 0) {
      atomicAdd(clk + K1_CLK_MMA_WAIT, (unsigned long long)c_wait);
      atomicAdd(clk + K1_CLK_MMA, (unsigned long long)c_work);
      if (g == 0) atomicAdd(clk + K1_CLK_TILES, (unsigned long long)n_blk);
    }
    }
  }
  __syncthreads();
  if (clk && threadIdx.x == 0) atomicAdd(clk + K1_CLK_CTA, (unsigned long long)(clock64() - t_start));
}

// ------------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D bf16 tensor map over a row-major [outer][inner] matrix with row stride `ld` elements, box = [box_outer][64]
static int make_map(CUtensorMap* m, const void* ptr, int64_t inner, int64_t outer, int64_t ld, int box_outer) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return B2RL_ERR_CUDA; }
  cuuint64_t gdim[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t gstr[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64u, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return B2RL_ERR_CUDA; }
  return B2RL_OK;
}

static int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

// CTA budget (b2rl_set_cta_budget): while set, the slab, dense and convolution weight-gradient launchers size their grids to
// at most this many CTAs instead of one per SM, so that two kernels on parallel graph branches can hold disjoint SMs.
// 0: every SM.  g_last_ctas: the CTAs of the last such launch (all its kernels), read by b2rl_last_grid_ctas.
static int g_cta_budget = 0;
static int g_last_ctas = 0;
static int grid_cap() { return g_cta_budget > 0 && g_cta_budget < sm_count() ? g_cta_budget : sm_count(); }

// shared memory one CTA may use, static + dynamic (227 KB on sm_90)
constexpr size_t SMEM_LIMIT = 227 * 1024;

// dynamic shared memory kernel `k` may request: the per-CTA limit of the device minus the kernel's own static shared memory
// (s_dbias and the alignment of the extern region); 0 if the runtime cannot tell
template <typename K>
static size_t dyn_smem_limit(K k) {
  static int optin = 0;
  if (!optin) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess || optin <= 0)
      optin = (int)SMEM_LIMIT;
  }
  cudaFuncAttributes a;
  if (cudaFuncGetAttributes(&a, reinterpret_cast<const void*>(k)) != cudaSuccess || a.sharedSizeBytes >= (size_t)optin) return 0;
  return (size_t)optin - a.sharedSizeBytes;
}

static bool has_ext(const GemmParams& p) { return p.mask || p.dbias || p.out_map >= 3; }

template <int BN, int STAGES, bool EXT>
static int launch_gemm_t(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ta2, const CUtensorMap& tb2,
                         const GemmParams& p, int splits, cudaStream_t st) {
  constexpr size_t smem = 1024 + (size_t)STAGES * (GEMM_BM * GEMM_BK * 2 + BN * GEMM_BK * 2) + acc_stage_bytes(BN) + 2 * STAGES * 8;
  static_assert(smem <= SMEM_LIMIT, "GEMM stages do not fit in shared memory");
  auto k = gemm_wgmma_kernel<BN, STAGES, EXT>;
  static const size_t limit = dyn_smem_limit(k);
  if (smem > limit) {
    set_error("b2rl_gemm_bf16: %zu bytes of shared memory per CTA exceed the %zu the device allows", smem, limit);
    return B2RL_ERR_ARG;
  }
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr_set = true;
  }
  const int tiles = ((p.M + GEMM_BM - 1) / GEMM_BM) * ((p.N + BN - 1) / BN);
  int ctas = sm_count() / splits / (p.dual ? 2 : 1);                 // per operand set
  if (ctas < 1) ctas = 1;
  if (ctas > tiles) ctas = tiles;
  dim3 grid(p.dual ? 2 * ctas : ctas, 1, splits);
  launch_pdl(k, dim3(grid), dim3(GEMM_THREADS), smem, st, ta, tb, ta2, tb2, p);
  return check_launch("b2rl_gemm_bf16");
}

// the backward extras (mask / bias gradient / scatter maps) are compiled into their own instantiation: the forward and
// weight-gradient kernels keep the lean epilogue
template <int BN, int STAGES>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ta2, const CUtensorMap& tb2,
                       const GemmParams& p, int splits, cudaStream_t st) {
  return has_ext(p) ? launch_gemm_t<BN, STAGES, true>(ta, tb, ta2, tb2, p, splits, st)
                    : launch_gemm_t<BN, STAGES, false>(ta, tb, ta2, tb2, p, splits, st);
}

static int gemm_dispatch(const uint16_t* A, int a_mn, int64_t lda, int64_t a_rows, int64_t a_cols, const uint16_t* B,
                         int b_mn, int64_t ldb, int64_t b_rows, int64_t b_cols, GemmParams p, int splits, int block_n,
                         cudaStream_t st, const uint16_t* A2 = nullptr, const uint16_t* B2 = nullptr) {
  CUtensorMap ta, tb, ta2, tb2;
  int rc;
  // the tensor map describes the matrix AS STORED: [a_rows][a_cols]; box = [128|64 rows][64 cols]
  rc = make_map(&ta, A, a_cols, a_rows, lda, a_mn ? 64 : GEMM_BM);
  if (rc) return rc;
  rc = make_map(&tb, B, b_cols, b_rows, ldb, b_mn ? 64 : block_n);
  if (rc) return rc;
  const int kt_total = (p.K + GEMM_BK - 1) / GEMM_BK;
  if (splits > kt_total) splits = kt_total;
  p.k_tiles_per_split = (kt_total + splits - 1) / splits;
  splits = (kt_total + p.k_tiles_per_split - 1) / p.k_tiles_per_split;
  ta2 = ta, tb2 = tb;
  if (p.dual) {                                                      // second operand set: same shapes and strides
    rc = make_map(&ta2, A2, a_cols, a_rows, lda, a_mn ? 64 : GEMM_BM);
    if (rc) return rc;
    rc = make_map(&tb2, B2, b_cols, b_rows, ldb, b_mn ? 64 : block_n);
    if (rc) return rc;
  }
  if (block_n == 32) return launch_gemm<32, 6>(ta, tb, ta2, tb2, p, splits, st);
  if (block_n == 64) return launch_gemm<64, 6>(ta, tb, ta2, tb2, p, splits, st);
  return launch_gemm<128, 4>(ta, tb, ta2, tb2, p, splits, st);
}

// ---- plain GEMMs: dense_gemm_kernel

// clusters of `S` CTAs of kernel `k` the device can hold at once (0: none -- e.g. no GPC has S free SMs for it)
template <typename K>
static int cluster_capacity(K k, size_t smem, int S) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(S);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = S;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, k, &cfg) != cudaSuccess) {
    cudaGetLastError();
    n = 0;
  }
  return n;
}

// Cluster size of a launch the caller leaves to the launcher, from the shape: per wave of tiles a CTA streams
// ceil(K tiles / S) k-tiles, and a cluster launch costs about CLUSTER_COST k-tiles more (the two cluster barriers, the
// DSMEM reduction and the epilogue on fewer rows; measured on fc4's forward, DESIGN section 7).  The size with the fewest
// k-tile steps, waves x (k-tiles per CTA [+ CLUSTER_COST]), wins; ties go to the smaller cluster.  fc4 forward at batch 512,
// BN 64 (32 tiles, 49 k-tiles): S = 2, since 32 clusters of 4 do not fit in one wave on an H100 SXM; the fc4 dgrad / weight
// gradient and the head GEMMs (8 k-tiles or fewer): S = 1.
// The wave count uses the clusters the device can hold (cap), not SMs / S: a GPC whose SMs do not divide by S leaves some idle.
constexpr int CLUSTER_COST = 16;
static int auto_cluster(int tiles, int kt_total, const int (&cap)[DENSE_MAX_CLUSTER + 1]) {
  int best = 1, best_cost = ((tiles + sm_count() - 1) / sm_count()) * kt_total;
  for (int S = 2; S <= 4; S *= 2) {
    if (cap[S] <= 0) continue;
    const int cost = ((tiles + cap[S] - 1) / cap[S]) * ((kt_total + S - 1) / S + CLUSTER_COST);
    if (cost < best_cost) best = S, best_cost = cost;
  }
  return best;
}

// cluster: 0 = chosen from the shape (auto_cluster), else the requested size (a power of two <= 8; halved while the device
// cannot hold a cluster of that size).  splits > 1 (atomic split-K over blockIdx.z) launches without clusters.
template <int BN, int STAGES, int TA, int TB, bool EXT>
static int launch_dense_t(const CUtensorMap& ta, const CUtensorMap& tb, GemmParams p, int splits, int cluster, cudaStream_t st) {
  constexpr size_t smem = 1024 + (size_t)STAGES * (GEMM_BM * GEMM_BK * 2 + BN * GEMM_BK * 2) + acc_stage_bytes(BN) + 2 * STAGES * 8;
  static_assert(smem <= SMEM_LIMIT, "GEMM stages do not fit in shared memory");
  auto k = dense_gemm_kernel<BN, STAGES, TA, TB, EXT>;
  static const size_t limit = dyn_smem_limit(k);
  if (smem > limit) {
    set_error("b2rl_gemm_bf16: %zu bytes of shared memory per CTA exceed the %zu the device allows", smem, limit);
    return B2RL_ERR_ARG;
  }
  static int cap[DENSE_MAX_CLUSTER + 1] = {};
  static bool init = false;
  if (!init) {
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    for (int S = 2; S <= DENSE_MAX_CLUSTER; S *= 2) cap[S] = cluster_capacity(k, smem, S);
    init = true;
  }
  const int tiles = ((p.M + GEMM_BM - 1) / GEMM_BM) * ((p.N + BN - 1) / BN);
  const int kt_total = (p.K + GEMM_BK - 1) / GEMM_BK;
  int S = 1;
  if (splits == 1 && !g_cta_budget) {                                // a CTA budget launches without clusters
    S = cluster > 0 ? cluster : auto_cluster(tiles, kt_total, cap);
    while (S > 1 && cap[S] <= 0) S >>= 1;
  }
  int ctas = S > 1 ? tiles * S : (tiles < grid_cap() / splits ? tiles : grid_cap() / splits);
  if (ctas < 1) ctas = 1;
  g_last_ctas = ctas * splits;
  if (S > 1) p.k_tiles_per_split = (kt_total + S - 1) / S;   // rank r: k-tiles [r kps, (r + 1) kps); trailing ranks may get none
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(ctas, 1, splits);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na++].val.programmaticStreamSerializationAllowed = 1;
  }
  if (S > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = S;
    attr[na].val.clusterDim.y = 1;
    attr[na++].val.clusterDim.z = 1;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  cudaLaunchKernelEx(&cfg, k, ta, tb, p);
  return check_launch("b2rl_gemm_bf16");
}

// instantiations: K-major or MN-major A and B (MN-major B from BN 64); the backward extras with a K-major A (dgrad)
template <int BN, int STAGES, bool EXT>
static int launch_dense_bn(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int splits, int cluster,
                           cudaStream_t st) {
  if constexpr (BN >= 64) {
    if (p.b_mn) {
      if (!p.a_mn) return launch_dense_t<BN, STAGES, 0, 1, EXT>(ta, tb, p, splits, cluster, st);
      if constexpr (!EXT) return launch_dense_t<BN, STAGES, 1, 1, false>(ta, tb, p, splits, cluster, st);
    }
  }
  if (!p.b_mn) {
    if (!p.a_mn) return launch_dense_t<BN, STAGES, 0, 0, EXT>(ta, tb, p, splits, cluster, st);
    if constexpr (!EXT) return launch_dense_t<BN, STAGES, 1, 0, false>(ta, tb, p, splits, cluster, st);
  }
  set_error("b2rl_gemm_bf16: no kernel for a_mn %d, b_mn %d, block_n %d%s", p.a_mn, p.b_mn, BN, EXT ? " with backward extras" : "");
  return B2RL_ERR_ARG;
}

static int dense_dispatch(const uint16_t* A, int a_mn, int64_t lda, int64_t a_rows, int64_t a_cols, const uint16_t* B,
                          int b_mn, int64_t ldb, int64_t b_rows, int64_t b_cols, GemmParams p, int splits, int block_n,
                          int cluster, cudaStream_t st) {
  CUtensorMap ta, tb;
  int rc = make_map(&ta, A, a_cols, a_rows, lda, a_mn ? 64 : GEMM_BM);
  if (rc) return rc;
  rc = make_map(&tb, B, b_cols, b_rows, ldb, b_mn ? 64 : block_n);
  if (rc) return rc;
  const int kt_total = (p.K + GEMM_BK - 1) / GEMM_BK;
  if (splits > kt_total) splits = kt_total;
  p.k_tiles_per_split = (kt_total + splits - 1) / splits;
  splits = (kt_total + p.k_tiles_per_split - 1) / p.k_tiles_per_split;
  const bool ext = has_ext(p);
  if (block_n == 32) return ext ? launch_dense_bn<32, 6, true>(ta, tb, p, splits, cluster, st)
                                : launch_dense_bn<32, 6, false>(ta, tb, p, splits, cluster, st);
  if (block_n == 64) return ext ? launch_dense_bn<64, 6, true>(ta, tb, p, splits, cluster, st)
                                : launch_dense_bn<64, 6, false>(ta, tb, p, splits, cluster, st);
  return ext ? launch_dense_bn<128, 4, true>(ta, tb, p, splits, cluster, st)
             : launch_dense_bn<128, 4, false>(ta, tb, p, splits, cluster, st);
}

template <int BN, bool EXT, bool U8, int TX, int TY, int CB, bool PAIR>
static auto slab_kernel() {
  if constexpr (PAIR) return &conv1_pair_wgmma_kernel;
  else return &conv_slab_wgmma_kernel<BN, EXT, U8, TX, TY, CB>;
}

template <int BN, bool EXT, bool U8, int TX, int TY, int CB, bool PAIR = false>
static int launch_slab_t(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ta2, const CUtensorMap& tb2,
                         SlabParams sp, cudaStream_t st) {
  const size_t w_bytes = (size_t)TX * TY * CB * BN * 128 + (PAIR ? (size_t)TX * TY * BN * 32 : 0);
  const size_t slab_bytes = (size_t)sp.slab_rows * 128 * CB + (PAIR ? pair_block_b_bytes(sp.slab_rows) : 0);
  const int tiles = (sp.g.M + GEMM_BM - 1) / GEMM_BM;
  // weights + slab ring + accumulator staging + barriers (+ uint8 staging) within the shared memory of one SM
  const size_t fixed = 1024 + acc_stage_bytes(BN) + (2 * 6 + 2) * 8 + 128;
  auto k = slab_kernel<BN, EXT, U8, TX, TY, CB, PAIR>();
  static const size_t limit = dyn_smem_limit(k);
  if (limit <= fixed) return 1;
  size_t u8_extra = 0;
  size_t budget = limit - fixed;
  if (U8) {
    // K1: three bf16 slabs are enough (shared -> shared conversion); everything else goes to uint8 staging tiles, each of which
    // is held for the copy latency plus the conversion
    const size_t ub = u8_stage_bytes(sp.slab_rows, sp.u8.G, sp.u8.frame_w, sp.u8.nf);
    if (w_bytes + 3 * slab_bytes + 2 * ub + 2 * U8_MAX_STAGES * 8 > budget) return 1;
    int us = (int)((budget - w_bytes - 3 * slab_bytes - 2 * U8_MAX_STAGES * 8) / ub);
    if (us > U8_MAX_STAGES) us = U8_MAX_STAGES;
    sp.u8.stages = us;
    u8_extra = (size_t)us * ub + 2 * U8_MAX_STAGES * 8;
    budget = w_bytes + 3 * slab_bytes;
  }
  if (w_bytes + 2 * slab_bytes > budget) return 1;                   // does not fit: caller falls back to tap addressing
  int stages = (int)((budget - w_bytes) / slab_bytes);
  if (stages > 6) stages = 6;
  sp.stages = stages;
  const size_t smem = fixed + w_bytes + stages * slab_bytes + u8_extra;
  static size_t attr = 0;
  if (attr < smem) {
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = smem;
  }
  int ctas = sp.g.dual ? grid_cap() / 2 : grid_cap();                 // per operand set
  if (ctas > tiles) ctas = tiles;
  if (ctas < 1) ctas = 1;
  g_last_ctas = sp.g.dual ? 2 * ctas : ctas;
  launch_pdl(k, dim3(sp.g.dual ? 2 * ctas : ctas), dim3(U8 ? SLAB_K1_THREADS : SLAB_THREADS), smem, st, ta, tb, ta2, tb2, sp);
  return check_launch("b2rl_conv_gemm_bf16(slab)");
}

// the slab kernel is instantiated for the layer shapes of NatureConvBody (taps_x x taps_y taps, col_blocks 64-channel blocks):
// conv1 forward (2x2, 1, block_n 32), conv2 forward (2x2, 2, 64), conv3 forward and dgrad (3x3, 1, 64), conv2 dgrad (2x2, 1,
// 128); returns 1 for any other shape (the caller falls back to tap addressing)
template <int BN, bool EXT>
static int launch_slab_shape(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ta2, const CUtensorMap& tb2,
                             const SlabParams& sp, cudaStream_t st) {
  const int tx = sp.g.taps_x, ty = sp.taps / sp.g.taps_x, cb = sp.col_blocks;
  if (tx * ty != sp.taps) return 1;
  if constexpr (BN == 32) {
    if (tx == 2 && ty == 2 && cb == 1) return launch_slab_t<32, EXT, false, 2, 2, 1>(ta, tb, ta2, tb2, sp, st);
  } else if constexpr (BN == 64) {
    if (tx == 2 && ty == 2 && cb == 2) return launch_slab_t<64, EXT, false, 2, 2, 2>(ta, tb, ta2, tb2, sp, st);
    if (tx == 3 && ty == 3 && cb == 1) return launch_slab_t<64, EXT, false, 3, 3, 1>(ta, tb, ta2, tb2, sp, st);
  } else {
    if (tx == 2 && ty == 2 && cb == 1) return launch_slab_t<128, EXT, false, 2, 2, 1>(ta, tb, ta2, tb2, sp, st);
  }
  return 1;
}

template <int BN>
static int launch_slab(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& ta2, const CUtensorMap& tb2,
                       SlabParams sp, cudaStream_t st) {
  if (sp.u8.frames) {                                                // K1: conv1 forward straight from the uint8 ring
    if constexpr (BN == 32) {
      if (!has_ext(sp.g) && !sp.g.dual && sp.col_blocks == 1 && sp.taps == 4 && sp.g.taps_x == 2)
        return launch_slab_t<32, false, true, 2, 2, 1>(ta, tb, ta2, tb2, sp, st);
    }
    set_error("the uint8-ring producer serves block_n 32, 2x2 taps of 64 channels, no backward extras, no dual launch");
    return B2RL_ERR_ARG;
  }
  return has_ext(sp.g) ? launch_slab_shape<BN, true>(ta, tb, ta2, tb2, sp, st)
                       : launch_slab_shape<BN, false>(ta, tb, ta2, tb2, sp, st);
}

// conv1_taps_conv_wgrad_wgmma_kernel: the 128-row k-blocks in equal contiguous ranges over at most one CTA per SM; returns
// the CTA count (= partial blocks written) through n_ctas, or 1 when the operand ring does not fit in shared memory
template <bool U8>
static int launch_conv1_wgrad(const CUtensorMap& tg, const CUtensorMap& tx, Conv1WgradParams w, cudaStream_t st, int* n_ctas) {
  auto k = conv1_taps_conv_wgrad_wgmma_kernel<U8>;
  static const size_t limit = dyn_smem_limit(k);
  const size_t stage = c1w_g_bytes(w.grid_w) + C1W_X_BYTES;
  // alignment of the ring + its barriers (+ U8: alignment of the uint8 staging tiles and their barriers)
  const size_t fixed = 1024 + 2 * 6 * 8 + (U8 ? 128 + 2 * U8_MAX_STAGES * 8 : 0);
  if (limit <= fixed) return 1;
  const size_t budget = limit - fixed;
  int stages = (int)(budget / stage);
  size_t u8_extra = 0;
  if (U8) {                                                          // K1: four operand stages, the rest for uint8 staging tiles
    const size_t ub = u8_stage_bytes(C1W_BK, w.u8.G, w.u8.frame_w, w.u8.nf);
    if (4 * stage + 2 * ub > budget) return 1;
    stages = 4;
    w.u8.stages = (int)((budget - 4 * stage) / ub);
    if (w.u8.stages > U8_MAX_STAGES) w.u8.stages = U8_MAX_STAGES;
    u8_extra = (size_t)w.u8.stages * ub;
  }
  if (stages > 6) stages = 6;
  if (stages < 2) return 1;
  w.stages = stages;
  const size_t smem = fixed + stages * stage + u8_extra;
  static size_t attr = 0;
  if (attr < smem) {
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = smem;
  }
  w.blocks = (w.rows + C1W_BK - 1) / C1W_BK;
  const int ctas = w.blocks < sm_count() ? w.blocks : sm_count();
  w.blocks_per_cta = (w.blocks + ctas - 1) / ctas;
  *n_ctas = (w.blocks + w.blocks_per_cta - 1) / w.blocks_per_cta;
  launch_pdl(k, dim3(*n_ctas), dim3(U8 ? SLAB_U8_THREADS : GEMM_THREADS), smem, st, tg, tx, w);
  return check_launch("conv1 weight gradient");
}

// conv_taps_wgrad_wgmma_kernel: the 128-row k-blocks in equal contiguous ranges over at most grid_cap() CTAs; returns the
// CTA count (= partial blocks written) through n_ctas, or 1 when the operand ring does not fit in shared memory
template <int C, int TAPS_X, int WGS>
static int launch_taps_wgrad(const CUtensorMap& tg, const CUtensorMap& tx, TapsWgradParams w, cudaStream_t st, int* n_ctas) {
  auto k = conv_taps_wgrad_wgmma_kernel<C, TAPS_X, WGS>;
  static const size_t limit = dyn_smem_limit(k);
  const size_t stage = ctw_g_bytes((TAPS_X - 1) * (w.grid_w + 1)) + (size_t)CTW_BK * 2 * C;
  const size_t fixed = 1024 + 2 * 6 * 8;                             // alignment of the ring + its barriers
  if (limit <= fixed) return 1;
  int stages = (int)((limit - fixed) / stage);
  if (stages > 6) stages = 6;
  if (stages < 2) return 1;
  w.stages = stages;
  const size_t smem = fixed + stages * stage;
  static size_t attr = 0;
  if (attr < smem) {
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = smem;
  }
  w.blocks = (w.rows + CTW_BK - 1) / CTW_BK;
  const int ctas = w.blocks < grid_cap() ? w.blocks : grid_cap();
  w.blocks_per_cta = (w.blocks + ctas - 1) / ctas;
  *n_ctas = (w.blocks + w.blocks_per_cta - 1) / w.blocks_per_cta;
  g_last_ctas = *n_ctas;
  launch_pdl(k, dim3(*n_ctas), dim3(ctw_threads<WGS>()), smem, st, tg, tx, w);
  return check_launch("conv2 / conv3 weight gradient");
}

}  // namespace b2rl

using namespace b2rl;

static int g_use_slab = 2;   // 2: shifted windows with base_offset 0 -- the 128B swizzle is a pure function of the smem address
static unsigned long long* g_k1_clocks = nullptr;
// Profiling hook of every slab launch (the K1 conv1 forwards b2rl_conv1_u8_fwd / b2rl_conv1_u8_fwd_pair, the slab forwards
// and dgrads of b2rl_conv_gemm_*) and of conv1's weight gradient (b2rl_conv1_u8_wgrad_partials, b2rl_conv1_wgrad_partials):
// while set, every launch adds its K1_CLK_SLOTS phase-cycle sums to clocks[] (scripts/slab_phase_time.py --phases,
// scripts/conv1_pair_time.py --phases, scripts/conv1_wgrad_time.py --phases).  Null (the default): no probe.
extern "C" int b2rl_conv1_set_phase_clocks(int64_t* clocks) {
  g_k1_clocks = reinterpret_cast<unsigned long long*>(clocks);
  return B2RL_OK;
}
extern "C" void b2rl_set_conv_slab(int32_t on) { g_use_slab = on; }

extern "C" int b2rl_set_cta_budget(int32_t ctas) {
  B2RL_REQUIRE(ctas >= 0, "the CTA budget is a CTA count (0: every SM)");
  g_cta_budget = ctas;
  return B2RL_OK;
}

extern "C" int b2rl_last_grid_ctas(int32_t* ctas) {
  B2RL_REQUIRE(ctas, "null pointer");
  *ctas = g_last_ctas;
  return B2RL_OK;
}

static int check_common(const void* A, const void* B, const void* D, int64_t lda, int64_t ldb, int M, int N, int K,
                        int out_mode, int splits, int block_n, int b_mn, int relu) {
  B2RL_REQUIRE(A && B && D, "null pointer");
  B2RL_REQUIRE(M > 0 && N > 0 && K > 0, "bad shape");
  B2RL_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "operand row strides must be multiples of 8 elements (16 bytes)");
  B2RL_REQUIRE((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) % 16 == 0, "operands must be 16-byte aligned");
  B2RL_REQUIRE(out_mode >= 0 && out_mode <= 2, "out_mode 0 (bf16) | 1 (fp32) | 2 (fp32 atomic add)");
  B2RL_REQUIRE(block_n == 32 || block_n == 64 || block_n == 128, "block_n must be 32, 64 or 128");
  B2RL_REQUIRE(!(b_mn && block_n < 64), "MN-major B needs block_n >= 64");
  B2RL_REQUIRE(splits >= 1 && (splits == 1 || out_mode == 2), "split-K needs out_mode 2 (atomic fp32 accumulation)");
  B2RL_REQUIRE(!(relu && out_mode == 2), "ReLU cannot be fused into an atomic accumulation");
  return B2RL_OK;
}

extern "C" int b2rl_gemm_bf16(const uint16_t* A, int32_t a_mn, int64_t lda, const uint16_t* B, int32_t b_mn, int64_t ldb,
                              void* D, int64_t ldd, int32_t M, int32_t N, int32_t K, const float* bias, int32_t relu,
                              int32_t out_mode, int32_t splits, int32_t block_n, void* stream) {
  int rc = check_common(A, B, D, lda, ldb, M, N, K, out_mode, splits, block_n, b_mn, relu);
  if (rc) return rc;
  GemmParams p = {};
  p.M = M; p.N = N; p.K = K; p.ldd = (int)ldd;
  p.a_mn = a_mn; p.b_mn = b_mn; p.relu = relu; p.out_mode = out_mode; p.bias = bias; p.D = D;
  p.taps_x = 1; p.shift_sign = 1;
  // K-major: stored [rows][K]; MN-major: stored [K][rows]
  return dense_dispatch(A, a_mn, lda, a_mn ? K : M, a_mn ? M : K, B, b_mn, ldb, b_mn ? K : N, b_mn ? N : K, p, splits,
                        block_n, 0, (cudaStream_t)stream);
}

// Convolution over a G x G grid as a shifted-row GEMM (see the header of this file).
//   mode 0 (forward / dgrad):  D[r, :] = sum_taps  X[r + shift(tap), :] * W[:, tap*C .. tap*C+C]^T
//        X: [rows][C] bf16 (C multiple of 64), W: [N][taps*C] bf16 K-major, shift(tap) = sign*((tap/taps_x)*grid_w + tap%taps_x)
//   mode 1 (wgrad):            D[n, tap*C + c] (+)= sum_r G[r, n] * X[r + shift(tap), c]
//        G: [rows][N_out] bf16, X: [rows][C] bf16 (C multiple of block_n), D: fp32 [N_out][taps*C], atomic accumulation
static int apply_ext(GemmParams& p, const b2rl_bwd_epilogue* ext, int N) {
  B2RL_REQUIRE(!ext->mask || (ext->mask_ld % 8 == 0 && reinterpret_cast<uintptr_t>(ext->mask) % 16 == 0 && N % 32 == 0),
               "mask rows must be 16-byte aligned and N a multiple of 32");
  B2RL_REQUIRE(!ext->dbias || (ext->dbias_mod >= 0 && ext->dbias_mod <= 128), "dbias_mod must be in [0, 128] (0: one bias per column)");
  B2RL_REQUIRE(p.out_map < 3 || (ext->sub_c > 0 && ext->sub_c % 32 == 0 && N % ext->sub_c == 0),
               "scatter maps need sub_c a multiple of 32 that divides N");
  p.mask = reinterpret_cast<const __nv_bfloat16*>(ext->mask);
  p.mask_ld = ext->mask_ld;
  p.dbias = ext->dbias;
  p.dbias_mod = ext->dbias ? ext->dbias_mod : 1;
  p.sub_c = ext->sub_c > 0 ? ext->sub_c : 32;
  return B2RL_OK;
}

static int conv_gemm_impl(int32_t mode, const uint16_t* X, int64_t rows, int32_t C, const uint16_t* W_or_G, int32_t n_out,
                          int32_t taps, int32_t taps_x, int32_t grid_w, int32_t shift_sign, void* D, int64_t ldd,
                          const float* bias, int32_t relu, int32_t out_mode, int32_t out_map, int32_t G, int32_t V,
                          int32_t splits, int32_t block_n, void* stream, const uint16_t* X2 = nullptr,
                          const uint16_t* W2 = nullptr, void* D2 = nullptr, const float* bias2 = nullptr,
                          const b2rl_bwd_epilogue* ext = nullptr) {
  B2RL_REQUIRE(mode == 0 || mode == 1, "mode 0 (forward/dgrad) or 1 (wgrad)");
  B2RL_REQUIRE(rows > 0 && C > 0 && taps > 0 && taps_x > 0 && n_out > 0, "bad shape");
  B2RL_REQUIRE(out_map >= 0 && out_map <= (ext ? 4 : 2), "bad out_map");
  GemmParams p = {};
  p.relu = relu; p.out_mode = out_mode; p.bias = bias; p.D = D; p.ldd = (int)ldd;
  p.taps_x = taps_x; p.grid_w = grid_w; p.shift_sign = shift_sign;
  p.out_map = out_map; p.G = G; p.V = V;
  p.dual = X2 != nullptr; p.D2 = D2; p.bias2 = bias2;
  if (ext) {
    int rc0 = apply_ext(p, ext, n_out);
    if (rc0) return rc0;
  }
  if (mode == 0) {
    B2RL_REQUIRE(C % 64 == 0, "forward/dgrad needs channels in multiples of 64");
    const int K = taps * C;
    int rc = check_common(X, W_or_G, D, C, K, (int)rows, n_out, K, out_mode, splits, block_n, 0, relu);
    if (rc) return rc;
    p.M = (int)rows; p.N = n_out; p.K = K; p.a_mn = 0; p.b_mn = 0; p.a_tap_tiles = C / 64;
    // the slab kernels' one output form (slab_epilogue_half): bf16 in whole 16-byte column groups; forwards with ReLU,
    // dgrads with mask and bias gradient.  Every other call goes to the tap-addressing kernel.
    const bool bf16_groups = out_mode == 0 && n_out % 8 == 0 && ldd % 8 == 0 &&
                             (reinterpret_cast<uintptr_t>(D) | reinterpret_cast<uintptr_t>(D2)) % 16 == 0;
    const bool slab_epilogue = ext ? (p.mask && p.dbias && !relu && !bias) : relu != 0;
    if (g_use_slab && splits == 1 && n_out <= block_n && bf16_groups && slab_epilogue) {
      const int max_shift = ((taps - 1) / taps_x) * grid_w + (taps - 1) % taps_x;
      SlabParams sp = {};
      sp.g = p; sp.taps = taps; sp.col_blocks = C / 64;
      sp.slab_rows = (GEMM_BM + max_shift + 7) / 8 * 8;
      sp.min_shift = shift_sign > 0 ? 0 : -max_shift;
      sp.base_offset_mode = g_use_slab;
      sp.clk = g_k1_clocks;
      if (sp.slab_rows <= 256) {
        CUtensorMap ta, tb, ta2, tb2;
        rc = make_map(&ta, X, C, rows, C, sp.slab_rows);            // box [slab_rows][64]
        if (rc) return rc;
        rc = make_map(&tb, W_or_G, K, n_out, K, block_n);           // box [block_n][64]
        if (rc) return rc;
        ta2 = ta, tb2 = tb;
        if (p.dual) {
          rc = make_map(&ta2, X2, C, rows, C, sp.slab_rows);
          if (rc) return rc;
          rc = make_map(&tb2, W2, K, n_out, K, block_n);
          if (rc) return rc;
        }
        int r2 = block_n == 32 ? launch_slab<32>(ta, tb, ta2, tb2, sp, (cudaStream_t)stream)
                 : block_n == 64 ? launch_slab<64>(ta, tb, ta2, tb2, sp, (cudaStream_t)stream)
                                 : launch_slab<128>(ta, tb, ta2, tb2, sp, (cudaStream_t)stream);
        if (r2 <= 0) return r2;                                      // launched (0) or failed (<0); 1 = does not fit
      }
    }
    return gemm_dispatch(X, 0, C, rows, C, W_or_G, 0, K, n_out, K, p, splits, block_n, (cudaStream_t)stream, X2, W2);
  }
  B2RL_REQUIRE(!p.dual, "the dual launch is for forward / dgrad GEMMs");
  B2RL_REQUIRE(C % block_n == 0, "wgrad needs channels in multiples of block_n");
  B2RL_REQUIRE(n_out % 8 == 0, "wgrad needs n_out in multiples of 8");
  int rc = check_common(W_or_G, X, D, n_out, C, n_out, taps * C, (int)rows, out_mode, splits, block_n, 1, relu);
  if (rc) return rc;
  B2RL_REQUIRE(out_mode == 2, "wgrad accumulates with out_mode 2");
  p.M = n_out; p.N = taps * C; p.K = (int)rows; p.a_mn = 1; p.b_mn = 1; p.b_tap_tiles = C / block_n;
  return gemm_dispatch(W_or_G, 1, n_out, rows, n_out, X, 1, C, rows, C, p, splits, block_n, (cudaStream_t)stream);
}

extern "C" int b2rl_conv_gemm_bf16(int32_t mode, const uint16_t* X, int64_t rows, int32_t C, const uint16_t* W_or_G,
                                   int32_t n_out, int32_t taps, int32_t taps_x, int32_t grid_w, int32_t shift_sign,
                                   void* D, int64_t ldd, const float* bias, int32_t relu, int32_t out_mode,
                                   int32_t out_map, int32_t G, int32_t V, int32_t splits, int32_t block_n, void* stream) {
  return conv_gemm_impl(mode, X, rows, C, W_or_G, n_out, taps, taps_x, grid_w, shift_sign, D, ldd, bias, relu, out_mode,
                        out_map, G, V, splits, block_n, stream);
}

// The same forward / dgrad convolution for TWO independent operand sets (online and target network) in one launch:
// D = conv(X, W) + bias and D2 = conv(X2, W2) + bias2, identical shapes.  Half of the CTAs work on each set.
extern "C" int b2rl_conv_gemm_dual_bf16(const uint16_t* X, const uint16_t* X2, int64_t rows, int32_t C, const uint16_t* W,
                                        const uint16_t* W2, int32_t n_out, int32_t taps, int32_t taps_x, int32_t grid_w,
                                        int32_t shift_sign, void* D, void* D2, int64_t ldd, const float* bias,
                                        const float* bias2, int32_t relu, int32_t out_mode, int32_t out_map, int32_t G,
                                        int32_t V, int32_t block_n, void* stream) {
  B2RL_REQUIRE(X2 && W2 && D2, "null pointer in the second operand set");
  B2RL_REQUIRE((reinterpret_cast<uintptr_t>(X2) | reinterpret_cast<uintptr_t>(W2)) % 16 == 0, "operands must be 16-byte aligned");
  B2RL_REQUIRE((bias == nullptr) == (bias2 == nullptr), "both or neither bias");
  return conv_gemm_impl(0, X, rows, C, W, n_out, taps, taps_x, grid_w, shift_sign, D, ldd, bias, relu, out_mode, out_map, G,
                        V, 1, block_n, stream, X2, W2, D2, bias2);
}

// D = A B^T + bias and D2 = A2 B2^T + bias2 (K-major operands, identical shapes) in one launch
extern "C" int b2rl_gemm_dual_bf16(const uint16_t* A, const uint16_t* A2, int64_t lda, const uint16_t* B, const uint16_t* B2,
                                   int64_t ldb, void* D, void* D2, int64_t ldd, int32_t M, int32_t N, int32_t K,
                                   const float* bias, const float* bias2, int32_t relu, int32_t out_mode, int32_t block_n,
                                   void* stream) {
  int rc = check_common(A, B, D, lda, ldb, M, N, K, out_mode, 1, block_n, 0, relu);
  if (rc) return rc;
  B2RL_REQUIRE(A2 && B2 && D2, "null pointer in the second operand set");
  B2RL_REQUIRE((reinterpret_cast<uintptr_t>(A2) | reinterpret_cast<uintptr_t>(B2)) % 16 == 0, "operands must be 16-byte aligned");
  B2RL_REQUIRE(out_mode != 2, "the dual launch stores (bf16 or fp32), it does not accumulate");
  B2RL_REQUIRE((bias == nullptr) == (bias2 == nullptr), "both or neither bias");
  GemmParams p = {};
  p.M = M; p.N = N; p.K = K; p.ldd = (int)ldd;
  p.relu = relu; p.out_mode = out_mode; p.bias = bias; p.D = D;
  p.taps_x = 1; p.shift_sign = 1;
  p.dual = 1; p.D2 = D2; p.bias2 = bias2;
  return gemm_dispatch(A, 0, lda, M, K, B, 0, ldb, N, K, p, 1, block_n, (cudaStream_t)stream, A2, B2);
}

// dgrad convolution with the backward extras fused into the epilogue (ReLU mask, bias gradient, grid scatter): D = mask .*
// conv_transpose(G_rows, W), see b2rl_bwd_epilogue in the header.  bf16 output.
extern "C" int b2rl_conv_gemm_bwd_bf16(const uint16_t* G_rows, int64_t rows, int32_t C, const uint16_t* W, int32_t n_out,
                                       int32_t taps, int32_t taps_x, int32_t grid_w, void* D, int64_t ldd, int32_t out_map,
                                       int32_t G, int32_t V, const b2rl_bwd_epilogue* ext, int32_t block_n, void* stream) {
  B2RL_REQUIRE(ext, "null epilogue description");
  B2RL_REQUIRE(out_map == 0 || out_map == 3, "dgrad output map 0 (same grid) or 3 (space-to-depth(2) -> grid)");
  return conv_gemm_impl(0, G_rows, rows, C, W, n_out, taps, taps_x, grid_w, -1, D, ldd, nullptr, 0, 0, out_map, G, V, 1,
                        block_n, stream, nullptr, nullptr, nullptr, nullptr, ext);
}

// D = mask .* (A B^T) with A [M][K] K-major and B K-major ([N][K]) or MN-major ([K][N]); same epilogue extras (fc4 dgrad)
extern "C" int b2rl_gemm_bwd_bf16(const uint16_t* A, int64_t lda, const uint16_t* B, int32_t b_mn, int64_t ldb, void* D,
                                  int64_t ldd, int32_t M, int32_t N, int32_t K, int32_t out_map, int32_t G, int32_t V,
                                  const b2rl_bwd_epilogue* ext, int32_t block_n, void* stream) {
  B2RL_REQUIRE(ext, "null epilogue description");
  B2RL_REQUIRE(out_map == 0 || out_map == 4, "output map 0 (plain) or 4 (per-image positions -> grid)");
  int rc = check_common(A, B, D, lda, ldb, M, N, K, 0, 1, block_n, b_mn, 0);
  if (rc) return rc;
  GemmParams p = {};
  p.M = M; p.N = N; p.K = K; p.ldd = (int)ldd;
  p.a_mn = 0; p.b_mn = b_mn; p.out_mode = 0; p.D = D;
  p.taps_x = 1; p.shift_sign = 1;
  p.out_map = out_map; p.G = G; p.V = V;
  rc = apply_ext(p, ext, N);
  if (rc) return rc;
  return dense_dispatch(A, 0, lda, M, K, B, b_mn, ldb, b_mn ? K : N, b_mn ? N : K, p, 1, block_n, 0, (cudaStream_t)stream);
}

// D = act(A B^T + bias) in bf16, K split over the `splits` CTAs of a cluster per output tile and the partials summed in
// distributed shared memory in rank order (dense_gemm_kernel): one launch, no scratch, the same bits in every launch.
// A [M][K], B [N][K] K-major bf16; splits 1, 2, 4 or 8 (1: one CTA per tile over all of K), or 0: the cluster size the
// launcher picks from the shape (auto_cluster).  fc4 of NatureConvBody (network_bodies.py:33).
extern "C" int b2rl_gemm_splitk_bf16(const uint16_t* A, int64_t lda, const uint16_t* B, int64_t ldb, void* D, int64_t ldd,
                                     int32_t M, int32_t N, int32_t K, const float* bias, int32_t relu, int32_t splits,
                                     int32_t block_n, void* stream) {
  B2RL_REQUIRE(splits == 0 || splits == 1 || splits == 2 || splits == 4 || splits == 8, "splits must be 0, 1, 2, 4 or 8");
  int rc = check_common(A, B, D, lda, ldb, M, N, K, 0, 1, block_n, 0, relu);
  if (rc) return rc;
  GemmParams p = {};
  p.M = M; p.N = N; p.K = K; p.ldd = (int)ldd;
  p.relu = relu; p.out_mode = 0; p.bias = bias; p.D = D;
  p.taps_x = 1; p.shift_sign = 1;
  return dense_dispatch(A, 0, lda, M, K, B, 0, ldb, N, K, p, 1, block_n, splits, (cudaStream_t)stream);
}


// ---------------------------------------------------------------------------------------------------------------
// K1 entry points: conv1 of NatureConvBody (network_bodies.py:27; 8x8 / stride 4 over `history` stacked frames = 2x2 taps
// over the space-to-depth(4) grid) reading the sampled frame stacks STRAIGHT FROM THE uint8 REPLAY RING (replay.py:124-134)
// -- no materialised batch.  frames: ring [capacity][row_bytes]; idx: int64 [batch] sampled ring indices; `first`: ring row
// of the oldest stacked frame relative to idx[b] (-(history-1) for the state, n_step-(history-1) for the next state).
// The frame values enter as exact integers 0..255; ImageNormalizer's 1/255 is folded into W (b2rl_nature_pack_weights).
// ---------------------------------------------------------------------------------------------------------------
// 3-D tensor map over the uint8 ring as 32-bit words: [capacity][G grid rows][frame_w words], box [nf frames][slots][frame_w]
static int make_ring_map(CUtensorMap* m, const uint8_t* frames, int64_t capacity, int64_t row_bytes, int frame_w, int slots,
                         int nf) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return B2RL_ERR_CUDA; }
  cuuint64_t gdim[3] = {(cuuint64_t)frame_w, (cuuint64_t)(frame_w / 4), (cuuint64_t)capacity};
  cuuint64_t gstr[2] = {(cuuint64_t)4 * frame_w, (cuuint64_t)row_bytes};
  cuuint32_t box[3] = {(cuuint32_t)frame_w, (cuuint32_t)slots, (cuuint32_t)nf};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<uint8_t*>(frames), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (uint8 ring) failed (%d)", (int)r); return B2RL_ERR_CUDA; }
  return B2RL_OK;
}

static int u8_src(U8Src& u, const uint8_t* frames, const int64_t* idx, int32_t first, int64_t row_bytes, int32_t frame_w,
                  int32_t batch, int32_t history) {
  B2RL_REQUIRE(frames && idx, "null pointer");
  B2RL_REQUIRE(history == 4, "the uint8-ring producer packs 4 frames x 16 pixels into the 64 channels of one slab column block");
  B2RL_REQUIRE(frame_w > 0 && frame_w % 4 == 0 && row_bytes % frame_w == 0 && row_bytes / frame_w == frame_w,
               "square frames with a side that is a multiple of 4");
  B2RL_REQUIRE(reinterpret_cast<uintptr_t>(frames) % 16 == 0 && row_bytes % 16 == 0 && (4 * frame_w) % 16 == 0 && frame_w <= 256,
               "ring rows and grid rows must be 16-byte aligned (TMA strides), frames at most 256 pixels wide");
  B2RL_REQUIRE(batch > 0 && (int64_t)batch * (frame_w / 4) * (frame_w / 4) < (1LL << 31), "bad batch");
  u.frames = frames; u.idx = idx; u.row_bytes = row_bytes; u.first = first; u.frame_w = frame_w; u.G = frame_w / 4;
  u.rows = batch * u.G * u.G;
  u.nf = history;
  return B2RL_OK;
}

// D = act(conv1(frames) + bias): rows (b, gy, gx) of the G x G grid, n_out <= 32 output channels, bf16, through the output row
// maps of b2rl_conv_gemm_bf16 (out_map 1 = space-to-depth(2) rows for conv2, valid V x V).  W: [n_out][4 taps * 64] bf16.
extern "C" int b2rl_conv1_u8_fwd(const uint8_t* frames, int64_t capacity, const int64_t* idx, int32_t first, int64_t row_bytes,
                                 int32_t frame_w, int32_t batch, int32_t history, const uint16_t* W, int32_t n_out, void* D, int64_t ldd,
                                 const float* bias, int32_t relu, int32_t out_map, int32_t V, void* stream) {
  SlabParams sp = {};
  int rc = u8_src(sp.u8, frames, idx, first, row_bytes, frame_w, batch, history);
  if (rc) return rc;
  B2RL_REQUIRE(W && D, "null pointer");
  B2RL_REQUIRE(n_out > 0 && n_out <= 32 && n_out % 8 == 0 && out_map >= 0 && out_map <= 2, "n_out 8, 16, 24 or 32, out_map 0..2");
  B2RL_REQUIRE((reinterpret_cast<uintptr_t>(W) | reinterpret_cast<uintptr_t>(D)) % 16 == 0 && ldd % 8 == 0,
               "operands and output must be 16-byte aligned, ldd a multiple of 8");
  B2RL_REQUIRE(relu, "the slab forward applies ReLU (conv1 of NatureConvBody)");
  const int G = sp.u8.G, C = 64, taps = 4, K = taps * C;
  GemmParams p = {};
  p.M = sp.u8.rows; p.N = n_out; p.K = K; p.ldd = (int)ldd;
  p.relu = relu; p.out_mode = 0; p.bias = bias; p.D = D;
  p.taps_x = 2; p.grid_w = G; p.shift_sign = 1; p.a_tap_tiles = 1;
  p.out_map = out_map; p.G = G; p.V = V;
  const int max_shift = G + 1;
  sp.g = p; sp.taps = taps; sp.col_blocks = 1;
  sp.slab_rows = (GEMM_BM + max_shift + 7) / 8 * 8;
  sp.min_shift = 0;
  sp.base_offset_mode = 2;
  B2RL_REQUIRE(sp.slab_rows <= 256, "frame too wide for one slab");
  B2RL_REQUIRE(capacity > 0, "bad capacity");
  CUtensorMap tb, tr;
  rc = make_map(&tb, W, K, n_out, K, 32);
  if (rc) return rc;
  rc = make_ring_map(&tr, frames, capacity, row_bytes, frame_w, u8_slots(sp.slab_rows, G), sp.u8.nf);
  if (rc) return rc;
  sp.clk = g_k1_clocks;
  int r2 = launch_slab<32>(tr, tb, tr, tb, sp, (cudaStream_t)stream);
  if (r2 > 0) { set_error("b2rl_conv1_u8_fwd: the slab does not fit in shared memory"); return B2RL_ERR_ARG; }
  return r2;
}

// 3-D bf16 tensor map over conv1's packed weights [32 n][4 taps][64 k] (K-major, tap-major columns), box [32 n][1 tap][box_k k]
static int make_w1_map(CUtensorMap* m, const uint16_t* W, int box_k, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return B2RL_ERR_CUDA; }
  cuuint64_t gdim[3] = {64u, 4u, 32u};
  cuuint64_t gstr[2] = {64u * 2, 4u * 64 * 2};
  cuuint32_t box[3] = {(cuuint32_t)box_k, 1u, 32u};
  cuuint32_t estr[3] = {1u, 1u, 1u};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<uint16_t*>(W), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (conv1 weights) failed (%d)", (int)r); return B2RL_ERR_CUDA; }
  return B2RL_OK;
}

// D = act(conv1_W(s) + bias) and D2 = act(conv1_W2(s') + bias2) in ONE launch (PAIR in conv_slab_wgmma_kernel), s the stacks
// idx[b] + first .. + 3 and s' the stacks one ring row later (n_step 1): both are read from the five ring rows
// idx[b] + first .. + 4.  W, W2: [32][4 taps * 64] as b2rl_conv1_u8_fwd takes them; D, D2: as its D (n_out 32, row stride ldd).
// The bits equal those of two b2rl_conv1_u8_fwd launches (first and first + 1).
extern "C" int b2rl_conv1_u8_fwd_pair(const uint8_t* frames, int64_t capacity, const int64_t* idx, int32_t first,
                                      int64_t row_bytes, int32_t frame_w, int32_t batch, int32_t history, const uint16_t* W,
                                      const uint16_t* W2, void* D, void* D2, int64_t ldd, const float* bias, const float* bias2,
                                      int32_t relu, int32_t out_map, int32_t V, void* stream) {
  SlabParams sp = {};
  int rc = u8_src(sp.u8, frames, idx, first, row_bytes, frame_w, batch, history);
  if (rc) return rc;
  B2RL_REQUIRE(W && W2 && D && D2, "null pointer");
  B2RL_REQUIRE(D != D2, "the two outputs must be distinct buffers");
  B2RL_REQUIRE((bias == nullptr) == (bias2 == nullptr), "both or neither bias");
  B2RL_REQUIRE(out_map >= 0 && out_map <= 2, "out_map 0..2");
  B2RL_REQUIRE(ldd >= (out_map == 1 ? 128 : 32) && ldd % 8 == 0, "ldd must hold the 32 output channels (x 4 for out_map 1), multiple of 8");
  B2RL_REQUIRE(frame_w == 84, "the paired forward serves 84 x 84 frames");
  B2RL_REQUIRE((reinterpret_cast<uintptr_t>(W) | reinterpret_cast<uintptr_t>(W2) | reinterpret_cast<uintptr_t>(D) |
                reinterpret_cast<uintptr_t>(D2)) % 16 == 0, "operands and outputs must be 16-byte aligned");
  B2RL_REQUIRE(capacity >= history + 1, "bad capacity");
  B2RL_REQUIRE(relu, "the slab forward applies ReLU (conv1 of NatureConvBody)");
  sp.u8.nf = history + 1;                                  // the window of s and s'
  const int G = sp.u8.G;
  GemmParams p = {};
  p.M = sp.u8.rows; p.N = 32; p.K = 4 * 64; p.ldd = (int)ldd;
  p.relu = relu; p.out_mode = 0; p.bias = bias; p.D = D; p.bias2 = bias2; p.D2 = D2;
  p.taps_x = 2; p.grid_w = G; p.shift_sign = 1; p.a_tap_tiles = 1;
  p.out_map = out_map; p.G = G; p.V = V;
  sp.g = p; sp.taps = 4; sp.col_blocks = 1;
  sp.slab_rows = (GEMM_BM + G + 1 + 7) / 8 * 8;
  sp.min_shift = 0;
  sp.base_offset_mode = 2;
  CUtensorMap tr, tw, tw2a, tw2b;
  rc = make_ring_map(&tr, frames, capacity, row_bytes, frame_w, u8_slots(sp.slab_rows, G), sp.u8.nf);
  if (rc) return rc;
  rc = make_w1_map(&tw, W, 64, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  rc = make_w1_map(&tw2a, W2, 64, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  rc = make_w1_map(&tw2b, W2, 16, CU_TENSOR_MAP_SWIZZLE_32B);
  if (rc) return rc;
  sp.clk = g_k1_clocks;
  int r2 = launch_slab_t<64, false, true, 2, 2, 1, true>(tr, tw, tw2a, tw2b, sp, (cudaStream_t)stream);
  if (r2 > 0) { set_error("b2rl_conv1_u8_fwd_pair: the slab does not fit in shared memory"); return B2RL_ERR_ARG; }
  return r2;
}

// 2-D bf16 tensor map over conv1's output gradient [rows][32] (64-byte rows), box [BK + G + 1 rows][32], 64-byte swizzle
static int make_g1_map(CUtensorMap* m, const uint16_t* G_rows, int64_t rows, int grid_w) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return B2RL_ERR_CUDA; }
  cuuint64_t gdim[2] = {32u, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {64u};
  cuuint32_t box[2] = {32u, (cuuint32_t)(C1W_BK + grid_w + 1)};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<uint16_t*>(G_rows), gdim, gstr, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (conv1 output gradient) failed (%d)", (int)r); return B2RL_ERR_CUDA; }
  return B2RL_OK;
}

static int conv1_wgrad_args(const uint16_t* G_rows, int32_t n_out, int grid_w, const float* partials, const int32_t* n_partials_host) {
  B2RL_REQUIRE(G_rows && partials && n_partials_host, "null pointer");
  B2RL_REQUIRE(n_out == 32, "conv1's weight gradient has n_out 32");
  B2RL_REQUIRE(grid_w > 0 && C1W_BK + grid_w + 1 <= 256, "grid too wide for one gradient box");
  B2RL_REQUIRE(reinterpret_cast<uintptr_t>(G_rows) % 16 == 0, "operands must be 16-byte aligned");
  B2RL_REQUIRE(reinterpret_cast<uintptr_t>(partials) % 8 == 0, "partials must be 8-byte aligned");
  return B2RL_OK;
}

// split-K partials of conv1's weight gradient dW[n][tap*64 + c] = sum_r G[r][n] * x[r + shift(tap)][c] with x read from the
// ring as above (G_rows: bf16 [batch*G*G][32], the masked output gradient on conv1's grid; n_out must be 32).  One partial
// per CTA, at most one per SM: partial i at partials + i * 32 * 256, *n_partials_host of them; the consumer sums them.  Same
// bits as b2rl_conv1_wgrad_partials on the materialised stacks.
extern "C" int b2rl_conv1_u8_wgrad_partials(const uint8_t* frames, int64_t capacity, const int64_t* idx, int32_t first,
                                            int64_t row_bytes, int32_t frame_w, int32_t batch, int32_t history, const uint16_t* G_rows,
                                            int32_t n_out, float* partials, int32_t* n_partials_host, void* stream) {
  Conv1WgradParams w = {};
  int rc = u8_src(w.u8, frames, idx, first, row_bytes, frame_w, batch, history);
  if (rc) return rc;
  rc = conv1_wgrad_args(G_rows, n_out, w.u8.G, partials, n_partials_host);
  if (rc) return rc;
  B2RL_REQUIRE(capacity > 0, "bad capacity");
  w.rows = w.u8.rows; w.grid_w = w.u8.G; w.D = partials; w.clk = g_k1_clocks;
  CUtensorMap tg, tr;
  rc = make_g1_map(&tg, G_rows, w.rows, w.grid_w);
  if (rc) return rc;
  rc = make_ring_map(&tr, frames, capacity, row_bytes, frame_w, u8_slots(C1W_BK, w.u8.G), w.u8.nf);
  if (rc) return rc;
  int n = 0;
  const int r2 = launch_conv1_wgrad<true>(tg, tr, w, (cudaStream_t)stream, &n);
  if (r2 > 0) { set_error("b2rl_conv1_u8_wgrad_partials: the operand ring does not fit in shared memory"); return B2RL_ERR_ARG; }
  *n_partials_host = n;
  return r2;
}

// The same partials from the materialised bf16 stacks X [rows][64] (conv1's space-to-depth(4) grid matrix, G = grid_w):
// conv1_taps_conv_wgrad_wgmma_kernel with a TMA-loaded activation block.
extern "C" int b2rl_conv1_wgrad_partials(const uint16_t* X, int64_t rows, int32_t grid_w, const uint16_t* G_rows, int32_t n_out,
                                         float* partials, int32_t* n_partials_host, void* stream) {
  int rc = conv1_wgrad_args(G_rows, n_out, grid_w, partials, n_partials_host);
  if (rc) return rc;
  B2RL_REQUIRE(X && reinterpret_cast<uintptr_t>(X) % 16 == 0, "operands must be 16-byte aligned");
  B2RL_REQUIRE(rows > 0 && rows < (1LL << 31), "bad shape");
  Conv1WgradParams w = {};
  w.rows = (int)rows; w.grid_w = grid_w; w.D = partials; w.clk = g_k1_clocks;
  CUtensorMap tg, tx;
  rc = make_g1_map(&tg, G_rows, rows, grid_w);
  if (rc) return rc;
  rc = make_map(&tx, X, 64, rows, 64, C1W_BK);                       // activation block: box [128 rows][64 c]
  if (rc) return rc;
  int n = 0;
  const int r2 = launch_conv1_wgrad<false>(tg, tx, w, (cudaStream_t)stream, &n);
  if (r2 > 0) { set_error("b2rl_conv1_wgrad_partials: the operand ring does not fit in shared memory"); return B2RL_ERR_ARG; }
  *n_partials_host = n;
  return r2;
}

// conv2's and conv3's weight-gradient partials, every tap of a k-block in one CTA (conv_taps_wgrad_wgmma_kernel): one
// partial per CTA (at most one per SM, or the CTA budget), partial i at partials + i * n_out * taps * C, *n_partials_host
// of them; the consumer (b2rl_nature_unpack_grads, b2rl_nature_grad_reduce) sums them.
extern "C" int b2rl_conv_taps_wgrad_partials(const uint16_t* X, int64_t rows, int32_t C, const uint16_t* G, int32_t n_out,
                                             int32_t taps, int32_t taps_x, int32_t grid_w, float* partials,
                                             int32_t* n_partials_host, void* stream) {
  B2RL_REQUIRE(X && G && partials && n_partials_host, "null pointer");
  B2RL_REQUIRE(n_out == 64 && ((C == 64 && taps == 9 && taps_x == 3) || (C == 128 && taps == 4 && taps_x == 2)),
               "the taps weight gradient serves n_out 64 with C 64 and 3 x 3 taps (conv3) or C 128 and 2 x 2 taps (conv2)");
  const int halo = (taps_x - 1) * (grid_w + 1);
  B2RL_REQUIRE(grid_w > 0 && CTW_BK + halo <= 256, "grid too wide for one gradient box");
  B2RL_REQUIRE(rows > 0 && rows < (1LL << 31), "bad shape");
  B2RL_REQUIRE((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(G)) % 16 == 0, "operands must be 16-byte aligned");
  B2RL_REQUIRE(reinterpret_cast<uintptr_t>(partials) % 8 == 0, "partials must be 8-byte aligned");
  TapsWgradParams w = {};
  w.rows = (int)rows; w.grid_w = grid_w; w.D = partials; w.clk = g_k1_clocks;
  CUtensorMap tg, tx;
  int rc = make_map(&tg, G, 64, rows, 64, CTW_BK + halo);             // gradient box: [BK + halo rows][64 n]
  if (rc) return rc;
  rc = make_map(&tx, X, C, rows, C, CTW_BK);                         // activation block: C / 64 boxes [128 rows][64 c]
  if (rc) return rc;
  int n = 0;
  const int r2 = C == 64 ? launch_taps_wgrad<64, 3, 3>(tg, tx, w, (cudaStream_t)stream, &n)
                         : launch_taps_wgrad<128, 2, 2>(tg, tx, w, (cudaStream_t)stream, &n);
  if (r2 > 0) { set_error("b2rl_conv_taps_wgrad_partials: the operand ring does not fit in shared memory"); return B2RL_ERR_ARG; }
  *n_partials_host = n;
  return r2;
}
