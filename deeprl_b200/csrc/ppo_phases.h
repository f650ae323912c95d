// ppo_phases.h -- the PPO minibatch update (PPO_agent.py:73-99, non-shared representation) written as PHASES of a single
// thread block: every function below takes (tid, NT) and is executed by all NT threads of the block, with a block barrier
// between consecutive phases (the sequence is ppo_sequence.inc).  csrc/ppo_persistent.cu runs the sequence as ONE persistent
// kernel over all minibatches of an iteration (weights in shared memory, Adam moments in L2); tests/host_emul/ppo_emul.cpp
// compiles the SAME functions with g++ and runs the threads of a phase one after another, which is how the arithmetic is
// checked against the oracle without a GPU.  Nothing here may depend on execution order inside a phase.
//
//   network   GaussianActorCriticNet (network_heads.py:173-214) with DummyBody phi, actor / critic FCBody(tanh) of two layers:
//             mean = tanh(fc_action(actor_body(x))), v = fc_critic(critic_body(x)), std = softplus(std_param)
//   losses    PPO_agent.py:79-88 (ratio, clipped surrogate, entropy bonus, value loss, approx_kl)
//   updates   PPO_agent.py:94-99: actor Adam step iff approx_kl <= 1.5 * target_kl; critic Adam step always
//             (torch.optim.Adam, _single_tensor_adam arithmetic, as csrc/optim.cu adam_kernel)
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define PPO_FN __device__ __forceinline__
#define PPO_HD __host__ __device__ inline
// the dense building blocks are called from several phases: ONE copy each (the kernel runs as a single block, and with every
// block inlined into every phase its code was 400 KB -- an order of magnitude beyond the 32 KB instruction cache).  Their pointer arguments are shared-memory addresses at every call site, which
// the compiler propagates into the one copy (LDS, not generic loads).
#define PPO_SUB __device__ __noinline__
#define PPO_LOOP _Pragma("unroll 1")
#else
#define PPO_FN static inline
#define PPO_HD static inline
#define PPO_SUB static
#define PPO_LOOP
#include <chrono>
#endif

namespace b2rl_ppo {

struct PpoArgs {
  // rollout rows (device): state [R][D], action [R][A], old log-prob / return / normalised advantage [R]
  const float* state; const float* action; const float* old_logp; const float* ret; const float* adv;
  int D, A, H1, H2, mb;
  const int64_t* perm;        // [n_batches][mb] row indices (np.random.permutation rows, misc.py:55-62)
  int n_batches;
  // flat arenas of the two FlatOptimizers (ops.py): parameters, exp_avg, exp_avg_sq, step count; tensor offsets inside them
  float* a_flat; float* a_m; float* a_v; int64_t* a_step; int a_off[7];     // w1 b1 w2 b2 fc_action.w fc_action.b std
  float* c_flat; float* c_m; float* c_v; int64_t* c_step; int c_off[6];     // w1 b1 w2 b2 fc_critic.w fc_critic.b
  float a_lr, a_b1, a_b2, a_eps, c_lr, c_b1, c_b2, c_eps;
  float clip, ent_w, gate_max;
  float* stats;               // [4]: policy loss, value loss, approx_kl of the LAST minibatch; actor steps taken in this call
  long long* clk;             // profiling hook (device only, normally null): clock64() of thread 0 after every phase barrier
};

struct PpoShared {
  float *aw1, *ab1, *aw2, *ab2, *aw3, *ab3, *sdp;      // actor weights (aw3 = fc_action), std parameter
  float *cw1, *cb1, *cw2, *cb2, *cw3, *cb3;            // critic weights (cw3 = fc_critic, one row)
  float *xb, *actb, *oldlpb, *advb, *retb;             // double-buffered minibatch rows: buffer s at + s * (x|act|row)_stride
  int x_stride, act_stride, row_stride;                // (no pointer arrays: a dynamically indexed member would push the struct to local memory)
  float *ah1, *ah2, *ad1, *ad2;                        // actor  [mb][ldh] activations / pre-activation gradients
  float *ch1, *ch2, *cd1, *cd2;                        // critic (the two networks run side by side, one half of the block each)
  float *mu, *dmu, *dsd;                               // [mb][A]
  float *v, *dv, *logp, *dlogp, *red;                  // [mb]; red [3*mb]
  float *sdv, *lsd;                                    // [A] softplus(std), log of it
  float *flag;                                         // [8]: 0 gate, 1 actor steps taken, 2 policy loss, 3 kl, 4 value loss
  int* steps;                                          // [2] Adam step counts: actor, critic
  int ld1, ldh, lda;                                   // row strides: multiples of 4 floats (16-byte rows for 128-bit loads); ld1 / ldh with an
                                                       // odd number of 16-byte pieces, so that a walk down a column is bank-conflict-free
};

PPO_HD int ppo_ld(int n) {                 // smallest multiple of 4 >= n whose quarter is odd (17 -> 20, 64 -> 68)
  int q = (n + 3) / 4;
  if ((q & 1) == 0) ++q;
  return 4 * q;
}

// carve the shared block (base may be a dummy when only the size is wanted); returns the number of floats used
PPO_HD size_t ppo_carve(PpoShared& S, float* base, int D, int A, int H1, int H2, int mb) {
  const int Hm = H1 > H2 ? H1 : H2;
  S.ld1 = ppo_ld(D);
  S.ldh = ppo_ld(Hm);
  S.lda = (A + 3) / 4 * 4;
  size_t off = 0;
#define PPO_TAKE(n) (base + (off += ((size_t)(n) + 3) / 4 * 4) - ((size_t)(n) + 3) / 4 * 4)
  const size_t w1 = (size_t)H1 * S.ld1, w2 = (size_t)H2 * S.ldh, act = (size_t)mb * S.ldh, ma = (size_t)mb * S.lda;
  S.aw1 = PPO_TAKE(w1); S.ab1 = PPO_TAKE(H1); S.aw2 = PPO_TAKE(w2); S.ab2 = PPO_TAKE(H2);
  S.aw3 = PPO_TAKE((size_t)A * S.ldh); S.ab3 = PPO_TAKE(A); S.sdp = PPO_TAKE(A);
  S.cw1 = PPO_TAKE(w1); S.cb1 = PPO_TAKE(H1); S.cw2 = PPO_TAKE(w2); S.cb2 = PPO_TAKE(H2);
  S.cw3 = PPO_TAKE(S.ldh); S.cb3 = PPO_TAKE(1);
  S.x_stride = (int)(((size_t)mb * S.ld1 + 3) / 4 * 4); S.act_stride = (int)(((size_t)mb * A + 3) / 4 * 4); S.row_stride = (mb + 3) / 4 * 4;
  S.xb = PPO_TAKE(2 * (size_t)S.x_stride); S.actb = PPO_TAKE(2 * (size_t)S.act_stride);
  S.oldlpb = PPO_TAKE(2 * (size_t)S.row_stride); S.advb = PPO_TAKE(2 * (size_t)S.row_stride); S.retb = PPO_TAKE(2 * (size_t)S.row_stride);
  S.ah1 = PPO_TAKE(act); S.ah2 = PPO_TAKE(act); S.ad1 = PPO_TAKE(act); S.ad2 = PPO_TAKE(act);
  S.ch1 = PPO_TAKE(act); S.ch2 = PPO_TAKE(act); S.cd1 = PPO_TAKE(act); S.cd2 = PPO_TAKE(act);
  S.mu = PPO_TAKE(ma); S.dmu = PPO_TAKE(ma); S.dsd = PPO_TAKE(ma);
  S.v = PPO_TAKE(mb); S.dv = PPO_TAKE(mb); S.logp = PPO_TAKE(mb); S.dlogp = PPO_TAKE(mb); S.red = PPO_TAKE((size_t)3 * mb);
  S.sdv = PPO_TAKE(A); S.lsd = PPO_TAKE(A);
  S.flag = PPO_TAKE(8);
  S.steps = reinterpret_cast<int*>(PPO_TAKE(4));
#undef PPO_TAKE
  return off;
}

// ------------------------------------------------------------------------------------------------ dense building blocks
// Every operand row starts on a 16-byte boundary and the reduction index runs along rows, so the inner loops read 4 floats
// per shared-memory load (LDS.128); a remainder of the reduction length (17 inputs, 6 actions) takes a scalar tail.  Tiles are
// 4 x 4 outputs per thread: 8 vector loads feed 64 FMAs (shared-memory bandwidth, not the FMA pipe, bounded the scalar form).
struct alignas(16) ppo_f4 { float x, y, z, w; };
PPO_FN ppo_f4 ppo_ld4(const float* p) { return *reinterpret_cast<const ppo_f4*>(p); }
PPO_FN void ppo_st4(float* p, const ppo_f4& v) { *reinterpret_cast<ppo_f4*>(p) = v; }
PPO_SUB float ppo_tanh(float x) { return tanhf(x); }
PPO_FN float ppo_dot4(const ppo_f4& a, const ppo_f4& b, float acc) {
  acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc); acc = fmaf(a.z, b.z, acc); return fmaf(a.w, b.w, acc);
}

// out[n][j] = f(sum_k in[n][k] * W[j][k] + bias[j])       n < M (M % 4 == 0), j < J, k < K
// tile = rows 4tn..4tn+3 x INTERLEAVED columns tj + tiles_j * c: consecutive threads read consecutive rows of W, which with
// an odd number of 16-byte pieces per row is conflict-free
PPO_FN void dense_fwd(const float* in, int ldin, const float* W, int ldw, const float* bias, float* out, int ldout, int M,
                      int K, int J, bool use_tanh, int tid, int NT) {
  const int tjn = (J + 3) / 4, tiles = (M / 4) * tjn, K4 = K & ~3;
  PPO_LOOP
  for (int t = tid; t < tiles; t += NT) {
    const int tn = t / tjn, tj = t - tn * tjn;
    int jj[4];
    bool ok[4];
    for (int c = 0; c < 4; ++c) {
      jj[c] = tj + tjn * c;
      ok[c] = jj[c] < J;
      if (!ok[c]) jj[c] = J - 1;
    }
    float acc[4][4];
    for (int i = 0; i < 4; ++i)
      for (int c = 0; c < 4; ++c) acc[i][c] = 0.0f;
    const float* xr = in + (size_t)(4 * tn) * ldin;
    PPO_LOOP
    for (int k = 0; k < K4; k += 4) {
      ppo_f4 xv[4], wv[4];
      for (int i = 0; i < 4; ++i) xv[i] = ppo_ld4(xr + i * ldin + k);
      for (int c = 0; c < 4; ++c) wv[c] = ppo_ld4(W + jj[c] * ldw + k);
      for (int i = 0; i < 4; ++i)
        for (int c = 0; c < 4; ++c) acc[i][c] = ppo_dot4(xv[i], wv[c], acc[i][c]);
    }
    PPO_LOOP
    for (int k = K4; k < K; ++k) {
      float xv[4], wv[4];
      for (int i = 0; i < 4; ++i) xv[i] = xr[i * ldin + k];
      for (int c = 0; c < 4; ++c) wv[c] = W[jj[c] * ldw + k];
      for (int i = 0; i < 4; ++i)
        for (int c = 0; c < 4; ++c) acc[i][c] = fmaf(xv[i], wv[c], acc[i][c]);
    }
    for (int i = 0; i < 4; ++i)
      for (int c = 0; c < 4; ++c)
        if (ok[c]) {
          const float s = acc[i][c] + bias[jj[c]];
          out[(size_t)(4 * tn + i) * ldout + jj[c]] = use_tanh ? ppo_tanh(s) : s;
        }
  }
}

// out[n][k] = (sum_j d[n][j] * W[j][k]) * (1 - h[n][k]^2)       back through a tanh layer whose output is h
// tile = rows 4tn..4tn+3 x CONSECUTIVE columns 4tk..4tk+3 (one 128-bit load per row of W); d rows 16-byte aligned unless ldd = 1
PPO_FN void dense_bwd_data(const float* d, int ldd, const float* W, int ldw, const float* h, int ldhh, float* out, int ldout,
                           int M, int J, int K, int tid, int NT) {
  const int tkn = (K + 3) / 4, tiles = (M / 4) * tkn, J4 = (ldd & 3) ? 0 : (J & ~3);
  PPO_LOOP
  for (int t = tid; t < tiles; t += NT) {
    const int tn = t / tkn, tk = t - tn * tkn;
    float acc[4][4];
    for (int i = 0; i < 4; ++i)
      for (int c = 0; c < 4; ++c) acc[i][c] = 0.0f;
    const float* dr = d + (size_t)(4 * tn) * ldd;
    const float* wc = W + 4 * tk;
    PPO_LOOP
    for (int j = 0; j < J4; j += 4) {
      ppo_f4 dv[4], wv[4];
      for (int i = 0; i < 4; ++i) dv[i] = ppo_ld4(dr + i * ldd + j);
      for (int q = 0; q < 4; ++q) wv[q] = ppo_ld4(wc + (j + q) * ldw);
      for (int i = 0; i < 4; ++i) {
        const float dq[4] = {dv[i].x, dv[i].y, dv[i].z, dv[i].w};
        for (int q = 0; q < 4; ++q) {
          acc[i][0] = fmaf(dq[q], wv[q].x, acc[i][0]); acc[i][1] = fmaf(dq[q], wv[q].y, acc[i][1]);
          acc[i][2] = fmaf(dq[q], wv[q].z, acc[i][2]); acc[i][3] = fmaf(dq[q], wv[q].w, acc[i][3]);
        }
      }
    }
    PPO_LOOP
    for (int j = J4; j < J; ++j) {
      const ppo_f4 wv = ppo_ld4(wc + j * ldw);
      for (int i = 0; i < 4; ++i) {
        const float dq = dr[i * ldd + j];
        acc[i][0] = fmaf(dq, wv.x, acc[i][0]); acc[i][1] = fmaf(dq, wv.y, acc[i][1]);
        acc[i][2] = fmaf(dq, wv.z, acc[i][2]); acc[i][3] = fmaf(dq, wv.w, acc[i][3]);
      }
    }
    for (int i = 0; i < 4; ++i) {
      const size_t row = (size_t)(4 * tn + i);
      const ppo_f4 hv = ppo_ld4(h + row * ldhh + 4 * tk);
      ppo_f4 o;
      o.x = acc[i][0] * (1.0f - hv.x * hv.x); o.y = acc[i][1] * (1.0f - hv.y * hv.y);
      o.z = acc[i][2] * (1.0f - hv.z * hv.z); o.w = acc[i][3] * (1.0f - hv.w * hv.w);
      float* op = out + row * ldout + 4 * tk;
      if (4 * tk + 3 < K) {
        ppo_st4(op, o);
      } else {                                             // ragged last tile: only the valid columns
        const float ov[4] = {o.x, o.y, o.z, o.w};
        for (int c = 0; c < 4; ++c)
          if (4 * tk + c < K) op[c] = ov[c];
      }
    }
  }
}

struct AdamCoef {
  float b1, b2, eps, step_size, bc2s;
};

// torch.optim.Adam, _single_tensor_adam (no amsgrad / weight decay / maximize): t = step count AFTER the increment
PPO_FN AdamCoef adam_coef(float lr, float b1, float b2, float eps, int t) {
  AdamCoef c;
  const float bc1 = 1.0f - powf(b1, (float)t), bc2 = 1.0f - powf(b2, (float)t);
  c.b1 = b1; c.b2 = b2; c.eps = eps;
  c.step_size = lr / bc1;
  c.bc2s = sqrtf(bc2);
  return c;
}

// The three updates are written as explicit fmaf, the same at every Adam site (adam_elem, wgrad_adam_tile): left to
// contraction, nvcc fused `p - step_size * q` into one FFMA in wgrad_adam_tile but rounded step_size * q first in the
// data-parallel reduce, so the W = 1 data-parallel kernel drifted from the single-process one by that rounding every step.
PPO_FN float adam_m(float m, float g, const AdamCoef& c) { return fmaf(1.0f - c.b1, g - m, m); }          // exp_avg.lerp_
PPO_FN float adam_v(float v, float g, const AdamCoef& c) { return fmaf((1.0f - c.b2) * g, g, c.b2 * v); } // .addcmul_
PPO_FN float adam_p(float p, float m, float v, const AdamCoef& c) {
  const float denom = sqrtf(v) / c.bc2s + c.eps;
  return fmaf(-c.step_size, m / denom, p);
}

PPO_FN float adam_elem(float p, float g, float* m, float* v, int idx, const AdamCoef& c) {
  const float mi = adam_m(m[idx], g, c), vi = adam_v(v[idx], g, c);
  m[idx] = mi;
  v[idx] = vi;
  return adam_p(p, mi, vi, c);
}

// Number of 4 x 4 tiles of a [J][K] weight
PPO_FN int wgrad_tiles(int J, int K) { return ((J + 3) / 4) * ((K + 3) / 4); }

// tile `t` of: g[j][k] = sum_n d[n][j] * in[n][k], then Adam on element j*K + k of the tensor at arena offset `off`
// (shared-memory copy W[j*ldw + k]; moments m / v [off + j*K + k]).  tile = rows 4tj..4tj+3 x columns 4tk..4tk+3 of the
// weight: one 128-bit load of d and one of `in` per sample (rows 16-byte aligned; ldd = 1, the value head, takes scalars)
// DP (data-parallel kernel): the same sums are stored to gout[off + j*K + k] (this rank's exchange slot) instead, and Adam
// runs after the exchange (ph_dp_reduce_adam)
template <bool DP = false>
PPO_FN void wgrad_adam_tile(int t, const float* d, int ldd, const float* in, int ldin, float* W, int ldw, int M, int J, int K,
                            float* m, float* v, int off, const AdamCoef& ac, float* gout = nullptr) {
  const int tkn = (K + 3) / 4;
  const int tj = t / tkn, tk = t - tj * tkn;
  float acc[4][4];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) acc[r][c] = 0.0f;
  if ((ldd & 3) == 0) {
    PPO_LOOP
    for (int n = 0; n < M; ++n) {
      const ppo_f4 dv = ppo_ld4(d + (size_t)n * ldd + 4 * tj), xv = ppo_ld4(in + (size_t)n * ldin + 4 * tk);
      const float dq[4] = {dv.x, dv.y, dv.z, dv.w};
      for (int r = 0; r < 4; ++r) {
        acc[r][0] = fmaf(dq[r], xv.x, acc[r][0]); acc[r][1] = fmaf(dq[r], xv.y, acc[r][1]);
        acc[r][2] = fmaf(dq[r], xv.z, acc[r][2]); acc[r][3] = fmaf(dq[r], xv.w, acc[r][3]);
      }
    }
  } else {
    PPO_LOOP
    for (int n = 0; n < M; ++n) {
      const ppo_f4 xv = ppo_ld4(in + (size_t)n * ldin + 4 * tk);
      for (int r = 0; r < 4; ++r) {
        const float dq = 4 * tj + r < J ? d[(size_t)n * ldd + 4 * tj + r] : 0.0f;
        acc[r][0] = fmaf(dq, xv.x, acc[r][0]); acc[r][1] = fmaf(dq, xv.y, acc[r][1]);
        acc[r][2] = fmaf(dq, xv.z, acc[r][2]); acc[r][3] = fmaf(dq, xv.w, acc[r][3]);
      }
    }
  }
  if constexpr (DP) {
    for (int r = 0; r < 4; ++r) {
      const int e = off + (4 * tj + r) * K + 4 * tk;
      if (4 * tj + r < J && (K & 3) == 0) {
        ppo_f4 g;
        g.x = acc[r][0]; g.y = acc[r][1]; g.z = acc[r][2]; g.w = acc[r][3]; ppo_st4(gout + e, g);
      } else if (4 * tj + r < J) {
        for (int c = 0; c < 4; ++c)
          if (4 * tk + c < K) gout[e + c] = acc[r][c];
      }
    }
    return;
  }
  // Adam.  The master copy `flat` is written once, when the kernel ends (ph_finish); the moments live in L2.  All moment
  // loads are issued before the arithmetic (independent round trips); rows of a weight whose K is a multiple of 4 are read
  // and written 128 bits at a time -- a warp then touches whole 32-byte sectors (the scalar form's 16-byte-strided stores
  // kept the load/store unit busy long into the NEXT phase)
  float mo[4][4], vo[4][4];
  const bool vec = (K & 3) == 0;
  for (int r = 0; r < 4; ++r) {
    const int j = 4 * tj + r < J ? 4 * tj + r : J - 1;
    if (vec) {
      const ppo_f4 mv = ppo_ld4(m + off + j * K + 4 * tk), vv = ppo_ld4(v + off + j * K + 4 * tk);
      mo[r][0] = mv.x; mo[r][1] = mv.y; mo[r][2] = mv.z; mo[r][3] = mv.w;
      vo[r][0] = vv.x; vo[r][1] = vv.y; vo[r][2] = vv.z; vo[r][3] = vv.w;
    } else {
      for (int c = 0; c < 4; ++c) {
        const int e = off + j * K + (4 * tk + c < K ? 4 * tk + c : K - 1);
        mo[r][c] = m[e];
        vo[r][c] = v[e];
      }
    }
  }
  for (int r = 0; r < 4; ++r) {
    if (4 * tj + r >= J) continue;
    float* wp = W + (4 * tj + r) * ldw + 4 * tk;
    float wn[4], mn[4], vn[4];
    for (int c = 0; c < 4; ++c) {
      const float g = acc[r][c];
      mn[c] = adam_m(mo[r][c], g, ac);
      vn[c] = adam_v(vo[r][c], g, ac);
      wn[c] = adam_p(4 * tk + c < K ? wp[c] : 0.0f, mn[c], vn[c], ac);
    }
    const int e = off + (4 * tj + r) * K + 4 * tk;
    if (vec) {
      ppo_f4 t;
      t.x = mn[0]; t.y = mn[1]; t.z = mn[2]; t.w = mn[3]; ppo_st4(m + e, t);
      t.x = vn[0]; t.y = vn[1]; t.z = vn[2]; t.w = vn[3]; ppo_st4(v + e, t);
      t.x = wn[0]; t.y = wn[1]; t.z = wn[2]; t.w = wn[3]; ppo_st4(wp, t);
    } else {
      for (int c = 0; c < 4; ++c)
        if (4 * tk + c < K) {
          m[e + c] = mn[c];
          v[e + c] = vn[c];
          wp[c] = wn[c];
        }
    }
  }
}

// element j of: g[j] = sum_n d[n][j], then Adam (bias vectors, the std parameter); DP: g stored to gout[off + j] instead
template <bool DP = false>
PPO_FN void bias_adam_elem(int j, const float* d, int ldd, float* Bv, int M, float* m, float* v, int off, const AdamCoef& ac,
                           float* gout = nullptr) {
  float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
  int n = 0;
  for (; n + 3 < M; n += 4) {
    s0 += d[(size_t)n * ldd + j]; s1 += d[(size_t)(n + 1) * ldd + j];
    s2 += d[(size_t)(n + 2) * ldd + j]; s3 += d[(size_t)(n + 3) * ldd + j];
  }
  for (; n < M; ++n) s0 += d[(size_t)n * ldd + j];
  if constexpr (DP) gout[off + j] = (s0 + s1) + (s2 + s3);
  else Bv[j] = adam_elem(Bv[j], (s0 + s1) + (s2 + s3), m, v, off + j, ac);
}

// all parameter gradients + Adam of one three-layer network, spread over the block as ONE index space:
//   [W2 tiles | W1 tiles | W3 tiles | b1 | b2 | b3 | extra (std)]
// d1 / d2 / d3: pre-activation gradients of the three layers; x / h1 / h2: their inputs.  DP: gradients only, into gout
template <bool DP = false>
PPO_FN void net_wgrad_adam(const float* x, int ldx, const float* h1, const float* h2, int ldh, const float* d1, const float* d2,
                           const float* d3, int ld3, int M, int D, int H1, int H2, int O, float* w1, int ld1, float* b1,
                           float* w2, float* b2, float* w3, float* b3, float* extra, const float* dextra, float* m, float* v,
                           const int* off, const AdamCoef& ac, int tid, int NT, float* gout = nullptr) {
  const int t2 = wgrad_tiles(H2, H1), t1 = wgrad_tiles(H1, D), t3 = wgrad_tiles(O, H2);
  const int nt = t2 + t1 + t3, nb = H1 + H2 + O + (extra ? O : 0);
  PPO_LOOP
  for (int t = tid; t < nt + nb; t += NT) {
    if (t < nt) {                                          // a 4 x 4 tile of one of the three weights: ONE copy of the tile code
      const float *d, *in;
      float* W;
      int u = t, ldd, ldin, ldw, J, K, o;
      if (u < t2) { d = d2; ldd = ldh; in = h1; ldin = ldh; W = w2; ldw = ldh; J = H2; K = H1; o = off[2]; }
      else if (u < t2 + t1) { u -= t2; d = d1; ldd = ldh; in = x; ldin = ldx; W = w1; ldw = ld1; J = H1; K = D; o = off[0]; }
      else { u -= t2 + t1; d = d3; ldd = ld3; in = h2; ldin = ldh; W = w3; ldw = ldh; J = O; K = H2; o = off[4]; }
      wgrad_adam_tile<DP>(u, d, ldd, in, ldin, W, ldw, M, J, K, m, v, o, ac, gout);
    } else {                                               // an element of a bias vector / the std parameter
      const float* d;
      float* Bv;
      int u = t - nt, ldd, o;
      if (u < H1) { d = d1; ldd = ldh; Bv = b1; o = off[1]; }
      else if (u < H1 + H2) { u -= H1; d = d2; ldd = ldh; Bv = b2; o = off[3]; }
      else if (u < H1 + H2 + O) { u -= H1 + H2; d = d3; ldd = ld3; Bv = b3; o = off[5]; }
      else { u -= H1 + H2 + O; d = dextra; ldd = ld3; Bv = extra; o = off[6]; }
      bias_adam_elem<DP>(u, d, ldd, Bv, M, m, v, o, ac, gout);
    }
  }
}

PPO_FN float ppo_softplus(float x) { return x > 20.0f ? x : log1pf(expf(x)); }      // F.softplus (beta 1, threshold 20)

// ------------------------------------------------------------------------------------------------ phases
PPO_FN void copy_rows_in(float* dst, int ld, const float* src, int rows, int cols, int tid, int NT) {
  for (int e = tid; e < rows * cols; e += NT) {
    const int j = e / cols, k = e - j * cols;
    dst[j * ld + k] = src[e];
  }
}

PPO_FN void ph_load_weights(PpoShared& S, const PpoArgs& a, int tid, int NT) {
  copy_rows_in(S.aw1, S.ld1, a.a_flat + a.a_off[0], a.H1, a.D, tid, NT);
  copy_rows_in(S.ab1, a.H1, a.a_flat + a.a_off[1], 1, a.H1, tid, NT);
  copy_rows_in(S.aw2, S.ldh, a.a_flat + a.a_off[2], a.H2, a.H1, tid, NT);
  copy_rows_in(S.ab2, a.H2, a.a_flat + a.a_off[3], 1, a.H2, tid, NT);
  copy_rows_in(S.aw3, S.ldh, a.a_flat + a.a_off[4], a.A, a.H2, tid, NT);
  copy_rows_in(S.ab3, a.A, a.a_flat + a.a_off[5], 1, a.A, tid, NT);
  copy_rows_in(S.sdp, a.A, a.a_flat + a.a_off[6], 1, a.A, tid, NT);
  copy_rows_in(S.cw1, S.ld1, a.c_flat + a.c_off[0], a.H1, a.D, tid, NT);
  copy_rows_in(S.cb1, a.H1, a.c_flat + a.c_off[1], 1, a.H1, tid, NT);
  copy_rows_in(S.cw2, S.ldh, a.c_flat + a.c_off[2], a.H2, a.H1, tid, NT);
  copy_rows_in(S.cb2, a.H2, a.c_flat + a.c_off[3], 1, a.H2, tid, NT);
  copy_rows_in(S.cw3, S.ldh, a.c_flat + a.c_off[4], 1, a.H2, tid, NT);
  copy_rows_in(S.cb3, 1, a.c_flat + a.c_off[5], 1, 1, tid, NT);
  if (tid == 0) {
    S.steps[0] = (int)*a.a_step;
    S.steps[1] = (int)*a.c_step;
    for (int i = 0; i < 8; ++i) S.flag[i] = 0.0f;
  }
}

// minibatch b -> buffer b & 1, by the threads [t0, NT) of the block (the idle half during the dense phases)
PPO_FN void ph_load_batch(PpoShared& S, const PpoArgs& a, int b, int tid, int NT, int t0) {
  if (b >= a.n_batches || tid < t0) return;
  const int s = b & 1, id = tid - t0, n_id = NT - t0;
  const int64_t* rows = a.perm + (int64_t)b * a.mb;
  for (int e = id; e < a.mb * a.D; e += n_id) {
    const int n = e / a.D, k = e - n * a.D;
    (S.xb + s * S.x_stride)[n * S.ld1 + k] = a.state[rows[n] * a.D + k];
  }
  for (int e = id; e < a.mb * a.A; e += n_id) {
    const int n = e / a.A, k = e - n * a.A;
    (S.actb + s * S.act_stride)[e] = a.action[rows[n] * a.A + k];
  }
  for (int n = id; n < a.mb; n += n_id) {
    (S.oldlpb + s * S.row_stride)[n] = a.old_logp[rows[n]];
    (S.advb + s * S.row_stride)[n] = a.adv[rows[n]];
    (S.retb + s * S.row_stride)[n] = a.ret[rows[n]];
  }
}

PPO_FN float sum_strided4(const float* p, int n) {       // fixed order, four independent chains
  float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
  int i = 0;
  for (; i + 3 < n; i += 4) { s0 += p[i]; s1 += p[i + 1]; s2 += p[i + 2]; s3 += p[i + 3]; }
  for (; i < n; ++i) s0 += p[i];
  return (s0 + s1) + (s2 + s3);
}

// ---- the two networks side by side: threads [0, NT/2) run the actor, [NT/2, NT) the critic
// P1: first layers (+ std = softplus(std_param), network_heads.py:205)
PPO_FN void ph1_fwd1(PpoShared& S, const PpoArgs& a, int b, int tid, int NT) {
  const int h = NT / 2, s = b & 1;
  if (tid < h) {
    dense_fwd((S.xb + s * S.x_stride), S.ld1, S.aw1, S.ld1, S.ab1, S.ah1, S.ldh, a.mb, a.D, a.H1, true, tid, h);
    for (int j = tid; j < a.A; j += h) {
      const float sd = ppo_softplus(S.sdp[j]);
      S.sdv[j] = sd;
      S.lsd[j] = logf(sd);
    }
  } else {
    dense_fwd((S.xb + s * S.x_stride), S.ld1, S.cw1, S.ld1, S.cb1, S.ch1, S.ldh, a.mb, a.D, a.H1, true, tid - h, h);
  }
}
// P2: second layers
PPO_FN void ph2_fwd2(PpoShared& S, const PpoArgs& a, int b, int tid, int NT) {
  const int h = NT / 2;
  if (tid < h) dense_fwd(S.ah1, S.ldh, S.aw2, S.ldh, S.ab2, S.ah2, S.ldh, a.mb, a.H1, a.H2, true, tid, h);
  else dense_fwd(S.ch1, S.ldh, S.cw2, S.ldh, S.cb2, S.ch2, S.ldh, a.mb, a.H1, a.H2, true, tid - h, h);
}
// P3: heads.  actor: mean = tanh(fc_action(.)); critic: v, value-loss terms, d value_loss / d v (PPO_agent.py:86) and the step
// count of its (unconditional) update
PPO_FN void ph3_heads(PpoShared& S, const PpoArgs& a, int b, int tid, int NT) {
  const int h = NT / 2, s = b & 1;
  if (tid < h) {
    dense_fwd(S.ah2, S.ldh, S.aw3, S.ldh, S.ab3, S.mu, S.lda, a.mb, a.H2, a.A, true, tid, h);
    return;
  }
  const float invM = 1.0f / (float)a.mb;
  for (int n = tid - h; n < a.mb; n += h) {
    float acc = 0.0f;
    for (int k = 0; k < a.H2; ++k) acc = fmaf(S.ch2[n * S.ldh + k], S.cw3[k], acc);
    const float v = acc + S.cb3[0];
    S.v[n] = v;
    const float e = (S.retb + s * S.row_stride)[n] - v;
    S.dv[n] = -e * invM;
    S.red[2 * a.mb + n] = e * e;
  }
  if (tid == NT - 1) S.steps[1] += 1;
}
// P4: actor: per sample log pi(a|s), ratio, clipped surrogate and its gradient (PPO_agent.py:79-84, 88);
//     critic: back through its head into layer 2
PPO_FN void ph4_loss(PpoShared& S, const PpoArgs& a, int b, int tid, int NT) {
  const int h = NT / 2, s = b & 1, A = a.A;
  if (tid >= h) {
    dense_bwd_data(S.dv, 1, S.cw3, S.ldh, S.ch2, S.ldh, S.cd2, S.ldh, a.mb, 1, a.H2, tid - h, h);
    if (tid == NT - 1) S.flag[4] = 0.5f * (sum_strided4(S.red + 2 * a.mb, a.mb) / (float)a.mb);
    return;
  }
  const float invM = 1.0f / (float)a.mb;
  for (int n = tid; n < a.mb; n += h) {
    float lp = 0.0f;
    for (int j = 0; j < A; ++j) {
      const float sd = S.sdv[j], t = (S.actb + s * S.act_stride)[n * A + j] - S.mu[n * S.lda + j];
      lp += -(t * t) / (2.0f * sd * sd) - S.lsd[j] - 0.91893853320467274178f;       // Normal.log_prob
    }
    S.logp[n] = lp;
    const float old = (S.oldlpb + s * S.row_stride)[n], adv = (S.advb + s * S.row_stride)[n];
    const float ratio = expf(lp - old);
    const float obj = ratio * adv;
    const float rc = fminf(fmaxf(ratio, 1.0f - a.clip), 1.0f + a.clip);
    const float objc = rc * adv;
    const bool inside = ratio >= 1.0f - a.clip && ratio <= 1.0f + a.clip;
    float g;                                               // d min(obj, objc) / d log pi (torch.min splits ties evenly)
    if (obj < objc) g = adv * ratio;
    else if (obj > objc) g = inside ? adv * ratio : 0.0f;
    else g = 0.5f * adv * ratio + (inside ? 0.5f * adv * ratio : 0.0f);
    S.dlogp[n] = -g * invM;
    S.red[n] = fminf(obj, objc);
    S.red[a.mb + n] = old - lp;
  }
}
// P5: actor: the reference's `if approx_kl <= 1.5 * target_kl` (PPO_agent.py:94), decided once for the block;
//     critic: back into layer 1.
//     DP: the gate is decided on the MEAN kl over ranks, after the exchange (ph_dp_wait); here this rank's kl and policy loss
//     are only recorded and the actor backward is switched on unconditionally (its gradient goes into the exchange slot)
template <bool DP = false>
PPO_FN void ph5_gate(PpoShared& S, const PpoArgs& a, int b, int tid, int NT) {
  const int h = NT / 2;
  if (tid >= h) {
    dense_bwd_data(S.cd2, S.ldh, S.cw2, S.ldh, S.ch1, S.ldh, S.cd1, S.ldh, a.mb, a.H2, a.H1, tid - h, h);
    return;
  }
  if (tid != 0) return;
  const float invM = 1.0f / (float)a.mb;
  const float kl = sum_strided4(S.red + a.mb, a.mb) * invM;
  float ent = 0.0f;
  for (int j = 0; j < a.A; ++j) ent += 0.5f + 0.91893853320467274178f + S.lsd[j];    // Normal.entropy, summed over actions
  if constexpr (DP) {
    S.flag[0] = 1.0f;
    S.flag[2] = -(sum_strided4(S.red, a.mb) * invM) - a.ent_w * ent;
    S.flag[3] = kl;
    return;
  }
  const bool gate = kl <= a.gate_max;
  S.flag[0] = gate ? 1.0f : 0.0f;
  S.flag[2] = -(sum_strided4(S.red, a.mb) * invM) - a.ent_w * ent;
  S.flag[3] = kl;
  if (gate) {
    S.steps[0] += 1;
    S.flag[1] += 1.0f;
  }
}
// P6: actor (if the gate is open): gradients at the policy head -- d / d pre-tanh mean, d / d std_param (through softplus);
//     the critic half fetches the rows of the NEXT minibatch into the other buffer
PPO_FN void ph6_head_bwd(PpoShared& S, const PpoArgs& a, int b, int tid, int NT) {
  const int h = NT / 2, s = b & 1, A = a.A;
  if (tid >= h) {
    ph_load_batch(S, a, b + 1, tid, NT, h);
    return;
  }
  if (S.flag[0] == 0.0f) return;
  const float dent = -a.ent_w / (float)a.mb;             // d(-w * mean(entropy)) / d entropy_n
  for (int e = tid; e < a.mb * A; e += h) {
    const int n = e / A, j = e - n * A;
    const float m_ = S.mu[n * S.lda + j], sd = S.sdv[j], t = (S.actb + s * S.act_stride)[e] - m_, gl = S.dlogp[n];
    S.dmu[n * S.lda + j] = gl * (t / (sd * sd)) * (1.0f - m_ * m_);
    const float p = S.sdp[j];
    const float sig = p > 20.0f ? 1.0f : 1.0f / (1.0f + expf(-p));                  // softplus'
    S.dsd[n * S.lda + j] = (gl * ((t * t) / (sd * sd * sd) - 1.0f / sd) + dent * (1.0f / sd)) * sig;
  }
}
// P7: actor (gate): back into layer 2; critic: all its parameter gradients + Adam (PPO_agent.py:97-99)
//     (DP: the critic's gradients into its part of the exchange slot, `gout`)
template <bool DP = false>
PPO_FN void ph7_critic_update(PpoShared& S, const PpoArgs& a, int b, int tid, int NT, float* gout = nullptr) {
  const int h = NT / 2;
  if (tid < h) {
    if (S.flag[0] != 0.0f) dense_bwd_data(S.dmu, S.lda, S.aw3, S.ldh, S.ah2, S.ldh, S.ad2, S.ldh, a.mb, a.A, a.H2, tid, h);
    return;
  }
  const AdamCoef ac = DP ? AdamCoef{} : adam_coef(a.c_lr, a.c_b1, a.c_b2, a.c_eps, S.steps[1]);
  net_wgrad_adam<DP>((S.xb + (b & 1) * S.x_stride), S.ld1, S.ch1, S.ch2, S.ldh, S.cd1, S.cd2, S.dv, 1, a.mb, a.D, a.H1, a.H2, 1, S.cw1, S.ld1, S.cb1,
                     S.cw2, S.cb2, S.cw3, S.cb3, nullptr, nullptr, a.c_m, a.c_v, a.c_off, ac, tid - h, h, gout);
}
// P8: actor (gate): back into layer 1
PPO_FN void ph8_actor_bwd1(PpoShared& S, const PpoArgs& a, int b, int tid, int NT) {
  if (S.flag[0] == 0.0f) return;
  dense_bwd_data(S.ad2, S.ldh, S.aw2, S.ldh, S.ah1, S.ldh, S.ad1, S.ldh, a.mb, a.H2, a.H1, tid, NT);
}
// P9: actor (gate): all its parameter gradients + Adam (PPO_agent.py:94-96), the whole block
//     (DP: the actor's gradients into the start of the exchange slot `gout`, and this rank's loss / kl values after them)
template <bool DP = false>
PPO_FN void ph9_actor_update(PpoShared& S, const PpoArgs& a, int b, int tid, int NT, float* gout = nullptr, int stat_at = 0) {
  if (S.flag[0] == 0.0f) return;
  const AdamCoef ac = DP ? AdamCoef{} : adam_coef(a.a_lr, a.a_b1, a.a_b2, a.a_eps, S.steps[0]);
  net_wgrad_adam<DP>((S.xb + (b & 1) * S.x_stride), S.ld1, S.ah1, S.ah2, S.ldh, S.ad1, S.ad2, S.dmu, S.lda, a.mb, a.D, a.H1, a.H2, a.A, S.aw1, S.ld1,
                     S.ab1, S.aw2, S.ab2, S.aw3, S.ab3, S.sdp, S.dsd, a.a_m, a.a_v, a.a_off, ac, tid, NT, gout);
  if constexpr (DP) {
    if (tid == NT - 1) {
      gout[stat_at + 0] = S.flag[2];
      gout[stat_at + 1] = S.flag[3];
      gout[stat_at + 2] = S.flag[4];
    }
  }
}

PPO_FN void copy_rows_out(float* dst, const float* src, int ld, int rows, int cols, int tid, int NT) {
  for (int e = tid; e < rows * cols; e += NT) {
    const int j = e / cols, k = e - j * cols;
    dst[e] = src[j * ld + k];
  }
}

// the master copies of the parameters (the optimizers' arenas), the step counts and the statistics of the last minibatch
PPO_FN void ph_finish(PpoShared& S, const PpoArgs& a, int tid, int NT) {
  copy_rows_out(a.a_flat + a.a_off[0], S.aw1, S.ld1, a.H1, a.D, tid, NT);
  copy_rows_out(a.a_flat + a.a_off[1], S.ab1, a.H1, 1, a.H1, tid, NT);
  copy_rows_out(a.a_flat + a.a_off[2], S.aw2, S.ldh, a.H2, a.H1, tid, NT);
  copy_rows_out(a.a_flat + a.a_off[3], S.ab2, a.H2, 1, a.H2, tid, NT);
  copy_rows_out(a.a_flat + a.a_off[4], S.aw3, S.ldh, a.A, a.H2, tid, NT);
  copy_rows_out(a.a_flat + a.a_off[5], S.ab3, a.A, 1, a.A, tid, NT);
  copy_rows_out(a.a_flat + a.a_off[6], S.sdp, a.A, 1, a.A, tid, NT);
  copy_rows_out(a.c_flat + a.c_off[0], S.cw1, S.ld1, a.H1, a.D, tid, NT);
  copy_rows_out(a.c_flat + a.c_off[1], S.cb1, a.H1, 1, a.H1, tid, NT);
  copy_rows_out(a.c_flat + a.c_off[2], S.cw2, S.ldh, a.H2, a.H1, tid, NT);
  copy_rows_out(a.c_flat + a.c_off[3], S.cb2, a.H2, 1, a.H2, tid, NT);
  copy_rows_out(a.c_flat + a.c_off[4], S.cw3, S.ldh, 1, a.H2, tid, NT);
  copy_rows_out(a.c_flat + a.c_off[5], S.cb3, 1, 1, 1, tid, NT);
  if (tid != 0) return;
  *a.a_step = (int64_t)S.steps[0];
  *a.c_step = (int64_t)S.steps[1];
  a.stats[0] = S.flag[2];
  a.stats[1] = S.flag[4];
  a.stats[2] = S.flag[3];
  a.stats[3] = S.flag[1];
}

// ------------------------------------------------------------------------------------------------ data parallel (ppo_dp_sequence.inc)
// W ranks, each with its own rollout rows and minibatch permutation; update b of every rank is ONE step of PPO_agent.py:68-99
// on the union of the ranks' b-th minibatches.  Every loss term is a mean over rows, so the union's gradients / losses / kl are
// the means over ranks of the per-rank values: each rank publishes its gradients and loss values in an exchange slot, waits for
// every peer's, sums them over ranks 0..W-1 in that order, scales by 1/W (exact for W = 1) and applies the same Adam
// arithmetic -- parameters, moments and step counts stay bit-identical on every rank.
//
// Exchange region of one rank (allocated by that rank, mapped into every peer):
//   int64 flag[8] (128-byte header) | slot 0 | slot 1          slot = [actor gradients | critic gradients | policy loss, kl, value loss]
// flag[p] of rank r's region = the last update rank p has published (written by rank p: flags are pushed, each rank polls
// only its own region).  Update b of a launch has the global sequence number seq = seq_base + b + 1 (monotonic across launches,
// never reset) and uses slot seq & 1.
constexpr int PPO_DP_MAX_WORLD = 8;
constexpr int PPO_DP_HEADER_FLOATS = 32;

struct PpoDp {
  float* region[PPO_DP_MAX_WORLD];   // exchange region of rank p, as seen from this rank
  int world, rank;
  int slot_floats, c_base, stat_at;  // floats per slot; slot offsets of the critic gradients and of the three loss values
  long long seq_base;                // updates exchanged before this launch
  long long timeout_ns;              // bound on the wait for one update's peers (%globaltimer)
  long long* status;                 // 0, or after a timeout 1 + peer + 16 * update (update index within the launch)
};

PPO_HD int ppo_dp_slot_floats(int a_n, int c_n, int* c_base, int* stat_at) {
  const int cb = (a_n + 3) / 4 * 4, sa = cb + (c_n + 3) / 4 * 4;
  if (c_base) *c_base = cb;
  if (stat_at) *stat_at = sa;
  return sa + 4;
}
PPO_HD long long* dp_flags(float* region) { return reinterpret_cast<long long*>(region); }
PPO_HD float* dp_slot(float* region, long long seq, int slot_floats) {
  return region + PPO_DP_HEADER_FLOATS + (int)(seq & 1) * slot_floats;
}

#ifdef __CUDACC__
PPO_FN void ppo_fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
PPO_FN void ppo_st_release_sys(long long* p, long long v) {
  asm volatile("st.release.sys.global.b64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
PPO_FN long long ppo_ld_acquire_sys(const long long* p) {
  long long v;
  asm volatile("ld.acquire.sys.global.b64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
PPO_FN float ppo_ld_peer(const float* p) { return __ldcg(p); }      // L2 / NVLink, never a (possibly stale) L1 line
PPO_FN unsigned long long ppo_now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
PPO_FN void ppo_backoff(unsigned ns) { __nanosleep(ns); }
#else
PPO_FN void ppo_fence_sys() { __atomic_thread_fence(__ATOMIC_ACQ_REL); }
PPO_FN void ppo_st_release_sys(long long* p, long long v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
PPO_FN long long ppo_ld_acquire_sys(const long long* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
PPO_FN float ppo_ld_peer(const float* p) { return *p; }
PPO_FN unsigned long long ppo_now_ns() {
  return (unsigned long long)std::chrono::duration_cast<std::chrono::nanoseconds>(
      std::chrono::steady_clock::now().time_since_epoch()).count();
}
PPO_FN void ppo_backoff(unsigned) {}
#endif

// Publish update b: this rank's slot was written in P7 / P9 and the block barrier after P9 orders those writes before this
// phase; thread 0 makes them visible at system scope and pushes seq into flag[rank] of every rank's region (release).
PPO_FN void ph_dp_publish(const PpoDp& d, int b, int tid) {
  if (tid != 0) return;
  const long long seq = d.seq_base + b + 1;
  ppo_fence_sys();
  for (int p = 0; p < d.world; ++p) ppo_st_release_sys(dp_flags(d.region[p]) + d.rank, seq);
}

// Wait for update b of every peer (thread 0, acquire loads of this rank's own flags, bounded by d.timeout_ns), then decide
// the KL gate on the MEAN kl over ranks (PPO_agent.py:94 on the union minibatch) and keep the mean losses as the statistics.
// On a timeout: status word, S.flag[6] = 1, and the sequence skips the remaining updates.
//
// Slot reuse: update b writes slot seq & 1, which update seq - 2 used.  This rank got here for seq - 1 only after it saw every
// peer's flag for seq - 1, and a peer publishes seq - 1 only after its reduce of seq - 2 (the last read of that slot) has
// finished: nobody still reads the slot this rank overwrites.  The barrier after this phase orders every thread's slot reads
// (ld.global.cg, which bypasses L1: a slot is reused, so an L1 line could be stale) after the acquire.
PPO_FN void ph_dp_wait(PpoShared& S, const PpoArgs& a, const PpoDp& d, int b, int tid) {
  if (tid != 0) return;
  const long long seq = d.seq_base + b + 1;
  const long long* fl = dp_flags(d.region[d.rank]);
  const unsigned long long t0 = ppo_now_ns();
  for (int p = 0; p < d.world; ++p) {
    unsigned ns = 32;
    while (ppo_ld_acquire_sys(fl + p) < seq) {
      if ((long long)(ppo_now_ns() - t0) > d.timeout_ns) {
        *d.status = 1 + p + 16LL * b;
        S.flag[6] = 1.0f;
        return;
      }
      ppo_backoff(ns);
      if (ns < 1024) ns *= 2;
    }
  }
  float v[3];
  for (int i = 0; i < 3; ++i) {
    v[i] = ppo_ld_peer(dp_slot(d.region[0], seq, d.slot_floats) + d.stat_at + i);
    for (int p = 1; p < d.world; ++p) v[i] += ppo_ld_peer(dp_slot(d.region[p], seq, d.slot_floats) + d.stat_at + i);
    v[i] *= 1.0f / (float)d.world;
  }
  const bool gate = v[1] <= a.gate_max;
  S.flag[0] = gate ? 1.0f : 0.0f;
  S.flag[2] = v[0];
  S.flag[3] = v[1];
  S.flag[4] = v[2];
  if (gate) {
    S.steps[0] += 1;
    S.flag[1] += 1.0f;
  }
}

// element e of the index space [critic tensors | actor tensors] (no arena padding): its shared-memory copy and arena offset
PPO_FN float* dp_param(PpoShared& S, const PpoArgs& a, int e, int nc, bool& actor, int& off) {
  actor = e >= nc;
  int u = actor ? e - nc : e;
#define PPO_DP_T(ptr, rows, cols, ld, o)                       \
  if (u < (rows) * (cols)) {                                   \
    const int j = u / (cols);                                  \
    off = (o) + u;                                             \
    return (ptr) + j * (ld) + (u - j * (cols));                \
  }                                                            \
  u -= (rows) * (cols);
  if (!actor) {
    PPO_DP_T(S.cw1, a.H1, a.D, S.ld1, a.c_off[0]) PPO_DP_T(S.cb1, 1, a.H1, 0, a.c_off[1])
    PPO_DP_T(S.cw2, a.H2, a.H1, S.ldh, a.c_off[2]) PPO_DP_T(S.cb2, 1, a.H2, 0, a.c_off[3])
    PPO_DP_T(S.cw3, 1, a.H2, 0, a.c_off[4])
    off = a.c_off[5];
    return S.cb3;
  }
  PPO_DP_T(S.aw1, a.H1, a.D, S.ld1, a.a_off[0]) PPO_DP_T(S.ab1, 1, a.H1, 0, a.a_off[1])
  PPO_DP_T(S.aw2, a.H2, a.H1, S.ldh, a.a_off[2]) PPO_DP_T(S.ab2, 1, a.H2, 0, a.a_off[3])
  PPO_DP_T(S.aw3, a.A, a.H2, S.ldh, a.a_off[4]) PPO_DP_T(S.ab3, 1, a.A, 0, a.a_off[5])
  off = a.a_off[6] + u;
  return S.sdp + u;
#undef PPO_DP_T
}

// Reduce + Adam: every element's gradient summed over ranks 0..W-1 in order, times 1/W, then adam_elem (the arithmetic of
// wgrad_adam_tile / bias_adam_elem).  Critic always (PPO_agent.py:97-99); actor iff the mean-kl gate is open (:94-96).
PPO_FN void ph_dp_reduce_adam(PpoShared& S, const PpoArgs& a, const PpoDp& d, int b, int tid, int NT) {
  const long long seq = d.seq_base + b + 1;
  const int nc = a.H1 * a.D + a.H1 + a.H2 * a.H1 + a.H2 + a.H2 + 1;
  const int na = a.H1 * a.D + a.H1 + a.H2 * a.H1 + a.H2 + a.A * a.H2 + 2 * a.A;
  const int n = nc + (S.flag[0] != 0.0f ? na : 0);
  const float invW = 1.0f / (float)d.world;
  const AdamCoef cc = adam_coef(a.c_lr, a.c_b1, a.c_b2, a.c_eps, S.steps[1]);
  const AdamCoef ca = adam_coef(a.a_lr, a.a_b1, a.a_b2, a.a_eps, S.steps[0]);
  PPO_LOOP
  for (int e0 = tid; e0 < n; e0 += 4 * NT) {                // four elements per thread in flight: 4 loads per peer round trip
    float* w[4];
    int so[4], off[4];
    bool act[4];
    float g[4];
    for (int q = 0; q < 4; ++q) {
      const int e = e0 + q * NT;
      so[q] = -1;
      if (e < n) {
        w[q] = dp_param(S, a, e, nc, act[q], off[q]);
        so[q] = (act[q] ? 0 : d.c_base) + off[q];
      }
    }
    const float* s0 = dp_slot(d.region[0], seq, d.slot_floats);
    for (int q = 0; q < 4; ++q) g[q] = so[q] >= 0 ? ppo_ld_peer(s0 + so[q]) : 0.0f;
    PPO_LOOP
    for (int p = 1; p < d.world; ++p) {
      const float* sp = dp_slot(d.region[p], seq, d.slot_floats);
      for (int q = 0; q < 4; ++q)
        if (so[q] >= 0) g[q] += ppo_ld_peer(sp + so[q]);
    }
    for (int q = 0; q < 4; ++q) {
      if (so[q] < 0) continue;
      *w[q] = act[q] ? adam_elem(*w[q], g[q] * invW, a.a_m, a.a_v, off[q], ca)
                     : adam_elem(*w[q], g[q] * invW, a.c_m, a.c_v, off[q], cc);
    }
  }
}

}  // namespace b2rl_ppo
