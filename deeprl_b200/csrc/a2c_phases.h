// a2c_phases.h -- the synchronous advantage actor-critic update (A2C_agent.py:22-64) and the forward of its actor step, written
// as PHASES of a single thread block: every function below takes (tid, NT) and is executed by all NT threads of the block, with a
// block barrier between consecutive phases (the update's sequence is a2c_sequence.inc).  csrc/a2c.cu runs the update as ONE
// launch of one block (weights, gradients and activations in shared memory, RMSprop moments in global memory) and the actor
// step's forward from the same functions; tests/host_emul/a2c_emul.cpp compiles the SAME functions with g++ and runs the
// threads of a phase one after another, which is how the arithmetic is checked against the oracle without a GPU.  Nothing here
// may depend on execution order inside a phase or on the number of threads: every sum runs over a fixed index range in a fixed
// order inside one thread.
//
//   networks  HEAD = CAT:   CategoricalActorCriticNet with an FCBody phi_body (SHARED trunk), DummyBody actor / critic:
//                           logits = fc_action(phi), v = fc_critic(phi)                                (network_heads.py:217-255)
//             HEAD = GAUSS: GaussianActorCriticNet with DummyBody phi, FCBody actor / critic bodies (separate trunks):
//                           mean = tanh(fc_action(actor_body(x))), v = fc_critic(critic_body(x)),
//                           std = softplus(std_param)                                                  (network_heads.py:173-214)
//             HEAD = Q:     VanillaNet on an FCBody (SHARED trunk), no critic: q = fc_head(phi)    (network_heads.py:11-21)
//             trunks: two Linear layers, each followed by GATE (tanh or ReLU)
//   update    forward of all (T + 1) N rows (row block T: the bootstrap value, A2C_agent.py:38-41); GAE (:43-53, the arithmetic of
//             gae_seq_kernel mode 0); -mean(log pi * adv) - w_ent mean(entropy) + w_v 0.5 mean((ret - v)^2) (:55-62); backward;
//             clip_grad_norm_ (:63); RMSprop on the FlatOptimizer arena (:64)
//   n-step Q  (NStepDQN_agent.py:26-67, nstep_sequence.inc) forward of the T N rollout rows, the target network on row block T
//             and its max over actions (:56-57), the return scan (:58-60), 0.5 mean((q[a] - ret)^2) (:63), backward, clip, RMSprop
//   replay Q  (DQN_agent.py:81-134, dqn_sequence.inc) HEAD = Q or DUEL (DuelingNet: q = v + (adv - mean(adv)), fc_advantage in
//             the fc_action slot, fc_value in the fc_critic slot): forward of the B sampled states (and of the B next states
//             with double_q), the target network on the next states, the TD target, delta, the PER priorities and importance
//             weights, 0.5 mean((w delta)^2), backward, clip, RMSprop
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "optim_elem.h"

#ifdef __CUDACC__
#define A2C_FN __device__ __forceinline__
#define A2C_HD __host__ __device__ inline
#define A2C_MUL(x, y) __fmul_rn(x, y)
#define A2C_ADD(x, y) __fadd_rn(x, y)
#define A2C_SUB(x, y) __fsub_rn(x, y)
#else
#define A2C_FN static inline
#define A2C_HD static inline
#define A2C_MUL(x, y) ((x) * (y))
#define A2C_ADD(x, y) ((x) + (y))
#define A2C_SUB(x, y) ((x) - (y))
#endif

namespace b2rl_a2c {

enum { CAT = 0, GAUSS = 1, Q = 2, DUEL = 3 };   // head kind
enum { TANH = 0, RELU = 1, LINEAR = 2 }; // gate of a layer
constexpr int A2C_MAX_TENSORS = 13;      // two trunks x (w1 b1 w2 b2) + fc_action w b + fc_critic w b + std
constexpr int A2C_CHUNK = 64;            // gradient elements per partial sum of the global norm

// the network's parameters: the FlatOptimizer arena and the offset of every tensor in it, in a2c_tensor order
struct A2cNet {
  float* flat;
  int off[A2C_MAX_TENSORS];
  int D, H1, H2, A;
};

struct A2cArgs {
  A2cNet net;
  const float* state;                    // rollout arena [T + 1][N][D] (rescaled states)
  const float* action;                   // [T][N][acols]: the category index as a float (CAT) or the action vector (GAUSS)
  const float* reward; const float* mask; // [T][N]
  int T, N;
  float* sq; float* ga; int64_t* step;   // RMSprop square_avg, grad_avg (centered only), step count: arena-shaped
  float lr, alpha, eps; int centered;
  float discount, tau; int use_gae;
  float ent_w, vw, max_norm;
  float* loss;                           // device scalar: the objective
};

// the n-step Q update's arguments besides A2cArgs (whose tau, use_gae, ent_w and vw it does not read)
struct NStepArgs {
  A2cArgs a;
  float* target;                         // the target network's arena: the layout of a.net.flat, the same offsets
  int sync;                              // copy the online arena into it first, and bootstrap from the online weights
};

// ------------------------------------------------------------------------------------------------ layout
// Tensor order: trunk t (t < ntr) w1 b1 w2 b2 at 4t..4t+3, then fc_action w b (Q: fc_head w b), fc_critic w b (not Q), std
// (GAUSS only).  The trunk serving the actor head is trunk 0, the critic's is trunk ntr - 1.
template <int HEAD, bool SHARED> struct A2cKind {
  static constexpr int ntr = SHARED ? 1 : 2;
  static constexpr int fa = 4 * ntr, ba = fa + 1, fc = fa + 2, bc = fa + 3, sd = fa + 4;
  static constexpr int ntensors = HEAD == Q ? 4 * ntr + 2 : 4 * ntr + 4 + (HEAD == GAUSS ? 1 : 0);
  static constexpr int critic_trunk = ntr - 1;
};

A2C_HD int a2c_odd(int n) { return n | 1; }   // odd row stride: consecutive rows of one column fall in different banks

struct TensorDesc { int rows, cols, ld, woff; };

// rows x cols of tensor i, its padded row stride and offset in the shared-memory copy (the gradient copy has the same layout)
A2C_HD TensorDesc a2c_tensor(int i, int ntr, int D, int H1, int H2, int A) {
  TensorDesc d = {0, 0, 0, 0};
  int woff = 0;
  for (int u = 0; u <= i; ++u) {
    int r, c, ld;
    if (u < 4 * ntr) {
      switch (u & 3) {
        case 0: r = H1; c = D; ld = a2c_odd(D); break;
        case 1: r = 1; c = H1; ld = H1; break;
        case 2: r = H2; c = H1; ld = a2c_odd(H1); break;
        default: r = 1; c = H2; ld = H2; break;
      }
    } else {
      switch (u - 4 * ntr) {
        case 0: r = A; c = H2; ld = a2c_odd(H2); break;
        case 1: r = 1; c = A; ld = A; break;
        case 2: r = 1; c = H2; ld = H2; break;
        case 3: r = 1; c = 1; ld = 1; break;
        default: r = 1; c = A; ld = A; break;
      }
    }
    if (u == i) { d.rows = r; d.cols = c; d.ld = ld; d.woff = woff; }
    woff += r * ld;
  }
  return d;
}

struct A2cShared {
  float* W;                              // parameters, tensor i at W + a2c_tensor(i).woff
  float* G;                              // their gradients (update only), same layout
  float* x;                              // [R][ldx] states
  float* h;                              // trunk t, layer l output at h + (2t + l) * hstride, [R][ldh]; the backward overwrites
                                         // them in place with the pre-activation gradients
  float *z, *dz;                         // [R][lda] logits (CAT) / mean (GAUSS) / q (Q); gradient w.r.t. the logits /
                                         // pre-tanh mean / q
  float *v, *dv, *adv, *ret, *logp, *ent, *lse;   // [R]
  float* red;                            // [3][M] per-row loss terms
  float* part;                           // [nchunks] sums of squares of the gradient
  float *sdv, *lsd;                      // [A] softplus(std), its log
  float* scal;                           // [4] objective, gradient norm
  int ldx, ldh, lda, hstride, R, M, nchunks;
};

// carve the shared block for R forward rows and M = T N loss rows (M = 0: actor step, no gradients); returns the floats used.
// The Q update's online forward covers only the M rollout rows (S.R = M): rows M..R-1 of h and z hold the target network's
// forward of the bootstrap states.  base may be a dummy when only the size is wanted.
template <int HEAD, bool SHARED>
A2C_HD size_t a2c_carve(A2cShared& S, float* base, int D, int H1, int H2, int A, int R, int M) {
  using K = A2cKind<HEAD, SHARED>;
  const bool upd = M > 0, critic = HEAD != Q;
  const TensorDesc last = a2c_tensor(K::ntensors - 1, K::ntr, D, H1, H2, A);
  const size_t wsize = (size_t)last.woff + (size_t)last.rows * last.ld;
  int nchunks = 0;
  for (int i = 0; i < K::ntensors; ++i) {
    const TensorDesc d = a2c_tensor(i, K::ntr, D, H1, H2, A);
    nchunks += (d.rows * d.cols + A2C_CHUNK - 1) / A2C_CHUNK;
  }
  S.ldx = a2c_odd(D);
  S.ldh = a2c_odd(H1 > H2 ? H1 : H2);
  S.lda = a2c_odd(A);
  S.hstride = R * S.ldh;
  S.R = critic || !upd ? R : M;
  S.M = M;
  S.nchunks = nchunks;
  size_t off = 0;
#define A2C_TAKE(n) (base + (off += ((size_t)(n) + 3) / 4 * 4) - ((size_t)(n) + 3) / 4 * 4)
  S.W = A2C_TAKE(wsize);
  S.G = upd ? A2C_TAKE(wsize) : nullptr;
  S.x = A2C_TAKE((size_t)S.R * S.ldx);
  S.h = A2C_TAKE((size_t)2 * K::ntr * S.hstride);
  S.z = A2C_TAKE((size_t)R * S.lda);
  S.dz = upd ? A2C_TAKE((size_t)M * S.lda) : nullptr;
  S.v = critic ? A2C_TAKE(R) : nullptr;
  S.dv = upd && critic ? A2C_TAKE(M) : nullptr;
  S.adv = upd && critic ? A2C_TAKE(M) : nullptr;
  S.ret = upd ? A2C_TAKE(M) : nullptr;
  S.logp = upd && critic ? A2C_TAKE(M) : nullptr;
  S.ent = upd && critic ? A2C_TAKE(M) : nullptr;
  S.lse = upd && critic ? A2C_TAKE(M) : nullptr;
  S.red = upd ? A2C_TAKE((size_t)(critic ? 3 : 1) * M) : nullptr;
  S.part = upd ? A2C_TAKE(nchunks) : nullptr;
  S.sdv = critic ? A2C_TAKE(A) : nullptr;
  S.lsd = critic ? A2C_TAKE(A) : nullptr;
  S.scal = A2C_TAKE(4);
#undef A2C_TAKE
  return off;
}

A2C_FN float* a2c_h(const A2cShared& S, int trunk, int layer) { return S.h + (2 * trunk + layer) * S.hstride; }

// ------------------------------------------------------------------------------------------------ dense building blocks
template <int GATE> A2C_FN float gate_f(float s) {
  if (GATE == TANH) return tanhf(s);
  if (GATE == RELU) return s > 0.0f ? s : 0.0f;
  return s;
}
// derivative of the gate from its OUTPUT h (tanh: 1 - h^2; relu: h > 0, as torch's threshold_backward on the result)
template <int GATE> A2C_FN float gate_d(float h) {
  if (GATE == TANH) return 1.0f - h * h;
  if (GATE == RELU) return h > 0.0f ? 1.0f : 0.0f;
  return 1.0f;
}

// out[n][j] = gate(sum_k in[n][k] W[j][k] + b[j]),  n < M, j < J, k < K; consecutive threads take consecutive j
template <int GATE>
A2C_FN void dense_fwd(const float* in, int ldin, const float* W, int ldw, const float* b, float* out, int ldout, int M, int K,
                      int J, int tid, int NT) {
  for (int e = tid; e < M * J; e += NT) {
    const int n = e / J, j = e - n * J;
    const float* xr = in + (size_t)n * ldin;
    const float* wr = W + (size_t)j * ldw;
    float acc = 0.0f;
    for (int k = 0; k < K; ++k) acc = fmaf(xr[k], wr[k], acc);
    out[(size_t)n * ldout + j] = gate_f<GATE>(acc + b[j]);
  }
}

// out[n][k] = (sum_j d[n][j] W[j][k] + sum_j d2[n][j] W2[j][k]) * gate'(h[n][k]),  n < M, k < K (J2 = 0: no second term).
// out may be h: every element is read and then written by the same thread.
template <int GATE>
A2C_FN void dense_bwd(const float* d, int ldd, const float* W, int ldw, int J, const float* d2, int ldd2, const float* W2,
                      int ldw2, int J2, const float* h, float* out, int ldh, int M, int K, int tid, int NT) {
  for (int e = tid; e < M * K; e += NT) {
    const int n = e / K, k = e - n * K;
    float acc = 0.0f;
    for (int j = 0; j < J; ++j) acc = fmaf(d[(size_t)n * ldd + j], W[(size_t)j * ldw + k], acc);
    for (int j = 0; j < J2; ++j) acc = fmaf(d2[(size_t)n * ldd2 + j], W2[(size_t)j * ldw2 + k], acc);
    const size_t o = (size_t)n * ldh + k;
    out[o] = acc * gate_d<GATE>(h[o]);
  }
}

// gradient of a Linear layer: G[j][k] = sum_n d[n][j] in[n][k] (J x K elements), then Gb[j] = sum_n d[n][j] (J elements),
// one index space over the block; every sum runs over n in order inside one thread
A2C_FN void dense_wgrad(const float* d, int ldd, const float* in, int ldin, float* G, int ldg, float* Gb, int M, int J, int K,
                        int tid, int NT) {
  const int nw = J * K;
  for (int e = tid; e < nw + J; e += NT) {
    if (e < nw) {
      const int j = e / K, k = e - j * K;
      float acc = 0.0f;
      for (int n = 0; n < M; ++n) acc = fmaf(d[(size_t)n * ldd + j], in[(size_t)n * ldin + k], acc);
      G[(size_t)j * ldg + k] = acc;
    } else {
      const int j = e - nw;
      float acc = 0.0f;
      for (int n = 0; n < M; ++n) acc += d[(size_t)n * ldd + j];
      Gb[j] = acc;
    }
  }
}

A2C_FN float a2c_softplus(float x) { return x > 20.0f ? x : log1pf(expf(x)); }      // F.softplus (beta 1, threshold 20)
constexpr float A2C_LOG_SQRT_2PI = 0.91893853320467274178f;

A2C_FN float sum4(const float* p, int n) {              // fixed order, four independent chains
  float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f, s3 = 0.0f;
  int i = 0;
  for (; i + 3 < n; i += 4) { s0 += p[i]; s1 += p[i + 1]; s2 += p[i + 2]; s3 += p[i + 3]; }
  for (; i < n; ++i) s0 += p[i];
  return (s0 + s1) + (s2 + s3);
}

// ------------------------------------------------------------------------------------------------ phases (forward)
// parameters from the arena into the padded shared-memory copy; actor_only: the tensors the actor step's forward reads
template <int HEAD, bool SHARED>
A2C_FN void ph_load_weights(A2cShared& S, const A2cNet& net, bool actor_only, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  for (int i = 0; i < K::ntensors; ++i) {
    const bool critic_only = i == K::fc || i == K::bc || (!SHARED && i >= 4 && i < 8);
    if (actor_only && critic_only) continue;
    const TensorDesc d = a2c_tensor(i, K::ntr, net.D, net.H1, net.H2, net.A);
    const float* src = net.flat + net.off[i];
    for (int e = tid; e < d.rows * d.cols; e += NT) {
      const int j = e / d.cols, k = e - j * d.cols;
      S.W[d.woff + j * d.ld + k] = src[e];
    }
  }
}

// update P0: weights and the R rollout rows
template <int HEAD, bool SHARED>
A2C_FN void ph_load(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  ph_load_weights<HEAD, SHARED>(S, a.net, false, tid, NT);
  const int D = a.net.D;
  for (int e = tid; e < S.R * D; e += NT) {
    const int n = e / D, k = e - n * D;
    S.x[n * S.ldx + k] = a.state[e];
  }
}

// first layer of every trunk (the actor step: trunk 0 only)
template <int HEAD, bool SHARED, int GATE>
A2C_FN void ph_fwd1(A2cShared& S, const A2cNet& net, bool actor_only, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  const int ntr = actor_only ? 1 : K::ntr;
  for (int t = 0; t < ntr; ++t) {
    const TensorDesc w = a2c_tensor(4 * t, K::ntr, net.D, net.H1, net.H2, net.A);
    const TensorDesc b = a2c_tensor(4 * t + 1, K::ntr, net.D, net.H1, net.H2, net.A);
    dense_fwd<GATE>(S.x, S.ldx, S.W + w.woff, w.ld, S.W + b.woff, a2c_h(S, t, 0), S.ldh, S.R, net.D, net.H1, tid, NT);
  }
}

template <int HEAD, bool SHARED, int GATE>
A2C_FN void ph_fwd2(A2cShared& S, const A2cNet& net, bool actor_only, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  const int ntr = actor_only ? 1 : K::ntr;
  for (int t = 0; t < ntr; ++t) {
    const TensorDesc w = a2c_tensor(4 * t + 2, K::ntr, net.D, net.H1, net.H2, net.A);
    const TensorDesc b = a2c_tensor(4 * t + 3, K::ntr, net.D, net.H1, net.H2, net.A);
    dense_fwd<GATE>(a2c_h(S, t, 0), S.ldh, S.W + w.woff, w.ld, S.W + b.woff, a2c_h(S, t, 1), S.ldh, S.R, net.H1, net.H2, tid, NT);
  }
}

// heads: logits / mean = tanh(fc_action(.)) / q = fc_head(.), v = fc_critic(.) (not in the actor step), softplus(std) (GAUSS)
template <int HEAD, bool SHARED>
A2C_FN void ph_heads(A2cShared& S, const A2cNet& net, bool actor_only, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  const TensorDesc fa = a2c_tensor(K::fa, K::ntr, net.D, net.H1, net.H2, net.A);
  const TensorDesc ba = a2c_tensor(K::ba, K::ntr, net.D, net.H1, net.H2, net.A);
  dense_fwd<HEAD == GAUSS ? TANH : LINEAR>(a2c_h(S, 0, 1), S.ldh, S.W + fa.woff, fa.ld, S.W + ba.woff, S.z, S.lda, S.R, net.H2,
                                           net.A, tid, NT);
  if (!actor_only && HEAD != Q) {
    const TensorDesc fc = a2c_tensor(K::fc, K::ntr, net.D, net.H1, net.H2, net.A);
    const TensorDesc bc = a2c_tensor(K::bc, K::ntr, net.D, net.H1, net.H2, net.A);
    dense_fwd<LINEAR>(a2c_h(S, K::critic_trunk, 1), S.ldh, S.W + fc.woff, fc.ld, S.W + bc.woff, S.v, 1, S.R, net.H2, 1, tid, NT);
  }
  if (HEAD == GAUSS) {
    const TensorDesc sd = a2c_tensor(K::sd, K::ntr, net.D, net.H1, net.H2, net.A);
    for (int j = tid; j < net.A; j += NT) {
      const float s = a2c_softplus(S.W[sd.woff + j]);
      S.sdv[j] = s;
      S.lsd[j] = logf(s);
    }
  }
}

// ------------------------------------------------------------------------------------------------ phases (update)
// GAE for every worker (one thread per worker, the time loop in the reference's order and association: gae_seq_kernel mode 0),
// and per loss row: log pi(a|s), entropy (and the log-sum-exp of the logits, CAT)
template <int HEAD, bool SHARED>
A2C_FN void ph_rows(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  const int N = a.N, T = a.T, A = a.net.A;
  for (int i = tid; i < N; i += NT) {
    float ret = S.v[T * N + i], adv = 0.0f, vnext = ret;
    for (int t = T - 1; t >= 0; --t) {
      const int o = t * N + i;
      const float r = a.reward[o], m = a.mask[o], v = S.v[o];
      const float gm = A2C_MUL(a.discount, m);
      ret = A2C_ADD(r, A2C_MUL(gm, ret));
      if (a.use_gae) {
        const float td = A2C_SUB(A2C_ADD(r, A2C_MUL(gm, vnext)), v);
        adv = A2C_ADD(A2C_MUL(A2C_MUL(A2C_MUL(adv, a.tau), a.discount), m), td);
      } else {
        adv = A2C_SUB(ret, v);
      }
      S.adv[o] = adv;
      S.ret[o] = ret;
      vnext = v;
    }
  }
  for (int n = tid; n < S.M; n += NT) {
    const float* z = S.z + (size_t)n * S.lda;
    if (HEAD == CAT) {                                    // Categorical(logits=z): log_softmax, -(p * log p).sum()
      float mx = z[0];
      for (int j = 1; j < A; ++j) mx = fmaxf(mx, z[j]);
      float s = 0.0f;
      for (int j = 0; j < A; ++j) s += expf(z[j] - mx);
      const float lse = mx + logf(s);
      float h = 0.0f;
      for (int j = 0; j < A; ++j) {
        const float lp = z[j] - lse;
        h -= lp * expf(lp);
      }
      S.lse[n] = lse;
      S.logp[n] = z[(int)a.action[n]] - lse;
      S.ent[n] = h;
    } else {                                              // Normal(mean, std): log_prob and entropy summed over actions
      const float* act = a.action + (size_t)n * A;
      float lp = 0.0f, h = 0.0f;
      for (int j = 0; j < A; ++j) {
        const float sd = S.sdv[j], t = act[j] - z[j];
        lp += -(t * t) / (2.0f * sd * sd) - S.lsd[j] - A2C_LOG_SQRT_2PI;
        h += 0.5f + A2C_LOG_SQRT_2PI + S.lsd[j];
      }
      S.logp[n] = lp;
      S.ent[n] = h;
    }
  }
}

// the objective's terms per row and its gradients: d / d v, and d / d logits (CAT) or d / d pre-tanh mean (GAUSS)
template <int HEAD, bool SHARED>
A2C_FN void ph_loss_grad(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  const int M = S.M, A = a.net.A;
  const float invM = 1.0f / (float)M;
  for (int n = tid; n < M; n += NT) {
    const float e = A2C_SUB(S.ret[n], S.v[n]);
    S.dv[n] = -a.vw * e * invM;
    S.red[n] = A2C_MUL(S.logp[n], S.adv[n]);
    S.red[M + n] = S.ent[n];
    S.red[2 * M + n] = A2C_MUL(e, e);
  }
  const float gent = -a.ent_w * invM;                   // d(-w_ent mean(entropy)) / d entropy_n
  for (int e = tid; e < M * A; e += NT) {
    const int n = e / A, j = e - n * A;
    const float glp = -S.adv[n] * invM;                 // d(-mean(log pi * adv)) / d log pi_n
    const float zj = S.z[(size_t)n * S.lda + j];
    float g;
    if (HEAD == CAT) {
      const float lp = zj - S.lse[n], p = expf(lp);
      const float onehot = (int)a.action[n] == j ? 1.0f : 0.0f;
      g = glp * (onehot - p) + gent * (-p * (lp + S.ent[n]));
    } else {
      const float sd = S.sdv[j], t = a.action[(size_t)n * A + j] - zj;
      g = glp * (t / (sd * sd)) * (1.0f - zj * zj);
    }
    S.dz[(size_t)n * S.lda + j] = g;
  }
}

// the heads' parameter gradients (fc_action / fc_head, fc_critic, std) and the objective (one thread)
template <int HEAD, bool SHARED>
A2C_FN void ph_head_wgrad(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  const A2cNet& net = a.net;
  const int M = S.M, A = net.A;
  const TensorDesc fa = a2c_tensor(K::fa, K::ntr, net.D, net.H1, net.H2, A);
  const TensorDesc ba = a2c_tensor(K::ba, K::ntr, net.D, net.H1, net.H2, A);
  const TensorDesc fc = a2c_tensor(K::fc, K::ntr, net.D, net.H1, net.H2, A);
  const TensorDesc bc = a2c_tensor(K::bc, K::ntr, net.D, net.H1, net.H2, A);
  dense_wgrad(S.dz, S.lda, a2c_h(S, 0, 1), S.ldh, S.G + fa.woff, fa.ld, S.G + ba.woff, M, A, net.H2, tid, NT);
  if (HEAD == Q) {
    if (tid == NT - 1) S.scal[0] = 0.5f * (sum4(S.red, M) * (1.0f / (float)M));   // NStepDQN_agent.py:63
    return;
  }
  dense_wgrad(S.dv, 1, a2c_h(S, K::critic_trunk, 1), S.ldh, S.G + fc.woff, fc.ld, S.G + bc.woff, M, 1, net.H2, tid, NT);
  if (HEAD == DUEL) {                                   // fc_value's gradient above; the objective of the Q head
    if (tid == NT - 1) S.scal[0] = 0.5f * (sum4(S.red, M) * (1.0f / (float)M));
    return;
  }
  if (HEAD == GAUSS) {                                  // d / d std_param: summed over rows, then through softplus
    const TensorDesc sd = a2c_tensor(K::sd, K::ntr, net.D, net.H1, net.H2, A);
    const float invM = 1.0f / (float)M, gent = -a.ent_w * invM;
    for (int j = tid; j < A; j += NT) {
      const float s = S.sdv[j];
      float acc = 0.0f;
      for (int n = 0; n < M; ++n) {
        const float t = a.action[(size_t)n * A + j] - S.z[(size_t)n * S.lda + j], glp = -S.adv[n] * invM;
        acc += glp * ((t * t) / (s * s * s) - 1.0f / s) + gent * (1.0f / s);
      }
      const float p = S.W[sd.woff + j];
      S.G[sd.woff + j] = acc * (p > 20.0f ? 1.0f : 1.0f / (1.0f + expf(-p)));
    }
  }
  if (tid == NT - 1) {                                  // A2C_agent.py:55-62, the association of a2c_loss_kernel
    const float invM = 1.0f / (float)M;
    const float pl = -(sum4(S.red, M) * invM), el = sum4(S.red + M, M) * invM, vl = 0.5f * (sum4(S.red + 2 * M, M) * invM);
    S.scal[0] = pl - a.ent_w * el + a.vw * vl;
  }
}

// back through the heads into the last layer of the trunk(s): in place over its output
template <int HEAD, bool SHARED, int GATE>
A2C_FN void ph_bwd2(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  const A2cNet& net = a.net;
  const TensorDesc fa = a2c_tensor(K::fa, K::ntr, net.D, net.H1, net.H2, net.A);
  const TensorDesc fc = a2c_tensor(K::fc, K::ntr, net.D, net.H1, net.H2, net.A);
  float* h0 = a2c_h(S, 0, 1);
  if (HEAD == Q) {
    dense_bwd<GATE>(S.dz, S.lda, S.W + fa.woff, fa.ld, net.A, nullptr, 0, nullptr, 0, 0, h0, h0, S.ldh, S.M, net.H2, tid, NT);
  } else if (SHARED) {
    dense_bwd<GATE>(S.dz, S.lda, S.W + fa.woff, fa.ld, net.A, S.dv, 1, S.W + fc.woff, fc.ld, 1, h0, h0, S.ldh, S.M, net.H2, tid, NT);
  } else {
    float* h1 = a2c_h(S, 1, 1);
    dense_bwd<GATE>(S.dz, S.lda, S.W + fa.woff, fa.ld, net.A, nullptr, 0, nullptr, 0, 0, h0, h0, S.ldh, S.M, net.H2, tid, NT);
    dense_bwd<GATE>(S.dv, 1, S.W + fc.woff, fc.ld, 1, nullptr, 0, nullptr, 0, 0, h1, h1, S.ldh, S.M, net.H2, tid, NT);
  }
}

// second layer's gradients (its pre-activation gradient x the first layer's output)
template <int HEAD, bool SHARED>
A2C_FN void ph_wgrad2(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  const A2cNet& net = a.net;
  for (int t = 0; t < K::ntr; ++t) {
    const TensorDesc w = a2c_tensor(4 * t + 2, K::ntr, net.D, net.H1, net.H2, net.A);
    const TensorDesc b = a2c_tensor(4 * t + 3, K::ntr, net.D, net.H1, net.H2, net.A);
    dense_wgrad(a2c_h(S, t, 1), S.ldh, a2c_h(S, t, 0), S.ldh, S.G + w.woff, w.ld, S.G + b.woff, S.M, net.H2, net.H1, tid, NT);
  }
}

// back into the first layer: in place over its output
template <int HEAD, bool SHARED, int GATE>
A2C_FN void ph_bwd1(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  const A2cNet& net = a.net;
  for (int t = 0; t < K::ntr; ++t) {
    const TensorDesc w = a2c_tensor(4 * t + 2, K::ntr, net.D, net.H1, net.H2, net.A);
    float* h = a2c_h(S, t, 0);
    dense_bwd<GATE>(a2c_h(S, t, 1), S.ldh, S.W + w.woff, w.ld, net.H2, nullptr, 0, nullptr, 0, 0, h, h, S.ldh, S.M, net.H1, tid, NT);
  }
}

template <int HEAD, bool SHARED>
A2C_FN void ph_wgrad1(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  const A2cNet& net = a.net;
  for (int t = 0; t < K::ntr; ++t) {
    const TensorDesc w = a2c_tensor(4 * t, K::ntr, net.D, net.H1, net.H2, net.A);
    const TensorDesc b = a2c_tensor(4 * t + 1, K::ntr, net.D, net.H1, net.H2, net.A);
    dense_wgrad(a2c_h(S, t, 0), S.ldh, S.x, S.ldx, S.G + w.woff, w.ld, S.G + b.woff, S.M, net.H1, net.D, tid, NT);
  }
}

// chunk c of the gradient (tensor order, A2C_CHUNK elements of one tensor per chunk): its sum of squares, in order
template <int HEAD, bool SHARED>
A2C_FN void ph_norm(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  const A2cNet& net = a.net;
  for (int c = tid; c < S.nchunks; c += NT) {
    int i = 0, c0 = 0;
    TensorDesc d = a2c_tensor(0, K::ntr, net.D, net.H1, net.H2, net.A);
    for (;;) {
      const int nc = (d.rows * d.cols + A2C_CHUNK - 1) / A2C_CHUNK;
      if (c < c0 + nc) break;
      c0 += nc;
      d = a2c_tensor(++i, K::ntr, net.D, net.H1, net.H2, net.A);
    }
    const int e1 = d.rows * d.cols, e0 = (c - c0) * A2C_CHUNK;
    float s = 0.0f;
    for (int e = e0; e < e1 && e < e0 + A2C_CHUNK; ++e) {
      const int j = e / d.cols, k = e - j * d.cols;
      const float g = S.G[d.woff + j * d.ld + k];
      s = fmaf(g, g, s);
    }
    S.part[c] = s;
  }
}

// clip_grad_norm_ (coefficient min(1, max_norm / (norm + 1e-6)), as optim.cu's sumsq_kernel) and RMSprop: every thread sums
// the chunk partials in the same order, so all see the same norm; new parameters and moments go to the arena
template <int HEAD, bool SHARED>
A2C_FN void ph_rmsprop(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  using K = A2cKind<HEAD, SHARED>;
  const A2cNet& net = a.net;
  const float norm = sqrtf(sum4(S.part, S.nchunks));
  const float coef = a.max_norm > 0.0f ? fminf(a.max_norm / (norm + 1e-6f), 1.0f) : 1.0f;
  for (int i = 0; i < K::ntensors; ++i) {
    const TensorDesc d = a2c_tensor(i, K::ntr, net.D, net.H1, net.H2, net.A);
    const int o = net.off[i];
    for (int e = tid; e < d.rows * d.cols; e += NT) {
      const int j = e / d.cols, k = e - j * d.cols, w = d.woff + j * d.ld + k;
      net.flat[o + e] = b2rl_elem::rmsprop_elem(S.W[w], S.G[w] * coef, a.sq, a.ga, (int64_t)o + e, a.lr, a.alpha, a.eps,
                                                a.centered);
    }
  }
  if (tid == 0) {
    *a.step += 1;
    *a.loss = S.scal[0];
  }
}

// ------------------------------------------------------------------------------------------------ phases (n-step Q)
// P0: ph_load, and the target sync (NStepDQN_agent.py:48-50): the online parameters do not change during a rollout, so a sync at
// any of its env steps is a copy of the arena as it is before this update
A2C_FN void ph_nstep_load(A2cShared& S, const NStepArgs& q, int tid, int NT) {
  using K = A2cKind<Q, true>;
  ph_load<Q, true>(S, q.a, tid, NT);
  if (!q.sync) return;
  const A2cNet& net = q.a.net;
  for (int i = 0; i < K::ntensors; ++i) {
    const TensorDesc d = a2c_tensor(i, K::ntr, net.D, net.H1, net.H2, net.A);
    for (int e = tid; e < d.rows * d.cols; e += NT) q.target[net.off[i] + e] = net.flat[net.off[i] + e];
  }
}

// layer l (0, 1: the trunk, 2: fc_head) of the target network on the N bootstrap states (row block T), into rows M.. of h / z.
// Its weights are read from the arena in global memory (rows of `cols` floats); after a sync they are the online ones, which
// the arena still holds until the last phase.  Runs in the same phase as the online forward's layer l (disjoint rows).
template <int GATE>
A2C_FN void ph_boot(A2cShared& S, const NStepArgs& q, int l, int tid, int NT) {
  using K = A2cKind<Q, true>;
  const A2cNet& net = q.a.net;
  const float* w = q.sync ? net.flat : q.target;
  const int N = q.a.N;
  const size_t rh = (size_t)S.M * S.ldh;
  if (l == 0)
    dense_fwd<GATE>(q.a.state + (size_t)S.M * net.D, net.D, w + net.off[0], net.D, w + net.off[1], a2c_h(S, 0, 0) + rh, S.ldh,
                    N, net.D, net.H1, tid, NT);
  else if (l == 1)
    dense_fwd<GATE>(a2c_h(S, 0, 0) + rh, S.ldh, w + net.off[2], net.H1, w + net.off[3], a2c_h(S, 0, 1) + rh, S.ldh, N, net.H1,
                    net.H2, tid, NT);
  else
    dense_fwd<LINEAR>(a2c_h(S, 0, 1) + rh, S.ldh, w + net.off[K::fa], net.H2, w + net.off[K::ba], S.z + (size_t)S.M * S.lda,
                      S.lda, N, net.H2, net.A, tid, NT);
}

// per worker (one thread each): the bootstrap max_a q_target(s_T) (:56-57) and the return scan ret = r + (discount mask) ret
// (:58-60), the arithmetic of ph_rows' ret (gae_seq_kernel mode 0)
A2C_FN void ph_nstep_returns(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  const int N = a.N, T = a.T, A = a.net.A;
  for (int i = tid; i < N; i += NT) {
    const float* zb = S.z + (size_t)(S.M + i) * S.lda;
    float ret = zb[0];
    for (int j = 1; j < A; ++j) ret = fmaxf(ret, zb[j]);
    for (int t = T - 1; t >= 0; --t) {
      const int o = t * N + i;
      ret = A2C_ADD(a.reward[o], A2C_MUL(A2C_MUL(a.discount, a.mask[o]), ret));
      S.ret[o] = ret;
    }
  }
}

// e_n = q[n][a_n] - ret_n, e_n^2 for the objective, and d(0.5 mean(e^2)) / dq[n][j] = (j == a_n) e_n / M
A2C_FN void ph_nstep_loss_grad(A2cShared& S, const A2cArgs& a, int tid, int NT) {
  const int M = S.M, A = a.net.A;
  const float invM = 1.0f / (float)M;
  for (int e = tid; e < M * A; e += NT) {
    const int n = e / A, j = e - n * A, an = (int)a.action[n];
    const float err = A2C_SUB(S.z[(size_t)n * S.lda + an], S.ret[n]);
    S.dz[(size_t)n * S.lda + j] = j == an ? A2C_MUL(err, invM) : 0.0f;
    if (j == 0) S.red[n] = A2C_MUL(err, err);
  }
}

// ------------------------------------------------------------------------------------------------ phases (replay Q)
#ifdef __CUDACC__
#define A2C_DIV(x, y) __fdiv_rn(x, y)
#else
#define A2C_DIV(x, y) ((x) / (y))
#endif

// the replay Q update's arguments besides A2cArgs, of which it reads net, the RMSprop fields, max_norm, loss, N (= B) and
// discount (= discount ** n_step)
struct DqnArgs {
  A2cArgs a;
  const void* state; const void* next_state;     // [B][D] sampled rows: float64 (f64) or float32
  int f64; double scale;                         // RescaleNormalizer: float32(scale * double(x)), rounded once
  const int64_t* action; const float* reward; const float* mask;   // [B]
  const float* target;                           // the target network's arena: the layout of a.net.flat, the same offsets
  int double_q;
  const float* prob; float beta, per_eps, per_alpha;   // PER when prob is set: sampling probabilities [B], beta, eps, alpha
  float* priority;                               // [B] (|delta| + eps)^alpha, PER only
  float* delta;                                  // [B] y - q[a], optional
};

struct DqnShared {
  A2cShared s;
  float *delta, *wt;                             // [B] delta, importance weights before the max-normalisation
};

// the shared block of the replay Q update: x holds the B states, then the B next states.  The online forward covers S.R rows
// (the states, and with double_q the next states too, for the argmax), the target network's forward the B rows after them in
// h / z / v.  The backward covers the first S.M = B rows.  base may be a dummy when only the size is wanted.
template <int HEAD>
A2C_HD size_t dqn_carve(DqnShared& DS, float* base, int D, int H1, int H2, int A, int B, int double_q) {
  using K = A2cKind<HEAD, true>;
  A2cShared& S = DS.s;
  const TensorDesc last = a2c_tensor(K::ntensors - 1, K::ntr, D, H1, H2, A);
  const size_t wsize = (size_t)last.woff + (size_t)last.rows * last.ld;
  int nchunks = 0;
  for (int i = 0; i < K::ntensors; ++i) {
    const TensorDesc d = a2c_tensor(i, K::ntr, D, H1, H2, A);
    nchunks += (d.rows * d.cols + A2C_CHUNK - 1) / A2C_CHUNK;
  }
  const int R = (double_q ? 2 : 1) * B, Rt = R + B;
  const bool duel = HEAD == DUEL;
  S.ldx = a2c_odd(D);
  S.ldh = a2c_odd(H1 > H2 ? H1 : H2);
  S.lda = a2c_odd(A);
  S.hstride = Rt * S.ldh;
  S.R = R;
  S.M = B;
  S.nchunks = nchunks;
  S.adv = S.ret = S.logp = S.ent = S.lse = S.sdv = S.lsd = nullptr;
  size_t off = 0;
#define A2C_TAKE(n) (base + (off += ((size_t)(n) + 3) / 4 * 4) - ((size_t)(n) + 3) / 4 * 4)
  S.W = A2C_TAKE(wsize);
  S.G = A2C_TAKE(wsize);
  S.x = A2C_TAKE((size_t)2 * B * S.ldx);
  S.h = A2C_TAKE((size_t)2 * S.hstride);
  S.z = A2C_TAKE((size_t)Rt * S.lda);
  S.dz = A2C_TAKE((size_t)B * S.lda);
  S.v = duel ? A2C_TAKE(Rt) : nullptr;
  S.dv = duel ? A2C_TAKE(B) : nullptr;
  S.red = A2C_TAKE(B);
  S.part = A2C_TAKE(nchunks);
  S.scal = A2C_TAKE(4);
  DS.delta = A2C_TAKE(B);
  DS.wt = A2C_TAKE(B);
#undef A2C_TAKE
  return off;
}

// at::pow(Tensor, Scalar)'s special cases (losses.cu pow_like_torch)
A2C_FN float a2c_pow_torch(float x, float e) {
  if (e == 0.5f) return sqrtf(x);
  if (e == 1.0f) return x;
  if (e == 2.0f) return x * x;
  if (e == -0.5f) return 1.0f / sqrtf(x);
  if (e == -1.0f) return 1.0f / x;
  return powf(x, e);
}

// DuelingNet (network_heads.py DuelingNet.forward): q = v + (adv - mean(adv)) in place over the advantages of rows 0..rows-1
A2C_FN void ph_duel_q(A2cShared& S, int rows, int A, int tid, int NT) {
  for (int n = tid; n < rows; n += NT) {
    float* z = S.z + (size_t)n * S.lda;
    float s = 0.0f;
    for (int j = 0; j < A; ++j) s += z[j];
    const float mean = A2C_DIV(s, (float)A), v = S.v[n];
    for (int j = 0; j < A; ++j) z[j] = A2C_ADD(v, A2C_SUB(z[j], mean));
  }
}

// P0: parameters, and the rescaled states / next states
template <int HEAD>
A2C_FN void ph_dqn_load(DqnShared& DS, const DqnArgs& d, int tid, int NT) {
  A2cShared& S = DS.s;
  ph_load_weights<HEAD, true>(S, d.a.net, false, tid, NT);
  const int D = d.a.net.D, n1 = S.M * D;
  for (int e = tid; e < 2 * n1; e += NT) {
    const int n = e / D, k = e - n * D, e1 = e < n1 ? e : e - n1;
    const void* src = e < n1 ? d.state : d.next_state;
    const double x = d.f64 ? static_cast<const double*>(src)[e1] : (double)static_cast<const float*>(src)[e1];
    S.x[n * S.ldx + k] = (float)(d.scale * x);
  }
}

// layer l (0, 1: the trunk, 2: the head) of the target network on the B next states, into the rows S.R.. of h / z (/ v).  Its
// weights are read from the target arena in global memory (rows of `cols` floats).  Runs in the phase of the online layer l.
template <int HEAD, int GATE>
A2C_FN void ph_dqn_target_fwd(DqnShared& DS, const DqnArgs& d, int l, int tid, int NT) {
  using K = A2cKind<HEAD, true>;
  A2cShared& S = DS.s;
  const A2cNet& net = d.a.net;
  const float* w = d.target;
  const int B = S.M;
  const size_t rh = (size_t)S.R * S.ldh;
  if (l == 0) {
    dense_fwd<GATE>(S.x + (size_t)B * S.ldx, S.ldx, w + net.off[0], net.D, w + net.off[1], a2c_h(S, 0, 0) + rh, S.ldh, B, net.D,
                    net.H1, tid, NT);
  } else if (l == 1) {
    dense_fwd<GATE>(a2c_h(S, 0, 0) + rh, S.ldh, w + net.off[2], net.H1, w + net.off[3], a2c_h(S, 0, 1) + rh, S.ldh, B, net.H1,
                    net.H2, tid, NT);
  } else {
    dense_fwd<LINEAR>(a2c_h(S, 0, 1) + rh, S.ldh, w + net.off[K::fa], net.H2, w + net.off[K::ba], S.z + (size_t)S.R * S.lda,
                      S.lda, B, net.H2, net.A, tid, NT);
    if (HEAD == DUEL)
      dense_fwd<LINEAR>(a2c_h(S, 0, 1) + rh, S.ldh, w + net.off[K::fc], net.H2, w + net.off[K::bc], S.v + S.R, 1, B, net.H2, 1,
                        tid, NT);
  }
}

// per sample (one thread each; the arithmetic of losses.cu dqn_loss_kernel): the bootstrap q (DQN_agent.py:88-92: the target's
// max, or with double_q the target's q at the online argmax, first maximal index), y = r + discount^n q_next mask (:95),
// delta = y - q[a] (:99); PER: the priority (|delta| + eps)^alpha (:121) and the unnormalised weight (P B + 1e-6)^-beta (:125)
template <int HEAD>
A2C_FN void ph_dqn_delta(DqnShared& DS, const DqnArgs& d, int tid, int NT) {
  A2cShared& S = DS.s;
  const int B = S.M, A = d.a.net.A;
  for (int n = tid; n < B; n += NT) {
    const float* zt = S.z + (size_t)(S.R + n) * S.lda;
    float qn;
    if (d.double_q) {
      const float* zo = S.z + (size_t)(B + n) * S.lda;
      int best = 0;
      float bv = zo[0];
      for (int j = 1; j < A; ++j)
        if (zo[j] > bv) { bv = zo[j]; best = j; }
      qn = zt[best];
    } else {
      qn = zt[0];
      for (int j = 1; j < A; ++j) qn = fmaxf(qn, zt[j]);
    }
    const float y = A2C_ADD(d.reward[n], A2C_MUL(A2C_MUL(d.a.discount, qn), d.mask[n]));
    const float dl = A2C_SUB(y, S.z[(size_t)n * S.lda + (int)d.action[n]]);
    DS.delta[n] = dl;
    if (d.delta) d.delta[n] = dl;
    if (d.prob) {
      d.priority[n] = a2c_pow_torch(A2C_ADD(fabsf(dl), d.per_eps), d.per_alpha);
      DS.wt[n] = a2c_pow_torch(A2C_ADD(A2C_MUL(d.prob[n], (float)B), 1e-6f), -d.beta);
    }
  }
}

// w = weight / max(weights) (:126, every thread takes the max in the same order), wl = delta w (:127), (wl)^2 for the objective
// 0.5 mean(wl^2) (:79), and its gradient d / dq[n][j] = (j == a_n) (-wl w / B); DUEL: through q = v + (adv - mean(adv)) into
// d / d adv (the fc_action slot) and d / d v (the fc_critic slot)
template <int HEAD>
A2C_FN void ph_dqn_loss_grad(DqnShared& DS, const DqnArgs& d, int tid, int NT) {
  A2cShared& S = DS.s;
  const int B = S.M, A = d.a.net.A;
  const float invB = 1.0f / (float)B;
  float wmax = 1.0f;
  if (d.prob) {
    wmax = 0.0f;
    for (int i = 0; i < B; ++i) wmax = fmaxf(wmax, DS.wt[i]);
  }
  for (int e = tid; e < B * A; e += NT) {
    const int n = e / A, j = e - n * A, an = (int)d.action[n];
    const float w = d.prob ? A2C_DIV(DS.wt[n], wmax) : 1.0f;
    const float wl = A2C_MUL(DS.delta[n], w);
    const float g = A2C_MUL(A2C_MUL(-wl, w), invB);
    float* dz = S.dz + (size_t)n * S.lda;
    if (HEAD == DUEL) {
      dz[j] = A2C_SUB(j == an ? g : 0.0f, A2C_DIV(g, (float)A));
      if (j == 0) S.dv[n] = g;
    } else {
      dz[j] = j == an ? g : 0.0f;
    }
    if (j == 0) S.red[n] = A2C_MUL(wl, wl);
  }
}

}  // namespace b2rl_a2c
