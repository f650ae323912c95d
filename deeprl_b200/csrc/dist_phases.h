// dist_phases.h -- the gradient update of the distributional DQN agents (CategoricalDQN_agent.py:60-89, C51;
// QuantileRegressionDQN_agent.py:55-77, QR-DQN) for a CategoricalNet / QuantileNet on a two-layer FCBody, written as PHASES of
// one thread block like a2c_phases.h, whose trunk, head, target-network, backward, clip and RMSprop phases it reuses with
// HEAD = Q: the distributional head is a Q head of width A K (K atoms / quantiles per action, row-major [A][K]).  The update's
// sequence is dist_sequence.inc; csrc/dist_dqn.cu runs it as one launch, tests/host_emul/dist_emul.cpp with the threads of a
// phase one after another.  Nothing here depends on the execution order inside a phase or on the number of threads.
//
//   C51  log_softmax of the online logits on the states and softmax of the next-state logits, per (row, action) over K; the
//        expected values sum_k p z_k of the target network (or with double_q of the online network) on the next states and
//        their first maximum a*; the projection m_j of the target's p(a*) onto the atoms; KL = sum m log(m + 1e-5) - m log p[a];
//        PER priorities and weights; mean(w KL); the gradient through log_softmax of the chosen action.  The arithmetic of
//        losses.cu c51_loss_kernel: float64 linspace atoms rounded once, float32 delta_atom.
//   QR   the target's first argmax of sum_k theta'; T_j = r + gamma^n m theta'_j(a*); the pairwise quantile-Huber terms
//        (kappa 1) summed over the online quantile i; the loss vector indexed by target quantile (mean over the batch) and its
//        mean; d theta_i = -sum_j psi(u) |tau_i - 1{u < 0}| / (B K) for the chosen action.  The arithmetic of qr_loss_kernel.
#pragma once
#include "a2c_phases.h"

#ifdef __CUDACC__
#define DIST_DMUL(x, y) __dmul_rn(x, y)
#define DIST_DADD(x, y) __dadd_rn(x, y)
#else
#define DIST_DMUL(x, y) ((x) * (y))
#define DIST_DADD(x, y) ((x) + (y))
#endif

namespace b2rl_dist {

using b2rl_a2c::A2cShared;
using b2rl_a2c::DqnArgs;
using b2rl_a2c::DqnShared;

enum { C51 = 0, QR = 1 };   // kind of the distributional head

// the update's arguments besides DqnArgs, whose net.A is A K.  DqnArgs.delta is not written; double_q and the PER fields are
// read by C51 only.
struct DistArgs {
  DqnArgs d;
  int A, K;
  double v_min, v_max;                       // C51: the support, np.linspace(v_min, v_max, K)
  float* loss_vec;                           // optional: per-sample KL [B] (C51) / the loss vector [K] (QR)
};

struct DistShared {
  DqnShared ds;
  float* atoms;                              // [K] (C51)
  float* astar;                              // [B] the bootstrap action, as a float
  float* mt;                                 // [B][K] C51: the projected target distribution m; QR: the target quantiles T
  float* rs;                                 // [B][K] QR: the quantile-Huber terms of (sample, target quantile) summed over i
  float* lv;                                 // [max(B, K)] per-sample KL (C51) / the loss vector (QR)
};

// dqn_carve<Q>'s block for a head of width A K (QR: no online forward of the next states), then the buffers above
template <int KIND>
A2C_HD size_t dist_carve(DistShared& T, float* base, int D, int H1, int H2, int A, int K, int B, int double_q) {
  size_t off = b2rl_a2c::dqn_carve<b2rl_a2c::Q>(T.ds, base, D, H1, H2, A * K, B, KIND == C51 ? double_q : 0);
#define DIST_TAKE(n) (base + (off += ((size_t)(n) + 3) / 4 * 4) - ((size_t)(n) + 3) / 4 * 4)
  T.atoms = KIND == C51 ? DIST_TAKE(K) : nullptr;
  T.astar = DIST_TAKE(B);
  T.mt = DIST_TAKE((size_t)B * K);
  T.rs = KIND == QR ? DIST_TAKE((size_t)B * K) : nullptr;
  T.lv = DIST_TAKE(B > K ? B : K);
#undef DIST_TAKE
  return off;
}

// np.linspace(v_min, v_max, K) in float64 (arange * step + start, the last point exactly v_max), then float32 (tensor())
A2C_FN float dist_atom(int k, int K, double v_min, double v_max) {
  if (k == K - 1) return (float)v_max;
  const double step = (v_max - v_min) / (double)(K - 1);
  return (float)DIST_DADD(DIST_DMUL((double)k, step), v_min);
}

A2C_FN float dist_delta_atom(const DistArgs& g) { return (float)((g.v_max - g.v_min) / (double)(g.K - 1)); }

// torch.clamp(x, v_min, v_max) with the bounds as float32
A2C_FN float dist_clamp(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }

// P0 (with ph_dqn_load): the atoms
template <int KIND>
A2C_FN void ph_dist_atoms(DistShared& T, const DistArgs& g, int tid, int NT) {
  if (KIND != C51) return;
  for (int k = tid; k < g.K; k += NT) T.atoms[k] = dist_atom(k, g.K, g.v_min, g.v_max);
}

// C51, per (row, action): log_softmax over K in place on the B state rows (network_heads.py CategoricalNet: F.log_softmax),
// softmax in place on the next-state rows (online with double_q, then the target's)
template <int KIND>
A2C_FN void ph_dist_softmax(DistShared& T, const DistArgs& g, int tid, int NT) {
  A2cShared& S = T.ds.s;
  const int B = S.M, A = g.A, K = g.K, rows = KIND == C51 ? S.R + B : 0;
  for (int e = tid; e < rows * A; e += NT) {
    const int n = e / A, a = e - n * A;
    float* z = S.z + (size_t)n * S.lda + a * K;
    float mx = z[0];
    for (int k = 1; k < K; ++k) mx = fmaxf(mx, z[k]);
    float s = 0.0f;
    for (int k = 0; k < K; ++k) s += expf(z[k] - mx);
    if (n < B) {
      const float ls = logf(s);
      for (int k = 0; k < K; ++k) z[k] = A2C_SUB(A2C_SUB(z[k], mx), ls);
    } else {
      for (int k = 0; k < K; ++k) z[k] = A2C_DIV(expf(z[k] - mx), s);
    }
  }
}

// per sample: the bootstrap action a*, the first maximum of -- C51: sum_k p z_k of the target network, or with double_q of
// the online network, on the next state (CategoricalDQN_agent.py:66-70); QR: sum_k theta' of the target (:60)
template <int KIND>
A2C_FN void ph_dist_argmax(DistShared& T, const DistArgs& g, int tid, int NT) {
  A2cShared& S = T.ds.s;
  const int B = S.M, A = g.A, K = g.K;
  for (int n = tid; n < B; n += NT) {
    const int row = KIND == C51 && g.d.double_q ? B + n : S.R + n;
    const float* z = S.z + (size_t)row * S.lda;
    int best = 0;
    float bv = 0.0f;
    for (int a = 0; a < A; ++a) {
      float s = 0.0f;
      for (int k = 0; k < K; ++k) s += KIND == C51 ? A2C_MUL(z[a * K + k], T.atoms[k]) : z[a * K + k];
      if (a == 0 || s > bv) { bv = s; best = a; }
    }
    T.astar[n] = (float)best;
  }
}

// per (sample, atom j) -- C51: the projection m_j = sum_k clamp(1 - |Tz_k - z_j| / delta_atom, 0, 1) p'_k(a*) with
// Tz_k = clamp(r + gamma^n mask z_k, v_min, v_max) (:75-80); QR: T_j = r + gamma^n mask theta'_j(a*) (:65)
template <int KIND>
A2C_FN void ph_dist_target(DistShared& T, const DistArgs& g, int tid, int NT) {
  A2cShared& S = T.ds.s;
  const int B = S.M, K = g.K;
  const float lo = (float)g.v_min, hi = (float)g.v_max, da = dist_delta_atom(g);
  for (int e = tid; e < B * K; e += NT) {
    const int n = e / K, j = e - n * K;
    const float r = g.d.reward[n], gm = A2C_MUL(g.d.a.discount, g.d.mask[n]);
    const float* pn = S.z + (size_t)(S.R + n) * S.lda + (int)T.astar[n] * K;
    if (KIND == C51) {
      const float zj = T.atoms[j];
      float m = 0.0f;
      for (int k = 0; k < K; ++k) {
        const float tz = dist_clamp(A2C_ADD(r, A2C_MUL(gm, T.atoms[k])), lo, hi);
        const float c = dist_clamp(A2C_SUB(1.0f, A2C_DIV(fabsf(A2C_SUB(tz, zj)), da)), 0.0f, 1.0f);
        m += A2C_MUL(c, pn[k]);
      }
      T.mt[e] = m;
    } else {
      T.mt[e] = A2C_ADD(r, A2C_MUL(gm, pn[j]));
    }
  }
}

A2C_FN float dist_tau(int i, int K) { return (float)((2.0 * i + 1.0) / (2.0 * K)); }   // QuantileRegressionDQN_agent.py:44-45

A2C_FN float dist_huber(float x) {                                                       // utils/torch_utils.py:47-48, k = 1
  const float ax = fabsf(x);
  return ax < 1.0f ? A2C_MUL(0.5f, A2C_MUL(x, x)) : A2C_SUB(ax, 0.5f);
}

// C51, per sample: KL = sum_j m_j log(m_j + 1e-5) - m_j log p_j(a) (:82-85), the PER priority (|KL| + eps)^alpha and the
// unnormalised weight (P B + 1e-6)^-beta (DQN_agent.py:121-125).  QR, per (sample, target quantile j): the quantile-Huber terms
// summed over the online quantiles i (:71-74)
template <int KIND>
A2C_FN void ph_dist_sample(DistShared& T, const DistArgs& g, int tid, int NT) {
  A2cShared& S = T.ds.s;
  const DqnArgs& d = g.d;
  const int B = S.M, K = g.K;
  if (KIND == C51) {
    for (int n = tid; n < B; n += NT) {
      const float* lp = S.z + (size_t)n * S.lda + (int)d.action[n] * K;
      const float* m = T.mt + (size_t)n * K;
      float kl = 0.0f;
      for (int j = 0; j < K; ++j) kl += A2C_SUB(A2C_MUL(m[j], logf(A2C_ADD(m[j], 1e-5f))), A2C_MUL(m[j], lp[j]));
      T.lv[n] = kl;
      if (g.loss_vec) g.loss_vec[n] = kl;
      if (d.prob) {
        d.priority[n] = b2rl_a2c::a2c_pow_torch(A2C_ADD(fabsf(kl), d.per_eps), d.per_alpha);
        T.ds.wt[n] = b2rl_a2c::a2c_pow_torch(A2C_ADD(A2C_MUL(d.prob[n], (float)B), 1e-6f), -d.beta);
      }
    }
  } else {
    for (int e = tid; e < B * K; e += NT) {
      const int n = e / K;
      const float tj = T.mt[e];
      const float* th = S.z + (size_t)n * S.lda + (int)d.action[n] * K;
      float s = 0.0f;
      for (int i = 0; i < K; ++i) {
        const float u = A2C_SUB(tj, th[i]);
        const float wq = fabsf(A2C_SUB(dist_tau(i, K), u < 0.0f ? 1.0f : 0.0f));
        s += A2C_MUL(dist_huber(u), wq);
      }
      T.rs[e] = s;
    }
  }
}

// the gradient w.r.t. the head's outputs (zero for every action but the chosen one), and the objective's terms.
// C51: w = weight / max(weights), d/dlogit_k = g_k - p_k sum_j g_j with g_j = -m_j w / B (log_softmax's backward; p_k =
// exp(log p_k)); S.red[n] = w KL.  QR: d theta_i = -sum_j psi(u) |tau_i - 1{u < 0}| / (B K); the loss vector
// lv[j] = sum_n rs[n][j] / B.
template <int KIND>
A2C_FN void ph_dist_loss_grad(DistShared& T, const DistArgs& g, int tid, int NT) {
  A2cShared& S = T.ds.s;
  const DqnArgs& d = g.d;
  const int B = S.M, K = g.K, AK = g.A * K;
  float wmax = 1.0f;
  if (KIND == C51 && d.prob) {
    wmax = 0.0f;
    for (int i = 0; i < B; ++i) wmax = fmaxf(wmax, T.ds.wt[i]);
  }
  const float gscale = 1.0f / ((float)B * (float)K);
  for (int e = tid; e < B * AK + (KIND == QR ? K : 0); e += NT) {
    if (e >= B * AK) {                                   // QR: the loss vector, .mean(1) over the batch
      const int j = e - B * AK;
      float s = 0.0f;
      for (int n = 0; n < B; ++n) s += T.rs[(size_t)n * K + j];
      T.lv[j] = A2C_DIV(s, (float)B);
      continue;
    }
    const int n = e / AK, c = e - n * AK, a = c / K, k = c - a * K, an = (int)d.action[n];
    const float* zr = S.z + (size_t)n * S.lda + an * K;
    float gk = 0.0f;
    if (a == an) {
      if (KIND == C51) {
        const float w = d.prob ? A2C_DIV(T.ds.wt[n], wmax) : 1.0f;
        const float scale = A2C_DIV(w, (float)B);
        const float* m = T.mt + (size_t)n * K;
        float gs = 0.0f;
        for (int j = 0; j < K; ++j) gs += A2C_MUL(-m[j], scale);
        gk = A2C_SUB(A2C_MUL(-m[k], scale), A2C_MUL(expf(zr[k]), gs));
        if (k == 0) S.red[n] = A2C_MUL(T.lv[n], w);
      } else {
        const float thi = zr[k], ti = dist_tau(k, K);
        for (int j = 0; j < K; ++j) {
          const float u = A2C_SUB(T.mt[(size_t)n * K + j], thi);
          const float wq = fabsf(A2C_SUB(ti, u < 0.0f ? 1.0f : 0.0f));
          const float hp = fabsf(u) < 1.0f ? u : (u > 0.0f ? 1.0f : -1.0f);
          gk -= A2C_MUL(A2C_MUL(gscale, hp), wq);
        }
      }
    }
    S.dz[(size_t)n * S.lda + c] = gk;
  }
}

// the objective into S.scal[0] (after ph_head_wgrad, whose Q branch writes it too): C51 mean(w KL) (:88-89), QR the mean of
// the loss vector (:76-77); and the optional QR loss vector out.  Runs in the phase of ph_bwd2, which reads neither.
template <int KIND>
A2C_FN void ph_dist_objective(DistShared& T, const DistArgs& g, int tid, int NT) {
  A2cShared& S = T.ds.s;
  const int B = S.M, K = g.K;
  if (KIND == QR && g.loss_vec)
    for (int j = tid; j < K; j += NT) g.loss_vec[j] = T.lv[j];
  if (tid == NT - 1) {
    float s = 0.0f;
    if (KIND == C51)
      for (int n = 0; n < B; ++n) s += S.red[n];
    else
      for (int j = 0; j < K; ++j) s += T.lv[j];
    S.scal[0] = A2C_DIV(s, (float)(KIND == C51 ? B : K));
  }
}

}  // namespace b2rl_dist
