// rainbow_phases.h -- the gradient update of CategoricalDQNAgent for a RainbowNet on a two-layer FCBody (rainbow_feature:
// NoisyLinear layers, a dueling categorical head, C51 + PER + double-Q + n-step), written as PHASES of one thread block like
// a2c_phases.h and dist_phases.h, whose phases it reuses by inclusion.  The update's sequence is rainbow_sequence.inc;
// csrc/rainbow.cu runs it as one launch, tests/host_emul/rainbow_emul.cpp with the threads of a phase one after another.
// Nothing here depends on the execution order inside a phase or on the number of threads.
//
//   layers    l = 0, 1: body.layers.l; l = 2: fc_advantage [A K][H2]; l = 3: fc_value [K][H2].  All four are NoisyLinear
//             (NOISY: weight_mu, weight_sigma, bias_mu, bias_sigma in the arena) or all four nn.Linear (weight, bias).
//   noise     per layer noise_in [in], noise_out_weight [out], noise_out_bias [out] (network_utils.py NoisyLinear.reset_noise),
//             the layers one after another: one "noise vector" of rb_noise_len floats per network.  f(x) = sign(x) sqrt|x|,
//             eps_w = f(out_w) (x) f(in), eps_b = f(out_b).  Only the f-transformed vectors live in shared memory.
//   effective W = mu + sigma eps_w, b = mu_b + sigma_b eps_b are formed while the online weights are loaded into shared memory,
//   weights   laid out as a2c_phases.h's HEAD = Q network whose head has (A + 1) K rows: fc_advantage's A K rows, then
//             fc_value's K rows.  ph_fwd1/2, ph_heads and the backward phases then apply unchanged and leave dW in S.G.  The
//             target network's effective weights are formed on the fly from the target arena.
//   dueling   q[a][k] = v[k] + (adv[a][k] - mean_a adv[.][k]) in place over the advantage columns of a row of z; backward
//             d adv[a][k] = dz[a][k] - mean_a dz[.][k], d v[k] = sum_a dz[a][k].
//   rows      h / z hold 2 B rows: the online forward covers the states and, with double_q, the next states, which are reduced
//             to the bootstrap action before the target network's forward overwrites rows B.. .
//   gradients d mu = dW, d sigma = dW eps_w, d mu_b = db, d sigma_b = db eps_b, formed from S.G and the noise vectors in the
//             norm and RMSprop phases.
#pragma once
#include "dist_phases.h"

namespace b2rl_rainbow {

using b2rl_a2c::A2cShared;
using b2rl_a2c::TensorDesc;
using b2rl_a2c::a2c_tensor;
using b2rl_dist::DistArgs;
using b2rl_dist::DistShared;

constexpr int RB_LAYERS = 4;
constexpr int RB_MAX_TENSORS = 16;

// the parameters in the optimizer's arena.  NOISY: layer l's weight_mu weight_sigma bias_mu bias_sigma at off[4 l .. 4 l + 3];
// plain: weight bias at off[2 l], off[2 l + 1]
struct RbNet {
  float* flat;
  int off[RB_MAX_TENSORS];
  int D, H1, H2, A, K;
};

A2C_HD int rb_in(const RbNet& n, int l) { return l == 0 ? n.D : l == 1 ? n.H1 : n.H2; }
A2C_HD int rb_out(const RbNet& n, int l) { return l == 0 ? n.H1 : l == 1 ? n.H2 : l == 2 ? n.A * n.K : n.K; }

// offset of layer l's noise_in in a noise vector (l = RB_LAYERS: its length)
A2C_HD int rb_noise_off(const RbNet& n, int l) {
  int o = 0;
  for (int u = 0; u < l; ++u) o += rb_in(n, u) + 2 * rb_out(n, u);
  return o;
}
A2C_HD int rb_noise_len(const RbNet& n) { return rb_noise_off(n, RB_LAYERS); }

// the noise arena the update writes for the online module: the noise vector, then every layer's bias_epsilon [out], then every
// layer's weight_epsilon [out][in]
A2C_HD int rb_beps_off(const RbNet& n, int l) {
  int o = rb_noise_len(n);
  for (int u = 0; u < l; ++u) o += rb_out(n, u);
  return o;
}
A2C_HD int rb_weps_off(const RbNet& n, int l) {
  int o = rb_beps_off(n, RB_LAYERS);
  for (int u = 0; u < l; ++u) o += rb_out(n, u) * rb_in(n, u);
  return o;
}
A2C_HD int rb_noise_arena_len(const RbNet& n) { return rb_weps_off(n, RB_LAYERS); }

// where layer l's effective weight rows and bias start in the shared-memory copy (and in the gradient copy)
struct RbEff { int w, ldw, b; };
A2C_HD RbEff rb_eff(const RbNet& n, int l) {
  const int AH = (n.A + 1) * n.K, row0 = l == 3 ? n.A * n.K : 0;
  const TensorDesc w = a2c_tensor(l < 2 ? 2 * l : 4, 1, n.D, n.H1, n.H2, AH);
  const TensorDesc b = a2c_tensor(l < 2 ? 2 * l + 1 : 5, 1, n.D, n.H1, n.H2, AH);
  RbEff e = {w.woff + row0 * w.ld, w.ld, b.woff + row0};
  return e;
}

// the update's arguments besides DistArgs, whose d.a.net describes the effective network (A = (A + 1) K; flat and off unused)
// and whose d.target is the target network's arena (the layout of net.flat, the same offsets)
struct RbArgs {
  DistArgs g;
  RbNet net;
  const float* given;                      // optional [2][noise_len]: the target's, then the online network's noise vector
  float* noise_out;                        // optional: the online module's noise arena (rb_noise_arena_len)
  float* target_noise_out;                 // optional [noise_len]: the target network's noise vector
  float noise_std;                         // Config.NOISY_LAYER_STD
};

struct RbShared {
  DistShared t;
  float* fo;                               // [noise_len] f(noise) of the online network
  float* ft;                               // [noise_len] f(noise) of the target network
};

template <bool NOISY> A2C_HD int rb_ntensors() { return NOISY ? 16 : 8; }
// arena tensor i = (layer, what): what 0 weight(_mu), 1 weight_sigma, 2 bias(_mu), 3 bias_sigma
template <bool NOISY> A2C_HD int rb_layer(int i) { return NOISY ? i >> 2 : i >> 1; }
template <bool NOISY> A2C_HD int rb_what(int i) { return NOISY ? i & 3 : 2 * (i & 1); }
template <bool NOISY> A2C_HD int rb_index(int l, int what) { return NOISY ? 4 * l + what : 2 * l + what / 2; }
A2C_HD int rb_numel(const RbNet& n, int l, int what) { return what < 2 ? rb_out(n, l) * rb_in(n, l) : rb_out(n, l); }
// network.parameters() lists fc_value, fc_advantage, then the body's layers: the order of the global norm's partial sums
A2C_HD int rb_param_layer(int p) { return p == 0 ? 3 : p == 1 ? 2 : p - 2; }

// the shared block of the update: the effective weights and their gradient copy, 2 B rows of x / h / z, B rows of dz, the C51
// buffers of dist_phases.h and both networks' transformed noise.  double_q does not change the size: the online forward of the
// next states uses the rows the target network's forward takes afterwards.  base may be a dummy when only the size is wanted.
template <bool NOISY>
A2C_HD size_t rb_carve(RbShared& RS, float* base, const RbNet& n, int B) {
  DistShared& T = RS.t;
  A2cShared& S = T.ds.s;
  const int AH = (n.A + 1) * n.K;
  const TensorDesc last = a2c_tensor(5, 1, n.D, n.H1, n.H2, AH);
  const size_t wsize = (size_t)last.woff + (size_t)last.rows * last.ld;
  int nchunks = 0;
  for (int i = 0; i < rb_ntensors<NOISY>(); ++i)
    nchunks += (rb_numel(n, rb_layer<NOISY>(i), rb_what<NOISY>(i)) + b2rl_a2c::A2C_CHUNK - 1) / b2rl_a2c::A2C_CHUNK;
  const int nz = NOISY ? rb_noise_len(n) : 0;
  S.ldx = b2rl_a2c::a2c_odd(n.D);
  S.ldh = b2rl_a2c::a2c_odd(n.H1 > n.H2 ? n.H1 : n.H2);
  S.lda = b2rl_a2c::a2c_odd(AH);
  S.hstride = 2 * B * S.ldh;
  S.R = B;
  S.M = B;
  S.nchunks = nchunks;
  S.v = S.dv = S.adv = S.ret = S.logp = S.ent = S.lse = S.sdv = S.lsd = nullptr;
  T.ds.delta = nullptr;
  T.rs = nullptr;
  size_t off = 0;
#define RB_TAKE(n) (base + (off += ((size_t)(n) + 3) / 4 * 4) - ((size_t)(n) + 3) / 4 * 4)
  S.W = RB_TAKE(wsize);
  S.G = RB_TAKE(wsize);
  S.x = RB_TAKE((size_t)2 * B * S.ldx);
  S.h = RB_TAKE((size_t)2 * S.hstride);
  S.z = RB_TAKE((size_t)2 * B * S.lda);
  S.dz = RB_TAKE((size_t)B * S.lda);
  S.red = RB_TAKE(B);
  S.part = RB_TAKE(nchunks);
  S.scal = RB_TAKE(4);
  T.ds.wt = RB_TAKE(B);
  T.atoms = RB_TAKE(n.K);
  T.astar = RB_TAKE(B);
  T.mt = RB_TAKE((size_t)B * n.K);
  T.lv = RB_TAKE(B);
  RS.fo = RB_TAKE(nz);
  RS.ft = RB_TAKE(nz);
#undef RB_TAKE
  return off;
}

// the online forward's view of the block: the B states, and with double_q the B next states too
A2C_FN A2cShared rb_online_rows(const A2cShared& S, int double_q) {
  A2cShared V = S;
  V.R = (double_q ? 2 : 1) * S.M;
  return V;
}

// rows row0.. of z as a block of its own for ph_dist_softmax: log_softmax on the first nlog rows, softmax on the next nsoft
A2C_FN DistShared rb_rows(const DistShared& T, int row0, int nlog, int nsoft) {
  DistShared V = T;
  V.ds.s.z = T.ds.s.z + (size_t)row0 * T.ds.s.lda;
  V.ds.s.M = nlog;
  V.ds.s.R = nsoft;
  return V;
}

// NoisyLinear.transform_noise: x.sign() * x.abs().sqrt()
A2C_FN float rb_f(float x) { return x < 0.0f ? -sqrtf(-x) : sqrtf(x); }

// mu + sigma * (f(out) f(in)), the roundings of NoisyLinear.forward on reset_noise's weight_epsilon
A2C_FN float rb_noisy(float mu, float sigma, float eps) { return A2C_ADD(mu, A2C_MUL(sigma, eps)); }

// one network's noise vector: the given one, or draw(base + i) * std for element i; written to raw_out when set, and its
// f-transform to f (shared memory)
template <bool NOISY, class DRAW>
A2C_FN void ph_rb_noise(const RbNet& n, float* f, const float* given, float* raw_out, float std, const DRAW& draw, int64_t base,
                        int tid, int NT) {
  if (!NOISY) return;
  const int nz = rb_noise_len(n);
  for (int i = tid; i < nz; i += NT) {
    const float x = given ? given[i] : A2C_MUL(draw(base + i), std);
    if (raw_out) raw_out[i] = x;
    f[i] = rb_f(x);
  }
}

// the online network's effective parameters into the padded shared-memory copy; with noise_out also weight_epsilon and
// bias_epsilon of every layer into the module's noise arena
template <bool NOISY>
A2C_FN void ph_rb_load_weights(A2cShared& S, const RbNet& n, const float* f, float* noise_out, int tid, int NT) {
  for (int l = 0; l < RB_LAYERS; ++l) {
    const int in = rb_in(n, l), out = rb_out(n, l);
    const RbEff ef = rb_eff(n, l);
    const float* fi = f + (NOISY ? rb_noise_off(n, l) : 0);
    const float *fow = fi + in, *fob = fow + out;
    const float* mu = n.flat + n.off[rb_index<NOISY>(l, 0)];
    const float* sg = n.flat + n.off[rb_index<NOISY>(l, 1)];
    const float* bmu = n.flat + n.off[rb_index<NOISY>(l, 2)];
    const float* bsg = n.flat + n.off[rb_index<NOISY>(l, 3)];
    float* weps = noise_out ? noise_out + rb_weps_off(n, l) : nullptr;
    float* beps = noise_out ? noise_out + rb_beps_off(n, l) : nullptr;
    for (int e = tid; e < out * in; e += NT) {
      const int j = e / in, k = e - j * in;
      float w = mu[e];
      if (NOISY) {
        const float eps = A2C_MUL(fow[j], fi[k]);
        w = rb_noisy(w, sg[e], eps);
        if (weps) weps[e] = eps;
      }
      S.W[ef.w + j * ef.ldw + k] = w;
    }
    for (int j = tid; j < out; j += NT) {
      float b = bmu[j];
      if (NOISY) {
        b = rb_noisy(b, bsg[j], fob[j]);
        if (beps) beps[j] = fob[j];
      }
      S.W[ef.b + j] = b;
    }
  }
}

// P0 of the update: the rescaled states and next states (ph_dqn_load's, without its parameter copy)
A2C_FN void ph_rb_load_states(A2cShared& S, const b2rl_a2c::DqnArgs& d, int D, int tid, int NT) {
  const int n1 = S.M * D;
  for (int e = tid; e < 2 * n1; e += NT) {
    const int n = e / D, k = e - n * D, e1 = e < n1 ? e : e - n1;
    const void* src = e < n1 ? d.state : d.next_state;
    const double x = d.f64 ? static_cast<const double*>(src)[e1] : (double)static_cast<const float*>(src)[e1];
    S.x[n * S.ldx + k] = (float)(d.scale * x);
  }
}

// out[m][j] = gate(sum_k in[m][k] W[j][k] + b[j]) with layer l's effective parameters formed from the arena `w` and the
// transformed noise `f` as they are read (dense_fwd's sums; consecutive threads take consecutive j)
template <bool NOISY, int GATE>
A2C_FN void rb_dense_fwd_arena(const float* in, int ldin, const RbNet& n, const float* w, const float* f, int l, float* out,
                               int ldout, int M, int tid, int NT) {
  const int K = rb_in(n, l), J = rb_out(n, l);
  const float* fi = f + (NOISY ? rb_noise_off(n, l) : 0);
  const float *fow = fi + K, *fob = fow + J;
  const float* mu = w + n.off[rb_index<NOISY>(l, 0)];
  const float* sg = w + n.off[rb_index<NOISY>(l, 1)];
  const float* bmu = w + n.off[rb_index<NOISY>(l, 2)];
  const float* bsg = w + n.off[rb_index<NOISY>(l, 3)];
  for (int e = tid; e < M * J; e += NT) {
    const int m = e / J, j = e - m * J;
    const float* xr = in + (size_t)m * ldin;
    const float *mr = mu + (size_t)j * K, *sr = sg + (size_t)j * K;
    float acc = 0.0f;
    if (NOISY) {
      const float fj = fow[j];
      for (int k = 0; k < K; ++k) acc = fmaf(xr[k], rb_noisy(mr[k], sr[k], A2C_MUL(fj, fi[k])), acc);
    } else {
      for (int k = 0; k < K; ++k) acc = fmaf(xr[k], mr[k], acc);
    }
    const float b = NOISY ? rb_noisy(bmu[j], bsg[j], fob[j]) : bmu[j];
    out[(size_t)m * ldout + j] = b2rl_a2c::gate_f<GATE>(acc + b);
  }
}

// step s (0, 1: the trunk, 2: fc_advantage and fc_value) of the target network on the B next states, into rows B.. of h / z
template <bool NOISY, int GATE>
A2C_FN void ph_rb_target_fwd(A2cShared& S, const RbNet& n, const float* target, const float* ft, int s, int tid, int NT) {
  const int B = S.M;
  const size_t rh = (size_t)B * S.ldh;
  float *h0 = b2rl_a2c::a2c_h(S, 0, 0) + rh, *h1 = b2rl_a2c::a2c_h(S, 0, 1) + rh, *z = S.z + (size_t)B * S.lda;
  if (s == 0) {
    rb_dense_fwd_arena<NOISY, GATE>(S.x + (size_t)B * S.ldx, S.ldx, n, target, ft, 0, h0, S.ldh, B, tid, NT);
  } else if (s == 1) {
    rb_dense_fwd_arena<NOISY, GATE>(h0, S.ldh, n, target, ft, 1, h1, S.ldh, B, tid, NT);
  } else {
    rb_dense_fwd_arena<NOISY, b2rl_a2c::LINEAR>(h1, S.ldh, n, target, ft, 2, z, S.lda, B, tid, NT);
    rb_dense_fwd_arena<NOISY, b2rl_a2c::LINEAR>(h1, S.ldh, n, target, ft, 3, z + n.A * n.K, S.lda, B, tid, NT);
  }
}

// RainbowNet.forward: q = value + (adv - adv.mean(1)) per (row, atom), in place over the advantages of rows row0..row0+rows-1
A2C_FN void ph_rb_duel(A2cShared& S, int A, int K, int row0, int rows, int tid, int NT) {
  for (int e = tid; e < rows * K; e += NT) {
    const int m = e / K, k = e - m * K;
    float* z = S.z + (size_t)(row0 + m) * S.lda;
    float s = 0.0f;
    for (int a = 0; a < A; ++a) s += z[a * K + k];
    const float mean = A2C_DIV(s, (float)A), v = z[A * K + k];
    for (int a = 0; a < A; ++a) z[a * K + k] = A2C_ADD(v, A2C_SUB(z[a * K + k], mean));
  }
}

// its backward per (sample, atom), in place over dz: d adv[a] = dz[a] - mean_a dz, d v = sum_a dz (into fc_value's columns)
A2C_FN void ph_rb_duel_bwd(A2cShared& S, int A, int K, int tid, int NT) {
  for (int e = tid; e < S.M * K; e += NT) {
    const int m = e / K, k = e - m * K;
    float* dz = S.dz + (size_t)m * S.lda;
    float s = 0.0f;
    for (int a = 0; a < A; ++a) s += dz[a * K + k];
    const float mean = A2C_DIV(s, (float)A);
    for (int a = 0; a < A; ++a) dz[a * K + k] = A2C_SUB(dz[a * K + k], mean);
    dz[A * K + k] = s;
  }
}

// element e of the gradient of arena tensor (l, what): dW / db from the gradient copy, times epsilon for the sigmas
template <bool NOISY>
A2C_FN float rb_grad(const A2cShared& S, const RbNet& n, const float* f, int l, int what, int e) {
  const int in = rb_in(n, l), out = rb_out(n, l);
  const RbEff ef = rb_eff(n, l);
  const float* fi = f + (NOISY ? rb_noise_off(n, l) : 0);
  if (what < 2) {
    const int j = e / in, k = e - j * in;
    const float g = S.G[ef.w + j * ef.ldw + k];
    return what == 1 ? A2C_MUL(g, A2C_MUL(fi[in + j], fi[k])) : g;
  }
  const float g = S.G[ef.b + e];
  return what == 3 ? A2C_MUL(g, fi[in + out + e]) : g;
}

// chunk c of the gradient (network.parameters() order, A2C_CHUNK elements of one tensor per chunk): its sum of squares
template <bool NOISY>
A2C_FN void ph_rb_norm(A2cShared& S, const RbNet& n, const float* f, int tid, int NT) {
  const int per = NOISY ? 4 : 2;
  for (int c = tid; c < S.nchunks; c += NT) {
    int p = 0, c0 = 0, l = 0, what = 0, ne = 0;
    for (;; ++p) {
      l = rb_param_layer(p / per);
      what = rb_what<NOISY>(p % per);
      ne = rb_numel(n, l, what);
      const int nc = (ne + b2rl_a2c::A2C_CHUNK - 1) / b2rl_a2c::A2C_CHUNK;
      if (c < c0 + nc) break;
      c0 += nc;
    }
    const int e0 = (c - c0) * b2rl_a2c::A2C_CHUNK;
    float s = 0.0f;
    for (int e = e0; e < ne && e < e0 + b2rl_a2c::A2C_CHUNK; ++e) {
      const float g = rb_grad<NOISY>(S, n, f, l, what, e);
      s = fmaf(g, g, s);
    }
    S.part[c] = s;
  }
}

// clip_grad_norm_ and RMSprop (ph_rmsprop's arithmetic) on every arena tensor; mu and sigma are read from the arena
template <bool NOISY>
A2C_FN void ph_rb_rmsprop(A2cShared& S, const RbNet& n, const b2rl_a2c::A2cArgs& a, const float* f, int tid, int NT) {
  const float norm = sqrtf(b2rl_a2c::sum4(S.part, S.nchunks));
  const float coef = a.max_norm > 0.0f ? fminf(a.max_norm / (norm + 1e-6f), 1.0f) : 1.0f;
  for (int i = 0; i < rb_ntensors<NOISY>(); ++i) {
    const int l = rb_layer<NOISY>(i), what = rb_what<NOISY>(i), ne = rb_numel(n, l, what), o = n.off[i];
    for (int e = tid; e < ne; e += NT)
      n.flat[o + e] = b2rl_elem::rmsprop_elem(n.flat[o + e], rb_grad<NOISY>(S, n, f, l, what, e) * coef, a.sq, a.ga,
                                              (int64_t)o + e, a.lr, a.alpha, a.eps, a.centered);
  }
  if (tid == 0) {
    *a.step += 1;
    *a.loss = S.scal[0];
  }
}

}  // namespace b2rl_rainbow
