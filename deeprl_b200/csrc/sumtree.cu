// sumtree.cu -- the prioritized-replay sum tree, resident in HBM, bit-identical to the reference.
// Reference: deep_rl/utils/sum_tree.py:6-67, deep_rl/component/replay.py:152-196.  sm_90a only.
//
// tree: float64 [2*cap-1] array heap (root 0, children 2i+1 / 2i+2, leaves [cap-1, 2cap-2]).
// The reference NEVER recomputes an internal node from its children: update() adds the same float64
// `change` to every ancestor, one += per node, in call order (sum_tree.py:16-20,58-60).  The bits of
// an internal node therefore depend on the ORDER of the additions it received.  A batch of B updates
// is applied here as
//   prep      (B threads)    first-occurrence + pending guard, change_i = p_i - leaf_i, leaf write
//   propagate (one CTA per tree DEPTH, B threads)   thread i owns node(depth, i) iff it is the first
//             row of the batch touching that node; it folds the changes of all later rows touching
//             the same node IN BATCH ORDER in a register (a chain of float64 adds), then stores.
// Different nodes are independent, so this is exactly the reference's sequence of additions per node.
#include "common.cuh"

namespace b2rl {

constexpr int ST_MAX_B = 1024;

// ancestor k (k >= 1) of heap node x: ((x+1) >> k) - 1; exists while (x+1) >> k >= 1
__device__ __forceinline__ int64_t ancestor(int64_t x, int k) { return ((x + 1) >> k) - 1; }

// mode 0: update_priorities rows (tree_idx given, float32 priorities, pending guard)
// mode 1: n x add(max_priority) at the write cursor
__global__ void __launch_bounds__(ST_MAX_B) sumtree_prep_kernel(double* __restrict__ tree, uint8_t* __restrict__ pending,
                                                                int64_t cap, const int64_t* __restrict__ tree_idx,
                                                                const float* __restrict__ prio, int B,
                                                                double* __restrict__ max_priority,
                                                                int64_t* __restrict__ ring_state, int mode,
                                                                double* __restrict__ change_out,
                                                                int64_t* __restrict__ idx_out) {
  __shared__ int64_t sidx[ST_MAX_B];
  __shared__ double red[32];
  const int i = threadIdx.x;
  int64_t idx = -1;
  double p = 0.0;
  if (i < B) {
    if (mode == 0) {
      idx = tree_idx[i];
      p = (double)prio[i];
      if (idx < cap - 1 || idx > 2 * cap - 2) idx = -1;   // not a leaf: the reference would corrupt the heap; we skip
    } else {
      idx = (ring_state[3] + i) % cap + cap - 1;          // sum_tree.py:40
      p = *max_priority;                                  // replay.py:162
    }
  }
  sidx[i] = idx;
  __syncthreads();
  bool active = false;
  if (i < B && idx >= 0) {
    if (mode == 0) {
      active = pending[idx - (cap - 1)] != 0;             // sum_tree.py:55-56
      for (int j = 0; j < i && active; ++j) active = sidx[j] != idx;   // an earlier row consumed the pending flag
    } else {
      active = true;                                      // add() marks the leaf pending itself (sum_tree.py:41)
    }
  }
  // max_priority = max(max_priority, p) over ALL rows, guarded or not (replay.py:195)
  if (mode == 0) {
    double m = block_reduce((i < B) ? p : -1e300, OpMax(), -1e300, red);
    if (i == 0 && m > *max_priority) *max_priority = m;
  }
  __syncthreads();
  double change = 0.0;
  if (active) {
    change = __dsub_rn(p, tree[idx]);                     // sum_tree.py:58
    tree[idx] = p;                                        // sum_tree.py:59
    pending[idx - (cap - 1)] = 0;                         // sum_tree.py:57
  }
  if (i < B) {
    change_out[i] = change;
    idx_out[i] = active ? idx : -1;
  }
  if (mode == 1 && i == 0) ring_state[3] = (ring_state[3] + B) % cap;   // sum_tree.py:48-50
}

__global__ void __launch_bounds__(ST_MAX_B) sumtree_propagate_kernel(double* __restrict__ tree,
                                                                     const double* __restrict__ change,
                                                                     const int64_t* __restrict__ idx, int B) {
  // One CTA per tree DEPTH d (root = depth 0): with a non-power-of-two capacity the leaves sit on two depths, so
  // the ancestor of row i at depth d is k_i = depth(leaf_i) - d levels up.  Indexing CTAs by depth (not by k)
  // guarantees that every node is owned by exactly one CTA.
  __shared__ int64_t node[ST_MAX_B];
  __shared__ double ch[ST_MAX_B];
  const int d = blockIdx.x;
  const int i = threadIdx.x;
  int64_t mine = -1;
  if (i < B) {
    int64_t x = idx[i];
    if (x >= 0) {
      const int depth = 63 - __clzll((unsigned long long)(x + 1));   // bitlength(x+1) - 1
      const int k = depth - d;
      if (k >= 1) mine = ancestor(x, k);
    }
    ch[i] = change[i];
  }
  node[i] = mine;
  __syncthreads();
  if (mine < 0) return;
  for (int j = 0; j < i; ++j)
    if (node[j] == mine) return;    // an earlier row owns this node
  double acc = tree[mine];
  for (int j = i; j < B; ++j)
    if (node[j] == mine) acc = __dadd_rn(acc, ch[j]);   // self.tree[parent] += change, batch order
  tree[mine] = acc;
}

// --------------------------------------------------------------------------------------------- sample
__device__ __forceinline__ bool per_valid_index(int64_t i, int64_t pos, int64_t size, int hl, int n) {
  if (i - hl + 1 >= 0 && i + n < pos) return true;
  if (i - hl + 1 >= pos && i + n < size) return true;
  return false;
}

__global__ void __launch_bounds__(ST_MAX_B) sumtree_sample_kernel(const double* __restrict__ tree,
                                                                  uint8_t* __restrict__ pending, int64_t cap,
                                                                  int64_t* __restrict__ ring_state,
                                                                  const double* __restrict__ uniforms,
                                                                  const int64_t* __restrict__ fills, uint64_t seed,
                                                                  int hl, int n, int B, int64_t* __restrict__ tidx_out,
                                                                  int64_t* __restrict__ didx_out,
                                                                  double* __restrict__ prob_out,
                                                                  int32_t* __restrict__ status) {
  __shared__ int64_t s_t[ST_MAX_B];
  __shared__ double s_p[ST_MAX_B];
  __shared__ int warp_tot[32];
  __shared__ int n_valid;
  const int i = threadIdx.x, lane = i & 31, w = i >> 5;
  const int64_t pos = ring_state[0], size = ring_state[1], ntree = 2 * cap - 1;
  const uint64_t ctr = (uint64_t)ring_state[4];
  const double total = tree[0];
  int v = 0;
  int64_t idx = 0;
  double prob = 0.0;
  if (i < B) {
    // replay.py:168-174 with CPython's random.uniform(a, b) = a + (b - a) * random()
    const double seg = __ddiv_rn(total, (double)B);
    const double a = __dmul_rn(seg, (double)i), bb = __dmul_rn(seg, (double)(i + 1));
    const double u = uniforms ? uniforms[i] : Philox::u53(seed, ctr + i, 2);
    double s = __dadd_rn(a, __dmul_rn(__dsub_rn(bb, a), u));
    // sum_tree.py:23-33
    while (true) {
      int64_t left = 2 * idx + 1;
      if (left >= ntree) break;
      double tl = tree[left];
      if (s <= tl) idx = left;
      else { s = __dsub_rn(s, tl); idx = left + 1; }
    }
    const int64_t data = idx - cap + 1;
    pending[data] = 1;                                    // sum_tree.py:66
    prob = __ddiv_rn(tree[idx], total);                   // replay.py:180
    v = per_valid_index(data, pos, size, hl, n) ? 1 : 0;  // construct_transition -> None when invalid
  }
  // order-preserving compaction of the valid rows
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_tot[w] = incl;
  __syncthreads();
  if (w == 0) {
    int x = warp_tot[lane], s2 = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, s2, o);
      if (lane >= o) s2 += y;
    }
    warp_tot[lane] = s2 - x;
    if (lane == 31) n_valid = s2;
  }
  __syncthreads();
  if (v) {
    int r = warp_tot[w] + incl - 1;
    s_t[r] = idx;
    s_p[r] = prob;
  }
  __syncthreads();
  if (i == 0) {
    int len = n_valid;
    status[0] = len;
    status[1] = 0;
    // replay.py:184-186: while len(sampled_data) < batch_size: sampled_data.append(random.choice(sampled_data))
    int k = 0;
    while (len > 0 && len < B) {
      int64_t pick = fills ? (fills[k] % len) : (int64_t)Philox::below(seed, ctr + B + k, 3, (uint64_t)len);
      s_t[len] = s_t[pick];
      s_p[len] = s_p[pick];
      ++len; ++k;
    }
    if (!uniforms || !fills) ring_state[4] = (int64_t)(ctr + 2ull * B);
  }
  __syncthreads();
  // With no valid draw the reference has nothing to back-fill from (random.choice raises).  The consumers (gather, conv1's
  // ring reads) use the outputs without a host check inside a captured graph, so they must still hold valid indices: as in
  // select_uniform_kernel, every row gets the smallest data index that cannot read below the ring (hl - 1), its leaf and that
  // leaf's probability.  status[0] = 0 tells the host check.
  if (i < B) {
    const int64_t t = n_valid > 0 ? s_t[i] : (int64_t)(hl - 1) + cap - 1;
    tidx_out[i] = t;
    didx_out[i] = t - cap + 1;
    prob_out[i] = n_valid > 0 ? s_p[i] : __ddiv_rn(tree[t], total);
  }
}

// SumTree.get for explicit prefix values (sum_tree.py:63-67), one thread per query
__global__ void sumtree_get_kernel(const double* __restrict__ tree, uint8_t* __restrict__ pending, int64_t cap,
                                   const double* __restrict__ prefix, int B, int64_t* __restrict__ tidx_out,
                                   double* __restrict__ prio_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  const int64_t ntree = 2 * cap - 1;
  double s = prefix[i];
  int64_t idx = 0;
  while (true) {
    int64_t left = 2 * idx + 1;
    if (left >= ntree) break;
    double tl = tree[left];
    if (s <= tl) idx = left;
    else { s = __dsub_rn(s, tl); idx = left + 1; }
  }
  pending[idx - cap + 1] = 1;
  tidx_out[i] = idx;
  prio_out[i] = tree[idx];
}

}  // namespace b2rl

using namespace b2rl;

static int tree_levels(int64_t cap) {
  // number of internal depths (0 .. depth(deepest leaf) - 1): bitlength(2cap-1) - 1
  int bl = 0;
  for (uint64_t x = (uint64_t)(2 * cap - 1); x; x >>= 1) ++bl;
  return bl - 1;
}

extern "C" int b2rl_sumtree_add(double* tree, uint8_t* pending, int64_t capacity, int64_t* ring_state,
                                const double* max_priority, int32_t n, double* scratch, void* stream) {
  B2RL_REQUIRE(tree && pending && ring_state && max_priority && scratch, "null pointer");
  B2RL_REQUIRE(capacity >= 2, "capacity must be >= 2 (the reference recurses forever at 1)");
  B2RL_REQUIRE(n >= 0 && n <= ST_MAX_B && n <= capacity, "n must be in [0, min(1024, capacity)]");
  if (n == 0) return B2RL_OK;
  cudaStream_t st = (cudaStream_t)stream;
  double* change = scratch;
  int64_t* idx = reinterpret_cast<int64_t*>(scratch + n);
  sumtree_prep_kernel<<<1, ST_MAX_B, 0, st>>>(tree, pending, capacity, nullptr, nullptr, n,
                                              const_cast<double*>(max_priority), ring_state, 1, change, idx);
  int rc = check_launch("b2rl_sumtree_add/prep");
  if (rc) return rc;
  sumtree_propagate_kernel<<<tree_levels(capacity), ST_MAX_B, 0, st>>>(tree, change, idx, n);
  return check_launch("b2rl_sumtree_add/propagate");
}

extern "C" int b2rl_sumtree_update(double* tree, uint8_t* pending, int64_t capacity, const int64_t* tree_idx,
                                   const float* priority, int32_t B, double* max_priority, void* scratch,
                                   void* stream) {
  B2RL_REQUIRE(tree && pending && tree_idx && priority && max_priority && scratch, "null pointer");
  B2RL_REQUIRE(capacity >= 2, "capacity must be >= 2");
  B2RL_REQUIRE(B > 0 && B <= ST_MAX_B, "B must be in [1, 1024]");
  cudaStream_t st = (cudaStream_t)stream;
  double* change = reinterpret_cast<double*>(scratch);
  int64_t* idx = reinterpret_cast<int64_t*>(change + B);
  sumtree_prep_kernel<<<1, ST_MAX_B, 0, st>>>(tree, pending, capacity, tree_idx, priority, B, max_priority, nullptr, 0,
                                              change, idx);
  int rc = check_launch("b2rl_sumtree_update/prep");
  if (rc) return rc;
  sumtree_propagate_kernel<<<tree_levels(capacity), ST_MAX_B, 0, st>>>(tree, change, idx, B);
  return check_launch("b2rl_sumtree_update/propagate");
}

extern "C" int b2rl_sumtree_sample(const double* tree, uint8_t* pending, int64_t capacity, int64_t* ring_state,
                                   const double* uniforms, const int64_t* fills, uint64_t seed, int32_t history,
                                   int32_t n_step, int32_t B, int64_t* tree_idx_out, int64_t* data_idx_out,
                                   double* sampling_prob_out, int32_t* status_out, void* stream) {
  B2RL_REQUIRE(tree && pending && ring_state && tree_idx_out && data_idx_out && sampling_prob_out && status_out,
               "null pointer");
  B2RL_REQUIRE(capacity >= 2, "capacity must be >= 2");
  B2RL_REQUIRE(B > 0 && B <= ST_MAX_B, "B must be in [1, 1024]");
  B2RL_REQUIRE(history >= 1 && history <= capacity, "history must be in [1, capacity]");
  sumtree_sample_kernel<<<1, ST_MAX_B, 0, (cudaStream_t)stream>>>(tree, pending, capacity, ring_state, uniforms, fills,
                                                                  seed, history, n_step, B, tree_idx_out, data_idx_out,
                                                                  sampling_prob_out, status_out);
  return check_launch("b2rl_sumtree_sample");
}

extern "C" int b2rl_sumtree_get(const double* tree, uint8_t* pending, int64_t capacity, const double* prefix, int32_t B,
                                int64_t* tree_idx_out, double* priority_out, void* stream) {
  B2RL_REQUIRE(tree && pending && prefix && tree_idx_out && priority_out, "null pointer");
  B2RL_REQUIRE(capacity >= 2 && B > 0, "bad shape");
  sumtree_get_kernel<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(tree, pending, capacity, prefix, B,
                                                                        tree_idx_out, priority_out);
  return check_launch("b2rl_sumtree_get");
}
