// reagent_b200 -- device-resident replay bookkeeping (SURVEY.md 8f rank 1): batched `add`,
// `set_priority` and the prioritized index draw, all on the GPU, so that an online loop
// (add one transition -> draw a minibatch -> train) is ONE CUDA-graph replay per step with the
// new transition as its only host->device traffic.
//
// Restates, with identical results (tests compare against the host path and the reference's
// golden vectors):
//   ReplayBuffer.add / _add_transition, validity bookkeeping
//                                    reagent/replay_memory/circular_replay_buffer.py:468-547, :430-438
//   PrioritizedReplayBuffer._add     reagent/replay_memory/prioritized_replay_buffer.py:62-84
//   SumTree.set (sequential fp64 delta propagation)        reagent/replay_memory/sum_tree.py:164-189
//   SumTree.stratified_sample / sample                     sum_tree.py:93-153
//   PrioritizedReplayBuffer.sample_index_batch (retries)   prioritized_replay_buffer.py:86-115
//   random.uniform / random.random of CPython (MT19937, Modules/_randommodule.c; the generator
//   is not part of the reference repo -- the stdlib module the reference calls at
//   sum_tree.py:113,152): state kept ON THE DEVICE in CPython's own layout (624 words +
//   position), uploaded from / downloaded to `random.getstate()` by the host wrapper.
//
// The add and draw kernels are single-CTA: the work is a few microseconds of latency-bound
// sequential-semantics bookkeeping.  The batched SumTree.set runs one CTA per tree level.
#include "rb200_common.cuh"

namespace rb200 {

constexpr int kMtN = 624, kMtM = 397;

__device__ __forceinline__ uint32_t mt_temper(uint32_t y) {
  y ^= (y >> 11);
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= (y >> 18);
  return y;
}
__device__ __forceinline__ uint32_t mt_mix(uint32_t cur, uint32_t nxt, uint32_t far_) {
  const uint32_t y = (cur & 0x80000000u) | (nxt & 0x7fffffffu);
  return far_ ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}

// state regeneration by the whole CTA (>= 256 threads): three phases whose reads all precede
// their writes (compute -> barrier -> store), then the last word
__device__ void mt_twist_block(uint32_t* s) {
  const int tid = threadIdx.x, nt = blockDim.x;
  uint32_t v[3];
  const int lo[3] = {0, kMtN - kMtM, 2 * (kMtN - kMtM)}, hi[3] = {kMtN - kMtM, 2 * (kMtN - kMtM), kMtN - 1};
  for (int ph = 0; ph < 3; ++ph) {
    int cnt = 0;
    for (int k = lo[ph] + tid; k < hi[ph]; k += nt)
      v[cnt++] = mt_mix(s[k], s[k + 1], ph == 0 ? s[k + kMtM] : s[k + (kMtM - kMtN)]);
    __syncthreads();
    cnt = 0;
    for (int k = lo[ph] + tid; k < hi[ph]; k += nt) s[k] = v[cnt++];
    __syncthreads();
  }
  if (tid == 0) s[kMtN - 1] = mt_mix(s[kMtN - 1], s[0], s[kMtM - 1]);
  __syncthreads();
}
// the same by ONE thread (retry path: a handful of extra draws after the stratified ones)
__device__ void mt_twist_serial(uint32_t* s) {
  int k = 0;
  for (; k < kMtN - kMtM; ++k) s[k] = mt_mix(s[k], s[k + 1], s[k + kMtM]);
  for (; k < kMtN - 1; ++k) s[k] = mt_mix(s[k], s[k + 1], s[k + (kMtM - kMtN)]);
  s[kMtN - 1] = mt_mix(s[kMtN - 1], s[0], s[kMtM - 1]);
}
// random.random(): 53-bit double in [0, 1) from two outputs (a >> 5, b >> 6)
__device__ __forceinline__ double mt_double(uint32_t a, uint32_t b) {
  return __dmul_rn(__dadd_rn(__dmul_rn((double)(a >> 5), 67108864.0), (double)(b >> 6)),
                   1.0 / 9007199254740992.0);
}

// SumTree.sample's descent (sum_tree.py:112-131) for a query already scaled by the root
__device__ __forceinline__ long long tree_walk(const double* __restrict__ tree, const double* top,
                                               int top_levels, int depth, double q) {
  long long node = 0;
  for (int lvl = 1; lvl <= depth; ++lvl) {
    const long long left = node * 2;
    const long long pos = ((1ll << lvl) - 1) + left;
    const double left_sum = (lvl < top_levels) ? top[pos] : __ldcg(tree + pos);
    if (q < left_sum) {
      node = left;
    } else {
      node = left + 1;
      q -= left_sum;
    }
  }
  return node;
}

constexpr int kDrawThreads = 1024;
constexpr int kDrawTop = 10;       // tree levels cached in shared memory (8 KB)
constexpr int kDrawChunk = 4096;   // strata per pass (32 KB of raw outputs)
constexpr int kDrawPer = kDrawChunk / kDrawThreads;  // descents per thread, interleaved

struct DrawDev {
  rb200_per_draw_args_t a;
};

__global__ void __launch_bounds__(kDrawThreads) per_draw_indices_kernel(const DrawDev d) {
  const rb200_per_draw_args_t& a = d.a;
  __shared__ uint32_t s_mt[kMtN];
  __shared__ uint32_t s_raw[2 * kDrawChunk];
  __shared__ double s_top[(1 << kDrawTop) - 1];
  __shared__ int s_pos, s_any;
  const int tid = threadIdx.x;
  for (int i = tid; i < kMtN; i += kDrawThreads) s_mt[i] = a.mt_state[i];
  const int top = min(a.tree_depth + 1, kDrawTop);
  for (int i = tid; i < (1 << top) - 1; i += kDrawThreads) s_top[i] = __ldcg(a.tree + i);
  if (tid == 0) { s_pos = (int)a.mt_state[kMtN]; s_any = 0; }
  __syncthreads();
  const double root = s_top[0];
  int pos = s_pos;
  bool any_invalid = false;
  for (int base = 0; base < a.batch; base += kDrawChunk) {
    const int m = min(kDrawChunk, a.batch - base);
    // ---- 2m tempered outputs of the stream ----
    int produced = 0;
    while (produced < 2 * m) {
      if (pos >= kMtN) { mt_twist_block(s_mt); pos = 0; }
      const int take = min(kMtN - pos, 2 * m - produced);
      for (int i = tid; i < take; i += kDrawThreads) s_raw[produced + i] = mt_temper(s_mt[pos + i]);
      pos += take;
      produced += take;
      __syncthreads();
    }
    // ---- stratified queries (sum_tree.py:149-152) and their descents: each thread walks
    // kDrawPer strata in lock-step so that their dependent loads overlap ----
    {
      double q[kDrawPer];
      long long node[kDrawPer];
      int bb[kDrawPer];
#pragma unroll
      for (int u = 0; u < kDrawPer; ++u) {
        const int i = tid + u * kDrawThreads;
        bb[u] = (i < m) ? base + i : -1;
        node[u] = 0;
        q[u] = 0.0;
        if (bb[u] >= 0) {
          const double r = mt_double(s_raw[2 * i], s_raw[2 * i + 1]);
          // random.uniform(lo, hi) = lo + (hi - lo) * random(): separately rounded operations
          const double lo = a.lo[bb[u]], hi = a.hi[bb[u]];
          const double qq = __dadd_rn(lo, __dmul_rn(__dadd_rn(hi, -lo), r));
          if (a.queries_out) a.queries_out[bb[u]] = qq;
          q[u] = __dmul_rn(qq, root);  // sum_tree.py:113
        }
      }
      for (int lvl = 1; lvl <= a.tree_depth; ++lvl) {
        double ls[kDrawPer];
#pragma unroll
        for (int u = 0; u < kDrawPer; ++u) {
          const long long p = ((1ll << lvl) - 1) + node[u] * 2;
          ls[u] = (lvl < top) ? s_top[p] : __ldcg(a.tree + p);
        }
#pragma unroll
        for (int u = 0; u < kDrawPer; ++u) {
          if (q[u] < ls[u]) {
            node[u] = node[u] * 2;
          } else {
            node[u] = node[u] * 2 + 1;
            q[u] -= ls[u];
          }
        }
      }
#pragma unroll
      for (int u = 0; u < kDrawPer; ++u) {
        if (bb[u] < 0) continue;
        a.indices_out[bb[u]] = node[u];
        if (!a.valid[node[u]]) any_invalid = true;
      }
    }
    __syncthreads();
  }
  if (any_invalid) s_any = 1;
  __syncthreads();
  // ---- retries, sequential as in prioritized_replay_buffer.py:95-113 ----
  if (tid == 0) {
    int used = 0;
    if (s_any) {
      int allowed = a.max_attempts;
      for (int b = 0; b < a.batch; ++b) {
        long long index = a.indices_out[b];
        if (a.valid[index]) continue;
        if (allowed == 0) { a.status[0] = 1; break; }  // "Max sample attempts" (sticky; host raises)
        while (!a.valid[index] && allowed > 0) {
          uint32_t w[2];
          for (int j = 0; j < 2; ++j) {
            if (pos >= kMtN) { mt_twist_serial(s_mt); pos = 0; }
            w[j] = mt_temper(s_mt[pos++]);
          }
          index = tree_walk(a.tree, s_top, top, a.tree_depth, __dmul_rn(mt_double(w[0], w[1]), root));
          --allowed;
          ++used;
        }
        a.indices_out[b] = index;
      }
    }
    a.status[1] = used;
    s_pos = pos;
  }
  __syncthreads();
  for (int i = tid; i < kMtN; i += kDrawThreads) a.mt_state[i] = s_mt[i];
  if (tid == 0) a.mt_state[kMtN] = (uint32_t)s_pos;
}

// ---------------------------------------------------------------------------
// SumTree.set of ONE transition (sum_tree.py:164-189) by one warp, for the add kernel: lane l
// owns level l of the root path
// ---------------------------------------------------------------------------
__device__ __forceinline__ void tree_set_warp(double* tree, int depth, long long leaf, double value,
                                              double* max_recorded, int lane) {
  // lane `depth` reads (and later writes) the leaf: same thread, program order
  double delta = 0.0;
  if (lane == depth) {
    delta = value - tree[((1ll << depth) - 1) + leaf];
    if (max_recorded && value > *max_recorded) *max_recorded = value;
  }
  delta = __shfl_sync(0xffffffffu, delta, depth);
  if (lane <= depth) {
    double* p = tree + ((1ll << lane) - 1) + (leaf >> (depth - lane));
    *p = __dadd_rn(*p, delta);
  }
  __syncwarp();
}

// ---------------------------------------------------------------------------
// SumTree.set for a batch, applied IN ORDER (sum_tree.py:164-189), bit-equal to the sequential
// loop.  Set k adds delta_k = v_k - (its leaf before set k) to every node on its root path, so a
// node's final value is its old value plus ITS deltas folded in k order.  Nodes are independent,
// which regroups the work without reassociating any fp64 sum:
//   deltas  sort the sets by (leaf, k); one thread folds each leaf's run in k order
//   levels  one CTA per inner level sorts the sets by (node, k) and folds each node's run
// The levels kernel reads the leaves and the leaf kernel then writes them (with max_recorded and
// the status word): two launches per chunk of kSetChunk sets, chunks in order.  The critical path
// is the root's fold, one dependent fp64 add per set.
// ---------------------------------------------------------------------------
constexpr int kSetThreads = 1024;
constexpr int kSetKBits = 12;
constexpr int kSetChunk = 1 << kSetKBits;
constexpr int kSetPer = kSetChunk / kSetThreads;
constexpr size_t kSetSmem = (size_t)kSetChunk * (sizeof(unsigned long long) + sizeof(double));

struct SetSrc {
  const long long* idx;      // [n] leaf of set i
  const double* val;         // [n] the values (set_priority), or NULL: PER priorities
  const float* td_target;    // [n]  p_i = ((double)|q_selected_i - td_target_i| + eps) ** alpha
  const float* q_selected;   // [n]
  const float* row_loss;     // [n] or NULL:  p_i = ((double)|row_loss_i| / divisor + eps) ** alpha
  double divisor;
  double alpha, eps;
  double* p_out;             // [n] or NULL: the values, written by the leaf kernel
  int n;
  bool per;                  // val path with PER semantics: a non-finite value applies none
};

__device__ __forceinline__ double set_value(const SetSrc& s, int i) {
  if (s.val) return s.val[i];
  const double e = s.row_loss ? __ddiv_rn(fabs((double)s.row_loss[i]), s.divisor)
                              : (double)fabsf(__fsub_rn(s.q_selected[i], s.td_target[i]));
  return pow(__dadd_rn(e, s.eps), s.alpha);
}

// How many sets apply: all, up to the first negative value (sum_tree.py raises there, after the
// earlier sets), or none when a PER priority is not finite.  *code = the status it sets (0, 2, 3).
__device__ int sets_applied(const SetSrc& s, int* code) {
  __shared__ int s_neg, s_bad;
  if (threadIdx.x == 0) { s_neg = s.n; s_bad = 0; }
  __syncthreads();
  int neg = s.n;
  bool bad = false;
  for (int i = threadIdx.x; i < s.n; i += blockDim.x) {
    const double v = set_value(s, i);
    if (v < 0.0 && i < neg) neg = i;
    if ((!s.val || s.per) && !isfinite(v)) bad = true;
  }
  if (neg < s.n) atomicMin(&s_neg, neg);
  if (bad) s_bad = 1;
  __syncthreads();
  *code = s_bad ? 3 : (s_neg < s.n ? 2 : 0);
  return s_bad ? 0 : s_neg;
}

// ascending bitonic sort of key[0, m) by the whole CTA (m <= kSetChunk)
__device__ void block_sort_u64(unsigned long long* key, int m) {
  int np = 1;
  while (np < m) np <<= 1;
  for (int i = m + threadIdx.x; i < np; i += blockDim.x) key[i] = ~0ull;
  __syncthreads();
  for (int size = 2; size <= np; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < np / 2; t += blockDim.x) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const unsigned long long x = key[lo], y = key[hi];
        if ((x > y) == ((lo & size) == 0)) { key[lo] = y; key[hi] = x; }
      }
      __syncthreads();
    }
  }
}

// end of the run of sorted key[j] that shares its group (key >> kSetKBits): binary search
__device__ __forceinline__ int run_end(const unsigned long long* key, int j, int m) {
  const unsigned long long lim = ((key[j] >> kSetKBits) + 1) << kSetKBits;
  int lo = j + 1, hi = m;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (key[mid] < lim) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Sets [c0, c0 + m) of the chunk: vals[k] <- delta_k (k = i - c0), each leaf's run folded in k
// order from its value in the tree; with write_leaves the leaves take their final values
__device__ void chunk_deltas(const SetSrc& s, double* leaves, int c0, int m,
                             unsigned long long* key, double* vals, bool write_leaves) {
  for (int k = threadIdx.x; k < m; k += blockDim.x) {
    vals[k] = set_value(s, c0 + k);
    key[k] = ((unsigned long long)s.idx[c0 + k] << kSetKBits) | (unsigned long long)k;
  }
  block_sort_u64(key, m);
  for (int j = threadIdx.x; j < m; j += blockDim.x) {
    const unsigned long long leaf = key[j] >> kSetKBits;
    if (j > 0 && (key[j - 1] >> kSetKBits) == leaf) continue;
    const int e = run_end(key, j, m);
    double cur = leaves[leaf];
    for (int r = j; r < e; ++r) {
      const int k = (int)(key[r] & (kSetChunk - 1));
      const double d = __dadd_rn(vals[k], -cur);  // sum_tree.py: delta = value - leaf
      vals[k] = d;
      cur = __dadd_rn(cur, d);
    }
    if (write_leaves) leaves[leaf] = cur;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kSetThreads) sumtree_levels_kernel(double* tree, int depth,
                                                                     const SetSrc s, int c0) {
  extern __shared__ __align__(16) unsigned long long set_smem[];
  unsigned long long* key = set_smem;
  double* vals = reinterpret_cast<double*>(set_smem + kSetChunk);
  int code;
  const int m = min(kSetChunk, sets_applied(s, &code) - c0);
  if (m <= 0) return;
  chunk_deltas(s, tree + ((1ll << depth) - 1), c0, m, key, vals, false);
  const int lvl = blockIdx.x, shift = depth - lvl;
  for (int k = threadIdx.x; k < m; k += blockDim.x)
    key[k] = ((unsigned long long)(s.idx[c0 + k] >> shift) << kSetKBits) | (unsigned long long)k;
  block_sort_u64(key, m);
  // deltas into sorted order (all reads before any write), so that each fold reads a contiguous run
  double dv[kSetPer];
#pragma unroll
  for (int u = 0; u < kSetPer; ++u) {
    const int j = threadIdx.x + u * kSetThreads;
    if (j < m) dv[u] = vals[key[j] & (kSetChunk - 1)];
  }
  __syncthreads();
#pragma unroll
  for (int u = 0; u < kSetPer; ++u) {
    const int j = threadIdx.x + u * kSetThreads;
    if (j < m) vals[j] = dv[u];
  }
  __syncthreads();
  double* level = tree + ((1ll << lvl) - 1);
  for (int j = threadIdx.x; j < m; j += blockDim.x) {
    const unsigned long long node = key[j] >> kSetKBits;
    if (j > 0 && (key[j - 1] >> kSetKBits) == node) continue;
    const int e = run_end(key, j, m);
    double acc = level[node];
#pragma unroll 8
    for (int r = j; r < e; ++r) acc = __dadd_rn(acc, vals[r]);
    level[node] = acc;
  }
}

__global__ void __launch_bounds__(kSetThreads) sumtree_leaves_kernel(double* tree, int depth,
                                                                     const SetSrc s, int c0,
                                                                     double* max_recorded,
                                                                     int* status) {
  extern __shared__ __align__(16) unsigned long long set_smem[];
  unsigned long long* key = set_smem;
  double* vals = reinterpret_cast<double*>(set_smem + kSetChunk);
  __shared__ double s_best[kSetThreads / 32];
  __shared__ int s_bestk[kSetThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int code;
  const int applied = sets_applied(s, &code);
  const int c1 = min(c0 + kSetChunk, s.n);
  if (s.p_out)
    for (int i = c0 + tid; i < c1; i += blockDim.x) s.p_out[i] = set_value(s, i);
  if (c0 == 0 && code && status && tid == 0) status[0] = code;
  const int m = min(kSetChunk, applied - c0);
  if (m <= 0) return;
  if (max_recorded) {
    // the sequential "if value > max_recorded" keeps the FIRST set holding the largest value
    double best = -INFINITY;
    int bk = 0x7fffffff;
    for (int k = tid; k < m; k += blockDim.x) {
      const double v = set_value(s, c0 + k);
      if (v > best) { best = v; bk = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
      if (ok != 0x7fffffff && (bk == 0x7fffffff || ob > best || (ob == best && ok < bk))) { best = ob; bk = ok; }
    }
    if (lane == 0) { s_best[warp] = best; s_bestk[warp] = bk; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < kSetThreads / 32; ++w) {
        const double ob = s_best[w];
        const int ok = s_bestk[w];
        if (ok != 0x7fffffff && (bk == 0x7fffffff || ob > best || (ob == best && ok < bk))) { best = ob; bk = ok; }
      }
      if (bk != 0x7fffffff && best > *max_recorded) *max_recorded = best;
    }
  }
  chunk_deltas(s, tree + ((1ll << depth) - 1), c0, m, key, vals, true);
}

static int sumtree_update(double* tree, int depth, const SetSrc& s, double* max_recorded,
                          int* status, cudaStream_t st) {
  cudaError_t e = opt_in_smem<sumtree_levels_kernel>(kSetSmem);
  if (e == cudaSuccess) e = opt_in_smem<sumtree_leaves_kernel>(kSetSmem);
  if (e != cudaSuccess) return check_cuda(e, "cudaFuncSetAttribute(sumtree)");
  for (int c0 = 0; c0 < s.n; c0 += kSetChunk) {
    if (depth > 0) sumtree_levels_kernel<<<depth, kSetThreads, kSetSmem, st>>>(tree, depth, s, c0);
    sumtree_leaves_kernel<<<1, kSetThreads, kSetSmem, st>>>(tree, depth, s, c0, max_recorded, status);
  }
  return check_cuda(cudaGetLastError(), "sumtree update launch");
}

// ---------------------------------------------------------------------------
// Data-parallel priority exchange (rb200_per_exchange_args_t): one CTA computes this rank's
// priorities with set_value, pushes them into every rank's receive buffer, then flags / waits
// as adam_soft_kernel does and copies the gathered vector out.  A few KB per update: the
// single CTA's latency is well under the tree update that follows it.
// ---------------------------------------------------------------------------
constexpr int kExchangeThreads = 1024;

struct ExchangeDev {
  rb200_per_exchange_args_t a;
};

__global__ void __launch_bounds__(kExchangeThreads) per_priority_exchange_kernel(const ExchangeDev d) {
  const rb200_per_exchange_args_t& a = d.a;
  SetSrc s = {};
  s.td_target = a.td_target;
  s.q_selected = a.q_selected;
  s.row_loss = a.row_loss;
  s.divisor = a.divisor;
  s.alpha = a.alpha;
  s.eps = a.eps;
  const int W = a.world, tid = threadIdx.x;
  if (W == 1) {
    for (int i = tid; i < a.n_local; i += kExchangeThreads) a.out[a.row0 + i] = set_value(s, i);
    return;
  }
  const uint32_t t = *a.epoch + 1u;
  const size_t par = t & 1u;
  const size_t slot = par * (size_t)a.B_global + a.row0;
  for (int i = tid; i < a.n_local; i += kExchangeThreads) {
    const double p = set_value(s, i);
    for (int r = 0; r < W; ++r) a.recv[r][slot + i] = p;  // own copy included
  }
  __syncthreads();
  if (tid == 0) {
    // one system-scope fence orders every push of the CTA (made visible to this thread by the
    // barrier) before the flags, which are then relaxed stores posted back to back
    __threadfence_system();
    for (int r = 0; r < W; ++r) {
      if (r == a.rank) continue;
      uint32_t* f = a.flags[r] + par * W + a.rank;
      asm volatile("st.relaxed.sys.global.u32 [%0], %1;\n" ::"l"(f), "r"(t) : "memory");
    }
  }
  if (tid < W && tid != a.rank) {
    const uint32_t* w = a.flags[a.rank] + par * W + tid;
    unsigned long long t0 = 0, now = 0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (;;) {
      uint32_t v;
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(w) : "memory");
      if (v == t) break;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
      if (now - t0 > 4000000000ull) __trap();  // 4 s: a lost peer fails the step, never hangs
    }
  }
  __syncthreads();
  const double* mine = a.recv[a.rank] + par * (size_t)a.B_global;
  for (int i = tid; i < a.B_global; i += kExchangeThreads) a.out[i] = __ldcg(mine + i);
  if (tid == 0) *a.epoch = t;
}

// ---------------------------------------------------------------------------
// PER importance weights (Schaul et al. 2016, normalised by the batch maximum as in Dopamine):
// w_i = (p_min / p_i) ** beta_t over the drawn leaves p_i; a zero leaf gets weight 0 and no say
// in p_min.  beta_t = min(1, beta0 + (1 - beta0) * t / beta_updates), t = *step.
// ---------------------------------------------------------------------------
constexpr int kWeightThreads = 1024;

__global__ void __launch_bounds__(kWeightThreads) per_weights_kernel(
    const double* tree, int depth, const long long* idx, int n, const long long* step,
    double beta0, double beta_updates, float* w, double* w64) {
  __shared__ double s_min[kWeightThreads / 32];
  const double* leaves = tree + ((1ll << depth) - 1);
  const int tid = threadIdx.x;
  double mn = INFINITY;
  for (int i = tid; i < n; i += kWeightThreads) {
    const double p = leaves[idx[i]];
    if (p > 0.0) mn = fmin(mn, p);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  if ((tid & 31) == 0) s_min[tid >> 5] = mn;
  __syncthreads();
  mn = s_min[0];
  for (int k = 1; k < kWeightThreads / 32; ++k) mn = fmin(mn, s_min[k]);
  const double t = (double)*step;
  const double beta = fmin(1.0, __dadd_rn(beta0, __ddiv_rn(__dmul_rn(__dadd_rn(1.0, -beta0), t), beta_updates)));
  for (int i = tid; i < n; i += kWeightThreads) {
    const double p = leaves[idx[i]];
    const double wi = p > 0.0 ? pow(__ddiv_rn(mn, p), beta) : 0.0;
    w[i] = (float)wi;
    if (w64) w64[i] = wi;
  }
}

// ---------------------------------------------------------------------------
// n consecutive ReplayBuffer.add() calls (stack_size == 1) from device staging rows
// ---------------------------------------------------------------------------
constexpr int kAddMax = 1024;

struct AddDev {
  rb200_add_args_t a;
};

__global__ void __launch_bounds__(256) replay_add_kernel(const AddDev d) {
  const rb200_add_args_t& a = d.a;
  const rb200_replay_dev_t& rb = a.rb;
  __shared__ long long s_cur[kAddMax];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long cap = rb.capacity;
  if (tid == 0) {
    // circular_replay_buffer.py:468-522 with stack_size == 1 (no padding transitions)
    long long add_count = rb.state[0], ep = rb.state[1], nvalid = rb.state[2];
    auto set_valid = [&](long long i, bool v) {  // set_index_valid_status, :430-438
      const bool old = rb.valid[i] != 0;
      if (old != v) { rb.valid[i] = v ? 1 : 0; nvalid += v ? 1 : -1; }
    };
    for (int t = 0; t < a.n; ++t) {
      const long long cur = add_count % cap;
      const long long last = (cur - 1 + cap) % cap;
      if (add_count == 0 || rb.terminal[last]) ep = 0;
      set_valid(cur, false);
      if (ep >= rb.update_horizon) set_valid(((cur - rb.update_horizon) % cap + cap) % cap, true);
      rb.terminal[cur] = a.terminal_in[t] ? 1 : 0;
      rb.reward[cur] = a.reward_in[t];
      s_cur[t] = cur;
      ++add_count;
      ++ep;
      if (a.terminal_in[t]) {
        const long long back = ep < rb.update_horizon ? ep : rb.update_horizon;
        for (long long k = 0; k < back; ++k) set_valid(((cur - k) % cap + cap) % cap, true);
      }
    }
    rb.state[0] = add_count;
    rb.state[1] = ep;
    rb.state[2] = nvalid;
  }
  __syncthreads();
  // priorities: prioritized_replay_buffer.py:76-84 -> SumTree.set(cursor, priority), in order
  if (warp == 0 && rb.tree && a.priority_in) {
    for (int t = 0; t < a.n; ++t) {
      double v = a.priority_in[t];
      // Schaul et al.'s rule for a transition without a priority: the largest one recorded so
      // far, read here, after the sets of the earlier transitions of this call
      if (a.priority_from_max && isnan(v)) v = *rb.max_priority;
      if (v < 0.0) { if (lane == 0) rb.state[3] = 2; break; }
      tree_set_warp(rb.tree, rb.tree_depth, s_cur[t], v, rb.max_priority, lane);
    }
  }
  // row copies (observation, action, extras): staging [n, row_bytes] -> store[cursor]
  for (int t = 0; t < a.n; ++t) {
    for (int g = 0; g < a.n_rows; ++g) {
      const rb200_gather_spec_t& sp = a.rows[g];
      const unsigned char* src = (const unsigned char*)sp.src + (size_t)t * sp.row_bytes;
      unsigned char* dst = (unsigned char*)sp.dst + (size_t)s_cur[t] * sp.row_bytes;
      if (((sp.row_bytes & 15) == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0) &&
          ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
        for (int c = tid; c < sp.row_bytes / 16; c += blockDim.x)
          reinterpret_cast<uint4*>(dst)[c] = reinterpret_cast<const uint4*>(src)[c];
      } else {
        for (int c = tid; c < sp.row_bytes; c += blockDim.x) dst[c] = src[c];
      }
    }
  }
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_per_draw_indices(const rb200_per_draw_args_t* a, void* stream) {
  if (!a || !a->mt_state || !a->lo || !a->hi || !a->tree || !a->valid || !a->indices_out || !a->status) {
    set_last_error("rb200_per_draw_indices: null argument"); return RB200_E_INVALID;
  }
  if (a->batch <= 0 || a->tree_depth < 0 || a->max_attempts < 0) { set_last_error("rb200_per_draw_indices: bad batch/depth/attempts"); return RB200_E_INVALID; }
  DrawDev d;
  d.a = *a;
  per_draw_indices_kernel<<<1, kDrawThreads, 0, (cudaStream_t)stream>>>(d);
  return check_cuda(cudaGetLastError(), "per_draw_indices_kernel launch");
}

extern "C" int rb200_sumtree_set_device(double* tree, int32_t depth, const int64_t* idx,
                                        const double* val, int32_t n, double* max_recorded,
                                        int32_t* status, void* stream) {
  if (!tree || !idx || !val || depth < 0 || depth > 31 || n < 0) { set_last_error("rb200_sumtree_set_device: bad argument"); return RB200_E_INVALID; }
  if (n == 0) return RB200_OK;
  SetSrc s = {};
  s.idx = (const long long*)idx;
  s.val = val;
  s.n = n;
  return sumtree_update(tree, depth, s, max_recorded, status, (cudaStream_t)stream);
}

extern "C" int rb200_per_priority_update(double* tree, int32_t depth, const int64_t* idx,
                                         const float* td_target, const float* q_selected,
                                         int32_t n, double alpha, double eps, double* p_out,
                                         double* max_recorded, int32_t* status, void* stream) {
  if (!tree || !idx || !td_target || !q_selected || !p_out || !status) { set_last_error("rb200_per_priority_update: null argument"); return RB200_E_INVALID; }
  if (depth < 0 || depth > 31 || n <= 0) { set_last_error("rb200_per_priority_update: bad depth/n"); return RB200_E_INVALID; }
  SetSrc s = {};
  s.idx = (const long long*)idx;
  s.td_target = td_target;
  s.q_selected = q_selected;
  s.alpha = alpha;
  s.eps = eps;
  s.p_out = p_out;
  s.n = n;
  return sumtree_update(tree, depth, s, max_recorded, status, (cudaStream_t)stream);
}

extern "C" int rb200_per_priority_update_rows(double* tree, int32_t depth, const int64_t* idx,
                                              const float* row_loss, int32_t n, double divisor,
                                              double alpha, double eps, double* p_out,
                                              double* max_recorded, int32_t* status, void* stream) {
  const char* null_arg = !tree ? "tree" : !idx ? "idx" : !row_loss ? "row_loss"
                         : !p_out ? "p_out" : !status ? "status" : nullptr;
  if (null_arg) { set_last_error("rb200_per_priority_update_rows: %s is null", null_arg); return RB200_E_INVALID; }
  if (depth < 0 || depth > 31 || n <= 0) { set_last_error("rb200_per_priority_update_rows: bad depth %d / n %d", depth, n); return RB200_E_INVALID; }
  if (!(divisor > 0.0) || !isfinite(divisor)) { set_last_error("rb200_per_priority_update_rows: divisor must be positive and finite, got %g", divisor); return RB200_E_INVALID; }
  SetSrc s = {};
  s.idx = (const long long*)idx;
  s.row_loss = row_loss;
  s.divisor = divisor;
  s.alpha = alpha;
  s.eps = eps;
  s.p_out = p_out;
  s.n = n;
  return sumtree_update(tree, depth, s, max_recorded, status, (cudaStream_t)stream);
}

extern "C" int rb200_per_priority_exchange(const rb200_per_exchange_args_t* a, void* stream) {
  if (!a) { set_last_error("rb200_per_priority_exchange: null argument"); return RB200_E_INVALID; }
  const char* null_arg = !a->out ? "out"
                         : a->row_loss ? nullptr
                         : !a->td_target ? "td_target" : !a->q_selected ? "q_selected" : nullptr;
  if (!null_arg && a->world > 1)
    null_arg = !a->recv ? "recv" : !a->flags ? "flags" : !a->epoch ? "epoch" : nullptr;
  if (null_arg) { set_last_error("rb200_per_priority_exchange: %s is null", null_arg); return RB200_E_INVALID; }
  if (a->world < 1 || a->world > 256 || a->rank < 0 || a->rank >= a->world) {
    set_last_error("rb200_per_priority_exchange: bad world %d / rank %d", a->world, a->rank);
    return RB200_E_INVALID;
  }
  if (a->n_local <= 0 || a->row0 < 0 || a->B_global <= 0 || (int64_t)a->row0 + a->n_local > a->B_global) {
    set_last_error("rb200_per_priority_exchange: rows [%d, %d + %d) outside B_global %d", a->row0,
                   a->row0, a->n_local, a->B_global);
    return RB200_E_INVALID;
  }
  if (a->row_loss && (!(a->divisor > 0.0) || !isfinite(a->divisor))) {
    set_last_error("rb200_per_priority_exchange: divisor must be positive and finite, got %g", a->divisor);
    return RB200_E_INVALID;
  }
  ExchangeDev d;
  d.a = *a;
  per_priority_exchange_kernel<<<1, kExchangeThreads, 0, (cudaStream_t)stream>>>(d);
  return check_cuda(cudaGetLastError(), "per_priority_exchange_kernel launch");
}

extern "C" int rb200_per_priority_apply(double* tree, int32_t depth, const int64_t* idx,
                                        const double* val, int32_t n, double* max_recorded,
                                        int32_t* status, void* stream) {
  const char* null_arg = !tree ? "tree" : !idx ? "idx" : !val ? "val" : !status ? "status" : nullptr;
  if (null_arg) { set_last_error("rb200_per_priority_apply: %s is null", null_arg); return RB200_E_INVALID; }
  if (depth < 0 || depth > 31 || n <= 0) { set_last_error("rb200_per_priority_apply: bad depth %d / n %d", depth, n); return RB200_E_INVALID; }
  SetSrc s = {};
  s.idx = (const long long*)idx;
  s.val = val;
  s.per = true;
  s.n = n;
  return sumtree_update(tree, depth, s, max_recorded, status, (cudaStream_t)stream);
}

extern "C" int rb200_per_weights(const double* tree, int32_t depth, const int64_t* idx, int32_t n,
                                 const int64_t* step, double beta0, double beta_updates,
                                 float* w_out, double* w64_out, void* stream) {
  if (!tree || !idx || !step || !w_out) { set_last_error("rb200_per_weights: null argument"); return RB200_E_INVALID; }
  if (depth < 0 || depth > 31 || n <= 0 || !(beta_updates > 0.0)) { set_last_error("rb200_per_weights: bad depth/n/beta_updates"); return RB200_E_INVALID; }
  per_weights_kernel<<<1, kWeightThreads, 0, (cudaStream_t)stream>>>(
      tree, depth, (const long long*)idx, n, (const long long*)step, beta0, beta_updates, w_out, w64_out);
  return check_cuda(cudaGetLastError(), "per_weights_kernel launch");
}

extern "C" int rb200_replay_add_device(const rb200_add_args_t* a, void* stream) {
  if (!a || !a->rb.state || !a->rb.valid || !a->rb.terminal || !a->rb.reward || !a->terminal_in || !a->reward_in) {
    set_last_error("rb200_replay_add_device: null argument"); return RB200_E_INVALID;
  }
  if (a->n <= 0 || a->n > kAddMax) { set_last_error("rb200_replay_add_device: n must be in [1, %d]", kAddMax); return RB200_E_INVALID; }
  if (a->rb.capacity <= 0 || a->rb.update_horizon <= 0 || a->n_rows < 0 || a->n_rows > RB200_MAX_GATHER_SPECS) { set_last_error("rb200_replay_add_device: bad capacity/horizon/rows"); return RB200_E_INVALID; }
  if (a->rb.tree && (a->rb.tree_depth < 0 || a->rb.tree_depth > 31)) { set_last_error("rb200_replay_add_device: bad tree depth"); return RB200_E_INVALID; }
  if (a->priority_from_max && (!a->rb.tree || !a->rb.max_priority)) { set_last_error("rb200_replay_add_device: priority_from_max needs the tree and max_priority"); return RB200_E_INVALID; }
  AddDev d;
  d.a = *a;
  replay_add_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(d);
  return check_cuda(cudaGetLastError(), "replay_add_kernel launch");
}
