// reagent_b200 -- loss head of SlateQTrainer (reagent/training/slate_q_trainer.py:199-276).
// The q networks around it are plain MLPs on the generic kernels: the target network scores
// every next-state candidate in one rb200_mlp_forward_tiled launch, and this head picks the next
// slate's values from those scores by index.  See include/reagent_b200.h for the contract.
#include "rb200_common.cuh"

namespace rb200 {

constexpr int kSqRows = RB200_SLATEQ_ROWS_PER_BLOCK;
constexpr int kCountThreads = 1024;

// Number of nonzero reward_mask entries.  An integer sum: the same count whatever the order.
__global__ void __launch_bounds__(kCountThreads) slateq_count_kernel(const float* rm, long long n,
                                                                     int32_t* out) {
  int c = 0;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) c += rm[i] != 0.f;
  c = __reduce_add_sync(0xffffffffu, c);
  __shared__ int s[kCountThreads / 32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kCountThreads / 32; ++w) t += s[w];
    *out = t;
  }
}

// torch's advanced indexing: an index in [-C, C) wraps into [0, C); anything else is the
// reference's IndexError, reported through `bad` (candidate 0 is used instead).
__device__ __forceinline__ int slate_index(long long v, int C, bool& bad) {
  if (v < 0) v += C;
  if (v < 0 || v >= C) {
    bad = true;
    return 0;
  }
  return (int)v;
}

// (k, i) before (bk, bi) in torch.topk's order with ties on the lowest index
__device__ __forceinline__ bool ranks_before(float k, int i, float bk, int bi) {
  return k > bk || (k == bk && i < bi);
}

__global__ void __launch_bounds__(32 * kSqRows) slateq_head_kernel(const rb200_slateq_args_t a) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.x * kSqRows + warp;
  const int C = a.num_candidates, K = a.slate_width;
  const bool single = a.single_selection != 0;
  float le = 0.f;
  if (b < a.batch) {  // whole warps: the block-level reduction below needs every thread
    const size_t cb = (size_t)b * C;
    const float* qn = a.q_next + cb;
    const float* nv = a.next_value + cb;
    const float* nm = a.next_mask + cb;
    const float nt = a.not_terminal[b];
    const bool terminal = nt == 0.f;
    const int Kn = a.maxq ? a.slate_size : a.next_width;
    bool bad = false;
    // lane j < Kn holds the candidate index of the next slate's entry j
    int idx = 0;
    if (a.maxq) {
      // _get_maxq_topk: top slate_size of q_target(s', c) * docs_value(c) over all candidates,
      // docs_value = softmax(value * mask) over C (single selection) or value * mask
      const auto dv = [nv, nm](int c) { return __fmul_rn(nv[c], nm[c]); };
      float mx = 0.f, sum = 1.f;
      if (single) warp_row_max_sumexp(dv, C, mx, sum);
      const auto key = [&](int c) {
        const float w = single ? __fdiv_rn(expf(__fsub_rn(dv(c), mx)), sum) : dv(c);
        return __fmul_rn(qn[c], w);
      };
      // entry j: the best candidate ranked after entry j - 1
      float pk = INFINITY;
      int pi = -1;
      for (int j = 0; j < Kn; ++j) {
        float bk = -INFINITY;
        int bi = C;
        for (int c = lane; c < C; c += 32) {
          const float k = key(c);
          if (ranks_before(pk, pi, k, c) && ranks_before(k, c, bk, bi)) { bk = k; bi = c; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          const float ok = __shfl_xor_sync(0xffffffffu, bk, o);
          const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
          if (ranks_before(ok, oi, bk, bi)) { bk = ok; bi = oi; }
        }
        if (lane == j) idx = bi < C ? bi : 0;  // bi == C only when every key left is NaN
        pk = bk;
        pi = bi;
      }
    } else if (lane < Kn && !terminal) {
      idx = slate_index(a.next_action[(size_t)b * Kn + lane], C, bad);
    }
    // _action_docs: a terminal row's next slate is candidate 0 (SARSA: in the caller's tensor)
    if (terminal) {
      idx = 0;
      if (!a.maxq && lane < Kn) a.next_action[(size_t)b * Kn + lane] = 0;
    }
    if (a.action && lane < K) slate_index(a.action[(size_t)b * K + lane], C, bad);
    if (bad) a.status[0] = 1;

    // sum over the next slate of q_target * docs_value(slate)
    float w = -INFINITY, q = 0.f;
    if (lane < Kn) {
      w = __fmul_rn(nv[idx], nm[idx]);
      q = qn[idx];
    }
    if (single) {
      const float m = warp_max(w);
      const float e = lane < Kn ? expf(__fsub_rn(w, m)) : 0.f;
      w = __fdiv_rn(e, warp_sum(e));
    }
    float next_q = warp_sum(lane < Kn ? __fmul_rn(q, w) : 0.f);
    if (!single) {  // _get_avg_by_slate_size: min(mask.sum(1), slate_size)
      const float* mk = (a.norm_method == RB200_SLATEQ_NORM_NEXT ? a.next_mask : a.cur_mask) + cb;
      float ms = 0.f;
      for (int c = lane; c < C; c += 32) ms += mk[c];
      next_q = __fdiv_rn(next_q, fminf(warp_sum(ms), (float)a.slate_size));
    }
    const float disc = a.time_diff ? powf(a.gamma, __fdiv_rn(a.time_diff[b], a.time_scale)) : a.gamma;
    const float future = __fmul_rn(disc, __fmul_rn(next_q, nt));
    if (lane < K) {
      const size_t e = (size_t)b * K + lane;
      const float tgt = __fadd_rn(a.reward[e], future);
      const float d = __fsub_rn(a.q_cur[e], tgt);
      // F.mse_loss: mean over the reward_mask entries or over all B * K entries
      const bool on = !single || a.reward_mask[e] != 0.f;
      const float n = single ? (float)*a.mask_count : (float)a.batch * (float)K;
      le = on ? __fmul_rn(d, d) : 0.f;
      a.dz[e] = on ? __fdiv_rn(__fmul_rn(2.f, d), n) : 0.f;
      if (a.target) a.target[e] = tgt;
    }
  }
  // deterministic mean: per-block partial of the rows in warp order, then finish_block
  __shared__ float s_l[kSqRows];
  __shared__ bool s_last;
  le = warp_sum(le);
  if (lane == 0) s_l[warp] = le;
  __syncthreads();
  float t = 0.f;
  if (tid == 0)
    for (int w = 0; w < kSqRows; ++w) t += s_l[w];
  finish_block(
      a.loss_partials, a.tile_counter, t, s_l, s_last, [](unsigned, float p) { return p; },
      [&](float t2) {
        const float n = single ? (float)*a.mask_count : (float)a.batch * (float)K;
        *a.loss = t2 / n;
      });
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_slateq_head(const rb200_slateq_args_t* a, void* stream) {
  if (!a) { set_last_error("rb200_slateq_head: args is null"); return RB200_E_INVALID; }
  const int C = a->num_candidates, K = a->slate_width;
  const int Kn = a->maxq ? a->slate_size : a->next_width;
  if (a->batch <= 0 || C < 1 || C > RB200_SLATEQ_MAX_CANDIDATES || K < 1 ||
      K > RB200_SLATEQ_MAX_SLATE || Kn < 1 || Kn > RB200_SLATEQ_MAX_SLATE || a->slate_size < 1 ||
      a->slate_size > C || a->slate_size > RB200_SLATEQ_MAX_SLATE) {
    set_last_error("rb200_slateq_head: need batch > 0, 1 <= C <= %d, 1 <= K, K_next <= %d and "
                   "1 <= slate_size <= min(C, %d) (got B %d, C %d, K %d, K_next %d, slate_size %d)",
                   RB200_SLATEQ_MAX_CANDIDATES, RB200_SLATEQ_MAX_SLATE, RB200_SLATEQ_MAX_SLATE,
                   a->batch, C, K, Kn, a->slate_size);
    return RB200_E_INVALID;
  }
  if (a->norm_method != RB200_SLATEQ_NORM_CURRENT && a->norm_method != RB200_SLATEQ_NORM_NEXT) {
    set_last_error("rb200_slateq_head: unknown norm_method %d", a->norm_method);
    return RB200_E_INVALID;
  }
  if (!a->q_cur || !a->q_next || !a->next_value || !a->next_mask || !a->reward ||
      !a->not_terminal || !a->dz || !a->status || !a->loss_partials || !a->loss ||
      !a->tile_counter || (!a->maxq && !a->next_action) ||
      (a->single_selection && (!a->reward_mask || !a->mask_count)) ||
      (!a->single_selection && a->norm_method == RB200_SLATEQ_NORM_CURRENT && !a->cur_mask)) {
    set_last_error("rb200_slateq_head: required pointer is null");
    return RB200_E_INVALID;
  }
  if (a->time_diff && !(a->time_scale != 0.f)) {
    set_last_error("rb200_slateq_head: time_diff needs a nonzero time_scale");
    return RB200_E_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (a->single_selection) {
    slateq_count_kernel<<<1, kCountThreads, 0, st>>>(a->reward_mask, (long long)a->batch * K,
                                                     a->mask_count);
    if (int rc = check_cuda(cudaGetLastError(), "slateq_count_kernel launch")) return rc;
  }
  slateq_head_kernel<<<ceil_div(a->batch, kSqRows), 32 * kSqRows, 0, st>>>(*a);
  return check_cuda(cudaGetLastError(), "slateq_head_kernel launch");
}
