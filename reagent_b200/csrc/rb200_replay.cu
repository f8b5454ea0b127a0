// reagent_b200 -- K1: fused replay-sample kernel (index selection + segment gather +
// n-step reward fold + on-the-fly feature normalisation + trainer-batch formatting).
//
// Restates, for device-resident storage,
//   SumTree.sample / stratified walk        reagent/replay_memory/sum_tree.py:93-153
//   ReplayBuffer.sample_index_batch         reagent/replay_memory/circular_replay_buffer.py:589-603
//   ReplayBuffer.sample_transition_batch    circular_replay_buffer.py:614-706, helpers :741-774
//   PrioritizedReplayBuffer probabilities   prioritized_replay_buffer.py:116-147
//   DiscreteDqnInputMaker / PolicyNetworkInputMaker   gym/preprocessors/trainer_preprocessor.py:72-227
//   Preprocessor.forward on state / next_state        preprocessing/preprocessor.py:115-170
//
// HBM-bound.  Algorithmic bytes per sampled transition (SURVEY.md 8d, K1):
//   d*8 (fp64 tree nodes) + 2*S*4 read + 2*S'*4 written + ~13 read + ~40 scalar outputs.
// Layout: one CTA = 32 samples, 4 per warp.  Lane u of a warp does the index selection and the
// scalar outputs of the warp's sample u (one dependent 8-byte load per deep tree level), so a
// CTA's 32 descents run in 8 warps whose latencies overlap; then the warp streams its 8 rows
// (state and next_state of 4 samples): all row loads are issued (coalesced 16-byte loads, one
// 512-byte request per row) before the first store.
#include "rb200_preproc.cuh"

namespace rb200 {

constexpr int kSPB = 32;  // samples per CTA
constexpr int kTopLevels = 10;  // 8 KB: small enough to share an SM with the wgmma TD kernel

struct SampleDev {
  rb200_sample_args_t a;
};

__device__ __forceinline__ long long wrap(long long i, long long cap) {
  i %= cap;
  return i < 0 ? i + cap : i;
}

__global__ void __launch_bounds__(kThreads) replay_sample_kernel(const SampleDev d) {
  const rb200_sample_args_t& a = d.a;
  // top kTopLevels levels of the fp64 sum tree (2^kTopLevels - 1 nodes, 8 KB): loaded once
  // per CTA with coalesced reads so that only the deep levels cost a dependent L2 round trip
  __shared__ double s_top[(1 << kTopLevels) - 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b0 = blockIdx.x * kSPB;
  const long long cap = a.capacity;
  if (a.mode == RB200_SAMPLE_PRIORITIZED) {
    const int top = min(a.tree_depth + 1, kTopLevels);
    const int n_top = (1 << top) - 1;
    for (int i = tid; i < n_top; i += kThreads) s_top[i] = __ldg(a.tree + i);
    __syncthreads();
  }

  // ---- index selection + scalar outputs: every warp owns kPerWarp samples, lane u does the
  // scalar work of sample u, so the 32 descents of a CTA run in 8 warps whose dependent loads
  // overlap (one warp doing all 32 in lock-step left 7 warps idle) ----
  constexpr int kPerWarp = kSPB / (kThreads / 32);  // 4
  long long idx = 0, next = 0;
  int term = 0;
  long long act = 0, nact = 0;
  {
    const int b = b0 + warp * kPerWarp + lane;
    if (lane < kPerWarp && b < a.batch) {
      if (a.mode == RB200_SAMPLE_PRIORITIZED) {
        // sum_tree.py:112-131: q *= root; descend comparing with the left child
        double q = a.query[b] * s_top[0];
        long long node = 0;
        for (int lvl = 1; lvl <= a.tree_depth; ++lvl) {
          const long long left = node * 2;
          const long long pos = ((1ll << lvl) - 1) + left;
          const double left_sum = (lvl < kTopLevels) ? s_top[pos] : __ldg(a.tree + pos);
          if (q < left_sum) {
            node = left;
          } else {
            node = left + 1;
            q -= left_sum;
          }
        }
        idx = node;
        for (int o = 0; o < a.n_override; ++o)
          if (a.override_pos[o] == b) idx = a.override_idx[o];
      } else if (a.mode == RB200_SAMPLE_UNIFORM) {
        // circular_replay_buffer.py:602-603: valid_indices[rank]; valid_indices is the
        // ascending list of valid slots -> select(rank) over the validity bitmap.
        const long long rank = a.ranks[b];
        int lo = 0, hi = a.n_valid_blocks;  // block_offsets has n_valid_blocks+1 entries
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if ((long long)a.valid_block_offsets[mid] <= rank) lo = mid; else hi = mid;
        }
        long long rem = rank - a.valid_block_offsets[lo];
        long long p = (long long)lo * RB200_VALID_BLOCK;
        const long long pend = min(cap, p + RB200_VALID_BLOCK);
        for (; p < pend; ++p) {
          if (a.valid[p]) {
            if (rem == 0) break;
            --rem;
          }
        }
        idx = p;
      } else {
        idx = a.indices_in[b];
      }
      // circular_replay_buffer.py:759-774 (_get_steps): first terminal within the horizon
      int steps = a.update_horizon;
      for (int k = 0; k < a.update_horizon - 1; ++k) {
        if (a.terminal[wrap(idx + k, cap)]) { steps = k + 1; break; }
      }
      // :741-747 (_reduce_multi_step_reward): sum_k r[i+k]*decay[k]*[k<steps]
      float rew = 0.f;
      for (int k = 0; k < a.update_horizon; ++k) {
        const float m = (k < steps) ? 1.f : 0.f;
        rew += __fmul_rn(__fmul_rn(a.reward[wrap(idx + k, cap)], a.decays[k]), m);
      }
      next = a.timeline_next ? wrap(idx + 1, cap) : wrap(idx + steps, cap);
      term = a.terminal[wrap(idx + steps - 1, cap)] ? 1 : 0;  // :658-660
      if (a.indices_out) a.indices_out[b] = idx;
      if (a.step_out) a.step_out[b] = steps;
      if (a.step_f32_out) a.step_f32_out[b] = (float)steps;
      if (a.reward_out) a.reward_out[b] = rew;
      if (a.next_reward_out) a.next_reward_out[b] = a.reward[next];
      if (a.terminal_out) a.terminal_out[b] = (uint8_t)term;
      if (a.not_terminal_out) a.not_terminal_out[b] = 1.f - (float)term;  // InputMaker :125,:187
      if (a.sampling_prob_out)  // prioritized_replay_buffer.py:136-140 (get_priority -> f32)
        a.sampling_prob_out[b] = (float)a.tree[((1ll << a.tree_depth) - 1) + idx];
      if (a.action_i64) {
        act = a.action_i64[idx];
        nact = a.action_i64[next];
        if (a.action_out_i64) a.action_out_i64[b] = act;
        if (a.next_action_out_i64) a.next_action_out_i64[b] = nact;
      }
    }
  }

  // ---- row gathers: the warp streams its kPerWarp samples ----
  long long s_idx[kPerWarp], s_next[kPerWarp];
  int s_term[kPerWarp];
#pragma unroll
  for (int u = 0; u < kPerWarp; ++u) {
    s_idx[u] = __shfl_sync(0xffffffffu, idx, u);
    s_next[u] = __shfl_sync(0xffffffffu, next, u);
    s_term[u] = __shfl_sync(0xffffffffu, term, u);
  }
  const int bw = b0 + warp * kPerWarp;  // first sample of this warp
  // one-hot actions (one_hot_actions, trainer_preprocessor.py:72-97): lanes over the actions
  if (a.action_i64 && a.action_onehot) {
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u) {
      const long long au = __shfl_sync(0xffffffffu, act, u), nu = __shfl_sync(0xffffffffu, nact, u);
      if (bw + u >= a.batch) continue;
      for (int c = lane; c < a.num_actions; c += 32) {
        a.action_onehot[(size_t)(bw + u) * a.num_actions + c] = (c == au) ? 1.f : 0.f;
        a.next_action_onehot[(size_t)(bw + u) * a.num_actions + c] = (!s_term[u] && c == nu) ? 1.f : 0.f;
      }
    }
  }
  // observation -> state / next_state (with optional normalisation)
  if (a.obs) {
    const bool vec = (a.cols == nullptr) && ((a.obs_dim & 3) == 0) &&
                     ((reinterpret_cast<uintptr_t>(a.obs) & 15) == 0) &&
                     (!a.state || (reinterpret_cast<uintptr_t>(a.state) & 15) == 0) &&
                     (!a.next_state || (reinterpret_cast<uintptr_t>(a.next_state) & 15) == 0);
    if (vec && a.obs_dim <= 128) {
      // all 2*kPerWarp row loads of the warp are issued before the first store: 8 independent
      // 512-byte requests in flight per warp instead of one
      float4 v[2 * kPerWarp];
      const int c = lane * 4;
#pragma unroll
      for (int u = 0; u < kPerWarp; ++u) {
        const bool on = bw + u < a.batch && c < a.obs_dim;
        v[2 * u] = (on && a.state) ? __ldg(reinterpret_cast<const float4*>(a.obs + (size_t)s_idx[u] * a.obs_dim + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
        v[2 * u + 1] = (on && a.next_state) ? __ldg(reinterpret_cast<const float4*>(a.obs + (size_t)s_next[u] * a.obs_dim + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < kPerWarp; ++u) {
        if (bw + u >= a.batch || c >= a.obs_dim) continue;
        if (a.state) *reinterpret_cast<float4*>(a.state + (size_t)(bw + u) * a.obs_dim + c) = v[2 * u];
        if (a.next_state) *reinterpret_cast<float4*>(a.next_state + (size_t)(bw + u) * a.obs_dim + c) = v[2 * u + 1];
      }
    } else {
#pragma unroll
      for (int u = 0; u < kPerWarp; ++u) {
        const int b = bw + u;
        if (b >= a.batch) continue;
        for (int which = 0; which < 2; ++which) {
          float* dst = which ? a.next_state : a.state;
          if (!dst) continue;
          const float* src = a.obs + (size_t)(which ? s_next[u] : s_idx[u]) * a.obs_dim;
          if (a.cols == nullptr) {
            float* drow = dst + (size_t)b * a.obs_dim;
            if (vec) {
              for (int c = lane * 4; c < a.obs_dim; c += 128)
                *reinterpret_cast<float4*>(drow + c) = __ldg(reinterpret_cast<const float4*>(src + c));
            } else {
              for (int c = lane; c < a.obs_dim; c += 32) drow[c] = src[c];
            }
          } else {
            float* drow = dst + (size_t)b * a.obs_out_dim;
            for (int j = lane; j < a.obs_out_dim; j += 32) {
              const rb200_feature_col_t f = a.cols[j];
              drow[j] = preprocess_value(src[f.src_col], 1.f, f, a.quantiles);
            }
          }
        }
      }
    }
  }
#pragma unroll
  for (int u = 0; u < kPerWarp; ++u) {
    const int b = bw + u;
    if (b >= a.batch) continue;
    const long long idx_u = s_idx[u], next_u = s_next[u];
    const int term_u = s_term[u];
    // continuous action -> rescaled action / next_action (PolicyNetworkInputMaker :176-196)
    if (a.action_f32) {
      const float* sa = a.action_f32 + (size_t)idx_u * a.action_dim;
      const float* sn = a.action_f32 + (size_t)next_u * a.action_dim;
      for (int c = lane; c < a.action_dim; c += 32) {
        float va = sa[c], vn = sn[c];
        if (a.action_out_raw) a.action_out_raw[(size_t)b * a.action_dim + c] = va;
        if (a.next_action_out_raw) a.next_action_out_raw[(size_t)b * a.action_dim + c] = vn;
        if (a.action_rescaled) {
          // rescale_actions (reagent/training/utils.py:13-29)
          const float lo = a.action_low[c], range = a.action_high[c] - a.action_low[c];
          const float nr = a.train_high - a.train_low;
          a.action_rescaled[(size_t)b * a.action_dim + c] =
              __fadd_rn(__fmul_rn(__fdiv_rn(__fsub_rn(va, lo), range), nr), a.train_low);
          a.next_action_rescaled[(size_t)b * a.action_dim + c] =
              term_u ? 0.f
                     : __fadd_rn(__fmul_rn(__fdiv_rn(__fsub_rn(vn, lo), range), nr), a.train_low);
        }
      }
    }
    // generic byte rows (extras, raw copies of any dense key)
    for (int g = 0; g < a.n_specs; ++g) {
      const rb200_gather_spec_t& sp = a.specs[g];
      const unsigned char* src =
          (const unsigned char*)sp.src + (size_t)(sp.which ? next_u : idx_u) * sp.row_bytes;
      unsigned char* dst = (unsigned char*)sp.dst + (size_t)b * sp.row_bytes;
      if (((sp.row_bytes & 3) == 0) && ((reinterpret_cast<uintptr_t>(src) & 3) == 0) &&
          ((reinterpret_cast<uintptr_t>(dst) & 3) == 0)) {
        for (int c = lane; c < sp.row_bytes / 4; c += 32)
          reinterpret_cast<uint32_t*>(dst)[c] = reinterpret_cast<const uint32_t*>(src)[c];
      } else {
        for (int c = lane; c < sp.row_bytes; c += 32) dst[c] = src[c];
      }
    }
  }
}

// ---- validity bitmap -> per-block counts -> exclusive offsets (uniform sampling) ----
__global__ void valid_count_kernel(const uint8_t* __restrict__ valid, long long cap,
                                   int* __restrict__ counts) {
  const long long base = (long long)blockIdx.x * RB200_VALID_BLOCK;
  int c = 0;
  for (int i = threadIdx.x; i < RB200_VALID_BLOCK; i += blockDim.x) {
    const long long p = base + i;
    if (p < cap && valid[p]) ++c;
  }
  c = (int)warp_sum((float)c);  // <= 256 per block: exact in fp32
  __shared__ int part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += part[w];
    counts[blockIdx.x] = t;
  }
}

__global__ void valid_scan_kernel(const int* __restrict__ counts, int n, int* __restrict__ offsets) {
  // single CTA, 1024 threads: chunked inclusive scan -> exclusive offsets[0..n]
  __shared__ int tot[1024];
  const int t = threadIdx.x, per = (n + 1023) / 1024;
  const int beg = t * per, end = min(n, beg + per);
  int s = 0;
  for (int i = beg; i < end; ++i) s += counts[i];
  tot[t] = s;
  __syncthreads();
  if (t == 0) {
    int run = 0;
    for (int i = 0; i < 1024; ++i) { const int v = tot[i]; tot[i] = run; run += v; }
  }
  __syncthreads();
  int run = tot[t];
  for (int i = beg; i < end; ++i) { offsets[i] = run; run += counts[i]; }
  if (end == n && beg <= n) offsets[n] = run;
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_replay_sample(const rb200_sample_args_t* a, void* stream) {
  if (!a) { set_last_error("rb200_replay_sample: null args"); return RB200_E_INVALID; }
  if (a->batch <= 0 || a->capacity <= 0 || a->update_horizon <= 0) { set_last_error("rb200_replay_sample: bad batch/capacity/horizon"); return RB200_E_INVALID; }
  if (!a->terminal || !a->reward || !a->decays) { set_last_error("rb200_replay_sample: terminal/reward/decays required"); return RB200_E_INVALID; }
  if (a->mode == RB200_SAMPLE_PRIORITIZED && (!a->tree || !a->query || a->tree_depth < 0)) { set_last_error("prioritized mode needs tree + query"); return RB200_E_INVALID; }
  if (a->mode == RB200_SAMPLE_UNIFORM && (!a->ranks || !a->valid || !a->valid_block_offsets)) { set_last_error("uniform mode needs ranks + validity index"); return RB200_E_INVALID; }
  if (a->mode == RB200_SAMPLE_GIVEN && !a->indices_in) { set_last_error("given mode needs indices_in"); return RB200_E_INVALID; }
  if (a->n_specs < 0 || a->n_specs > RB200_MAX_GATHER_SPECS) { set_last_error("too many gather specs"); return RB200_E_INVALID; }
  if (a->sampling_prob_out && !a->tree) { set_last_error("sampling probabilities need the tree"); return RB200_E_INVALID; }
  if (a->action_onehot && (!a->next_action_onehot || a->num_actions <= 0)) { set_last_error("one-hot output needs next_action_onehot and num_actions"); return RB200_E_INVALID; }
  if (a->action_rescaled && (!a->next_action_rescaled || !a->action_low || !a->action_high)) { set_last_error("rescaled action output needs bounds"); return RB200_E_INVALID; }
  SampleDev d;
  d.a = *a;
  const int grid = ceil_div(a->batch, kSPB);
  replay_sample_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(d);
  return check_cuda(cudaGetLastError(), "replay_sample_kernel launch");
}

extern "C" int rb200_valid_index_build(const uint8_t* valid, int64_t capacity, int32_t* counts,
                                       int32_t* offsets, void* stream) {
  if (!valid || !counts || !offsets || capacity <= 0) { set_last_error("rb200_valid_index_build: bad argument"); return RB200_E_INVALID; }
  const int nblk = (int)((capacity + RB200_VALID_BLOCK - 1) / RB200_VALID_BLOCK);
  valid_count_kernel<<<nblk, 256, 0, (cudaStream_t)stream>>>(valid, capacity, counts);
  valid_scan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(counts, nblk, offsets);
  return check_cuda(cudaGetLastError(), "valid index kernels launch");
}
