// reagent_b200 -- loss heads of the two remaining DQN-family trainers (SURVEY.md 8f rank 3).
// The networks around them are plain MLPs evaluated by the generic forward / backward /
// weight-gradient kernels of this library; these kernels do what sits in between.
//
//   rb200_pdqn_head  ParametricDQNTrainer.train_step_gen
//       reagent/training/parametric_dqn_trainer.py:109-173: masked (double-)max over the tiled
//       possible next actions (dqn_trainer_base.py:33-77) or the SARSA value, TD target,
//       mse | huber loss and d loss / d q.
//   rb200_c51_head   C51Trainer.train_step_gen, reagent/training/c51_trainer.py:98-173:
//       log-softmax over the atoms (reagent/models/categorical_dqn.py:33-35), expected values,
//       masked arg max, target distribution, categorical projection onto the support (with the
//       reference's l == u corner-case adjustment), cross-entropy loss and d loss / d logits.
//   rb200_bc_xent_head  BehavioralCloningTrainer.train_step_gen / validation_step,
//       reagent/training/behavioral_cloning_trainer.py:38-66: masked logits
//       (reagent/models/dqn.py:55-63), mean cross entropy against each row's logged action and
//       d loss / d logits.
#include "rb200_common.cuh"

namespace rb200 {

// ---------------------------------------------------------------------------
struct PdqnDev {
  rb200_pdqn_args_t a;
};

__global__ void __launch_bounds__(256) pdqn_head_kernel(const PdqnDev d) {
  const rb200_pdqn_args_t& a = d.a;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  float le = 0.f;
  if (b < a.batch) {
    float next_q;
    const int M = a.max_num_action;
    if (M > 0) {
      // get_max_q_values_with_target: q += -1e9 * (1 - mask) on both nets; double-Q: arg max
      // of the online values, value of the target net there; else max of the target values
      float best = 0.f, sel = 0.f;
      int bi = -1;
      for (int c = 0; c < M; ++c) {
        const float pen = -1e9f * (1.f - (a.mask ? a.mask[(size_t)b * M + c] : 1.f));
        const float vt = a.next_q_target[(size_t)b * M + c] + pen;
        const float key = (a.double_q && a.next_q) ? a.next_q[(size_t)b * M + c] + pen : vt;
        if (bi < 0 || key > best) { best = key; bi = c; sel = vt; }
      }
      next_q = sel;
    } else {
      next_q = a.next_q_target[b];
    }
    const float disc = (a.discount_mode == RB200_DISCOUNT_POW && a.discount_src)
                           ? powf(a.gamma, a.discount_src[b]) : a.gamma;
    // parametric_dqn_trainer.py:159: reward + not_terminal * discount * next_q
    const float tgt = a.reward[b] + (a.not_terminal[b] * disc) * next_q;
    const float dq = a.q_values[b] - tgt;
    const float inv = 1.f / (float)a.batch;
    float g;
    if (a.loss_kind == RB200_LOSS_HUBER) {
      const float ad = fabsf(dq);
      le = ad < 1.f ? 0.5f * dq * dq : ad - 0.5f;
      g = (dq < -1.f ? -1.f : (dq > 1.f ? 1.f : dq)) * inv;
    } else {
      le = dq * dq;
      g = 2.f * dq * inv;
    }
    a.dz[b] = g;
    if (a.td_target) a.td_target[b] = tgt;
  }
  __shared__ float s_l[8];
  le = warp_sum(le);
  if ((threadIdx.x & 31) == 0) s_l[threadIdx.x >> 5] = le;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += s_l[w];
    finish_serial<1>(a.loss_partials, a.tile_counter, {t},
                     [&](const float (&tot)[1]) { *a.loss = tot[0] / (float)a.batch; });
  }
}

// ---------------------------------------------------------------------------
// C51: one CTA per batch row; smem: logits of three [A, N] heads as log-probabilities
// ---------------------------------------------------------------------------
struct C51Dev {
  rb200_c51_args_t a;
};

// in-place log_softmax over the last dim of x[A][N] (one warp per action row, round-robin)
__device__ void c51_log_softmax(float* x, int A, int N) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int r = warp; r < A; r += nw) {
    float* row = x + (size_t)r * N;
    float mx = -INFINITY;
    for (int c = lane; c < N; c += 32) mx = fmaxf(mx, row[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float s = 0.f;
    for (int c = lane; c < N; c += 32) s += expf(row[c] - mx);
    s = warp_sum(s);
    const float lse = mx + logf(s);
    for (int c = lane; c < N; c += 32) row[c] -= lse;
  }
}

// kWeighted: prioritized-replay importance weights (a.sample_weight), a separate instantiation so
// that the unweighted kernel stays exactly as it is.  Row b's dz_logits is scaled by w_b and the
// loss is mean_b(w_b * loss_partials[b]); loss_partials keeps the unweighted row cross entropies
// (the priorities are computed from them).
template <bool kWeighted>
__global__ void __launch_bounds__(256) c51_head_kernel(const C51Dev d) {
  const rb200_c51_args_t& a = d.a;
  extern __shared__ float sm[];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int A = a.num_actions, N = a.num_atoms, AN = A * N;
  float* lt = sm;             // log dist of the target net on s'      [A][N]
  float* lo = lt + AN;        // log dist of the online net on s' (double-Q) or alias of lt
  float* lc = lo + AN;        // log dist of the online net on s       [A][N]
  float* nd = lc + AN;        // next_dist of the chosen action         [N]
  float* m = nd + N;          // projected target distribution          [N]
  float* qv = m + N;          // expected values per action             [A]
  __shared__ int s_next;
  for (int i = tid; i < AN; i += blockDim.x) {
    lt[i] = a.logits_next_target[(size_t)b * AN + i];
    lc[i] = a.logits_cur[(size_t)b * AN + i];
    if (a.logits_next_online) lo[i] = a.logits_next_online[(size_t)b * AN + i];
  }
  __syncthreads();
  c51_log_softmax(lt, A, N);
  c51_log_softmax(lc, A, N);
  if (a.logits_next_online) c51_log_softmax(lo, A, N);
  __syncthreads();
  // expected next values: (dist * support).sum(2), c51_trainer.py:117-124
  const float* lq = (a.double_q && a.logits_next_online) ? lo : lt;
  if (a.maxq) {
    for (int r = tid >> 5; r < A; r += blockDim.x >> 5) {
      float s = 0.f;
      for (int c = tid & 31; c < N; c += 32) s += expf(lq[(size_t)r * N + c]) * a.support[c];
      s = warp_sum(s);
      if ((tid & 31) == 0) qv[r] = s;
    }
    __syncthreads();
    if (tid == 0) {  // argmax_with_mask: q + -1e9 * (1 - mask), first maximum
      float best = 0.f;
      int bi = -1;
      for (int c = 0; c < A; ++c) {
        const float mk = a.possible_next_actions_mask ? a.possible_next_actions_mask[(size_t)b * A + c] : 1.f;
        const float v = qv[c] + (-1e9f) * (1.f - mk);
        if (bi < 0 || v > best) { best = v; bi = c; }
      }
      s_next = bi;
      if (a.next_action_idx) a.next_action_idx[b] = bi;
    }
    __syncthreads();
    for (int c = tid; c < N; c += blockDim.x) nd[c] = expf(lt[(size_t)s_next * N + c]);
  } else {  // SARSA: (next_dist * next_action.unsqueeze(-1)).sum(1)
    for (int c = tid; c < N; c += blockDim.x) {
      float s = 0.f;
      for (int r = 0; r < A; ++r) s += expf(lt[(size_t)r * N + c]) * a.next_action[(size_t)b * A + r];
      nd[c] = s;
    }
  }
  for (int c = tid; c < N; c += blockDim.x) m[c] = 0.f;
  __syncthreads();
  // target support, projection (c51_trainer.py:135-160); atoms in order so that the
  // scatter_add of the reference (index order) is reproduced per destination
  if (tid == 0) {
    float rew = a.reward[b];
    if (a.reward_boost) {
      float bs = 0.f;
      for (int c = 0; c < A; ++c) bs += a.action[(size_t)b * A + c] * a.reward_boost[c];
      rew += bs;
    }
    const float disc = (a.discount_src) ? powf(a.gamma, a.discount_src[b]) : a.gamma;
    const float nt = a.not_terminal[b];
    // position b of atom j's target on the support grid and its neighbours l, u.  A NaN target
    // keeps b NaN (fminf / fmaxf would clamp it to qmin) and lands on atom 0, so that m, the
    // row's cross entropy and the loss turn NaN.  In float32 (qmax - qmin) / scale_support can
    // exceed N - 1 by an ulp; b is clamped so that u stays inside m.
    const auto project = [&](int j, int& l, int& u) {
      float tq = rew + (disc * nt) * a.support[j];
      if (tq != tq) { l = u = 0; return tq; }
      tq = fminf(fmaxf(tq, a.qmin), a.qmax);
      const float bb = fminf((tq - a.qmin) / a.scale_support, (float)(N - 1));
      l = (int)floorf(bb);
      u = (int)ceilf(bb);
      if (u > 0 && l == u) l -= 1;
      if (l < N - 1 && l == u) u += 1;
      return bb;
    };
    for (int j = 0; j < N; ++j) {
      int l, u;
      const float bb = project(j, l, u);
      m[l] += nd[j] * ((float)u - bb);
    }
    for (int j = 0; j < N; ++j) {
      int l, u;
      const float bb = project(j, l, u);
      m[u] += nd[j] * (bb - (float)l);
    }
  }
  __syncthreads();
  // loss = -(m * (log_dist * action).sum(1)).sum(1).mean(); gradient w.r.t. the logits of s:
  // d/dlogit[r][c] = action[r] * (softmax[r][c] * sum_j m_j - m_c) / B
  float msum = 0.f;
  for (int c = 0; c < N; ++c) msum += m[c];
  float le = 0.f;
  const float invB = 1.f / (float)a.batch;
  const float w_row = kWeighted ? a.sample_weight[b] : 1.f;
  for (int i = tid; i < AN; i += blockDim.x) {
    const int r = i / N, c = i - r * N;
    const float aw = a.action[(size_t)b * A + r];
    le -= m[c] * lc[i] * aw;
    float dz = aw * (expf(lc[i]) * msum - m[c]) * invB;
    if (kWeighted) dz *= w_row;
    a.dz_logits[(size_t)b * AN + i] = dz;
  }
  if (a.all_q_values) {
    for (int r = tid >> 5; r < A; r += blockDim.x >> 5) {
      float s = 0.f;
      for (int c = tid & 31; c < N; c += 32) s += expf(lc[(size_t)r * N + c]) * a.support[c];
      s = warp_sum(s);
      if ((tid & 31) == 0) a.all_q_values[(size_t)b * A + r] = s;
    }
  }
  __shared__ float s_l[8];
  __shared__ bool s_last;
  le = warp_sum(le);
  if ((tid & 31) == 0) s_l[tid >> 5] = le;
  __syncthreads();
  float t = 0.f;
  if (tid == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_l[w];
  finish_block(
      a.loss_partials, a.tile_counter, t, s_l, s_last,
      [&](unsigned i, float p) { return kWeighted ? __fmul_rn(p, a.sample_weight[i]) : p; },
      [&](float t2) { *a.loss = t2 * invB; });
}

// ---------------------------------------------------------------------------
// Behavioral cloning: one warp per row, lanes striding over the actions
// ---------------------------------------------------------------------------
constexpr int kBcRowsPerBlock = RB200_BC_ROWS_PER_BLOCK;

__global__ void __launch_bounds__(32 * kBcRowsPerBlock) bc_xent_head_kernel(const rb200_bc_xent_args_t a) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row = blockIdx.x * kBcRowsPerBlock + warp;
  const int A = a.num_actions;
  float le = 0.f;
  if (row < a.batch) {  // whole warps: the block-level reduction below needs every thread
    const size_t base = (size_t)row * A;
    const float* x = a.logits + base;
    const float* m = a.mask + base;
    const float* lab = a.labels + base;
    // z = scores + (-1e10) * (1 - mask), each operation rounded as torch does it
    const auto z = [x, m](int c) { return __fadd_rn(x[c], __fmul_rn(-1e10f, __fsub_rn(1.f, m[c]))); };
    // label = torch.argmax(labels, dim=1)
    const int li = warp_first_argmax(lab, A);
    // log_softmax: (z - max) - log(sum exp(z - max)); row loss -log_softmax[label]
    float mx, sum;
    warp_row_max_sumexp(z, A, mx, sum);
    const float lsum = logf(sum);
    le = lane == 0 ? -__fsub_rn(__fsub_rn(z(li), mx), lsum) : 0.f;
    if (a.dz) {  // (softmax - onehot) / B
      const float invB = 1.f / (float)a.batch;
      for (int c = lane; c < A; c += 32) {
        const float p = expf(__fsub_rn(__fsub_rn(z(c), mx), lsum));
        a.dz[base + c] = __fmul_rn(__fsub_rn(p, c == li ? 1.f : 0.f), invB);
      }
    }
  }
  // deterministic mean: per-block partial of the rows in warp order, then finish_block
  __shared__ float s_l[kBcRowsPerBlock];
  __shared__ bool s_last;
  if (lane == 0) s_l[warp] = le;
  __syncthreads();
  float t = 0.f;
  if (tid == 0)
    for (int w = 0; w < kBcRowsPerBlock; ++w) t += s_l[w];
  finish_block(
      a.loss_partials, a.tile_counter, t, s_l, s_last, [](unsigned, float p) { return p; },
      [&](float t2) { *a.loss = t2 / (float)a.batch; });
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_bc_xent_head(const rb200_bc_xent_args_t* a, void* stream) {
  if (!a) { set_last_error("rb200_bc_xent_head: args is null"); return RB200_E_INVALID; }
  if (a->batch <= 0 || a->num_actions < 1 || a->num_actions > 1024) {
    set_last_error("rb200_bc_xent_head: need batch > 0 and 1 <= num_actions <= 1024 (got %d, %d)",
                   a->batch, a->num_actions);
    return RB200_E_INVALID;
  }
  if (!a->logits || !a->labels || !a->mask || !a->loss_partials || !a->loss || !a->tile_counter) {
    set_last_error("rb200_bc_xent_head: required pointer is null");
    return RB200_E_INVALID;
  }
  bc_xent_head_kernel<<<ceil_div(a->batch, kBcRowsPerBlock), 32 * kBcRowsPerBlock, 0,
                        (cudaStream_t)stream>>>(*a);
  return check_cuda(cudaGetLastError(), "bc_xent_head_kernel launch");
}

extern "C" int rb200_pdqn_head(const rb200_pdqn_args_t* a, void* stream) {
  if (!a || a->batch <= 0 || a->max_num_action < 0) { set_last_error("rb200_pdqn_head: bad argument"); return RB200_E_INVALID; }
  if (!a->next_q_target || !a->reward || !a->not_terminal || !a->q_values || !a->dz ||
      !a->loss_partials || !a->loss || !a->tile_counter) { set_last_error("rb200_pdqn_head: required pointer is null"); return RB200_E_INVALID; }
  if (a->discount_mode == RB200_DISCOUNT_POW && !a->discount_src) { set_last_error("POW discount needs discount_src"); return RB200_E_INVALID; }
  PdqnDev d;
  d.a = *a;
  pdqn_head_kernel<<<ceil_div(a->batch, 256), 256, 0, (cudaStream_t)stream>>>(d);
  return check_cuda(cudaGetLastError(), "pdqn_head_kernel launch");
}

extern "C" int rb200_c51_head(const rb200_c51_args_t* a, void* stream) {
  if (!a || a->batch <= 0 || a->num_actions <= 0 || a->num_atoms < 2) { set_last_error("rb200_c51_head: bad argument"); return RB200_E_INVALID; }
  if (!a->logits_next_target || !a->logits_cur || !a->action || !a->reward || !a->not_terminal ||
      !a->support || !a->dz_logits || !a->loss_partials || !a->loss || !a->tile_counter) { set_last_error("rb200_c51_head: required pointer is null"); return RB200_E_INVALID; }
  if (!a->maxq && !a->next_action) { set_last_error("SARSA update needs next_action"); return RB200_E_INVALID; }
  if (a->double_q && a->maxq && !a->logits_next_online) { set_last_error("double-Q needs logits_next_online"); return RB200_E_INVALID; }
  C51Dev d;
  d.a = *a;
  const size_t smem = ((size_t)3 * a->num_actions * a->num_atoms + 2 * a->num_atoms + a->num_actions) * sizeof(float);
  if (smem > 200 * 1024) { set_last_error("rb200_c51_head: too many atoms/actions for one CTA"); return RB200_E_SMEM; }
  cudaStream_t st = (cudaStream_t)stream;
  const char* what = "c51_head_kernel launch";
  return a->sample_weight ? launch<c51_head_kernel<true>>(a->batch, 256, smem, st, what, d)
                          : launch<c51_head_kernel<false>>(a->batch, 256, smem, st, what, d);
}
