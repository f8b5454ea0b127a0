// reagent_b200 -- QR-DQN: fused quantile-regression loss head.
//
// The loss of QRDQNTrainer.train_step_gen (reagent/training/qrdqn_trainer.py:108-194) on the
// (B, A, N) output of a network whose last layer is [hidden -> A*N] (FullyConnectedDQN with
// num_atoms, reagent/models/fully_connected_network.py:166-217), one CTA per batch row:
//   qr_head_kernel   mean over atoms -> masked argmax -> target distribution -> pairwise
//                    quantile-Huber loss and its gradient WITHOUT materialising the
//                    (N, B, N) tensor (qrdqn_trainer.py:125-155, :210-218).
// The network around it runs on the layer kernels of rb200_mlp.cu.
#include "rb200_common.cuh"

namespace rb200 {

// ---------------- fused distributional head: one CTA per batch row ----------------
struct QrDev {
  rb200_qrdqn_args_t a;
};

// kWeighted: prioritized-replay importance weights (a.sample_weight), a separate instantiation so
// that the unweighted kernel stays exactly as it is.  Row b's dz_head is scaled by w_b and the loss
// is mean_b(w_b * loss_partials[b] / N^2); loss_partials keeps the unweighted row sums (the
// priorities are computed from them).
template <bool kWeighted>
__global__ void __launch_bounds__(256) qr_head_kernel(const QrDev d) {
  const rb200_qrdqn_args_t& a = d.a;
  extern __shared__ __align__(16) float sm[];
  const int A = a.num_actions, N = a.num_atoms;
  float* tq = sm;            // [N] target distribution
  float* cq = tq + N;        // [N] current distribution of the taken action
  float* means = cq + N;     // [A]
  float* red = means + A;    // [256]
  __shared__ int s_best;
  __shared__ float s_act[64], s_nact[64], s_mask[64];  // per-row action weights / mask (A <= 64 staged)
  __shared__ bool s_last;
  const int b = blockIdx.x, tid = threadIdx.x;
  const size_t base = (size_t)b * A * N;

  const bool staged = A <= 64;
  if (staged && tid < A) {
    s_act[tid] = a.action[(size_t)b * A + tid];
    s_nact[tid] = (!a.maxq && a.next_action) ? a.next_action[(size_t)b * A + tid] : 0.f;
    s_mask[tid] = a.possible_next_actions_mask ? a.possible_next_actions_mask[(size_t)b * A + tid] : 1.f;
  }
  // mean over atoms of the selection network (qrdqn_trainer.py:127-133)
  const float* sel = a.double_q ? a.q_next_online : a.q_next_target;
  // (16-byte loads when the rows allow it: lane sums differ from the scalar path only in order)
  const bool vec4 = (N & 3) == 0 && (reinterpret_cast<uintptr_t>(sel) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(a.q_cur) & 15) == 0;
  auto row_mean = [&](const float* src, int act) {
    float s = 0.f;
    if (vec4) {
      const float4* r4 = reinterpret_cast<const float4*>(src + base + (size_t)act * N);
      for (int n = tid & 31; n < N / 4; n += 32) { const float4 v = __ldg(r4 + n); s += (v.x + v.y) + (v.z + v.w); }
    } else {
      for (int n = tid & 31; n < N; n += 32) s += src[base + (size_t)act * N + n];
    }
    return warp_sum(s) / (float)N;
  };
  for (int act = tid >> 5; act < A; act += 8) {
    const float m = row_mean(sel, act);
    if ((tid & 31) == 0) means[act] = m;
  }
  __syncthreads();
  if (tid == 0) {
    int bi = 0;
    if (a.maxq) {  // argmax_with_mask (:210-214)
      float best = 0.f;
      bi = -1;
      for (int c = 0; c < A; ++c) {
        const float m = staged ? s_mask[c]
                               : (a.possible_next_actions_mask ? a.possible_next_actions_mask[(size_t)b * A + c] : 1.f);
        const float v = means[c] + -1e9f * (1.f - m);
        if (bi < 0 || v > best) { best = v; bi = c; }
      }
    }
    s_best = bi;
    if (a.next_action_idx) a.next_action_idx[b] = bi;
  }
  __syncthreads();
  float rew = a.reward[b];
  if (a.reward_boost) {
    float bs = 0.f;
    for (int c = 0; c < A; ++c) bs += (staged ? s_act[c] : a.action[(size_t)b * A + c]) * a.reward_boost[c];
    rew += bs;
  }
  const float disc = a.discount_src ? powf(a.gamma, a.discount_src[b]) : a.gamma;
  const float nd = a.not_terminal[b];
  bool finite = true;
  for (int n = tid; n < N; n += blockDim.x) {
    float nq;
    if (a.maxq) {
      nq = a.q_next_target[base + (size_t)s_best * N + n];            // :137
    } else {
      nq = 0.f;                                                         // SARSA (:139)
      for (int c = 0; c < A; ++c)
        nq += a.q_next_target[base + (size_t)c * N + n] * (staged ? s_nact[c] : a.next_action[(size_t)b * A + c]);
    }
    tq[n] = rew + disc * nd * nq;                                       // :142
    finite = finite && isfinite(tq[n]);
    float cur = 0.f;                                                    // :149
    for (int c = 0; c < A; ++c) {
      const float w = staged ? s_act[c] : a.action[(size_t)b * A + c];
      if (w != 0.f) cur += a.q_cur[base + (size_t)c * N + n] * w;
    }
    cq[n] = cur;
  }
  const bool tq_finite = __syncthreads_and(finite);
  // pairwise quantile-Huber (:152-155): td[i,b,j] = target[i] - current[j], weight |tau_j - 1[td<0]|
  const float norm = 1.f / ((float)N * (float)a.batch * (float)N);
  const float w_row = kWeighted ? a.sample_weight[b] : 1.f;
  float lsum = 0.f;
  for (int j = tid; j < N; j += blockDim.x) {
    const float c = cq[j];
    const float tau = (0.5f + (float)j) / (float)N;   // :70-73
    float g = 0.f;
    // |tau - 1[td < 0]| takes two values; huber'(td) = clamp(td, -1, 1) =: gs and
    // huber(td) = gs * (td - gs / 2) (= td^2 / 2 inside, |td| - 1/2 outside: the same roundings
    // as the two-branch form, multiplication by 1/2 being exact)
    const float w_neg = fabsf(tau - 1.f), w_pos = fabsf(tau);
    float l2 = 0.f, g2 = 0.f;  // second accumulators: two independent dependency chains
    int i = 0;
    for (; i + 1 < N; i += 2) {
      const float td0 = tq[i] - c, td1 = tq[i + 1] - c;
      const float gs0 = fmaxf(-1.f, fminf(1.f, td0)), gs1 = fmaxf(-1.f, fminf(1.f, td1));
      const float w0 = td0 < 0.f ? w_neg : w_pos, w1 = td1 < 0.f ? w_neg : w_pos;
      lsum += (gs0 * (td0 - 0.5f * gs0)) * w0;                          // huber (:217-218)
      l2 += (gs1 * (td1 - 0.5f * gs1)) * w1;
      g += gs0 * w0;
      g2 += gs1 * w1;
    }
    if (i < N) {
      const float td0 = tq[i] - c;
      const float gs0 = fmaxf(-1.f, fminf(1.f, td0));
      const float w0 = td0 < 0.f ? w_neg : w_pos;
      lsum += (gs0 * (td0 - 0.5f * gs0)) * w0;
      g += gs0 * w0;
    }
    lsum += l2;
    g += g2;
    // fminf / fmaxf turn a NaN td into a derivative of 1; autograd keeps the NaN.  A NaN td
    // needs a non-finite target or current value, so only such columns look for one.
    if (!(tq_finite && isfinite(c)))
      for (int i2 = 0; i2 < N; ++i2) {
        const float td = tq[i2] - c;
        if (td != td) g = td;
      }
    float dcur = -g * norm;   // d loss / d current[j]
    if (kWeighted) dcur *= w_row;
    // d loss / d head output [b, a, j] = action[b,a] * dcur  (linear head)
    for (int cact = 0; cact < A; ++cact)
      a.dz_head[base + (size_t)cact * N + j] = (staged ? s_act[cact] : a.action[(size_t)b * A + cact]) * dcur;
  }
  lsum = warp_sum(lsum);
  if ((tid & 31) == 0) red[tid >> 5] = lsum;
  __syncthreads();
  float s = 0.f;
  if (tid == 0)
    for (int i = 0; i < (int)blockDim.x / 32; ++i) s += red[i];
  finish_block(
      a.loss_partials, a.tile_counter, s, red, s_last,
      [&](unsigned i, float p) { return kWeighted ? __fmul_rn(p, a.sample_weight[i]) : p; },
      [&](float t2) { *a.loss = t2 * norm; });
  // mean over atoms of q(s) for reporting (all_q_values, :146)
  if (a.all_q_values) {
    for (int act = tid >> 5; act < A; act += 8) {
      const float m = row_mean(a.q_cur, act);
      if ((tid & 31) == 0) a.all_q_values[(size_t)b * A + act] = m;
    }
  }
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_qrdqn_head(const rb200_qrdqn_args_t* a, void* stream) {
  if (!a || a->batch <= 0 || a->num_actions <= 0 || a->num_atoms <= 0) { set_last_error("rb200_qrdqn_head: bad argument"); return RB200_E_INVALID; }
  if (!a->q_next_target || !a->q_cur || !a->action || !a->reward || !a->not_terminal || !a->dz_head ||
      !a->loss_partials || !a->loss || !a->tile_counter) { set_last_error("rb200_qrdqn_head: required pointer is null"); return RB200_E_INVALID; }
  // the atom means are read from q_next_online whenever double_q is set, SARSA included
  if (a->double_q && !a->q_next_online) { set_last_error("double-Q needs q_next_online"); return RB200_E_INVALID; }
  if (!a->maxq && !a->next_action) { set_last_error("SARSA update needs next_action"); return RB200_E_INVALID; }
  QrDev d;
  d.a = *a;
  const size_t smem = (size_t)(2 * a->num_atoms + a->num_actions + 256) * sizeof(float);
  if (smem > 48 * 1024) { set_last_error("rb200_qrdqn_head: too many atoms/actions for one CTA"); return RB200_E_SMEM; }
  // opted in: the kernel's static shared memory comes on top of the 48 KB of dynamic
  cudaStream_t st = (cudaStream_t)stream;
  const char* what = "qr_head_kernel launch";
  return a->sample_weight ? launch<qr_head_kernel<true>>(a->batch, 256, smem, st, what, d)
                          : launch<qr_head_kernel<false>>(a->batch, 256, smem, st, what, d);
}
