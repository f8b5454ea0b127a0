// reagent_b200 -- counterfactual-policy-evaluation heads of the DQN step (SURVEY.md 8f rank 4).
//
// Restates DQNTrainerBaseLightning._calculate_cpes (reagent/training/dqn_trainer_base.py:332-452)
// between the network evaluations: the reward network and the CPE q-network are plain MLPs
// evaluated by rb200_mlp_forward; this kernel does everything in between for one batch row
// per thread --
//   masked_softmax of q(s') over the allowed next actions   reagent/core/torch_utils.py:62-73
//   gather of the logged action's outputs per metric         dqn_trainer_base.py:392-399,:404-406
//   reward loss  = mse(reward_est[logged], metrics_reward)   :397-399
//   CPE targets  = metric_i + discount * not_done * sum_a q_cpe_target(s')[i,a] * p(a|s')   :407-423
//   CPE loss     = mse | huber(q_cpe(s)[logged], target)     :425-428
// and writes d loss / d output of both networks (dense [B, M*A], zero off the logged action), which
// rb200_mlp_backward + rb200_mlp_wgrad turn into parameter gradients.
#include "rb200_common.cuh"

namespace rb200 {

struct CpeDev {
  rb200_cpe_args_t a;
};

__global__ void __launch_bounds__(256) cpe_heads_kernel(const CpeDev d) {
  const rb200_cpe_args_t& a = d.a;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const int A = a.num_actions, M = a.num_metrics;
  float rl = 0.f, ql = 0.f;
  if (b < a.batch) {
    // ---- model propensities on the next state: masked_softmax(q(s'), mask, temperature) ----
    const float* x = a.next_scores + (size_t)b * A;
    const float* mk = a.mask ? a.mask + (size_t)b * A : nullptr;
    float mx, den;
    masked_softmax_stats(x, mk, a.temperature, A, mx, den);
    // logged action: torch.argmax(action, dim=1) -- first maximum
    const float* act = a.action + (size_t)b * A;
    int logged = 0;
    float best = act[0];
    for (int c = 1; c < A; ++c)
      if (act[c] > best) { best = act[c]; logged = c; }
    const float disc = (a.discount_mode == RB200_DISCOUNT_POW && a.discount_src)
                           ? powf(a.gamma, a.discount_src[b]) : a.gamma;
    const float nd = a.not_terminal[b];
    const float inv = 1.f / ((float)a.batch * (float)M);
    for (int i = 0; i < M; ++i) {
      const size_t row = (size_t)b * M * A + (size_t)i * A;
      for (int c = 0; c < A; ++c) { a.dz_reward[row + c] = 0.f; a.dz_qcpe[row + c] = 0.f; }
      const float t = a.metrics_reward[(size_t)b * M + i];
      const float dr = a.reward_est[row + logged] - t;
      rl += dr * dr;
      a.dz_reward[row + logged] = 2.f * dr * inv;
      float nq = 0.f;
      for (int c = 0; c < A; ++c) {
        const float p = masked_softmax_p(x[c], mk ? mk[c] : 1.f, a.temperature, mx, den);
        if (i == 0 && a.propensities_next) a.propensities_next[(size_t)b * A + c] = p;
        nq += a.qcpe_target_next[row + c] * p;
      }
      const float tq = t + disc * (nq * nd);
      const float dq = a.qcpe[row + logged] - tq;
      if (a.loss_kind == RB200_LOSS_HUBER) {
        const float ad = fabsf(dq);
        ql += ad < 1.f ? 0.5f * dq * dq : ad - 0.5f;
        a.dz_qcpe[row + logged] = (dq < -1.f ? -1.f : (dq > 1.f ? 1.f : dq)) * inv;
      } else {
        ql += dq * dq;
        a.dz_qcpe[row + logged] = 2.f * dq * inv;
      }
    }
  }
  // block sums -> partials -> the last block publishes both mean losses (fixed order)
  __shared__ float s_r[8], s_q[8];
  rl = warp_sum(rl);
  ql = warp_sum(ql);
  if ((threadIdx.x & 31) == 0) { s_r[threadIdx.x >> 5] = rl; s_q[threadIdx.x >> 5] = ql; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float r = 0.f, q = 0.f;
    for (int w = 0; w < 8; ++w) { r += s_r[w]; q += s_q[w]; }
    finish_serial<2>(a.loss_partials, a.tile_counter, {r, q}, [&](const float (&tot)[2]) {
      const float inv = 1.f / ((float)a.batch * (float)M);
      a.loss[0] = tot[0] * inv;
      a.loss[1] = tot[1] * inv;
    });
  }
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_cpe_heads(const rb200_cpe_args_t* a, void* stream) {
  if (!a || a->batch <= 0 || a->num_actions <= 0 || a->num_metrics <= 0) { set_last_error("rb200_cpe_heads: bad argument"); return RB200_E_INVALID; }
  if (!a->next_scores || !a->action || !a->metrics_reward || !a->not_terminal || !a->reward_est ||
      !a->qcpe || !a->qcpe_target_next || !a->dz_reward || !a->dz_qcpe || !a->loss_partials ||
      !a->loss || !a->tile_counter) { set_last_error("rb200_cpe_heads: required pointer is null"); return RB200_E_INVALID; }
  if (!(a->temperature > 0.f)) { set_last_error("rb200_cpe_heads: temperature must be positive"); return RB200_E_INVALID; }
  if (a->discount_mode == RB200_DISCOUNT_POW && !a->discount_src) { set_last_error("POW discount needs discount_src"); return RB200_E_INVALID; }
  CpeDev d;
  d.a = *a;
  cpe_heads_kernel<<<ceil_div(a->batch, 256), 256, 0, (cudaStream_t)stream>>>(d);
  return check_cuda(cudaGetLastError(), "cpe_heads_kernel launch");
}
