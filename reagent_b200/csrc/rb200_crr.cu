// reagent_b200 -- loss heads of DiscreteCRRTrainer (reagent/training/discrete_crr_trainer.py).
//
// Both kernels are row-local: one warp per batch row, lanes striding over the A <= 1024 actions,
// softmax in torch's order (row max, exp(x - max), sum; see warp_row_max_sumexp).  The networks
// around them run on rb200_mlp_forward / rb200_mlp_backward / rb200_mlp_wgrad.
//
//   crr_critic_head_kernel   compute_target_q_values + compute_td_loss (:198-218) for one or two
//                            critics, and d loss / d q of each
//   crr_actor_head_kernel    compute_actor_loss (:220-288) and d loss / d (pre-activation of the
//                            actor's last layer)
//
// The actor's logits are FullyConnectedActor.forward's output (reagent/models/actor.py:90-110):
// l = act(z), and with exploration noise l = clamp(act(z) + noise, -1, 1).  `noise` is the draw
// itself (already scaled); NULL means an actor without exploration_variance, which does not clamp.
// Each kernel leaves two batch means, summed in a fixed order by finish_serial.
#include "rb200_common.cuh"

namespace rb200 {

constexpr int kCrrRowsPerBlock = RB200_CRR_ROWS_PER_BLOCK;  // one warp per row

// The logit of column c and whether the clamp passes its gradient (torch.clamp does on the
// closed interval).
struct CrrLogits {
  const float* y;      // act(z), one row
  const float* noise;  // one row or nullptr
  __device__ __forceinline__ float raw(int c) const { return noise ? __fadd_rn(y[c], noise[c]) : y[c]; }
  __device__ __forceinline__ float operator()(int c) const {
    const float u = raw(c);
    return noise ? fminf(fmaxf(u, -1.f), 1.f) : u;
  }
  __device__ __forceinline__ bool passes(int c) const {
    if (!noise) return true;
    const float u = raw(c);
    return u >= -1.f && u <= 1.f;
  }
};

// Per-block tail shared by both heads: the two per-row terms of the block's warps are added in
// warp order, then finish_serial adds the blocks in block order.
template <typename Fin>
__device__ __forceinline__ void crr_finish(float v0, float v1, float* partials, uint32_t* counter,
                                           Fin fin) {
  __shared__ float s_v[2][kCrrRowsPerBlock];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_v[0][warp] = v0; s_v[1][warp] = v1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float mine[2] = {0.f, 0.f};
    for (int w = 0; w < kCrrRowsPerBlock; ++w) { mine[0] += s_v[0][w]; mine[1] += s_v[1][w]; }
    finish_serial<2>(partials, counter, mine, fin);
  }
}

__global__ void __launch_bounds__(32 * kCrrRowsPerBlock)
crr_critic_head_kernel(const rb200_crr_critic_args_t a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row = blockIdx.x * kCrrRowsPerBlock + warp;
  const int A = a.num_actions;
  float l1 = 0.f, l2 = 0.f;
  if (row < a.batch) {  // whole warps: the block-level tail below needs every thread
    const size_t base = (size_t)row * A;
    const CrrLogits lg{a.actor_next + base, a.noise_next ? a.noise_next + base : nullptr};
    float mx, sum;
    warp_row_max_sumexp(lg, A, mx, sum);
    // V' = sum_a softmax(l')_a * q_target(s')_a, per critic; q(s, a) = sum_a q * action
    const float* act = a.action + base;
    float v1 = 0.f, v2 = 0.f, s1 = 0.f, s2 = 0.f, boost = 0.f;
    for (int c = lane; c < A; c += 32) {
      const float p = __fdiv_rn(expf(__fsub_rn(lg(c), mx)), sum);
      v1 = __fadd_rn(v1, __fmul_rn(a.q1_target_next[base + c], p));
      s1 = __fadd_rn(s1, __fmul_rn(a.q1[base + c], act[c]));
      if (a.q2) {
        v2 = __fadd_rn(v2, __fmul_rn(a.q2_target_next[base + c], p));
        s2 = __fadd_rn(s2, __fmul_rn(a.q2[base + c], act[c]));
      }
      if (a.reward_boost) boost = __fadd_rn(boost, __fmul_rn(act[c], a.reward_boost[c]));
    }
    v1 = warp_sum(v1);
    s1 = warp_sum(s1);
    if (a.q2) { v1 = fminf(v1, warp_sum(v2)); s2 = warp_sum(s2); }
    float r = a.reward[row];
    if (a.reward_boost) r = __fadd_rn(r, warp_sum(boost));
    const float y = __fadd_rn(r, __fmul_rn(__fmul_rn(a.gamma, v1), a.not_terminal[row]));
    const float d1 = __fsub_rn(s1, y), d2 = __fsub_rn(s2, y);
    const float k = 2.f / (float)a.batch;
    if (lane == 0) {
      a.td_target[row] = y;
      a.q1_selected[row] = s1;
      if (a.q2) a.q2_selected[row] = s2;
    }
    l1 = __fmul_rn(d1, d1);
    if (a.q2) l2 = __fmul_rn(d2, d2);
    for (int c = lane; c < A; c += 32) {
      a.dz_q1[base + c] = __fmul_rn(__fmul_rn(k, d1), act[c]);
      if (a.q2) a.dz_q2[base + c] = __fmul_rn(__fmul_rn(k, d2), act[c]);
    }
  }
  const float invB = 1.f / (float)a.batch;
  float* loss = a.loss;
  crr_finish(l1, l2, a.loss_partials, a.tile_counter, [loss, invB](const float (&t)[2]) {
    loss[0] = t[0] * invB;
    loss[1] = t[1] * invB;
  });
}

__global__ void __launch_bounds__(32 * kCrrRowsPerBlock)
crr_actor_head_kernel(const rb200_crr_actor_args_t a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row = blockIdx.x * kCrrRowsPerBlock + warp;
  const int A = a.num_actions;
  float t0 = 0.f, t1 = 0.f;
  if (row < a.batch) {
    const size_t base = (size_t)row * A;
    const CrrLogits lg{a.actor_out + base, a.noise ? a.noise + base : nullptr};
    // logged action: torch.argmax(action, dim=1)
    const int li = warp_first_argmax(a.action + base, A);
    float mx, sum;
    warp_row_max_sumexp(lg, A, mx, sum);
    const float lsum = logf(sum);
    // V = sum_a pi_a * Q_a
    float v = 0.f;
    for (int c = lane; c < A; c += 32)
      v = __fadd_rn(v, __fmul_rn(a.q1[base + c], __fdiv_rn(expf(__fsub_rn(lg(c), mx)), sum)));
    v = warp_sum(v);
    const float adv = __fsub_rn(a.q1[base + li], v);
    // exp overflows to +inf before the clamp, which then gives max_weight
    const float w = fminf(fmaxf(expf(__fmul_rn(a.inv_beta, adv)), 0.f), a.max_weight);
    const float log_pi = __fsub_rn(__fsub_rn(lg(li), mx), lsum);
    const float pi_t = __fdiv_rn(expf(__fsub_rn(lg(li), mx)), sum);
    // d loss_row / d log_pi, with the ratio's own dependence on the logits folded in:
    // d(ratio * log_pi) = (ratio + log_pi * ratio_raw * [unclipped]) * d log_pi
    float coef = -w;
    t0 = __fmul_rn(-log_pi, w);
    t1 = t0;
    if (a.entropy_coeff > 0.f) {
      const float raw = __fdiv_rn(pi_t, a.action_probability[row]);
      const float ratio = fminf(fmaxf(raw, 1e-4f), a.clip_limit);
      const bool open = raw >= 1e-4f && raw <= a.clip_limit;
      t1 = __fadd_rn(t0, __fmul_rn(a.entropy_coeff, __fmul_rn(ratio, log_pi)));
      coef = __fadd_rn(coef, __fmul_rn(a.entropy_coeff,
                                       __fadd_rn(ratio, open ? __fmul_rn(log_pi, raw) : 0.f)));
    }
    if (lane == 0 && a.weight) a.weight[row] = w;
    if (lane != 0) { t0 = 0.f; t1 = 0.f; }
    if (a.dz) {
      const float k = coef / (float)a.batch;
      for (int c = lane; c < A; c += 32) {
        const float p = __fdiv_rn(expf(__fsub_rn(lg(c), mx)), sum);
        const float g = __fmul_rn(k, __fsub_rn(c == li ? 1.f : 0.f, p));
        const float y = a.actor_out[base + c];
        a.dz[base + c] = lg.passes(c) ? __fmul_rn(g, act_bwd_from_out(y, a.action_activation)) : 0.f;
      }
    }
  }
  const float invB = 1.f / (float)a.batch;
  float* loss = a.loss;
  crr_finish(t0, t1, a.loss_partials, a.tile_counter, [loss, invB](const float (&t)[2]) {
    loss[0] = t[0] * invB;
    loss[1] = t[1] * invB;
  });
}

static int crr_check_shape(const char* who, int batch, int A) {
  if (batch <= 0 || A < 1 || A > 1024) {
    set_last_error("%s: need batch > 0 and 1 <= num_actions <= 1024 (got %d, %d)", who, batch, A);
    return RB200_E_INVALID;
  }
  return RB200_OK;
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_crr_critic_head(const rb200_crr_critic_args_t* a, void* stream) {
  if (!a) { set_last_error("rb200_crr_critic_head: args is null"); return RB200_E_INVALID; }
  if (int rc = crr_check_shape("rb200_crr_critic_head", a->batch, a->num_actions)) return rc;
  if (!a->actor_next || !a->q1_target_next || !a->q1 || !a->action || !a->reward ||
      !a->not_terminal || !a->td_target || !a->q1_selected || !a->dz_q1 || !a->loss_partials ||
      !a->loss || !a->tile_counter) {
    set_last_error("rb200_crr_critic_head: required pointer is null");
    return RB200_E_INVALID;
  }
  if (a->q2 && (!a->q2_target_next || !a->q2_selected || !a->dz_q2)) {
    set_last_error("rb200_crr_critic_head: q2 needs q2_target_next, q2_selected and dz_q2");
    return RB200_E_INVALID;
  }
  if (!a->q2 && a->q2_target_next) {
    set_last_error("rb200_crr_critic_head: q2_target_next is only read with q2");
    return RB200_E_INVALID;
  }
  return launch<crr_critic_head_kernel>(ceil_div(a->batch, kCrrRowsPerBlock),
                                        32 * kCrrRowsPerBlock, 0, (cudaStream_t)stream,
                                        "crr_critic_head_kernel launch", *a);
}

extern "C" int rb200_crr_actor_head(const rb200_crr_actor_args_t* a, void* stream) {
  if (!a) { set_last_error("rb200_crr_actor_head: args is null"); return RB200_E_INVALID; }
  if (int rc = crr_check_shape("rb200_crr_actor_head", a->batch, a->num_actions)) return rc;
  if (!a->actor_out || !a->q1 || !a->action || !a->loss_partials || !a->loss || !a->tile_counter) {
    set_last_error("rb200_crr_actor_head: required pointer is null");
    return RB200_E_INVALID;
  }
  if (a->entropy_coeff > 0.f && !a->action_probability) {
    set_last_error("rb200_crr_actor_head: entropy_coeff > 0 needs action_probability");
    return RB200_E_INVALID;
  }
  if (a->action_activation < RB200_ACT_LINEAR || a->action_activation > RB200_ACT_SOFTPLUS) {
    set_last_error("rb200_crr_actor_head: unknown action_activation %d", a->action_activation);
    return RB200_E_INVALID;
  }
  return launch<crr_actor_head_kernel>(ceil_div(a->batch, kCrrRowsPerBlock),
                                       32 * kCrrRowsPerBlock, 0, (cudaStream_t)stream,
                                       "crr_actor_head_kernel launch", *a);
}
