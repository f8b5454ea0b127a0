// reagent_b200 -- batch-constrained Q-learning (BCQ) filter over imitator logits.
//
// Restates get_valid_actions_from_imitator (reagent/training/imitator_training.py:12-25) and the
// act-time penalty of BatchConstrainedDQN.forward (reagent/models/bcq.py:26-35) for one batch row
// per warp, lanes striding over the actions:
//   p    = softmax(logits)                  row max, expf(x - max), sum, p = e / sum
//   r    = p / max(p)
//   keep = r >= drop_threshold
// in that order (not the algebraic shortcut r = exp(x - max)), with IEEE expf and divisions, so
// that keep flips only where r lies within fp32 noise of the threshold.  Then either
//   mask_out = mask_in * keep                         (trainer: DQNTrainer, dqn_trainer.py:206-220)
//   q_out    = q_in + (-1e10) * (1 - keep)            (model:   BatchConstrainedDQN)
// Row-local and deterministic (fixed reduction order, no atomics), so it can be captured into a
// CUDA graph and its mask fed to K2 as possible_next_actions_mask.
#include "rb200_common.cuh"

namespace rb200 {

constexpr int kBcqRowsPerBlock = 8;  // one warp per row

__global__ void __launch_bounds__(32 * kBcqRowsPerBlock)
bcq_filter_kernel(const float* __restrict__ logits, int batch, int A, float thr,
                  const float* __restrict__ mask_in, float* __restrict__ mask_out,
                  const float* q_in, float* q_out) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * kBcqRowsPerBlock + (threadIdx.x >> 5);
  if (row >= batch) return;  // whole warps leave together: no block-level barrier below
  const size_t base = (size_t)row * A;
  const float* x = logits + base;
  float mx, sum;
  warp_row_max_sumexp([x](int c) { return x[c]; }, A, mx, sum);
  float pmax = 0.f;
  for (int c = lane; c < A; c += 32) pmax = fmaxf(pmax, __fdiv_rn(expf(__fsub_rn(x[c], mx)), sum));
  pmax = warp_max(pmax);
  for (int c = lane; c < A; c += 32) {
    const float p = __fdiv_rn(expf(__fsub_rn(x[c], mx)), sum);
    const float keep = __fdiv_rn(p, pmax) >= thr ? 1.f : 0.f;
    if (mask_out)
      mask_out[base + c] = mask_in ? __fmul_rn(mask_in[base + c], keep) : keep;
    else
      q_out[base + c] = __fadd_rn(q_in[base + c], __fmul_rn(-1e10f, __fsub_rn(1.f, keep)));
  }
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_bcq_filter(const float* imitator_logits, int32_t batch, int32_t num_actions,
                                float drop_threshold, const float* mask_in, float* mask_out,
                                const float* q_in, float* q_out, void* stream) {
  if (batch <= 0 || num_actions < 1 || num_actions > 1024) {
    set_last_error("rb200_bcq_filter: need batch > 0 and 1 <= num_actions <= 1024 (got %d, %d)",
                   batch, num_actions);
    return RB200_E_INVALID;
  }
  if (!imitator_logits) { set_last_error("rb200_bcq_filter: imitator_logits is null"); return RB200_E_INVALID; }
  if (drop_threshold != drop_threshold) { set_last_error("rb200_bcq_filter: drop_threshold is NaN"); return RB200_E_INVALID; }
  const bool trainer_mode = mask_out != nullptr, model_mode = q_out != nullptr;
  if (trainer_mode == model_mode) {
    set_last_error("rb200_bcq_filter: pass exactly one of mask_out (trainer) and q_out (model)");
    return RB200_E_INVALID;
  }
  if (model_mode && !q_in) { set_last_error("rb200_bcq_filter: q_out needs q_in"); return RB200_E_INVALID; }
  if (trainer_mode && q_in) { set_last_error("rb200_bcq_filter: q_in is only read with q_out"); return RB200_E_INVALID; }
  if (model_mode && mask_in) { set_last_error("rb200_bcq_filter: mask_in is only read with mask_out"); return RB200_E_INVALID; }
  bcq_filter_kernel<<<ceil_div(batch, kBcqRowsPerBlock), 32 * kBcqRowsPerBlock, 0,
                      (cudaStream_t)stream>>>(imitator_logits, batch, num_actions, drop_threshold,
                                              mask_in, mask_out, q_in, q_out);
  return check_cuda(cudaGetLastError(), "bcq_filter_kernel launch");
}
