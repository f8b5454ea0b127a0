// reagent_b200 -- returns and loss heads of ReinforceTrainer and PPOTrainer
// (reagent/training/reinforce_trainer.py, reagent/training/ppo_trainer.py).
//
// Both kernels take a packed batch: the rows of n_traj trajectories one after another, with
// offsets[n_traj + 1] marking where each begins.
//
//   pg_returns_kernel   discounted_returns (reagent/training/utils.py:42-54) of every trajectory,
//                       then whiten (:32-39) or mean subtraction, then clamp(min=0).  One warp per
//                       trajectory.  The reverse chain running = r_t + gamma * running is run by
//                       one lane, in order, with the product and the sum each rounded to fp32 (no
//                       FMA) -- what the reference's 0-dim tensor ops compute -- so the returns
//                       are bit-identical to its loop.  A parallel scan would regroup the powers
//                       of gamma and lose that.  The warp stages the next chunk of rewards into
//                       registers while the lane walks the current one, so the chain waits on
//                       its own adds and multiplies, not on loads.
//   pg_head_kernel      one warp per row, A <= 1024: the masked, tempered log-softmax at the
//                       logged action, the advantage, the REINFORCE or PPO loss term of the row,
//                       d loss / d scores and the value net's d loss / d V.
#include "rb200_common.cuh"

namespace rb200 {

constexpr int kPgRowsPerBlock = RB200_PG_ROWS_PER_BLOCK;  // head: one warp per row
constexpr int kPgTrajPerBlock = 4;                        // returns: one warp per trajectory
constexpr int kPgChunk = 128;                             // rewards staged per warp and step
constexpr int kPgPerLane = kPgChunk / 32;

// ----------------------------------------------------------------------------
// returns
// ----------------------------------------------------------------------------
__device__ __forceinline__ float pg_clip(float r, float hi) { return r > hi ? hi : r; }  // NaN stays

__global__ void __launch_bounds__(32 * kPgTrajPerBlock)
pg_returns_kernel(const rb200_pg_returns_args_t a) {
  __shared__ float s_chunk[kPgTrajPerBlock][kPgChunk];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int traj = blockIdx.x * kPgTrajPerBlock + warp;
  if (traj >= a.n_traj) return;  // no block-level synchronisation below
  const int beg = a.offsets[traj], end = a.offsets[traj + 1];
  const int n = end - beg;
  if (n <= 0) return;
  float* sc = s_chunk[warp];
  const float* rw = a.reward + beg;
  float* out = a.returns + beg;
  if (a.gamma == 0.f) {  // discounted_returns returns the clamped rewards as they are
    for (int i = lane; i < n; i += 32) out[i] = pg_clip(rw[i], a.reward_clip);
  } else {
    // chunks from the end: chunk k covers [max(0, n - (k+1)*kPgChunk), n - k*kPgChunk)
    float next[kPgPerLane];
    auto load = [&](int hi, float (&v)[kPgPerLane]) {
#pragma unroll
      for (int j = 0; j < kPgPerLane; ++j) {
        const int i = hi - kPgChunk + j * 32 + lane;
        v[j] = (i >= 0 && i < hi) ? pg_clip(rw[i], a.reward_clip) : 0.f;
      }
    };
    load(n, next);
    float running = 0.f;
    for (int hi = n; hi > 0; hi -= kPgChunk) {
#pragma unroll
      for (int j = 0; j < kPgPerLane; ++j) sc[j * 32 + lane] = next[j];
      __syncwarp();
      if (hi - kPgChunk > 0) load(hi - kPgChunk, next);  // in flight while lane 0 walks the chain
      const int lo = hi - kPgChunk < 0 ? 0 : hi - kPgChunk;
      if (lane == 0) {
#pragma unroll 8
        for (int i = hi - 1; i >= lo; --i) {
          float& s = sc[i - (hi - kPgChunk)];
          running = __fadd_rn(s, __fmul_rn(a.gamma, running));
          s = running;
        }
      }
      __syncwarp();
#pragma unroll
      for (int j = 0; j < kPgPerLane; ++j) {
        const int i = hi - kPgChunk + j * 32 + lane;
        if (i >= lo && i < hi) out[i] = sc[j * 32 + lane];
      }
      __syncwarp();
    }
  }
  if (a.norm == RB200_PG_NORM_NONE && !a.offset_clamp_min) return;
  __syncwarp();  // this warp's global writes above are visible to all its lanes
  float mean_f = 0.f, den = 1.f;
  if (a.norm != RB200_PG_NORM_NONE) {
    double s = 0.0;
    for (int i = lane; i < n; i += 32) s += (double)out[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const double mean = s / (double)n;
    mean_f = (float)mean;
    if (a.norm != RB200_PG_NORM_SUBTRACT_MEAN) {
      // whiten: population std (unbiased=False), then + EPS in fp32
      double q = 0.0;
      for (int i = lane; i < n; i += 32) {
        const double d = (double)out[i] - mean;
        q += d * d;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      den = __fadd_rn((float)sqrt(q / (double)n), (float)RB200_PG_WHITEN_EPS);
    }
  }
  const bool sub = a.norm == RB200_PG_NORM_WHITEN || a.norm == RB200_PG_NORM_SUBTRACT_MEAN;
  const bool div = a.norm == RB200_PG_NORM_WHITEN || a.norm == RB200_PG_NORM_WHITEN_NO_MEAN;
  for (int i = lane; i < n; i += 32) {
    float x = out[i];
    if (sub) x = __fsub_rn(x, mean_f);
    if (div) x = __fdiv_rn(x, den);
    if (a.offset_clamp_min) x = x < 0.f ? 0.f : x;
    out[i] = x;
  }
}

// ----------------------------------------------------------------------------
// loss head
// ----------------------------------------------------------------------------
// The logits of one row: (z + INVALID_ACTION_CONSTANT * (1 - mask)) / temperature.
struct PgLogits {
  const float* z;
  const float* mask;  // nullptr: no mask
  float temperature;
  __device__ __forceinline__ float operator()(int c) const {
    const float s = mask ? __fadd_rn(z[c], __fmul_rn(-1e10f, __fsub_rn(1.f, mask[c]))) : z[c];
    return __fdiv_rn(s, temperature);
  }
};

// The trajectory of a row: the last t with offsets[t] <= row.
__device__ __forceinline__ int pg_traj_of(const int32_t* offsets, int n_traj, int row) {
  int lo = 0, hi = n_traj - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (offsets[mid] <= row) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(32 * kPgRowsPerBlock)
pg_head_kernel(const rb200_pg_head_args_t a) {
  __shared__ float s_v[2][kPgRowsPerBlock];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row = blockIdx.x * kPgRowsPerBlock + warp;
  const int A = a.num_actions;
  float t_pol = 0.f, t_val = 0.f;
  if (row < a.rows) {  // whole warps: the block-level tail below needs every thread
    const size_t base = (size_t)row * A;
    const PgLogits lg{a.scores + base, a.mask ? a.mask + base : nullptr, a.temperature};
    // logged action: Categorical.log_prob(action.argmax(1))
    const int li = warp_first_argmax(a.action + base, A);
    float mx, sum;
    warp_row_max_sumexp(lg, A, mx, sum);
    const float lse = __fadd_rn(mx, logf(sum));
    const float log_pi = __fsub_rn(lg(li), lse);

    // advantage, and the value net's regression target y
    float adv, y = 0.f, v = 0.f;
    if (a.advantage_kind == RB200_PG_ADV_TD) {
      v = a.value[row];
      float vn;
      float nt;
      if (a.next_value) {
        vn = a.next_value[row];
        nt = a.not_terminal ? a.not_terminal[row] : 1.f;
        if (!a.not_terminal) {
          const int t = pg_traj_of(a.offsets, a.n_traj, row);
          if (row == a.offsets[t + 1] - 1) nt = 0.f;
        }
      } else {
        const int t = pg_traj_of(a.offsets, a.n_traj, row);
        const bool last = row == a.offsets[t + 1] - 1;
        vn = last ? 0.f : a.value[row + 1];
        nt = a.not_terminal ? a.not_terminal[row] : (last ? 0.f : 1.f);
      }
      const float r = pg_clip(a.reward[row], a.reward_clip);
      y = __fadd_rn(r, __fmul_rn(__fmul_rn(a.gamma, nt), vn));
      adv = __fsub_rn(y, v);
      if (a.offset_clamp_min) adv = adv < 0.f ? 0.f : adv;
    } else {
      adv = a.returns[row];
      if (a.advantage_kind == RB200_PG_ADV_BASELINE) {
        v = a.value[row];
        y = adv;
        adv = __fsub_rn(adv, v);
      }
    }

    // d loss_row / d log_pi, and the row's loss term
    float g;
    float ent = 0.f;
    if (a.loss_kind == RB200_PG_LOSS_REINFORCE) {
      float elig = log_pi;
      g = -adv;
      if (a.logged_log_prob) {  // off_policy: exp(min(log_pi - logged, log(clip_param)))
        const float d = __fsub_rn(log_pi, a.logged_log_prob[row]);
        elig = expf(fminf(d, a.log_clip_param));
        g = d <= a.log_clip_param ? __fmul_rn(-adv, elig) : 0.f;
      }
      t_pol = -__fmul_rn(adv, elig);
    } else {
      const float ratio = expf(__fsub_rn(log_pi, a.logged_log_prob[row]));
      const float lo = a.ppo_clip_lo, hi = a.ppo_clip_hi;
      const float rc = fminf(fmaxf(ratio, lo), hi);
      const float s1 = __fmul_rn(adv, ratio), s2 = __fmul_rn(adv, rc);
      // torch.minimum sends the gradient to the smaller side, half to each on a tie;
      // torch.clamp passes it on the closed interval
      const float g1 = s1 < s2 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
      const float g2 = s2 < s1 ? 1.f : (s1 == s2 ? 0.5f : 0.f);
      const float pass = (ratio >= lo && ratio <= hi) ? 1.f : 0.f;
      g = -__fmul_rn(__fmul_rn(adv, __fadd_rn(g1, __fmul_rn(g2, pass))), ratio);
      t_pol = -fminf(s1, s2);
      if (a.entropy_weight != 0.f) {  // H = -sum_c p_c log p_c
        float h = 0.f;
        for (int c = lane; c < A; c += 32) {
          const float l = __fsub_rn(lg(c), lse);
          h = __fadd_rn(h, __fmul_rn(expf(l), l));
        }
        ent = -warp_sum(h);
        t_pol = __fsub_rn(t_pol, __fmul_rn(a.entropy_weight, ent));
      }
    }
    if (a.value) {
      const float d = __fsub_rn(v, y);
      t_val = __fmul_rn(d, d);
      if (lane == 0 && a.dz_value) a.dz_value[row] = __fmul_rn(d, __fmul_rn(2.f, a.value_scale));
    }
    if (lane == 0 && a.advantage_out) a.advantage_out[row] = adv;
    if (lane != 0) { t_pol = 0.f; t_val = 0.f; }
    if (a.dz) {
      // d loss / d x_c = g * (onehot_c - p_c) - entropy_weight * dH/dx_c,
      // dH/dx_c = -p_c (log p_c + H); then / temperature for d / d z_c
      for (int c = lane; c < A; c += 32) {
        const float l = __fsub_rn(lg(c), lse);
        const float p = expf(l);
        float d = __fmul_rn(g, __fsub_rn(c == li ? 1.f : 0.f, p));
        if (a.entropy_weight != 0.f)
          d = __fadd_rn(d, __fmul_rn(a.entropy_weight, __fmul_rn(p, __fadd_rn(l, ent))));
        a.dz[base + c] = __fdiv_rn(d, a.temperature);
      }
    }
  }
  if (lane == 0) { s_v[0][warp] = t_pol; s_v[1][warp] = t_val; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float mine[2] = {0.f, 0.f};
    for (int w = 0; w < kPgRowsPerBlock; ++w) { mine[0] += s_v[0][w]; mine[1] += s_v[1][w]; }
    float* loss = a.loss;
    const float k = a.value_scale;
    finish_serial<2>(a.loss_partials, a.tile_counter, mine, [loss, k](const float (&t)[2]) {
      loss[0] = t[0];
      loss[1] = t[1] * k;
    });
  }
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_pg_returns(const rb200_pg_returns_args_t* a, void* stream) {
  if (!a) { set_last_error("rb200_pg_returns: args is null"); return RB200_E_INVALID; }
  if (a->n_traj <= 0 || !a->offsets || !a->reward || !a->returns) {
    set_last_error("rb200_pg_returns: need n_traj > 0, offsets, reward and returns");
    return RB200_E_INVALID;
  }
  if (a->norm < RB200_PG_NORM_NONE || a->norm > RB200_PG_NORM_SUBTRACT_MEAN) {
    set_last_error("rb200_pg_returns: unknown norm %d", a->norm);
    return RB200_E_INVALID;
  }
  return launch<pg_returns_kernel>(ceil_div(a->n_traj, kPgTrajPerBlock), 32 * kPgTrajPerBlock, 0,
                                   (cudaStream_t)stream, "pg_returns_kernel launch", *a);
}

extern "C" int rb200_pg_head(const rb200_pg_head_args_t* a, void* stream) {
  if (!a) { set_last_error("rb200_pg_head: args is null"); return RB200_E_INVALID; }
  if (a->rows <= 0 || a->num_actions < 1 || a->num_actions > 1024 || a->n_traj <= 0) {
    set_last_error("rb200_pg_head: need rows > 0, n_traj > 0 and 1 <= num_actions <= 1024 "
                   "(got %d, %d, %d)", a->rows, a->n_traj, a->num_actions);
    return RB200_E_INVALID;
  }
  if (!a->scores || !a->action || !a->offsets || !a->loss_partials || !a->loss ||
      !a->tile_counter) {
    set_last_error("rb200_pg_head: required pointer is null");
    return RB200_E_INVALID;
  }
  if (a->loss_kind != RB200_PG_LOSS_REINFORCE && a->loss_kind != RB200_PG_LOSS_PPO) {
    set_last_error("rb200_pg_head: unknown loss_kind %d", a->loss_kind);
    return RB200_E_INVALID;
  }
  if (a->loss_kind == RB200_PG_LOSS_PPO && !a->logged_log_prob) {
    set_last_error("rb200_pg_head: the PPO loss needs logged_log_prob");
    return RB200_E_INVALID;
  }
  switch (a->advantage_kind) {
    case RB200_PG_ADV_RETURNS:
      if (!a->returns || a->value) {
        set_last_error("rb200_pg_head: returns advantage needs returns and no value");
        return RB200_E_INVALID;
      }
      break;
    case RB200_PG_ADV_BASELINE:
      if (!a->returns || !a->value) {
        set_last_error("rb200_pg_head: baseline advantage needs returns and value");
        return RB200_E_INVALID;
      }
      break;
    case RB200_PG_ADV_TD:
      if (!a->value || !a->reward) {
        set_last_error("rb200_pg_head: TD advantage needs value and reward");
        return RB200_E_INVALID;
      }
      break;
    default:
      set_last_error("rb200_pg_head: unknown advantage_kind %d", a->advantage_kind);
      return RB200_E_INVALID;
  }
  return launch<pg_head_kernel>(ceil_div(a->rows, kPgRowsPerBlock), 32 * kPgRowsPerBlock, 0,
                                (cudaStream_t)stream, "pg_head_kernel launch", *a);
}
