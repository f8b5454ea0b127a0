// reagent_b200 -- fused SAC / TD3 update kernels over row tiles.
//
//   ac_critic_rows_kernel : TD target + both critic losses + critic backward (dZ chains)
//       SAC  reagent/training/sac_trainer.py:214-248   TD3  reagent/training/td3_trainer.py:138-178
//       actor forward on s' (Gaussian reparameterised / deterministic target actor + clipped
//       noise), q1_target / q2_target on (s', a'), min, entropy term, r + gamma*V*not_done,
//       then q1(s,a), q2(s,a), MSE and the dZ chains of both critics.
//   ac_actor_rows_kernel  : actor loss + backward THROUGH the (already updated) critics
//       SAC  sac_trainer.py:254-322 (incl. the alpha loss)   TD3  td3_trainer.py:181-194
//       actor forward on s, q1/q2 on (s, pi(s)), min-of-two, d loss / d action through the
//       critics (input gradient), Gaussian log-prob / tanh-squash backward
//       (reagent/models/actor.py:169-261), dZ chain of the actor.
// Everything is row-local; weight gradients are produced afterwards by rb200_mlp_wgrad.
#include "rb200_rows.cuh"

namespace rb200 {

struct AcDev {
  rb200_ac_args_t a;
  rb200_net_ws_t ws_actor, ws_q1, ws_q2;
  int ld_c, ld_h, ld_o;  // strides: critic-input tile, hidden tiles, actor-output tile
  int has_q2;
};

constexpr float kLogProbMin = -2.f, kLogProbMax = 2.f;   // reagent/models/actor.py:18-19
constexpr float kActEps = 1e-6f;                         // actor.py:165
constexpr float kLogSqrt2Pi = 0.91893853320467274178f;   // log(sqrt(2*pi)), actor.py:164

// Gaussian actor head for one row (GaussianFullyConnectedActor.forward + get_log_prob,
// reagent/models/actor.py:202-261).  out = [loc | scale_log] (2A), noise = N(0,1) draws.
// Writes the squashed action to act_out[0..A) and returns sum_j log_prob_j.
__device__ __forceinline__ float gaussian_head_row(const float* __restrict__ out,
                                                   const float* __restrict__ noise, int A,
                                                   float* __restrict__ act_out) {
  float lp = 0.f;
  for (int j = 0; j < A; ++j) {
    const float loc = out[j];
    const float sl = fminf(fmaxf(out[A + j], kLogProbMin), kLogProbMax);
    const float sigma = expf(sl);
    const float raw = __fadd_rn(loc, __fmul_rn(noise[j], sigma));
    const float a = fminf(fmaxf(tanhf(raw), -1.f + kActEps), 1.f - kActEps);
    // get_log_prob recomputes r from the squashed action (actor.py:243-261)
    const float r2 = __fdiv_rn(__fsub_rn(atanhf(a), loc), sigma);
    const float e = __fsub_rn(__fsub_rn(__fdiv_rn(-__fmul_rn(r2, r2), 2.f), sl), kLogSqrt2Pi);
    const float corr = logf(__fadd_rn(__fsub_rn(1.f, __fmul_rn(a, a)), kActEps));
    lp += __fsub_rn(e, corr);
    act_out[j] = a;
  }
  return lp;
}

// ---------------------------------------------------------------------------------------
// kWeighted: prioritized replay, a separate instantiation so that the unweighted kernel keeps
// its code.  Row b's loss element and dz are multiplied by a.sample_weight[b] (1 when that
// pointer is NULL) as the last operation, so unit weights reproduce the unweighted update bit
// for bit, and the row's TD error max_c |q_c(s,a) - y| (the twin-critic priority of Fujimoto,
// Meger & Precup 2020) goes to a.td_error_out.  Only the critics are weighted: the importance
// weights correct the bias of the critics' regression towards the TD target (Schaul et al.
// 2016); the actor and alpha losses do not regress on the sampled targets.
//
// kValueTarget: SAC with a state-value network (sac_trainer.py:214-217).  q1t is then the
// value-network target V' [S -> 1]; its forward on the s' columns replaces the actor forward
// on s', both target critics and the entropy term (no noise_next is read).  Everything from
// the TD target on is the same code.
template <int NT, int TM, int KC, bool kWeighted, bool kValueTarget = false>
__global__ void __launch_bounds__(NT, 1)
ac_critic_rows_kernel(const Mlp actor, const Mlp q1, const Mlp q2, const Mlp q1t, const Mlp q2t,
                      const AcDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  const rb200_ac_args_t& a = p.a;
  const int tid = threadIdx.x;
  const int ld_c = p.ld_c, ld_h = p.ld_h, ld_o = p.ld_o;
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* cin = Wst + 2 * wstage_floats<KC>();  // [R, ld_c] critic input cat(state, action)
  float* hA = cin + R * ld_c;
  float* hB = hA + R * ld_h;
  float* hC = hB + R * ld_h;
  float* aout = hC + R * ld_h;                 // [R, ld_o] actor output / small tiles
  float* v1 = aout + R * ld_o;                 // [R, 8] critic outputs (width 1, stride 8)
  float* v2 = v1 + R * 8;
  float* rowv = v2 + R * 8;                    // [4R]: target, logp, loss1, loss2
  const int B = a.batch, row0 = blockIdx.x * R;
  const int S = actor.dims[0];
  const int A = q1.dims[0] - S;
  const bool sac = a.algo == RB200_ALGO_SAC;

  if constexpr (kValueTarget) {
    // ---- V'(s'): the value-network target on next_state ----
    tile_load_rows<NT, R>(cin, ld_c, a.next_state, S, S, row0, B);
    __syncthreads();
    tile_mlp_fwd<NT, TM, KC>(q1t, cin, ld_c, hA, hB, ld_h, v1, 8, Wst, nullptr, row0, B);
    if (tid < R) {
      const int r = tid, row = row0 + r;
      float tgt = 0.f;
      if (row < B) {
        tgt = a.gamma > 0.f
                  ? __fadd_rn(a.reward[row], __fmul_rn(__fmul_rn(a.gamma, v1[r * 8]), a.not_terminal[row]))
                  : a.reward[row];                                    // :233-239
        if (a.td_target) a.td_target[row] = tgt;
      }
      rowv[r] = tgt;
    }
    __syncthreads();
  } else {
  // ---- next action from the (target) actor on next_state ----
  tile_load_rows<NT, R>(cin, ld_c, a.next_state, S, S, row0, B);
  __syncthreads();
  tile_mlp_fwd<NT, TM, KC>(actor, cin, ld_c, hA, hB, ld_h, aout, ld_o, Wst, nullptr, row0, B);
  if (tid < R) {
    const int r = tid, row = row0 + r;
    float lp = 0.f;
    if (row < B) {
      const float* nz = a.noise_next + (size_t)row * A;
      if (sac) {
        lp = gaussian_head_row(aout + r * ld_o, nz, A, cin + r * ld_c + S);
      } else {
        // td3_trainer.py:139-144
        for (int j = 0; j < A; ++j) {
          const float n = fminf(fmaxf(__fmul_rn(nz[j], a.noise_variance), -a.noise_clip), a.noise_clip);
          cin[r * ld_c + S + j] = fminf(fmaxf(__fadd_rn(aout[r * ld_o + j], n), -1.f), 1.f);
        }
      }
      if (a.next_action_out)
        for (int j = 0; j < A; ++j) a.next_action_out[(size_t)row * A + j] = cin[r * ld_c + S + j];
    } else {
      for (int j = 0; j < A; ++j) cin[r * ld_c + S + j] = 0.f;
    }
    for (int j = S + A; j < round_up4(S + A); ++j) cin[r * ld_c + j] = 0.f;
    rowv[R + r] = lp;
  }
  __syncthreads();

  // ---- target critics on (s', a') ----
  tile_mlp_fwd<NT, TM, KC>(q1t, cin, ld_c, hA, hB, ld_h, v1, 8, Wst, nullptr, row0, B);
  if (p.has_q2)
    tile_mlp_fwd<NT, TM, KC>(q2t, cin, ld_c, hA, hB, ld_h, v2, 8, Wst, nullptr, row0, B);
  if (tid < R) {
    const int r = tid, row = row0 + r;
    float tgt = 0.f;
    if (row < B) {
      float nsv = v1[r * 8];
      if (p.has_q2) nsv = fminf(nsv, v2[r * 8]);
      if (sac) {
        const float lpc = fminf(fmaxf(rowv[R + r], kLogProbMin), kLogProbMax);
        nsv = __fsub_rn(nsv, __fmul_rn(*a.alpha, lpc));               // sac_trainer.py:228-231
        tgt = a.gamma > 0.f
                  ? __fadd_rn(a.reward[row], __fmul_rn(__fmul_rn(a.gamma, nsv), a.not_terminal[row]))
                  : a.reward[row];                                    // :233-239
        if (a.log_prob_out) a.log_prob_out[row] = rowv[R + r];
      } else {
        tgt = __fadd_rn(a.reward[row], __fmul_rn(__fmul_rn(a.gamma, nsv), a.not_terminal[row]));
      }
      if (a.td_target) a.td_target[row] = tgt;
    }
    rowv[r] = tgt;
  }
  __syncthreads();
  }  // !kValueTarget

  // ---- critics on (s, a): loss + backward ----
  {
    const int D = S + A, D4 = round_up4(D);
    for (int idx = tid; idx < R * D4; idx += NT) {
      const int r = idx / D4, c = idx - r * D4;
      float v = 0.f;
      if (row0 + r < B) {
        if (c < S) v = a.state[(size_t)(row0 + r) * S + c];
        else if (c < D) v = a.action[(size_t)(row0 + r) * A + (c - S)];
      }
      cin[r * ld_c + c] = v;
    }
    __syncthreads();
    if (p.ws_q1.input) tile_store_rows<NT, R>(cin, ld_c, p.ws_q1.input, D, D, row0, B);
  }
  float td_err = 0.f;  // kWeighted: row tid's max_c |q_c - y|, kept across both critics
  for (int which = 0; which < (p.has_q2 ? 2 : 1); ++which) {
    const Mlp& q = which ? q2 : q1;
    const rb200_net_ws_t& ws = which ? p.ws_q2 : p.ws_q1;
    float* v = which ? v2 : v1;
    tile_mlp_fwd<NT, TM, KC>(q, cin, ld_c, hA, hB, ld_h, v, 8, Wst, ws.hidden, row0, B);
    if (tid < R) {
      const int r = tid, row = row0 + r;
      float le = 0.f, g = 0.f;
      if (row < B) {
        const float qv = v[r * 8];
        const float d = __fsub_rn(qv, rowv[r]);
        le = d * d;                                   // F.mse_loss, mean over B
        g = 2.f / (float)B * d;
        const int lact = q.act[q.n_layers - 1];
        if (lact != RB200_ACT_LINEAR) g *= act_bwd_from_out(qv, lact);
        if (kWeighted) {
          const float w = a.sample_weight ? a.sample_weight[row] : 1.f;
          le = __fmul_rn(le, w);
          g = __fmul_rn(g, w);
          // torch.maximum: a NaN from either critic propagates (status 3 on write-back)
          const float e = fabsf(d);
          td_err = (which == 0 || e > td_err || e != e) ? e : td_err;
        }
        float* qo = which ? a.q2_value : a.q1_value;
        if (qo) qo[row] = qv;
      }
      aout[r * ld_o + 0] = g;                         // dz of the (1-wide) last layer
      aout[r * ld_o + 1] = 0.f; aout[r * ld_o + 2] = 0.f; aout[r * ld_o + 3] = 0.f;
      rowv[(2 + which) * R + r] = le;
    }
    __syncthreads();
    tile_mlp_bwd<NT, TM, KC>(q, aout, ld_o, hA, hB, hC, ld_h, Wst, ws.hidden, ws.dz, row0, B,
                             nullptr, 0, 0, 0);
    __syncthreads();
  }
  if (kWeighted && a.td_error_out && tid < R && row0 + tid < B) a.td_error_out[row0 + tid] = td_err;
  if (tid == 0) {
    float s1 = 0.f, s2 = 0.f;
    for (int r = 0; r < R; ++r) { s1 += rowv[2 * R + r]; s2 += rowv[3 * R + r]; }
    finish_serial<2>(a.loss_partials, a.tile_counter, {s1, s2}, [&](const float (&tot)[2]) {
      a.loss[0] = tot[0] / (float)B;
      a.loss[1] = tot[1] / (float)B;
    });
  }
}

// ---------------------------------------------------------------------------------------
// kCrr: Critic Regularized Regression weighting of the SAC actor loss (sac_trainer.py:23-48,
// :265-276).  vn is the current value network V [S -> 1]; the row's loss element is
// -clamp(lp) * w(min_q - V(s)), w detached, so the only gradient is through log_prob and the
// input-gradient pass through the critics is skipped (dact stays zero).
template <int NT, int TM, int KC, bool kCrr = false>
__global__ void __launch_bounds__(NT, 1)
ac_actor_rows_kernel(const Mlp actor, const Mlp q1, const Mlp q2, const Mlp vn, const AcDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  const rb200_ac_args_t& a = p.a;
  const int tid = threadIdx.x;
  const int ld_c = p.ld_c, ld_h = p.ld_h, ld_o = p.ld_o;
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* cin = Wst + 2 * wstage_floats<KC>();
  float* hA = cin + R * ld_c;
  float* hB = hA + R * ld_h;
  float* hC = hB + R * ld_h;
  float* aout = hC + R * ld_h;   // [R, ld_o] actor output, later its dz
  float* dact = aout + R * ld_o; // [R, ld_o] d loss / d action (sum over critics)
  float* dtmp = dact + R * ld_o; // [R, ld_o] per-critic input gradient / 1-wide dz tile
  float* v1 = dtmp + R * ld_o;
  float* v2 = v1 + R * 8;
  float* rowv = v2 + R * 8;      // [4R]: logp, wq1, wq2, actor loss element
  const int B = a.batch, row0 = blockIdx.x * R;
  const int S = actor.dims[0];
  const int A = q1.dims[0] - S;
  const bool sac = a.algo == RB200_ALGO_SAC;
  const float invB = 1.f / (float)B;

  // ---- actor on state (saved for its backward) ----
  tile_load_rows<NT, R>(cin, ld_c, a.state, S, S, row0, B);
  __syncthreads();
  tile_mlp_fwd<NT, TM, KC>(actor, cin, ld_c, hA, hB, ld_h, aout, ld_o, Wst, p.ws_actor.hidden,
                           row0, B);
  if (tid < R) {
    const int r = tid, row = row0 + r;
    float lp = 0.f;
    if (row < B) {
      if (sac) lp = gaussian_head_row(aout + r * ld_o, a.noise_cur + (size_t)row * A, A, cin + r * ld_c + S);
      else for (int j = 0; j < A; ++j) cin[r * ld_c + S + j] = aout[r * ld_o + j];
      if (a.next_action_out)
        for (int j = 0; j < A; ++j) a.next_action_out[(size_t)row * A + j] = cin[r * ld_c + S + j];
      if (a.log_prob_out) a.log_prob_out[row] = lp;
    } else {
      for (int j = 0; j < A; ++j) cin[r * ld_c + S + j] = 0.f;
    }
    for (int j = S + A; j < round_up4(S + A); ++j) cin[r * ld_c + j] = 0.f;
    rowv[r] = lp;
  }
  __syncthreads();

  // ---- critics (updated weights) on (s, pi(s)); hidden activations to their workspaces ----
  tile_mlp_fwd<NT, TM, KC>(q1, cin, ld_c, hA, hB, ld_h, v1, 8, Wst, p.ws_q1.hidden, row0, B);
  const bool use_q2 = sac && p.has_q2;  // TD3's actor loss uses q1 only (td3_trainer.py:183-184)
  if (use_q2)
    tile_mlp_fwd<NT, TM, KC>(q2, cin, ld_c, hA, hB, ld_h, v2, 8, Wst, p.ws_q2.hidden, row0, B);
  // V(s) on the state columns of cin.  Exact despite the action columns after S: the staged
  // weights are zero for k >= S and the actions are finite.
  if constexpr (kCrr)
    tile_mlp_fwd<NT, TM, KC>(vn, cin, ld_c, hA, hB, ld_h, dtmp, ld_o, Wst, nullptr, row0, B);
  if (tid < R) {
    const int r = tid, row = row0 + r;
    float w1 = 0.f, w2 = 0.f, le = 0.f;
    if (row < B) {
      const float qa = v1[r * 8];
      float minq = qa;
      if (use_q2) {
        // torch.min(a, b) backward: ties split the gradient evenly
        const float qb = v2[r * 8];
        if (qa < qb) w1 = 1.f; else if (qa > qb) w2 = 1.f; else { w1 = 0.5f; w2 = 0.5f; }
        minq = fminf(qa, qb);
        const float lpc = fminf(fmaxf(rowv[r], kLogProbMin), kLogProbMax);
        le = __fsub_rn(__fmul_rn(*a.alpha, lpc), minq);       // sac_trainer.py:278
      } else if (sac) {
        w1 = 1.f;
        const float lpc = fminf(fmaxf(rowv[r], kLogProbMin), kLogProbMax);
        le = __fsub_rn(__fmul_rn(*a.alpha, lpc), qa);
      } else {
        w1 = 1.f;
        le = -qa;                                             // td3_trainer.py:184
      }
      if (a.min_q_out) a.min_q_out[row] = minq;
      if constexpr (kCrr) {
        // CRRWeightFn.get_weight_from_advantage (sac_trainer.py:38-48); w1 carries w
        const float adv = __fsub_rn(minq, dtmp[r * ld_o]);
        if (a.crr_mode == RB200_CRR_INDICATOR) {
          w1 = adv >= a.crr_threshold ? 1.f : 0.f;
        } else {
          w1 = expf(__fdiv_rn(adv, a.crr_beta));
          if (a.crr_clamp > 0.f) w1 = fminf(fmaxf(w1, 0.f), a.crr_clamp);
        }
        le = -__fmul_rn(fminf(fmaxf(rowv[r], kLogProbMin), kLogProbMax), w1);
      }
    }
    rowv[R + r] = w1;
    rowv[2 * R + r] = w2;
    rowv[3 * R + r] = le;
  }
  __syncthreads();

  // ---- d loss / d action through the critics: loss = mean(... - minQ) ----
  for (int which = 0; which < (kCrr ? 0 : (use_q2 ? 2 : 1)); ++which) {
    const Mlp& q = which ? q2 : q1;
    const rb200_net_ws_t& ws = which ? p.ws_q2 : p.ws_q1;
    const float* v = which ? v2 : v1;
    if (tid < R) {
      const int r = tid;
      float g = -invB * rowv[(1 + which) * R + r];
      const int lact = q.act[q.n_layers - 1];
      if (lact != RB200_ACT_LINEAR) g *= act_bwd_from_out(v[r * 8], lact);
      dtmp[r * ld_o + 0] = (row0 + r < B) ? g : 0.f;
      dtmp[r * ld_o + 1] = 0.f; dtmp[r * ld_o + 2] = 0.f; dtmp[r * ld_o + 3] = 0.f;
    }
    __syncthreads();
    float* din = which ? dtmp + 4 : dact;  // q2's input gradient lands after the dz quad
    // input gradient of the action columns [S, S+A)
    tile_mlp_bwd<NT, TM, KC>(q, dtmp, ld_o, hA, hB, hC, ld_h, Wst, ws.hidden, nullptr, row0, B,
                             which ? (dtmp + 8) : dact, ld_o, S, A);
    __syncthreads();
    if (which) {
      const int A4 = round_up4(A);
      for (int idx = tid; idx < R * A4; idx += NT) {
        const int r = idx / A4, c = idx - r * A4;
        dact[r * ld_o + c] += dtmp[r * ld_o + 8 + c];
      }
      __syncthreads();
    }
    (void)din;
  }

  // ---- actor output gradient ----
  if (tid < R) {
    const int r = tid, row = row0 + r;
    const int NO = actor.dims[actor.n_layers];
    const int NO4 = round_up4(NO);
    if (row < B) {
      if (sac) {
        const float lp = rowv[r];
        const bool in_clamp = (lp >= kLogProbMin) && (lp <= kLogProbMax);
        float glp = (a.backprop_through_log_prob && in_clamp) ? (*a.alpha) * invB : 0.f;
        if constexpr (kCrr) glp = in_clamp ? -(rowv[R + r] * invB) : 0.f;
        const float* nz = a.noise_cur + (size_t)row * A;
        for (int j = 0; j < A; ++j) {
          const float loc = aout[r * ld_o + j];
          const float slr = aout[r * ld_o + A + j];
          const float sl = fminf(fmaxf(slr, kLogProbMin), kLogProbMax);
          const float sigma = expf(sl);
          const float raw = __fadd_rn(loc, __fmul_rn(nz[j], sigma));
          const float t = tanhf(raw);
          const float av = fminf(fmaxf(t, -1.f + kActEps), 1.f - kActEps);
          const float r2 = (atanhf(av) - loc) / sigma;
          const float om = 1.f - av * av;
          // d lp_j / d a  (through atanh and the squash correction)
          const float dlp_da = -r2 / (sigma * om) + 2.f * av / (om + kActEps);
          float ga = dact[r * ld_o + j] + glp * dlp_da;
          if (!(t >= -1.f + kActEps && t <= 1.f - kActEps)) ga = 0.f;   // clamp backward
          const float graw = ga * (1.f - t * t);
          const float dloc = graw + glp * (r2 / sigma);
          float dsl = graw * (nz[j] * sigma) + glp * (r2 * r2 - 1.f);
          if (!(slr >= kLogProbMin && slr <= kLogProbMax)) dsl = 0.f;     // clamp backward
          aout[r * ld_o + j] = dloc;
          aout[r * ld_o + A + j] = dsl;
        }
      } else {
        const int lact = actor.act[actor.n_layers - 1];
        for (int j = 0; j < A; ++j) {
          const float y = aout[r * ld_o + j];
          aout[r * ld_o + j] = dact[r * ld_o + j] * act_bwd_from_out(y, lact);
        }
      }
      for (int j = NO; j < NO4; ++j) aout[r * ld_o + j] = 0.f;
    } else {
      for (int j = 0; j < NO4; ++j) aout[r * ld_o + j] = 0.f;
    }
  }
  __syncthreads();
  tile_mlp_bwd<NT, TM, KC>(actor, aout, ld_o, hA, hB, hC, ld_h, Wst, p.ws_actor.hidden,
                           p.ws_actor.dz, row0, B, nullptr, 0, 0, 0);

  // ---- losses: actor loss mean, alpha loss / gradient (sac_trainer.py:311-322) ----
  if (tid == 0) {
    float s = 0.f, ent = 0.f;
    for (int r = 0; r < R; ++r) {
      s += rowv[3 * R + r];
      if (sac && row0 + r < B)
        ent += fminf(fmaxf(rowv[r], kLogProbMin), kLogProbMax) + a.target_entropy;
    }
    finish_serial<2>(a.loss_partials, a.tile_counter, {s, ent}, [&](const float (&tot)[2]) {
      a.loss[0] = tot[0] * invB;
      if (sac && a.alpha_grad) {
        const float m = tot[1] * invB;        // mean(clamp(logp) + target_entropy)
        a.alpha_grad[0] = -m;                 // d/d log_alpha of -(log_alpha * m)
        if (a.log_alpha) a.loss[1] = -((*a.log_alpha) * m);
      }
    });
  }
}

// ---------------------------------------------------------------------------------------
// Value step (sac_trainer.py:329-343): V(s) forward with the hidden activations saved, the
// per-row target min_q (logged_action_uniform_prior) or min_q - alpha * clamp(log_prob) with
// the post-update alpha, MSE against the detached target and the value network's dZ chain.
template <int NT, int TM, int KC>
__global__ void __launch_bounds__(NT, 1)
ac_value_rows_kernel(const Mlp vn, const AcDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  const rb200_ac_args_t& a = p.a;
  const int tid = threadIdx.x;
  const int ld_c = p.ld_c, ld_h = p.ld_h;
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* cin = Wst + 2 * wstage_floats<KC>();  // [R, ld_c] state
  float* hA = cin + R * ld_c;
  float* hB = hA + R * ld_h;
  float* hC = hB + R * ld_h;
  float* v = hC + R * ld_h;                     // [R, 8] V(s), then its dz
  float* rowv = v + R * 8;                      // [R] loss element
  const int B = a.batch, row0 = blockIdx.x * R;
  const int S = vn.dims[0];
  const rb200_net_ws_t& ws = p.ws_q1;

  tile_load_rows<NT, R>(cin, ld_c, a.state, S, S, row0, B);
  __syncthreads();
  tile_mlp_fwd<NT, TM, KC>(vn, cin, ld_c, hA, hB, ld_h, v, 8, Wst, ws.hidden, row0, B);
  if (tid < R) {
    const int r = tid, row = row0 + r;
    float le = 0.f, g = 0.f;
    if (row < B) {
      const float sv = v[r * 8];
      float tgt = a.min_q_out[row];
      if (!a.logged_action_uniform_prior) {
        const float lpc = fminf(fmaxf(a.log_prob_out[row], kLogProbMin), kLogProbMax);
        tgt = __fsub_rn(tgt, __fmul_rn(*a.alpha, lpc));
      }
      const float d = __fsub_rn(sv, tgt);
      le = d * d;                                     // F.mse_loss, mean over B
      g = 2.f / (float)B * d;
      const int lact = vn.act[vn.n_layers - 1];
      if (lact != RB200_ACT_LINEAR) g *= act_bwd_from_out(sv, lact);
    }
    v[r * 8] = g;                                     // dz of the (1-wide) last layer
    rowv[r] = le;
  }
  __syncthreads();
  tile_mlp_bwd<NT, TM, KC>(vn, v, 8, hA, hB, hC, ld_h, Wst, ws.hidden, ws.dz, row0, B,
                           nullptr, 0, 0, 0);
  if (tid == 0) {
    float s = 0.f;
    for (int r = 0; r < R; ++r) s += rowv[r];
    finish_serial<1>(a.loss_partials, a.tile_counter, {s}, [&](const float (&tot)[1]) {
      a.loss[0] = tot[0] / (float)B;
    });
  }
}

// A state-value network V [S -> 1] for the step that `who` names.
static int check_value_net(const rb200_mlp_t* v, int S, const rb200_ac_args_t* a, const char* who) {
  if (!v) { set_last_error("%s: value network descriptor is null", who); return RB200_E_INVALID; }
  if (int rc = validate_mlp(v, who)) return rc;
  if (v->dims[0] != S || v->dims[v->n_layers] != 1) { set_last_error("%s: value network must map the state (%d wide) to 1 output (got %d -> %d)", who, S, v->dims[0], v->dims[v->n_layers]); return RB200_E_INVALID; }
  if (a->algo != RB200_ALGO_SAC) { set_last_error("%s: a value network needs SAC (TD3 has none)", who); return RB200_E_INVALID; }
  return RB200_OK;
}

static int ac_common_checks(const rb200_mlp_t* actor, const rb200_mlp_t* q1, const rb200_mlp_t* q2,
                            const rb200_ac_args_t* a) {
  if (!actor || !q1 || !a) { set_last_error("actor-critic step: null argument"); return RB200_E_INVALID; }
  if (int rc = validate_mlp(actor, "actor")) return rc;
  if (int rc = validate_mlp(q1, "q1_network")) return rc;
  if (q2) if (int rc = validate_mlp(q2, "q2_network")) return rc;
  const int S = actor->dims[0], A = q1->dims[0] - S;
  if (A <= 0) { set_last_error("critic input must be cat(state, action)"); return RB200_E_INVALID; }
  const int NO = actor->dims[actor->n_layers];
  if (a->algo == RB200_ALGO_SAC && NO != 2 * A) { set_last_error("Gaussian actor must output 2*action_dim (got %d, A=%d)", NO, A); return RB200_E_INVALID; }
  if (a->algo == RB200_ALGO_TD3 && NO != A) { set_last_error("deterministic actor must output action_dim"); return RB200_E_INVALID; }
  if (q1->dims[q1->n_layers] != 1 || (q2 && q2->dims[q2->n_layers] != 1)) { set_last_error("critics must have a single output"); return RB200_E_INVALID; }
  if (q2 && q2->dims[0] != q1->dims[0]) { set_last_error("q1 / q2 input widths differ"); return RB200_E_INVALID; }
  if (a->batch <= 0 || !a->state || !a->loss_partials || !a->loss || !a->tile_counter) { set_last_error("actor-critic step: required pointer is null"); return RB200_E_INVALID; }
  if (a->algo == RB200_ALGO_SAC && !a->alpha) { set_last_error("SAC needs the entropy temperature pointer"); return RB200_E_INVALID; }
  return RB200_OK;
}

// `value`: the value network the launch runs (critic step: the value target; actor step with
// CRR: the value network), or NULL.
static RowsCfg ac_cfg(const rb200_mlp_t* actor, const rb200_mlp_t* q1, const rb200_mlp_t* q2,
                      const rb200_mlp_t* value, int batch, int n_out_tiles, int* ld_o) {
  int hmax = mlp_max_hidden(actor);
  const int h1 = mlp_max_hidden(q1);
  hmax = h1 > hmax ? h1 : hmax;
  if (q2) { const int h2 = mlp_max_hidden(q2); hmax = h2 > hmax ? h2 : hmax; }
  if (value) { const int hv = mlp_max_hidden(value); hmax = hv > hmax ? hv : hmax; }
  const int NO = actor->dims[actor->n_layers];
  *ld_o = round_up4(NO > 8 ? NO : 8) + 12;  // room for a 1-wide dz quad + an A-wide gradient
  return pick_rows_cfg(batch, q1->dims[0], hmax, 1, 3, n_out_tiles * (*ld_o) + 16 + 4, 0);
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_ac_critic_step(const rb200_mlp_t* actor, const rb200_mlp_t* q1,
                                    const rb200_mlp_t* q2, const rb200_mlp_t* q1_target,
                                    const rb200_mlp_t* q2_target, const rb200_ac_args_t* args,
                                    const rb200_net_ws_t* ws_q1, const rb200_net_ws_t* ws_q2,
                                    void* stream) {
  if (int rc = ac_common_checks(actor, q1, q2, args)) return rc;
  const rb200_mlp_t* vt = args->value_target;
  if (vt) {
    // the value target replaces the actor forward on s' and both q targets
    if (int rc = check_value_net(vt, actor->dims[0], args, "value_network_target")) return rc;
    if (!ws_q1 || (q2 && !ws_q2)) { set_last_error("critic step: workspaces required"); return RB200_E_INVALID; }
    if (!args->action || !args->next_state || !args->reward || !args->not_terminal) { set_last_error("critic step: batch pointer is null"); return RB200_E_INVALID; }
  } else {
    if (!q1_target || (q2 && !q2_target) || !ws_q1 || (q2 && !ws_q2)) { set_last_error("critic step: target nets / workspaces required"); return RB200_E_INVALID; }
    if (int rc = validate_mlp(q1_target, "q1_network_target")) return rc;
    if (q2) if (int rc = validate_mlp(q2_target, "q2_network_target")) return rc;
    if (!args->action || !args->next_state || !args->reward || !args->not_terminal || !args->noise_next) { set_last_error("critic step: batch pointer is null"); return RB200_E_INVALID; }
  }
  AcDev p;
  p.a = *args;
  p.ws_q1 = *ws_q1;
  p.ws_q2 = q2 ? *ws_q2 : *ws_q1;
  p.ws_actor = *ws_q1;
  p.has_q2 = q2 ? 1 : 0;
  RowsCfg cfg = ac_cfg(actor, q1, q2, vt, args->batch, 1, &p.ld_o);
  if (cfg.tm == 0) { set_last_error("actor-critic tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_c = cfg.ld_in;
  p.ld_h = cfg.ld_h;
  const Mlp ma = make_mlp(actor), m1 = make_mlp(q1), m2 = make_mlp(q2 ? q2 : q1);
  // with a value network, t1 carries the value target (t2 is unused)
  const Mlp t1 = make_mlp(vt ? vt : q1_target);
  const Mlp t2 = make_mlp(vt ? vt : (q2 ? q2_target : q1_target));
  const int grid = ceil_div(args->batch, rows_per_tile(cfg));
  cudaStream_t st = (cudaStream_t)stream;
  // prioritized replay: weights and / or TD errors take the weighted instantiation
  const bool weighted = args->sample_weight || args->td_error_out;
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    const char* what = "ac_critic_rows_kernel launch";
    if (vt)
      return weighted
                 ? launch<ac_critic_rows_kernel<NT(), 4, KC(), true, true>>(
                       grid, NT(), cfg.smem_bytes, st, what, ma, m1, m2, t1, t2, p)
                 : launch<ac_critic_rows_kernel<NT(), 4, KC(), false, true>>(
                       grid, NT(), cfg.smem_bytes, st, what, ma, m1, m2, t1, t2, p);
    return weighted
               ? launch<ac_critic_rows_kernel<NT(), 4, KC(), true>>(grid, NT(), cfg.smem_bytes, st,
                                                                     what, ma, m1, m2, t1, t2, p)
               : launch<ac_critic_rows_kernel<NT(), 4, KC(), false>>(grid, NT(), cfg.smem_bytes, st,
                                                                      what, ma, m1, m2, t1, t2, p);
  });
}

extern "C" int rb200_ac_actor_step(const rb200_mlp_t* actor, const rb200_mlp_t* q1,
                                   const rb200_mlp_t* q2, const rb200_ac_args_t* args,
                                   const rb200_net_ws_t* ws_actor, const rb200_net_ws_t* ws_q1,
                                   const rb200_net_ws_t* ws_q2, void* stream) {
  if (int rc = ac_common_checks(actor, q1, q2, args)) return rc;
  if (!ws_actor || !ws_q1 || (q2 && !ws_q2)) { set_last_error("actor step: workspaces required"); return RB200_E_INVALID; }
  if (args->algo == RB200_ALGO_SAC && !args->noise_cur) { set_last_error("SAC actor step needs noise_cur"); return RB200_E_INVALID; }
  const bool crr = args->crr_mode != RB200_CRR_NONE;
  if (crr) {
    if (args->crr_mode != RB200_CRR_INDICATOR && args->crr_mode != RB200_CRR_EXPONENT) { set_last_error("actor step: unknown crr_mode %d", args->crr_mode); return RB200_E_INVALID; }
    if (!args->value_net) { set_last_error("actor step: CRR needs a value network"); return RB200_E_INVALID; }
    if (int rc = check_value_net(args->value_net, actor->dims[0], args, "value_network")) return rc;
    if (!args->backprop_through_log_prob) { set_last_error("actor step: the CRR loss has no gradient without backprop_through_log_prob"); return RB200_E_INVALID; }
    if (args->crr_mode == RB200_CRR_EXPONENT && !(args->crr_beta > 0.f)) { set_last_error("actor step: crr_beta must be > 0"); return RB200_E_INVALID; }
  }
  AcDev p;
  p.a = *args;
  p.ws_actor = *ws_actor;
  p.ws_q1 = *ws_q1;
  p.ws_q2 = q2 ? *ws_q2 : *ws_q1;
  p.has_q2 = q2 ? 1 : 0;
  RowsCfg cfg = ac_cfg(actor, q1, q2, crr ? args->value_net : nullptr, args->batch, 3, &p.ld_o);
  if (cfg.tm == 0) { set_last_error("actor-critic tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_c = cfg.ld_in;
  p.ld_h = cfg.ld_h;
  const Mlp ma = make_mlp(actor), m1 = make_mlp(q1), m2 = make_mlp(q2 ? q2 : q1);
  const Mlp mv = make_mlp(crr ? args->value_net : q1);
  const int grid = ceil_div(args->batch, rows_per_tile(cfg));
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    const char* what = "ac_actor_rows_kernel launch";
    return crr ? launch<ac_actor_rows_kernel<NT(), 4, KC(), true>>(grid, NT(), cfg.smem_bytes, st,
                                                                   what, ma, m1, m2, mv, p)
               : launch<ac_actor_rows_kernel<NT(), 4, KC()>>(grid, NT(), cfg.smem_bytes, st, what,
                                                             ma, m1, m2, mv, p);
  });
}

extern "C" int rb200_ac_value_step(const rb200_mlp_t* value, const rb200_ac_args_t* args,
                                   const rb200_net_ws_t* ws_value, void* stream) {
  if (!args) { set_last_error("value step: null argument"); return RB200_E_INVALID; }
  if (!value) { set_last_error("value step: value network descriptor is null"); return RB200_E_INVALID; }
  if (int rc = check_value_net(value, value->dims[0], args, "value_network")) return rc;
  if (!ws_value || args->batch <= 0 || !args->state || !args->min_q_out || !args->loss_partials || !args->loss || !args->tile_counter) { set_last_error("value step: required pointer is null"); return RB200_E_INVALID; }
  if (!args->logged_action_uniform_prior && (!args->log_prob_out || !args->alpha)) { set_last_error("value step: the entropy target needs log_prob_out and alpha"); return RB200_E_INVALID; }
  AcDev p;
  p.a = *args;
  p.ws_actor = p.ws_q1 = p.ws_q2 = *ws_value;
  p.has_q2 = 0;
  p.ld_o = 8;
  RowsCfg cfg = pick_rows_cfg(args->batch, value->dims[0], mlp_max_hidden(value), 1, 3, 8 + 1, 0);
  if (cfg.tm == 0) { set_last_error("value tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_c = cfg.ld_in;
  p.ld_h = cfg.ld_h;
  const Mlp mv = make_mlp(value);
  const int grid = ceil_div(args->batch, rows_per_tile(cfg));
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    return launch<ac_value_rows_kernel<NT(), 4, KC()>>(grid, NT(), cfg.smem_bytes, st,
                                                       "ac_value_rows_kernel launch", mv, p);
  });
}
