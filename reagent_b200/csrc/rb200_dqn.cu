// reagent_b200 -- fused DQN TD-target / loss / backward kernel (K2 + K2').
//
// One launch, one CTA per tile of R batch rows, everything row-local:
//   q(s'), q_target(s')            dqn_trainer.py:157-164  (get_detached_model_outputs)
//   mask -> -1e9, argmax / gather  dqn_trainer_base.py:33-77
//   r + boost, gamma^k             dqn_trainer_base.py:216-241, dqn_trainer.py:166-177
//   target = r + disc*next_q*nt    dqn_trainer.py:229-231
//   q(s), sum(q*action)            dqn_trainer.py:234-237
//   mse | smooth_l1 (mean)         dqn_trainer.py:238
//   d loss / d pre-activations of every layer of q_network (autograd's backward)
// Algorithmic work per launch (SURVEY.md 8d, K2+K2'):
//   FLOPs = 2*B*Sigma(net)*(3 fwd) + 2*B*Sigma(net minus first layer)*(1 bwd-dX)
//   bytes = B*(2S + 2A + 3)*4 read + B*(sum hidden + sum dz + A)*4 written + params.
#include "rb200_rows.cuh"

namespace rb200 {

struct DqnDev {
  rb200_dqn_args_t a;
  rb200_net_ws_t ws;
  int ld_in, ld_h, ld_q;
};

// kWeighted: prioritized-replay importance weights (a.sample_weight), a separate instantiation so
// that the unweighted kernels stay exactly as they are
template <int NT, int TM, int KC, bool kWeighted>
__global__ void __launch_bounds__(NT, 1)
dqn_td_rows_kernel(const Mlp q, const Mlp qt, const DqnDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  const rb200_dqn_args_t& a = p.a;
  const int tid = threadIdx.x;
  const int ld_in = p.ld_in, ld_h = p.ld_h, ld_q = p.ld_q;
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* xin = Wst + 2 * wstage_floats<KC>();
  float* hA = xin + R * ld_in;
  float* hB = hA + R * ld_h;
  float* hC = hB + R * ld_h;
  float* qa = hC + R * ld_h;   // q(s') online, later dz of the last layer
  float* qb = qa + R * ld_q;   // q_target(s')
  float* qc = qb + R * ld_q;   // q(s)
  float* rowv = qc + R * ld_q; // [2R] per-row scalars: td target, per-row loss
  const int B = a.batch;
  const int row0 = blockIdx.x * R;
  const int L = q.n_layers;
  const int S = q.dims[0], A = q.dims[L];

  // ---- TD target on next_state (no grad) ----
  tile_load_rows<NT, R>(xin, ld_in, a.next_state, S, S, row0, B);
  __syncthreads();
  if (a.double_q)
    tile_mlp_fwd<NT, TM, KC>(q, xin, ld_in, hA, hB, ld_h, qa, ld_q, Wst, nullptr, row0, B);
  tile_mlp_fwd<NT, TM, KC>(qt, xin, ld_in, hA, hB, ld_h, qb, ld_q, Wst, nullptr, row0, B);
  if (tid < R) {
    const int r = tid, row = row0 + r;
    float tgt = 0.f;
    if (row < B) {
      const float* mask = a.maxq ? a.possible_next_actions_mask : a.next_action;
      float best = 0.f, sel = 0.f;
      int bi = -1;
      for (int c = 0; c < A; ++c) {
        const float m = mask ? mask[(size_t)row * A + c] : 1.f;
        const float pen = -1e9f * (1.f - m);
        const float vt = qb[r * ld_q + c] + pen;
        const float key = a.double_q ? (qa[r * ld_q + c] + pen) : vt;
        if (bi < 0 || key > best) { best = key; bi = c; sel = vt; }
      }
      float rew = a.reward[row];
      if (a.reward_boost) {
        float bsum = 0.f;
        for (int c = 0; c < A; ++c) bsum += a.action[(size_t)row * A + c] * a.reward_boost[c];
        rew += bsum;
      }
      const float disc = (a.discount_mode == RB200_DISCOUNT_POW)
                             ? powf(a.gamma, a.discount_src[row]) : a.gamma;
      const float filtered = sel * a.not_terminal[row];
      tgt = rew + disc * filtered;
      if (a.td_target) a.td_target[row] = tgt;
      if (a.next_action_idx) a.next_action_idx[row] = bi;
    }
    rowv[r] = tgt;
  }
  __syncthreads();

  // ---- online network on state (with grad): save hidden activations ----
  tile_load_rows<NT, R>(xin, ld_in, a.state, S, S, row0, B);
  __syncthreads();
  tile_mlp_fwd<NT, TM, KC>(q, xin, ld_in, hA, hB, ld_h, qc, ld_q, Wst,
                       a.do_backward ? p.ws.hidden : nullptr, row0, B);
  if (a.all_action_scores) tile_store_rows<NT, R>(qc, ld_q, a.all_action_scores, A, A, row0, B);

  // ---- loss and d loss / d q_network output ----
  if (tid < R) {
    const int r = tid, row = row0 + r;
    const int A4 = round_up4(A);
    float le = 0.f;
    if (row < B) {
      float qsel = 0.f;
      for (int c = 0; c < A; ++c) qsel += qc[r * ld_q + c] * a.action[(size_t)row * A + c];
      const float d = qsel - rowv[r];
      const float invB = 1.f / (float)B;
      float g;
      if (a.loss_kind == RB200_LOSS_HUBER) {
        const float ad = fabsf(d);
        le = ad < 1.f ? 0.5f * d * d : ad - 0.5f;
        g = (d < -1.f) ? -invB : (d > 1.f ? invB : invB * d);
      } else {
        le = d * d;
        g = 2.f * invB * d;
      }
      if (kWeighted) {
        const float w = a.sample_weight[row];
        le *= w;
        g *= w;
      }
      if (a.q_selected) a.q_selected[row] = qsel;
      const int lact = q.act[L - 1];
      for (int c = 0; c < A4; ++c) {
        float v = 0.f;
        if (c < A) {
          v = g * a.action[(size_t)row * A + c];
          if (lact != RB200_ACT_LINEAR) v *= act_bwd_from_out(qc[r * ld_q + c], lact);
        }
        qa[r * ld_q + c] = v;
      }
    } else {
      for (int c = 0; c < A4; ++c) qa[r * ld_q + c] = 0.f;
    }
    rowv[R + r] = le;
  }
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
    for (int r = 0; r < R; ++r) s += rowv[R + r];
    finish_serial<1>(a.loss_partials, a.tile_counter, {s},
                     [&](const float (&tot)[1]) { *a.loss = tot[0] / (float)B; });
  }

  // ---- backward: dZ chain of q_network ----
  if (a.do_backward)
    tile_mlp_bwd<NT, TM, KC>(q, qa, ld_q, hA, hB, hC, ld_h, Wst, p.ws.hidden, p.ws.dz, row0, B,
                         nullptr, 0, 0, 0);
}

static RowsCfg dqn_cfg(const rb200_mlp_t* q, int batch, int* ld_q) {
  const int A = q->dims[q->n_layers];
  *ld_q = round_up4(A) + 4;
  // 1 input tile, 3 hidden tiles, 3 q tiles + 2 scalars per row
  return pick_rows_cfg(batch, q->dims[0], mlp_max_hidden(q), 1, 3, 3 * (*ld_q) + 2, 0);
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_dqn_td_step(const rb200_mlp_t* q_net, const rb200_mlp_t* q_target,
                                 const rb200_dqn_args_t* args, const rb200_net_ws_t* ws,
                                 void* stream) {
  if (!q_net || !q_target || !args || !ws) { set_last_error("rb200_dqn_td_step: null argument"); return RB200_E_INVALID; }
  if (int rc = validate_mlp(q_net, "q_network")) return rc;
  if (int rc = validate_mlp(q_target, "q_network_target")) return rc;
  if (q_net->n_layers != q_target->n_layers) { set_last_error("q_network / target layer count mismatch"); return RB200_E_INVALID; }
  for (int l = 0; l <= q_net->n_layers; ++l)
    if (q_net->dims[l] != q_target->dims[l]) { set_last_error("q_network / target dims mismatch at %d", l); return RB200_E_INVALID; }
  if (args->batch <= 0) { set_last_error("batch must be positive"); return RB200_E_INVALID; }
  if (!args->state || !args->next_state || !args->action || !args->reward || !args->not_terminal ||
      !args->loss_partials || !args->loss || !args->tile_counter) {
    set_last_error("rb200_dqn_td_step: required pointer is null"); return RB200_E_INVALID;
  }
  if (!args->maxq && !args->next_action) { set_last_error("SARSA update needs next_action"); return RB200_E_INVALID; }
  if (args->discount_mode == RB200_DISCOUNT_POW && !args->discount_src) { set_last_error("POW discount needs discount_src"); return RB200_E_INVALID; }
  if (args->do_backward) {
    for (int l = 0; l < q_net->n_layers; ++l) {
      if (!ws->dz[l] || (l < q_net->n_layers - 1 && !ws->hidden[l])) { set_last_error("workspace buffer missing for layer %d", l); return RB200_E_INVALID; }
    }
  }
  DqnDev p;
  p.a = *args;
  p.ws = *ws;
  RowsCfg cfg = dqn_cfg(q_net, args->batch, &p.ld_q);
  if (cfg.tm == 0) { set_last_error("DQN tile does not fit in shared memory (dims too large)"); return RB200_E_SMEM; }
  p.ld_in = cfg.ld_in;
  p.ld_h = cfg.ld_h;
  const Mlp q = make_mlp(q_net), qt = make_mlp(q_target);
  const int grid = ceil_div(args->batch, rows_per_tile(cfg));
  cudaStream_t st = (cudaStream_t)stream;
  const bool weighted = args->sample_weight != nullptr;
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    const char* what = "dqn_td_rows_kernel launch";
    return weighted
               ? launch<dqn_td_rows_kernel<NT(), 4, KC(), true>>(grid, NT(), cfg.smem_bytes, st,
                                                                  what, q, qt, p)
               : launch<dqn_td_rows_kernel<NT(), 4, KC(), false>>(grid, NT(), cfg.smem_bytes, st,
                                                                   what, q, qt, p);
  });
}

extern "C" int rb200_num_row_tiles(int batch, int max_dim_in, int max_dim_hidden) {
  RowsCfg cfg = pick_rows_cfg(batch, max_dim_in, max_dim_hidden, 1, 3, 64, 0);
  if (cfg.tm == 0) return ceil_div(batch, 16);
  return ceil_div(batch, rows_per_tile(cfg));
}
