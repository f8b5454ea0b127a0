// reagent_b200 -- QR-DQN: wide-head layer kernels + fused quantile-regression head.
//
// QRDQNTrainer.train_step_gen (reagent/training/qrdqn_trainer.py:108-194) on a network whose
// last layer is [hidden -> A*N] (FullyConnectedDQN with num_atoms, reagent/models/
// fully_connected_network.py:166-217).  The (B, A, N) head output does not fit a row tile's
// shared memory, so the head layer runs as a 2-D tiled launch (row tiles x column blocks) built
// from the same tile primitives, and the distributional loss is one CTA per batch row:
//   qr_head_kernel   mean over atoms -> masked argmax -> target distribution -> pairwise
//                    quantile-Huber loss and its gradient WITHOUT materialising the
//                    (N, B, N) tensor (qrdqn_trainer.py:125-155, :210-218).
#include "rb200_rows.cuh"

namespace rb200 {

constexpr int kColBlock = 512;  // head columns per CTA

// ---------------- wide single Linear layer forward: out = act(in . W^T + b) ----------------
struct LinFwdDev {
  const float* in; int K;
  const float* W; const float* b; int N; int act;
  float* out; int batch; int ld_in, ld_o;
};

template <int NT, int TM, int KC>
__global__ void __launch_bounds__(NT, 1) linear_fwd_wide_kernel(const LinFwdDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* xin = Wst + 2 * wstage_floats<KC>();
  float* xo = xin + R * p.ld_in;
  const int row0 = blockIdx.x * R;
  const int c0 = blockIdx.y * kColBlock;
  const int nloc = min(kColBlock, p.N - c0);
  tile_load_rows<NT, R>(xin, p.ld_in, p.in, p.K, p.K, row0, p.batch);
  __syncthreads();
  tile_linear_fwd<NT, TM, KC>(xin, p.ld_in, p.K, p.W + (size_t)c0 * p.K, p.K,
                              p.b ? p.b + c0 : nullptr, nloc, p.act, xo, p.ld_o, Wst);
  tile_store_rows<NT, R>(xo, p.ld_o, p.out + c0, p.N, nloc, row0, p.batch);
}

// -------- wide contraction backward: dz_prev = (dz . W) * act'(h_prev), N large --------
struct LinBwdDev {
  const float* dz; int N;       // [B, N]
  const float* W; int K;        // [N, K]
  const float* h_prev; int act_prev;  // [B, K] output of the previous layer (or nullptr)
  float* out;                   // [B, K]
  int batch, ld_z, ld_k;
};

template <int NT, int TM, int KC>
__global__ void __launch_bounds__(NT, 1) linear_bwd_wide_kernel(const LinBwdDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* zs = Wst + 2 * wstage_floats<KC>();  // [R, ld_z] slab of dz
  float* accb = zs + R * p.ld_z;              // [R, ld_k] running sum
  float* tmp = accb + R * p.ld_k;             // [R, ld_k] per-slab result
  const int row0 = blockIdx.x * R;
  const int K4 = round_up4(p.K);
  for (int idx = threadIdx.x; idx < R * p.ld_k; idx += NT) accb[idx] = 0.f;
  for (int n0 = 0; n0 < p.N; n0 += kColBlock) {
    const int nloc = min(kColBlock, p.N - n0);
    // slab of dz columns [n0, n0+nloc)
    tile_load_rows<NT, R>(zs, p.ld_z, p.dz + n0, p.N, nloc, row0, p.batch);
    __syncthreads();
    tile_linear_bwd<NT, TM, KC>(zs, p.ld_z, nloc, p.W + (size_t)n0 * p.K, p.K, p.K, nullptr, 0, 0,
                                tmp, p.ld_k, Wst);
    for (int idx = threadIdx.x; idx < R * K4; idx += NT) {
      const int r = idx / K4, c = idx - r * K4;
      accb[r * p.ld_k + c] += tmp[r * p.ld_k + c];
    }
    __syncthreads();
  }
  for (int idx = threadIdx.x; idx < R * K4; idx += NT) {
    const int r = idx / K4, c = idx - r * K4;
    const int row = row0 + r;
    if (row < p.batch && c < p.K) {
      float g = accb[r * p.ld_k + c];
      if (p.h_prev) g *= act_bwd_from_out(p.h_prev[(size_t)row * p.K + c], p.act_prev);
      p.out[(size_t)row * p.K + c] = g;
    }
  }
}

// ---------------- whole-MLP backward (dZ chain) from a given last-layer dz ----------------
struct MlpBwdDev {
  const float* dz_last;  // [B, dims[L]] pre-activation gradient of the last layer
  rb200_net_ws_t ws;
  int batch, ld_h, ld_o;
};

template <int NT, int TM, int KC>
__global__ void __launch_bounds__(NT, 1) mlp_bwd_rows_kernel(const Mlp net, const MlpBwdDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* gA = Wst + 2 * wstage_floats<KC>();
  float* gB = gA + R * p.ld_h;
  float* hb = gB + R * p.ld_h;
  float* zl = hb + R * p.ld_h;
  const int row0 = blockIdx.x * R;
  const int DL = net.dims[net.n_layers];
  tile_load_rows<NT, R>(zl, p.ld_o, p.dz_last, DL, DL, row0, p.batch);
  __syncthreads();
  // dz of the last layer is already in global memory: do not store it again
  rb200_net_ws_t ws = p.ws;
  float* keep = ws.dz[net.n_layers - 1];
  ws.dz[net.n_layers - 1] = nullptr;
  tile_mlp_bwd<NT, TM, KC>(net, zl, p.ld_o, gA, gB, hb, p.ld_h, Wst, ws.hidden, ws.dz, row0,
                           p.batch, nullptr, 0, 0, 0);
  (void)keep;
}

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

extern "C" int rb200_linear_forward_tc(const float* W, const float* b, int32_t act, int32_t K,
                                       int32_t N, const float* in, int32_t batch, float* out,
                                       void* stream);

extern "C" int rb200_linear_forward(const float* W, const float* b, int32_t act, int32_t K,
                                    int32_t N, const float* in, int32_t batch, float* out,
                                    void* stream) {
  if (!W || !in || !out || K <= 0 || N <= 0 || batch <= 0) { set_last_error("rb200_linear_forward: bad argument"); return RB200_E_INVALID; }
  // GEMM-shaped problems (>= one full 128x128 tile) go to the wgmma kernel
  static const bool no_tc = getenv("RB200_DISABLE_WGMMA") != nullptr;  // debugging aid
  if (!no_tc && batch >= 128 && N >= 128) return rb200_linear_forward_tc(W, b, act, K, N, in, batch, out, stream);
  LinFwdDev p{in, K, W, b, N, act, out, batch, 0, kColBlock + 4};
  RowsCfg cfg = pick_rows_cfg(batch, K, 4, 1, 0, p.ld_o, 0);
  if (cfg.tm == 0) { set_last_error("rb200_linear_forward: tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_in = cfg.ld_in;
  dim3 grid(ceil_div(batch, rows_per_tile(cfg)), ceil_div(N, kColBlock));
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    return launch<linear_fwd_wide_kernel<NT(), 4, KC()>>(grid, NT(), cfg.smem_bytes, (cudaStream_t)stream,
                                                         "linear_fwd_wide_kernel launch", p);
  });
}

extern "C" int rb200_linear_backward_dx(const float* W, int32_t K, int32_t N, const float* dz,
                                        const float* h_prev, int32_t act_prev, int32_t batch,
                                        float* out, void* stream) {
  if (!W || !dz || !out || K <= 0 || N <= 0 || batch <= 0) { set_last_error("rb200_linear_backward_dx: bad argument"); return RB200_E_INVALID; }
  LinBwdDev p{dz, N, W, K, h_prev, act_prev, out, batch, kColBlock + 4, round_up4(K) + 4};
  RowsCfg cfg = pick_rows_cfg(batch, kColBlock, 4, 1, 0, 2 * p.ld_k, 0);
  if (cfg.tm == 0) { set_last_error("rb200_linear_backward_dx: tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_z = cfg.ld_in;
  dim3 grid(ceil_div(batch, rows_per_tile(cfg)));
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    return launch<linear_bwd_wide_kernel<NT(), 4, KC()>>(grid, NT(), cfg.smem_bytes, (cudaStream_t)stream,
                                                         "linear_bwd_wide_kernel launch", p);
  });
}

extern "C" int rb200_mlp_backward(const rb200_mlp_t* net, const float* dz_last, int32_t batch,
                                  const rb200_net_ws_t* ws, void* stream) {
  if (!net || !dz_last || !ws || batch <= 0) { set_last_error("rb200_mlp_backward: bad argument"); return RB200_E_INVALID; }
  if (int rc = validate_mlp(net, "net")) return rc;
  if (net->n_layers < 2) return RB200_OK;  // nothing below the last layer
  MlpBwdDev p;
  p.dz_last = dz_last;
  p.ws = *ws;
  p.batch = batch;
  const int DL = net->dims[net->n_layers];
  p.ld_o = round_up4(DL) + 4;
  RowsCfg cfg = pick_rows_cfg(batch, 4, mlp_max_hidden(net), 0, 3, p.ld_o, 0);
  if (cfg.tm == 0) { set_last_error("rb200_mlp_backward: tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_h = cfg.ld_h;
  const Mlp m = make_mlp(net);
  dim3 grid(ceil_div(batch, rows_per_tile(cfg)));
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    return launch<mlp_bwd_rows_kernel<NT(), 4, KC()>>(grid, NT(), cfg.smem_bytes, (cudaStream_t)stream,
                                                      "mlp_bwd_rows_kernel launch", m, p);
  });
}

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
