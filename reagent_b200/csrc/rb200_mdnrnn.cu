// reagent_b200 -- MDN-RNN: a multi-layer LSTM with a mixture-density head
// (reagent/models/mdn_rnn.py MDNRNN.forward and gmm_loss, reagent/training/world_model/
// mdnrnn_trainer.py get_loss).
//
// Rows of an LSTM are independent across the batch, so one CTA carries a tile of R = 16 rows
// through every step and every layer with no grid-wide synchronisation, on the row-tile LSTM step
// of rb200_lstm.cuh.  The backward walks time in reverse per row tile and writes dGates[l, t];
// the weight gradients are one launch of the shared split-K kernel (rb200_wgrad.cuh) over the
// T * B rows.  The world-model evaluators (reagent/evaluation/world_model_evaluator.py) run the
// forward's step, without its training outputs, over a second grid dimension of perturbed
// copies of one batch.
#include <math.h>

#include "rb200_lstm.cuh"
#include "rb200_wgrad.cuh"

namespace rb200 {

constexpr int kMdnNT = kLstmNT, kMdnTM = kLstmTM, kMdnKC = kLstmKC;
constexpr int kMdnR = kLstmR;  // 16 rows per CTA
static_assert(kMdnR == RB200_MDNRNN_ROWS_PER_BLOCK, "rows per block");
constexpr float kLogSqrt2Pi = 0.91893853320467274f;  // math.log(math.sqrt(2 * math.pi))

struct MdnDims {
  int T, B, S, A, H, L, G, NG, DX;  // DX = A + S
  int ld_x, ld_h, ld_s;             // smem strides: input tile, h / c tiles, scratch
};

__host__ __device__ inline MdnDims mdn_dims(const rb200_mdnrnn_args_t& a) {
  MdnDims d;
  d.T = a.seq_len; d.B = a.batch; d.S = a.state_dim; d.A = a.action_dim; d.H = a.hidden;
  d.L = a.layers; d.G = a.gaussians;
  d.NG = (2 * d.S + 1) * d.G + 2;
  d.DX = d.A + d.S;
  d.ld_x = round_up4(d.DX) + 4;
  d.ld_h = round_up4(d.H) + 4;
  const int ld_g = round_up4(4 * d.H) + 4, ld_y = round_up4(d.NG) + 4;
  d.ld_s = 2 * ld_g > ld_y ? 2 * ld_g : ld_y;
  return d;
}

inline size_t mdn_fwd_smem(const MdnDims& d) {
  return sizeof(float) * (2 * (size_t)wstage_floats<kMdnKC>() +
                          (size_t)kMdnR * (d.ld_x + 2 * d.L * d.ld_h + d.ld_s) + 3 * kMdnR);
}
inline size_t mdn_bwd_smem(const MdnDims& d) {
  return sizeof(float) * (2 * (size_t)wstage_floats<kMdnKC>() +
                          (size_t)kMdnR * ((2 * d.L + 1) * d.ld_h + d.ld_s));
}

__device__ __forceinline__ size_t hc_idx(const MdnDims& d, int l, int s, int b) {
  return lstm_hc_idx(d.T, d.B, d.H, l, s, b);
}

// ---------------------------------------------------------------------------
// One forward step of a row tile for mdnrnn_eval_kernel: stage the input, every LSTM layer,
// gmm_linear, and each row's nll / bce / squared error (thread 0 adds them to `acc` in row
// order).  These are mdnrnn_fwd_kernel's operations in its order, minus the training outputs,
// so the same input gives the same bits; the GPU tests hold every variant to the forward with
// torch.equal.  The forward keeps its own copy: calling this from it cost it 2-3 % of its time
// on the H100 (more registers, 135 against 124), on the training path of MDN-RNN and CEM.
//   x(b, c):     input column c of row b < B at this step
//   mus:         [T][B][G*S] means, or nullptr
// ---------------------------------------------------------------------------
struct MdnSmem {
  float* Wst;    // weight staging
  float* xs;     // [R][ld_x] the step's input
  float* hsm;    // [L][R][ld_h]
  float* csm;    // [L][R][ld_h]
  float* scr;    // [R][ld_s]: G1 | G2, then the head output
  float* s_row;  // [3][R] per-row nll, bce, squared error
};

__device__ __forceinline__ MdnSmem mdn_smem(const MdnDims& d, float* smem) {
  constexpr int R = kMdnR;
  MdnSmem m;
  m.Wst = smem;
  m.xs = m.Wst + 2 * wstage_floats<kMdnKC>();
  m.hsm = m.xs + R * d.ld_x;
  m.csm = m.hsm + d.L * R * d.ld_h;
  m.scr = m.csm + d.L * R * d.ld_h;
  m.s_row = m.scr + R * d.ld_s;
  return m;
}

template <typename X>
__device__ __forceinline__ void mdn_step(const rb200_mdnrnn_args_t& a, const MdnDims& d,
                                         float* smem, int t, int row0, float* mus, X x,
                                         float (&acc)[3]) {
  const MdnSmem m = mdn_smem(d, smem);
  constexpr int NT = kMdnNT, R = kMdnR;
  const int ld_g = round_up4(4 * d.H) + 4;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float* P = a.params;
  const int H = d.H, GS = d.G * d.S;
  float* xs = m.xs;
  float* scr = m.scr;
  float* s_row = m.s_row;
  // x = cat(action, state), action first (MDNRNN.forward)
  const size_t tb = (size_t)t * d.B;
  for (int i = tid; i < R * d.DX; i += NT) {
    const int r = i / d.DX, c = i - r * d.DX, b = row0 + r;
    float v = 0.f;
    if (b < d.B) v = x(b, c);
    xs[r * d.ld_x + c] = v;
  }
  __syncthreads();
  lstm_tile_step<true>(a, d.L, H, d.B, row0, xs, d.ld_x, d.DX, m.hsm, m.csm, d.ld_h, scr, d.ld_s,
                       ld_g, m.Wst,
                       [](int, int, int, int, float, float, float, float, float, float) {});
  // gmm_linear on the top layer's h_t
  tile_linear_fwd<NT, kMdnTM, kMdnKC>(m.hsm + (d.L - 1) * R * d.ld_h, d.ld_h, H,
                                      P + a.w_gmm_off, H, P + a.b_gmm_off, d.NG,
                                      RB200_ACT_LINEAR, scr, d.ld_s, m.Wst);
  const bool in_loss = !a.fit_only_one_next_step || t == d.T - 1;
  // one warp per row; lane k < G carries gaussian k
  for (int r = warp; r < R; r += NT / 32) {
    const int b = row0 + r;
    if (b >= d.B) {
      if (lane == 0) { s_row[r] = 0.f; s_row[R + r] = 0.f; s_row[2 * R + r] = 0.f; }
      continue;
    }
    const float* y = scr + r * d.ld_s;
    const bool gl = lane < d.G;
    // logpi = log_softmax(y[2GS .. 2GS+G))
    const float rp = gl ? y[2 * GS + lane] : -INFINITY;
    const float pm = warp_max(rp);
    const float pe = warp_sum(gl ? expf(__fsub_rn(rp, pm)) : 0.f);
    const float logpi = gl ? __fsub_rn(__fsub_rn(rp, pm), logf(pe)) : -INFINITY;
    float* o = mus ? mus + (tb + b) * GS : nullptr;
    const float* xt = in_loss ? a.next_state + (tb + b) * d.S : nullptr;
    float lp = 0.f;
    if (gl) {
      for (int s = 0; s < d.S; ++s) {
        const float mu = y[lane * d.S + s];
        const float sg = expf(y[GS + lane * d.S + s]);
        if (o) o[lane * d.S + s] = mu;
        if (xt) {
          // Normal.log_prob: -(x - mu)^2 / (2 var) - log(sigma) - log(sqrt(2 pi))
          const float df = __fsub_rn(xt[s], mu);
          const float q = __fdiv_rn(-__fmul_rn(df, df), __fmul_rn(2.f, __fmul_rn(sg, sg)));
          lp = __fadd_rn(lp, __fsub_rn(__fsub_rn(q, logf(sg)), kLogSqrt2Pi));
        }
      }
    }
    if (!in_loss) {
      if (lane == 0) { s_row[r] = 0.f; s_row[R + r] = 0.f; s_row[2 * R + r] = 0.f; }
      continue;
    }
    // log-sum-exp over gaussians, shifted by the max
    const float z = gl ? __fadd_rn(logpi, lp) : -INFINITY;
    const float zm = warp_max(z);
    const float ez = gl ? expf(__fsub_rn(z, zm)) : 0.f;
    const float zs = warp_sum(ez);
    const float log_prob = __fadd_rn(zm, logf(zs));
    const float rh = y[d.NG - 2], nt = y[d.NG - 1];
    const float rt = a.reward[tb + b], yt = a.not_terminal[tb + b];
    if (lane == 0) {
      // binary_cross_entropy_with_logits: (1 - y) x - log_sigmoid(x)
      const float ls = __fsub_rn(fminf(nt, 0.f), log1pf(expf(-fabsf(nt))));
      const float dr = __fsub_rn(rh, rt);
      s_row[r] = -log_prob;
      s_row[R + r] = __fsub_rn(__fmul_rn(__fsub_rn(1.f, yt), nt), ls);
      s_row[2 * R + r] = __fmul_rn(dr, dr);
    }
  }
  __syncthreads();
  if (tid == 0 && in_loss) {
    for (int r = 0; r < R; ++r) {
      acc[0] += s_row[r];
      acc[1] += s_row[R + r];
      acc[2] += s_row[2 * R + r];
    }
  }
}

// The last tile's means of a launch's three sums, weighted, and
// loss = gmm / gmm_divisor + bce + mse, into loss[4] (thread 0 of every tile calls it).
__device__ __forceinline__ void mdn_finish(const rb200_mdnrnn_args_t& a, const MdnDims& d,
                                           float* partials, uint32_t* counter, float* loss,
                                           const float (&acc)[3]) {
  const float n_rows = a.fit_only_one_next_step ? (float)d.B : (float)d.T * (float)d.B;
  const float w0 = a.next_state_weight, w1 = a.not_terminal_weight, w2 = a.reward_weight;
  const float div = a.gmm_divisor;
  finish_serial<3>(partials, counter, acc, [=](const float (&s)[3]) {
    const float gmm = __fmul_rn(__fdiv_rn(s[0], n_rows), w0);
    const float bce = __fmul_rn(__fdiv_rn(s[1], n_rows), w1);
    const float mse = __fmul_rn(__fdiv_rn(s[2], n_rows), w2);
    loss[0] = gmm;
    loss[1] = bce;
    loss[2] = mse;
    loss[3] = __fadd_rn(__fadd_rn(__fdiv_rn(gmm, div), bce), mse);
  });
}

// ---------------------------------------------------------------------------
// Forward (+ loss and dL/d(gmm_outs) with targets)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kMdnNT, 1) mdnrnn_fwd_kernel(const rb200_mdnrnn_args_t a) {
  constexpr int NT = kMdnNT, R = kMdnR;
  const MdnDims d = mdn_dims(a);
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* xs = Wst + 2 * wstage_floats<kMdnKC>();
  float* hsm = xs + R * d.ld_x;             // [L][R][ld_h]
  float* csm = hsm + d.L * R * d.ld_h;      // [L][R][ld_h]
  float* scr = csm + d.L * R * d.ld_h;      // [R][ld_s]: G1 | G2, then the head output
  float* s_row = scr + R * d.ld_s;          // [3][R] per-row nll, bce, squared error
  const int ld_g = round_up4(4 * d.H) + 4;
  const int row0 = blockIdx.x * R;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool has_loss = a.next_state != nullptr;
  const bool train = a.dy != nullptr;
  const float* P = a.params;
  const int H = d.H, GS = d.G * d.S;
  const float n_rows = a.fit_only_one_next_step ? (float)d.B : (float)d.T * (float)d.B;
  float acc[3] = {0.f, 0.f, 0.f};  // thread 0: this block's sums, rows and steps in order

  // slot 0 of hs / cs: the zero initial state read by the backward and the weight gradients
  for (int i = tid; i < d.L * R * H; i += NT) {
    const int l = i / (R * H), r = (i / H) % R, j = i % H;
    if (row0 + r < d.B) {
      a.hs[hc_idx(d, l, 0, row0 + r) + j] = 0.f;
      a.cs[hc_idx(d, l, 0, row0 + r) + j] = 0.f;
    }
  }

  for (int t = 0; t < d.T; ++t) {
    // x = cat(action, state), action first (MDNRNN.forward)
    const size_t tb = (size_t)t * d.B;
    for (int i = tid; i < R * d.DX; i += NT) {
      const int r = i / d.DX, c = i - r * d.DX, b = row0 + r;
      float v = 0.f;
      if (b < d.B)
        v = c < d.A ? a.action[(tb + b) * d.A + c] : a.state[(tb + b) * d.S + (c - d.A)];
      xs[r * d.ld_x + c] = v;
      if (train && b < d.B) a.xin[(tb + b) * d.DX + c] = v;
    }
    __syncthreads();
    lstm_tile_step<true>(a, d.L, H, d.B, row0, xs, d.ld_x, d.DX, hsm, csm, d.ld_h, scr, d.ld_s,
                         ld_g, Wst,
                         [&](int l, int r, int b, int j, float gi, float gf, float gg, float go,
                             float cn, float hn) {
                           a.hs[hc_idx(d, l, t + 1, b) + j] = hn;
                           a.cs[hc_idx(d, l, t + 1, b) + j] = cn;
                           if (train) {
                             float* ga = a.acts + lstm_gate_idx(d.T, d.B, H, l, t, b);
                             ga[j] = gi; ga[H + j] = gf; ga[2 * H + j] = gg; ga[3 * H + j] = go;
                           }
                         });
    // gmm_linear on the top layer's h_t
    tile_linear_fwd<NT, kMdnTM, kMdnKC>(hsm + (d.L - 1) * R * d.ld_h, d.ld_h, H,
                                        P + a.w_gmm_off, H, P + a.b_gmm_off, d.NG,
                                        RB200_ACT_LINEAR, scr, d.ld_s, Wst);
    const bool in_loss = has_loss && (!a.fit_only_one_next_step || t == d.T - 1);
    // one warp per row; lane k < G carries gaussian k
    for (int r = warp; r < R; r += NT / 32) {
      const int b = row0 + r;
      if (b >= d.B) {
        if (lane == 0) { s_row[r] = 0.f; s_row[R + r] = 0.f; s_row[2 * R + r] = 0.f; }
        continue;
      }
      const float* y = scr + r * d.ld_s;
      const bool gl = lane < d.G;
      // logpi = log_softmax(y[2GS .. 2GS+G))
      const float rp = gl ? y[2 * GS + lane] : -INFINITY;
      const float pm = warp_max(rp);
      const float pe = warp_sum(gl ? expf(__fsub_rn(rp, pm)) : 0.f);
      const float logpi = gl ? __fsub_rn(__fsub_rn(rp, pm), logf(pe)) : -INFINITY;
      float* o = a.out ? a.out + (tb + b) * d.NG : nullptr;
      const float* x = in_loss ? a.next_state + (tb + b) * d.S : nullptr;
      float lp = 0.f;
      if (gl) {
        for (int s = 0; s < d.S; ++s) {
          const float mu = y[lane * d.S + s];
          const float sg = expf(y[GS + lane * d.S + s]);
          if (o) { o[lane * d.S + s] = mu; o[GS + lane * d.S + s] = sg; }
          if (x) {
            // Normal.log_prob: -(x - mu)^2 / (2 var) - log(sigma) - log(sqrt(2 pi))
            const float df = __fsub_rn(x[s], mu);
            const float q = __fdiv_rn(-__fmul_rn(df, df), __fmul_rn(2.f, __fmul_rn(sg, sg)));
            lp = __fadd_rn(lp, __fsub_rn(__fsub_rn(q, logf(sg)), kLogSqrt2Pi));
          }
        }
        if (o) o[2 * GS + lane] = logpi;
      }
      if (o && lane == 0) { o[d.NG - 2] = y[d.NG - 2]; o[d.NG - 1] = y[d.NG - 1]; }
      if (!has_loss) continue;
      float* dy = train ? a.dy + (tb + b) * d.NG : nullptr;
      if (!in_loss) {
        if (dy)
          for (int c = lane; c < d.NG; c += 32) dy[c] = 0.f;
        if (lane == 0) { s_row[r] = 0.f; s_row[R + r] = 0.f; s_row[2 * R + r] = 0.f; }
        continue;
      }
      // log-sum-exp over gaussians, shifted by the max
      const float z = gl ? __fadd_rn(logpi, lp) : -INFINITY;
      const float zm = warp_max(z);
      const float ez = gl ? expf(__fsub_rn(z, zm)) : 0.f;
      const float zs = warp_sum(ez);
      const float log_prob = __fadd_rn(zm, logf(zs));
      const float rh = y[d.NG - 2], nt = y[d.NG - 1];
      const float rt = a.reward[tb + b], yt = a.not_terminal[tb + b];
      if (lane == 0) {
        // binary_cross_entropy_with_logits: (1 - y) x - log_sigmoid(x)
        const float ls = __fsub_rn(fminf(nt, 0.f), log1pf(expf(-fabsf(nt))));
        const float dr = __fsub_rn(rh, rt);
        s_row[r] = -log_prob;
        s_row[R + r] = __fsub_rn(__fmul_rn(__fsub_rn(1.f, yt), nt), ls);
        s_row[2 * R + r] = __fmul_rn(dr, dr);
      }
      if (!dy) continue;
      // d loss / d log_prob of this row = -(w_ns / N) / gmm_divisor
      const float cg = -__fdiv_rn(__fdiv_rn(a.next_state_weight, n_rows), a.gmm_divisor);
      const float dz = gl ? __fmul_rn(cg, __fdiv_rn(ez, zs)) : 0.f;  // d/dz_k
      if (gl) {
        for (int s = 0; s < d.S; ++s) {
          const float mu = y[lane * d.S + s];
          const float sg = expf(y[GS + lane * d.S + s]);
          const float var = __fmul_rn(sg, sg);
          const float df = __fsub_rn(x[s], mu);
          dy[lane * d.S + s] = __fmul_rn(dz, __fdiv_rn(df, var));
          dy[GS + lane * d.S + s] = __fmul_rn(dz, __fsub_rn(__fdiv_rn(__fmul_rn(df, df), var), 1.f));
        }
      }
      // log_softmax backward: d raw_j = dz_j - softmax_j * sum_k dz_k
      const float dzs = warp_sum(dz);
      if (gl) dy[2 * GS + lane] = __fsub_rn(dz, __fmul_rn(expf(logpi), dzs));
      if (lane == 0) {
        dy[d.NG - 2] = __fmul_rn(__fdiv_rn(a.reward_weight, n_rows), __fmul_rn(2.f, __fsub_rn(rh, rt)));
        dy[d.NG - 1] = __fmul_rn(__fdiv_rn(a.not_terminal_weight, n_rows), __fsub_rn(sigmoidf(nt), yt));
      }
    }
    __syncthreads();
    if (has_loss && tid == 0 && in_loss) {
      for (int r = 0; r < R; ++r) {
        acc[0] += s_row[r];
        acc[1] += s_row[R + r];
        acc[2] += s_row[2 * R + r];
      }
    }
  }
  if (has_loss && tid == 0) {
    float* loss = a.loss;
    const float w0 = a.next_state_weight, w1 = a.not_terminal_weight, w2 = a.reward_weight;
    const float div = a.gmm_divisor;
    finish_serial<3>(a.loss_partials, a.tile_counter, acc, [=](const float (&s)[3]) {
      const float gmm = __fmul_rn(__fdiv_rn(s[0], n_rows), w0);
      const float bce = __fmul_rn(__fdiv_rn(s[1], n_rows), w1);
      const float mse = __fmul_rn(__fdiv_rn(s[2], n_rows), w2);
      loss[0] = gmm;
      loss[1] = bce;
      loss[2] = mse;
      loss[3] = __fadd_rn(__fadd_rn(__fdiv_rn(gmm, div), bce), mse);
    });
  }
}

// ---------------------------------------------------------------------------
// Variant-batched loss (world-model feature importance and sensitivity): CTA (j, v) carries row
// tile j of variant v through the forward of mdn_step.  Variant v replaces columns
// [col_begin[v], col_end[v]) of x by fill[fill_off[v] ...] at every step and row, and variant
// perm_variant reads action row perm[b] for row b.  Targets are never changed.  Nothing of the
// training workspace is written; mus (when given) gets variant v's means at [v][T][B][G*S].
// Each variant reduces its own tiles in finish_serial's order into loss[4 v ...], so variant v's
// four numbers are the forward's on the batch with the replacement made.  A perm entry outside
// [0, B) reads NaN as the action, so that variant's results are NaN.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kMdnNT, 1) mdnrnn_eval_kernel(const rb200_mdnrnn_eval_args_t e) {
  constexpr int NT = kMdnNT, R = kMdnR;
  const rb200_mdnrnn_args_t& a = e.net;
  const MdnDims d = mdn_dims(a);
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  const int row0 = blockIdx.x * R;
  const int v = blockIdx.y;
  const int c0 = e.col_begin[v], c1 = e.col_end[v];
  const float* fill = e.fill + e.fill_off[v] - c0;  // fill[c] for c in [c0, c1)
  const int64_t* perm = v == e.perm_variant ? e.perm : nullptr;
  const int GS = d.G * d.S;
  float* mus = e.mus ? e.mus + (size_t)v * d.T * d.B * GS : nullptr;  // [T][B][G*S] of v
  float acc[3] = {0.f, 0.f, 0.f};

  for (int t = 0; t < d.T; ++t) {
    const size_t tb = (size_t)t * d.B;
    mdn_step(
        a, d, smem, t, row0, mus,
        [&](int b, int c) {
          if (c >= c0 && c < c1) return fill[c];
          if (c >= d.A) return a.state[(tb + b) * d.S + (c - d.A)];
          if (!perm) return a.action[(tb + b) * d.A + c];
          const int64_t pb = perm[b];
          return pb >= 0 && pb < d.B ? a.action[(tb + pb) * d.A + c] : NAN;
        },
        acc);
  }
  if (threadIdx.x == 0)
    mdn_finish(a, d, e.loss_partials + (size_t)v * 3 * gridDim.x, e.tile_counter + v,
               e.loss + 4 * v, acc);
}

// ---------------------------------------------------------------------------
// Backward through time: dGates[l, t] for every layer and step
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kMdnNT, 1) mdnrnn_bwd_kernel(const rb200_mdnrnn_args_t a) {
  constexpr int NT = kMdnNT, R = kMdnR;
  const MdnDims d = mdn_dims(a);
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* dhr = Wst + 2 * wstage_floats<kMdnKC>();  // [L][R][ld_h] dL/dh_{t-1} through W_hh
  float* dcs = dhr + d.L * R * d.ld_h;             // [L][R][ld_h] dL/dc_{t-1} through f
  float* dx = dcs + d.L * R * d.ld_h;              // [R][ld_h] dL/dh_t from above
  float* scr = dx + R * d.ld_h;                    // [R][ld_s]: dY of the step, then dGates
  const int row0 = blockIdx.x * R;
  const float* P = a.params;
  const int H = d.H;
  for (int t = d.T - 1; t >= 0; --t) {
    tile_load_rows<NT, R>(scr, d.ld_s, a.dy + (size_t)t * d.B * d.NG, d.NG, d.NG, row0, d.B);
    __syncthreads();
    // dh_top = dY . W_gmm
    tile_linear_bwd<NT, kMdnTM, kMdnKC>(scr, d.ld_s, d.NG, P + a.w_gmm_off, H, H, nullptr, 0, 0,
                                        dx, d.ld_h, Wst);
    lstm_tile_bwd_step(a, d.T, d.B, d.H, d.L, t, row0, dhr, dcs, dx, d.ld_h, scr, d.ld_s, Wst);
  }
}

// ---------------------------------------------------------------------------
// Feature fill values and sensitivity (reagent/evaluation/world_model_evaluator.py): one CTA
// per feature group; sums in fp64 over a fixed thread-strided order, so both are deterministic.
// ---------------------------------------------------------------------------
constexpr int kEvalNT = 256;

// compute_median_feature_value of group g over the rows of x = cat(action, state): a width-1
// group gets its column mean; a wider (enum) group a one-hot at the first column whose count
// (column sum) equals the lower median of the counts (torch.median).
__global__ void __launch_bounds__(kEvalNT) mdnrnn_fill_kernel(const rb200_mdnrnn_fill_args_t f) {
  __shared__ double s_warp[kEvalNT / 32];
  __shared__ double s_cnt[RB200_MDNRNN_MAX_INPUT];
  __shared__ double s_sorted[RB200_MDNRNN_MAX_INPUT];
  const int g = blockIdx.x, c0 = f.group_begin[g], w = f.group_begin[g + 1] - c0;
  for (int k = 0; k < w; ++k) {
    const int c = c0 + k;
    double s = 0.0;
    for (int i = threadIdx.x; i < f.rows; i += kEvalNT)
      s += c < f.action_dim ? f.action[(size_t)i * f.action_dim + c]
                            : f.state[(size_t)i * f.state_dim + (c - f.action_dim)];
    s = block_sum_f64(s, s_warp);
    if (threadIdx.x == 0) s_cnt[k] = s;
  }
  if (threadIdx.x != 0) return;
  if (w == 1) {
    f.fill[c0] = (float)(s_cnt[0] / (double)f.rows);
    return;
  }
  for (int k = 0; k < w; ++k) {  // insertion sort: at most 256 counts
    const double x = s_cnt[k];
    int j = k;
    for (; j > 0 && s_sorted[j - 1] > x; --j) s_sorted[j] = s_sorted[j - 1];
    s_sorted[j] = x;
  }
  const double med = s_sorted[(w - 1) / 2];
  int first = w - 1;
  for (int k = w - 1; k >= 0; --k)
    if (s_cnt[k] == med) first = k;
  for (int k = 0; k < w; ++k) f.fill[c0 + k] = k == first ? 1.f : 0.f;
}

// Group g of the state columns: mean over (rows, G) of sum_{s in g} |mus1 - mus0|.
__global__ void __launch_bounds__(kEvalNT) mdnrnn_sensitivity_kernel(
    const rb200_mdnrnn_sensitivity_args_t f) {
  __shared__ double s_warp[kEvalNT / 32];
  const int g = blockIdx.x, c0 = f.group_begin[g], c1 = f.group_begin[g + 1];
  const int n = f.rows * f.gaussians;
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += kEvalNT) {
    const float* m0 = f.mus0 + (size_t)i * f.state_dim;
    const float* m1 = f.mus1 + (size_t)i * f.state_dim;
    float r = 0.f;
    for (int c = c0; c < c1; ++c) r = __fadd_rn(r, fabsf(__fsub_rn(m1[c], m0[c])));
    s += r;
  }
  s = block_sum_f64(s, s_warp);
  if (threadIdx.x == 0) f.out[g] = (float)(s / (double)n);
}

static int mdn_validate(const rb200_mdnrnn_args_t* a, const char* who, bool need_hc = true) {
  if (!a) { set_last_error("%s: args is null", who); return RB200_E_INVALID; }
  if (int rc = rb200_mdnrnn_check_shape(a->state_dim, a->action_dim, a->hidden, a->layers,
                                        a->gaussians))
    return rc;
  if (a->seq_len <= 0 || a->batch <= 0) {
    set_last_error("%s: seq_len %d and batch %d must be positive", who, a->seq_len, a->batch);
    return RB200_E_INVALID;
  }
  if ((long long)a->seq_len * a->batch > INT32_MAX / 4) {
    set_last_error("%s: seq_len * batch = %lld is too large", who,
                   (long long)a->seq_len * a->batch);
    return RB200_E_INVALID;
  }
  if (!a->params || (need_hc && (!a->hs || !a->cs))) {
    set_last_error(need_hc ? "%s: params, hs and cs are required" : "%s: params is required",
                   who);
    return RB200_E_INVALID;
  }
  return RB200_OK;
}

// Feature groups [begin[g], begin[g + 1]) for g < n: 1 <= n, begin[0] >= 0, strictly
// increasing, begin[n] <= width.
static int groups_validate(int n, const int32_t* begin, int width, const char* who) {
  if (n < 1 || n > RB200_MDNRNN_MAX_INPUT) {
    set_last_error("%s: num_groups %d must be in [1, %d]", who, n, RB200_MDNRNN_MAX_INPUT);
    return RB200_E_INVALID;
  }
  if (begin[0] < 0 || begin[n] > width) {
    set_last_error("%s: groups span [%d, %d), outside [0, %d)", who, begin[0], begin[n], width);
    return RB200_E_INVALID;
  }
  for (int g = 0; g < n; ++g)
    if (begin[g + 1] <= begin[g]) {
      set_last_error("%s: group boundaries must increase strictly (group %d: [%d, %d))", who, g,
                     begin[g], begin[g + 1]);
      return RB200_E_INVALID;
    }
  return RB200_OK;
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_mdnrnn_check_shape(int32_t S, int32_t A, int32_t H, int32_t L, int32_t G) {
  if (S < 1 || A < 1 || H < 1 || L < 1 || G < 1) {
    set_last_error("rb200_mdnrnn: state_dim %d, action_dim %d, hidden %d, layers %d and "
                   "gaussians %d must be positive", S, A, H, L, G);
    return RB200_E_INVALID;
  }
  const long long ng = (2LL * S + 1) * G + 2;
  if (H > RB200_MDNRNN_MAX_HIDDEN || L > RB200_MDNRNN_MAX_LAYERS ||
      G > RB200_MDNRNN_MAX_GAUSSIANS || S + A > RB200_MDNRNN_MAX_INPUT ||
      ng > RB200_MDNRNN_MAX_OUT) {
    set_last_error("rb200_mdnrnn: unsupported shape (hidden %d <= %d, layers %d <= %d, "
                   "gaussians %d <= %d, state_dim + action_dim %d <= %d, (2 state_dim + 1) "
                   "gaussians + 2 = %lld <= %d)", H, RB200_MDNRNN_MAX_HIDDEN, L,
                   RB200_MDNRNN_MAX_LAYERS, G, RB200_MDNRNN_MAX_GAUSSIANS, S + A,
                   RB200_MDNRNN_MAX_INPUT, ng, RB200_MDNRNN_MAX_OUT);
    return RB200_E_INVALID;
  }
  return RB200_OK;
}

extern "C" int rb200_mdnrnn_forward(const rb200_mdnrnn_args_t* a, void* stream) {
  if (int rc = mdn_validate(a, "rb200_mdnrnn_forward")) return rc;
  if (!a->state || !a->action) {
    set_last_error("rb200_mdnrnn_forward: state and action are required");
    return RB200_E_INVALID;
  }
  const int n_tgt = !!a->next_state + !!a->reward + !!a->not_terminal;
  const int n_train = !!a->xin + !!a->acts + !!a->dy;
  if ((n_tgt != 0 && n_tgt != 3) || (n_train != 0 && n_train != 3) || (n_train && !n_tgt) ||
      (n_tgt && (!a->loss_partials || !a->tile_counter || !a->loss)) ||
      (n_tgt && !(a->gmm_divisor > 0.f))) {
    set_last_error("rb200_mdnrnn_forward: targets (next_state, reward, not_terminal) need loss "
                   "buffers and gmm_divisor > 0; training (xin, acts, dy) needs the targets");
    return RB200_E_INVALID;
  }
  const MdnDims d = mdn_dims(*a);
  return launch<mdnrnn_fwd_kernel>(ceil_div(d.B, kMdnR), kMdnNT, mdn_fwd_smem(d),
                                   (cudaStream_t)stream, "mdnrnn_fwd_kernel launch", *a);
}

extern "C" int rb200_mdnrnn_backward(const rb200_mdnrnn_args_t* a, void* stream) {
  if (int rc = mdn_validate(a, "rb200_mdnrnn_backward")) return rc;
  if (!a->acts || !a->dy || !a->dgates) {
    set_last_error("rb200_mdnrnn_backward: acts, dy and dgates are required");
    return RB200_E_INVALID;
  }
  const MdnDims d = mdn_dims(*a);
  return launch<mdnrnn_bwd_kernel>(ceil_div(d.B, kMdnR), kMdnNT, mdn_bwd_smem(d),
                                   (cudaStream_t)stream, "mdnrnn_bwd_kernel launch", *a);
}

extern "C" int rb200_mdnrnn_wgrad(const rb200_mdnrnn_args_t* a, void* stream) {
  if (int rc = mdn_validate(a, "rb200_mdnrnn_wgrad")) return rc;
  if (!a->xin || !a->dgates || !a->dy || !a->gpart || a->splits <= 0) {
    set_last_error("rb200_mdnrnn_wgrad: xin, dgates, dy, gpart and splits > 0 are required");
    return RB200_E_INVALID;
  }
  const MdnDims d = mdn_dims(*a);
  const size_t TB = (size_t)d.T * d.B, slot = (size_t)(d.T + 1) * d.B * d.H;
  WgradLayer jobs[kWgradMaxJobs] = {};
  int n = 0;
  for (int l = 0; l < d.L; ++l) {
    const float* dz = a->dgates + (size_t)l * TB * 4 * d.H;
    // dW_ih = dGates^T . x (x: the network input, or h_t of the layer below); db_ih = sum dGates
    WgradLayer& ih = jobs[n++];
    ih.A = l == 0 ? a->xin : a->hs + (size_t)(l - 1) * slot + (size_t)d.B * d.H;
    ih.dZ = dz; ih.K = l == 0 ? d.DX : d.H; ih.N = 4 * d.H;
    ih.w_off = a->w_ih_off[l]; ih.b_off = a->b_ih_off[l];
    // dW_hh = dGates^T . h_{t-1} (slots 0 .. T-1, slot 0 the zero state); db_hh = sum dGates
    WgradLayer& hh = jobs[n++];
    hh.A = a->hs + (size_t)l * slot;
    hh.dZ = dz; hh.K = d.H; hh.N = 4 * d.H;
    hh.w_off = a->w_hh_off[l]; hh.b_off = a->b_hh_off[l];
  }
  WgradLayer& head = jobs[n++];
  head.A = a->hs + (size_t)(d.L - 1) * slot + (size_t)d.B * d.H;
  head.dZ = a->dy; head.K = d.H; head.N = d.NG;
  head.w_off = a->w_gmm_off; head.b_off = a->b_gmm_off;
  return wgrad_jobs_launch(jobs, n, (int)TB, a->splits, a->gpart, a->n_params,
                           (cudaStream_t)stream, "rb200_mdnrnn_wgrad");
}

extern "C" int rb200_mdnrnn_eval(const rb200_mdnrnn_eval_args_t* e, void* stream) {
  const char* who = "rb200_mdnrnn_eval";
  if (!e) { set_last_error("%s: args is null", who); return RB200_E_INVALID; }
  const rb200_mdnrnn_args_t* a = &e->net;
  if (int rc = mdn_validate(a, who, false)) return rc;
  if (!a->state || !a->action || !a->next_state || !a->reward || !a->not_terminal ||
      !(a->gmm_divisor > 0.f) || !e->loss_partials || !e->tile_counter || !e->loss) {
    set_last_error("%s: state, action, the targets (next_state, reward, not_terminal), "
                   "loss_partials, tile_counter, loss and gmm_divisor > 0 are required", who);
    return RB200_E_INVALID;
  }
  const MdnDims d = mdn_dims(*a);
  const int V = e->num_variants;
  if (V < 1 || V > 1 + d.A + d.S || V > RB200_MDNRNN_EVAL_MAX_VARIANTS) {
    set_last_error("%s: num_variants %d must be in [1, 1 + action_dim + state_dim = %d]", who, V,
                   1 + d.A + d.S);
    return RB200_E_INVALID;
  }
  for (int v = 0; v < V; ++v) {
    const int c0 = e->col_begin[v], c1 = e->col_end[v];
    if (c0 == c1) continue;
    if (c0 < 0 || c1 < c0 || c1 > d.DX) {
      set_last_error("%s: variant %d replaces columns [%d, %d), outside [0, %d)", who, v, c0, c1,
                     d.DX);
      return RB200_E_INVALID;
    }
    if (!e->fill || e->fill_off[v] < 0 || (int64_t)e->fill_off[v] + (c1 - c0) > e->fill_len) {
      set_last_error("%s: variant %d reads fill[%d, %lld), outside the %d fill values", who, v,
                     e->fill_off[v], (long long)e->fill_off[v] + (c1 - c0), e->fill_len);
      return RB200_E_INVALID;
    }
  }
  if (e->perm_variant < -1 || e->perm_variant >= V || (e->perm_variant >= 0 && !e->perm)) {
    set_last_error("%s: perm_variant %d must be -1 or a variant < %d with a perm", who,
                   e->perm_variant, V);
    return RB200_E_INVALID;
  }
  return launch<mdnrnn_eval_kernel>(dim3(ceil_div(d.B, kMdnR), V), kMdnNT, mdn_fwd_smem(d),
                                    (cudaStream_t)stream, "mdnrnn_eval_kernel launch", *e);
}

extern "C" int rb200_mdnrnn_fill_values(const rb200_mdnrnn_fill_args_t* f, void* stream) {
  const char* who = "rb200_mdnrnn_fill_values";
  if (!f) { set_last_error("%s: args is null", who); return RB200_E_INVALID; }
  if (f->rows <= 0 || f->action_dim < 0 || f->state_dim < 0 ||
      f->action_dim + f->state_dim > RB200_MDNRNN_MAX_INPUT || !f->fill ||
      (f->action_dim && !f->action) || (f->state_dim && !f->state)) {
    set_last_error("%s: rows %d > 0, action_dim %d + state_dim %d <= %d, action / state of "
                   "those widths and fill are required", who, f->rows, f->action_dim,
                   f->state_dim, RB200_MDNRNN_MAX_INPUT);
    return RB200_E_INVALID;
  }
  if (int rc = groups_validate(f->num_groups, f->group_begin, f->action_dim + f->state_dim, who))
    return rc;
  return launch<mdnrnn_fill_kernel>(f->num_groups, kEvalNT, 0, (cudaStream_t)stream,
                                    "mdnrnn_fill_kernel launch", *f);
}

extern "C" int rb200_mdnrnn_sensitivity(const rb200_mdnrnn_sensitivity_args_t* f, void* stream) {
  const char* who = "rb200_mdnrnn_sensitivity";
  if (!f) { set_last_error("%s: args is null", who); return RB200_E_INVALID; }
  if (f->rows <= 0 || f->state_dim < 1 || f->state_dim > RB200_MDNRNN_MAX_INPUT ||
      f->gaussians < 1 || f->gaussians > RB200_MDNRNN_MAX_GAUSSIANS ||
      (long long)f->rows * f->gaussians > INT32_MAX || !f->mus0 || !f->mus1 || !f->out) {
    set_last_error("%s: rows %d > 0, 1 <= state_dim %d <= %d, 1 <= gaussians %d <= %d, "
                   "rows * gaussians < 2^31, mus0, mus1 and out are required", who, f->rows,
                   f->state_dim, RB200_MDNRNN_MAX_INPUT, f->gaussians,
                   RB200_MDNRNN_MAX_GAUSSIANS);
    return RB200_E_INVALID;
  }
  if (int rc = groups_validate(f->num_groups, f->group_begin, f->state_dim, who)) return rc;
  return launch<mdnrnn_sensitivity_kernel>(f->num_groups, kEvalNT, 0, (cudaStream_t)stream,
                                           "mdnrnn_sensitivity_kernel launch", *f);
}
