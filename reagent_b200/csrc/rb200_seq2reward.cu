// reagent_b200 -- Seq2Reward (reagent/models/seq2reward_model.py, reagent/training/world_model/
// seq2reward_trainer.py get_mse_loss / get_Q, compress_model_trainer.py get_loss).
//
// The network is an LSTM over the one-hot action sequence whose every layer starts from
// h = map_linear(state[0]), c = 0, and a width-1 head lstm_linear on the top h of the last valid
// step.  The forward, backward and plan carry 16-row tiles through every step and layer on the
// LSTM step of rb200_lstm.cuh, without tile_linear_fwd's k-chunk rotation: a row's outputs then
// do not depend on the CTA that computes it, so every node of the plan's prefix tree is
// bit-identical to the same sequence's row in a forward over the expanded batch.
#include <math.h>

#include "rb200_lstm.cuh"
#include "rb200_wgrad.cuh"

namespace rb200 {

constexpr int kS2rNT = kLstmNT, kS2rR = kLstmR;
static_assert(kS2rR == RB200_SEQ2REWARD_ROWS_PER_BLOCK, "rows per block");
constexpr int kS2rHeadNT = 256;  // rows per block of the compress head
constexpr size_t kS2rSmemLimit = 227 * 1024;  // H100 opt-in shared memory per CTA

struct S2rDims {
  int T, B, S, A, H, L;
  int ld_x, ld_h, ld_g, ld_s;  // smem strides: input tile, h / c tiles, one gate product, scratch
};

__host__ __device__ inline S2rDims s2r_dims(const rb200_seq2reward_args_t& a) {
  S2rDims d;
  d.T = a.seq_len; d.B = a.batch; d.S = a.state_dim; d.A = a.action_dim; d.H = a.hidden;
  d.L = a.layers;
  d.ld_x = round_up4(d.S > d.A ? d.S : d.A) + 4;
  d.ld_h = round_up4(d.H) + 4;
  d.ld_g = round_up4(4 * d.H) + 4;
  d.ld_s = 2 * d.ld_g;
  return d;
}

inline size_t s2r_fwd_smem(const S2rDims& d) {
  return sizeof(float) * (2 * (size_t)wstage_floats<kLstmKC>() +
                          (size_t)kS2rR * (d.ld_x + (2 * d.L + 1) * d.ld_h + d.ld_s + 1)) +
         sizeof(int) * kS2rR;
}
inline size_t s2r_bwd_smem(const S2rDims& d) {
  return sizeof(float) * (2 * (size_t)wstage_floats<kLstmKC>() +
                          (size_t)kS2rR * ((2 * d.L + 1) * d.ld_h + d.ld_s));
}
inline size_t s2r_plan_smem(const S2rDims& d) {
  return sizeof(float) * (2 * (size_t)wstage_floats<kLstmKC>() +
                          (size_t)kS2rR * (d.ld_x + 2 * d.L * d.ld_h + d.ld_s));
}

struct S2rNoStore {
  __device__ void operator()(int, int, int, int, float, float, float, float, float, float) const {}
};

// h0 = map_linear(state row of each tile row) into every layer's h; c stays 0.  xs holds the
// state rows (S columns); rows r >= nvalid get 0.
__device__ __forceinline__ void s2r_initial_state(const rb200_seq2reward_args_t& a,
                                                  const S2rDims& d, const float* xs, float* hsm,
                                                  float* scr, float* Wst, int nvalid) {
  constexpr int NT = kS2rNT, R = kS2rR;
  const float* P = a.params;
  tile_linear_fwd<NT, kLstmTM, kLstmKC, false>(xs, d.ld_x, d.S, P + a.w_map_off, d.S,
                                               P + a.b_map_off, d.H, RB200_ACT_LINEAR, scr,
                                               d.ld_s, Wst);
  for (int i = threadIdx.x; i < d.L * R * d.H; i += NT) {
    const int l = i / (R * d.H), r = (i / d.H) % R, j = i % d.H;
    hsm[(l * R + r) * d.ld_h + j] = r < nvalid ? scr[r * d.ld_s + j] : 0.f;
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// Forward (+ target, MSE and dL/dacc_reward; step labels)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kS2rNT, 1) s2r_fwd_kernel(const rb200_seq2reward_args_t a) {
  constexpr int NT = kS2rNT, R = kS2rR;
  const S2rDims d = s2r_dims(a);
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* xs = Wst + 2 * wstage_floats<kLstmKC>();  // [R][ld_x]: the state, then the actions
  float* hsm = xs + R * d.ld_x;                     // [L][R][ld_h]
  float* csm = hsm + d.L * R * d.ld_h;              // [L][R][ld_h]
  float* hsel = csm + d.L * R * d.ld_h;             // [R][ld_h]: top h of step valid - 1
  float* scr = hsel + R * d.ld_h;                   // [R][ld_s]
  float* s_row = scr + R * d.ld_s;                  // [R] squared errors
  int* s_valid = reinterpret_cast<int*>(s_row + R); // [R] valid step, clamped to [1, T]
  const int row0 = blockIdx.x * R, tid = threadIdx.x;
  const int T = d.T, B = d.B, H = d.H;
  const bool train = a.hs != nullptr;
  if (tid < R) {
    const int b = row0 + tid;
    int v = T;
    if (a.valid_step && b < B) {
      const long long x = a.valid_step[b];
      v = x < 1 ? 1 : (x > T ? T : (int)x);
    }
    s_valid[tid] = v;
  }
  tile_load_rows<NT, R>(xs, d.ld_x, a.state, d.S, d.S, row0, B);
  __syncthreads();
  s2r_initial_state(a, d, xs, hsm, scr, Wst, B - row0);
  if (train) {
    for (int i = tid; i < d.L * R * H; i += NT) {
      const int l = i / (R * H), r = (i / H) % R, j = i % H, b = row0 + r;
      if (b < B) {
        a.hs[lstm_hc_idx(T, B, H, l, 0, b) + j] = hsm[(l * R + r) * d.ld_h + j];
        a.cs[lstm_hc_idx(T, B, H, l, 0, b) + j] = 0.f;
      }
    }
  }
  for (int i = tid; i < R * d.ld_x; i += NT) xs[i] = 0.f;
  __syncthreads();

  for (int t = 0; t < T; ++t) {
    tile_load_rows<NT, R>(xs, d.ld_x, a.action + (size_t)t * B * d.A, d.A, d.A, row0, B);
    __syncthreads();
    lstm_tile_step<false>(a, d.L, H, B, row0, xs, d.ld_x, d.A, hsm, csm, d.ld_h, scr, d.ld_s,
                          d.ld_g, Wst,
                          [&](int l, int r, int b, int j, float gi, float gf, float gg, float go,
                              float cn, float hn) {
                            if (!train) return;
                            a.hs[lstm_hc_idx(T, B, H, l, t + 1, b) + j] = hn;
                            a.cs[lstm_hc_idx(T, B, H, l, t + 1, b) + j] = cn;
                            float* ga = a.acts + lstm_gate_idx(T, B, H, l, t, b);
                            ga[j] = gi; ga[H + j] = gf; ga[2 * H + j] = gg; ga[3 * H + j] = go;
                          });
    const float* top = hsm + (d.L - 1) * R * d.ld_h;
    for (int i = tid; i < R * H; i += NT) {
      const int r = i / H, j = i - r * H;
      if (s_valid[r] == t + 1) hsel[r * d.ld_h + j] = top[r * d.ld_h + j];
    }
    __syncthreads();
  }
  // acc_reward = lstm_linear(h_top at valid - 1)
  const float* P = a.params;
  tile_linear_fwd<NT, kLstmTM, kLstmKC, false>(hsel, d.ld_h, H, P + a.w_lin_off, H,
                                               P + a.b_lin_off, 1, RB200_ACT_LINEAR, scr, d.ld_s,
                                               Wst);
  const bool has_loss = a.reward != nullptr;
  if (tid < R) {
    const int r = tid, b = row0 + r, v = s_valid[r];
    float sq = 0.f;
    if (b < B) {
      const float y = scr[r * d.ld_s];
      a.acc_reward[b] = y;
      if (a.step_labels)
        for (int m = 0; m < a.multi_steps; ++m)
          a.step_labels[(size_t)b * a.multi_steps + m] = m == v - 1 ? 1.f : 0.f;
      if (has_loss) {
        // cumsum(reward * fp32(gamma ** t))[v - 1]: fp32 products, an fp64 sum rounded once
        double s = 0.0;
        for (int t = 0; t < v; ++t)
          s = __dadd_rn(s, (double)__fmul_rn(a.reward[(size_t)t * B + b], a.discount[t]));
        const float tg = __double2float_rn(s);
        if (a.target) a.target[b] = tg;
        const float df = __fsub_rn(y, tg);
        sq = __fmul_rn(df, df);
        if (a.dy) {
          const float g = __fmul_rn(__fdiv_rn(2.f, (float)B), df);
          for (int t = 0; t < T; ++t) a.dy[(size_t)t * B + b] = t == v - 1 ? g : 0.f;
        }
      }
    }
    s_row[r] = sq;
  }
  __syncthreads();
  if (has_loss && tid == 0) {
    float acc[1] = {0.f};
    for (int r = 0; r < R; ++r) acc[0] += s_row[r];
    float* loss = a.loss;
    const float n = (float)B;
    finish_serial<1>(a.loss_partials, a.tile_counter, acc,
                     [=](const float (&s)[1]) { loss[0] = __fdiv_rn(s[0], n); });
  }
}

// ---------------------------------------------------------------------------
// Backward through time: dGates[l, t], then dh0 = sum_l dL/dh_{-1}
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kS2rNT, 1) s2r_bwd_kernel(const rb200_seq2reward_args_t a) {
  constexpr int NT = kS2rNT, R = kS2rR;
  const S2rDims d = s2r_dims(a);
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* dhr = Wst + 2 * wstage_floats<kLstmKC>();  // [L][R][ld_h]
  float* dcs = dhr + d.L * R * d.ld_h;              // [L][R][ld_h]
  float* dx = dcs + d.L * R * d.ld_h;               // [R][ld_h]
  float* scr = dx + R * d.ld_h;                     // [R][ld_s]
  const int row0 = blockIdx.x * R, tid = threadIdx.x;
  const int T = d.T, B = d.B, H = d.H;
  const float* wl = a.params + a.w_lin_off;
  for (int t = T - 1; t >= 0; --t) {
    // dh_top = dy[t] . W_lin: nonzero only on the row's valid step
    for (int i = tid; i < R * H; i += NT) {
      const int r = i / H, j = i - r * H, b = row0 + r;
      dx[r * d.ld_h + j] = b < B ? __fmul_rn(a.dy[(size_t)t * B + b], wl[j]) : 0.f;
    }
    __syncthreads();
    lstm_tile_bwd_step(a, T, B, H, d.L, t, row0, dhr, dcs, dx, d.ld_h, scr, d.ld_s, Wst);
    __syncthreads();
  }
  // every layer's initial h is the same map_linear output
  for (int i = tid; i < R * H; i += NT) {
    const int r = i / H, j = i - r * H, b = row0 + r;
    if (b >= B) continue;
    float s = dhr[r * d.ld_h + j];
    for (int l = 1; l < d.L; ++l) s = __fadd_rn(s, dhr[(l * R + r) * d.ld_h + j]);
    a.dh0[(size_t)b * H + j] = s;
  }
}

// ---------------------------------------------------------------------------
// Plan: one level of the prefix tree for states [b0, b0 + nb)
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t s2r_ordered(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float s2r_unordered(uint32_t u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__host__ __device__ inline long long s2r_pow(int a, int e) {
  long long p = 1;
  for (int i = 0; i < e; ++i) p *= a;
  return p;
}

__global__ void __launch_bounds__(kS2rNT, 1)
    s2r_plan_kernel(const rb200_seq2reward_plan_args_t pa, int level, int b0, int nb) {
  constexpr int NT = kS2rNT, R = kS2rR;
  const rb200_seq2reward_args_t& a = pa.net;
  const S2rDims d = s2r_dims(a);
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* xs = Wst + 2 * wstage_floats<kLstmKC>();
  float* hsm = xs + R * d.ld_x;
  float* csm = hsm + d.L * R * d.ld_h;
  float* scr = csm + d.L * R * d.ld_h;
  const int tid = threadIdx.x, A = d.A, H = d.H, L = d.L, k = pa.multi_steps;
  const int PP = R / A;                          // parents per CTA; their children fill PP * A rows
  const long long Ap = s2r_pow(A, level - 1);    // nodes per state at the parents' level
  const long long n_par = (long long)nb * Ap;
  const long long p0 = (long long)blockIdx.x * PP;
  const int nvalid = (int)(n_par - p0 < PP ? n_par - p0 : PP) * A;
  const size_t node = (size_t)L * 2 * H;         // floats of one stored node
  if (level == 1) {
    // the root of each state: h0 = map_linear(state)
    for (int i = tid; i < R * d.S; i += NT) {
      const int r = i / d.S, c = i - r * d.S;
      xs[r * d.ld_x + c] = r < nvalid ? pa.state[(size_t)(b0 + p0 + r / A) * d.S + c] : 0.f;
    }
    __syncthreads();
    s2r_initial_state(a, d, xs, hsm, scr, Wst, nvalid);
    for (int i = tid; i < R * d.ld_x; i += NT) xs[i] = 0.f;
  } else {
    const long long stride = s2r_pow(A, k - level);  // parents' row stride (level - 1)
    for (int i = tid; i < L * R * H; i += NT) {
      const int l = i / (R * H), r = (i / H) % R, j = i % H;
      if (r >= nvalid) continue;
      const float* src = pa.workspace + (size_t)((p0 + r / A) * stride) * node + (size_t)l * 2 * H;
      hsm[(l * R + r) * d.ld_h + j] = src[j];
      csm[(l * R + r) * d.ld_h + j] = src[H + j];
    }
  }
  __syncthreads();
  if (tid < nvalid) xs[tid * d.ld_x + tid % A] = 1.f;
  __syncthreads();
  lstm_tile_step<false>(a, L, H, nvalid, 0, xs, d.ld_x, A, hsm, csm, d.ld_h, scr, d.ld_s, d.ld_g,
                        Wst, S2rNoStore());
  const float* P = a.params;
  tile_linear_fwd<NT, kLstmTM, kLstmKC, false>(hsm + (L - 1) * R * d.ld_h, d.ld_h, H,
                                               P + a.w_lin_off, H, P + a.b_lin_off, 1,
                                               RB200_ACT_LINEAR, scr, d.ld_s, Wst);
  if (tid < nvalid && (pa.q_all || level == k)) {
    const long long n = (p0 + tid / A) * A + tid % A;  // this node, within the chunk's level
    const long long b = n / (Ap * A), a0 = (n / Ap) % A;
    atomicMax(pa.qbits + ((size_t)(b0 + b) * k + (level - 1)) * A + a0,
              s2r_ordered(scr[tid * d.ld_s]));
  }
  if (level < k) {
    const long long stride = s2r_pow(A, k - 1 - level);
    for (int i = tid; i < L * R * H; i += NT) {
      const int l = i / (R * H), r = (i / H) % R, j = i % H;
      if (r >= nvalid) continue;
      const long long n = (p0 + r / A) * A + r % A;
      float* dst = pa.workspace + (size_t)(n * stride) * node + (size_t)l * 2 * H;
      dst[j] = hsm[(l * R + r) * d.ld_h + j];
      dst[H + j] = csm[(l * R + r) * d.ld_h + j];
    }
  }
}

__global__ void s2r_plan_finish_kernel(const rb200_seq2reward_plan_args_t pa) {
  const int A = pa.net.action_dim, k = pa.multi_steps;
  const long long n = (long long)pa.batch * k * A;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const float v = s2r_unordered(pa.qbits[i]);
    if (pa.q_all) pa.q_all[i] = v;
    if ((i / A) % k == k - 1) pa.q[(i / ((long long)k * A)) * A + i % A] = v;
  }
}

// ---------------------------------------------------------------------------
// Compress head: MSE over B * A, dL/dout, argmax agreement
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(kS2rHeadNT) s2r_compress_kernel(
    const rb200_seq2reward_compress_args_t a) {
  __shared__ float s_sq[kS2rHeadNT], s_ok[kS2rHeadNT];
  const int tid = threadIdx.x, b = blockIdx.x * kS2rHeadNT + tid, A = a.num_action;
  const float n = __fmul_rn((float)a.batch, (float)A);
  float sq = 0.f, ok = 0.f;
  if (b < a.batch) {
    const float* o = a.out + (size_t)b * A;
    const float* q = a.q + (size_t)b * A;
    int bo = 0, bq = 0;
    for (int c = 0; c < A; ++c) {
      const float df = __fsub_rn(o[c], q[c]);
      sq = __fadd_rn(sq, __fmul_rn(df, df));
      if (a.dout) a.dout[(size_t)b * A + c] = __fmul_rn(__fdiv_rn(2.f, n), df);
      if (o[c] > o[bo]) bo = c;  // first maximum
      if (q[c] > q[bq]) bq = c;
    }
    ok = bo == bq ? 1.f : 0.f;
  }
  s_sq[tid] = sq;
  s_ok[tid] = ok;
  __syncthreads();
  if (tid == 0) {
    float acc[2] = {0.f, 0.f};
    for (int r = 0; r < kS2rHeadNT; ++r) { acc[0] += s_sq[r]; acc[1] += s_ok[r]; }
    float* out = a.out_loss;
    const float nb = (float)a.batch;
    finish_serial<2>(a.loss_partials, a.tile_counter, acc, [=](const float (&s)[2]) {
      out[0] = __fdiv_rn(s[0], n);
      out[1] = __fdiv_rn(s[1], nb);
    });
  }
}

static int s2r_validate(const rb200_seq2reward_args_t* a, const char* who) {
  if (!a) { set_last_error("%s: args is null", who); return RB200_E_INVALID; }
  if (int rc = rb200_seq2reward_check_shape(a->state_dim, a->action_dim, a->hidden, a->layers, 1))
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
  if (!a->params || !a->state || !a->action) {
    set_last_error("%s: params, state and action are required", who);
    return RB200_E_INVALID;
  }
  return RB200_OK;
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_seq2reward_check_shape(int32_t S, int32_t A, int32_t H, int32_t L,
                                            int32_t k) {
  if (S < 1 || A < 1 || H < 1 || L < 1 || k < 1 || H > RB200_MDNRNN_MAX_HIDDEN ||
      L > RB200_MDNRNN_MAX_LAYERS || S > RB200_SEQ2REWARD_MAX_STATE ||
      A > RB200_SEQ2REWARD_MAX_ACTIONS || k > RB200_SEQ2REWARD_MAX_STEPS ||
      s2r_pow(A, k) > RB200_SEQ2REWARD_MAX_PERMUTATIONS) {
    set_last_error("rb200_seq2reward: unsupported shape (state_dim %d in [1, %d], action_dim %d "
                   "in [1, %d], hidden %d in [1, %d], layers %d in [1, %d], multi_steps %d in "
                   "[1, %d], action_dim ** multi_steps <= %d)", S, RB200_SEQ2REWARD_MAX_STATE, A,
                   RB200_SEQ2REWARD_MAX_ACTIONS, H, RB200_MDNRNN_MAX_HIDDEN, L,
                   RB200_MDNRNN_MAX_LAYERS, k, RB200_SEQ2REWARD_MAX_STEPS,
                   RB200_SEQ2REWARD_MAX_PERMUTATIONS);
    return RB200_E_INVALID;
  }
  // the tiles of the forward, backward and plan must fit the opt-in shared memory of one CTA
  rb200_seq2reward_args_t a = {};
  a.state_dim = S; a.action_dim = A; a.hidden = H; a.layers = L;
  const S2rDims d = s2r_dims(a);
  size_t smem = s2r_fwd_smem(d);
  if (s2r_bwd_smem(d) > smem) smem = s2r_bwd_smem(d);
  if (s2r_plan_smem(d) > smem) smem = s2r_plan_smem(d);
  if (smem > kS2rSmemLimit) {
    set_last_error("rb200_seq2reward: unsupported shape (state_dim %d, action_dim %d, hidden %d, "
                   "layers %d need %zu bytes of shared memory per CTA, more than %zu)", S, A, H,
                   L, smem, kS2rSmemLimit);
    return RB200_E_INVALID;
  }
  return RB200_OK;
}

extern "C" int rb200_seq2reward_forward(const rb200_seq2reward_args_t* a, void* stream) {
  if (int rc = s2r_validate(a, "rb200_seq2reward_forward")) return rc;
  const bool loss = a->reward || a->discount || a->loss_partials || a->tile_counter || a->loss;
  const bool train = a->hs || a->cs || a->acts || a->dy;
  if (!a->acc_reward ||
      (loss && !(a->reward && a->discount && a->loss_partials && a->tile_counter && a->loss)) ||
      (train && !(a->hs && a->cs && a->acts && a->dy && a->reward)) ||
      (a->step_labels && a->multi_steps < 1)) {
    set_last_error("rb200_seq2reward_forward: acc_reward is required; the loss needs reward, "
                   "discount, loss_partials, tile_counter and loss; training (hs, cs, acts, dy) "
                   "needs the loss; step_labels needs multi_steps >= 1");
    return RB200_E_INVALID;
  }
  const S2rDims d = s2r_dims(*a);
  return launch<s2r_fwd_kernel>(ceil_div(d.B, kS2rR), kS2rNT, s2r_fwd_smem(d),
                                (cudaStream_t)stream, "s2r_fwd_kernel launch", *a);
}

extern "C" int rb200_seq2reward_backward(const rb200_seq2reward_args_t* a, void* stream) {
  if (int rc = s2r_validate(a, "rb200_seq2reward_backward")) return rc;
  if (!a->cs || !a->acts || !a->dy || !a->dgates || !a->dh0) {
    set_last_error("rb200_seq2reward_backward: cs, acts, dy, dgates and dh0 are required");
    return RB200_E_INVALID;
  }
  const S2rDims d = s2r_dims(*a);
  return launch<s2r_bwd_kernel>(ceil_div(d.B, kS2rR), kS2rNT, s2r_bwd_smem(d),
                                (cudaStream_t)stream, "s2r_bwd_kernel launch", *a);
}

extern "C" int rb200_seq2reward_wgrad(const rb200_seq2reward_args_t* a, void* stream) {
  if (int rc = s2r_validate(a, "rb200_seq2reward_wgrad")) return rc;
  if (!a->hs || !a->dgates || !a->dy || !a->dh0 || !a->gpart || a->splits <= 0) {
    set_last_error("rb200_seq2reward_wgrad: hs, dgates, dy, dh0, gpart and splits > 0 are "
                   "required");
    return RB200_E_INVALID;
  }
  const S2rDims d = s2r_dims(*a);
  const size_t TB = (size_t)d.T * d.B, slot = (size_t)(d.T + 1) * d.B * d.H;
  WgradLayer jobs[kWgradMaxJobs] = {};
  int n = 0;
  for (int l = 0; l < d.L; ++l) {
    const float* dz = a->dgates + (size_t)l * TB * 4 * d.H;
    // dW_ih = dGates^T . x (x: the one-hot actions, or h_t of the layer below)
    WgradLayer& ih = jobs[n++];
    ih.A = l == 0 ? a->action : a->hs + (size_t)(l - 1) * slot + (size_t)d.B * d.H;
    ih.dZ = dz; ih.K = l == 0 ? d.A : d.H; ih.N = 4 * d.H;
    ih.w_off = a->w_ih_off[l]; ih.b_off = a->b_ih_off[l];
    // dW_hh = dGates^T . h_{t-1} (slot 0 = h0)
    WgradLayer& hh = jobs[n++];
    hh.A = a->hs + (size_t)l * slot;
    hh.dZ = dz; hh.K = d.H; hh.N = 4 * d.H;
    hh.w_off = a->w_hh_off[l]; hh.b_off = a->b_hh_off[l];
  }
  // lstm_linear over every step: dy is zero off each row's valid step
  WgradLayer& head = jobs[n++];
  head.A = a->hs + (size_t)(d.L - 1) * slot + (size_t)d.B * d.H;
  head.dZ = a->dy; head.K = d.H; head.N = 1;
  head.w_off = a->w_lin_off; head.b_off = a->b_lin_off;
  if (int rc = wgrad_jobs_launch(jobs, n, (int)TB, a->splits, a->gpart, a->n_params,
                                 (cudaStream_t)stream, "rb200_seq2reward_wgrad"))
    return rc;
  // map_linear over the B first states
  WgradLayer map = {};
  map.A = a->state; map.dZ = a->dh0; map.K = d.S; map.N = d.H;
  map.w_off = a->w_map_off; map.b_off = a->b_map_off;
  return wgrad_jobs_launch(&map, 1, d.B, a->splits, a->gpart, a->n_params, (cudaStream_t)stream,
                           "rb200_seq2reward_wgrad(map_linear)");
}

static long long s2r_plan_node_bytes(int A, int k, int H, int L) {
  return k < 2 ? 0 : s2r_pow(A, k - 1) * L * 2 * H * (long long)sizeof(float);
}

extern "C" int64_t rb200_seq2reward_plan_workspace_bytes(int32_t batch, int32_t A, int32_t k,
                                                         int32_t H, int32_t L) {
  if (batch < 1 || rb200_seq2reward_check_shape(1, A, H, L, k)) return -1;
  const long long per = s2r_plan_node_bytes(A, k, H, L);
  if (per == 0) return 0;
  long long nb = RB200_SEQ2REWARD_PLAN_BUDGET_BYTES / per;
  if (nb > batch) nb = batch;
  if (nb < 1) nb = 1;
  return nb * per;
}

extern "C" int rb200_seq2reward_plan(const rb200_seq2reward_plan_args_t* pa, void* stream) {
  if (!pa) { set_last_error("rb200_seq2reward_plan: args is null"); return RB200_E_INVALID; }
  const rb200_seq2reward_args_t& a = pa->net;
  if (int rc = rb200_seq2reward_check_shape(a.state_dim, a.action_dim, a.hidden, a.layers,
                                            pa->multi_steps))
    return rc;
  const int A = a.action_dim, k = pa->multi_steps, B = pa->batch;
  const long long per = s2r_plan_node_bytes(A, k, a.hidden, a.layers);
  if (B < 1 || !a.params || !pa->state || !pa->q || !pa->qbits ||
      (per > 0 && (!pa->workspace || pa->workspace_bytes < per))) {
    set_last_error("rb200_seq2reward_plan: batch %d must be positive; params, state, q and qbits "
                   "are required, and a workspace of at least %lld bytes", B, per);
    return RB200_E_INVALID;
  }
  const cudaStream_t st = (cudaStream_t)stream;
  if (int rc = check_cuda(cudaMemsetAsync(pa->qbits, 0, sizeof(uint32_t) * (size_t)B * k * A, st),
                          "rb200_seq2reward_plan memset"))
    return rc;
  const int chunk = per > 0 ? (int)(pa->workspace_bytes / per < B ? pa->workspace_bytes / per : B)
                            : B;
  const S2rDims d = s2r_dims(a);
  const int PP = kS2rR / A;
  for (int b0 = 0; b0 < B; b0 += chunk) {
    const int nb = B - b0 < chunk ? B - b0 : chunk;
    for (int level = 1; level <= k; ++level) {
      const long long parents = (long long)nb * s2r_pow(A, level - 1);
      const long long grid = (parents + PP - 1) / PP;
      if (int rc = launch<s2r_plan_kernel>((unsigned)grid, kS2rNT, s2r_plan_smem(d), st,
                                           "s2r_plan_kernel launch", *pa, level, b0, nb))
        return rc;
    }
  }
  const long long n = (long long)B * k * A;
  const int blocks = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
  s2r_plan_finish_kernel<<<blocks, 256, 0, st>>>(*pa);
  return check_cuda(cudaGetLastError(), "s2r_plan_finish_kernel launch");
}

extern "C" int rb200_seq2reward_compress_head(const rb200_seq2reward_compress_args_t* a,
                                              void* stream) {
  if (!a || a->batch < 1 || a->num_action < 1 || !a->out || !a->q || !a->loss_partials ||
      !a->tile_counter || !a->out_loss) {
    set_last_error("rb200_seq2reward_compress_head: batch and num_action must be positive; out, "
                   "q, loss_partials, tile_counter and out_loss are required");
    return RB200_E_INVALID;
  }
  return launch<s2r_compress_kernel>(ceil_div(a->batch, kS2rHeadNT), kS2rHeadNT, 0,
                                     (cudaStream_t)stream, "s2r_compress_kernel launch", *a);
}
