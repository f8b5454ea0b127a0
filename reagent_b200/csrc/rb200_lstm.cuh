// reagent_b200 -- the row-tile LSTM step shared by the MDN-RNN (rb200_mdnrnn.cu) and Seq2Reward
// (rb200_seq2reward.cu) kernels.
//
// One CTA of kLstmNT threads carries kLstmR rows; h and c of every layer stay in shared memory and
// the weights stream through the 3xTF32 row-tile primitives of rb200_tile.cuh.  Gates follow
// ATen's CPU LSTM cell:
//   gates = (h . W_hh^T + b_hh) + (x . W_ih^T + b_ih),   i, f, g, o = chunk(gates, 4)
//   c' = f * c + i * g  (each product rounded),   h' = o * tanh(c')
// The argument struct `a` of either kernel provides `params` (the arena) and the per-layer
// offsets w_ih_off / w_hh_off / b_ih_off / b_hh_off; the backward also reads acts / cs and writes
// dgates in the layouts below.
#pragma once
#include <math.h>

#include "rb200_tile.cuh"

namespace rb200 {

constexpr int kLstmNT = 256, kLstmTM = 4, kLstmKC = 32;
constexpr int kLstmR = (kLstmNT / 64) * kLstmTM;  // 16 rows per CTA

// hs / cs [L, T+1, B, H]: slot s (0 = the initial state) of layer l, row b
__device__ __forceinline__ size_t lstm_hc_idx(int T, int B, int H, int l, int s, int b) {
  return (((size_t)l * (T + 1) + s) * B + b) * H;
}
// acts / dgates [L, T, B, 4H] (i, f, g, o): layer l, step t, row b
__device__ __forceinline__ size_t lstm_gate_idx(int T, int B, int H, int l, int t, int b) {
  return (((size_t)l * T + t) * B + b) * (size_t)(4 * H);
}

// One step of every layer for the tile's rows row0 + r, r < kLstmR.  xs: the step's input
// (K0 columns, stride ld_x); hsm / csm: [L][R][ld_h], the previous step's h / c, overwritten with
// this step's (rows >= B zeroed); scr: [R][ld_s] with the two gate products at columns 0 and ld_g.
// store(l, r, b, j, gi, gf, gg, go, cn, hn) runs for every element of a row b < B.  kRotate is
// tile_linear_fwd's k-chunk rotation by blockIdx.x.
template <bool kRotate, typename Args, typename Store>
__device__ __forceinline__ void lstm_tile_step(const Args& a, int L, int H, int B, int row0,
                                               const float* xs, int ld_x, int K0, float* hsm,
                                               float* csm, int ld_h, float* scr, int ld_s, int ld_g,
                                               float* Wst, Store store) {
  constexpr int NT = kLstmNT, R = kLstmR;
  const int tid = threadIdx.x, H4 = 4 * H;
  const float* P = a.params;
  for (int l = 0; l < L; ++l) {
    float* h = hsm + l * R * ld_h;
    float* c = csm + l * R * ld_h;
    const float* in = l == 0 ? xs : hsm + (l - 1) * R * ld_h;
    const int K = l == 0 ? K0 : H, ld_in = l == 0 ? ld_x : ld_h;
    tile_linear_fwd<NT, kLstmTM, kLstmKC, kRotate>(in, ld_in, K, P + a.w_ih_off[l], K,
                                                   P + a.b_ih_off[l], H4, RB200_ACT_LINEAR, scr,
                                                   ld_s, Wst);
    tile_linear_fwd<NT, kLstmTM, kLstmKC, kRotate>(h, ld_h, H, P + a.w_hh_off[l], H,
                                                   P + a.b_hh_off[l], H4, RB200_ACT_LINEAR,
                                                   scr + ld_g, ld_s, Wst);
    for (int i = tid; i < R * H; i += NT) {
      const int r = i / H, j = i - r * H, b = row0 + r;
      const float* g1 = scr + r * ld_s;
      const float* g2 = g1 + ld_g;
      const float gi = sigmoidf(__fadd_rn(g2[j], g1[j]));
      const float gf = sigmoidf(__fadd_rn(g2[H + j], g1[H + j]));
      const float gg = tanhf(__fadd_rn(g2[2 * H + j], g1[2 * H + j]));
      const float go = sigmoidf(__fadd_rn(g2[3 * H + j], g1[3 * H + j]));
      const float cn = __fadd_rn(__fmul_rn(gf, c[r * ld_h + j]), __fmul_rn(gi, gg));
      const float hn = __fmul_rn(go, tanhf(cn));
      c[r * ld_h + j] = b < B ? cn : 0.f;
      h[r * ld_h + j] = b < B ? hn : 0.f;
      if (b < B) store(l, r, b, j, gi, gf, gg, go, cn, hn);
    }
    __syncthreads();
  }
}

// Backward through every layer at step t (top layer first) for the tile's rows.  On entry dx
// holds dL/dh_t of the top layer from the head; dhr / dcs ([L][R][ld_h]) carry each layer's
// dL/dh_t and dL/dc_t through the recurrence and leave with dL/dh_{t-1} and dL/dc_{t-1}.  Writes
// dGates[l, t] of rows < B into a.dgates; scr ([R][ld_s]) holds the step's dGates.
template <typename Args>
__device__ __forceinline__ void lstm_tile_bwd_step(const Args& a, int T, int B, int H, int L,
                                                   int t, int row0, float* dhr, float* dcs,
                                                   float* dx, int ld_h, float* scr, int ld_s,
                                                   float* Wst) {
  constexpr int NT = kLstmNT, R = kLstmR;
  const int tid = threadIdx.x, H4 = 4 * H;
  const float* P = a.params;
  for (int l = L - 1; l >= 0; --l) {
    float* dh_rec = dhr + l * R * ld_h;
    float* dc = dcs + l * R * ld_h;
    for (int i = tid; i < R * H; i += NT) {
      const int r = i / H, j = i - r * H, b = row0 + r;
      float* dg = scr + r * ld_s;
      if (b >= B) {
        dg[j] = dg[H + j] = dg[2 * H + j] = dg[3 * H + j] = 0.f;
        continue;
      }
      const float* ga = a.acts + lstm_gate_idx(T, B, H, l, t, b);
      const float gi = ga[j], gf = ga[H + j], gg = ga[2 * H + j], go = ga[3 * H + j];
      const float cn = a.cs[lstm_hc_idx(T, B, H, l, t + 1, b) + j];
      const float cp = a.cs[lstm_hc_idx(T, B, H, l, t, b) + j];
      const float tc = tanhf(cn);
      const float dh = __fadd_rn(dx[r * ld_h + j], dh_rec[r * ld_h + j]);
      const float dct = __fadd_rn(dc[r * ld_h + j],
                                  __fmul_rn(__fmul_rn(dh, go), __fsub_rn(1.f, __fmul_rn(tc, tc))));
      const float di = __fmul_rn(__fmul_rn(dct, gg), __fmul_rn(__fsub_rn(1.f, gi), gi));
      const float df = __fmul_rn(__fmul_rn(dct, cp), __fmul_rn(__fsub_rn(1.f, gf), gf));
      const float dgg = __fmul_rn(__fmul_rn(dct, gi), __fsub_rn(1.f, __fmul_rn(gg, gg)));
      const float dgo = __fmul_rn(__fmul_rn(dh, tc), __fmul_rn(__fsub_rn(1.f, go), go));
      dc[r * ld_h + j] = __fmul_rn(dct, gf);
      dg[j] = di; dg[H + j] = df; dg[2 * H + j] = dgg; dg[3 * H + j] = dgo;
      float* out = a.dgates + lstm_gate_idx(T, B, H, l, t, b);
      out[j] = di; out[H + j] = df; out[2 * H + j] = dgg; out[3 * H + j] = dgo;
    }
    __syncthreads();
    // dL/dh_{t-1} of this layer, and dL/dh_t of the layer below
    tile_linear_bwd<NT, kLstmTM, kLstmKC>(scr, ld_s, H4, P + a.w_hh_off[l], H, H, nullptr, 0, 0,
                                          dh_rec, ld_h, Wst);
    if (l > 0)
      tile_linear_bwd<NT, kLstmTM, kLstmKC>(scr, ld_s, H4, P + a.w_ih_off[l], H, H, nullptr, 0, 0,
                                            dx, ld_h, Wst);
  }
}

}  // namespace rb200
