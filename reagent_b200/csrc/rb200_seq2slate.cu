// reagent_b200 -- Seq2Slate transformer (reagent/models/seq2slate.py): encoder, teacher-forced
// decoder with the per-symbol / per-sequence log-probability heads, and the whole ranking decode,
// each as ONE launch.  One CTA carries one slate at a time through every layer; a slate's
// activations, the cross-attention keys / values of the memory and the self-attention cache of
// every decoder layer live in that CTA's workspace slice: shared memory when it fits, else the
// caller's global workspace.
//
// The decoder runs one position at a time, teacher-forced or not: position t's output at every
// layer depends only on positions <= t (causal self-attention) and its cross-attention mask only
// on tgt_in_idx[0..t], so computing row t from the cached keys / values of rows < t gives the
// reference's full-recompute result.  See include/reagent_b200.h for the contract.
#include "rb200_common.cuh"

namespace rb200 {

constexpr int kS2sThreads = 256;
constexpr int kS2sWarps = kS2sThreads / 32;
constexpr int kS2sMaxN = RB200_SEQ2SLATE_MAX_CANDIDATES;
constexpr int kS2sMaxCtas = RB200_SEQ2SLATE_MAX_CTAS;
constexpr float kLayerNormEps = 1e-5f;
// A CTA's workspace slice goes to shared memory when it takes at most this many bytes (every
// shape of the reference's tests, and d 128 / FFN 512 at N 32): the decoder's one-row steps are
// latency-bound, and shared memory answers in a tenth of an L2 round trip.
constexpr size_t kS2sSmemMax = 200 * 1024;
constexpr float kProbFloor = 1e-40f;  // fp32 denormal: the library is built without FTZ

// offsets of the parameters in the reference's parameters() order
enum EncParam { E_IN_W, E_IN_B, E_OUT_W, E_OUT_B, E_L1_W, E_L1_B, E_L2_W, E_L2_B, E_N1_W, E_N1_B,
                E_N2_W, E_N2_B, E_COUNT };
enum DecParam { D_SA_IN_W, D_SA_IN_B, D_SA_OUT_W, D_SA_OUT_B, D_CA_IN_W, D_CA_IN_B, D_CA_OUT_W,
                D_CA_OUT_B, D_L1_W, D_L1_B, D_L2_W, D_L2_B, D_N1_W, D_N1_B, D_N2_W, D_N2_B,
                D_N3_W, D_N3_B, D_COUNT };

struct S2sShape {
  int N, T, S, C, se, ce, d, H, hd, F, L, wide;
};

__host__ __device__ inline S2sShape s2s_shape(const rb200_seq2slate_args_t& a) {
  S2sShape s;
  s.N = a.src_len;
  s.T = a.tgt_len;
  s.S = a.state_dim;
  s.C = a.candidate_dim;
  s.se = a.state_embed_dim;
  s.ce = a.dim_model - a.state_embed_dim;
  s.d = a.dim_model;
  s.H = a.num_heads;
  s.hd = a.dim_model / a.num_heads;
  s.F = a.dim_feedforward;
  s.L = a.layers;
  s.wide = 3 * s.d > s.F ? 3 * s.d : s.F;
  return s;
}

// Floats of one CTA's workspace slice (see S2sWs).
__host__ __device__ inline long long s2s_ws_floats(const S2sShape& s) {
  auto r4 = [](long long n) { return (n + 3) & ~3LL; };
  return r4((long long)s.N * s.d) * 2 + r4((long long)s.N * s.wide) +
         r4((long long)s.L * 2 * s.N * s.d) + r4((long long)s.L * 2 * s.T * s.d) +
         r4((long long)s.H * s.N) + r4(s.N) + 4 * r4(s.d) + r4(s.wide) + r4(s.C);
}

struct S2sWs {
  float *X, *Z, *Y, *kvc, *kvs, *hp, *score, *x, *z, *q, *se, *y, *feat;
  __device__ S2sWs(float* base, const S2sShape& s) {
    auto r4 = [](long long n) { return (n + 3) & ~3LL; };
    float* p = base;
    X = p; p += r4((long long)s.N * s.d);
    Z = p; p += r4((long long)s.N * s.d);
    Y = p; p += r4((long long)s.N * s.wide);
    kvc = p; p += r4((long long)s.L * 2 * s.N * s.d);
    kvs = p; p += r4((long long)s.L * 2 * s.T * s.d);
    hp = p; p += r4((long long)s.H * s.N);
    score = p; p += r4(s.N);
    x = p; p += r4(s.d);
    z = p; p += r4(s.d);
    q = p; p += r4(s.d);
    se = p; p += r4(s.d);
    y = p; p += r4(s.wide);
    feat = p;
  }
};

// out[r, o] = act((in[r, :K] . W[o, :K] (+ W[o, K] * extra) + b[o]) * scale) for r < rows, o < O.
// W rows are `ldw` apart (the positional encoding's [d, d + 1] weight passes its last column as
// `extra`).  Four rows per thread share each weight load.  Ends with a block barrier.
__device__ void s2s_linear(const float* in, int ld_in, int rows, int K, const float* W, int ldw,
                           const float* b, float* out, int ld_out, int O, float scale, bool relu,
                           bool has_extra = false, float extra = 0.f) {
  const int groups = (rows + 3) >> 2;
  for (int w = threadIdx.x; w < groups * O; w += blockDim.x) {
    const int o = w % O, r0 = (w / O) * 4;
    const int nr = min(4, rows - r0);
    const float* __restrict__ wr = W + (size_t)o * ldw;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const float* i0 = in + (size_t)r0 * ld_in;
    for (int k = 0; k < K; ++k) {
      const float wk = __ldg(wr + k);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < nr) acc[j] = fmaf(i0[(size_t)j * ld_in + k], wk, acc[j]);
    }
    const float tail = has_extra ? __ldg(wr + K) * extra : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j >= nr) break;
      float v = (acc[j] + tail + __ldg(b + o)) * scale;
      if (relu) v = fmaxf(v, 0.f);
      out[(size_t)(r0 + j) * ld_out + o] = v;
    }
  }
  __syncthreads();
}

// x[r] = LayerNorm(x[r] + y[r]) over d (biased variance, eps 1e-5), one warp per row.
__device__ void s2s_add_layernorm(float* x, const float* y, int ld_y, int rows, int d,
                                  const float* g, const float* bt) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < rows; r += kS2sWarps) {
    float* xr = x + (size_t)r * d;
    const float* yr = y + (size_t)r * ld_y;
    float v[RB200_SEQ2SLATE_MAX_DIM_MODEL / 32];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < RB200_SEQ2SLATE_MAX_DIM_MODEL / 32; ++i) {
      const int c = lane + 32 * i;
      v[i] = c < d ? xr[c] + yr[c] : 0.f;
      s += v[i];
    }
    const float mean = warp_sum(s) / (float)d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < RB200_SEQ2SLATE_MAX_DIM_MODEL / 32; ++i) {
      const int c = lane + 32 * i;
      const float dv = c < d ? v[i] - mean : 0.f;
      q = fmaf(dv, dv, q);
    }
    const float rstd = rsqrtf(warp_sum(q) / (float)d + kLayerNormEps);
#pragma unroll
    for (int i = 0; i < RB200_SEQ2SLATE_MAX_DIM_MODEL / 32; ++i) {
      const int c = lane + 32 * i;
      if (c < d) xr[c] = (v[i] - mean) * rstd * g[c] + bt[c];
    }
  }
  __syncthreads();
}

// Softmax weights of one query head over `nk` keys, in one warp: p[j] = softmax_j(q . k_j /
// sqrt(hd)) with keys where masked(j) is true at -inf.  Returns the weights in p (shared).
template <typename Masked>
__device__ __forceinline__ void s2s_head_weights(const float* q, const float* k, int ldk, int nk,
                                                 int hd, float scale, const Masked& masked,
                                                 float* p) {
  const int lane = threadIdx.x & 31;
  float mx = -INFINITY;
  for (int j = lane; j < nk; j += 32) {
    float s = -INFINITY;
    if (!masked(j)) {
      const float* kj = k + (size_t)j * ldk;
      float dot = 0.f;
      for (int c = 0; c < hd; ++c) dot = fmaf(q[c], kj[c], dot);
      s = dot * scale;
    }
    p[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < nk; j += 32) {
    const float e = p[j] == -INFINITY ? 0.f : expf(p[j] - mx);
    p[j] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  __syncwarp();
  for (int j = lane; j < nk; j += 32) p[j] = p[j] / sum;
  __syncwarp();
}

// out[i, h*hd + c] = sum_j softmax(...)[j] v[j, h*hd + c] for `nq` query rows and every head:
// one warp per (row, head).
template <typename Masked>
__device__ void s2s_attention(const float* Q, int ldq, int nq, const float* K, const float* V,
                              int ldkv, int nk, const S2sShape& s, const Masked& masked,
                              float* out, int ldo, float (*s_p)[kS2sMaxN]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float scale = 1.f / sqrtf((float)s.hd);
  for (int w = warp; w < nq * s.H; w += kS2sWarps) {
    const int i = w / s.H, h = w % s.H;
    float* p = s_p[warp];
    s2s_head_weights(Q + (size_t)i * ldq + h * s.hd, K + h * s.hd, ldkv, nk, s.hd, scale,
                     [&](int j) { return masked(i, j); }, p);
    for (int c = lane; c < s.hd; c += 32) {
      float acc = 0.f;
      for (int j = 0; j < nk; ++j) acc = fmaf(p[j], V[(size_t)j * ldkv + h * s.hd + c], acc);
      out[(size_t)i * ldo + h * s.hd + c] = acc;
    }
    __syncwarp();
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kS2sThreads, 4) seq2slate_kernel(const rb200_seq2slate_args_t a,
                                                                 bool smem_ws) {
  extern __shared__ float4 s_dyn[];
  const S2sShape s = s2s_shape(a);
  const float* P = a.params;
  auto enc = [&](int l, int p) { return P + a.off[l * E_COUNT + p]; };
  const int dec0 = s.L * E_COUNT + 2;
  auto dec = [&](int l, int p) { return P + a.off[dec0 + l * D_COUNT + p]; };
  const float* w_score = P + a.off[s.L * E_COUNT];
  const float* b_score = P + a.off[s.L * E_COUNT + 1];
  const int tail = dec0 + s.L * D_COUNT;
  const float* w_pe = P + a.off[tail];
  const float* b_pe = P + a.off[tail + 1];
  const float* w_st = P + a.off[tail + 2];
  const float* b_st = P + a.off[tail + 3];
  const float* w_ca = P + a.off[tail + 4];
  const float* b_ca = P + a.off[tail + 5];
  const float sq_se = (float)sqrt((double)s.se), sq_ce = (float)sqrt((double)s.ce);
  const int NC = s.N + 2, d = s.d;
  const bool forced = a.decode == RB200_SEQ2SLATE_DECODE_FORCED;
  const bool frechet = a.arch == RB200_SEQ2SLATE_ARCH_FRECHET_SORT;

  __shared__ float s_p[kS2sWarps][kS2sMaxN];
  __shared__ float s_probs[kS2sMaxN + 2];
  __shared__ unsigned char s_masked[kS2sMaxN + 2];
  __shared__ int s_idx;
  __shared__ float s_prod;

  S2sWs ws(smem_ws ? reinterpret_cast<float*>(s_dyn)
                   : a.workspace + (size_t)blockIdx.x * s2s_ws_floats(s), s);
  const int tid = threadIdx.x;

  for (int b = blockIdx.x; b < a.batch; b += gridDim.x) {
    const float* src = a.src_seq + (size_t)b * s.N * s.C;
    // ---- embedders: X = cat(state_embed repeated, candidate_embed) ----
    s2s_linear(a.state + (size_t)b * s.S, s.S, 1, s.S, w_st, s.S, b_st, ws.se, s.se, s.se, sq_se,
               false);
    s2s_linear(src, s.C, s.N, s.C, w_ca, s.C, b_ca, ws.X + s.se, d, s.ce, sq_ce, false);
    for (int i = tid; i < s.N * s.se; i += blockDim.x) ws.X[(i / s.se) * d + i % s.se] = ws.se[i % s.se];
    __syncthreads();
    // ---- post-norm encoder layers ----
    for (int l = 0; l < s.L; ++l) {
      s2s_linear(ws.X, d, s.N, d, enc(l, E_IN_W), d, enc(l, E_IN_B), ws.Y, 3 * d, 3 * d, 1.f, false);
      s2s_attention(ws.Y, 3 * d, s.N, ws.Y + d, ws.Y + 2 * d, 3 * d, s.N, s,
                    [](int, int) { return false; }, ws.Z, d, s_p);
      s2s_linear(ws.Z, d, s.N, d, enc(l, E_OUT_W), d, enc(l, E_OUT_B), ws.Y, d, d, 1.f, false);
      s2s_add_layernorm(ws.X, ws.Y, d, s.N, d, enc(l, E_N1_W), enc(l, E_N1_B));
      s2s_linear(ws.X, d, s.N, d, enc(l, E_L1_W), d, enc(l, E_L1_B), ws.Y, s.F, s.F, 1.f, true);
      s2s_linear(ws.Y, s.F, s.N, s.F, enc(l, E_L2_W), s.F, enc(l, E_L2_B), ws.Z, d, d, 1.f, false);
      s2s_add_layernorm(ws.X, ws.Z, d, s.N, d, enc(l, E_N2_W), enc(l, E_N2_B));
    }
    // ---- memory-side work done once per slate ----
    if (frechet) {
      s2s_linear(ws.X, d, s.N, d, w_score, d, b_score, ws.score, 1, 1, 1.f, false);
    } else {
      for (int l = 0; l < s.L; ++l)  // K, V of the cross-attention (only K is read in the last)
        s2s_linear(ws.X, d, s.N, d, dec(l, D_CA_IN_W) + (size_t)d * d, d, dec(l, D_CA_IN_B) + d,
                   ws.kvc + (size_t)l * 2 * s.N * d, 2 * d, l + 1 < s.L ? 2 * d : d, 1.f, false);
    }
    for (int i = tid; i < NC; i += blockDim.x) s_masked[i] = 0;
    if (tid == 0) s_prod = 1.f;
    __syncthreads();

    // ---- decoder, one position per step ----
    for (int t = 0; t < s.T; ++t) {
      if (tid == 0) {
        long long v;
        if (forced) v = a.tgt_in_idx[(size_t)b * s.T + t];
        else v = t == 0 ? 1 : a.ranked_idx[(size_t)b * s.T + t - 1];
        s_idx = (int)v;
        if (v >= 0 && v < NC) s_masked[v] = 1;  // pytorch_decoder_mask / mask_logits_by_idx
      }
      __syncthreads();
      const int in_idx = s_idx;
      if (frechet) {
        // softmax over the scores of the candidates not yet masked; columns 0, 1 are -inf
        if (tid < 32) {
          float mx = -INFINITY;
          for (int j = tid; j < s.N; j += 32)
            if (!s_masked[j + 2]) mx = fmaxf(mx, ws.score[j]);
          mx = warp_max(mx);
          float sum = 0.f;
          for (int j = tid; j < s.N; j += 32) {
            const float e = s_masked[j + 2] ? 0.f : expf(ws.score[j] - mx);
            s_probs[j + 2] = e;
            sum += e;
          }
          sum = warp_sum(sum);
          __syncwarp();
          for (int j = tid; j < s.N; j += 32) s_probs[j + 2] = s_probs[j + 2] / sum;
          if (tid < 2) s_probs[tid] = 0.f;
        }
        __syncthreads();
      } else {
        // decoder input: cat(state_embed, candidate_embed(features of in_idx)), then
        // relu(pos_embed(cat(x, t)))
        const float* feat;
        if (forced) {
          feat = a.tgt_in_seq + ((size_t)b * s.T + t) * s.C;
        } else if (in_idx >= 2) {
          feat = src + (size_t)(in_idx - 2) * s.C;
        } else {
          for (int c = tid; c < s.C; c += blockDim.x) ws.feat[c] = 0.f;
          __syncthreads();
          feat = ws.feat;
        }
        s2s_linear(feat, s.C, 1, s.C, w_ca, s.C, b_ca, ws.z + s.se, s.ce, s.ce, sq_ce, false);
        for (int c = tid; c < s.se; c += blockDim.x) ws.z[c] = ws.se[c];
        __syncthreads();
        s2s_linear(ws.z, d, 1, d, w_pe, d + 1, b_pe, ws.x, d, d, 1.f, true, true, (float)t);
        for (int l = 0; l < s.L; ++l) {
          float* kc = ws.kvs + (size_t)l * 2 * s.T * d;  // [T, 2d]: k, v of each position
          // causal self-attention: this row's q, k, v; k, v appended to the cache
          s2s_linear(ws.x, d, 1, d, dec(l, D_SA_IN_W), d, dec(l, D_SA_IN_B), ws.y, 3 * d, 3 * d,
                     1.f, false);
          for (int c = tid; c < 2 * d; c += blockDim.x) kc[(size_t)t * 2 * d + c] = ws.y[d + c];
          __syncthreads();
          s2s_attention(ws.y, 3 * d, 1, kc, kc + d, 2 * d, t + 1, s,
                        [](int, int) { return false; }, ws.z, d, s_p);
          s2s_linear(ws.z, d, 1, d, dec(l, D_SA_OUT_W), d, dec(l, D_SA_OUT_B), ws.y, d, d, 1.f,
                     false);
          s2s_add_layernorm(ws.x, ws.y, d, 1, d, dec(l, D_N1_W), dec(l, D_N1_B));
          // cross-attention over the memory, candidates chosen so far masked
          s2s_linear(ws.x, d, 1, d, dec(l, D_CA_IN_W), d, dec(l, D_CA_IN_B), ws.q, d, d, 1.f,
                     false);
          const float* kv = ws.kvc + (size_t)l * 2 * s.N * d;
          const auto cross_masked = [&](int, int j) { return s_masked[j + 2] != 0; };
          if (l + 1 < s.L) {
            s2s_attention(ws.q, d, 1, kv, kv + d, 2 * d, s.N, s, cross_masked, ws.z, d, s_p);
            s2s_linear(ws.z, d, 1, d, dec(l, D_CA_OUT_W), d, dec(l, D_CA_OUT_B), ws.y, d, d, 1.f,
                       false);
            s2s_add_layernorm(ws.x, ws.y, d, 1, d, dec(l, D_N2_W), dec(l, D_N2_B));
            s2s_linear(ws.x, d, 1, d, dec(l, D_L1_W), d, dec(l, D_L1_B), ws.y, s.F, s.F, 1.f, true);
            s2s_linear(ws.y, s.F, 1, s.F, dec(l, D_L2_W), s.F, dec(l, D_L2_B), ws.z, d, d, 1.f,
                       false);
            s2s_add_layernorm(ws.x, ws.z, d, 1, d, dec(l, D_N3_W), dec(l, D_N3_B));
          } else {
            // DecoderLastLayerPytorch: the head-averaged attention weights are the probabilities
            const int lane = tid & 31, warp = tid >> 5;
            const float scale = 1.f / sqrtf((float)s.hd);
            for (int h = warp; h < s.H; h += kS2sWarps) {
              float* p = s_p[warp];
              s2s_head_weights(ws.q + h * s.hd, kv + h * s.hd, 2 * d, s.N, s.hd, scale,
                               [&](int j) { return cross_masked(0, j); }, p);
              for (int j = lane; j < s.N; j += 32) ws.hp[(size_t)h * s.N + j] = p[j];
              __syncwarp();
            }
            __syncthreads();
            for (int j = tid; j < s.N; j += blockDim.x) {
              float acc = 0.f;
              for (int h = 0; h < s.H; ++h) acc += ws.hp[(size_t)h * s.N + j];
              s_probs[j + 2] = acc / (float)s.H;
            }
            if (tid < 2) s_probs[tid] = 0.f;
            __syncthreads();
          }
        }
      }

      // ---- this step's probabilities: outputs, the next symbol, the sequence product ----
      float* prow = a.probs ? a.probs + ((size_t)b * s.T + t) * NC : nullptr;
      if (frechet && a.decode == RB200_SEQ2SLATE_DECODE_GREEDY) {
        // _greedy_rank: argsort of the first step's probabilities (ties: lowest index first),
        // every selected symbol's probability set to 1
        if (tid == 0) {
          for (int r = 0; r < s.T; ++r) {
            int best = -1;
            for (int j = 2; j < NC; ++j)
              if (s_masked[j] != 2 && (best < 0 || s_probs[j] > s_probs[best])) best = j;
            s_masked[best] = 2;
            a.ranked_idx[(size_t)b * s.T + r] = best;
          }
          a.seq_prob[b] = 1.f;
        }
        __syncthreads();
        if (a.probs)
          for (int i = tid; i < s.T * NC; i += blockDim.x) {
            const int r = i / NC, j = i % NC;
            a.probs[(size_t)b * s.T * NC + i] = a.ranked_idx[(size_t)b * s.T + r] == j ? 1.f : 0.f;
          }
        __syncthreads();
        break;
      }
      if (prow)
        for (int j = tid; j < NC; j += blockDim.x) prow[j] = s_probs[j];
      if (forced && a.log_probs) {
        float* lrow = a.log_probs + ((size_t)b * s.T + t) * NC;
        for (int j = tid; j < NC; j += blockDim.x) lrow[j] = logf(fmaxf(s_probs[j], kProbFloor));
      }
      if (tid == 0) {
        int out;
        if (forced) {
          const long long v = a.tgt_out_idx[(size_t)b * s.T + t];
          out = v >= 0 && v < NC ? (int)v : -1;
        } else if (a.decode == RB200_SEQ2SLATE_DECODE_GREEDY) {
          out = 0;  // torch.max: the first maximal index
          for (int j = 1; j < NC; ++j)
            if (s_probs[j] > s_probs[out]) out = j;
        } else {
          // inverse CDF over the candidate order: the first j with cumsum(p)[j] > u * sum(p),
          // among the symbols of nonzero probability
          float total = 0.f;
          for (int j = 0; j < NC; ++j) total += s_probs[j];
          const float u = a.noise[(size_t)b * s.T + t] * total;
          float c = 0.f;
          out = -1;
          int last = 0;
          for (int j = 0; j < NC; ++j) {
            if (s_probs[j] <= 0.f) continue;
            last = j;
            c += s_probs[j];
            if (c > u) { out = j; break; }
          }
          if (out < 0) out = last;
        }
        if (!forced) a.ranked_idx[(size_t)b * s.T + t] = out;
        s_prod *= out >= 0 ? s_probs[out] : NAN;
      }
      __syncthreads();
    }
    if (tid == 0 && !(frechet && a.decode == RB200_SEQ2SLATE_DECODE_GREEDY)) {
      const float pr = fmaxf(s_prod, kProbFloor);  // per_symbol_to_per_seq_probs
      if (forced) {
        if (a.seq_log_prob) a.seq_log_prob[b] = logf(pr);
      } else {
        a.seq_prob[b] = pr;
      }
    }
    __syncthreads();
  }
}

int s2s_check(int32_t S, int32_t C, int32_t se, int32_t d, int32_t H, int32_t F, int32_t L,
              int32_t N, int32_t T, const char* who) {
  if (S < 1 || S > RB200_SEQ2SLATE_MAX_INPUT || C < 1 || C > RB200_SEQ2SLATE_MAX_INPUT ||
      d < 2 || d > RB200_SEQ2SLATE_MAX_DIM_MODEL || H < 1 || d % H != 0 || se < 1 || se >= d ||
      F < 1 || F > RB200_SEQ2SLATE_MAX_FEEDFORWARD || L < 1 || L > RB200_SEQ2SLATE_MAX_LAYERS ||
      N < 1 || N > RB200_SEQ2SLATE_MAX_CANDIDATES || T < 1 || T > N) {
    set_last_error("%s: need 1 <= state_dim, candidate_dim <= %d, 2 <= dim_model <= %d divisible "
                   "by num_heads, 1 <= state_embed_dim < dim_model, 1 <= dim_feedforward <= %d, "
                   "1 <= num_stacked_layers <= %d, 1 <= src_seq_len <= %d and 1 <= tgt_seq_len "
                   "<= src_seq_len (got state_dim %d, candidate_dim %d, state_embed_dim %d, "
                   "dim_model %d, num_heads %d, dim_feedforward %d, layers %d, src_seq_len %d, "
                   "tgt_seq_len %d)",
                   who, RB200_SEQ2SLATE_MAX_INPUT, RB200_SEQ2SLATE_MAX_DIM_MODEL,
                   RB200_SEQ2SLATE_MAX_FEEDFORWARD, RB200_SEQ2SLATE_MAX_LAYERS,
                   RB200_SEQ2SLATE_MAX_CANDIDATES, S, C, se, d, H, F, L, N, T);
    return RB200_E_INVALID;
  }
  return 0;
}

int s2s_validate(const rb200_seq2slate_args_t* a, const char* who) {
  if (!a) { set_last_error("%s: args is null", who); return RB200_E_INVALID; }
  if (int rc = s2s_check(a->state_dim, a->candidate_dim, a->state_embed_dim, a->dim_model,
                         a->num_heads, a->dim_feedforward, a->layers, a->src_len, a->tgt_len, who))
    return rc;
  if (a->batch < 1) { set_last_error("%s: batch %d < 1", who, a->batch); return RB200_E_INVALID; }
  if (a->arch != RB200_SEQ2SLATE_ARCH_AUTOREGRESSIVE && a->arch != RB200_SEQ2SLATE_ARCH_FRECHET_SORT) {
    set_last_error("%s: unknown arch %d", who, a->arch);
    return RB200_E_INVALID;
  }
  if (!a->params || !a->state || !a->src_seq ||
      (!a->workspace && rb200_seq2slate_workspace_bytes(a) > 0)) {
    set_last_error("%s: required pointer is null", who);
    return RB200_E_INVALID;
  }
  for (int i = 0; i < 30 * a->layers + 8; ++i)
    if (a->off[i] < 0 || a->off[i] >= a->n_params) {
      set_last_error("%s: parameter offset %d (%lld) outside the arena of %lld floats", who, i,
                     (long long)a->off[i], (long long)a->n_params);
      return RB200_E_INVALID;
    }
  const long long need = rb200_seq2slate_workspace_bytes(a);
  if (a->workspace_bytes < need) {
    set_last_error("%s: workspace of %lld bytes, need %lld", who, (long long)a->workspace_bytes,
                   need);
    return RB200_E_INVALID;
  }
  return 0;
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_seq2slate_check_shape(int32_t state_dim, int32_t candidate_dim,
                                           int32_t state_embed_dim, int32_t dim_model,
                                           int32_t num_heads, int32_t dim_feedforward,
                                           int32_t layers, int32_t max_src_seq_len,
                                           int32_t max_tgt_seq_len) {
  return s2s_check(state_dim, candidate_dim, state_embed_dim, dim_model, num_heads,
                   dim_feedforward, layers, max_src_seq_len, max_tgt_seq_len,
                   "rb200_seq2slate_check_shape");
}

// Bytes of one CTA's workspace slice; the slice lives in shared memory up to kS2sSmemMax.
static size_t s2s_slice_bytes(const rb200_seq2slate_args_t* a) {
  return (size_t)s2s_ws_floats(s2s_shape(*a)) * sizeof(float);
}

extern "C" int64_t rb200_seq2slate_workspace_bytes(const rb200_seq2slate_args_t* a) {
  if (!a || a->batch < 1 || s2s_slice_bytes(a) <= kS2sSmemMax) return 0;
  const int ctas = a->batch < kS2sMaxCtas ? a->batch : kS2sMaxCtas;
  return (int64_t)ctas * (int64_t)s2s_slice_bytes(a);
}

// CTAs of a launch: min(B, RB200_SEQ2SLATE_MAX_CTAS), and on the shared-memory path no more than
// fit on the device at once.  CTA c carries slates c, c + ctas, c + 2 ctas, ...
static int s2s_ctas(const rb200_seq2slate_args_t* a, int* ctas) {
  const size_t slice = s2s_slice_bytes(a);
  *ctas = a->batch < kS2sMaxCtas ? a->batch : kS2sMaxCtas;
  if (slice > kS2sSmemMax) return 0;
  if (cudaError_t e = opt_in_smem<seq2slate_kernel>(slice))
    return check_cuda(e, "seq2slate_kernel smem opt-in");
  int per_sm = 0, dev = 0, sms = 0;
  if (cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, seq2slate_kernel,
                                                                     kS2sThreads, slice))
    return check_cuda(e, "seq2slate_kernel occupancy");
  if (cudaError_t e = cudaGetDevice(&dev)) return check_cuda(e, "cudaGetDevice");
  if (cudaError_t e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev))
    return check_cuda(e, "cudaDeviceGetAttribute");
  const long long fit = (long long)(per_sm > 0 ? per_sm : 1) * sms;
  if (fit < *ctas) *ctas = (int)fit;
  return 0;
}

static int s2s_launch(const rb200_seq2slate_args_t* a, void* stream) {
  const size_t slice = s2s_slice_bytes(a);
  const bool smem = slice <= kS2sSmemMax;
  int ctas = 0;
  if (int rc = s2s_ctas(a, &ctas)) return rc;
  seq2slate_kernel<<<ctas, kS2sThreads, smem ? slice : 0, (cudaStream_t)stream>>>(*a, smem);
  return check_cuda(cudaGetLastError(), "seq2slate_kernel launch");
}

extern "C" int rb200_seq2slate_ctas(const rb200_seq2slate_args_t* a) {
  const char* who = "rb200_seq2slate_ctas";
  if (!a) { set_last_error("%s: args is null", who); return RB200_E_INVALID; }
  if (int rc = s2s_check(a->state_dim, a->candidate_dim, a->state_embed_dim, a->dim_model,
                         a->num_heads, a->dim_feedforward, a->layers, a->src_len, a->tgt_len, who))
    return rc;
  if (a->batch < 1) { set_last_error("%s: batch %d < 1", who, a->batch); return RB200_E_INVALID; }
  int ctas = 0;
  if (int rc = s2s_ctas(a, &ctas)) return rc;
  return ctas;
}

extern "C" int rb200_seq2slate_forward(const rb200_seq2slate_args_t* a, void* stream) {
  const char* who = "rb200_seq2slate_forward";
  if (int rc = s2s_validate(a, who)) return rc;
  if (a->decode != RB200_SEQ2SLATE_DECODE_FORCED || !a->tgt_in_idx || !a->tgt_out_idx ||
      (a->arch == RB200_SEQ2SLATE_ARCH_AUTOREGRESSIVE && !a->tgt_in_seq) ||
      (!a->probs && !a->log_probs && !a->seq_log_prob)) {
    set_last_error("%s: needs decode FORCED, tgt_in_idx, tgt_out_idx, tgt_in_seq "
                   "(AUTOREGRESSIVE) and at least one output", who);
    return RB200_E_INVALID;
  }
  return s2s_launch(a, stream);
}

extern "C" int rb200_seq2slate_rank(const rb200_seq2slate_args_t* a, void* stream) {
  const char* who = "rb200_seq2slate_rank";
  if (int rc = s2s_validate(a, who)) return rc;
  if ((a->decode != RB200_SEQ2SLATE_DECODE_GREEDY && a->decode != RB200_SEQ2SLATE_DECODE_SAMPLE) ||
      !a->ranked_idx || !a->seq_prob || (a->decode == RB200_SEQ2SLATE_DECODE_SAMPLE && !a->noise)) {
    set_last_error("%s: needs decode GREEDY or SAMPLE, ranked_idx, seq_prob and (SAMPLE) noise",
                   who);
    return RB200_E_INVALID;
  }
  return s2s_launch(a, stream);
}
