// reagent_b200 -- row-tile MLP primitives (tensor cores: mma.sync TF32 with 3xTF32 split).
//
// A CTA of NT (256 or 512) threads owns a tile of R = (NT/64)*TM batch rows and walks whole MLPs
// over it with every activation resident in shared memory; only weights stream
// through (cp.async, double buffered, out of L2 where all CTAs share them).
//
//   tile_linear_fwd : C[R,N]  = act(A[R,K] . W[N,K]^T + b)        (nn.Linear forward)
//   tile_linear_bwd : dA[R,K] = dZ[R,N] . W[N,K]                  (input gradient)
//
// The inner products run on the tensor cores (see "Tensor-core inner product" below).
#pragma once
#include "rb200_common.cuh"

namespace rb200 {

constexpr int kNC = 256;  // output-column chunk processed per pass

template <int KC>
__host__ __device__ constexpr int wstage_floats() {
  // one stage must hold either the fwd chunk [256][KC+4] or the bwd chunk [KC][256+8]
  return (kNC * (KC + 4) > KC * (kNC + 8)) ? kNC * (KC + 4) : KC * (kNC + 8);
}

// ---------------------------------------------------------------------------
// Tensor-core inner product: mma.sync.m16n8k8 TF32 with 3xTF32 error compensation
// (split_tf32 / mma_3xtf32, rb200_common.cuh), with far fewer issue slots than an FFMA loop.
// Fragment <-> shared-memory mapping (g = lane/4, t = lane%4), all LDS.32 conflict-free:
//   A (16x8, row-major tile of the activations, stride == 4 mod 32): a0 (g,t) a1 (g+8,t)
//                                                                   a2 (g,t+4) a3 (g+8,t+4)
//   B fwd (W chunk staged [n][KC+4], stride == 4 mod 32):  b0 = Ws[n0+g][k+t], b1 = Ws[n0+g][k+t+4]
//   B bwd (W chunk staged [n][256+8], stride == 8 mod 32): b0 = Ws[n+t][c0+g], b1 = Ws[n+t+4][c0+g]
//   C: c0 (g,2t) c1 (g,2t+1) c2 (g+8,2t) c3 (g+8,2t+1)
// A warp owns ALL row tiles (R/16) and the 8-column tiles  warp, warp+NW, ...  of the chunk, so
// narrow layers still spread over every warp.
// ---------------------------------------------------------------------------
constexpr int kLWB = kNC + 8;  // bwd staging row stride (== 8 mod 32)

// ---------------------------------------------------------------------------
// forward:  Cs[r, 0..N) = act(As[r, 0..K) . Wg[n, 0..K) + bg[n])
//   As : smem, row stride lda (== 4 mod 32), finite everywhere, 0 in columns K..round_up4(K)-1
//   Cs : smem, row stride ldc (multiple of 4); columns N..round_up4(N)-1 are zeroed
//   Wst: smem staging, 2 * wstage_floats<KC>() floats, 16B aligned; W chunk staged as
//        Ws[256][KC+4] (K contiguous), k >= K zero filled
// All NT threads must call (contains __syncthreads).
// ---------------------------------------------------------------------------
template <int NT, int TM, int KC, bool kRotate = true>
__device__ __noinline__ void tile_linear_fwd(const float* __restrict__ As, int lda, int K,
                                             const float* __restrict__ Wg, int ldw,
                                             const float* __restrict__ bg, int N, int act,
                                             float* __restrict__ Cs, int ldc,
                                             float* __restrict__ Wst) {
  constexpr int LW = KC + 4;
  constexpr int STAGE = wstage_floats<KC>();
  constexpr int QPR = KC / 4;  // 16B quads per staged row
  constexpr int NW = NT / 32;
  constexpr int R = (NT / 64) * TM;
  constexpr int MT = R / 16;          // 16-row MMA tiles
  constexpr int NTW = (kNC / 8) / NW; // 8-column tiles per warp at full chunk width
  static_assert(R % 16 == 0, "row tile must be a multiple of the MMA M");
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int nk = ceil_div(K, KC), nn = ceil_div(N, kNC), total = nk * nn;
  const bool vec = ((ldw & 3) == 0) && ((reinterpret_cast<uintptr_t>(Wg) & 15) == 0);
  // every CTA walks the k-chunks in a different rotation: all CTAs stream the SAME weights,
  // and in lock-step they would hammer the same L2 lines at the same time.  Without kRotate a
  // row's result does not depend on the CTA that computes it.
  const int rot = kRotate ? blockIdx.x % nk : 0;

  // staging map: thread -> (quad lq of the k-chunk, rows lr0, lr0+RPI, ...): fixed per thread
  constexpr int RPI = NT / QPR;
  const int lq = tid % QPR, lr0 = tid / QPR;
  auto load_chunk = [&](int c, int stage) {
    const int nci = c / nk, kci = c - nci * nk;
    const int n0 = nci * kNC, k0 = ((kci + rot) % nk) * KC;
    float* dst = Wst + stage * STAGE;
    const int rows = min(kNC, N - n0);
    const int k = k0 + 4 * lq;
    const bool fast = vec && (k + 3 < K);
#pragma unroll
    for (int it = 0; it < kNC / RPI; ++it) {
      const int row = lr0 + it * RPI;
      if (row < rows) {
        float* d = dst + row * LW + 4 * lq;
        const float* src = Wg + (size_t)(n0 + row) * ldw;
        if (fast) {
          cp_async16(d, src + k);
        } else {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (k < K) v.x = src[k];
          if (k + 1 < K) v.y = src[k + 1];
          if (k + 2 < K) v.z = src[k + 2];
          if (k + 3 < K) v.w = src[k + 3];
          *reinterpret_cast<float4*>(d) = v;
        }
      }
    }
  };

  float acc[MT][NTW][4];
  load_chunk(0, 0);
  cp_async_commit();
  for (int c = 0; c < total; ++c) {
    const int nci = c / nk, kci = c - nci * nk;
    const int n0 = nci * kNC, k0 = ((kci + rot) % nk) * KC;
    const int ncols = min(kNC, N - n0);
    const int ntiles = ceil_div(ncols, 8);
    if (kci == 0) {
#pragma unroll
      for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int j = 0; j < NTW; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[m][j][e] = 0.f;
    }
    if (c + 1 < total) {
      load_chunk(c + 1, (c + 1) & 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* Ws = Wst + (c & 1) * STAGE;
    if (warp < ntiles) {
      const int klen = min(KC, (K - k0 + 7) & ~7);
      const float* ab = As + g * lda + k0 + t;
      for (int kk = 0; kk < klen; kk += 8) {
        uint32_t ah[MT][4], al[MT][4];
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          const float* ap = ab + m * 16 * lda + kk;
          split_tf32(ap[0], ah[m][0], al[m][0]);
          split_tf32(ap[8 * lda], ah[m][1], al[m][1]);
          split_tf32(ap[4], ah[m][2], al[m][2]);
          split_tf32(ap[8 * lda + 4], ah[m][3], al[m][3]);
        }
#pragma unroll
        for (int j = 0; j < NTW; ++j) {
          const int nt = warp + j * NW;
          if (nt < ntiles) {
            const float* bp = Ws + (nt * 8 + g) * LW + kk + t;
            uint32_t bh[2], bl[2];
            split_tf32(bp[0], bh[0], bl[0]);
            split_tf32(bp[4], bh[1], bl[1]);
#pragma unroll
            for (int m = 0; m < MT; ++m) mma_3xtf32(acc[m][j], ah[m], al[m], bh, bl);
          }
        }
      }
    }
    if (kci == nk - 1) {
      const int n4 = round_up4(N);
#pragma unroll
      for (int j = 0; j < NTW; ++j) {
        const int nt = warp + j * NW;
        if (nt < ntiles) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = n0 + nt * 8 + 2 * t + e;
            if (col < n4) {
              const bool real = col < N;
              const float b = (real && bg != nullptr) ? bg[col] : 0.f;
#pragma unroll
              for (int m = 0; m < MT; ++m) {
                Cs[(m * 16 + g) * ldc + col] = real ? act_fwd(acc[m][j][e] + b, act) : 0.f;
                Cs[(m * 16 + g + 8) * ldc + col] = real ? act_fwd(acc[m][j][2 + e] + b, act) : 0.f;
              }
            }
          }
        }
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// backward (input gradient):  dAs[r, 0..Kout) = dZs[r, 0..N) . Wg[n, kcol0 .. kcol0+Kout)
//   then, if Hs != nullptr, multiplied elementwise by act'(Hs[r,k]) (Hs = the
//   activation OUTPUT that produced this input, same column indexing as dAs).
//   dZs: smem, stride ldz (== 4 mod 32), finite everywhere, 0 in columns N..round_up4(N)-1.
//   dAs: smem, stride lda; columns Kout..round_up4(Kout)-1 are zeroed.
//   Wg points at W[0][kcol0]; ldw is the full row stride of W.  W chunk staged as
//   Ws[KC][256+8] (rows = contraction index n, zero filled for n >= N).
// ---------------------------------------------------------------------------
template <int NT, int TM, int KC>
__device__ __noinline__ void tile_linear_bwd(const float* __restrict__ dZs, int ldz, int N,
                                             const float* __restrict__ Wg, int ldw, int Kout,
                                             const float* __restrict__ Hs, int ldh, int hact,
                                             float* __restrict__ dAs, int lda,
                                             float* __restrict__ Wst) {
  constexpr int LW = kLWB;
  constexpr int STAGE = wstage_floats<KC>();
  constexpr int NR = KC;  // contraction rows per staged chunk
  constexpr int NW = NT / 32;
  constexpr int R = (NT / 64) * TM;
  constexpr int MT = R / 16;
  constexpr int NTW = (kNC / 8) / NW;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int nnc = ceil_div(N, NR), nkc = ceil_div(Kout, kNC), total = nnc * nkc;
  const bool vec = ((ldw & 3) == 0) && ((reinterpret_cast<uintptr_t>(Wg) & 15) == 0);
  const int rot = blockIdx.x % nnc;

  // staging map: thread -> (quad lq of the 256-wide row, rows lr0, lr0+RPI, ...)
  constexpr int QPRB = kNC / 4;
  constexpr int RPI = NT / QPRB;
  const int lq = tid % QPRB, lr0 = tid / QPRB;
  auto load_chunk = [&](int c, int stage) {
    const int kci = c / nnc, nci = c - kci * nnc;
    const int k0 = kci * kNC, n0 = ((nci + rot) % nnc) * NR;
    float* dst = Wst + stage * STAGE;
    const int k = k0 + 4 * lq;
    if (k < ((Kout - k0 + 7) & ~7) + k0) {
      const bool fast = vec && (k + 3 < Kout);
#pragma unroll
      for (int it = 0; it < (NR + RPI - 1) / RPI; ++it) {
        const int row = lr0 + it * RPI;
        if (row < NR) {
          const int n = n0 + row;
          float* d = dst + row * LW + 4 * lq;
          if (n < N && fast) {
            cp_async16(d, Wg + (size_t)n * ldw + k);
          } else {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (n < N) {
              const float* src = Wg + (size_t)n * ldw;
              if (k < Kout) v.x = src[k];
              if (k + 1 < Kout) v.y = src[k + 1];
              if (k + 2 < Kout) v.z = src[k + 2];
              if (k + 3 < Kout) v.w = src[k + 3];
            }
            *reinterpret_cast<float4*>(d) = v;
          }
        }
      }
    }
  };

  float acc[MT][NTW][4];
  load_chunk(0, 0);
  cp_async_commit();
  for (int c = 0; c < total; ++c) {
    const int kci = c / nnc, nci = c - kci * nnc;
    const int k0 = kci * kNC, n0 = ((nci + rot) % nnc) * NR;
    const int kcols = min(kNC, Kout - k0);
    const int ntiles = ceil_div(kcols, 8);
    if (nci == 0) {
#pragma unroll
      for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int j = 0; j < NTW; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[m][j][e] = 0.f;
    }
    if (c + 1 < total) {
      load_chunk(c + 1, (c + 1) & 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* Ws = Wst + (c & 1) * STAGE;
    if (warp < ntiles) {
      const int nlen = min(NR, (N - n0 + 7) & ~7);
      const float* zb = dZs + g * ldz + n0 + t;
      for (int nn = 0; nn < nlen; nn += 8) {
        uint32_t ah[MT][4], al[MT][4];
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          const float* zp = zb + m * 16 * ldz + nn;
          split_tf32(zp[0], ah[m][0], al[m][0]);
          split_tf32(zp[8 * ldz], ah[m][1], al[m][1]);
          split_tf32(zp[4], ah[m][2], al[m][2]);
          split_tf32(zp[8 * ldz + 4], ah[m][3], al[m][3]);
        }
#pragma unroll
        for (int j = 0; j < NTW; ++j) {
          const int nt = warp + j * NW;
          if (nt < ntiles) {
            const float* bp = Ws + (nn + t) * LW + nt * 8 + g;
            uint32_t bh[2], bl[2];
            split_tf32(bp[0], bh[0], bl[0]);
            split_tf32(bp[4 * LW], bh[1], bl[1]);
#pragma unroll
            for (int m = 0; m < MT; ++m) mma_3xtf32(acc[m][j], ah[m], al[m], bh, bl);
          }
        }
      }
    }
    if (nci == nnc - 1) {
      const int k4 = round_up4(Kout);
#pragma unroll
      for (int j = 0; j < NTW; ++j) {
        const int nt = warp + j * NW;
        if (nt < ntiles) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int k = k0 + nt * 8 + 2 * t + e;
            if (k < k4) {
#pragma unroll
              for (int m = 0; m < MT; ++m) {
#pragma unroll
                for (int hrow = 0; hrow < 2; ++hrow) {
                  const int r = m * 16 + g + 8 * hrow;
                  float gv = 0.f;
                  if (k < Kout) {
                    gv = acc[m][j][2 * hrow + e];
                    if (Hs != nullptr) gv *= act_bwd_from_out(Hs[r * ldh + k], hact);
                  }
                  dAs[r * lda + k] = gv;
                }
              }
            }
          }
        }
      }
    }
    __syncthreads();
  }
}

// zero a shared-memory region (all NT threads): activations tiles must be finite everywhere
// because the MMA consumes their padding columns against zero-filled weights.
template <int NT>
__device__ __forceinline__ void tile_smem_zero_all(float* smem) {
  unsigned nbytes;
  asm("mov.u32 %0, %%dynamic_smem_size;" : "=r"(nbytes));
  const int nfloats = (int)(nbytes / 4);
  for (int i = threadIdx.x * 4; i + 3 < nfloats; i += NT * 4)
    *reinterpret_cast<float4*>(smem + i) = make_float4(0.f, 0.f, 0.f, 0.f);
  if (threadIdx.x < (nfloats & 3)) smem[(nfloats & ~3) + threadIdx.x] = 0.f;
  __syncthreads();
}

// ---------------------------------------------------------------------------
// cooperative tile <-> global copies (all NT threads)
// ---------------------------------------------------------------------------
// smem[r, 0..round_up4(D)) <- g[(row0+r), 0..D), zero padded; rows >= nrows zeroed.
template <int NT, int R>
__device__ void tile_load_rows(float* __restrict__ s, int lds, const float* __restrict__ g,
                               int ldg, int D, int row0, int nrows) {
  const int d4 = round_up4(D) / 4;
  const bool vec = ((ldg & 3) == 0) && ((reinterpret_cast<uintptr_t>(g) & 15) == 0);
  for (int idx = threadIdx.x; idx < R * d4; idx += NT) {
    const int r = idx / d4, q = idx - r * d4;
    const int c = 4 * q;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + r < nrows) {
      const float* src = g + (size_t)(row0 + r) * ldg;
      if (vec && c + 3 < D) {
        v = *reinterpret_cast<const float4*>(src + c);
      } else {
        if (c < D) v.x = src[c];
        if (c + 1 < D) v.y = src[c + 1];
        if (c + 2 < D) v.z = src[c + 2];
        if (c + 3 < D) v.w = src[c + 3];
      }
    }
    *reinterpret_cast<float4*>(s + r * lds + c) = v;
  }
}

// g[(row0+r), 0..D) <- smem[r, 0..D) for rows < nrows
template <int NT, int R>
__device__ void tile_store_rows(const float* __restrict__ s, int lds, float* __restrict__ g,
                                int ldg, int D, int row0, int nrows) {
  const int d4 = round_up4(D) / 4;
  const bool vec = ((ldg & 3) == 0) && ((reinterpret_cast<uintptr_t>(g) & 15) == 0);
  for (int idx = threadIdx.x; idx < R * d4; idx += NT) {
    const int r = idx / d4, q = idx - r * d4;
    const int c = 4 * q;
    if (row0 + r >= nrows) continue;
    const float4 v = *reinterpret_cast<const float4*>(s + r * lds + c);
    float* dst = g + (size_t)(row0 + r) * ldg;
    if (vec && c + 3 < D) {
      *reinterpret_cast<float4*>(dst + c) = v;
    } else {
      if (c < D) dst[c] = v.x;
      if (c + 1 < D) dst[c + 1] = v.y;
      if (c + 2 < D) dst[c + 2] = v.z;
      if (c + 3 < D) dst[c + 3] = v.w;
    }
  }
}

// ---------------------------------------------------------------------------
// Whole-MLP forward over the tile.  Input in `in` (stride ld_in).  Hidden
// activations ping-pong between hA and hB (stride ldh each); the final layer's
// output lands in `out` (stride ld_out).  If save != nullptr, save[l] (global,
// [B, dims[l+1]] dense) receives layer l's output for l < n_layers-1 (hidden
// only) -- the activations the weight-gradient kernel and the backward need.
// ---------------------------------------------------------------------------
template <int NT, int TM, int KC>
__device__ void tile_mlp_fwd(const Mlp& net, const float* in, int ld_in, float* hA, float* hB,
                             int ldh, float* out, int ld_out, float* Wst,
                             float* const* save, int row0, int nrows) {
  constexpr int R = (NT / 64) * TM;
  const float* cur = in;
  int ldc = ld_in;
  for (int l = 0; l < net.n_layers; ++l) {
    const bool last = (l == net.n_layers - 1);
    float* dst = last ? out : ((l & 1) ? hB : hA);
    const int ldd = last ? ld_out : ldh;
    tile_linear_fwd<NT, TM, KC>(cur, ldc, net.dims[l], net.params + net.w_off[l], net.dims[l],
                            net.params + net.b_off[l], net.dims[l + 1], net.act[l], dst, ldd,
                            Wst);
    if (!last && save != nullptr && save[l] != nullptr)
      tile_store_rows<NT, R>(dst, ldd, save[l], net.dims[l + 1], net.dims[l + 1], row0, nrows);
    cur = dst;
    ldc = ldd;
  }
}

// ---------------------------------------------------------------------------
// Whole-MLP backward (dZ chain) over the tile.
//   dz_last: smem [R, round_up4(dims[L])] = dLoss/d(pre-activation of last layer)
//   hidden[l] (global, dense [B, dims[l+1]]): saved outputs of layer l (l < L-1)
//   dz_out[l] (global, dense [B, dims[l+1]]): receives dLoss/d(pre-act of layer l)
//   On return, if din != nullptr it holds dLoss/d(input columns [in_col0, in_col0+in_cols))
//   in smem (stride ld_din).
// Buffers gA/gB (stride ldg) ping-pong the hidden dZ tiles; hbuf (stride ldg) is
// scratch for re-loading saved activations.
// ---------------------------------------------------------------------------
template <int NT, int TM, int KC>
__device__ void tile_mlp_bwd(const Mlp& net, float* dz_last, int ld_last, float* gA, float* gB,
                             float* hbuf, int ldg, float* Wst, const float* const* hidden,
                             float* const* dz_out, int row0, int nrows, float* din, int ld_din,
                             int in_col0, int in_cols) {
  constexpr int R = (NT / 64) * TM;
  const int L = net.n_layers;
  float* cur = dz_last;
  int ldc = ld_last;
  if (dz_out != nullptr && dz_out[L - 1] != nullptr)
    tile_store_rows<NT, R>(cur, ldc, dz_out[L - 1], net.dims[L], net.dims[L], row0, nrows);
  for (int l = L - 1; l >= 1; --l) {
    // dZ_{l-1} = (dZ_l . W_l) * act'_{l-1}(H_{l-1})
    tile_load_rows<NT, R>(hbuf, ldg, hidden[l - 1], net.dims[l], net.dims[l], row0, nrows);
    __syncthreads();
    float* dst = (l & 1) ? gA : gB;
    tile_linear_bwd<NT, TM, KC>(cur, ldc, net.dims[l + 1], net.params + net.w_off[l], net.dims[l],
                            net.dims[l], hbuf, ldg, net.act[l - 1], dst, ldg, Wst);
    if (dz_out != nullptr && dz_out[l - 1] != nullptr)
      tile_store_rows<NT, R>(dst, ldg, dz_out[l - 1], net.dims[l], net.dims[l], row0, nrows);
    cur = dst;
    ldc = ldg;
  }
  if (din != nullptr) {
    tile_linear_bwd<NT, TM, KC>(cur, ldc, net.dims[1], net.params + net.w_off[0] + in_col0,
                            net.dims[0], in_cols, nullptr, 0, 0, din, ld_din, Wst);
  }
}

}  // namespace rb200
