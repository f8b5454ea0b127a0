// reagent_b200 -- weight-gradient, gradient-reduce, fused Adam + soft-update kernels (K3).
#include <math.h>

#include "rb200_dqn_tc_layout.cuh"
#include "rb200_wgrad.cuh"

namespace rb200 {

// ---------------------------------------------------------------------------
// dW_l[n,k] = sum_b dZ_l[b,n] * A_{l-1}[b,k];  db_l[n] = sum_b dZ_l[b,n]
// One CTA = one 64(n) x 64(k) tile of one layer over one batch split; 8 warps, each a
// 32(n) x 16(k) block = 2x2 mma.sync.m16n8k8 tiles, contraction over 8 batch rows per step,
// 3xTF32 error compensation like the row-tile kernels.  Operands are staged [batch][64+8]
// (stride == 8 mod 32): the A fragment (dZ^T: row n, col b) and the B fragment (row b, col k)
// are conflict-free LDS.32.  Deterministic: split s of the batch sum goes to its own slab.
// ---------------------------------------------------------------------------
constexpr int kWgTile = 64;
constexpr int kWgRows = 32;  // batch rows staged per step
constexpr int kWgLd = kWgTile + 8;

// (WgradLayer: rb200_wgrad.cuh)  kJobs is the capacity of the job list passed by value.
template <int kJobs>
struct WgradParamsN {
  int n_layers;
  WgradLayer L[kJobs];
  int B, splits, rows_per_split;
  float* gpart;
  long long P;
};
using WgradParams = WgradParamsN<kMaxLayers>;

template <int kJobs>
__global__ void __launch_bounds__(kThreads) wgrad_kernel(const WgradParamsN<kJobs> p) {
  __shared__ __align__(16) float zs[2][kWgRows][kWgLd];
  __shared__ __align__(16) float as[2][kWgRows][kWgLd];
  int li = 0;
  while (li + 1 < p.n_layers && (int)blockIdx.x >= p.L[li + 1].tile_start) ++li;
  const WgradLayer& Ly = p.L[li];
  const int tl = blockIdx.x - Ly.tile_start;
  const int tn = tl / Ly.tiles_k, tk = tl - tn * Ly.tiles_k;
  const int n0 = tn * kWgTile, k0 = tk * kWgTile;
  const int split = blockIdx.y;
  const int b_begin = split * p.rows_per_split;
  const int b_end = min(p.B, b_begin + p.rows_per_split);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int wn = (warp >> 2) * 32;  // warp block origin inside the 64x64 tile
  const int wk = (warp & 3) * 16;
  const int N = Ly.N, K = Ly.K;
  const bool vz = ((N & 3) == 0) && ((reinterpret_cast<uintptr_t>(Ly.dZ) & 15) == 0);
  const bool va = ((K & 3) == 0) && ((reinterpret_cast<uintptr_t>(Ly.A) & 15) == 0);

  float acc[2][2][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
  float bsum = 0.f;  // thread tid < 64: column sum of dZ for n0 + tid (bias gradient)

  auto stage = [&](int b0, int buf) {
    for (int idx = tid; idx < kWgRows * 16; idx += kThreads) {
      const int r = idx >> 4, qd = idx & 15;
      const int b = b0 + r;
      {
        const int n = n0 + 4 * qd;
        float* d = &zs[buf][r][4 * qd];
        if (b < b_end && vz && n + 3 < N) {
          cp_async16(d, Ly.dZ + (size_t)b * N + n);
        } else {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (b < b_end) {
            const float* s = Ly.dZ + (size_t)b * N;
            if (n < N) v.x = s[n];
            if (n + 1 < N) v.y = s[n + 1];
            if (n + 2 < N) v.z = s[n + 2];
            if (n + 3 < N) v.w = s[n + 3];
          }
          *reinterpret_cast<float4*>(d) = v;
        }
      }
      {
        const int k = k0 + 4 * qd;
        float* d = &as[buf][r][4 * qd];
        if (b < b_end && va && k + 3 < K) {
          cp_async16(d, Ly.A + (size_t)b * K + k);
        } else {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (b < b_end) {
            const float* s = Ly.A + (size_t)b * K;
            if (k < K) v.x = s[k];
            if (k + 1 < K) v.y = s[k + 1];
            if (k + 2 < K) v.z = s[k + 2];
            if (k + 3 < K) v.w = s[k + 3];
          }
          *reinterpret_cast<float4*>(d) = v;
        }
      }
    }
  };

  const int nsteps = ceil_div(max(b_end - b_begin, 0), kWgRows);
  if (nsteps > 0) {
    stage(b_begin, 0);
    cp_async_commit();
  }
  for (int s = 0; s < nsteps; ++s) {
    if (s + 1 < nsteps) {
      stage(b_begin + (s + 1) * kWgRows, (s + 1) & 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int buf = s & 1;
#pragma unroll
    for (int bb = 0; bb < kWgRows; bb += 8) {
      // A = dZ^T block: element (row n, col b) = zs[b][n]
      uint32_t ah[2][4], al[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int n = wn + 16 * i + g;
        split_tf32(zs[buf][bb + t][n], ah[i][0], al[i][0]);
        split_tf32(zs[buf][bb + t][n + 8], ah[i][1], al[i][1]);
        split_tf32(zs[buf][bb + t + 4][n], ah[i][2], al[i][2]);
        split_tf32(zs[buf][bb + t + 4][n + 8], ah[i][3], al[i][3]);
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int k = wk + 8 * j + g;
        uint32_t bh[2], bl[2];
        split_tf32(as[buf][bb + t][k], bh[0], bl[0]);
        split_tf32(as[buf][bb + t + 4][k], bh[1], bl[1]);
#pragma unroll
        for (int i = 0; i < 2; ++i) mma_3xtf32(acc[i][j], ah[i], al[i], bh, bl);
      }
    }
    if (tk == 0 && tid < kWgTile) {
#pragma unroll 8
      for (int r = 0; r < kWgRows; ++r) bsum += zs[buf][r][tid];
    }
    __syncthreads();
  }

  float* gp = p.gpart + (size_t)split * p.P;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int n = n0 + wn + 16 * i + g + ((e >> 1) ? 8 : 0);
        const int k = k0 + wk + 8 * j + 2 * t + (e & 1);
        if (n < N && k < K) gp[Ly.w_off + (size_t)n * K + k] = acc[i][j][e];
      }
  if (tk == 0 && tid < kWgTile && n0 + tid < N) gp[Ly.b_off + n0 + tid] = bsum;
}

int wgrad_jobs_launch(WgradLayer* jobs, int n_jobs, int rows, int splits, float* gpart,
                      long long P, cudaStream_t st, const char* what) {
  if (n_jobs < 1 || n_jobs > kWgradMaxJobs || rows <= 0 || splits <= 0) {
    set_last_error("%s: bad job count %d, rows %d or splits %d", what, n_jobs, rows, splits);
    return RB200_E_INVALID;
  }
  WgradParamsN<kWgradMaxJobs> p = {};
  p.n_layers = n_jobs;
  p.B = rows;
  p.splits = splits;
  p.rows_per_split = ceil_div(ceil_div(rows, splits), kWgRows) * kWgRows;
  p.gpart = gpart;
  p.P = P;
  int tiles = 0;
  for (int j = 0; j < n_jobs; ++j) {
    WgradLayer& L = jobs[j];
    L.tiles_n = ceil_div(L.N, kWgTile);
    L.tiles_k = ceil_div(L.K, kWgTile);
    L.tile_start = tiles;
    tiles += L.tiles_n * L.tiles_k;
    p.L[j] = L;
  }
  for (int j = n_jobs; j < kWgradMaxJobs; ++j) p.L[j].tile_start = 1 << 30;
  return launch<wgrad_kernel<kWgradMaxJobs>>(dim3(tiles, splits), kThreads, 0, st, what, p);
}

// g[i] = sum_s gpart[s*P + i]
__global__ void grad_reduce_kernel(const float* __restrict__ gpart, int splits, long long n,
                                   float* __restrict__ g) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    float s = gpart[i];
    for (int k = 1; k < splits; ++k) s += gpart[(size_t)k * n + i];
    g[i] = s;
  }
}

// ---------------------------------------------------------------------------
// Fused Adam (+ Polyak).  Mirrors torch.optim.Adam's single-tensor path
// (non-amsgrad, non-capturable):
//   g   = sum_s grad[s] * grad_scale (+ wd * p)
//   m   = lerp(m, g, 1-b1);  v = v*b2 + (1-b2)*g*g
//   (the weight decay term and the lerp are fused multiply-adds, like ATen's)
//   bc1 = 1 - b1^t, bc2 = 1 - b2^t (double), step_size = lr/bc1
//   p  -= step_size * m / (sqrt(v)/sqrt(bc2) + eps)
// then target = tau*p + (1-tau)*target  (SoftUpdate.step on the updated source).
// kDecoupled (AdamW): no wd term in g; instead p *= float(1 - lr*wd) (double, like Python)
// before the moment updates.  kAmsgrad: vmax = maximum(vmax, v) with NaN propagating like
// torch.maximum, and the denominator uses vmax.  Adam is <false, false>: no per-element work
// is added to it.
// ---------------------------------------------------------------------------
struct AdamDev {
  rb200_adam_args_t a;
  TcPackView pv;
};

// images of one updated weight (and of its updated target) for the wgmma TD kernel
__device__ __forceinline__ void adam_pack_weight(const TcPackView& pv, long long i, float p,
                                                 bool has_target, float tgt) {
  for (int l = 0; l < pv.n_layers; ++l) {
    const int N = pv.dims[l + 1], K = pv.dims[l];
    const long long rel = i - pv.w_off[l];
    if (rel < 0 || rel >= (long long)N * K) continue;
    const int m = (int)(rel / K), k = (int)(rel - (long long)m * K);
    const uint32_t pos = image_elem(N, K, m, k);
    pv.pack[pv.on_fwd[l] / 4 + pos] = p;
    if (has_target) pv.pack[pv.tg_fwd[l] / 4 + pos] = tgt;
    // transposed operand of the backward: rows = K_l features, contraction = N_l
    if (pv.has_bwd && l >= 1) pv.pack[pv.on_bwd[l] / 4 + image_elem(K, N, k, m)] = p;
    return;
  }
}

// maximum that returns NaN when either input is NaN (fmaxf returns the other input)
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

template <bool kDecoupled, bool kAmsgrad>
__global__ void __launch_bounds__(256) adam_soft_kernel(const AdamDev d) {
  const rb200_adam_args_t& a = d.a;
  // bias corrections in double like torch (Python floats), once per block
  __shared__ long long s_t;
  __shared__ float s_step_size, s_bc2_sqrt;
  if (threadIdx.x == 0) {
    const long long tt = *a.step + 1;
    const double bc1 = 1.0 - pow(a.beta1, (double)tt);
    const double bc2 = 1.0 - pow(a.beta2, (double)tt);
    s_t = tt;
    s_step_size = (float)(a.lr / bc1);
    s_bc2_sqrt = (float)sqrt(bc2);
  }
  __syncthreads();
  const long long t = s_t;
  const float step_size = s_step_size;
  const float bc2_sqrt = s_bc2_sqrt;
  const float eps = (float)a.eps;
  const float w1 = (float)(1.0 - a.beta1);
  const bool w1_small = fabsf(w1) < 0.5f;
  const float w1m1 = w1 - 1.f;
  const float b2 = (float)a.beta2;
  const float w2 = (float)(1.0 - a.beta2);
  const float wd = (float)a.weight_decay;
  const float decay = kDecoupled ? (float)(1.0 - a.lr * a.weight_decay) : 1.f;
  const long long n = a.n;
  const long long stride = (long long)gridDim.x * blockDim.x;
  // split-K partials: loads issued 8 at a time, summed in slab order (deterministic)
  auto local_grad = [&](long long i) {
    float g = 0.f;
    for (int s0 = 0; s0 < a.splits; s0 += 8) {
      float part[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        part[u] = (s0 + u < a.splits) ? a.grad[(size_t)(s0 + u) * n + i] : 0.f;
#pragma unroll
      for (int u = 0; u < 8; ++u)
        if (s0 + u < a.splits) g = (s0 + u == 0) ? part[u] : g + part[u];
    }
    return g;
  };
  const int W = a.dp_world;
  const float* dp_mine = nullptr;
  if (W > 1) {
    // ---- fused gradient exchange over NVLink peer memory (see rb200_adam_args_t) ----
    const unsigned par = (unsigned)(t & 1);
    const size_t slot = ((size_t)par * W + a.dp_rank) * (size_t)a.dp_stride;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
      const float g = local_grad(i);
      for (int r = 0; r < W; ++r) a.dp_recv[r][slot + i] = g;  // own copy included
    }
    __syncthreads();
    const size_t fslot = ((size_t)par * W) * a.dp_max_blocks + blockIdx.x;
    if (threadIdx.x == 0) {
      // ONE system-scope fence orders every push of this block (made visible to this thread by
      // the barrier) before the flags; the W-1 flag stores themselves are then relaxed and
      // posted back to back (a release store per peer would pay the fence W-1 times)
      __threadfence_system();
      for (int r = 0; r < W; ++r) {
        if (r == a.dp_rank) continue;
        uint32_t* f = a.dp_flags[r] + fslot + (size_t)a.dp_rank * a.dp_max_blocks;
        asm volatile("st.relaxed.sys.global.u32 [%0], %1;\n" ::"l"(f), "r"((uint32_t)t) : "memory");
      }
    }
    if ((int)threadIdx.x < W && (int)threadIdx.x != a.dp_rank) {
      // wait for that peer's push of the same slice (it never waits before pushing)
      const uint32_t* w = a.dp_flags[a.dp_rank] + fslot + (size_t)threadIdx.x * a.dp_max_blocks;
      unsigned long long t0 = 0, now = 0;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      for (;;) {
        uint32_t v;
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];\n" : "=r"(v) : "l"(w) : "memory");
        if (v == (uint32_t)t) break;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        if (now - t0 > 4000000000ull) __trap();  // 4 s: a lost peer fails the step, never hangs
      }
    }
    __syncthreads();
    dp_mine = a.dp_recv[a.dp_rank] + (size_t)par * W * (size_t)a.dp_stride;
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    float g;
    if (W > 1) {
      g = __ldcg(dp_mine + i);
      for (int r = 1; r < W; ++r) g += __ldcg(dp_mine + (size_t)r * a.dp_stride + i);
    } else {
      g = local_grad(i);
    }
    g *= a.grad_scale;
    float p = a.params[i];
    if (kDecoupled) {
      if (wd != 0.f) p = __fmul_rn(p, decay);
    } else if (wd != 0.f) {
      g = fmaf(wd, p, g);
    }
    float m = a.exp_avg[i];
    float v = a.exp_avg_sq[i];
    // rounding mirrors ATen's CPU kernels:
    //   lerp:    fma(w, g-m, m) for |w| < 0.5, else fma(w-1, g-m, g)  (at::lerp's two branches)
    //   addcmul: self + (value*t1)*t2 with every product and the sum rounded separately.  ATen's
    //            AVX2 / AVX-512 builds contract the last multiply-add into an fma; the two differ
    //            by at most 1 ulp of exp_avg_sq per step, and this form is kept so that training
    //            runs reproduce the library's earlier results exactly.
    //   addcdiv: self + (value*t1)/t2, each product / quotient rounded separately
    const float gm = __fsub_rn(g, m);
    m = w1_small ? fmaf(w1, gm, m) : fmaf(w1m1, gm, g);
    v = __fadd_rn(__fmul_rn(v, b2), __fmul_rn(__fmul_rn(w2, g), g));
    float vd = v;
    if (kAmsgrad) {
      vd = fmax_nan(a.max_exp_avg_sq[i], v);
      a.max_exp_avg_sq[i] = vd;
    }
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vd), bc2_sqrt), eps);
    p = __fadd_rn(p, __fdiv_rn(__fmul_rn(-step_size, m), denom));
    a.params[i] = p;
    a.exp_avg[i] = m;
    a.exp_avg_sq[i] = v;
    if (a.exp_out) a.exp_out[i] = expf(p);
    float tn = 0.f;
    if (a.target) {
      const float tg = a.target[i];
      tn = __fadd_rn(__fmul_rn(a.tau, p), __fmul_rn(a.one_minus_tau, tg));
      a.target[i] = tn;
    }
    if (d.pv.pack) adam_pack_weight(d.pv, i, p, a.target != nullptr, tn);
  }
  // last block to finish bumps the step counter (every block has read it by then)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned done = atomicAdd(a.block_counter, 1u);
    if (done == gridDim.x - 1) {
      *a.step = t;
      *a.block_counter = 0u;
    }
  }
}

__global__ void soft_update_kernel(float* __restrict__ target, const float* __restrict__ src,
                                   long long n, float tau, float omt) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    target[i] = __fadd_rn(__fmul_rn(tau, src[i]), __fmul_rn(omt, target[i]));
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_wgrad_splits(int batch) {
  // enough batch splits that even a single 64x64 tile layer fills a good part of the
  // SMs: 256 rows per split, a multiple of the 32-row staging step.
  int s = batch / 256;
  if (s < 1) s = 1;
  if (s > 64) s = 64;
  return s;
}

extern "C" int rb200_mlp_wgrad(const rb200_mlp_t* net, const float* net_input, int32_t batch,
                               const rb200_net_ws_t* ws, float* gpart, int32_t splits,
                               void* stream) {
  if (!net || !ws || !gpart) { set_last_error("rb200_mlp_wgrad: null argument"); return RB200_E_INVALID; }
  if (int rc = validate_mlp(net, "net")) return rc;
  if (batch <= 0 || splits <= 0) { set_last_error("rb200_mlp_wgrad: bad batch/splits"); return RB200_E_INVALID; }
  WgradParams p = {};
  p.n_layers = net->n_layers;
  p.B = batch;
  p.splits = splits;
  p.rows_per_split = ceil_div(ceil_div(batch, splits), kWgRows) * kWgRows;
  p.gpart = gpart;
  p.P = net->n_params;
  int tiles = 0;
  for (int l = 0; l < net->n_layers; ++l) {
    WgradLayer& L = p.L[l];
    L.A = (l == 0) ? (net_input ? net_input : ws->input) : ws->hidden[l - 1];
    L.dZ = ws->dz[l];
    if (!L.A || !L.dZ) { set_last_error("rb200_mlp_wgrad: missing activation / dz for layer %d", l); return RB200_E_INVALID; }
    L.K = net->dims[l];
    L.N = net->dims[l + 1];
    L.w_off = net->w_off[l];
    L.b_off = net->b_off[l];
    L.tiles_n = ceil_div(L.N, kWgTile);
    L.tiles_k = ceil_div(L.K, kWgTile);
    L.tile_start = tiles;
    tiles += L.tiles_n * L.tiles_k;
  }
  for (int l = net->n_layers; l < kMaxLayers; ++l) p.L[l].tile_start = 1 << 30;
  dim3 grid(tiles, splits);
  wgrad_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(p);
  return check_cuda(cudaGetLastError(), "wgrad_kernel launch");
}

extern "C" int rb200_grad_reduce(const float* gpart, int32_t splits, int64_t n, float* g,
                                 void* stream) {
  if (!gpart || !g || n <= 0 || splits <= 0) { set_last_error("rb200_grad_reduce: bad argument"); return RB200_E_INVALID; }
  int blocks = (int)((n + 255) / 256);
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  grad_reduce_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(gpart, splits, (long long)n, g);
  return check_cuda(cudaGetLastError(), "grad_reduce_kernel launch");
}

extern "C" int rb200_adam_soft_update(const rb200_adam_args_t* a, void* stream) {
  if (!a || !a->params || !a->grad || !a->exp_avg || !a->exp_avg_sq || !a->step || !a->block_counter) {
    set_last_error("rb200_adam_soft_update: null argument"); return RB200_E_INVALID;
  }
  if (a->n <= 0 || a->splits <= 0) { set_last_error("rb200_adam_soft_update: bad n/splits"); return RB200_E_INVALID; }
  if ((a->decoupled_weight_decay != 0 && a->decoupled_weight_decay != 1) ||
      (a->amsgrad != 0 && a->amsgrad != 1)) {
    set_last_error("rb200_adam_soft_update: decoupled_weight_decay and amsgrad must be 0 or 1"); return RB200_E_INVALID;
  }
  if (a->amsgrad && !a->max_exp_avg_sq) { set_last_error("rb200_adam_soft_update: amsgrad needs max_exp_avg_sq"); return RB200_E_INVALID; }
  AdamDev d;
  d.a = *a;
  d.a.tc_net = nullptr;  // host pointer: not for the device
  d.pv.pack = nullptr;
  if (a->tc_net && a->tc_pack_ws) {
    const rb200_mlp_t* q = a->tc_net;
    if (int rc = validate_mlp(q, "tc_net")) return rc;
    if (q->params != a->params || !a->target) { set_last_error("rb200_adam_soft_update: tc packing needs tc_net->params == params and a target"); return RB200_E_INVALID; }
    const TcImages im = tc_images(q, a->tc_do_backward);
    if (a->tc_pack_ws_bytes < im.total_bytes) { set_last_error("rb200_adam_soft_update: pack workspace too small"); return RB200_E_INVALID; }
    d.pv.n_layers = q->n_layers;
    for (int l = 0; l <= kMaxLayers; ++l) d.pv.dims[l] = im.dims[l];
    for (int l = 0; l < kMaxLayers; ++l) {
      d.pv.w_off[l] = l < q->n_layers ? q->w_off[l] : 0;
      d.pv.on_fwd[l] = im.on_fwd[l];
      d.pv.tg_fwd[l] = im.tg_fwd[l];
      d.pv.on_bwd[l] = im.on_bwd[l];
    }
    d.pv.has_bwd = im.has_bwd;
    d.pv.pack = static_cast<float*>(a->tc_pack_ws);
  }
  const int blocks = rb200_adam_blocks(a->n);
  if (a->dp_world > 1) {
    if (!a->dp_recv || !a->dp_flags || a->dp_rank < 0 || a->dp_rank >= a->dp_world ||
        a->dp_world > 256 || a->dp_stride < a->n || a->dp_max_blocks < blocks) {
      set_last_error("rb200_adam_soft_update: bad data-parallel exchange arguments"); return RB200_E_INVALID;
    }
  } else {
    d.a.dp_world = 1;
  }
  void (*kernel)(const AdamDev) =
      a->decoupled_weight_decay ? (a->amsgrad ? adam_soft_kernel<true, true> : adam_soft_kernel<true, false>)
                                : (a->amsgrad ? adam_soft_kernel<false, true> : adam_soft_kernel<false, false>);
  kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(d);
  return check_cuda(cudaGetLastError(), "adam_soft_kernel launch");
}

// grid of rb200_adam_soft_update for an arena of n floats (all blocks co-resident on the SMs)
extern "C" int rb200_adam_blocks(int64_t n) {
  int blocks = (int)((n + 255) / 256);
  if (blocks > kNumSMs * 4) blocks = kNumSMs * 4;
  return blocks < 1 ? 1 : blocks;
}

extern "C" int rb200_soft_update(float* target, const float* source, int64_t n, float tau,
                                 float one_minus_tau, void* stream) {
  if (!target || !source || n <= 0) { set_last_error("rb200_soft_update: bad argument"); return RB200_E_INVALID; }
  if (target == source) return RB200_OK;  // aliased: soft_update.py:64-67 skips
  int blocks = (int)((n + 255) / 256);
  if (blocks > kNumSMs * 4) blocks = kNumSMs * 4;
  soft_update_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(target, source, (long long)n, tau, one_minus_tau);
  return check_cuda(cudaGetLastError(), "soft_update_kernel launch");
}
