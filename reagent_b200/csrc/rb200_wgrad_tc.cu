// reagent_b200 -- weight gradients on the Hopper tensor cores.
//
//   dW_l[n, k] = sum_b dZ_l[b, n] * A_{l-1}[b, k],   db_l[n] = sum_b dZ_l[b, n]
// (autograd's Linear backward reached from loss.backward() in the reference's Lightning loop,
// reagent/training/reagent_lightning_module.py:108-133) as wgmma kind tf32 with 3xTF32 error
// compensation and the accumulators in registers.
//
// The contraction runs over the BATCH, and both factors are stored batch-row-major in HBM
// ([B, N] and [B, K]), i.e. transposed with respect to the K-major operand layout the MMA
// reads.  The kernel transposes while staging: a 32-row chunk of both matrices is loaded with
// 16-byte loads (a lane = one row x 4 features; 16 rows x 32 B per instruction: whole sectors),
// split into TF32 hi / lo in registers, and every scalar goes straight to its place in the
// canonical K-major no-swizzle layout
//     [batch row / 4][feature][4 batch rows]   (row-quad stride = LBO, 8 features = SBO = 128 B)
// with bank-conflict-free 4-byte stores (the padded row-quad stride spreads a warp's 32 stores
// over the 32 banks); every 8-row k step issues  D += A_hi.B_hi + A_lo.B_hi + A_hi.B_lo  with
// M = 64 output features of dZ_l per warpgroup (two warpgroups: 128) and N <= 256 input
// features of A_{l-1}.
//
// One CTA = (layer, 128-feature tile of dZ_l, 256-feature tile of A_{l-1}, batch slab); the
// slabs are summed later by the Adam kernel in slab order (deterministic), exactly like the
// mma.sync kernel this one replaces for shapes that fit (rb200_optim.cu keeps that kernel for
// the rest).  Two smem stages; the loads of chunk c+1 are in flight while chunk c's MMAs run.
#include "rb200_wgmma.cuh"

namespace rb200 {

constexpr int kWtRows = 32;                       // batch rows per stage = 4 MMA k steps
constexpr int kWtM = 128;                         // dZ features per tile (two m64 warpgroups)
constexpr int kWtN = 256;                         // input features per tile (wgmma N <= 256)
constexpr int kWtQuadA = kWtM * 16 + 16;          // bytes per 4-row group of the dZ operand
constexpr int kWtQuadB = kWtN * 16 + 16;          // ... of the activation operand
constexpr int kWtPlaneA = (kWtRows / 4) * kWtQuadA;
constexpr int kWtPlaneB = (kWtRows / 4) * kWtQuadB;
constexpr int kWtStage = 2 * (kWtPlaneA + kWtPlaneB);  // A_hi, A_lo, B_hi, B_lo
constexpr int kWtThreads = 256;
constexpr int kWtSmem = 2 * kWtStage + 64;

struct WtLayer {
  const float* A;   // [B, K]
  const float* dZ;  // [B, N]
  int K, N;
  long long w_off, b_off;
  int tiles_m, tiles_k, job_start;
};
struct WtParams {
  int n_layers;
  WtLayer L[kMaxLayers];
  int B, rows_per_split;
  float* gpart;
  long long P;
};

// the three MMAs of one k step at wgmma N = NT (the staged columns rounded up; columns past the
// matrix only reach accumulator columns that are not stored)
template <int NT>
__device__ __forceinline__ void wt_kstep(float* acc, uint64_t dah, uint64_t dal, uint64_t dbh,
                                         uint64_t dbl) {
  if constexpr (NT == 32) {
    wgmma_ss_n32(acc, dah, dbh, 1u); wgmma_ss_n32(acc, dal, dbh, 1u); wgmma_ss_n32(acc, dah, dbl, 1u);
  } else if constexpr (NT == 64) {
    wgmma_ss_n64(acc, dah, dbh, 1u); wgmma_ss_n64(acc, dal, dbh, 1u); wgmma_ss_n64(acc, dah, dbl, 1u);
  } else if constexpr (NT == 128) {
    wgmma_ss_n128(acc, dah, dbh, 1u); wgmma_ss_n128(acc, dal, dbh, 1u); wgmma_ss_n128(acc, dah, dbl, 1u);
  } else {
    wgmma_ss_n256(acc, dah, dbh, 1u); wgmma_ss_n256(acc, dal, dbh, 1u); wgmma_ss_n256(acc, dah, dbl, 1u);
  }
}

__global__ void __launch_bounds__(kWtThreads, 1) wgrad_tc_kernel(const WtParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;  // warpgroup: dZ features [64 wg, 64 wg + 64) of the tile
  int li = 0;
  while (li + 1 < p.n_layers && (int)blockIdx.x >= p.L[li + 1].job_start) ++li;
  const WtLayer& Ly = p.L[li];
  const int job = blockIdx.x - Ly.job_start;
  const int tm = job / Ly.tiles_k, tk = job - tm * Ly.tiles_k;
  const int n0 = tm * kWtM, k0 = tk * kWtN;
  const int N = Ly.N, K = Ly.K;
  const int nrows_m = min(kWtM, N - n0);             // valid dZ features of this tile
  const int ncols = min(kWtN, K - k0);               // valid input features of this tile
  const int n_mma = ncols <= 32 ? 32 : (ncols <= 64 ? 64 : (ncols <= 128 ? 128 : 256));
  const int split = blockIdx.y;
  const int b_begin = split * p.rows_per_split;
  const int b_end = min(p.B, b_begin + p.rows_per_split);
  const int nchunks = ceil_div(max(b_end - b_begin, 0), kWtRows);

  // No zero-fill of the stages: every staged feature row is rewritten per chunk (zeros past the
  // slab end); features past the matrix are never written, and whatever they hold only reaches
  // accumulator rows / columns that are not stored (D[m][n] depends on A row m and B row n only).

  // A chunk (32 batch rows) is moved in "units" of 16 rows x 8 features: lane = (row, 4-feature
  // piece) loads one float4 (16 rows x 32 B: whole sectors), splits it into TF32 hi / lo and
  // stores the 2 x 4 scalars transposed into the K-major planes -- element (row r, feature f)
  // at [r / 4][f][r % 4].  With the 16-byte padded row-quad stride the 32 stores of a warp hit
  // 32 different banks.  Units of a chunk: 2 halves x (feature pairs of A + of B), dealt to the
  // 8 warps round-robin; the loads of chunk c+1 are in flight while chunk c's MMAs run.
  const int fa = (nrows_m + 7) & ~7, fb = (ncols + 7) & ~7;  // staged features (multiples of 8)
  const int ua = 2 * (fa / 8), utotal = ua + 2 * (fb / 8);
  constexpr int kMaxUnits = (2 * (kWtM / 8) + 2 * (kWtN / 8)) / (kWtThreads / 32);  // 12
  const int r_l = lane & 15, qsel = lane >> 4;
  float4 regs[kMaxUnits];
  auto chunk_fetch = [&](int c) {
    const int r0 = b_begin + c * kWtRows;
#pragma unroll
    for (int u = 0; u < kMaxUnits; ++u) {
      const int unit = warp + u * (kWtThreads / 32);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (unit < utotal) {
        const bool isb = unit >= ua;
        const int j = isb ? unit - ua : unit;
        const int h = j & 1, fp = j >> 1;
        const int row = r0 + 16 * h + r_l;
        const int f = (isb ? k0 : n0) + 8 * fp + 4 * qsel;
        const int F = isb ? K : N;
        if (row < b_end && f < F) {
          const float* src = (isb ? Ly.A : Ly.dZ) + (size_t)row * F + f;
          if (f + 3 < F && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
            v = __ldg(reinterpret_cast<const float4*>(src));
          } else {
            v.x = src[0];
            if (f + 1 < F) v.y = src[1];
            if (f + 2 < F) v.z = src[2];
            if (f + 3 < F) v.w = src[3];
          }
        }
      }
      regs[u] = v;
    }
  };
  auto chunk_store = [&](int st) {
    unsigned char* base = smem + st * kWtStage;
#pragma unroll
    for (int u = 0; u < kMaxUnits; ++u) {
      const int unit = warp + u * (kWtThreads / 32);
      if (unit >= utotal) continue;
      const bool isb = unit >= ua;
      const int j = isb ? unit - ua : unit;
      const int h = j & 1, fp = j >> 1;
      const int r = 16 * h + r_l;
      const int fl = 8 * fp + 4 * qsel;
      float* hi = reinterpret_cast<float*>(base + (isb ? 2 * kWtPlaneA + (r >> 2) * kWtQuadB
                                                       : (r >> 2) * kWtQuadA) + fl * 16) + (r & 3);
      float* lo = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(hi) + (isb ? kWtPlaneB : kWtPlaneA));
      float4 hh, ll;
      split4(regs[u], hh, ll);
      hi[0] = hh.x; hi[4] = hh.y; hi[8] = hh.z; hi[12] = hh.w;
      lo[0] = ll.x; lo[4] = ll.y; lo[8] = ll.z; lo[12] = ll.w;
    }
  };
  // bias gradient: column sums of dZ over the chunk (hi + lo is the exact value)
  float bsum = 0.f;
  auto chunk_bias = [&](int st) {
    if (tk != 0 || tid >= kWtM) return;
    const unsigned char* base = smem + st * kWtStage;
#pragma unroll
    for (int rq = 0; rq < kWtRows / 4; ++rq) {
      const float4 a = *reinterpret_cast<const float4*>(base + rq * kWtQuadA + tid * 16);
      const float4 b = *reinterpret_cast<const float4*>(base + kWtPlaneA + rq * kWtQuadA + tid * 16);
      bsum += ((a.x + b.x) + (a.y + b.y)) + ((a.z + b.z) + (a.w + b.w));
    }
  };

  float acc[kWtN / 2];
#pragma unroll
  for (int i = 0; i < kWtN / 2; ++i) acc[i] = 0.f;
  auto chunk_mma = [&](int st) {
    const uint32_t sb = smem_u32(smem + st * kWtStage);
    const uint32_t a_hi = sb + (uint32_t)wg * 64 * 16, a_lo = a_hi + kWtPlaneA;
    const uint32_t b_hi = sb + 2 * kWtPlaneA, b_lo = b_hi + kWtPlaneB;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kWtRows / 8; ++ks) {
      // K-major no-swizzle: leading offset = next 4-row group, stride offset = 8 features
      const uint32_t oa = ks * 2 * kWtQuadA, ob = ks * 2 * kWtQuadB;
      const uint64_t dah = wgmma_desc(a_hi + oa, kWtQuadA, 128), dal = wgmma_desc(a_lo + oa, kWtQuadA, 128);
      const uint64_t dbh = wgmma_desc(b_hi + ob, kWtQuadB, 128), dbl = wgmma_desc(b_lo + ob, kWtQuadB, 128);
      switch (n_mma) {
        case 32: wt_kstep<32>(acc, dah, dal, dbh, dbl); break;
        case 64: wt_kstep<64>(acc, dah, dal, dbh, dbl); break;
        case 128: wt_kstep<128>(acc, dah, dal, dbh, dbl); break;
        default: wt_kstep<256>(acc, dah, dal, dbh, dbl); break;
      }
    }
    wgmma_commit();
  };

  if (nchunks > 0) chunk_fetch(0);
  for (int c = 0; c < nchunks; ++c) {
    const int st = c & 1;
    // the MMAs of chunk c-2 read this stage: every warpgroup waited for them (wait_group 1 at
    // the end of chunk c-1) before the barrier of chunk c-1
    chunk_store(st);
    if (c + 1 < nchunks) chunk_fetch(c + 1);  // in flight during the barrier and the MMAs
    fence_proxy_async_smem();
    __syncthreads();
    chunk_bias(st);
    // (a warpgroup whose dZ features lie past the matrix multiplies stale rows that are never
    // stored: issuing unconditionally keeps the MMAs out of divergent code)
    chunk_mma(st);
    wgmma_wait<1>();  // chunk c-1's group retired: its stage is free for chunk c+1
    __syncthreads();
  }
  wgmma_wait<0>();
  __syncthreads();  // all MMAs retired: the operand stages become the output tile

  // ---- epilogue: accumulators -> shared memory (the operand stages are dead) -> this slab's
  // gradient partial with coalesced 16-byte stores ----
  float* gp = p.gpart + (size_t)split * p.P;
  constexpr int kLdT = kWtN + 4;  // floats per staged row: 16-byte aligned
  float* tile = reinterpret_cast<float*>(smem);
  {
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < kWtN / 8; ++j) {
      if (8 * j < n_mma) {
        *reinterpret_cast<float2*>(tile + (size_t)r * kLdT + 8 * j + cq) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(tile + (size_t)(r + 8) * kLdT + 8 * j + cq) =
            make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
  }
  if (tid < kWtM && tk == 0 && n0 + tid < N) gp[Ly.b_off + n0 + tid] = bsum;
  __syncthreads();
  {
    const bool v4 = ((K & 3) == 0) && ((k0 & 3) == 0) && ((Ly.w_off & 3) == 0) &&
                    ((reinterpret_cast<uintptr_t>(gp) & 15) == 0);
    for (int r = warp; r < nrows_m; r += kWtThreads / 32) {
      float* dst = gp + Ly.w_off + (size_t)(n0 + r) * K + k0;
      const float* src = tile + (size_t)r * kLdT;
      if (v4) {
        for (int c = lane * 4; c < ncols; c += 128)
          *reinterpret_cast<float4*>(dst + c) = *reinterpret_cast<const float4*>(src + c);
      } else {
        for (int c = lane; c < ncols; c += 32) dst[c] = src[c];
      }
    }
  }
}

}  // namespace rb200

using namespace rb200;

// Launch the wgmma weight-gradient kernel.
int rb200_wgrad_tc_launch(const rb200_mlp_t* net, const float* net_input, int32_t batch,
                          const rb200_net_ws_t* ws, float* gpart, int32_t splits, void* stream) {
  WtParams p = {};
  p.n_layers = net->n_layers;
  p.B = batch;
  p.rows_per_split = ceil_div(ceil_div(batch, splits), kWtRows) * kWtRows;
  p.gpart = gpart;
  p.P = net->n_params;
  int jobs = 0;
  for (int l = 0; l < net->n_layers; ++l) {
    WtLayer& L = p.L[l];
    L.A = (l == 0) ? (net_input ? net_input : ws->input) : ws->hidden[l - 1];
    L.dZ = ws->dz[l];
    if (!L.A || !L.dZ) { set_last_error("rb200_mlp_wgrad: missing activation / dz for layer %d", l); return RB200_E_INVALID; }
    L.K = net->dims[l];
    L.N = net->dims[l + 1];
    L.w_off = net->w_off[l];
    L.b_off = net->b_off[l];
    L.tiles_m = ceil_div(L.N, kWtM);
    L.tiles_k = ceil_div(L.K, kWtN);
    L.job_start = jobs;
    jobs += L.tiles_m * L.tiles_k;
  }
  for (int l = net->n_layers; l < kMaxLayers; ++l) p.L[l].job_start = 1 << 30;
  dim3 grid(jobs, splits);
  return launch<wgrad_tc_kernel>(grid, kWtThreads, kWtSmem, (cudaStream_t)stream,
                                 "wgrad_tc_kernel launch", p);
}
