// reagent_b200 -- wide Linear forward on the Hopper tensor cores: wgmma (kind tf32) with the
// accumulators in registers, 3xTF32 error compensation.
//
//   out[B, N] = act(in[B, K] . W[N, K]^T + b)          (nn.Linear forward, wide N)
//
// Used for the QR-DQN head ([hidden -> A*N], reagent/models/fully_connected_network.py:
// 190-217 / reagent/training/qrdqn_trainer.py:125-149): at config 3 it is a
// 4096 x 6400 x 128 GEMM, the only genuinely GEMM-shaped op of the path.
//
// One CTA = one 128 (rows) x 128 (cols) output tile = two warpgroups, each owning 64 rows
// (wgmma m64n128k8, 64 fp32 accumulators per thread).  K is walked in 32-element chunks through
// ONE shared-memory stage; the next chunk's global loads are held in registers while the
// tensor cores consume the stage, and two CTAs share an SM so that one CTA's loads overlap the
// other's MMAs / epilogue.  Per chunk all 256 threads load 16 B pieces of in / W with LDG.128,
// split every value into hi = rna_tf32(x) and lo = x - hi and store both planes in the
// canonical K-major no-swizzle layout  [k/4][row][4 floats]  (core matrix = 8 rows x 16 B
// contiguous; SBO = 128 B between 8-row groups, LBO = rows*16 B + 16 B pad between the two
// 16-byte k-slices of one K=8 MMA).  Each warpgroup then issues, per K=8 step, the three MMAs
//   D += A_lo.B_hi ;  D += A_hi.B_lo ;  D += A_hi.B_hi
// and waits for them before the stage is overwritten.
// Epilogue: registers -> smem tile -> bias + activation -> coalesced global stores.
#include "rb200_wgmma.cuh"

namespace rb200 {

constexpr int kTcM = 128;     // rows per CTA (two m64 warpgroups)
constexpr int kTcN = 128;     // cols per CTA (wgmma N)
constexpr int kTcKC = 32;     // k elements per stage
constexpr int kTcThreads = 256;
constexpr int kTcCtasPerSm = 2;
constexpr int kTcQuadStride = kTcM * 4 + 4;            // floats between k quads: 2048 B + 16 B pad
constexpr int kTcPlane = (kTcKC / 4) * kTcQuadStride;  // floats per operand plane per stage
constexpr int kTcStageFloats = 4 * kTcPlane;           // A_hi, A_lo, B_hi, B_lo
constexpr int kTcLdo = kTcN + 4;                       // padded stride of the epilogue tile
constexpr int kTcBufFloats = (kTcM * kTcLdo > kTcStageFloats) ? kTcM * kTcLdo : kTcStageFloats;
constexpr size_t kTcSmemBytes = kTcBufFloats * sizeof(float) + 64;
constexpr int kTcIters = kTcM * (kTcKC / 4) / kTcThreads;  // 16 B pieces per thread per operand

struct TcDev {
  const float* in; const float* W; const float* b; float* out;
  int batch, K, N, act;
  // split-K (blockIdx.z): slice z walks chunks [z * chunks_per_split, ...) and stores its RAW
  // partial tile (no bias / activation) to out + z * batch * N; 0 = no split
  int chunks_per_split;
};

__global__ void __launch_bounds__(kTcThreads, kTcCtasPerSm) tc_linear_fwd_kernel(const TcDev p) {
  // Two CTAs per SM (66 KB smem, 64 accumulator registers per thread each): while one CTA's
  // MMAs or epilogue run, the other loads -- the overlap a deeper ring would give.
  extern __shared__ __align__(128) float smem[];
  float* a_hi = smem;
  float* a_lo = a_hi + kTcPlane;
  float* b_hi = a_lo + kTcPlane;
  float* b_lo = b_hi + kTcPlane;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = warp >> 2;  // warpgroup: rows [64 wg, 64 wg + 64) of the tile
  const int row0 = blockIdx.x * kTcM, col0 = blockIdx.y * kTcN;
  const int K = p.K;
  int c_begin = 0, nchunks = ceil_div(K, kTcKC);
  const bool raw = p.chunks_per_split > 0;
  if (raw) {
    c_begin = (int)blockIdx.z * p.chunks_per_split;
    nchunks = nchunks < c_begin + p.chunks_per_split ? nchunks : c_begin + p.chunks_per_split;
  }
  float* const outp = raw ? p.out + (size_t)blockIdx.z * p.batch * p.N : p.out;
  const bool vin = ((K & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.in) & 15) == 0);
  const bool vw = ((K & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.W) & 15) == 0);

  // thread -> pieces (row = idx / 8, quad = idx % 8), idx = tid + it*256: a warp reads 4 rows x
  // 128 contiguous bytes of global memory and stores them to the [k quad][row][4] layout whose
  // quad stride is padded by 16 B, so the 32 pieces of a warp spread evenly over the banks
  // (4 wavefronts for 512 B: optimal).
  float4 ra[kTcIters], rb[kTcIters];
  auto load_regs = [&](int c) {
    const int k0 = c * kTcKC;
#pragma unroll
    for (int it = 0; it < kTcIters; ++it) {
      const int idx = tid + it * kTcThreads;
      const int r = idx >> 3, q = idx & 7;
      const int k = k0 + 4 * q;
      float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = make_float4(0.f, 0.f, 0.f, 0.f);
      const int row = row0 + r, col = col0 + r;
      if (row < p.batch) {
        const float* sp = p.in + (size_t)row * K;
        if (vin && k + 3 < K) va = __ldg(reinterpret_cast<const float4*>(sp + k));
        else {
          if (k < K) va.x = sp[k];
          if (k + 1 < K) va.y = sp[k + 1];
          if (k + 2 < K) va.z = sp[k + 2];
          if (k + 3 < K) va.w = sp[k + 3];
        }
      }
      if (col < p.N) {
        const float* sp = p.W + (size_t)col * K;
        if (vw && k + 3 < K) vb = __ldg(reinterpret_cast<const float4*>(sp + k));
        else {
          if (k < K) vb.x = sp[k];
          if (k + 1 < K) vb.y = sp[k + 1];
          if (k + 2 < K) vb.z = sp[k + 2];
          if (k + 3 < K) vb.w = sp[k + 3];
        }
      }
      ra[it] = va;
      rb[it] = vb;
    }
  };

  float acc[kTcN / 2];
#pragma unroll
  for (int i = 0; i < kTcN / 2; ++i) acc[i] = 0.f;
  constexpr uint32_t LBO = kTcQuadStride * 4;  // bytes between the two 16 B k-slices of an MMA
  constexpr uint32_t SBO = 128;                // bytes between 8-row groups
  const uint32_t a_row_off = (uint32_t)wg * 64 * 16;

  load_regs(c_begin);
  for (int c = c_begin; c < nchunks; ++c) {
    // the MMAs of the previous chunk (both warpgroups) have completed: the stage is free
    if (c > c_begin) __syncthreads();
#pragma unroll
    for (int it = 0; it < kTcIters; ++it) {
      const int idx = tid + it * kTcThreads;
      const int r = idx >> 3, q = idx & 7;
      const int off = q * kTcQuadStride + r * 4;  // [k quad][row][4], padded quad stride
      float4 h, l;
      split_tf32(ra[it], h, l);
      *reinterpret_cast<float4*>(a_hi + off) = h;
      *reinterpret_cast<float4*>(a_lo + off) = l;
      split_tf32(rb[it], h, l);
      *reinterpret_cast<float4*>(b_hi + off) = h;
      *reinterpret_cast<float4*>(b_lo + off) = l;
    }
    // make the generic-proxy stores visible to the tensor cores (async proxy)
    fence_proxy_async_smem();
    __syncthreads();
    wgmma_fence();
#pragma unroll
    for (int s4 = 0; s4 < kTcKC / 8; ++s4) {
      const uint32_t koff = (uint32_t)(2 * s4) * LBO;  // k quad 2*s4
      const uint64_t dah = wgmma_desc(smem_u32(a_hi) + koff + a_row_off, LBO, SBO);
      const uint64_t dal = wgmma_desc(smem_u32(a_lo) + koff + a_row_off, LBO, SBO);
      const uint64_t dbh = wgmma_desc(smem_u32(b_hi) + koff, LBO, SBO);
      const uint64_t dbl = wgmma_desc(smem_u32(b_lo) + koff, LBO, SBO);
      wgmma_ss_n128(acc, dal, dbh, 1u);
      wgmma_ss_n128(acc, dah, dbl, 1u);
      wgmma_ss_n128(acc, dah, dbh, 1u);
    }
    wgmma_commit();
    // global loads of the next chunk fly while the tensor cores work on this one
    if (c + 1 < nchunks) load_regs(c + 1);
    wgmma_wait<0>();
  }
  __syncthreads();  // every warpgroup is done with the operand stage: it becomes the output tile

  // ---- epilogue: registers -> smem tile -> bias + activation -> coalesced global ----
  {
    constexpr int LDO = kTcLdo;    // padded row stride of the output tile in smem
    float* otile = smem;           // 128 x 132 floats, reuses the operand stage
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < kTcN / 8; ++j) {
      *reinterpret_cast<float2*>(otile + r * LDO + 8 * j + cq) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(otile + (r + 8) * LDO + 8 * j + cq) =
          make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    __syncthreads();
    // each warp writes whole 512-byte row segments; bias + activation applied on the way out
    const bool vo = ((p.N & 3) == 0) && ((reinterpret_cast<uintptr_t>(outp) & 15) == 0);
    for (int idx = tid; idx < kTcM * (kTcN / 4); idx += kTcThreads) {
      const int rr = idx >> 5, c4 = (idx & 31) * 4;
      const int row = row0 + rr, col = col0 + c4;
      if (row >= p.batch || col >= p.N) continue;
      float4 o = *reinterpret_cast<const float4*>(otile + rr * LDO + c4);
      float ov[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (!raw && col + j < p.N) ov[j] = act_fwd(ov[j] + (p.b ? __ldg(p.b + col + j) : 0.f), p.act);
      float* dst = outp + (size_t)row * p.N + col;
      if (vo && col + 3 < p.N) {
        *reinterpret_cast<float4*>(dst) = make_float4(ov[0], ov[1], ov[2], ov[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (col + j < p.N) dst[j] = ov[j];
      }
    }
  }
}

// ---- nn.Linear backward w.r.t. its input on the same kernel (split-K) ----------------------
// Wt[k][n] = W[n][k]: the GEMM above wants both operands contiguous along the contraction
__global__ void __launch_bounds__(256) tc_transpose_kernel(const float* __restrict__ W, int N, int K,
                                                          float* __restrict__ Wt) {
  __shared__ float tile[32][33];
  const int n0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int j = ty; j < 32; j += 8) {
    const int n = n0 + j, k = k0 + tx;
    tile[j][tx] = (n < N && k < K) ? W[(size_t)n * K + k] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int k = k0 + j, n = n0 + tx;
    if (k < K && n < N) Wt[(size_t)k * N + n] = tile[tx][j];
  }
}

// out[b][k] = (sum over slices of partial[s][b][k]) * act'(h_prev[b][k]), slices added in order
__global__ void __launch_bounds__(256) tc_dx_reduce_kernel(const float* __restrict__ partial, int splits,
                                                          size_t slice, const float* __restrict__ h_prev,
                                                          int act_prev, float* __restrict__ out, size_t n4) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 acc = reinterpret_cast<const float4*>(partial)[i];
  for (int s = 1; s < splits; ++s) {
    const float4 v = reinterpret_cast<const float4*>(partial + (size_t)s * slice)[i];
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  if (h_prev && act_prev != RB200_ACT_LINEAR) {
    const float4 h = reinterpret_cast<const float4*>(h_prev)[i];
    acc.x *= act_bwd_from_out(h.x, act_prev); acc.y *= act_bwd_from_out(h.y, act_prev);
    acc.z *= act_bwd_from_out(h.z, act_prev); acc.w *= act_bwd_from_out(h.w, act_prev);
  }
  reinterpret_cast<float4*>(out)[i] = acc;
}

struct DxPlan { int splits, chunks_per_split; size_t wt_floats, partial_floats; };
// the tensor-core path pays off for a wide layer (N = out features is the contraction here)
static bool dx_plan(int K, int N, int batch, DxPlan* pl) {
  if (N < 1024 || batch < 256 || (K & 3) != 0 || (N & 3) != 0) return false;
  const int tiles = ceil_div(batch, kTcM) * ceil_div(K, kTcN);
  const int nchunks = ceil_div(N, kTcKC);
  int splits = (kTcCtasPerSm * kNumSMs) / tiles;
  splits = splits < 1 ? 1 : (splits > nchunks ? nchunks : splits);
  pl->chunks_per_split = ceil_div(nchunks, splits);
  pl->splits = ceil_div(nchunks, pl->chunks_per_split);
  pl->wt_floats = ((size_t)K * N + 31) & ~(size_t)31;
  pl->partial_floats = (size_t)pl->splits * batch * K;
  return true;
}

}  // namespace rb200

using namespace rb200;

// Scratch bytes rb200_linear_backward_dx_tc needs for this shape; 0 = shape not taken by the
// tensor-core path (use rb200_linear_backward_dx).
extern "C" int64_t rb200_linear_backward_dx_tc_scratch_bytes(int32_t K, int32_t N, int32_t batch) {
  DxPlan pl;
  if (K <= 0 || N <= 0 || batch <= 0 || !dx_plan(K, N, batch, &pl)) return 0;
  return (int64_t)((pl.wt_floats + pl.partial_floats) * sizeof(float));
}

// Same contract as rb200_linear_backward_dx (W is the nn.Linear weight [N out x K in], dz [B, N],
// out [B, K] = (dz . W) * act'(h_prev)) on wgmma: W is transposed into the scratch, the
// contraction over N runs as split-K slices of tc_linear_fwd_kernel, a last pass adds the
// slices in order and applies act'.
extern "C" int rb200_linear_backward_dx_tc(const float* W, int32_t K, int32_t N, const float* dz,
                                           const float* h_prev, int32_t act_prev, int32_t batch,
                                           float* out, void* scratch, int64_t scratch_bytes,
                                           void* stream) {
  if (!W || !dz || !out || !scratch || K <= 0 || N <= 0 || batch <= 0) { set_last_error("rb200_linear_backward_dx_tc: bad argument"); return RB200_E_INVALID; }
  DxPlan pl;
  if (!dx_plan(K, N, batch, &pl)) { set_last_error("rb200_linear_backward_dx_tc: shape not supported (N >= 1024, batch >= 256, K and N multiples of 4)"); return RB200_E_INVALID; }
  if (scratch_bytes < (int64_t)((pl.wt_floats + pl.partial_floats) * sizeof(float))) { set_last_error("rb200_linear_backward_dx_tc: scratch too small"); return RB200_E_INVALID; }
  if ((reinterpret_cast<uintptr_t>(scratch) & 15) || (reinterpret_cast<uintptr_t>(out) & 15) ||
      (h_prev && (reinterpret_cast<uintptr_t>(h_prev) & 15))) { set_last_error("rb200_linear_backward_dx_tc: buffers must be 16-byte aligned"); return RB200_E_INVALID; }
  cudaStream_t st = (cudaStream_t)stream;
  if (cudaError_t e = opt_in_smem<tc_linear_fwd_kernel>(kTcSmemBytes))
    return check_cuda(e, "cudaFuncSetAttribute(tc_linear_fwd)");
  float* Wt = static_cast<float*>(scratch);
  float* partial = Wt + pl.wt_floats;
  tc_transpose_kernel<<<dim3(ceil_div(N, 32), ceil_div(K, 32)), 256, 0, st>>>(W, N, K, Wt);
  TcDev p{dz, Wt, nullptr, partial, batch, /*contraction*/ N, /*columns*/ K, RB200_ACT_LINEAR, pl.chunks_per_split};
  dim3 grid(ceil_div(batch, kTcM), ceil_div(K, kTcN), pl.splits);
  tc_linear_fwd_kernel<<<grid, kTcThreads, kTcSmemBytes, st>>>(p);
  const size_t n4 = (size_t)batch * K / 4;
  tc_dx_reduce_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, st>>>(partial, pl.splits, (size_t)batch * K, h_prev,
                                                                   act_prev, out, n4);
  return check_cuda(cudaGetLastError(), "rb200_linear_backward_dx_tc launch");
}

// Same contract as rb200_linear_forward; chosen by it for large shapes.
extern "C" int rb200_linear_forward_tc(const float* W, const float* b, int32_t act, int32_t K,
                                       int32_t N, const float* in, int32_t batch, float* out,
                                       void* stream) {
  if (!W || !in || !out || K <= 0 || N <= 0 || batch <= 0) { set_last_error("rb200_linear_forward_tc: bad argument"); return RB200_E_INVALID; }
  TcDev p{in, W, b, out, batch, K, N, act, 0};
  dim3 grid(ceil_div(batch, kTcM), ceil_div(N, kTcN));
  return launch<tc_linear_fwd_kernel>(grid, kTcThreads, kTcSmemBytes, (cudaStream_t)stream,
                                      "tc_linear_fwd_kernel launch", p);
}
