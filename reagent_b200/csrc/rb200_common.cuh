// reagent_b200 -- common device/host helpers (sm_90a only).
//
// Data layout conventions used by every kernel in this library
//   * all batch tensors are dense row-major fp32, one transition per row;
//   * an MLP's parameters live in ONE flat fp32 arena laid out
//       [W0 (d1 x d0, row-major = nn.Linear.weight), b0 (d1), W1, b1, ...]
//     which is exactly torch's `parameters()` order for the reference's
//     FullyConnectedNetwork (reagent/models/fully_connected_network.py:101-153),
//     so Adam / Polyak / all-reduce are single launches over the arena;
//   * gradient partials, Adam moments and target networks use the same layout.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/reagent_b200.h"

namespace rb200 {

constexpr int kThreads = 256;          // every row-tile kernel uses 8 warps
constexpr int kNumSMs = 132;           // H100 SXM: grid sizes that fill the GPU a whole number of times
constexpr int kMaxLayers = RB200_MAX_LAYERS;

// Device-side view of one MLP (passed by value as a kernel parameter).
struct Mlp {
  int n_layers;
  int dims[kMaxLayers + 1];
  int act[kMaxLayers];
  const float* params;                 // arena base (device)
  long long w_off[kMaxLayers];         // float offsets into the arena
  long long b_off[kMaxLayers];
  long long n_params;
};

inline Mlp make_mlp(const rb200_mlp_t* d) {
  Mlp m;
  m.n_layers = d->n_layers;
  for (int l = 0; l <= kMaxLayers; ++l) m.dims[l] = (l <= d->n_layers) ? d->dims[l] : 0;
  for (int l = 0; l < kMaxLayers; ++l) {
    const bool on = l < d->n_layers;
    m.act[l] = on ? d->act[l] : 0;
    m.w_off[l] = on ? d->w_off[l] : 0;
    m.b_off[l] = on ? d->b_off[l] : 0;
  }
  m.params = d->params;
  m.n_params = d->n_params;
  return m;
}
int validate_mlp(const rb200_mlp_t* d, const char* name);

__host__ __device__ __forceinline__ int round_up4(int x) { return (x + 3) & ~3; }
__host__ __device__ __forceinline__ int ceil_div(int a, int b) { return (a + b - 1) / b; }

// ----------------------------------------------------------------------------
// activations (reagent/models/fully_connected_network.py:37-44)
// ----------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ float act_fwd(float x, int act) {
  switch (act) {
    case RB200_ACT_RELU: return x > 0.f ? x : 0.f;
    case RB200_ACT_TANH: return tanhf(x);
    case RB200_ACT_LEAKY_RELU: return x > 0.f ? x : 0.01f * x;
    case RB200_ACT_SIGMOID: return sigmoidf(x);
    case RB200_ACT_SOFTPLUS: return x > 20.f ? x : log1pf(expf(x));
    default: return x;
  }
}
// derivative of the activation expressed through its OUTPUT y
__device__ __forceinline__ float act_bwd_from_out(float y, int act) {
  switch (act) {
    case RB200_ACT_RELU: return y > 0.f ? 1.f : 0.f;
    case RB200_ACT_TANH: return 1.f - y * y;
    case RB200_ACT_LEAKY_RELU: return y > 0.f ? 1.f : 0.01f;
    case RB200_ACT_SIGMOID: return y * (1.f - y);
    case RB200_ACT_SOFTPLUS: return 1.f - expf(-y);
    default: return 1.f;
  }
}

// ----------------------------------------------------------------------------
// cp.async (LDGSTS) helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// torch.argmax of a one-hot row of n values held by one warp (lanes take c = lane, lane + 32,
// ...): the column of the first maximum, on every lane.  A row with no value above -inf (all
// NaN, say) gives 0, as torch.argmax does for a row of NaNs.
__device__ __forceinline__ int warp_first_argmax(const float* row, int n) {
  const int lane = threadIdx.x & 31;
  float lv = -INFINITY;
  int li = n;
  for (int c = lane; c < n; c += 32) {
    const float v = row[c];
    if (v > lv) { lv = v; li = c; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, lv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, li, o);
    if (ov > lv || (ov == lv && oi < li)) { lv = ov; li = oi; }
  }
  if (li >= n) li = 0;
  return li;
}

// Sum over the CTA of one fp64 value per thread, in a fixed order (butterfly within each warp,
// then warps 0, 1, ... from 0.0); every thread gets the total.  The CTA has 32 * kWarps threads
// and s_warp is shared memory with one slot per warp.
template <int kWarps>
__device__ __forceinline__ double block_sum_f64(double v, double (&s_warp)[kWarps]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < kWarps; ++w) t += s_warp[w];
  return t;
}

// ----------------------------------------------------------------------------
// TF32 tensor-core products with 3xTF32 error compensation
// ----------------------------------------------------------------------------
// x = hi + lo with hi = x rounded to TF32;  a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi with fp32
// accumulation in the MMA.  The dropped a_lo*b_lo term is ~2^-22 relative, which keeps the 1e-5
// fp32 parity that plain TF32 (~1e-3) cannot hold.
//
// hi = x rounded to nearest (ties away) at 10 explicit mantissa bits, done with integer ops
// (ptxas expands cvt.rna.tf32.f32 to 5 instructions; this is 2).  lo = x - hi is exact in fp32
// and is handed to the MMA as is: the tensor core drops its low 13 bits, an error
// <= 2^-11 |lo| <= 2^-22 |x|, the same order as the dropped lo*lo term, and unbiased because hi
// is rounded to nearest.  3 instructions per element.
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
  lo = x - hi;
}
// the same split as mma.sync operand registers
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  float h, l;
  split_tf32(x, h, l);
  hi = __float_as_uint(h);
  lo = __float_as_uint(l);
}
__device__ __forceinline__ void split_tf32(const float4 v, float4& hi, float4& lo) {
  split_tf32(v.x, hi.x, lo.x);
  split_tf32(v.y, hi.y, lo.y);
  split_tf32(v.z, hi.z, lo.z);
  split_tf32(v.w, hi.w, lo.w);
}

// c += a . b on mma.sync.m16n8k8 (TF32 operands, fp32 accumulators)
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4],
                                         const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, "
      "{%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ void mma_3xtf32(float (&c)[4], const uint32_t (&ah)[4],
                                           const uint32_t (&al)[4], const uint32_t (&bh)[2],
                                           const uint32_t (&bl)[2]) {
  mma_tf32(c, al, bh);
  mma_tf32(c, ah, bl);
  mma_tf32(c, ah, bh);
}

// First two passes of a softmax over one row held by one warp (lanes take c = lane, lane + 32,
// ...), in torch's order: mx = max_c x(c), sum = sum_c exp(x(c) - mx).  `x` is a callable
// returning element c.  Xor butterflies: every lane ends with the same bits.  The rounded
// intrinsics keep the subtraction out of expf's FMA; c51_log_softmax lets the compiler fuse it
// and keeps its own loop so that its results stay as they are.
template <typename Row>
__device__ __forceinline__ void warp_row_max_sumexp(const Row& x, int n, float& mx, float& sum) {
  const int lane = threadIdx.x & 31;
  float m = -INFINITY;
  for (int c = lane; c < n; c += 32) m = fmaxf(m, x(c));
  m = warp_max(m);
  float s = 0.f;
  for (int c = lane; c < n; c += 32) s = __fadd_rn(s, expf(__fsub_rn(x(c), m)));
  mx = m;
  sum = warp_sum(s);
}

// masked_softmax(x, mask, temperature) of one row held by one thread (reagent/core/torch_utils.py:
// 62-73): logit(c) = x/t - (1 - m)*1e20, mx its max, den = sum_c exp(logit - mx)*m in column order,
// p(c) = exp(logit - mx)*m / den with NaN (a fully masked row) -> 0.  The CPE heads of the training
// step and the evaluation page share these, so both give the same propensity bits.
__device__ __forceinline__ float masked_softmax_logit(float x, float m, float t) {
  return __fsub_rn(__fdiv_rn(x, t), __fmul_rn(__fsub_rn(1.f, m), 1e20f));
}
__device__ __forceinline__ void masked_softmax_stats(const float* x, const float* mk, float t, int A,
                                                     float& mx, float& den) {
  mx = -INFINITY;
  for (int c = 0; c < A; ++c) mx = fmaxf(mx, masked_softmax_logit(x[c], mk ? mk[c] : 1.f, t));
  den = 0.f;
  for (int c = 0; c < A; ++c) {
    const float m = mk ? mk[c] : 1.f;
    den += __fmul_rn(expf(__fsub_rn(masked_softmax_logit(x[c], m, t), mx)), m);
  }
}
__device__ __forceinline__ float masked_softmax_p(float x, float m, float t, float mx, float den) {
  const float p = __fdiv_rn(__fmul_rn(expf(__fsub_rn(masked_softmax_logit(x, m, t), mx)), m), den);
  return p != p ? 0.f : p;
}

// ----------------------------------------------------------------------------
// deterministic loss means
// ----------------------------------------------------------------------------
// A loss kernel's mean over the batch: every block publishes its partial(s) to `partials`, and
// the last block to take `counter` sums them in a fixed order, hands the totals to `fin` and
// re-arms the counter for the next launch.  There are two summation orders, and each kernel keeps
// the one it has, since another order changes the loss bits:
//   finish_serial, called by ONE thread of each block: kCh partials per block at
//     partials[kCh * block + c]; the last block's thread adds each channel in block order.
//   finish_block, called by ALL threads (one CTA per batch row, so grids of thousands of
//     blocks): `mine` is read from thread 0; the last block's thread t adds load(i, partials[i])
//     over i = t, t + blockDim, ..., the warps combine with warp_sum, and thread 0 adds the warp
//     sums in order into s_warp[blockDim / 32] (the caller's shared memory).  One thread walking
//     4096 dependent loads instead cost ~20 us of kernel tail.
template <int kCh, typename Fin>
__device__ __forceinline__ void finish_serial(float* partials, uint32_t* counter,
                                              const float (&mine)[kCh], Fin fin) {
#pragma unroll
  for (int c = 0; c < kCh; ++c) partials[kCh * blockIdx.x + c] = mine[c];
  __threadfence();
  if (atomicAdd(counter, 1u) == gridDim.x - 1) {
    __threadfence();
    float tot[kCh] = {};
    for (unsigned i = 0; i < gridDim.x; ++i) {
#pragma unroll
      for (int c = 0; c < kCh; ++c) tot[c] += ((volatile float*)partials)[kCh * i + c];
    }
    fin(tot);
    *counter = 0u;
  }
}

template <typename Load, typename Fin>
__device__ __forceinline__ void finish_block(float* partials, uint32_t* counter, float mine,
                                             float* s_warp, bool& s_last, Load load, Fin fin) {
  const unsigned tid = threadIdx.x;
  if (tid == 0) {
    partials[blockIdx.x] = mine;
    __threadfence();
    s_last = atomicAdd(counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (s_last) {
    __threadfence();
    float tot = 0.f;
    for (unsigned i = tid; i < gridDim.x; i += blockDim.x) tot += load(i, ((volatile float*)partials)[i]);
    tot = warp_sum(tot);
    __syncthreads();
    if ((tid & 31) == 0) s_warp[tid >> 5] = tot;
    __syncthreads();
    if (tid == 0) {
      float t2 = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t2 += s_warp[w];
      fin(t2);
      *counter = 0u;
    }
  }
}

// Error plumbing shared by the C-ABI translation units.
void set_last_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);

// Dynamic shared-memory opt-in of `Kernel`, remembered PER DEVICE (the attribute is per device
// and per function): a high-water mark indexed by the current device id, so the first launch on
// a second GPU of the same process opts in as well.  Racing threads at worst set the attribute
// twice.  Raised outside CUDA-graph capture by the first eager call.
template <auto Kernel>
inline cudaError_t opt_in_smem(size_t bytes) {
  static size_t configured[64] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev >= 0 && dev < 64 && configured[dev] >= bytes) return cudaSuccess;
  e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess && dev >= 0 && dev < 64) configured[dev] = bytes;
  return e;
}

// Opts `Kernel` in to `smem` bytes of dynamic shared memory and launches it; errors of either
// step are reported under `what`.
template <auto Kernel, typename... Args>
inline int launch(dim3 grid, dim3 block, size_t smem, cudaStream_t st, const char* what,
                  Args... args) {
  if (cudaError_t e = opt_in_smem<Kernel>(smem)) return check_cuda(e, what);
  Kernel<<<grid, block, smem, st>>>(args...);
  return check_cuda(cudaGetLastError(), what);
}

}  // namespace rb200
