// reagent_b200 -- dueling head (reagent/models/dueling_q_network.py:92-103) folded into a Linear.
//
//   q[a, n] = value[n] + (advantage[a, n] - mean_{a', n'} advantage[a', n'])
// (n = atom index; N = 1 for plain DQN, the mean runs over ALL non-batch dims, :98-101) with
//   value = W_v.h_v + b_v  (W_v [N, H]),   advantage = W_a.h_a + b_a  (W_a [A*N, H])
// is linear in the concatenated head activations h = [h_a | h_v] (H each), so a dueling network
// is a plain MLP whose last layer, with output row r = a*N + n (the (B, A, N) view of
// fully_connected_network.py:215-217), is
//   W_q[r, j]     = W_a[r, j] - mean_r' W_a[r', j]      (j <  H)
//   W_q[r, H + j] = W_v[r % N, j]                       (j <  H)
//   b_q[r]        = b_a[r] - mean(b_a) + b_v[r % N]
// and every fused kernel of the path (TD step, forward, weight gradients) runs on it unchanged.
// The TRUE parameters stay (W_a, b_a, W_v, b_v): `fold` rebuilds W_q / b_q from them before a
// step, `unfold` maps the gradient of the folded layer back with the transposed linear map
//   dW_a[r, j] = dW_q[r, j] - mean_r' dW_q[r', j],  dW_v[n, j] = sum_a dW_q[a*N + n, H + j],
//   db_a[r]    = db_q[r]    - mean(db_q),           db_v[n]    = sum_a db_q[a*N + n]
// (per gradient partial slab) and clears the folded layer's gradient so that the fused Adam
// kernel, which also sweeps the derived region of the arena, leaves it untouched (g = 0, m = v = 0).
//
// Two launches each: column sums over the R = A*N rows (one CTA of 1024 threads per 32
// columns, rows strided over the 32 warps, coalesced 128-byte row segments), then an
// element-parallel apply.  `scratch` holds the sums: >= (2H + 2) floats per slab.
#include "rb200_common.cuh"

namespace rb200 {

// sums[c] = sum_r src[r*ld + c] for c < ncols; sums[ncols] = sum_r bias[r]   (per slab)
__global__ void __launch_bounds__(1024) dueling_colsum_kernel(
    const float* __restrict__ src, const float* __restrict__ bias, long long slab_stride, int R,
    int ncols, int ld, float* __restrict__ sums, int sums_stride) {
  __shared__ float red[32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* s = src + (size_t)blockIdx.y * slab_stride;
  const float* b = bias + (size_t)blockIdx.y * slab_stride;
  float* out = sums + (size_t)blockIdx.y * sums_stride;
  const int ngroups = ceil_div(ncols, 32);
  float acc = 0.f;
  if ((int)blockIdx.x < ngroups) {
    const int c = blockIdx.x * 32 + lane;
    if (c < ncols)
      for (int r = warp; r < R; r += 32) acc += s[(size_t)r * ld + c];
  } else {  // the extra CTA: bias sum
    for (int r = threadIdx.x; r < R; r += 1024) acc += b[r];
    acc = warp_sum(acc);
  }
  red[warp][lane] = acc;
  __syncthreads();
  if (warp == 0) {
    if ((int)blockIdx.x < ngroups) {
      float t = 0.f;
      for (int w = 0; w < 32; ++w) t += red[w][lane];
      const int c = blockIdx.x * 32 + lane;
      if (c < ncols) out[c] = t;
    } else if (lane == 0) {
      float t = 0.f;
      for (int w = 0; w < 32; ++w) t += red[w][0];
      out[ncols] = t;
    }
  }
}

__global__ void dueling_fold_apply_kernel(const float* __restrict__ Wa, const float* __restrict__ ba,
                                          const float* __restrict__ Wv, const float* __restrict__ bv,
                                          int R, int N, int H, const float* __restrict__ sums,
                                          float* __restrict__ Wq, float* __restrict__ bq) {
  const long long total = (long long)R * 2 * H;
  const float invR = 1.f / (float)R;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total + R;
       i += (long long)gridDim.x * blockDim.x) {
    if (i < total) {
      const int r = (int)(i / (2 * H)), j = (int)(i - (long long)r * 2 * H);
      Wq[i] = (j < H) ? Wa[(size_t)r * H + j] - sums[j] * invR : Wv[(size_t)(r % N) * H + (j - H)];
    } else {
      const int r = (int)(i - total);
      bq[r] = ba[r] - sums[H] * invR + bv[r % N];
    }
  }
}

// per slab: dW_a, db_a from the folded gradient; the folded gradient (dW_q and db_q) is cleared
__global__ void dueling_unfold_apply_kernel(float* __restrict__ g, long long slab_stride, int R,
                                            int N, int H, long long o_wq, long long o_bq,
                                            long long o_wa, long long o_ba,
                                            const float* __restrict__ sums, int sums_stride) {
  float* s = g + (size_t)blockIdx.y * slab_stride;
  const float* sm = sums + (size_t)blockIdx.y * sums_stride;
  const long long total = (long long)R * 2 * H;
  const float invR = 1.f / (float)R;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total + R;
       i += (long long)gridDim.x * blockDim.x) {
    if (i < total) {
      const int r = (int)(i / (2 * H)), j = (int)(i - (long long)r * 2 * H);
      if (j < H) s[o_wa + (size_t)r * H + j] = s[o_wq + i] - sm[j] * invR;
      s[o_wq + i] = 0.f;
    } else {
      const int r = (int)(i - total);
      s[o_ba + r] = s[o_bq + r] - sm[2 * H] * invR;
      s[o_bq + r] = 0.f;
    }
  }
}

// per slab: dW_v[n, j] = sum_a dW_q[a*N + n, H + j], db_v[n] = sum_a db_q[a*N + n]; runs BEFORE
// the apply kernel clears the folded gradient
__global__ void dueling_unfold_value_kernel(float* __restrict__ g, long long slab_stride, int A,
                                            int N, int H, long long o_wq, long long o_bq,
                                            long long o_wv, long long o_bv) {
  float* s = g + (size_t)blockIdx.y * slab_stride;
  const int total = N * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total + N; i += gridDim.x * blockDim.x) {
    float acc = 0.f;
    if (i < total) {
      const int n = i / H, j = i - n * H;
      for (int a = 0; a < A; ++a) acc += s[o_wq + ((size_t)a * N + n) * 2 * H + H + j];
      s[o_wv + i] = acc;
    } else {
      const int n = i - total;
      for (int a = 0; a < A; ++a) acc += s[o_bq + (size_t)a * N + n];
      s[o_bv + n] = acc;
    }
  }
}

}  // namespace rb200

using namespace rb200;

extern "C" int64_t rb200_dueling_scratch_floats(int32_t head_hidden, int32_t splits) {
  return (int64_t)(2 * head_hidden + 2) * (splits < 1 ? 1 : splits);
}

extern "C" int rb200_dueling_fold(const float* W_adv, const float* b_adv, const float* w_val,
                                  const float* b_val, int32_t num_actions, int32_t num_atoms,
                                  int32_t head_hidden, float* W_q, float* b_q, float* scratch,
                                  void* stream) {
  if (!W_adv || !b_adv || !w_val || !b_val || !W_q || !b_q || !scratch || num_actions <= 0 ||
      num_atoms <= 0 || head_hidden <= 0) {
    set_last_error("rb200_dueling_fold: bad argument");
    return RB200_E_INVALID;
  }
  const int R = num_actions * num_atoms, H = head_hidden;
  cudaStream_t st = (cudaStream_t)stream;
  dueling_colsum_kernel<<<dim3(ceil_div(H, 32) + 1, 1), 1024, 0, st>>>(W_adv, b_adv, 0, R, H, H,
                                                                      scratch, 0);
  const long long work = (long long)R * 2 * H + R;
  int blocks = (int)((work + 255) / 256);
  if (blocks > kNumSMs * 8) blocks = kNumSMs * 8;
  dueling_fold_apply_kernel<<<blocks, 256, 0, st>>>(W_adv, b_adv, w_val, b_val, R, num_atoms, H,
                                                    scratch, W_q, b_q);
  return check_cuda(cudaGetLastError(), "dueling fold kernels launch");
}

extern "C" int rb200_dueling_unfold(float* grad, int64_t slab_stride, int32_t splits,
                                    int32_t num_actions, int32_t num_atoms, int32_t head_hidden,
                                    int64_t off_W_q, int64_t off_b_q, int64_t off_W_adv,
                                    int64_t off_b_adv, int64_t off_w_val, int64_t off_b_val,
                                    float* scratch, void* stream) {
  if (!grad || !scratch || splits <= 0 || num_actions <= 0 || num_atoms <= 0 || head_hidden <= 0) {
    set_last_error("rb200_dueling_unfold: bad argument");
    return RB200_E_INVALID;
  }
  const int R = num_actions * num_atoms, H = head_hidden;
  cudaStream_t st = (cudaStream_t)stream;
  const int sstride = 2 * H + 2;
  dueling_colsum_kernel<<<dim3(ceil_div(2 * H, 32) + 1, splits), 1024, 0, st>>>(
      grad + off_W_q, grad + off_b_q, slab_stride, R, 2 * H, 2 * H, scratch, sstride);
  dueling_unfold_value_kernel<<<dim3(ceil_div(num_atoms * H + num_atoms, 256), splits), 256, 0, st>>>(
      grad, slab_stride, num_actions, num_atoms, H, off_W_q, off_b_q, off_w_val, off_b_val);
  const long long work = (long long)R * 2 * H + R;
  int blocks = (int)((work + 255) / 256);
  if (blocks > kNumSMs * 2) blocks = kNumSMs * 2;
  dueling_unfold_apply_kernel<<<dim3(blocks, splits), 256, 0, st>>>(
      grad, slab_stride, R, num_atoms, H, off_W_q, off_b_q, off_W_adv, off_b_adv, scratch, sstride);
  return check_cuda(cudaGetLastError(), "dueling unfold kernels launch");
}
