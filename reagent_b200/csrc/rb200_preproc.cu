// reagent_b200 -- stand-alone Preprocessor.forward kernel (HBM-bound, elementwise).
#include "rb200_preproc.cuh"

namespace rb200 {

// one thread per output element; a warp covers 32 consecutive output columns of a row
// (coalesced stores; the loads hit the same 128B lines of the input row).
__global__ void preprocess_kernel(const float* __restrict__ in, const uint8_t* __restrict__ presence,
                                  int presence_is_float, long long rows, int f_in, int f_out,
                                  const rb200_feature_col_t* __restrict__ cols,
                                  const float* __restrict__ quantiles, float* __restrict__ out) {
  const long long total = rows * (long long)f_out;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const long long r = i / f_out;
    const int j = (int)(i - r * f_out);
    const rb200_feature_col_t f = cols[j];
    const float x = in[r * f_in + f.src_col];
    float p = 1.f;
    if (presence != nullptr) {
      p = presence_is_float ? reinterpret_cast<const float*>(presence)[r * f_in + f.src_col]
                            : (float)presence[r * f_in + f.src_col];
    }
    out[i] = preprocess_value(x, p, f, quantiles);
  }
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_preprocess(const float* input, const void* presence, int32_t presence_is_float,
                                int64_t rows, int32_t f_in, int32_t f_out,
                                const rb200_feature_col_t* cols, const float* quantiles,
                                float* out, void* stream) {
  if (!input || !cols || !out || rows < 0 || f_in <= 0 || f_out <= 0) {
    set_last_error("rb200_preprocess: bad argument");
    return RB200_E_INVALID;
  }
  if (rows == 0) return RB200_OK;
  const long long total = rows * (long long)f_out;
  long long blocks = (total + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  preprocess_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(
      input, (const uint8_t*)presence, presence_is_float, rows, f_in, f_out, cols, quantiles, out);
  return check_cuda(cudaGetLastError(), "preprocess_kernel launch");
}
