// reagent_b200 -- the split-K weight-gradient launch over a list of (input, dZ) products.
// The kernel is rb200_optim.cu's wgrad_kernel; rb200_mlp_wgrad builds its job list from an MLP,
// rb200_mdnrnn_wgrad from the LSTM layers and the mixture head.
#pragma once
#include "rb200_common.cuh"

namespace rb200 {

// dW[n, k] = sum_b dZ[b, n] * A[b, k] into gpart + split * P + w_off, and the column sums of dZ
// into gpart + split * P + b_off (when b_off >= 0)
struct WgradLayer {
  const float* A;   // [B, K] input activations of this product
  const float* dZ;  // [B, N] pre-activation gradients
  int K, N;
  long long w_off, b_off;
  int tiles_n, tiles_k, tile_start;
};

constexpr int kWgradMaxJobs = 9;  // 2 * RB200_MDNRNN_MAX_LAYERS + 1

// Fills the tile bookkeeping of jobs[0..n_jobs) and launches over `rows` batch rows split into
// `splits` fixed slabs (deterministic).  n_jobs <= kWgradMaxJobs.
int wgrad_jobs_launch(WgradLayer* jobs, int n_jobs, int rows, int splits, float* gpart,
                      long long P, cudaStream_t st, const char* what);

}  // namespace rb200
