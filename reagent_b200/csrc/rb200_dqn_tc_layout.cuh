// reagent_b200 -- layout of the packed weight images of the wgmma TD kernel
// (rb200_dqn_tc.cu), shared with the Adam kernel, which can write the images of the updated
// parameters itself (rb200_optim.cu) instead of a separate packing launch.
//
// Image of an operand A[N rows x K] (N = output features, K = contraction): for every
// (128-row tile t, kQKC-wide k chunk c) one block of fp32 values laid out [k/4][row][4 floats]
// with the k-quad stride (LBO) padded by 16 B, so that (a) one 1-D bulk copy moves a whole
// chunk and (b) the TD kernel reads its wgmma A fragments (rows g / g+8, k t / t+4 of a
// warp's 16 x 8 slice) as conflict-free 4-byte shared-memory loads.  The TF32 hi/lo split
// happens in the TD kernel on the way into registers (the A operand of the MMAs), so the image
// holds every parameter ONCE.
// Rows / k past the matrix are zero (the buffer is zero-initialised once and those positions
// are never written).
#pragma once
#include "rb200_common.cuh"

namespace rb200 {

constexpr int kQKC = 32;                                  // contraction elements per weight chunk
constexpr int kQFullLbo = 128 * 16 + 16;                  // A quad stride of a full 128-row tile

__host__ __device__ __forceinline__ int round_up8(int x) { return (x + 7) & ~7; }

struct ChunkGeo {
  uint32_t off, bytes, lbo;
  int ksteps, k0q;
};
// geometry of chunk (feature tile t, k chunk c) inside the image of an [N x K] operand
__host__ __device__ __forceinline__ ChunkGeo chunk_geo(int N, int K, int t, int c) {
  ChunkGeo g;
  const int rows = N - 128 * t;
  const int rows8 = round_up8(rows < 128 ? rows : 128);
  g.lbo = (uint32_t)(rows8 * 16 + 16);
  const int kl = K - kQKC * c;
  const int kl8 = round_up8(kl < kQKC ? kl : kQKC);
  g.bytes = (uint32_t)(kl8 / 4) * g.lbo;
  g.off = (uint32_t)t * ((uint32_t)(round_up8(K) / 4) * kQFullLbo) +
          (uint32_t)c * ((kQKC / 4) * g.lbo);
  g.ksteps = kl8 / 8;
  g.k0q = c * (kQKC / 4);
  return g;
}
inline uint32_t image_bytes(int N, int K) {
  uint32_t tot = 0;
  for (int t = 0; t < ceil_div(N, 128); ++t) {
    const int rows = N - 128 * t;
    const int rows8 = round_up8(rows < 128 ? rows : 128);
    tot += (uint32_t)(round_up8(K) / 4) * (uint32_t)(rows8 * 16 + 16);
  }
  return tot;
}

// float offset of element (m, k) of an [N x K] operand inside its image
__host__ __device__ __forceinline__ uint32_t image_elem(int N, int K, int m, int k) {
  const int t = m >> 7, c = k / kQKC;
  const ChunkGeo g = chunk_geo(N, K, t, c);
  const int r = m & 127, kk = k - c * kQKC;
  return g.off / 4 + (uint32_t)((kk >> 2) * (int)(g.lbo / 4) + r * 4 + (kk & 3));
}

// Where the images of one Q-network pair live in the pack buffer (byte offsets); the order is
// the one make_plan() in rb200_dqn_tc.cu streams them in.
struct TcImages {
  int n_layers;
  int dims[kMaxLayers + 1];
  uint32_t on_fwd[kMaxLayers], tg_fwd[kMaxLayers], on_bwd[kMaxLayers];  // on_bwd[0] unused
  int has_bwd;
  int64_t total_bytes;
};
inline TcImages tc_images(const rb200_mlp_t* q, int do_backward) {
  TcImages im = {};
  im.n_layers = q->n_layers;
  for (int l = 0; l <= kMaxLayers; ++l) im.dims[l] = l <= q->n_layers ? q->dims[l] : 0;
  uint32_t off = 0;
  for (int l = 0; l < q->n_layers; ++l) { im.on_fwd[l] = off; off += image_bytes(q->dims[l + 1], q->dims[l]); }
  for (int l = 0; l < q->n_layers; ++l) { im.tg_fwd[l] = off; off += image_bytes(q->dims[l + 1], q->dims[l]); }
  im.has_bwd = do_backward ? 1 : 0;
  im.on_bwd[0] = 0;
  for (int l = 1; l < q->n_layers; ++l) {
    im.on_bwd[l] = off;
    if (do_backward) off += image_bytes(q->dims[l], q->dims[l + 1]);
  }
  im.total_bytes = (int64_t)off + 4096;  // slack: partial tiles are over-read by design (in smem only)
  return im;
}

// device view used by the Adam kernel to write the images of the parameters it updates
struct TcPackView {
  int n_layers;
  int dims[kMaxLayers + 1];
  long long w_off[kMaxLayers];
  uint32_t on_fwd[kMaxLayers], tg_fwd[kMaxLayers], on_bwd[kMaxLayers];
  int has_bwd;
  float* pack;  // nullptr: no packing
};

}  // namespace rb200
