// Host-only consistency check of the wgmma weight-image layout (rb200_dqn_tc_layout.cuh):
// the element -> offset map used by the Adam kernel (image_elem) must be a bijection onto the
// positions the pack kernel writes (chunk_geo + its in-chunk formula), chunks must not collide,
// and everything must stay inside image_bytes().  Compiled with nvcc, run on the CPU.
#include <cstdio>
#include <cstdlib>
#include <set>
#include <vector>

#include "../../reagent_b200/csrc/rb200_dqn_tc_layout.cuh"

using namespace rb200;

static int check(int N, int K) {
  const uint32_t total = image_bytes(N, K) / 4;  // floats
  std::vector<int> owner(total, -1);
  // positions written by the pack kernel: per (tile, chunk) block, rows8 x kl8 elements
  for (int t = 0; t < ceil_div(N, 128); ++t)
    for (int c = 0; c < ceil_div(K, kQKC); ++c) {
      const ChunkGeo g = chunk_geo(N, K, t, c);
      const int rows8 = (int)(g.lbo - 16) / 16, kl8 = g.ksteps * 8;
      if (g.off + g.bytes > total * 4) { printf("chunk beyond image N=%d K=%d\n", N, K); return 1; }
      for (int m = 0; m < rows8; ++m)
        for (int kk = 0; kk < kl8; ++kk) {
          const uint32_t hi = g.off / 4 + (kk >> 2) * (g.lbo / 4) + m * 4 + (kk & 3);
          if (hi >= total) { printf("oob N=%d K=%d\n", N, K); return 1; }
          if (owner[hi] != -1) { printf("collision N=%d K=%d\n", N, K); return 1; }
          const bool real = 128 * t + m < N && kQKC * c + kk < K;
          owner[hi] = real ? 1 : 0;
        }
    }
  // the Adam-side map hits exactly the "real" positions
  long long real_hi = 0;
  for (uint32_t i = 0; i < total; ++i) real_hi += owner[i] == 1;
  if (real_hi != (long long)N * K) { printf("count N=%d K=%d\n", N, K); return 1; }
  for (int m = 0; m < N; ++m)
    for (int k = 0; k < K; ++k) {
      const uint32_t hi = image_elem(N, K, m, k);
      if (hi >= total || owner[hi] != 1) {
        printf("image_elem mismatch N=%d K=%d m=%d k=%d\n", N, K, m, k);
        return 1;
      }
      owner[hi] = 3;  // each position exactly once
    }
  return 0;
}

int main() {
  const int shapes[][2] = {{256, 128}, {128, 256}, {16, 128}, {128, 16}, {300, 36}, {130, 300},
                           {20, 130}, {9, 20}, {1, 8}, {5, 40}, {40, 7}, {512, 33}, {129, 1}};
  for (auto& s : shapes)
    if (check(s[0], s[1])) return 1;
  // image table of a whole network: consecutive, non-overlapping, same order as make_plan()
  rb200_mlp_t q = {};
  q.n_layers = 3;
  const int dims[] = {128, 256, 128, 16};
  for (int i = 0; i < 4; ++i) q.dims[i] = dims[i];
  const TcImages im = tc_images(&q, 1);
  uint32_t expect = 0;
  for (int l = 0; l < 3; ++l) { if (im.on_fwd[l] != expect) return 2; expect += image_bytes(dims[l + 1], dims[l]); }
  for (int l = 0; l < 3; ++l) { if (im.tg_fwd[l] != expect) return 2; expect += image_bytes(dims[l + 1], dims[l]); }
  for (int l = 1; l < 3; ++l) { if (im.on_bwd[l] != expect) return 2; expect += image_bytes(dims[l], dims[l + 1]); }
  if (im.total_bytes != (int64_t)expect + 4096) return 2;
  printf("ok\n");
  return 0;
}
