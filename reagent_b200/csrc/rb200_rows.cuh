// reagent_b200 -- host-side tile configuration shared by the row-tile kernels.
#pragma once
#include <stdio.h>
#include <stdlib.h>

#include <type_traits>

#include "rb200_tile.cuh"

namespace rb200 {

constexpr int kSmemLimit = 227 * 1024;  // H100 opt-in maximum per CTA

struct RowsCfg {
  int nt;      // threads per CTA (256 or 512)
  int tm;      // rows per thread (tile rows R = (nt/64)*tm)
  int kc;      // staged k-chunk
  int ld_in;   // smem stride of the input tile
  int ld_h;    // smem stride of hidden tiles
  size_t smem_bytes;
};

// Pick the largest tile that fits: n_in input buffers of width din, n_h hidden
// buffers of width hmax, plus `extra_per_row` floats per tile row and `extra`
// floats flat.  Returns tm == 0 when nothing fits.
inline RowsCfg pick_rows_cfg(int batch, int din, int hmax, int n_in, int n_h, int extra_per_row,
                             int extra) {
  RowsCfg best{0, 0, 0, 0, 0, 0};
  const int ld_in = round_up4(din) + 4;
  const int ld_h = round_up4(hmax > 0 ? hmax : 4) + 4;
  // (threads, rows/thread, k-chunk): 16 warps per SM hide the LDS->FMA latency of the
  // 4x4 register tile; the 16-row tile serves small batches (more CTAs than SMs).
  const int cand[4][3] = {{512, 4, 32}, {512, 4, 16}, {256, 4, 32}, {256, 4, 16}};
  const char* force = getenv("RB200_FORCE_CFG");  // tuning / profiling only: "nt,kc"
  int fnt = 0, fkc = 0;
  if (force) sscanf(force, "%d,%d", &fnt, &fkc);
  for (int c = 0; c < 4; ++c) {
    const int nt = cand[c][0], tm = cand[c][1], kc = cand[c][2];
    const int R = (nt / 64) * tm;
    if (fnt) { if (nt != fnt || kc != fkc) continue; }
    else if (R == 32 && batch <= 16 * kNumSMs) continue;  // small batch: prefer 16-row tiles
    const size_t stage = (size_t)(kc == 32 ? wstage_floats<32>() : wstage_floats<16>());
    const size_t floats = 2 * stage + (size_t)R * ((size_t)n_in * ld_in + (size_t)n_h * ld_h +
                                                   (size_t)extra_per_row) + (size_t)extra;
    const size_t bytes = floats * sizeof(float);
    if (bytes <= (size_t)kSmemLimit) {
      best = RowsCfg{nt, tm, kc, ld_in, ld_h, bytes};
      break;
    }
  }
  return best;
}

inline int rows_per_tile(const RowsCfg& c) { return (c.nt / 64) * c.tm; }

inline int mlp_max_hidden(const rb200_mlp_t* m) {
  int h = 0;
  for (int l = 1; l < m->n_layers; ++l) h = m->dims[l] > h ? m->dims[l] : h;
  return h;
}

// Calls f(NT, KC) with the tile of `cfg` as std::integral_constant<int, ...> arguments, so that
// a call site instantiates its kernel once per tile of pick_rows_cfg (TM is 4 on every tile).
template <typename F>
inline auto dispatch_rows(const RowsCfg& cfg, F&& f) {
  using std::integral_constant;
  if (cfg.nt == 512 && cfg.kc == 32) return f(integral_constant<int, 512>{}, integral_constant<int, 32>{});
  if (cfg.nt == 512 && cfg.kc == 16) return f(integral_constant<int, 512>{}, integral_constant<int, 16>{});
  if (cfg.nt == 256 && cfg.kc == 32) return f(integral_constant<int, 256>{}, integral_constant<int, 32>{});
  return f(integral_constant<int, 256>{}, integral_constant<int, 16>{});
}

}  // namespace rb200
