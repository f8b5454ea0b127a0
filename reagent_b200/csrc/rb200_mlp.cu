// reagent_b200 -- the generic MLP and Linear-layer kernels over row tiles.
//   mlp_fwd_rows_kernel      whole-MLP forward: the nn.Module.forward of the models in
//                            reagent_b200/models (the reference's FullyConnectedNetwork.forward,
//                            reagent/models/fully_connected_network.py:157-163, and the critic's
//                            cat(state, action) input, reagent/models/critic.py:76-92)
//   mlp_fwd_tiled_kernel     ParametricDQN's max-Q forward over tiled (state, action) rows
//   linear_fwd_wide_kernel   one Linear layer too wide for a row tile (QR-DQN / C51 heads):
//                            row tiles x column blocks; GEMM-sized shapes go to rb200_tc_gemm.cu
//   linear_bwd_wide_kernel   dz_prev = (dz . W) * act'(h_prev) of such a layer
//   mlp_bwd_rows_kernel      dZ chain of the layers below a given last-layer dz, which every
//                            trainer's backward runs before rb200_mlp_wgrad (rb200_optim.cu)
#include "rb200_rows.cuh"

namespace rb200 {

struct FwdDev {
  const float* in0; int d0;   // [B, d0]
  const float* in1; int d1;   // [B, d1] or nullptr (concatenated after in0)
  float* out;                 // [B, dims[L]]
  int batch, ld_in, ld_h, ld_o;
  rb200_net_ws_t ws;
  int save;
};

template <int NT, int TM, int KC>
__global__ void __launch_bounds__(NT, 1) mlp_fwd_rows_kernel(const Mlp net, const FwdDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* xin = Wst + 2 * wstage_floats<KC>();
  float* hA = xin + R * p.ld_in;
  float* hB = hA + R * p.ld_h;
  float* xo = hB + R * p.ld_h;
  const int row0 = blockIdx.x * R;
  // cat(in0, in1): in0 occupies columns [0,d0), in1 columns [d0, d0+d1)
  if (p.in1 == nullptr) {
    tile_load_rows<NT, R>(xin, p.ld_in, p.in0, p.d0, p.d0, row0, p.batch);
  } else {
    const int D = p.d0 + p.d1, D4 = round_up4(D);
    for (int idx = threadIdx.x; idx < R * D4; idx += NT) {
      const int r = idx / D4, c = idx - r * D4;
      float v = 0.f;
      if (row0 + r < p.batch) {
        if (c < p.d0) v = p.in0[(size_t)(row0 + r) * p.d0 + c];
        else if (c < D) v = p.in1[(size_t)(row0 + r) * p.d1 + (c - p.d0)];
      }
      xin[r * p.ld_in + c] = v;
    }
  }
  __syncthreads();
  tile_mlp_fwd<NT, TM, KC>(net, xin, p.ld_in, hA, hB, p.ld_h, xo, p.ld_o, Wst,
                           p.save ? p.ws.hidden : nullptr, row0, p.batch);
  const int DO = net.dims[net.n_layers];
  tile_store_rows<NT, R>(xo, p.ld_o, p.out, DO, DO, row0, p.batch);
}

// Tiled forward of ParametricDQN's max-Q target: row r of the B*M rows is
// cat(state[r / M], actions[r]) (FeatureData.get_tiled_batch + the possible next actions),
// built in shared memory by the loader, so the tiled input never exists in HBM.  Every network
// of the launch (online and target: same dims / act) runs over the SAME input tile.  The tile,
// its shared-memory layout and the grid mapping are those of mlp_fwd_rows_kernel on the
// materialised [B*M, S+K] input, and so are the bits of every output.
struct TiledFwdDev {
  const float* state; int S;     // [B, S]
  const float* actions; int K;   // [B*M, K]
  float* out[2];                 // [B*M, dims[L]] per network
  int n_nets, rows, M;           // rows = B*M
  int ld_in, ld_h, ld_o;
};

template <int NT, int TM, int KC>
__global__ void __launch_bounds__(NT, 1) mlp_fwd_tiled_kernel(const Mlp net0, const Mlp net1,
                                                              const TiledFwdDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* xin = Wst + 2 * wstage_floats<KC>();
  float* hA = xin + R * p.ld_in;
  float* hB = hA + R * p.ld_h;
  float* xo = hB + R * p.ld_h;
  const int row0 = blockIdx.x * R;
  const int D = p.S + p.K, D4 = round_up4(D);
  for (int idx = threadIdx.x; idx < R * D4; idx += NT) {
    const int r = idx / D4, c = idx - r * D4;
    const int gr = row0 + r;
    float v = 0.f;
    if (gr < p.rows) {
      if (c < p.S) v = p.state[(size_t)(gr / p.M) * p.S + c];
      else if (c < D) v = p.actions[(size_t)gr * p.K + (c - p.S)];
    }
    xin[r * p.ld_in + c] = v;
  }
  __syncthreads();
  const int DO = net0.dims[net0.n_layers];
  tile_mlp_fwd<NT, TM, KC>(net0, xin, p.ld_in, hA, hB, p.ld_h, xo, p.ld_o, Wst, nullptr, row0,
                           p.rows);
  tile_store_rows<NT, R>(xo, p.ld_o, p.out[0], DO, DO, row0, p.rows);
  if (p.n_nets < 2) return;
  // the second network starts from the state the first one saw: hidden and output tiles zero
  // (their padding columns feed the MMA against zero weights), the input tile untouched
  __syncthreads();
  for (int i = threadIdx.x; i < R * (2 * p.ld_h + p.ld_o); i += NT) hA[i] = 0.f;
  __syncthreads();
  tile_mlp_fwd<NT, TM, KC>(net1, xin, p.ld_in, hA, hB, p.ld_h, xo, p.ld_o, Wst, nullptr, row0,
                           p.rows);
  tile_store_rows<NT, R>(xo, p.ld_o, p.out[1], DO, DO, row0, p.rows);
}

constexpr int kColBlock = 512;  // head columns per CTA

// ---------------- wide single Linear layer forward: out = act(in . W^T + b) ----------------
struct LinFwdDev {
  const float* in; int K;
  const float* W; const float* b; int N; int act;
  float* out; int batch; int ld_in, ld_o;
};

template <int NT, int TM, int KC>
__global__ void __launch_bounds__(NT, 1) linear_fwd_wide_kernel(const LinFwdDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* xin = Wst + 2 * wstage_floats<KC>();
  float* xo = xin + R * p.ld_in;
  const int row0 = blockIdx.x * R;
  const int c0 = blockIdx.y * kColBlock;
  const int nloc = min(kColBlock, p.N - c0);
  tile_load_rows<NT, R>(xin, p.ld_in, p.in, p.K, p.K, row0, p.batch);
  __syncthreads();
  tile_linear_fwd<NT, TM, KC>(xin, p.ld_in, p.K, p.W + (size_t)c0 * p.K, p.K,
                              p.b ? p.b + c0 : nullptr, nloc, p.act, xo, p.ld_o, Wst);
  tile_store_rows<NT, R>(xo, p.ld_o, p.out + c0, p.N, nloc, row0, p.batch);
}

// -------- wide contraction backward: dz_prev = (dz . W) * act'(h_prev), N large --------
struct LinBwdDev {
  const float* dz; int N;       // [B, N]
  const float* W; int K;        // [N, K]
  const float* h_prev; int act_prev;  // [B, K] output of the previous layer (or nullptr)
  float* out;                   // [B, K]
  int batch, ld_z, ld_k;
};

template <int NT, int TM, int KC>
__global__ void __launch_bounds__(NT, 1) linear_bwd_wide_kernel(const LinBwdDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* zs = Wst + 2 * wstage_floats<KC>();  // [R, ld_z] slab of dz
  float* accb = zs + R * p.ld_z;              // [R, ld_k] running sum
  float* tmp = accb + R * p.ld_k;             // [R, ld_k] per-slab result
  const int row0 = blockIdx.x * R;
  const int K4 = round_up4(p.K);
  for (int idx = threadIdx.x; idx < R * p.ld_k; idx += NT) accb[idx] = 0.f;
  for (int n0 = 0; n0 < p.N; n0 += kColBlock) {
    const int nloc = min(kColBlock, p.N - n0);
    // slab of dz columns [n0, n0+nloc)
    tile_load_rows<NT, R>(zs, p.ld_z, p.dz + n0, p.N, nloc, row0, p.batch);
    __syncthreads();
    tile_linear_bwd<NT, TM, KC>(zs, p.ld_z, nloc, p.W + (size_t)n0 * p.K, p.K, p.K, nullptr, 0, 0,
                                tmp, p.ld_k, Wst);
    for (int idx = threadIdx.x; idx < R * K4; idx += NT) {
      const int r = idx / K4, c = idx - r * K4;
      accb[r * p.ld_k + c] += tmp[r * p.ld_k + c];
    }
    __syncthreads();
  }
  for (int idx = threadIdx.x; idx < R * K4; idx += NT) {
    const int r = idx / K4, c = idx - r * K4;
    const int row = row0 + r;
    if (row < p.batch && c < p.K) {
      float g = accb[r * p.ld_k + c];
      if (p.h_prev) g *= act_bwd_from_out(p.h_prev[(size_t)row * p.K + c], p.act_prev);
      p.out[(size_t)row * p.K + c] = g;
    }
  }
}

// ---------------- whole-MLP backward (dZ chain) from a given last-layer dz ----------------
struct MlpBwdDev {
  const float* dz_last;  // [B, dims[L]] pre-activation gradient of the last layer
  rb200_net_ws_t ws;
  int batch, ld_h, ld_o;
};

template <int NT, int TM, int KC>
__global__ void __launch_bounds__(NT, 1) mlp_bwd_rows_kernel(const Mlp net, const MlpBwdDev p) {
  constexpr int R = (NT / 64) * TM;
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* gA = Wst + 2 * wstage_floats<KC>();
  float* gB = gA + R * p.ld_h;
  float* hb = gB + R * p.ld_h;
  float* zl = hb + R * p.ld_h;
  const int row0 = blockIdx.x * R;
  const int DL = net.dims[net.n_layers];
  tile_load_rows<NT, R>(zl, p.ld_o, p.dz_last, DL, DL, row0, p.batch);
  __syncthreads();
  // dz of the last layer is already in global memory: do not store it again
  rb200_net_ws_t ws = p.ws;
  float* keep = ws.dz[net.n_layers - 1];
  ws.dz[net.n_layers - 1] = nullptr;
  tile_mlp_bwd<NT, TM, KC>(net, zl, p.ld_o, gA, gB, hb, p.ld_h, Wst, ws.hidden, ws.dz, row0,
                           p.batch, nullptr, 0, 0, 0);
  (void)keep;
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_mlp_forward(const rb200_mlp_t* net, const float* in0, int32_t d0,
                                 const float* in1, int32_t d1, int32_t batch, float* out,
                                 const rb200_net_ws_t* save_hidden, void* stream) {
  if (!net || !in0 || !out) { set_last_error("rb200_mlp_forward: null argument"); return RB200_E_INVALID; }
  if (int rc = validate_mlp(net, "net")) return rc;
  if (batch <= 0) { set_last_error("rb200_mlp_forward: batch must be positive"); return RB200_E_INVALID; }
  if (d0 + (in1 ? d1 : 0) != net->dims[0]) {
    set_last_error("rb200_mlp_forward: input width %d != dims[0]=%d", d0 + (in1 ? d1 : 0), net->dims[0]);
    return RB200_E_INVALID;
  }
  FwdDev p;
  p.in0 = in0; p.d0 = d0; p.in1 = in1; p.d1 = in1 ? d1 : 0; p.out = out; p.batch = batch;
  p.save = save_hidden ? 1 : 0;
  if (save_hidden) p.ws = *save_hidden; else p.ws = rb200_net_ws_t{};
  const int DO = net->dims[net->n_layers];
  const int hmax = mlp_max_hidden(net);
  p.ld_o = round_up4(DO) + 4;
  if (p.ld_o > 1024 + 4) { set_last_error("rb200_mlp_forward: output width %d too large for the row-tile kernel", DO); return RB200_E_SMEM; }
  RowsCfg cfg = pick_rows_cfg(batch, net->dims[0], hmax, 1, 2, p.ld_o, 0);
  if (cfg.tm == 0) { set_last_error("rb200_mlp_forward: tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_in = cfg.ld_in; p.ld_h = cfg.ld_h;
  const Mlp m = make_mlp(net);
  const int grid = ceil_div(batch, rows_per_tile(cfg));
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    return launch<mlp_fwd_rows_kernel<NT(), 4, KC()>>(grid, NT(), cfg.smem_bytes, st,
                                                      "mlp_fwd_rows_kernel launch", m, p);
  });
}

extern "C" int rb200_mlp_forward_tiled(const rb200_mlp_t* net0, const rb200_mlp_t* net1,
                                       const float* state, int32_t state_dim,
                                       const float* actions, int32_t action_dim, int32_t batch,
                                       int32_t num_tiled, float* out0, float* out1,
                                       void* stream) {
  if (!net0 || !state || !actions || !out0 || (net1 != nullptr) != (out1 != nullptr)) {
    set_last_error("rb200_mlp_forward_tiled: null argument (net1 and out1 go together)");
    return RB200_E_INVALID;
  }
  if (int rc = validate_mlp(net0, "net0")) return rc;
  if (net1) {
    if (int rc = validate_mlp(net1, "net1")) return rc;
    bool same = net1->n_layers == net0->n_layers;
    for (int l = 0; same && l <= net0->n_layers; ++l) same = net1->dims[l] == net0->dims[l];
    for (int l = 0; same && l < net0->n_layers; ++l) same = net1->act[l] == net0->act[l];
    if (!same) {
      set_last_error("rb200_mlp_forward_tiled: net0 and net1 differ in dims or activations");
      return RB200_E_INVALID;
    }
  }
  if (batch <= 0 || num_tiled <= 0) {
    set_last_error("rb200_mlp_forward_tiled: batch %d and num_tiled %d must be positive", batch,
                   num_tiled);
    return RB200_E_INVALID;
  }
  if ((long long)batch * num_tiled > INT32_MAX) {
    set_last_error("rb200_mlp_forward_tiled: batch * num_tiled = %lld overflows int32",
                   (long long)batch * num_tiled);
    return RB200_E_INVALID;
  }
  if (state_dim <= 0 || action_dim <= 0 || state_dim + action_dim != net0->dims[0]) {
    set_last_error("rb200_mlp_forward_tiled: input width %d + %d != dims[0]=%d", state_dim,
                   action_dim, net0->dims[0]);
    return RB200_E_INVALID;
  }
  const int rows = batch * num_tiled;
  TiledFwdDev p;
  p.state = state; p.S = state_dim; p.actions = actions; p.K = action_dim;
  p.out[0] = out0; p.out[1] = out1; p.n_nets = net1 ? 2 : 1;
  p.rows = rows; p.M = num_tiled;
  const int DO = net0->dims[net0->n_layers];
  const int hmax = mlp_max_hidden(net0);
  p.ld_o = round_up4(DO) + 4;
  if (p.ld_o > 1024 + 4) { set_last_error("rb200_mlp_forward_tiled: output width %d too large for the row-tile kernel", DO); return RB200_E_SMEM; }
  // the tile of rb200_mlp_forward on the materialised [rows, S+K] input: the k-chunk rotation
  // of tile_linear_fwd depends on the tile and the CTA, so this keeps every output bit-equal
  RowsCfg cfg = pick_rows_cfg(rows, net0->dims[0], hmax, 1, 2, p.ld_o, 0);
  if (cfg.tm == 0) { set_last_error("rb200_mlp_forward_tiled: tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_in = cfg.ld_in; p.ld_h = cfg.ld_h;
  const Mlp m0 = make_mlp(net0);
  const Mlp m1 = make_mlp(net1 ? net1 : net0);
  const int grid = ceil_div(rows, rows_per_tile(cfg));
  cudaStream_t st = (cudaStream_t)stream;
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    return launch<mlp_fwd_tiled_kernel<NT(), 4, KC()>>(grid, NT(), cfg.smem_bytes, st,
                                                       "mlp_fwd_tiled_kernel launch", m0, m1, p);
  });
}

extern "C" int rb200_linear_forward_tc(const float* W, const float* b, int32_t act, int32_t K,
                                       int32_t N, const float* in, int32_t batch, float* out,
                                       void* stream);

extern "C" int rb200_linear_forward(const float* W, const float* b, int32_t act, int32_t K,
                                    int32_t N, const float* in, int32_t batch, float* out,
                                    void* stream) {
  if (!W || !in || !out || K <= 0 || N <= 0 || batch <= 0) { set_last_error("rb200_linear_forward: bad argument"); return RB200_E_INVALID; }
  // GEMM-shaped problems (>= one full 128x128 tile) go to the wgmma kernel
  if (batch >= 128 && N >= 128) return rb200_linear_forward_tc(W, b, act, K, N, in, batch, out, stream);
  LinFwdDev p{in, K, W, b, N, act, out, batch, 0, kColBlock + 4};
  RowsCfg cfg = pick_rows_cfg(batch, K, 4, 1, 0, p.ld_o, 0);
  if (cfg.tm == 0) { set_last_error("rb200_linear_forward: tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_in = cfg.ld_in;
  dim3 grid(ceil_div(batch, rows_per_tile(cfg)), ceil_div(N, kColBlock));
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    return launch<linear_fwd_wide_kernel<NT(), 4, KC()>>(grid, NT(), cfg.smem_bytes, (cudaStream_t)stream,
                                                         "linear_fwd_wide_kernel launch", p);
  });
}

extern "C" int rb200_linear_backward_dx(const float* W, int32_t K, int32_t N, const float* dz,
                                        const float* h_prev, int32_t act_prev, int32_t batch,
                                        float* out, void* stream) {
  if (!W || !dz || !out || K <= 0 || N <= 0 || batch <= 0) { set_last_error("rb200_linear_backward_dx: bad argument"); return RB200_E_INVALID; }
  LinBwdDev p{dz, N, W, K, h_prev, act_prev, out, batch, kColBlock + 4, round_up4(K) + 4};
  RowsCfg cfg = pick_rows_cfg(batch, kColBlock, 4, 1, 0, 2 * p.ld_k, 0);
  if (cfg.tm == 0) { set_last_error("rb200_linear_backward_dx: tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_z = cfg.ld_in;
  dim3 grid(ceil_div(batch, rows_per_tile(cfg)));
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    return launch<linear_bwd_wide_kernel<NT(), 4, KC()>>(grid, NT(), cfg.smem_bytes, (cudaStream_t)stream,
                                                         "linear_bwd_wide_kernel launch", p);
  });
}

extern "C" int rb200_mlp_backward(const rb200_mlp_t* net, const float* dz_last, int32_t batch,
                                  const rb200_net_ws_t* ws, void* stream) {
  if (!net || !dz_last || !ws || batch <= 0) { set_last_error("rb200_mlp_backward: bad argument"); return RB200_E_INVALID; }
  if (int rc = validate_mlp(net, "net")) return rc;
  if (net->n_layers < 2) return RB200_OK;  // nothing below the last layer
  MlpBwdDev p;
  p.dz_last = dz_last;
  p.ws = *ws;
  p.batch = batch;
  const int DL = net->dims[net->n_layers];
  p.ld_o = round_up4(DL) + 4;
  RowsCfg cfg = pick_rows_cfg(batch, 4, mlp_max_hidden(net), 0, 3, p.ld_o, 0);
  if (cfg.tm == 0) { set_last_error("rb200_mlp_backward: tile does not fit in shared memory"); return RB200_E_SMEM; }
  p.ld_h = cfg.ld_h;
  const Mlp m = make_mlp(net);
  dim3 grid(ceil_div(batch, rows_per_tile(cfg)));
  return dispatch_rows(cfg, [&](auto NT, auto KC) {
    return launch<mlp_bwd_rows_kernel<NT(), 4, KC()>>(grid, NT(), cfg.smem_bytes, (cudaStream_t)stream,
                                                      "mlp_bwd_rows_kernel launch", m, p);
  });
}
