// reagent_b200 -- K2 on the Hopper tensor cores: the fused DQN TD-target / loss / backward step
// (same contract as rb200_dqn.cu) with every matrix product issued as warpgroup MMAs (wgmma,
// kind tf32, 3xTF32 error compensation) and the accumulators in registers.
//
// Formulation.  A CTA owns 32 batch rows and computes every layer TRANSPOSED:
//     D_l^T [features x 32 rows]  =  W_l [features x K]  .  H_{l-1}^T [K x 32 rows]
// so the WEIGHTS are the wgmma A operand (M = 64 output features per warpgroup, always a full
// tensor-core tile however small the batch tile is) and the ACTIVATIONS are the B operand
// (N = 32).  4096 rows therefore spread over 128 SMs instead of the 32 an M = 64-row tile
// would use, and the accumulator of a 64-feature slice is only 32 registers per thread.
//
//   weights      pre-tiled once per update (by the Adam kernel, or dqn_tc_pack_kernel) into one
//                fp32 image per (128-feature tile, 32-k chunk) -- [k/4][row][4 floats].  The TD
//                kernel streams the images through a shared-memory ring with 1-D bulk copies
//                (cp.async.bulk -> mbarrier complete_tx, one producer warp; a stage = two chunk
//                images).  The two MMA warpgroups read their A fragments straight from the
//                ring (conflict-free 4-byte loads), split them into TF32 hi / lo in registers
//                and issue the MMAs with A FROM REGISTERS: every weight byte crosses shared
//                memory once in and once out as raw fp32.  The MMAs of a 32-k chunk go out as
//                one chain while the next chunk's fragments are read and split.
//   activations  live in shared memory as hi/lo planes in the canonical K-major layout (rows =
//                batch rows); the epilogue of layer l (registers -> bias -> activation -> split)
//                writes them straight into the B operand of layer l+1 and, for the online
//                pass on `state`, to the global buffers the weight-gradient kernel reads.
//   backward     dZ_{l-1}^T = W_l^T . dZ_l^T uses pre-transposed weight images; the epilogue
//                multiplies by act'(h_{l-1}) and stores dZ_{l-1}.
//
// Warps 0-7 (two warpgroups; warpgroup g owns features [64 g, 64 g + 64) of every 128-feature
// tile) issue the MMAs and run the epilogues and the loss; warp 8 streams the weights.  Ring
// synchronisation is mbarrier-only:
//     full[s]   bulk copy landed in smem stage s     sfree[s]  the eight MMA warps have read it
// and the hand-over of an activation operand between layers is a named barrier of warps 0-7.
//
// Reference semantics: reagent/training/dqn_trainer.py:157-239, dqn_trainer_base.py:33-77,
// 216-241 (see rb200_dqn.cu for the line-by-line map; the loss code is the same).
#include <string.h>

#include <type_traits>

#include "rb200_dqn_tc_layout.cuh"
#include "rb200_wgmma.cuh"

namespace rb200 {

constexpr int kQR = 32;                                   // batch rows per CTA
// A ring stage holds kQSub consecutive 32-k chunk images of one feature tile (they are
// contiguous in the image: the k-quad sequence simply continues).  Each mbarrier hand-over has
// a fixed cost, so the stage is the unit that amortises it.
constexpr int kQSub = 2;
constexpr int kQStages = 3;                               // shared-memory ring depth
constexpr int kQStageBytes = kQSub * (kQKC / 4) * kQFullLbo;  // kQSub chunk images
// B operand (activations): per k quad 64 rows of 16 B -- rows 0-31 hold the hi parts of the 32
// batch rows, rows 32-63 their lo parts -- plus 16 B of padding.  One N = 64 MMA against W_hi
// then yields W_hi.X_hi in accumulator columns 0-31 and W_hi.X_lo in columns 32-63; a second
// N = 32 MMA adds W_lo.X_hi to columns 0-31.  Two MMAs per k step instead of three, and the
// epilogue adds the two column groups.
constexpr int kQLboB = 64 * 16 + 16;
constexpr int kQLoOff = 32 * 4;                           // floats from a hi element to its lo
constexpr int kQEpiThreads = 256;                         // the two MMA / epilogue warpgroups
constexpr int kQThreads = kQEpiThreads + 32;              // + the producer warp
constexpr int kQMaxTiles = 4;                             // widest layer: 4 x 128 features
constexpr int kQMaxSteps = 4 * kMaxLayers;
constexpr int kQMaxSmem = 232448;                         // 227 KB opt-in limit of sm_90
static_assert(kQKC == 32, "a chunk is four K = 8 MMA steps");

enum { kStepHidden = 0, kStepLast = 1, kStepBwd = 2 };

struct QStep {
  uint32_t pack_off;  // byte offset of the weight image in the pack buffer
  int16_t N, K;       // A-operand rows (output features) and contraction length
  int8_t layer, kind, net, in_buf, load_x, save, qdst, out_buf;
};

struct QDev {
  rb200_dqn_args_t a;
  rb200_net_ws_t ws;
  const unsigned char* pack;
  int nsteps, last_fwd_step;
  int buf_off[3];  // operand buffers (bytes from the smem base); [2] holds dZ of the last layer
  int q_off, ldq, lin_off, bar_off;
  int need_zero;    // some layer width is not a multiple of 8: clear the operand buffers first
  QStep steps[kQMaxSteps];
};

// ---------------------------------------------------------------------------
// weight packing: fp32 arena -> tiled chunk images
// ---------------------------------------------------------------------------
struct PackJob {
  const float* W;   // nn.Linear weight [rows_src x ld]
  int N, K;         // operand rows / contraction length (after the optional transpose)
  int ld;           // source row stride
  int transpose;    // 0: A[m][k] = W[m][k]; 1: A[m][k] = W[k][m]
  uint32_t pack_off;
  int chunk0;       // index of this job's first chunk in the grid
};
struct PackDev {
  PackJob jobs[3 * kMaxLayers];
  int njobs;
  unsigned char* pack;
};

constexpr int kPackParts = 4;  // blocks per chunk: one round of loads per thread at KC = 32

__global__ void __launch_bounds__(256) dqn_tc_pack_kernel(const PackDev p) {
  const int chunk = (int)blockIdx.x / kPackParts, part = (int)blockIdx.x % kPackParts;
  int j = 0;
  while (j + 1 < p.njobs && chunk >= p.jobs[j + 1].chunk0) ++j;
  const PackJob job = p.jobs[j];
  const int local = chunk - job.chunk0;
  const int kch = ceil_div(job.K, kQKC);
  const int t = local / kch, c = local - t * kch;
  const ChunkGeo g = chunk_geo(job.N, job.K, t, c);
  const int rows8 = (int)(g.lbo - 16) / 16, kl8 = g.ksteps * 8;
  float* img = reinterpret_cast<float*>(p.pack + job.pack_off + g.off);
  const int m0 = 128 * t, k0 = kQKC * c;
  const int total = rows8 * kl8;
  constexpr int U = 4;
  for (int base = (part * 256 + (int)threadIdx.x); base < total; base += kPackParts * 256 * U) {
    float v[U];
    int o[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int idx = base + u * kPackParts * 256;
      int m, kk;
      if (job.transpose) { kk = idx / rows8; m = idx - kk * rows8; }
      else { m = idx / kl8; kk = idx - m * kl8; }
      v[u] = 0.f;
      o[u] = -1;
      if (idx < total) {
        o[u] = (kk >> 2) * (int)(g.lbo / 4) + m * 4 + (kk & 3);
        if (m0 + m < job.N && k0 + kk < job.K)
          v[u] = job.transpose ? __ldg(job.W + (size_t)(k0 + kk) * job.ld + m0 + m)
                               : __ldg(job.W + (size_t)(m0 + m) * job.ld + k0 + kk);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (o[u] >= 0) img[o[u]] = v[u];
  }
}

// ---------------------------------------------------------------------------
// the TD kernel
// ---------------------------------------------------------------------------
// activations other than ReLU / linear go through out-of-line calls so that the unrolled
// epilogues stay small enough for the instruction cache
__device__ __noinline__ float act_fwd_slow(float x, int act) { return act_fwd(x, act); }
__device__ __noinline__ float act_bwd_slow(float y, int act) { return act_bwd_from_out(y, act); }

constexpr int kQCK = kQKC / 8;  // K = 8 MMA steps in a chunk

// The MMAs of one chunk of NK k steps, issued as one chain: one fence, per k step
// W_hi . [X_hi | X_lo] then W_lo . X_hi into the same accumulators, in k order, one commit.
// b0 is the shared-memory address of the chunk's first k quad in the B operand.
template <int NK>
__device__ __forceinline__ void chunk_mma(float (&acc)[32], const uint32_t (&ah)[kQCK][4],
                                          const uint32_t (&al)[kQCK][4], uint32_t b0) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < NK; ++kk) {
    const uint64_t bd = wgmma_desc(b0 + (uint32_t)(2 * kk) * kQLboB, kQLboB, 128);
    wgmma_rs_n64(acc, ah[kk], bd, 1u);  // W_hi . [X_hi | X_lo]
    wgmma_rs_n32(acc, al[kk], bd, 1u);  // W_lo . X_hi
  }
  wgmma_commit();
}
// f(std::integral_constant<int, nk>()) for a run-time nk in [1, NK]
template <int NK, typename F>
__device__ __forceinline__ void with_ksteps(int nk, F&& f) {
  if (nk == NK) f(std::integral_constant<int, NK>());
  else if constexpr (NK > 1) with_ksteps<NK - 1>(nk, f);
}

// kWeighted: prioritized-replay importance weights (a.sample_weight), a separate instantiation so
// that the unweighted kernel stays exactly as it is
template <bool kWeighted>
__global__ void __launch_bounds__(kQThreads, 1)
dqn_td_tc_kernel(const Mlp q, const Mlp qt, const QDev p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const rb200_dqn_args_t& a = p.a;
  const int B = a.batch;
  const int row0 = blockIdx.x * kQR;
  const int L = q.n_layers;
  const int A = q.dims[L];

  // operand padding (k up to the next multiple of 8) must be finite.  With every layer width a
  // multiple of 8 there is no padding: all operand quads, all 64 B-operand rows (rows past the
  // batch are stored as zeros) and the loss inputs are fully written before they are read, and
  // the ~115 KB clear (about 1 us per CTA) is skipped.
  if (p.need_zero) {
    unsigned nbytes;
    asm("mov.u32 %0, %%dynamic_smem_size;" : "=r"(nbytes));
    // (the weight ring is fully overwritten by the bulk copies; fragment rows past a partial
    // tile are read as zeros)
    for (unsigned i = (unsigned)p.buf_off[0] + tid * 16u; i + 15u < nbytes; i += kQThreads * 16u)
      *reinterpret_cast<float4*>(smem_raw + i) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();

  unsigned char* ring = smem_raw;
  float* qarr = reinterpret_cast<float*>(smem_raw + p.q_off);  // [3][kQR][ldq]: q(s') online, target, q(s)
  float* act_s = reinterpret_cast<float*>(smem_raw + p.lin_off);  // [kQR][A] action weights
  float* mask_s = act_s + kQR * A;                                // [kQR][A] next-action mask
  float* scal_s = mask_s + kQR * A;                               // [kQR][4] reward, not_terminal, discount src
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + p.bar_off);
  uint64_t* sfree = full + kQStages;
  const int ldq = p.ldq;

  if (tid == 0) {
    for (int s = 0; s < kQStages; ++s) { mbar_init(full + s, 1); mbar_init(sfree + s, kQEpiThreads / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncthreads();

  // warp-uniform role index (the shuffle lets the compiler keep the role loops in uniform registers)
  const int role = __shfl_sync(0xffffffffu, warp, 0);
  if (role == kQEpiThreads / 32) {
    // =====================  weight producer warp (bulk copies)  =====================
    // Free-running over the static chunk list; the `sfree` barriers of the ring are the only
    // back-pressure, so up to kQStages stages are in flight ahead of the MMA warps.
    const bool leader = elect_one();
    int stage = 0;
    uint32_t par = 1;  // parity of the PREVIOUS use of `stage` (first lap: passes immediately)
    for (int s = 0; s < p.nsteps; ++s) {
      const QStep st = p.steps[s];
      const int mt = ceil_div(st.N, 128), kch = ceil_div(st.K, kQKC);
      const uint32_t tile_stride = (uint32_t)(round_up8(st.K) / 4) * kQFullLbo;
      for (int t = 0; t < mt; ++t) {
        const int rows = st.N - 128 * t;
        const uint32_t lbo = (uint32_t)(round_up8(rows < 128 ? rows : 128) * 16 + 16);
        const uint32_t full_bytes = (kQKC / 4) * lbo;
        const int klast = st.K - kQKC * (kch - 1);
        const uint32_t last_bytes = (uint32_t)(round_up8(klast) / 4) * lbo;
        const unsigned char* src = p.pack + st.pack_off + (size_t)t * tile_stride;
        for (int c = 0; c < kch; c += kQSub) {
          const int nsub = kch - c < kQSub ? kch - c : kQSub;
          const uint32_t bytes = (uint32_t)(nsub - 1) * full_bytes + ((c + nsub == kch) ? last_bytes : full_bytes);
          mbar_wait(sfree + stage, par);
          if (leader) {
            mbar_expect_tx(full + stage, bytes);
            bulk_g2s(ring + stage * kQStageBytes, src, bytes, full + stage);
          }
          src += bytes;
          if (++stage == kQStages) { stage = 0; par ^= 1u; }
        }
      }
    }
  } else {
    // =====================  MMA / epilogue warpgroups  =====================
    const int wg = warp >> 2, w4 = warp & 3, g = lane >> 2, tq = lane & 3;
    int ss = 0;
    uint32_t spar = 0;  // ring position (every MMA warp walks the whole chunk sequence)

    // The input tile of a pass: global -> registers (x_fetch, issued early so that the load
    // latency hides behind the previous layer) -> hi/lo split -> B operand (x_store).
    constexpr int kXQ = 4;  // float4 pieces per thread held in flight (covers S <= 128)
    const int xS = q.dims[0];
    const int xnq = round_up8(xS) / 4;
    const bool x_in_regs = kQR * xnq <= kXQ * kQEpiThreads;
    float4 xr[kXQ];
    auto x_fetch_one = [&](const float* src, int idx) {
      const bool vec = ((xS & 3) == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
      const int r = idx / xnq, qd = idx - r * xnq;
      const int k = 4 * qd, row = row0 + r;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < kQR * xnq && row < B) {
        const float* sp = src + (size_t)row * xS;
        if (vec && k + 3 < xS) {
          // volatile: keep the load HERE (the compiler would sink it next to its use)
          asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];\n"
                       : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                       : "l"(sp + k));
        } else {
          if (k < xS) v.x = sp[k];
          if (k + 1 < xS) v.y = sp[k + 1];
          if (k + 2 < xS) v.z = sp[k + 2];
          if (k + 3 < xS) v.w = sp[k + 3];
        }
      }
      return v;
    };
    auto x_store_one = [&](int idx, const float4 v) {
      if (idx >= kQR * xnq) return;
      float* base = reinterpret_cast<float*>(smem_raw + p.buf_off[0]);
      const int r = idx / xnq, qd = idx - r * xnq;
      float4 h, l;
      split_tf32(v, h, l);
      const int o = qd * (kQLboB / 4) + r * 4;
      *reinterpret_cast<float4*>(base + o) = h;
      *reinterpret_cast<float4*>(base + o + kQLoOff) = l;
    };
    auto x_fetch = [&](const float* src) {
      if (!x_in_regs) return;
#pragma unroll
      for (int i = 0; i < kXQ; ++i) xr[i] = x_fetch_one(src, tid + i * kQEpiThreads);
    };
    auto x_store = [&](const float* src) {
      if (x_in_regs) {
#pragma unroll
        for (int i = 0; i < kXQ; ++i) x_store_one(tid + i * kQEpiThreads, xr[i]);
      } else {
        for (int idx = tid; idx < kQR * xnq; idx += kQEpiThreads) x_store_one(idx, x_fetch_one(src, idx));
      }
    };
    // per-row inputs of the loss, staged while the first layers run
    auto load_loss_inputs = [&]() {
      const float* mask = a.maxq ? a.possible_next_actions_mask : a.next_action;
      for (int idx = tid; idx < kQR * A; idx += kQEpiThreads) {
        const int r = idx / A;
        const bool in = row0 + r < B;
        const size_t g = (size_t)row0 * A + idx;
        act_s[idx] = in ? a.action[g] : 0.f;
        mask_s[idx] = (in && mask) ? mask[g] : 1.f;
      }
      if (tid < kQR) {
        const int row = row0 + tid;
        const bool in = row < B;
        scal_s[tid * 4 + 0] = in ? a.reward[row] : 0.f;
        scal_s[tid * 4 + 1] = in ? a.not_terminal[row] : 0.f;
        scal_s[tid * 4 + 2] = (in && a.discount_mode == RB200_DISCOUNT_POW) ? a.discount_src[row] : 0.f;
      }
    };
    // One step (layer): per 128-feature tile, warpgroup wg accumulates features
    // [128 t + 64 wg, +64) x 64 columns (32 batch rows hi, then lo) over the weight stream, then
    // its epilogue writes them out.  The thread holds features n and n + 8 (n = 128 t + 64 wg +
    // 16 w4 + g) of batch rows 8 i + 2 tq + e (i < 4, e < 2), in acc[4 i + 2 h + e] (+ the lo
    // column group acc[4 (i + 4) + 2 h + e]).
    auto step_tiles = [&](const QStep& st) {
      const Mlp& net = st.net ? qt : q;
      const int l = st.layer, N = st.N;
      const int mt = ceil_div(N, 128), kch = ceil_div(st.K, kQKC);
      float* obase = reinterpret_cast<float*>(smem_raw + p.buf_off[st.out_buf]);
      const uint32_t bbase = smem_u32(smem_raw + p.buf_off[st.in_buf]);
      for (int t = 0; t < mt; ++t) {
        const int rows = N - 128 * t;
        const int rows8 = round_up8(rows < 128 ? rows : 128);
        const uint32_t lbo = (uint32_t)(rows8 * 16 + 16);
        const bool live = 64 * wg < rows;  // warpgroup-uniform: this half of the tile has features
        const int m0 = 64 * wg + 16 * w4 + g;
        const bool ok0 = live && m0 < rows8, ok1 = live && m0 + 8 < rows8;
        float acc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          acc[i] = 0.f;
          wgmma_fence_operand(acc[i]);
        }
        // The MMAs are issued a chunk (kQCK k steps, 8 MMAs) at a time, each chunk as one
        // unbroken chain, and the next chunk's A fragments are read and split while that chain
        // runs.  Chunk c is chunk c % 2 of its ring stage and uses fragment buffer c % 2; wait<1>
        // before a read retires the chain that last used the buffer it overwrites.  Buffers of
        // a whole stage (2 x 64 registers) do not fit: with 9 warps, 3 share an SM
        // sub-partition's 64 KB register file, which caps the kernel at 168 registers per
        // thread.  A short last chunk (K not a multiple of 32) is issued after the others have
        // retired: inside the loop, its extra code paths make ptxas serialise all the MMAs of the
        // kernel (notes C7512 / C7513).
        static_assert(kQSub == 2, "one fragment buffer per chunk of a ring stage");
        const int kfull = st.K / kQKC;                            // chunks of kQCK k steps
        const int nk_last = round_up8(st.K - kQKC * kfull) / 8;  // k steps of a short last chunk
        uint32_t ah[2][kQCK][4], al[2][kQCK][4];
        // A fragments of chunk c: raw fp32 from the ring (k steps past nk and rows past the tile
        // read as zeros), the ring stage released once both its chunks are in registers, then
        // TF32 hi / lo, every register final before the chunk's MMAs are issued
        auto fetch = [&](uint32_t (&fh)[kQCK][4], uint32_t (&fl)[kQCK][4], int c, int nk) {
          if (c % 2 == 0) mbar_wait(full + ss, spar);
          float v[kQCK][4];
#pragma unroll
          for (int kk = 0; kk < kQCK; ++kk) {
            v[kk][0] = v[kk][1] = v[kk][2] = v[kk][3] = 0.f;
            const unsigned char* s0 = ring + ss * kQStageBytes + (uint32_t)((c % 2) * (kQKC / 4) + 2 * kk) * lbo + tq * 4;  // k = 8 kk + tq
            const unsigned char* s1 = s0 + lbo;                                                                         // k = 8 kk + 4 + tq
            if (kk < nk && ok0) { v[kk][0] = *reinterpret_cast<const float*>(s0 + m0 * 16); v[kk][2] = *reinterpret_cast<const float*>(s1 + m0 * 16); }
            if (kk < nk && ok1) { v[kk][1] = *reinterpret_cast<const float*>(s0 + (m0 + 8) * 16); v[kk][3] = *reinterpret_cast<const float*>(s1 + (m0 + 8) * 16); }
          }
          if (c % 2 == 1 || c + 1 == kch) {
            // the stage's values are in registers: the ring stage can be refilled
            __syncwarp();
            if (lane == 0) mbar_arrive(sfree + ss);
            if (++ss == kQStages) { ss = 0; spar ^= 1u; }
          }
#pragma unroll
          for (int kk = 0; kk < kQCK; ++kk)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              split_tf32(v[kk][e], fh[kk][e], fl[kk][e]);
              wgmma_fence_operand(fh[kk][e]);
              wgmma_fence_operand(fl[kk][e]);
            }
        };
        auto b_of = [&](int c) { return bbase + (uint32_t)(2 * kQCK * c) * kQLboB; };
        // (a warpgroup without features in this tile multiplies zeros: issuing unconditionally
        // keeps the MMAs out of divergent code, which the compiler would serialise)
        if (kfull > 0) fetch(ah[0], al[0], 0, kQCK);
        for (int c = 0; c < kfull; c += 2) {
          chunk_mma<kQCK>(acc, ah[0], al[0], b_of(c));
          if (c + 1 == kfull) break;
          wgmma_wait<1>();  // chunk c - 1 retired: buffer 1 is free
          fetch(ah[1], al[1], c + 1, kQCK);
          chunk_mma<kQCK>(acc, ah[1], al[1], b_of(c + 1));
          if (c + 2 == kfull) break;
          wgmma_wait<1>();  // chunk c retired: buffer 0 is free
          fetch(ah[0], al[0], c + 2, kQCK);
        }
        if (kfull < kch) {
          // the short last chunk: its k-step count is a template argument, so no branch either
          wgmma_wait<0>();
          fetch(ah[0], al[0], kfull, nk_last);
          with_ksteps<kQCK>(nk_last, [&](auto nk_c) {
            chunk_mma<decltype(nk_c)::value>(acc, ah[0], al[0], b_of(kfull));
          });
        }
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < 32; ++i) wgmma_fence_operand(acc[i]);
        if (!live) continue;

        // ---- epilogue of this tile ----
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int n = 128 * t + m0 + 8 * hh;
          const bool valid = n < N;
          float x[8];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int e = 0; e < 2; ++e) x[2 * i + e] = acc[4 * i + 2 * hh + e] + acc[4 * (i + 4) + 2 * hh + e];
          auto rowof = [&](int k) { return 8 * (k >> 1) + 2 * tq + (k & 1); };
          float* ob = obase + (n >> 2) * (kQLboB / 4) + (n & 3);  // + 4 r for batch row r
          bool to_operand, to_global;
          float* gdst = nullptr;
          if (st.kind == kStepBwd) {
            // act'(h_{l-1}) from the forward operand still resident in shared memory (h = hi + lo
            // exactly); dZ_{l-1} then replaces it in place as the next B operand
            const int hact = q.act[l - 1];
            // st.save: the shared-memory copy of h_{l-1} was overwritten by a later forward layer
            // (networks with >= 3 hidden layers ping-pong over the same two buffers); read the
            // copy saved for the weight-gradient kernel instead
            float hv[8];
            if (st.save) {
              const float* hs = p.ws.hidden[l - 1];
#pragma unroll
              for (int k = 0; k < 8; ++k) {
                const int row = row0 + rowof(k);
                hv[k] = (valid && row < B) ? hs[(size_t)row * N + n] : 0.f;
              }
            } else {
#pragma unroll
              for (int k = 0; k < 8; ++k) hv[k] = valid ? ob[rowof(k) * 4] + ob[rowof(k) * 4 + kQLoOff] : 0.f;
            }
            if (hact == RB200_ACT_RELU) {
#pragma unroll
              for (int k = 0; k < 8; ++k) x[k] = hv[k] > 0.f ? x[k] : 0.f;
            } else if (hact != RB200_ACT_LINEAR) {
#pragma unroll
              for (int k = 0; k < 8; ++k) x[k] = valid ? x[k] * act_bwd_slow(hv[k], hact) : 0.f;
            }
            to_operand = l - 1 >= 1;
            to_global = true;
            gdst = p.ws.dz[l - 1];
          } else {
            const float bias = valid ? __ldg(net.params + net.b_off[l] + n) : 0.f;
            const int act = net.act[l];
            if (act == RB200_ACT_RELU) {
#pragma unroll
              for (int k = 0; k < 8; ++k) x[k] = fmaxf(x[k] + bias, 0.f);
            } else if (act == RB200_ACT_LINEAR) {
#pragma unroll
              for (int k = 0; k < 8; ++k) x[k] += bias;
            } else {
#pragma unroll
              for (int k = 0; k < 8; ++k) x[k] = act_fwd_slow(x[k] + bias, act);
            }
            to_operand = st.kind != kStepLast;
            to_global = st.save != 0 && st.kind != kStepLast;
            gdst = to_global ? p.ws.hidden[l] : nullptr;
          }
          if (!valid) continue;
          if (st.kind == kStepLast) {
            float* qd = qarr + st.qdst * kQR * ldq + n;
#pragma unroll
            for (int k = 0; k < 8; ++k) qd[rowof(k) * ldq] = x[k];
            continue;
          }
          if (to_operand) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              float h, lo_;
              split_tf32(row0 + rowof(k) < B ? x[k] : 0.f, h, lo_);
              ob[rowof(k) * 4] = h;
              ob[rowof(k) * 4 + kQLoOff] = lo_;
            }
          }
          if (to_global) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              const int row = row0 + rowof(k);
              if (row < B) gdst[(size_t)row * N + n] = x[k];
            }
          }
        }
      }
    };
    auto loss_stage = [&]() {
      // same arithmetic as rb200_dqn.cu (dqn_trainer.py:157-239); 8 lanes per batch row, the
      // actions strided over them, combined with shuffles inside the 8-lane group
      const float* qa = qarr;
      const float* qb = qarr + kQR * ldq;
      const float* qc = qarr + 2 * kQR * ldq;
      const int r = tid >> 3, sub = tid & 7;
      const int row = row0 + r;
      const bool in = row < B;
      // arg max over the (masked) next-state values: first index wins ties, as a sequential
      // "key > best" scan does
      float best = 0.f, sel = 0.f, qsel = 0.f, bsum = 0.f;
      int bi = 0x7fffffff;
      for (int c = sub; c < A; c += 8) {
        const float pen = -1e9f * (1.f - mask_s[r * A + c]);
        const float vt = qb[r * ldq + c] + pen;
        const float key = a.double_q ? (qa[r * ldq + c] + pen) : vt;
        if (bi == 0x7fffffff || key > best) { best = key; bi = c; sel = vt; }
        const float aw = act_s[r * A + c];
        qsel += qc[r * ldq + c] * aw;
        if (a.reward_boost) bsum += aw * a.reward_boost[c];
      }
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const float os = __shfl_xor_sync(0xffffffffu, sel, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        qsel += __shfl_xor_sync(0xffffffffu, qsel, o);
        bsum += __shfl_xor_sync(0xffffffffu, bsum, o);
        if (oi != 0x7fffffff && (bi == 0x7fffffff || ob > best || (ob == best && oi < bi))) {
          best = ob; bi = oi; sel = os;
        }
      }
      float le = 0.f, g = 0.f;
      if (in) {
        const float rew = scal_s[r * 4 + 0] + bsum;
        const float disc = (a.discount_mode == RB200_DISCOUNT_POW)
                               ? powf(a.gamma, scal_s[r * 4 + 2]) : a.gamma;
        const float tgt = rew + disc * (sel * scal_s[r * 4 + 1]);
        const float d = qsel - tgt;
        const float invB = 1.f / (float)B;
        if (a.loss_kind == RB200_LOSS_HUBER) {
          const float ad = fabsf(d);
          le = ad < 1.f ? 0.5f * d * d : ad - 0.5f;
          g = (d < -1.f) ? -invB : (d > 1.f ? invB : invB * d);
        } else {
          le = d * d;
          g = 2.f * invB * d;
        }
        if (kWeighted) {
          const float w = a.sample_weight[row];
          le *= w;
          g *= w;
        }
        if (sub == 0) {
          if (a.td_target) a.td_target[row] = tgt;
          if (a.next_action_idx) a.next_action_idx[row] = bi;
          if (a.q_selected) a.q_selected[row] = qsel;
        }
      }
      const int A8 = round_up8(A);
      const int lact = q.act[L - 1];
      float* zb = reinterpret_cast<float*>(smem_raw + p.buf_off[2]) + r * 4;
      for (int c = sub; c < A8; c += 8) {
        float v = 0.f;
        if (in && c < A) {
          v = g * act_s[r * A + c];
          if (lact != RB200_ACT_LINEAR) v *= act_bwd_slow(qc[r * ldq + c], lact);
          if (a.all_action_scores) a.all_action_scores[(size_t)row * A + c] = qc[r * ldq + c];
          if (a.do_backward) p.ws.dz[L - 1][(size_t)row * A + c] = v;
        }
        if (a.do_backward) {
          float h, lo_;
          split_tf32(v, h, lo_);
          float* o = zb + (c >> 2) * (kQLboB / 4) + (c & 3);
          o[0] = h;
          o[kQLoOff] = lo_;
        }
      }
      const float ws = warp_sum(sub == 0 ? le : 0.f);
      if (lane == 0) scal_s[kQR * 4 + warp] = ws;  // per-warp loss sums, combined by thread 0 at the end
    };


    auto x_src = [&](int lx) { return lx == 1 ? a.state : a.next_state; };
    // hand-over between the MMA warpgroups: every thread makes its operand stores visible to
    // the async proxy (the wgmma operand reads), then warps 0-7 meet at a named barrier
    auto handover = [&]() {
      fence_proxy_async_smem();
      asm volatile("bar.sync 1, %0;\n" ::"n"(kQEpiThreads) : "memory");
    };
    if (p.steps[0].load_x) { x_fetch(x_src(p.steps[0].load_x)); x_store(x_src(p.steps[0].load_x)); }
    load_loss_inputs();
    handover();
    for (int s = 0; s < p.nsteps; ++s) {
      const QStep st = p.steps[s];
      const int lx = (s + 1 < p.nsteps) ? p.steps[s + 1].load_x : 0;
      if (lx) x_fetch(x_src(lx));  // in flight during this step's MMAs and epilogue
      step_tiles(st);
      handover();  // this step's operand complete, and every MMA that read its input retired
      if (s == p.last_fwd_step) {
        loss_stage();
        handover();
      }
      if (lx) {
        x_store(x_src(lx));
        handover();
      }
    }

    // publish the loss (off the critical path of the step loop): last tile reduces
    if (tid == 0) {
      float loss_partial = 0.f;
      for (int w = 0; w < kQEpiThreads / 32; ++w) loss_partial += scal_s[kQR * 4 + w];
      finish_serial<1>(a.loss_partials, a.tile_counter, {loss_partial},
                       [&](const float (&tot)[1]) { *a.loss = tot[0] / (float)B; });
    }
  }
}

// ---------------------------------------------------------------------------
// host side: plan (steps, pack jobs, shared-memory layout)
// ---------------------------------------------------------------------------
struct QPlan {
  QDev dev;
  PackDev pack;
  int pack_chunks;
  size_t smem_bytes;
  int64_t pack_bytes;
  bool ok;
};

static QPlan make_plan(const rb200_mlp_t* qn, const rb200_mlp_t* qtn, int double_q, int do_backward) {
  QPlan pl;
  memset(&pl, 0, sizeof(pl));
  pl.ok = false;
  const int L = qn->n_layers;
  if (L < 1 || L > kMaxLayers) return pl;
  for (int l = 1; l <= L; ++l)
    if (qn->dims[l] > 128 * kQMaxTiles || qn->dims[l] > 32000) return pl;
  if (qn->dims[0] > 32000 || qn->dims[L] > 256) return pl;

  // weight images: online fwd, target fwd, online bwd (transposed)
  uint32_t off = 0;
  uint32_t off_on[kMaxLayers], off_tg[kMaxLayers], off_bw[kMaxLayers];
  int nj = 0, nchunks = 0;
  auto add_job = [&](const rb200_mlp_t* net, int l, int transpose) {
    PackJob& j = pl.pack.jobs[nj++];
    j.W = net->params + net->w_off[l];
    j.ld = net->dims[l];
    j.transpose = transpose;
    j.N = transpose ? net->dims[l] : net->dims[l + 1];
    j.K = transpose ? net->dims[l + 1] : net->dims[l];
    j.pack_off = off;
    j.chunk0 = nchunks;
    nchunks += ceil_div(j.N, 128) * ceil_div(j.K, kQKC);
    const uint32_t o = off;
    off += image_bytes(j.N, j.K);
    return o;
  };
  for (int l = 0; l < L; ++l) off_on[l] = add_job(qn, l, 0);
  if (qtn) for (int l = 0; l < L; ++l) off_tg[l] = add_job(qtn, l, 0);
  else for (int l = 0; l < L; ++l) { off_tg[l] = off; off += image_bytes(qn->dims[l + 1], qn->dims[l]); nj++; }
  if (do_backward) for (int l = 1; l < L; ++l) off_bw[l] = add_job(qn, l, 1);
  pl.pack.njobs = nj;
  pl.pack_chunks = nchunks;
  {
    // the Adam kernel writes the same images from rb200_dqn_tc_layout.cuh's table
    const TcImages im = tc_images(qn, do_backward);
    pl.pack_bytes = im.total_bytes;
    bool same = im.total_bytes == (int64_t)off + 4096;
    for (int l = 0; l < L; ++l) same = same && im.on_fwd[l] == off_on[l] && im.tg_fwd[l] == off_tg[l];
    if (do_backward) for (int l = 1; l < L; ++l) same = same && im.on_bwd[l] == off_bw[l];
    if (!same) return pl;  // ok stays false: layout tables disagree (a bug, not a user error)
  }

  // steps
  int ns = 0;
  auto add_pass = [&](int net, int load_x, int save, int qdst) {
    for (int l = 0; l < L; ++l) {
      QStep& s = pl.dev.steps[ns++];
      s.pack_off = net ? off_tg[l] : off_on[l];
      s.N = (int16_t)qn->dims[l + 1];
      s.K = (int16_t)qn->dims[l];
      s.layer = (int8_t)l;
      s.kind = (l == L - 1) ? kStepLast : kStepHidden;
      s.net = (int8_t)net;
      s.in_buf = (int8_t)(l & 1);
      s.out_buf = (int8_t)((l + 1) & 1);
      s.load_x = (int8_t)(l == 0 ? load_x : 0);
      s.save = (int8_t)save;
      s.qdst = (int8_t)qdst;
    }
  };
  add_pass(1, 2, 0, 1);                    // q_target(next_state)
  if (double_q) add_pass(0, 2, 0, 0);      // q(next_state)
  add_pass(0, 1, do_backward ? 1 : 0, 2);  // q(state)
  pl.dev.last_fwd_step = ns - 1;
  if (do_backward) {
    for (int l = L - 1; l >= 1; --l) {
      QStep& s = pl.dev.steps[ns++];
      s.pack_off = off_bw[l];
      s.N = (int16_t)qn->dims[l];
      s.K = (int16_t)qn->dims[l + 1];
      s.layer = (int8_t)l;
      s.kind = kStepBwd;
      s.net = 0;
      // dZ of the last layer sits in its own buffer so that the forward operands h_{l-1}
      // (the activation derivatives) survive until their backward step; dZ_{l-1} then
      // overwrites h_{l-1} in place
      s.in_buf = (int8_t)(l == L - 1 ? 2 : ((l + 1) & 1));
      s.out_buf = (int8_t)(l & 1);
      s.save = (int8_t)(l <= L - 3 ? 1 : 0);  // h_{l-1} clobbered by h_{l+1}: use the global copy
    }
  }
  pl.dev.nsteps = ns;
  pl.dev.need_zero = 0;
  for (int l = 0; l <= L; ++l)
    if (qn->dims[l] % 8 != 0) pl.dev.need_zero = 1;

  // shared memory
  int maxd[3] = {8, 8, qn->dims[L]};
  for (int i = 0; i < L; ++i) if (qn->dims[i] > maxd[i & 1]) maxd[i & 1] = qn->dims[i];
  size_t o = (size_t)kQStages * kQStageBytes;
  for (int b = 0; b < 3; ++b) {
    pl.dev.buf_off[b] = (int)o;
    o += (size_t)(round_up8(maxd[b]) / 4) * kQLboB;
  }
  pl.dev.ldq = qn->dims[L] + 1;
  pl.dev.q_off = (int)o;
  o += (size_t)3 * kQR * pl.dev.ldq * sizeof(float);
  o = (o + 15) & ~(size_t)15;
  pl.dev.lin_off = (int)o;
  o += ((size_t)2 * kQR * qn->dims[L] + 4 * kQR + 8) * sizeof(float);
  o = (o + 15) & ~(size_t)15;
  pl.dev.bar_off = (int)o;
  o += 2 * kQStages * sizeof(uint64_t);
  pl.smem_bytes = (o + 15) & ~(size_t)15;
  pl.ok = pl.smem_bytes <= (size_t)kQMaxSmem;
  return pl;
}

}  // namespace rb200

using namespace rb200;

extern "C" int64_t rb200_dqn_tc_workspace_bytes(const rb200_mlp_t* q_net, int32_t double_q,
                                                int32_t do_backward) {
  if (!q_net || validate_mlp(q_net, "q_network")) return 0;
  const QPlan pl = make_plan(q_net, nullptr, double_q, do_backward);
  return pl.ok ? pl.pack_bytes : 0;
}

extern "C" int rb200_dqn_tc_pack(const rb200_mlp_t* q_net, const rb200_mlp_t* q_target,
                                 int32_t double_q, int32_t do_backward, void* pack_ws,
                                 int64_t pack_ws_bytes, void* stream) {
  if (!q_net || !q_target || !pack_ws) { set_last_error("rb200_dqn_tc_pack: null argument"); return RB200_E_INVALID; }
  if (int rc = validate_mlp(q_net, "q_network")) return rc;
  if (int rc = validate_mlp(q_target, "q_network_target")) return rc;
  if (q_net->n_layers != q_target->n_layers) { set_last_error("q_network / target layer count mismatch"); return RB200_E_INVALID; }
  for (int l = 0; l <= q_net->n_layers; ++l)
    if (q_net->dims[l] != q_target->dims[l]) { set_last_error("q_network / target dims mismatch at %d", l); return RB200_E_INVALID; }
  if ((reinterpret_cast<uintptr_t>(pack_ws) & 127) != 0) { set_last_error("pack workspace must be 128-byte aligned"); return RB200_E_INVALID; }
  QPlan pl = make_plan(q_net, q_target, double_q, do_backward);
  if (!pl.ok) { set_last_error("rb200_dqn_tc_pack: shapes do not fit the wgmma path"); return RB200_E_SMEM; }
  if (pack_ws_bytes < pl.pack_bytes) { set_last_error("pack workspace too small: %lld < %lld", (long long)pack_ws_bytes, (long long)pl.pack_bytes); return RB200_E_INVALID; }
  pl.pack.pack = static_cast<unsigned char*>(pack_ws);
  dqn_tc_pack_kernel<<<pl.pack_chunks * kPackParts, 256, 0, (cudaStream_t)stream>>>(pl.pack);
  return check_cuda(cudaGetLastError(), "dqn_tc_pack_kernel launch");
}

extern "C" int rb200_dqn_td_step_tc(const rb200_mlp_t* q_net, const rb200_mlp_t* q_target,
                                    const rb200_dqn_args_t* args, const rb200_net_ws_t* ws,
                                    void* pack_ws, int64_t pack_ws_bytes, int32_t weights_packed,
                                    void* stream) {
  if (!q_net || !q_target || !args || !ws || !pack_ws) { set_last_error("rb200_dqn_td_step_tc: null argument"); return RB200_E_INVALID; }
  if (!weights_packed) {
    if (int rc = rb200_dqn_tc_pack(q_net, q_target, args->double_q, args->do_backward, pack_ws, pack_ws_bytes, stream)) return rc;
  }
  if (int rc = validate_mlp(q_net, "q_network")) return rc;
  if (int rc = validate_mlp(q_target, "q_network_target")) return rc;
  if (q_net->n_layers != q_target->n_layers) { set_last_error("q_network / target layer count mismatch"); return RB200_E_INVALID; }
  for (int l = 0; l <= q_net->n_layers; ++l)
    if (q_net->dims[l] != q_target->dims[l]) { set_last_error("q_network / target dims mismatch at %d", l); return RB200_E_INVALID; }
  if (args->batch <= 0) { set_last_error("batch must be positive"); return RB200_E_INVALID; }
  if (!args->state || !args->next_state || !args->action || !args->reward || !args->not_terminal ||
      !args->loss_partials || !args->loss || !args->tile_counter) {
    set_last_error("rb200_dqn_td_step_tc: required pointer is null"); return RB200_E_INVALID;
  }
  if (!args->maxq && !args->next_action) { set_last_error("SARSA update needs next_action"); return RB200_E_INVALID; }
  if (args->discount_mode == RB200_DISCOUNT_POW && !args->discount_src) { set_last_error("POW discount needs discount_src"); return RB200_E_INVALID; }
  if (args->do_backward) {
    for (int l = 0; l < q_net->n_layers; ++l)
      if (!ws->dz[l] || (l < q_net->n_layers - 1 && !ws->hidden[l])) { set_last_error("workspace buffer missing for layer %d", l); return RB200_E_INVALID; }
  }
  if ((reinterpret_cast<uintptr_t>(pack_ws) & 127) != 0) { set_last_error("pack workspace must be 128-byte aligned"); return RB200_E_INVALID; }
  QPlan pl = make_plan(q_net, q_target, args->double_q, args->do_backward);
  if (!pl.ok) { set_last_error("rb200_dqn_td_step_tc: shapes do not fit the wgmma path"); return RB200_E_SMEM; }
  if (pack_ws_bytes < pl.pack_bytes) { set_last_error("pack workspace too small: %lld < %lld", (long long)pack_ws_bytes, (long long)pl.pack_bytes); return RB200_E_INVALID; }
  pl.dev.a = *args;
  pl.dev.ws = *ws;
  pl.dev.pack = static_cast<const unsigned char*>(pack_ws);
  cudaStream_t st = (cudaStream_t)stream;
  const bool weighted = args->sample_weight != nullptr;
  if (cudaError_t e = weighted ? opt_in_smem<dqn_td_tc_kernel<true>>(pl.smem_bytes)
                               : opt_in_smem<dqn_td_tc_kernel<false>>(pl.smem_bytes))
    return check_cuda(e, "cudaFuncSetAttribute(dqn_td_tc)");
  // Launched at the device's greatest priority.  A CTA of this kernel needs nearly a whole SM
  // (~210 KB of shared memory, 9 warps at ~160 registers), so when an independent kernel becomes
  // ready at the same time -- the next update's replay sample in a captured training loop --
  // and its CTAs are placed first, K2's CTAs wait for them to drain and the whole chain of K2
  // slips (config 2: 80 us instead of 61 us per launch on an H100).  With the higher priority
  // the block scheduler places K2's CTAs first and the other kernel fills what is left.  The
  // priority is recorded in captured graph nodes; it takes effect where the graph is
  // instantiated with cudaGraphInstantiateFlagUseNodePriority, as torch.cuda.CUDAGraph does.
  static int greatest[64] = {};
  static bool have_greatest[64] = {};
  int dev = 0;
  if (cudaError_t e = cudaGetDevice(&dev)) return check_cuda(e, "cudaGetDevice");
  int prio = 0;
  if (dev >= 0 && dev < 64 && have_greatest[dev]) {
    prio = greatest[dev];
  } else {
    int least = 0;
    if (cudaError_t e = cudaDeviceGetStreamPriorityRange(&least, &prio))
      return check_cuda(e, "cudaDeviceGetStreamPriorityRange");
    if (dev >= 0 && dev < 64) { greatest[dev] = prio; have_greatest[dev] = true; }
  }
  const Mlp q = make_mlp(q_net), qt = make_mlp(q_target);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)ceil_div(args->batch, kQR));
  cfg.blockDim = dim3(kQThreads);
  cfg.dynamicSmemBytes = pl.smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributePriority;
  attr[0].val.priority = prio;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const cudaError_t e = weighted ? cudaLaunchKernelEx(&cfg, dqn_td_tc_kernel<true>, q, qt, pl.dev)
                                 : cudaLaunchKernelEx(&cfg, dqn_td_tc_kernel<false>, q, qt, pl.dev);
  return check_cuda(e, "dqn_td_tc_kernel launch");
}
