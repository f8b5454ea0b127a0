// reagent_b200 -- cross-entropy-method planner (reagent/models/cem_planner.py): the rollout of
// one CEM iteration and its reduction, in one launch.
//
// The reference evaluates a solution by calling the world model once per planned step with a
// [1, 1, .] input and no hidden state, so every step is a T = 1 MDN-RNN forward from h = c = 0:
//   gates = (0 + b_hh) + (x . W_ih^T + b_ih),   c' = i * g,   h' = o * tanh(c')
// W_hh never contributes, and f multiplies a zero cell.  The per-step products below keep the
// operand order and roundings of mdnrnn_fwd_kernel (0 . W sums to exactly 0 and f * 0 = 0), so
// each step's head outputs are bit-identical to MemoryNetwork.forward on the same rows.
//
// The trajectories of an iteration are independent, so CTA (j, m) carries the j-th group of 16
// trajectories that drew world model m through every step with the row-tile primitives of
// rb200_tile.cuh, and samples the mixture, the next state and (with terminal_effective) the
// terminal in place from the caller's noise.  The last CTA to finish (atomic counter, as
// finish_serial) selects the elites and updates mean / var in fp64, or tallies first actions.
#include <math.h>

#include "rb200_tile.cuh"

namespace rb200 {

constexpr int kCemNT = 256, kCemTM = 4, kCemKC = 32;
constexpr int kCemR = (kCemNT / 64) * kCemTM;  // 16 trajectories per CTA
static_assert(kCemR == RB200_CEM_ROWS_PER_BLOCK, "rows per block");

struct CemDims {
  int S, A, H, L, G, NG, DX, GS, NS;  // NS = S + 2 noise floats per step
  int P, HOR, HA;
  int ld_x, ld_h, ld_s;
};

__host__ __device__ inline CemDims cem_dims(const rb200_cem_args_t& a) {
  CemDims d;
  d.S = a.net.state_dim; d.A = a.net.action_dim; d.H = a.net.hidden; d.L = a.net.layers;
  d.G = a.net.gaussians;
  d.NG = (2 * d.S + 1) * d.G + 2;
  d.DX = d.A + d.S;
  d.GS = d.G * d.S;
  d.NS = d.S + 2;
  d.P = a.population; d.HOR = a.horizon; d.HA = a.horizon * d.A;
  d.ld_x = round_up4(d.DX) + 4;
  d.ld_h = round_up4(d.H) + 4;
  const int ld_g = round_up4(4 * d.H) + 4, ld_y = round_up4(d.NG) + 4;
  d.ld_s = ld_g > ld_y ? ld_g : ld_y;
  return d;
}

// floats of the rollout's shared memory; the reduction reuses the weight staging area
inline size_t cem_smem(const CemDims& d) {
  const size_t f = 2 * (size_t)wstage_floats<kCemKC>() +
                   (size_t)kCemR * (d.ld_x + 2 * d.ld_h + d.ld_s + 32);
  return sizeof(float) * f + sizeof(double) * kCemR + sizeof(int) * (2 * kCemR + 4);
}

// sqrt(constrained_variance) of plan element c: min(((mean - lb) / 2)^2, ((ub - mean) / 2)^2,
// var), every operation rounded as numpy rounds it
__device__ __forceinline__ double cem_scale(const rb200_cem_args_t& a, int c, double mean,
                                            double var) {
  const double lo = __ddiv_rn(__dsub_rn(mean, a.lower[c]), 2.0);
  const double hi = __ddiv_rn(__dsub_rn(a.upper[c], mean), 2.0);
  return __dsqrt_rn(fmin(fmin(__dmul_rn(lo, lo), __dmul_rn(hi, hi)), var));
}

// solution element c of trajectory p in this iteration: z * sqrt(constrained var) + mean
__device__ __forceinline__ double cem_solution(const rb200_cem_args_t& a, const CemDims& d, int p,
                                               int c, double mean, double scale) {
  const double z = a.truncnorm[((size_t)a.iter * d.P + p) * d.HA + c];
  return __dadd_rn(__dmul_rn(z, scale), mean);
}

__device__ void cem_reduce(const rb200_cem_args_t& a, const CemDims& d, float* smem) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = kCemNT / 32;
  const int it = a.iter;
  double* v = reinterpret_cast<double*>(smem);  // [P]
  for (int p = tid; p < d.P; p += kCemNT) v[p] = __ldcg(a.values + (size_t)it * d.P + p);
  __syncthreads();
  if (a.discrete) {
    if (tid == 0) {
      // reward_tally / first_action_tally, both fp64 in solution order; nanargmax skips the
      // actions never drawn first (0 / 0)
      double* cnt = v + d.P;
      double* sum = cnt + d.A;
      for (int c = 0; c < d.A; ++c) cnt[c] = sum[c] = 0.0;
      for (int p = 0; p < d.P; ++p) {
        const int f = a.action_idx[(size_t)p * d.HOR];
        cnt[f] = __dadd_rn(cnt[f], 1.0);
        sum[f] = __dadd_rn(sum[f], v[p]);
      }
      int best = -1;
      double bv = 0.0;
      for (int c = 0; c < d.A; ++c) {
        const double r = __ddiv_rn(sum[c], cnt[c]);
        if (!isnan(r) && (best < 0 || r > bv)) { best = c; bv = r; }
      }
      if (best < 0) best = 0;
      a.action_out[0] = best;
      for (int c = 0; c < d.A; ++c) a.one_hot[c] = c == best ? 1.f : 0.f;
      *a.n_iters = 1;
      *a.done = 1;
    }
    return;
  }
  // elites: the num_elites largest values, ties to the larger index, stored in ascending order
  // (np.argsort(values)[-num_elites:])
  const int E = a.num_elites;
  int* el = reinterpret_cast<int*>(v + d.P);
  for (int i = tid; i < E; i += kCemNT) el[i] = 0;
  __syncthreads();
  for (int p = tid; p < d.P; p += kCemNT) {
    const double vp = v[p];
    int rank = 0;
    for (int q = 0; q < d.P; ++q) rank += (v[q] > vp) || (v[q] == vp && q > p);
    if (rank < E) el[E - 1 - rank] = p;
  }
  __syncthreads();
  for (int i = tid; i < E; i += kCemNT) a.elites[(size_t)it * E + i] = el[i];
  // mean / var of the elites (np.mean, np.var with ddof 0: sequential over the elites), then
  // mean <- alpha mean + (1 - alpha) mean(elites), likewise var
  const double al = a.alpha, om = __dsub_rn(1.0, a.alpha);
  double vmax = -INFINITY;
  for (int c = tid; c < d.HA; c += kCemNT) {
    const double mc = a.mean[c], vc = a.var[c];
    const double sc = cem_scale(a, c, mc, vc);
    double s = 0.0;
    for (int i = 0; i < E; ++i) s = __dadd_rn(s, cem_solution(a, d, el[i], c, mc, sc));
    const double nm = __ddiv_rn(s, (double)E);
    double q = 0.0;
    for (int i = 0; i < E; ++i) {
      const double x = __dsub_rn(cem_solution(a, d, el[i], c, mc, sc), nm);
      q = __dadd_rn(q, __dmul_rn(x, x));
    }
    const double nv = __ddiv_rn(q, (double)E);
    const double m2 = __dadd_rn(__dmul_rn(al, mc), __dmul_rn(om, nm));
    const double v2 = __dadd_rn(__dmul_rn(al, vc), __dmul_rn(om, nv));
    a.mean[c] = m2;
    a.var[c] = v2;
    a.mean_hist[(size_t)it * d.HA + c] = m2;
    a.var_hist[(size_t)it * d.HA + c] = v2;
    vmax = fmax(vmax, v2);
  }
  for (int o = 16; o > 0; o >>= 1) vmax = fmax(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
  __syncthreads();  // the elite list is no longer read
  double* wm = v;
  if (lane == 0) wm[warp] = vmax;
  __syncthreads();
  if (tid == 0) {
    double m = wm[0];
    for (int w = 1; w < NW; ++w) m = fmax(m, wm[w]);
    *a.n_iters = it + 1;
    if (m <= a.epsilon || it + 1 >= a.iters) *a.done = 1;
  }
}

__global__ void __launch_bounds__(kCemNT, 1) cem_rollout_kernel(const rb200_cem_args_t a) {
  constexpr int NT = kCemNT, R = kCemR;
  if (*(volatile const int32_t*)a.done) return;  // converged in an earlier launch
  const CemDims d = cem_dims(a);
  extern __shared__ __align__(16) float smem[];
  tile_smem_zero_all<NT>(smem);
  float* Wst = smem;
  float* xs = Wst + 2 * wstage_floats<kCemKC>();  // [R][ld_x]: action | state
  float* hA = xs + R * d.ld_x;                   // [R][ld_h]: h of even layers
  float* hB = hA + R * d.ld_h;                   // [R][ld_h]: h of odd layers
  float* scr = hB + R * d.ld_h;                  // [R][ld_s]: gates, then the head output
  float* lps = scr + R * d.ld_s;                 // [R][32]: logpi
  double* acc = reinterpret_cast<double*>(lps + R * 32);
  int* rows = reinterpret_cast<int*>(acc + R);   // trajectory of each row, or -1
  int* alive = rows + R;
  int* s_last = alive + R;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m = blockIdx.y, j = blockIdx.x, it = a.iter;
  const int H = d.H, GS = d.GS;

  // the j-th group of R trajectories that drew model m, in solution order
  if (warp == 0) {
    const int32_t* midx = a.model_idx + (size_t)it * d.P;
    if (lane < R) rows[lane] = -1;
    __syncwarp();
    int seen = 0;
    for (int base = 0; base < d.P && seen < (j + 1) * R; base += 32) {
      const int p = base + lane;
      const bool hit = p < d.P && midx[p] == m;
      const unsigned bal = __ballot_sync(0xffffffffu, hit);
      const int rank = seen + __popc(bal & ((1u << lane) - 1u));
      if (hit && rank >= j * R && rank < (j + 1) * R) rows[rank - j * R] = p;
      seen += __popc(bal);
    }
  }
  __syncthreads();

  if (rows[0] >= 0) {
    const float* P = a.params[m];
    if (tid < R) { acc[tid] = 0.0; alive[tid] = rows[tid] >= 0; }
    for (int i = tid; i < R * d.S; i += NT) {
      const int r = i / d.S, s = i - r * d.S;
      xs[r * d.ld_x + d.A + s] = rows[r] >= 0 ? a.state[s] : 0.f;
    }
    for (int step = 0; step < d.HOR; ++step) {
      // this step's action: a one-hot, or the fp64 solution cast to fp32
      for (int i = tid; i < R * d.A; i += NT) {
        const int r = i / d.A, c = i - r * d.A, p = rows[r];
        if (p < 0) continue;
        float x;
        if (a.discrete) {
          x = a.action_idx[(size_t)p * d.HOR + step] == c ? 1.f : 0.f;
        } else {
          const int k = step * d.A + c;
          const double mc = a.mean[k];
          x = __double2float_rn(cem_solution(a, d, p, k, mc, cem_scale(a, k, mc, a.var[k])));
        }
        xs[r * d.ld_x + c] = x;
      }
      __syncthreads();
      const float* in = xs;
      int K = d.DX, ld_in = d.ld_x;
      float* hout = hA;
      for (int l = 0; l < d.L; ++l) {
        tile_linear_fwd<NT, kCemTM, kCemKC>(in, ld_in, K, P + a.net.w_ih_off[l], K,
                                            P + a.net.b_ih_off[l], 4 * H, RB200_ACT_LINEAR, scr,
                                            d.ld_s, Wst);
        const float* bhh = P + a.net.b_hh_off[l];  // h . W_hh^T + b_hh with h = 0
        for (int i = tid; i < R * H; i += NT) {
          const int r = i / H, jj = i - r * H;
          const float* g1 = scr + r * d.ld_s;
          const float gi = sigmoidf(__fadd_rn(bhh[jj], g1[jj]));
          const float gg = tanhf(__fadd_rn(bhh[2 * H + jj], g1[2 * H + jj]));
          const float go = sigmoidf(__fadd_rn(bhh[3 * H + jj], g1[3 * H + jj]));
          const float cn = __fmul_rn(gi, gg);
          hout[r * d.ld_h + jj] = rows[r] >= 0 ? __fmul_rn(go, tanhf(cn)) : 0.f;
        }
        __syncthreads();
        in = hout;
        K = H;
        ld_in = d.ld_h;
        hout = hout == hA ? hB : hA;
      }
      tile_linear_fwd<NT, kCemTM, kCemKC>(in, d.ld_h, H, P + a.net.w_gmm_off, H,
                                          P + a.net.b_gmm_off, d.NG, RB200_ACT_LINEAR, scr,
                                          d.ld_s, Wst);
      // one warp per row: logpi, then the draws of sample_reward_next_state_terminal
      for (int r = warp; r < R; r += NT / 32) {
        const int p = rows[r];
        if (p < 0 || !alive[r]) continue;
        const float* y = scr + r * d.ld_s;
        const bool gl = lane < d.G;
        const float rp = gl ? y[2 * GS + lane] : -INFINITY;
        const float pm = warp_max(rp);
        const float pe = warp_sum(gl ? expf(__fsub_rn(rp, pm)) : 0.f);
        const float logpi = gl ? __fsub_rn(__fsub_rn(rp, pm), logf(pe)) : -INFINITY;
        if (gl) lps[r * 32 + lane] = logpi;
        __syncwarp();
        if (a.dump && it == 0) {
          float* o = a.dump + ((size_t)p * d.HOR + step) * (d.DX + d.NG);
          for (int c = lane; c < d.DX; c += 32) o[c] = xs[r * d.ld_x + c];
          o += d.DX;
          for (int c = lane; c < GS; c += 32) { o[c] = y[c]; o[GS + c] = expf(y[GS + c]); }
          if (gl) o[2 * GS + lane] = logpi;
          if (lane == 0) { o[d.NG - 2] = y[d.NG - 2]; o[d.NG - 1] = y[d.NG - 1]; }
        }
        const float* nz = a.step_noise + (((size_t)it * d.P + p) * d.HOR + step) * d.NS;
        // mixture k ~ Categorical(exp(logpi)): the first k with u * sum(p) < cumsum(p)_k
        int k = d.G - 1;
        if (lane == 0) {
          float tot = 0.f;
          for (int q = 0; q < d.G; ++q) tot = __fadd_rn(tot, expf(lps[r * 32 + q]));
          const float thr = __fmul_rn(nz[0], tot);
          float cum = 0.f;
          for (int q = 0; q < d.G; ++q) {
            cum = __fadd_rn(cum, expf(lps[r * 32 + q]));
            if (thr < cum) { k = q; break; }
          }
        }
        k = __shfl_sync(0xffffffffu, k, 0);
        // next_state = mus[k] + sigmas[k] * z
        for (int s = lane; s < d.S; s += 32)
          xs[r * d.ld_x + d.A + s] =
              __fadd_rn(y[k * d.S + s], __fmul_rn(expf(y[GS + k * d.S + s]), nz[1 + s]));
        if (lane == 0) {
          // reward * gamma ** j in fp32, accumulated in fp64; stop after a terminal draw
          acc[r] = __dadd_rn(acc[r], (double)__fmul_rn(y[d.NG - 2], a.discount[step]));
          if (a.terminal_effective && !(nz[d.S + 1] < sigmoidf(y[d.NG - 1]))) alive[r] = 0;
        }
      }
      if (!__syncthreads_or(tid < R && rows[tid] >= 0 && alive[tid])) break;
    }
    if (tid < R && rows[tid] >= 0) a.values[(size_t)it * d.P + rows[tid]] = acc[tid];
  }

  __threadfence();
  __syncthreads();
  if (tid == 0) s_last[0] = atomicAdd(a.counter, 1u) == gridDim.x * gridDim.y - 1;
  __syncthreads();
  if (!s_last[0]) return;
  __threadfence();
  cem_reduce(a, d, smem);
  if (tid == 0) *a.counter = 0u;
}

}  // namespace rb200

using namespace rb200;

extern "C" int rb200_cem_check_shape(int32_t S, int32_t A, int32_t H, int32_t L, int32_t G,
                                     int32_t P, int32_t K, int32_t horizon, int32_t E) {
  if (int rc = rb200_mdnrnn_check_shape(S, A, H, L, G)) return rc;
  if (P < 1 || K < 1 || horizon < 1 || P > RB200_CEM_MAX_POPULATION ||
      K > RB200_CEM_MAX_MODELS || (long long)horizon * A > RB200_CEM_MAX_PLAN || E < 1 || E > P) {
    set_last_error("rb200_cem: unsupported shape (population %d in [1, %d], world models %d in "
                   "[1, %d], horizon %d >= 1 with horizon * action_dim %lld <= %d, num_elites "
                   "%d in [1, population])", P, RB200_CEM_MAX_POPULATION, K,
                   RB200_CEM_MAX_MODELS, horizon, (long long)horizon * A, RB200_CEM_MAX_PLAN, E);
    return RB200_E_INVALID;
  }
  return RB200_OK;
}

extern "C" int rb200_cem_rollout(const rb200_cem_args_t* a, void* stream) {
  if (!a) { set_last_error("rb200_cem_rollout: args is null"); return RB200_E_INVALID; }
  const rb200_mdnrnn_args_t& n = a->net;
  if (int rc = rb200_cem_check_shape(n.state_dim, n.action_dim, n.hidden, n.layers, n.gaussians,
                                     a->population, a->num_models, a->horizon, a->num_elites))
    return rc;
  bool ok = a->iters >= 1 && a->iter >= 0 && a->iter < a->iters && a->state && a->discount &&
            a->model_idx && a->step_noise && a->values && a->done && a->n_iters && a->counter;
  for (int m = 0; m < a->num_models; ++m) ok = ok && a->params[m];
  if (a->discrete)
    ok = ok && a->iters == 1 && a->action_idx && a->action_out && a->one_hot;
  else
    ok = ok && a->lower && a->upper && a->truncnorm && a->mean && a->var && a->elites &&
         a->mean_hist && a->var_hist;
  if (!ok) {
    set_last_error("rb200_cem_rollout: iteration %d of %d (discrete plans run one), or a "
                   "required buffer is null", a->iter, a->iters);
    return RB200_E_INVALID;
  }
  const CemDims d = cem_dims(*a);
  const dim3 grid(ceil_div(d.P, kCemR), a->num_models);
  return launch<cem_rollout_kernel>(grid, kCemNT, cem_smem(d), (cudaStream_t)stream,
                                    "cem_rollout_kernel launch", *a);
}
