// reagent_b200 -- counterfactual policy evaluation (reagent/evaluation/*.py) on the device.
//
// The networks of an EvaluationDataPage run on rb200_mlp_forward; these kernels do the rest.
// Every kernel is deterministic: no floating-point atomics, fixed summation orders.
//   page          evaluation_data_page.py:309-462  one row per thread
//   episode_marks :542-626 (validate's episode checks) and the episode boundaries
//   logged_values :523-540 compute_values_for_mdps, one thread per episode
//   sdr           sequential_doubly_robust_estimator.py:29-96, one thread per episode
//   dr_rows       doubly_robust_estimator.py:219-340, one row per thread
//   boot_means    cpe.py:176-191 bootstrapped_std_error_of_mean's sample means, one CTA per sample
//   wsdr_rows / wsdr_returns / seg_sum / cov
//                 weighted_sequential_doubly_robust_estimator.py:27-384 in episode (CSR) layout
// Float32 recursions use the rounded intrinsics, so no FMA contraction changes their bits.
#include <curand_kernel.h>

#include "rb200_common.cuh"

namespace rb200 {

constexpr int kOpeThreads = 256;

// ---------------------------------------------------------------------------------------------
// page: boosted reward, masked_softmax(q), masked arg max, logged-action gathers
// ---------------------------------------------------------------------------------------------
struct PageArgs {
  int n, A, K;  // K metrics besides the reward
  const float *q, *reward_out, *qcpe_out, *mask, *action, *reward, *boost;
  float temperature;
  float *boosted, *prop;
  int64_t* eval_idx;
  float *mr_logged, *mm_logged, *mmv_logged;
};

// torch.sum(x * w, dim=1) of one row in the order of torch's CPU reduction over a short
// contiguous axis: k = 8 (A >= 8) or 4 (A >= 4) strided accumulators, added in order.  This is
// the order measured for A <= 5, 8, 9 and 16; for A = 6 and 7 torch's order is different and the
// last bit can differ.
__device__ __forceinline__ float dot_seq(const float* x, const float* w, int A) {
  const int k = A >= 8 ? 8 : (A >= 4 ? 4 : 1);
  float s = 0.f;
  for (int j = 0; j < k && j < A; ++j) {
    float a = __fmul_rn(x[j], w[j]);
    for (int i = j + k; i < A; i += k) a = __fadd_rn(a, __fmul_rn(x[i], w[i]));
    s = j == 0 ? a : __fadd_rn(s, a);
  }
  return s;
}

__global__ void __launch_bounds__(kOpeThreads) ope_page_kernel(const PageArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.n) return;
  const int A = a.A, W = (a.K + 1) * A;
  const float* act = a.action + (size_t)b * A;
  const float* q = a.q + (size_t)b * A;
  const float* mk = a.mask + (size_t)b * A;
  // boost_rewards (dqn_trainer_base.py:216-241)
  a.boosted[b] = a.boost ? __fadd_rn(a.reward[b], dot_seq(act, a.boost, A)) : a.reward[b];
  // masked_softmax(model_outputs, possible_actions_mask, rl_temperature)
  float mx, den;
  masked_softmax_stats(q, mk, a.temperature, A, mx, den);
  for (int c = 0; c < A; ++c)
    a.prop[(size_t)b * A + c] = masked_softmax_p(q[c], mk[c], a.temperature, mx, den);
  // get_max_q_values: q + (-1e9) * (1 - mask), torch.max's first maximum
  int best = 0;
  float bv = __fadd_rn(q[0], __fmul_rn(-1e9f, __fsub_rn(1.f, mk[0])));
  for (int c = 1; c < A; ++c) {
    const float v = __fadd_rn(q[c], __fmul_rn(-1e9f, __fsub_rn(1.f, mk[c])));
    if (v > bv || (v != v && bv == bv)) { bv = v; best = c; }
  }
  a.eval_idx[b] = best;
  const float* ro = a.reward_out + (size_t)b * W;
  const float* qo = a.qcpe_out + (size_t)b * W;
  a.mr_logged[b] = dot_seq(ro, act, A);
  for (int i = 0; i < a.K; ++i) {
    a.mm_logged[(size_t)b * a.K + i] = dot_seq(ro + (i + 1) * A, act, A);
    a.mmv_logged[(size_t)b * a.K + i] = dot_seq(qo + (i + 1) * A, act, A);
  }
}

// ---------------------------------------------------------------------------------------------
// episode marks: is_start[i] = (i == 0 || mdp[i] != mdp[i-1]); flags[0] = first row whose
// sequence_number does not increase inside its run (n if none), flags[1] = number of runs.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kOpeThreads)
ope_marks_kernel(int n, const int64_t* mdp, const int64_t* seq, uint8_t* is_start, int* flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool start = i == 0 || mdp[i] != mdp[i - 1];
  is_start[i] = start;
  if (start) atomicAdd(&flags[1], 1);
  else if (seq[i] <= seq[i - 1]) atomicMin(&flags[0], i);
}

// compute_values_for_mdps: values = x; for rows from the end, values[r, 0] +=
// values[r+1, 0] * disc[r] inside an episode, where disc[r] = (float)math.pow(gamma,
// seq[r+1] - seq[r]) comes from the host.  Only column 0 recurses, as in the reference; the
// other columns are copies.
__global__ void __launch_bounds__(kOpeThreads)
ope_values_kernel(int E, const int* off, const float* disc, int C, const float* x, float* out) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int lo = off[e], hi = off[e + 1];
  for (int r = lo; r < hi; ++r)
    for (int c = 1; c < C; ++c) out[(size_t)r * C + c] = x[(size_t)r * C + c];
  float v = x[(size_t)(hi - 1) * C];
  out[(size_t)(hi - 1) * C] = v;
  for (int r = hi - 2; r >= lo; --r) {
    v = __fadd_rn(x[(size_t)r * C], __fmul_rn(v, disc[r]));
    out[(size_t)r * C] = v;
  }
}

// sequential DR of one episode, from its last row back:
//   dr = V(s) + w * (r + gamma * dr - Q(s, a)),  value = value * gamma + r    (float32)
__global__ void __launch_bounds__(kOpeThreads)
ope_sdr_kernel(int E, const int* off, int A, const float* prop, const float* qv, const float* am,
               const float* r, const float* lp, float gamma, float* ep_dr, float* ep_val) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  float dr = 0.f, val = 0.f;
  for (int j = off[e + 1] - 1; j >= off[e]; --j) {
    const float* p = prop + (size_t)j * A;
    const float* q = qv + (size_t)j * A;
    const float* m = am + (size_t)j * A;
    const float v = dot_seq(p, q, A);
    const float ql = dot_seq(q, m, A);
    const float w = __fdiv_rn(dot_seq(p, m, A), lp[j]);
    dr = __fadd_rn(v, __fmul_rn(w, __fsub_rn(__fadd_rn(r[j], __fmul_rn(gamma, dr)), ql)));
    val = __fadd_rn(__fmul_rn(val, gamma), r[j]);
  }
  ep_dr[e] = dr;
  ep_val[e] = val;
}

// DM = sum_a p * R(s, a); IPS = w * r; DR = w * (r - R(s, a_log)) + DM, w = p(a_log) / mu
__global__ void __launch_bounds__(kOpeThreads)
ope_dr_rows_kernel(int n, int A, const float* prop, const float* mr, const float* am, const float* r,
                   const float* mrl, const float* lp, float* dm, float* ips, float* dr) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n) return;
  const float* p = prop + (size_t)b * A;
  const float w = __fdiv_rn(dot_seq(p, am + (size_t)b * A, A), lp[b]);
  const float d = dot_seq(p, mr + (size_t)b * A, A);
  dm[b] = d;
  ips[b] = __fmul_rn(w, r[b]);
  dr[b] = __fadd_rn(__fmul_rn(w, __fsub_rn(r[b], mrl[b])), d);
}

// one CTA per bootstrap sample: the mean of data[idx[s, :]] as an fp64 sum over fp64 (the caller
// rounds it to float32 where the reference's sample is float32).  idx == NULL: index k of sample s is drawn
// from Philox(seed, subsequence s * 256 + thread, offset) as a 64-bit value modulo n.
__global__ void __launch_bounds__(kOpeThreads)
ope_boot_kernel(const float* data, int n, const int* idx, int k, unsigned long long seed,
                unsigned long long offset, double* means) {
  __shared__ double s_warp[kOpeThreads / 32];
  const int s = blockIdx.x;
  double acc = 0.0;
  if (idx) {
    const int* row = idx + (size_t)s * k;
    for (int i = threadIdx.x; i < k; i += blockDim.x) acc += (double)data[row[i]];
  } else {
    curandStatePhilox4_32_10_t st;
    curand_init(seed, (unsigned long long)s * blockDim.x + threadIdx.x, offset, &st);
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
      const unsigned long long hi = curand(&st);
      const unsigned long long u = (hi << 32) | curand(&st);
      acc += (double)data[u % (unsigned long long)n];
    }
  }
  const double t = block_sum_f64(acc, s_warp);
  if (threadIdx.x == 0) means[s] = t / (double)k;
}

// numpy's pairwise sum of n < 128 values (8 accumulators, then a fixed tree), the order of
// np.sum(..., axis=-1) over the action axis
template <typename T, typename F>
__device__ __forceinline__ T np_sum(int n, F f) {
  if (n < 8) {
    T s = (T)0;  // numpy starts from -0.0 and adds in order; 0 + x == x for every x but -0
    for (int i = 0; i < n; ++i) s = i == 0 ? f(0) : s + f(i);
    return s;
  }
  T r[8];
  for (int j = 0; j < 8; ++j) r[j] = f(j);
  int i = 8;
  for (; i + 8 <= n; i += 8)
    for (int j = 0; j < 8; ++j) r[j] += f(i + j);
  T s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
  for (; i < n; ++i) s += f(i);
  return s;
}

// WSDR rows in the weight precision T: w = cumprod(p(a_log) / mu) along the episode,
// V(s) = sum_a p * Q, Q(s, a_log) = sum_a Q * action_mask
template <typename T>
__global__ void __launch_bounds__(kOpeThreads)
ope_wsdr_rows_kernel(int E, const int* off, int A, const float* prop, const float* qv, const float* am,
                     const float* lp, T* w, T* sv, T* ql) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  T c = (T)1;
  for (int j = off[e]; j < off[e + 1]; ++j) {
    const float* p = prop + (size_t)j * A;
    const float* q = qv + (size_t)j * A;
    const float* m = am + (size_t)j * A;
    const T tp = np_sum<T>(A, [&](int i) { return (T)p[i] * (T)m[i]; });
    const T x = tp / (T)lp[j];
    c = j == off[e] ? x : c * x;
    w[j] = c;
    sv[j] = np_sum<T>(A, [&](int i) { return (T)p[i] * (T)q[i]; });
    ql[j] = np_sum<T>(A, [&](int i) { return (T)q[i] * (T)m[i]; });
  }
}

// out[s] = sum of x[perm[i]] (or x[i]) for i in [seg_off[s], seg_off[s+1]), accumulated in T
template <typename T>
__global__ void __launch_bounds__(kOpeThreads)
ope_seg_sum_kernel(const T* x, const int64_t* perm, const int64_t* off, T* out) {
  __shared__ double s_warp[kOpeThreads / 32];
  const int s = blockIdx.x;
  double acc = 0.0;
  for (int64_t i = off[s] + threadIdx.x; i < off[s + 1]; i += blockDim.x)
    acc += (double)x[perm ? perm[i] : i];
  const double t = block_sum_f64(acc, s_warp);
  if (threadIdx.x == 0) out[s] = (T)t;
}

// normalize_importance_weights for one row: w / column sum, or 1 / n where the column sums to 0
template <typename T>
__device__ __forceinline__ double norm_w(T w, T col, int n) {
  return col == (T)0 ? (double)((T)1 / (T)n) : (double)(w / col);
}

struct WsdrRet {
  int E, L, J, S;
  const int* off;
  const double* disc;
  const float* r;
  const int* js;
  const int* sub_off;
  double *ret, *sub_ret, *ev;
};

// calculate_step_return of every j-step for one trajectory, walking it once.  With prefix sums
// ISR(k) = sum_{s<=k} wd_s r_s and CV(k) = sum_{s<=k} (wd_s Q_s - wde_s V_s), where wd = disc * w
// and wde = disc * w_{s-1} (w_{-1} = 1/n):  ret_j = ISR(j) + wde_{j+1} V_{j+1} - CV(j), the middle
// term 0 past the trajectory (padding has V = 0).  Also the inf-step return under the weights of
// the trajectory's subset, and sum_s disc_s r_s.
template <typename T>
__global__ void __launch_bounds__(kOpeThreads)
ope_wsdr_returns_kernel(const WsdrRet a, const T* w, const T* sv, const T* ql, const T* col,
                        const T* sub_col) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.E) return;
  const int lo = a.off[e], len = a.off[e + 1] - lo;
  int sub = -1;
  for (int k = 0; k < a.S; ++k)
    if (e >= a.sub_off[k] && e < a.sub_off[k + 1]) sub = k;
  const int nsub = sub >= 0 ? a.sub_off[sub + 1] - a.sub_off[sub] : 1;
  double isr = 0.0, cv = 0.0, isr_s = 0.0, cv_s = 0.0, ev = 0.0;
  double prev = 1.0 / (double)a.E, prev_s = 1.0 / (double)nsub;
  for (int s = 0; s < len; ++s) {
    const int j = lo + s;
    const double d = a.disc[s], v = (double)sv[j], q = (double)ql[j], r = (double)a.r[j];
    const double wde = d * prev;
    for (int k = 0; k < a.J; ++k)
      if (a.js[k] == s - 1) a.ret[(size_t)k * a.E + e] = (isr + wde * v) - cv;
    const double wn = norm_w(w[j], col[s], a.E), wd = d * wn;
    isr += wd * r;
    cv += wd * q - wde * v;
    prev = wn;
    if (sub >= 0) {
      const double wns = norm_w(w[j], sub_col[(size_t)sub * a.L + s], nsub), wds = d * wns;
      isr_s += wds * r;
      cv_s += wds * q - d * prev_s * v;
      prev_s = wns;
    }
    ev += r * d;
  }
  for (int k = 0; k < a.J; ++k)
    if (a.js[k] >= len - 1) a.ret[(size_t)k * a.E + e] = isr - cv;
  a.sub_ret[e] = sub >= 0 ? isr_s - cv_s : 0.0;
  a.ev[e] = ev;
}

// np.cov(x) of [J, T] rows (ddof 1): one CTA per (j, k), j <= k, mirrored
__global__ void __launch_bounds__(kOpeThreads)
ope_cov_kernel(const double* x, int J, int T, double* cov) {
  __shared__ double s_warp[kOpeThreads / 32];
  __shared__ double s_mean[2];
  const int j = blockIdx.x, k = blockIdx.y;
  if (k < j) return;
  for (int h = 0; h < 2; ++h) {
    const double* row = x + (size_t)(h ? k : j) * T;
    double acc = 0.0;
    for (int t = threadIdx.x; t < T; t += blockDim.x) acc += row[t];
    const double m = block_sum_f64(acc, s_warp);
    if (threadIdx.x == 0) s_mean[h] = m / (double)T;
    __syncthreads();
  }
  const double mj = s_mean[0], mk = s_mean[1];
  double acc = 0.0;
  for (int t = threadIdx.x; t < T; t += blockDim.x)
    acc += (x[(size_t)j * T + t] - mj) * (x[(size_t)k * T + t] - mk);
  const double c = block_sum_f64(acc, s_warp);
  if (threadIdx.x == 0) cov[(size_t)j * J + k] = cov[(size_t)k * J + j] = c / (double)(T - 1);
}

}  // namespace rb200

using namespace rb200;

#define OPE_REQUIRE(cond, msg)                 \
  do {                                         \
    if (!(cond)) {                             \
      set_last_error("%s", msg);               \
      return RB200_E_INVALID;                  \
    }                                          \
  } while (0)

static dim3 ope_grid(int n) { return dim3((unsigned)ceil_div(n > 0 ? n : 1, kOpeThreads)); }

extern "C" int rb200_ope_page(int32_t n, int32_t A, int32_t K, const float* q, const float* reward_out,
                              const float* qcpe_out, const float* mask, const float* action,
                              const float* reward, const float* boost, float temperature,
                              float* boosted, float* prop, int64_t* eval_idx, float* mr_logged,
                              float* mm_logged, float* mmv_logged, void* stream) {
  OPE_REQUIRE(n > 0 && A > 0 && K >= 0, "rb200_ope_page: bad shape");
  OPE_REQUIRE(q && reward_out && qcpe_out && mask && action && reward && boosted && prop && eval_idx &&
                  mr_logged && (K == 0 || (mm_logged && mmv_logged)),
              "rb200_ope_page: required pointer is null");
  OPE_REQUIRE(temperature > 0.f, "rb200_ope_page: temperature must be positive");
  PageArgs a{n, A, K, q, reward_out, qcpe_out, mask, action, reward, boost, temperature,
             boosted, prop, eval_idx, mr_logged, mm_logged, mmv_logged};
  return launch<ope_page_kernel>(ope_grid(n), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                 "ope_page_kernel", a);
}

extern "C" int rb200_ope_episode_marks(int32_t n, const int64_t* mdp, const int64_t* seq,
                                       uint8_t* is_start, int32_t* flags, void* stream) {
  OPE_REQUIRE(n > 0 && mdp && seq && is_start && flags, "rb200_ope_episode_marks: bad argument");
  const int32_t init[2] = {n, 0};
  if (int rc = check_cuda(cudaMemcpyAsync(flags, init, sizeof(init), cudaMemcpyHostToDevice,
                                          (cudaStream_t)stream), "ope flags"))
    return rc;
  return launch<ope_marks_kernel>(ope_grid(n), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                  "ope_marks_kernel", n, mdp, seq, is_start, (int*)flags);
}

extern "C" int rb200_ope_logged_values(int32_t E, const int32_t* off, const float* disc, int32_t C,
                                       const float* x, float* out, void* stream) {
  OPE_REQUIRE(E > 0 && C > 0 && off && disc && x && out, "rb200_ope_logged_values: bad argument");
  return launch<ope_values_kernel>(ope_grid(E), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                   "ope_values_kernel", E, off, disc, C, x, out);
}

extern "C" int rb200_ope_sdr(int32_t E, const int32_t* off, int32_t A, const float* prop,
                             const float* qv, const float* am, const float* r, const float* lp,
                             float gamma, float* ep_dr, float* ep_val, void* stream) {
  OPE_REQUIRE(E > 0 && A > 0 && off && prop && qv && am && r && lp && ep_dr && ep_val,
              "rb200_ope_sdr: bad argument");
  return launch<ope_sdr_kernel>(ope_grid(E), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                "ope_sdr_kernel", E, off, A, prop, qv, am, r, lp, gamma, ep_dr, ep_val);
}

extern "C" int rb200_ope_dr_rows(int32_t n, int32_t A, const float* prop, const float* mr,
                                 const float* am, const float* r, const float* mrl, const float* lp,
                                 float* dm, float* ips, float* dr, void* stream) {
  OPE_REQUIRE(n > 0 && A > 0 && prop && mr && am && r && mrl && lp && dm && ips && dr,
              "rb200_ope_dr_rows: bad argument");
  return launch<ope_dr_rows_kernel>(ope_grid(n), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                    "ope_dr_rows_kernel", n, A, prop, mr, am, r, mrl, lp, dm, ips, dr);
}

extern "C" int rb200_ope_boot_means(const float* data, int32_t n, const int32_t* idx, int32_t samples,
                                    int32_t k, int64_t seed, int64_t offset, double* means,
                                    void* stream) {
  OPE_REQUIRE(data && means && n > 0 && samples > 0 && k > 0, "rb200_ope_boot_means: bad argument");
  return launch<ope_boot_kernel>(dim3(samples), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                 "ope_boot_kernel", data, n, (const int*)idx, k,
                                 (unsigned long long)seed, (unsigned long long)offset, means);
}

extern "C" int rb200_ope_wsdr_rows(int32_t E, const int32_t* off, int32_t A, int32_t fp64,
                                   const float* prop, const float* qv, const float* am,
                                   const float* lp, void* w, void* sv, void* ql, void* stream) {
  OPE_REQUIRE(E > 0 && A > 0 && A < 128 && off && prop && qv && am && lp && w && sv && ql,
              "rb200_ope_wsdr_rows: bad argument");
  if (fp64)
    return launch<ope_wsdr_rows_kernel<double>>(ope_grid(E), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                                "ope_wsdr_rows_kernel", E, off, A, prop, qv, am, lp,
                                                (double*)w, (double*)sv, (double*)ql);
  return launch<ope_wsdr_rows_kernel<float>>(ope_grid(E), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                             "ope_wsdr_rows_kernel", E, off, A, prop, qv, am, lp,
                                             (float*)w, (float*)sv, (float*)ql);
}

extern "C" int rb200_ope_seg_sum(int32_t fp64, const void* x, const int64_t* perm,
                                 const int64_t* seg_off, int32_t nseg, void* out, void* stream) {
  OPE_REQUIRE(x && seg_off && out && nseg > 0, "rb200_ope_seg_sum: bad argument");
  if (fp64)
    return launch<ope_seg_sum_kernel<double>>(dim3(nseg), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                              "ope_seg_sum_kernel", (const double*)x, perm, seg_off,
                                              (double*)out);
  return launch<ope_seg_sum_kernel<float>>(dim3(nseg), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                           "ope_seg_sum_kernel", (const float*)x, perm, seg_off,
                                           (float*)out);
}

extern "C" int rb200_ope_wsdr_returns(int32_t E, const int32_t* off, int32_t fp64, const void* w,
                                      const void* sv, const void* ql, const float* r,
                                      const double* disc, int32_t L, const void* col, int32_t J,
                                      const int32_t* js, int32_t S, const int32_t* sub_off,
                                      const void* sub_col, double* ret, double* sub_ret, double* ev,
                                      void* stream) {
  OPE_REQUIRE(E > 0 && L > 0 && J > 0 && J <= RB200_OPE_MAX_J && S >= 0 && off && w && sv && ql &&
                  r && disc && col && js && ret && sub_ret && ev && (S == 0 || (sub_off && sub_col)),
              "rb200_ope_wsdr_returns: bad argument");
  WsdrRet a{E, L, J, S, off, disc, r, js, sub_off, ret, sub_ret, ev};
  if (fp64)
    return launch<ope_wsdr_returns_kernel<double>>(
        ope_grid(E), dim3(kOpeThreads), 0, (cudaStream_t)stream, "ope_wsdr_returns_kernel", a,
        (const double*)w, (const double*)sv, (const double*)ql, (const double*)col, (const double*)sub_col);
  return launch<ope_wsdr_returns_kernel<float>>(
      ope_grid(E), dim3(kOpeThreads), 0, (cudaStream_t)stream, "ope_wsdr_returns_kernel", a,
      (const float*)w, (const float*)sv, (const float*)ql, (const float*)col, (const float*)sub_col);
}

extern "C" int rb200_ope_cov(const double* x, int32_t J, int32_t T, double* cov, void* stream) {
  OPE_REQUIRE(x && cov && J > 0 && J <= RB200_OPE_MAX_J && T > 0, "rb200_ope_cov: bad argument");
  return launch<ope_cov_kernel>(dim3(J, J), dim3(kOpeThreads), 0, (cudaStream_t)stream,
                                "ope_cov_kernel", x, J, T, cov);
}
