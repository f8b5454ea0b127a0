// reagent_b200 -- C-ABI plumbing: error text, validation, device queries.
#include <stdarg.h>
#include <string.h>
#include <stdio.h>

#include "rb200_common.cuh"

namespace rb200 {

static thread_local char g_err[512] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return RB200_OK;
  set_last_error("%s: %s", what, cudaGetErrorString(e));
  return RB200_E_CUDA;
}

int validate_mlp(const rb200_mlp_t* d, const char* name) {
  if (d->n_layers < 1 || d->n_layers > RB200_MAX_LAYERS) {
    set_last_error("%s: n_layers=%d out of range [1,%d]", name, d->n_layers, RB200_MAX_LAYERS);
    return RB200_E_INVALID;
  }
  if (!d->params) { set_last_error("%s: params is null", name); return RB200_E_INVALID; }
  for (int l = 0; l <= d->n_layers; ++l)
    if (d->dims[l] <= 0) { set_last_error("%s: dims[%d]=%d", name, l, d->dims[l]); return RB200_E_INVALID; }
  for (int l = 0; l < d->n_layers; ++l) {
    if (d->act[l] < RB200_ACT_LINEAR || d->act[l] > RB200_ACT_SOFTPLUS) {
      set_last_error("%s: unsupported activation %d at layer %d", name, d->act[l], l);
      return RB200_E_INVALID;
    }
    const long long wend = d->w_off[l] + (long long)d->dims[l] * d->dims[l + 1];
    const long long bend = d->b_off[l] + d->dims[l + 1];
    if (d->w_off[l] < 0 || d->b_off[l] < 0 || wend > d->n_params || bend > d->n_params) {
      set_last_error("%s: layer %d offsets outside the arena", name, l);
      return RB200_E_INVALID;
    }
  }
  return RB200_OK;
}

}  // namespace rb200

extern "C" const char* rb200_last_error(void) { return rb200::g_err; }
extern "C" int rb200_version(void) { return RB200_VERSION; }

// sizeof() of the structs that cross the C ABI, so that a binding (ctypes / cgo / JNI) can
// check its own mirror against the library it loaded
extern "C" int64_t rb200_abi_sizeof(const char* type_name) {
  if (!type_name) return -1;
#define RB200_SZ(T) if (!strcmp(type_name, #T)) return (int64_t)sizeof(T)
  RB200_SZ(rb200_mlp_t);
  RB200_SZ(rb200_net_ws_t);
  RB200_SZ(rb200_feature_col_t);
  RB200_SZ(rb200_dqn_args_t);
  RB200_SZ(rb200_qrdqn_args_t);
  RB200_SZ(rb200_ac_args_t);
  RB200_SZ(rb200_adam_args_t);
  RB200_SZ(rb200_gather_spec_t);
  RB200_SZ(rb200_sample_args_t);
  RB200_SZ(rb200_replay_dev_t);
  RB200_SZ(rb200_cpe_args_t);
  RB200_SZ(rb200_pdqn_args_t);
  RB200_SZ(rb200_slateq_args_t);
  RB200_SZ(rb200_c51_args_t);
  RB200_SZ(rb200_bc_xent_args_t);
  RB200_SZ(rb200_crr_critic_args_t);
  RB200_SZ(rb200_crr_actor_args_t);
  RB200_SZ(rb200_pg_returns_args_t);
  RB200_SZ(rb200_pg_head_args_t);
  RB200_SZ(rb200_add_args_t);
  RB200_SZ(rb200_per_draw_args_t);
  RB200_SZ(rb200_per_exchange_args_t);
  RB200_SZ(rb200_mdnrnn_args_t);
  RB200_SZ(rb200_mdnrnn_eval_args_t);
  RB200_SZ(rb200_mdnrnn_fill_args_t);
  RB200_SZ(rb200_mdnrnn_sensitivity_args_t);
  RB200_SZ(rb200_cem_args_t);
  RB200_SZ(rb200_seq2reward_args_t);
  RB200_SZ(rb200_seq2reward_plan_args_t);
  RB200_SZ(rb200_seq2reward_compress_args_t);
  RB200_SZ(rb200_seq2slate_args_t);
#undef RB200_SZ
  return -1;
}
extern "C" int rb200_device_info(int* sm_count, int* max_smem_optin) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return rb200::check_cuda(e, "cudaGetDevice");
  if (sm_count) {
    e = cudaDeviceGetAttribute(sm_count, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return rb200::check_cuda(e, "cudaDeviceGetAttribute(sm count)");
  }
  if (max_smem_optin) {
    e = cudaDeviceGetAttribute(max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (e != cudaSuccess) return rb200::check_cuda(e, "cudaDeviceGetAttribute(smem optin)");
  }
  return RB200_OK;
}
