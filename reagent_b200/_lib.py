"""ctypes binding of libreagent_b200.so (the C ABI in include/reagent_b200.h).

The product path has NO fallback: if the CUDA library is missing or a call fails this
module raises.  Build with `python -c "import __graft_entry__ as g; g.build()"` or
`reagent_b200/csrc/build.sh`.
"""
import ctypes as C
import os

MAX_LAYERS = 8

ACT = {"linear": 0, "relu": 1, "tanh": 2, "leaky_relu": 3, "sigmoid": 4, "softplus": 5}
E_SMEM = -3  # RB200_E_SMEM: a row tile does not fit in shared memory
LOSS_MSE, LOSS_HUBER = 0, 1
DISCOUNT_CONST, DISCOUNT_POW = 0, 1

_f32p = C.POINTER(C.c_float)
_vp = C.c_void_p


class MlpT(C.Structure):
    _fields_ = [
        ("n_layers", C.c_int32),
        ("dims", C.c_int32 * (MAX_LAYERS + 1)),
        ("act", C.c_int32 * MAX_LAYERS),
        ("params", _vp),
        ("w_off", C.c_int64 * MAX_LAYERS),
        ("b_off", C.c_int64 * MAX_LAYERS),
        ("n_params", C.c_int64),
    ]


class NetWsT(C.Structure):
    _fields_ = [
        ("hidden", _vp * MAX_LAYERS),
        ("dz", _vp * MAX_LAYERS),
        ("input", _vp),
    ]


class DqnArgsT(C.Structure):
    _fields_ = [
        ("batch", C.c_int32),
        ("state", _vp),
        ("next_state", _vp),
        ("action", _vp),
        ("next_action", _vp),
        ("reward", _vp),
        ("not_terminal", _vp),
        ("possible_next_actions_mask", _vp),
        ("discount_src", _vp),
        ("reward_boost", _vp),
        ("gamma", C.c_float),
        ("discount_mode", C.c_int32),
        ("double_q", C.c_int32),
        ("maxq", C.c_int32),
        ("loss_kind", C.c_int32),
        ("do_backward", C.c_int32),
        ("all_action_scores", _vp),
        ("td_target", _vp),
        ("q_selected", _vp),
        ("next_action_idx", _vp),
        ("loss_partials", _vp),
        ("loss", _vp),
        ("tile_counter", _vp),
        ("sample_weight", _vp),
    ]


class AdamArgsT(C.Structure):
    _fields_ = [
        ("params", _vp),
        ("grad", _vp),
        ("splits", C.c_int32),
        ("n", C.c_int64),
        ("exp_avg", _vp),
        ("exp_avg_sq", _vp),
        ("step", _vp),
        ("block_counter", _vp),
        ("lr", C.c_double),
        ("beta1", C.c_double),
        ("beta2", C.c_double),
        ("eps", C.c_double),
        ("weight_decay", C.c_double),
        ("grad_scale", C.c_float),
        ("target", _vp),
        ("tau", C.c_float),
        ("one_minus_tau", C.c_float),
        ("exp_out", _vp),
        ("tc_net", C.POINTER(MlpT)),
        ("tc_pack_ws", _vp),
        ("tc_pack_ws_bytes", C.c_int64),
        ("tc_do_backward", C.c_int32),
        ("dp_world", C.c_int32),
        ("dp_rank", C.c_int32),
        ("dp_recv", _vp),
        ("dp_flags", _vp),
        ("dp_stride", C.c_int64),
        ("dp_max_blocks", C.c_int32),
        ("decoupled_weight_decay", C.c_int32),
        ("amsgrad", C.c_int32),
        ("max_exp_avg_sq", _vp),
    ]


ALGO_SAC, ALGO_TD3 = 0, 1
CRR_NONE, CRR_INDICATOR, CRR_EXPONENT = 0, 1, 2


class AcArgsT(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("algo", C.c_int32),
        ("state", _vp), ("action", _vp), ("next_state", _vp), ("reward", _vp),
        ("not_terminal", _vp), ("noise_next", _vp), ("noise_cur", _vp),
        ("gamma", C.c_float), ("alpha", _vp), ("log_alpha", _vp),
        ("target_entropy", C.c_float), ("backprop_through_log_prob", C.c_int32),
        ("noise_variance", C.c_float), ("noise_clip", C.c_float),
        ("loss_partials", _vp), ("loss", _vp), ("tile_counter", _vp), ("alpha_grad", _vp),
        ("td_target", _vp), ("next_action_out", _vp), ("log_prob_out", _vp),
        ("q1_value", _vp), ("q2_value", _vp),
        ("value_target", C.POINTER(MlpT)), ("value_net", C.POINTER(MlpT)), ("min_q_out", _vp),
        ("crr_mode", C.c_int32), ("crr_threshold", C.c_float), ("crr_beta", C.c_float),
        ("crr_clamp", C.c_float), ("logged_action_uniform_prior", C.c_int32),
        ("sample_weight", _vp), ("td_error_out", _vp),
    ]


class FeatureColT(C.Structure):
    _fields_ = [("src_col", C.c_int32), ("type", C.c_int32), ("p0", C.c_float), ("p1", C.c_float),
                ("p2", C.c_float), ("p3", C.c_float), ("q_off", C.c_int32), ("q_cnt", C.c_int32)]


MAX_GATHER_SPECS = 12
VALID_BLOCK = 256
SAMPLE_PRIORITIZED, SAMPLE_UNIFORM, SAMPLE_GIVEN = 0, 1, 2


class GatherSpecT(C.Structure):
    _fields_ = [("src", _vp), ("dst", _vp), ("row_bytes", C.c_int32), ("which", C.c_int32)]


class SampleArgsT(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("capacity", C.c_int32), ("update_horizon", C.c_int32),
        ("mode", C.c_int32), ("timeline_next", C.c_int32),
        ("tree", _vp), ("tree_depth", C.c_int32), ("query", _vp),
        ("override_pos", _vp), ("override_idx", _vp), ("n_override", C.c_int32),
        ("ranks", _vp), ("valid", _vp), ("valid_block_offsets", _vp),
        ("n_valid_blocks", C.c_int32), ("indices_in", _vp),
        ("terminal", _vp), ("reward", _vp), ("decays", _vp),
        ("obs", _vp), ("obs_dim", C.c_int32), ("obs_out_dim", C.c_int32),
        ("cols", _vp), ("quantiles", _vp), ("state", _vp), ("next_state", _vp),
        ("action_i64", _vp), ("num_actions", C.c_int32),
        ("action_out_i64", _vp), ("next_action_out_i64", _vp),
        ("action_onehot", _vp), ("next_action_onehot", _vp),
        ("action_f32", _vp), ("action_dim", C.c_int32),
        ("action_out_raw", _vp), ("next_action_out_raw", _vp),
        ("action_rescaled", _vp), ("next_action_rescaled", _vp),
        ("action_low", _vp), ("action_high", _vp),
        ("train_low", C.c_float), ("train_high", C.c_float),
        ("reward_out", _vp), ("next_reward_out", _vp), ("terminal_out", _vp),
        ("not_terminal_out", _vp), ("indices_out", _vp), ("step_out", _vp),
        ("step_f32_out", _vp), ("sampling_prob_out", _vp),
        ("n_specs", C.c_int32), ("specs", GatherSpecT * MAX_GATHER_SPECS),
    ]


class PdqnArgsT(C.Structure):
    _fields_ = [("batch", C.c_int32), ("max_num_action", C.c_int32), ("next_q", _vp),
                ("next_q_target", _vp), ("mask", _vp), ("reward", _vp), ("not_terminal", _vp),
                ("discount_src", _vp), ("gamma", C.c_float), ("discount_mode", C.c_int32),
                ("double_q", C.c_int32), ("loss_kind", C.c_int32), ("q_values", _vp), ("dz", _vp),
                ("td_target", _vp), ("loss_partials", _vp), ("loss", _vp), ("tile_counter", _vp)]


class C51ArgsT(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_actions", C.c_int32), ("num_atoms", C.c_int32),
                ("logits_next_online", _vp), ("logits_next_target", _vp), ("logits_cur", _vp),
                ("action", _vp), ("next_action", _vp), ("possible_next_actions_mask", _vp),
                ("reward", _vp), ("not_terminal", _vp), ("discount_src", _vp),
                ("reward_boost", _vp), ("support", _vp), ("gamma", C.c_float), ("qmin", C.c_float),
                ("qmax", C.c_float), ("scale_support", C.c_float), ("double_q", C.c_int32),
                ("maxq", C.c_int32), ("dz_logits", _vp), ("all_q_values", _vp),
                ("next_action_idx", _vp), ("loss_partials", _vp), ("loss", _vp),
                ("tile_counter", _vp), ("sample_weight", _vp)]


BC_ROWS_PER_BLOCK = 8  # rb200_bc_xent_head: loss_partials holds ceil(batch / 8) floats


class BcXentArgsT(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_actions", C.c_int32), ("logits", _vp),
                ("labels", _vp), ("mask", _vp), ("dz", _vp), ("loss_partials", _vp),
                ("loss", _vp), ("tile_counter", _vp)]


CRR_ROWS_PER_BLOCK = 16  # rb200_crr_*_head: loss_partials holds 2 * ceil(batch / 16) floats


class CrrCriticArgsT(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_actions", C.c_int32), ("actor_next", _vp),
                ("noise_next", _vp), ("q1_target_next", _vp), ("q2_target_next", _vp),
                ("q1", _vp), ("q2", _vp), ("action", _vp), ("reward", _vp),
                ("reward_boost", _vp), ("not_terminal", _vp), ("gamma", C.c_float),
                ("td_target", _vp), ("q1_selected", _vp), ("q2_selected", _vp), ("dz_q1", _vp),
                ("dz_q2", _vp), ("loss_partials", _vp), ("loss", _vp), ("tile_counter", _vp)]


class CrrActorArgsT(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_actions", C.c_int32), ("actor_out", _vp),
                ("noise", _vp), ("q1", _vp), ("action", _vp), ("action_probability", _vp),
                ("inv_beta", C.c_float), ("max_weight", C.c_float), ("entropy_coeff", C.c_float),
                ("clip_limit", C.c_float), ("action_activation", C.c_int32), ("weight", _vp),
                ("dz", _vp), ("loss_partials", _vp), ("loss", _vp), ("tile_counter", _vp)]


PG_ROWS_PER_BLOCK = 8  # rb200_pg_head: loss_partials holds 2 * ceil(rows / 8) floats
PG_NORM_NONE, PG_NORM_WHITEN, PG_NORM_WHITEN_NO_MEAN, PG_NORM_SUBTRACT_MEAN = 0, 1, 2, 3
PG_LOSS_REINFORCE, PG_LOSS_PPO = 0, 1
PG_ADV_RETURNS, PG_ADV_BASELINE, PG_ADV_TD = 0, 1, 2


class PgReturnsArgsT(C.Structure):
    _fields_ = [("n_traj", C.c_int32), ("offsets", _vp), ("reward", _vp),
                ("reward_clip", C.c_float), ("gamma", C.c_float), ("norm", C.c_int32),
                ("offset_clamp_min", C.c_int32), ("returns", _vp)]


class PgHeadArgsT(C.Structure):
    _fields_ = [("rows", C.c_int32), ("num_actions", C.c_int32), ("n_traj", C.c_int32),
                ("offsets", _vp), ("scores", _vp), ("mask", _vp), ("action", _vp),
                ("logged_log_prob", _vp), ("returns", _vp), ("value", _vp),
                ("next_value", _vp), ("reward", _vp), ("not_terminal", _vp),
                ("temperature", C.c_float), ("gamma", C.c_float), ("reward_clip", C.c_float),
                ("log_clip_param", C.c_float), ("entropy_weight", C.c_float),
                ("ppo_clip_lo", C.c_float), ("ppo_clip_hi", C.c_float), ("value_scale", C.c_float),
                ("loss_kind", C.c_int32), ("advantage_kind", C.c_int32),
                ("offset_clamp_min", C.c_int32), ("advantage_out", _vp), ("dz", _vp),
                ("dz_value", _vp), ("loss_partials", _vp), ("loss", _vp),
                ("tile_counter", _vp)]


class CpeArgsT(C.Structure):
    _fields_ = [("batch", C.c_int32), ("num_actions", C.c_int32), ("num_metrics", C.c_int32),
                ("next_scores", _vp), ("mask", _vp), ("temperature", C.c_float), ("action", _vp),
                ("metrics_reward", _vp), ("discount_src", _vp), ("gamma", C.c_float),
                ("discount_mode", C.c_int32), ("not_terminal", _vp), ("reward_est", _vp),
                ("qcpe", _vp), ("qcpe_target_next", _vp), ("loss_kind", C.c_int32),
                ("dz_reward", _vp), ("dz_qcpe", _vp), ("propensities_next", _vp),
                ("loss_partials", _vp), ("loss", _vp), ("tile_counter", _vp)]


class ReplayDevT(C.Structure):
    _fields_ = [("state", _vp), ("capacity", C.c_int32), ("update_horizon", C.c_int32),
                ("valid", _vp), ("terminal", _vp), ("reward", _vp), ("tree", _vp),
                ("tree_depth", C.c_int32), ("max_priority", _vp)]


class AddArgsT(C.Structure):
    _fields_ = [("rb", ReplayDevT), ("n", C.c_int32), ("terminal_in", _vp), ("reward_in", _vp),
                ("priority_in", _vp), ("n_rows", C.c_int32),
                ("rows", GatherSpecT * MAX_GATHER_SPECS), ("priority_from_max", C.c_int32)]


class PerDrawArgsT(C.Structure):
    _fields_ = [("mt_state", _vp), ("batch", C.c_int32), ("lo", _vp), ("hi", _vp), ("tree", _vp),
                ("tree_depth", C.c_int32), ("valid", _vp), ("max_attempts", C.c_int32),
                ("indices_out", _vp), ("queries_out", _vp), ("status", _vp)]


class QrdqnArgsT(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("num_actions", C.c_int32), ("num_atoms", C.c_int32),
        ("q_next_online", _vp), ("q_next_target", _vp), ("q_cur", _vp), ("action", _vp),
        ("next_action", _vp), ("possible_next_actions_mask", _vp), ("reward", _vp),
        ("not_terminal", _vp), ("discount_src", _vp), ("reward_boost", _vp),
        ("gamma", C.c_float), ("double_q", C.c_int32), ("maxq", C.c_int32),
        ("dz_head", _vp), ("all_q_values", _vp), ("next_action_idx", _vp),
        ("loss_partials", _vp), ("loss", _vp), ("tile_counter", _vp),
        ("sample_weight", _vp),
    ]


MDNRNN_MAX_LAYERS = 4
MDNRNN_ROWS_PER_BLOCK = 16  # rb200_mdnrnn_forward: loss_partials holds 3 * ceil(batch / 16) floats


class MdnrnnArgsT(C.Structure):
    _fields_ = [
        ("seq_len", C.c_int32), ("batch", C.c_int32), ("state_dim", C.c_int32),
        ("action_dim", C.c_int32), ("hidden", C.c_int32), ("layers", C.c_int32),
        ("gaussians", C.c_int32), ("params", _vp), ("n_params", C.c_int64),
        ("w_ih_off", C.c_int64 * MDNRNN_MAX_LAYERS), ("w_hh_off", C.c_int64 * MDNRNN_MAX_LAYERS),
        ("b_ih_off", C.c_int64 * MDNRNN_MAX_LAYERS), ("b_hh_off", C.c_int64 * MDNRNN_MAX_LAYERS),
        ("w_gmm_off", C.c_int64), ("b_gmm_off", C.c_int64),
        ("state", _vp), ("action", _vp), ("next_state", _vp), ("reward", _vp),
        ("not_terminal", _vp), ("next_state_weight", C.c_float),
        ("not_terminal_weight", C.c_float), ("reward_weight", C.c_float),
        ("gmm_divisor", C.c_float), ("fit_only_one_next_step", C.c_int32),
        ("out", _vp), ("hs", _vp), ("cs", _vp), ("xin", _vp), ("acts", _vp), ("dgates", _vp),
        ("dy", _vp), ("loss_partials", _vp), ("tile_counter", _vp), ("loss", _vp),
        ("gpart", _vp), ("splits", C.c_int32),
    ]


CEM_MAX_MODELS = 8
CEM_ROWS_PER_BLOCK = 16


class CemArgsT(C.Structure):
    _fields_ = [
        ("net", MdnrnnArgsT), ("num_models", C.c_int32), ("params", _vp * CEM_MAX_MODELS),
        ("population", C.c_int32), ("horizon", C.c_int32), ("iters", C.c_int32),
        ("num_elites", C.c_int32), ("discrete", C.c_int32), ("terminal_effective", C.c_int32),
        ("iter", C.c_int32), ("alpha", C.c_double), ("epsilon", C.c_double),
        ("state", _vp), ("discount", _vp), ("lower", _vp), ("upper", _vp),
        ("model_idx", _vp), ("action_idx", _vp), ("truncnorm", _vp), ("step_noise", _vp),
        ("mean", _vp), ("var", _vp), ("values", _vp), ("elites", _vp), ("mean_hist", _vp),
        ("var_hist", _vp), ("done", _vp), ("n_iters", _vp), ("action_out", _vp),
        ("one_hot", _vp), ("counter", _vp), ("dump", _vp),
    ]


class Rb200Error(RuntimeError):
    pass


_LIB = None
# RB200_LIB selects another build of the SAME library (e.g. the profiling build with the
# clock64 timeline compiled in); there is no other implementation to fall back to.
LIB_PATH = os.environ.get("RB200_LIB") or os.path.join(
    os.path.dirname(os.path.abspath(__file__)), "libreagent_b200.so")


def _declare(lib):
    lib.rb200_last_error.restype = C.c_char_p
    lib.rb200_version.restype = C.c_int
    lib.rb200_abi_sizeof.argtypes = [C.c_char_p]
    lib.rb200_abi_sizeof.restype = C.c_int64
    lib.rb200_device_info.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.rb200_num_row_tiles.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.rb200_dqn_td_step.argtypes = [C.POINTER(MlpT), C.POINTER(MlpT), C.POINTER(DqnArgsT),
                                      C.POINTER(NetWsT), _vp]
    lib.rb200_dueling_scratch_floats.argtypes = [C.c_int32, C.c_int32]
    lib.rb200_dueling_scratch_floats.restype = C.c_int64
    lib.rb200_dueling_fold.argtypes = [_vp, _vp, _vp, _vp, C.c_int32, C.c_int32, C.c_int32, _vp, _vp,
                                       _vp, _vp]
    lib.rb200_dueling_unfold.argtypes = [_vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                         C.c_int64, _vp, _vp]
    lib.rb200_dqn_tc_workspace_bytes.argtypes = [C.POINTER(MlpT), C.c_int32, C.c_int32]
    lib.rb200_dqn_tc_workspace_bytes.restype = C.c_int64
    lib.rb200_dqn_tc_pack.argtypes = [C.POINTER(MlpT), C.POINTER(MlpT), C.c_int32, C.c_int32, _vp,
                                      C.c_int64, _vp]
    lib.rb200_dqn_td_step_tc.argtypes = [C.POINTER(MlpT), C.POINTER(MlpT), C.POINTER(DqnArgsT),
                                         C.POINTER(NetWsT), _vp, C.c_int64, C.c_int32, _vp]
    lib.rb200_mlp_forward.argtypes = [C.POINTER(MlpT), _vp, C.c_int32, _vp, C.c_int32, C.c_int32,
                                      _vp, C.POINTER(NetWsT), _vp]
    lib.rb200_mlp_forward_tiled.argtypes = [C.POINTER(MlpT), C.POINTER(MlpT), _vp, C.c_int32, _vp,
                                            C.c_int32, C.c_int32, C.c_int32, _vp, _vp, _vp]
    lib.rb200_linear_forward.argtypes = [_vp, _vp, C.c_int32, C.c_int32, C.c_int32, _vp,
                                         C.c_int32, _vp, _vp]
    lib.rb200_linear_backward_dx.argtypes = [_vp, C.c_int32, C.c_int32, _vp, _vp, C.c_int32,
                                             C.c_int32, _vp, _vp]
    lib.rb200_linear_backward_dx_tc_scratch_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.rb200_linear_backward_dx_tc_scratch_bytes.restype = C.c_int64
    lib.rb200_linear_backward_dx_tc.argtypes = [_vp, C.c_int32, C.c_int32, _vp, _vp, C.c_int32,
                                                C.c_int32, _vp, _vp, C.c_int64, _vp]
    lib.rb200_mlp_backward.argtypes = [C.POINTER(MlpT), _vp, C.c_int32, C.POINTER(NetWsT), _vp]
    lib.rb200_qrdqn_head.argtypes = [C.POINTER(QrdqnArgsT), _vp]
    lib.rb200_preprocess.argtypes = [_vp, _vp, C.c_int32, C.c_int64, C.c_int32, C.c_int32, _vp,
                                     _vp, _vp, _vp]
    lib.rb200_replay_sample.argtypes = [C.POINTER(SampleArgsT), _vp]
    lib.rb200_valid_index_build.argtypes = [_vp, C.c_int64, _vp, _vp, _vp]
    lib.rb200_mt19937_uniform_host.argtypes = [_vp, C.POINTER(C.c_int32), _vp, _vp, _vp, C.c_int64]
    lib.rb200_mt19937_uniform_host.restype = None
    lib.rb200_sumtree_set_host.argtypes = [_vp, C.c_int32, _vp, _vp, C.c_int64, _vp]
    lib.rb200_sumtree_sample_host.argtypes = [_vp, C.c_int32, C.c_double]
    lib.rb200_sumtree_sample_host.restype = C.c_int64
    lib.rb200_sumtree_sample_many_host.argtypes = [_vp, C.c_int32, _vp, _vp, C.c_int64, _vp]
    lib.rb200_sumtree_sample_many_host.restype = None
    lib.rb200_replay_add_batch_host.argtypes = [_vp, C.c_int64, C.c_int64, C.c_int32, _vp, _vp, _vp]
    lib.rb200_replay_add_batch_host.restype = None
    lib.rb200_ac_critic_step.argtypes = [C.POINTER(MlpT), C.POINTER(MlpT), C.POINTER(MlpT),
                                         C.POINTER(MlpT), C.POINTER(MlpT), C.POINTER(AcArgsT),
                                         C.POINTER(NetWsT), C.POINTER(NetWsT), _vp]
    lib.rb200_ac_actor_step.argtypes = [C.POINTER(MlpT), C.POINTER(MlpT), C.POINTER(MlpT),
                                        C.POINTER(AcArgsT), C.POINTER(NetWsT), C.POINTER(NetWsT),
                                        C.POINTER(NetWsT), _vp]
    lib.rb200_ac_value_step.argtypes = [C.POINTER(MlpT), C.POINTER(AcArgsT), C.POINTER(NetWsT), _vp]
    lib.rb200_wgrad_splits.argtypes = [C.c_int]
    lib.rb200_wgrad_splits_for.argtypes = [C.POINTER(MlpT), C.c_int32]
    lib.rb200_mlp_wgrad.argtypes = [C.POINTER(MlpT), _vp, C.c_int32, C.POINTER(NetWsT), _vp,
                                    C.c_int32, _vp]
    lib.rb200_grad_reduce.argtypes = [_vp, C.c_int32, C.c_int64, _vp, _vp]
    lib.rb200_adam_soft_update.argtypes = [C.POINTER(AdamArgsT), _vp]
    lib.rb200_soft_update.argtypes = [_vp, _vp, C.c_int64, C.c_float, C.c_float, _vp]
    lib.rb200_cpe_heads.argtypes = [C.POINTER(CpeArgsT), _vp]
    lib.rb200_bcq_filter.argtypes = [_vp, C.c_int32, C.c_int32, C.c_float, _vp, _vp, _vp, _vp, _vp]
    lib.rb200_pdqn_head.argtypes = [C.POINTER(PdqnArgsT), _vp]
    lib.rb200_c51_head.argtypes = [C.POINTER(C51ArgsT), _vp]
    lib.rb200_bc_xent_head.argtypes = [C.POINTER(BcXentArgsT), _vp]
    lib.rb200_crr_critic_head.argtypes = [C.POINTER(CrrCriticArgsT), _vp]
    lib.rb200_crr_actor_head.argtypes = [C.POINTER(CrrActorArgsT), _vp]
    lib.rb200_pg_returns.argtypes = [C.POINTER(PgReturnsArgsT), _vp]
    lib.rb200_pg_head.argtypes = [C.POINTER(PgHeadArgsT), _vp]
    lib.rb200_replay_add_device.argtypes = [C.POINTER(AddArgsT), _vp]
    lib.rb200_sumtree_set_device.argtypes = [_vp, C.c_int32, _vp, _vp, C.c_int32, _vp, _vp, _vp]
    lib.rb200_per_draw_indices.argtypes = [C.POINTER(PerDrawArgsT), _vp]
    lib.rb200_per_weights.argtypes = [_vp, C.c_int32, _vp, C.c_int32, _vp, C.c_double, C.c_double,
                                      _vp, _vp, _vp]
    lib.rb200_per_priority_update.argtypes = [_vp, C.c_int32, _vp, _vp, _vp, C.c_int32, C.c_double,
                                              C.c_double, _vp, _vp, _vp, _vp]
    lib.rb200_per_priority_update_rows.argtypes = [_vp, C.c_int32, _vp, _vp, C.c_int32, C.c_double,
                                                   C.c_double, C.c_double, _vp, _vp, _vp, _vp]
    lib.rb200_mdnrnn_check_shape.argtypes = [C.c_int32] * 5
    for f in ("rb200_mdnrnn_forward", "rb200_mdnrnn_backward", "rb200_mdnrnn_wgrad"):
        getattr(lib, f).argtypes = [C.POINTER(MdnrnnArgsT), _vp]
    lib.rb200_cem_check_shape.argtypes = [C.c_int32] * 9
    lib.rb200_cem_rollout.argtypes = [C.POINTER(CemArgsT), _vp]
    lib.rb200_adam_blocks.argtypes = [C.c_int64]
    lib.rb200_dp_alloc.argtypes = [C.c_int64, C.POINTER(_vp)]
    lib.rb200_dp_free.argtypes = [_vp]
    lib.rb200_dp_ipc_handle.argtypes = [_vp, _vp]
    lib.rb200_dp_ipc_open.argtypes = [_vp, C.POINTER(_vp)]
    lib.rb200_dp_ipc_close.argtypes = [_vp]


def lib():
    """Load (once) and return the shared library; raise loudly if it is missing."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise Rb200Error(
                f"{LIB_PATH} not found: the CUDA extension is not built. "
                "Run reagent_b200/csrc/build.sh (there is no CPU fallback).")
        _LIB = C.CDLL(LIB_PATH)
        _declare(_LIB)
    return _LIB


def check(rc, what=""):
    if rc != 0:
        msg = lib().rb200_last_error().decode("utf-8", "replace")
        raise Rb200Error(f"{what} failed (rc={rc}): {msg}")


def ptr(t, device=None):
    """Device pointer of a torch tensor (None -> NULL).  A host tensor -- or one on another
    GPU than `device` -- would reach the kernel as a wild pointer (illegal address, sticky
    context error), so it is refused here with a Python exception instead."""
    if t is None:
        return None
    if not t.is_cuda:
        raise Rb200Error("reagent_b200: a CPU tensor reached a CUDA entry point (call "
                         "trainer.cuda() / batch.cuda() first; there is no CPU path)")
    if device is not None and t.device != device:
        raise Rb200Error(f"reagent_b200: tensor on {t.device}, expected {device}")
    return t.data_ptr()


def on_device(t, device):
    """`t` on `device` (moved once if it was created elsewhere, e.g. trainer-owned constants
    of a trainer that was built from already-CUDA networks and never .cuda()'d)."""
    if t is None or (t.is_cuda and t.device == device):
        return t
    return t.to(device)


def cur_stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


def require_current_device(device):
    """Launches go to the CURRENT device's stream; tensors elsewhere would be wild pointers
    there.  Multi-GPU callers run one process per GPU or wrap calls in torch.cuda.device()."""
    import torch

    if device.type != "cuda" or torch.cuda.current_device() != (device.index or 0):
        raise Rb200Error(f"reagent_b200: tensors live on {device} but the current CUDA device is "
                         f"cuda:{torch.cuda.current_device()} -- wrap the call in "
                         f"torch.cuda.device({device.index})")
