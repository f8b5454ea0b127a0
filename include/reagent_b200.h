/* reagent_b200 -- C ABI of the H100-native off-policy training hot path.
 *
 * The reference (facebookresearch/ReAgent) has no FFI for this path: it is plain
 * Python over torch (SURVEY.md section 8b).  This header is the boundary one level
 * beneath the Python surface: every entry point replaces a chain of eager aten ops
 * in the reference file:line it cites.  All pointers are DEVICE pointers except:
 *   - a pointer to an rb200_*_t struct, parameter or field: a HOST descriptor
 *     (rb200_mlp_t, rb200_net_ws_t, the *_args_t, ...) read during the call.  The one
 *     exception is rb200_feature_col_t, whose pointers are device arrays;
 *   - a parameter whose name ends in `_host`.
 * Every function takes the CUDA stream to launch on (as void*), owns no memory, starts
 * no threads and returns 0 on success or a negative RB200_E_* code (text via
 * rb200_last_error()).
 */
#ifndef REAGENT_B200_H_
#define REAGENT_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RB200_VERSION 1
#define RB200_MAX_LAYERS 8

#define RB200_OK 0
#define RB200_E_INVALID (-1)   /* bad argument / unsupported shape            */
#define RB200_E_CUDA (-2)      /* CUDA runtime error                          */
#define RB200_E_SMEM (-3)      /* tile does not fit in 227 KB shared memory   */

/* activations: reagent/models/fully_connected_network.py:37-44 */
#define RB200_ACT_LINEAR 0
#define RB200_ACT_RELU 1
#define RB200_ACT_TANH 2
#define RB200_ACT_LEAKY_RELU 3
#define RB200_ACT_SIGMOID 4
#define RB200_ACT_SOFTPLUS 5

/* losses: reagent/training/dqn_trainer_base.py:146-155 */
#define RB200_LOSS_MSE 0
#define RB200_LOSS_HUBER 1

/* discount modes: reagent/training/dqn_trainer.py:166-177 */
#define RB200_DISCOUNT_CONST 0     /* gamma                          */
#define RB200_DISCOUNT_POW 1       /* gamma ** discount_src[b]       */

/* One fully connected network (reagent/models/fully_connected_network.py:67-163,
 * in-scope subset: Linear + activation, no BN/LN/dropout/residual).  Parameters live
 * in one flat fp32 arena; layer l's weight is [dims[l+1], dims[l]] row-major at
 * params + w_off[l] (== nn.Linear.weight), its bias at params + b_off[l]. */
typedef struct rb200_mlp {
  int32_t n_layers;
  int32_t dims[RB200_MAX_LAYERS + 1];
  int32_t act[RB200_MAX_LAYERS];
  const float* params;
  int64_t w_off[RB200_MAX_LAYERS];
  int64_t b_off[RB200_MAX_LAYERS];
  int64_t n_params; /* arena length in floats (including alignment padding) */
} rb200_mlp_t;

/* Per-network training workspace (caller allocated, all dense row-major):
 *   hidden[l]  [B, dims[l+1]]  output of layer l, l < n_layers-1
 *   dz[l]      [B, dims[l+1]]  dLoss/d(pre-activation of layer l)
 *   input      [B, dims[0]]    the (concatenated) network input, or NULL when the
 *                              batch tensor itself is the input               */
typedef struct rb200_net_ws {
  float* hidden[RB200_MAX_LAYERS];
  float* dz[RB200_MAX_LAYERS];
  float* input;
} rb200_net_ws_t;

/* feature types: reagent/preprocessing/identify_types.py:9-30 (FEATURE_TYPES order) */
#define RB200_FT_BINARY 0
#define RB200_FT_PROBABILITY 1
#define RB200_FT_CONTINUOUS 2
#define RB200_FT_BOXCOX 3
#define RB200_FT_ENUM 4
#define RB200_FT_QUANTILE 5
#define RB200_FT_CONTINUOUS_ACTION 6
#define RB200_FT_DISCRETE_ACTION 7
#define RB200_FT_DO_NOT_PREPROCESS 8
#define RB200_FT_CLIP_LOG 9

/* One OUTPUT column of the dense preprocessor (reagent/preprocessing/preprocessor.py):
 * out[:, j] = transform_type(in[:, src_col]; p0..p3 [, quantiles q_off..q_off+q_cnt)).
 *   PROBABILITY: p0=1e-5 p1=1-1e-5 (as f32)     CONTINUOUS: p0=mean p1=stddev
 *   BOXCOX: p0=mean p1=stddev p2=shift p3=lambda ENUM: p0=possible value of this column
 *   QUANTILE: p0=len(quantiles)-1 p1=max p2=min, q_* = padded boundaries
 *   CONTINUOUS_ACTION: p0=min_serving p1=scaling_factor p2=min_training p3=-1+EPS */
typedef struct rb200_feature_col {
  int32_t src_col;
  int32_t type;
  float p0, p1, p2, p3;
  int32_t q_off, q_cnt;
} rb200_feature_col_t;

const char* rb200_last_error(void);
int rb200_version(void);
/* sizeof() of an ABI struct by name ("rb200_adam_args_t", ...), -1 if unknown: lets a binding
 * verify its mirror of the struct against the library it loaded */
int64_t rb200_abi_sizeof(const char* type_name);
/* number of SMs / max opt-in smem of the current device (host query helpers) */
int rb200_device_info(int* sm_count, int* max_smem_optin);

/* P1: Preprocessor.forward(input, input_presence_byte) -- reagent/preprocessing/
 * preprocessor.py:115-170.  `cols` / `quantiles` are device arrays; presence may be NULL
 * (all present), uint8/bool [rows,f_in] or float [rows,f_in]. */
int rb200_preprocess(const float* input, const void* presence, int32_t presence_is_float,
                     int64_t rows, int32_t f_in, int32_t f_out, const rb200_feature_col_t* cols,
                     const float* quantiles, float* out, void* stream);

/* Fused whole-MLP forward out = net(cat(in0, in1)) over row tiles; in1 may be NULL.
 * Replaces FullyConnectedNetwork.forward (reagent/models/fully_connected_network.py:157-163)
 * and FullyConnectedCritic.forward's cat (reagent/models/critic.py:76-92).  When
 * save_hidden != NULL the hidden layer outputs go to save_hidden->hidden[l] (training). */
int rb200_mlp_forward(const rb200_mlp_t* net, const float* in0, int32_t d0, const float* in1,
                      int32_t d1, int32_t batch, float* out, const rb200_net_ws_t* save_hidden,
                      void* stream);

/* Tiled forward of the max-Q target of ParametricDQNTrainer (reagent/training/
 * parametric_dqn_trainer.py:101-110, FeatureData.get_tiled_batch): for each of the
 * batch * num_tiled rows r, out_n[r] = net_n(cat(state[r / num_tiled], actions[r])).
 * state [batch, state_dim]; actions [batch * num_tiled, action_dim]; out0 / out1
 * [batch * num_tiled, dims[L]].  net1 (with out1) is optional and must have net0's dims and
 * activations; both networks run over one input tile built in shared memory, so the tiled
 * input is never written to HBM.  Every output is bit-equal to rb200_mlp_forward on the
 * materialised cat(state.repeat_interleave(num_tiled), actions).  RB200_E_INVALID on null
 * pointers, differing descriptors, widths that do not sum to dims[0] or batch * num_tiled
 * past int32; RB200_E_SMEM where rb200_mlp_forward's tile would not fit. */
int rb200_mlp_forward_tiled(const rb200_mlp_t* net0, const rb200_mlp_t* net1,
                            const float* state, int32_t state_dim, const float* actions,
                            int32_t action_dim, int32_t batch, int32_t num_tiled, float* out0,
                            float* out1, void* stream);

/* ------------------------------------------------------------------------- */
/* Dueling head folded into a Linear (rb200_dueling.cu).  Replaces the head arithmetic of     */
/* DuelingQNetwork._get_values (reagent/models/dueling_q_network.py:92-103), with atoms:       */
/*   q[a,n] = value[n] + advantage[a,n] - mean_{a',n'}(advantage)     (num_atoms = 1: DQN)     */
/* `fold` builds the equivalent last layer W_q [A*N, 2H] / b_q [A*N] (row a*N+n) from the true  */
/* parameters (advantage head W_adv [A*N,H], b_adv [A*N]; value head w_val [N,H], b_val [N]) so */
/* that every MLP kernel of this library runs a dueling network as a plain MLP; `unfold` maps   */
/* the gradient of that layer back onto the true parameters in each of `splits` gradient slabs  */
/* (offsets in floats from the slab start) and zeroes the folded layer's gradient.  `scratch`:  */
/* rb200_dueling_scratch_floats(H, splits) floats of device memory.                             */
/* ------------------------------------------------------------------------- */
int64_t rb200_dueling_scratch_floats(int32_t head_hidden, int32_t splits);
int rb200_dueling_fold(const float* W_adv, const float* b_adv, const float* w_val,
                       const float* b_val, int32_t num_actions, int32_t num_atoms,
                       int32_t head_hidden, float* W_q, float* b_q, float* scratch, void* stream);
int rb200_dueling_unfold(float* grad, int64_t slab_stride, int32_t splits, int32_t num_actions,
                         int32_t num_atoms, int32_t head_hidden, int64_t off_W_q, int64_t off_b_q,
                         int64_t off_W_adv, int64_t off_b_adv, int64_t off_w_val,
                         int64_t off_b_val, float* scratch, void* stream);

/* ------------------------------------------------------------------------- */
/* K2 (+K2'): fused DQN TD-target / loss / backward over row tiles.            */
/* Replaces DQNTrainer.compute_td_loss + get_max_q_values_with_target +        */
/* boost_rewards + compute_discount_tensor (reagent/training/dqn_trainer.py:   */
/* 157-239, dqn_trainer_base.py:33-77,216-241) and, with do_backward, autograd's*/
/* backward through q_network down to every layer's pre-activation gradient.    */
/* ------------------------------------------------------------------------- */
typedef struct rb200_dqn_args {
  int32_t batch;                 /* B */
  const float* state;            /* [B,S] */
  const float* next_state;       /* [B,S] */
  const float* action;           /* [B,A] float weights (one-hot in practice) */
  const float* next_action;      /* [B,A] (SARSA only, may be NULL)          */
  const float* reward;           /* [B]   */
  const float* not_terminal;     /* [B]   */
  const float* possible_next_actions_mask; /* [B,A] or NULL (= ones)          */
  const float* discount_src;     /* [B] time_diff or step (POW mode) or NULL  */
  const float* reward_boost;     /* [A] or NULL                                */
  float gamma;
  int32_t discount_mode;         /* RB200_DISCOUNT_*  */
  int32_t double_q;              /* dqn_trainer_base.py:64-75 */
  int32_t maxq;                  /* 0 = SARSA (mask := next_action)           */
  int32_t loss_kind;             /* RB200_LOSS_*      */
  int32_t do_backward;           /* 0: forward/loss only (validation_step)    */
  /* outputs */
  float* all_action_scores;      /* [B,A] q_network(state) (detached) or NULL */
  float* td_target;              /* [B] or NULL                                */
  float* q_selected;             /* [B] or NULL                                */
  int32_t* next_action_idx;      /* [B] argmax index or NULL                   */
  float* loss_partials;          /* [>= ceil(B/16)]                */
  float* loss;                   /* [1] mean loss (written by the last tile)   */
  uint32_t* tile_counter;        /* [1] zero-initialised scratch, self-resetting */
  const float* sample_weight;    /* [B] or NULL: loss = mean(w * loss_row), dZ row scaled by w */
} rb200_dqn_args_t;

int rb200_num_row_tiles(int batch, int max_dim_in, int max_dim_hidden);
int rb200_dqn_td_step(const rb200_mlp_t* q_net, const rb200_mlp_t* q_target,
                      const rb200_dqn_args_t* args, const rb200_net_ws_t* ws, void* stream);

/* The same step on the Hopper tensor cores (warpgroup MMAs, wgmma kind tf32 with 3xTF32 error
 * compensation, accumulators in registers, weights streamed by bulk async copies):
 * rb200_dqn_tc.cu.  Same arguments, semantics and reference lines as rb200_dqn_td_step plus a
 * caller-owned scratch buffer for the packed hi/lo weight images (re-packed on every call,
 * because the weights change on every update).
 *   rb200_dqn_tc_workspace_bytes: bytes the scratch buffer needs for this network, or 0 when
 *       the shapes do not fit the tensor-core path (then use rb200_dqn_td_step).
 *   rb200_dqn_tc_pack: (re)build the hi/lo weight images from the current parameters.  It only
 *       depends on the parameters, so a caller may run it on a side stream as soon as the
 *       previous optimizer step is done (e.g. concurrently with replay sampling) and pass
 *       weights_packed = 1; with weights_packed = 0 the step packs first, on `stream`.
 *       The images depend on (double_q, do_backward) only through which ones are built.
 *   pack_ws: device buffer, 128-byte aligned, zero-initialised ONCE by the caller. */
int64_t rb200_dqn_tc_workspace_bytes(const rb200_mlp_t* q_net, int32_t double_q,
                                     int32_t do_backward);
int rb200_dqn_tc_pack(const rb200_mlp_t* q_net, const rb200_mlp_t* q_target, int32_t double_q,
                      int32_t do_backward, void* pack_ws, int64_t pack_ws_bytes, void* stream);
int rb200_dqn_td_step_tc(const rb200_mlp_t* q_net, const rb200_mlp_t* q_target,
                         const rb200_dqn_args_t* args, const rb200_net_ws_t* ws, void* pack_ws,
                         int64_t pack_ws_bytes, int32_t weights_packed, void* stream);

/* ------------------------------------------------------------------------- */
/* Batch-constrained Q-learning filter (rb200_bcq.cu).  Replaces                 */
/* get_valid_actions_from_imitator (reagent/training/imitator_training.py:12-25) */
/* as used by DQNTrainer (dqn_trainer.py:206-220, 282-297) and the penalty of    */
/* BatchConstrainedDQN.forward (reagent/models/bcq.py:26-35):                    */
/*   r = softmax(logits) / max(softmax(logits)),  keep = r >= drop_threshold     */
/* per row of imitator_logits [batch, num_actions], 1 <= num_actions <= 1024.    */
/* Exactly one output mode:                                                       */
/*   trainer: mask_out [B,A] = mask_in * keep   (mask_in [B,A] or NULL = ones;    */
/*            q_in must be NULL)                                                  */
/*   model:   q_out [B,A] = q_in + (-1e10) * (1 - keep)  (mask_in must be NULL;   */
/*            q_out may equal q_in)                                               */
/* Row-local, deterministic, no atomics, no allocation (graph-capturable).        */
/* ------------------------------------------------------------------------- */
int rb200_bcq_filter(const float* imitator_logits, int32_t batch, int32_t num_actions,
                     float drop_threshold, const float* mask_in, float* mask_out,
                     const float* q_in, float* q_out, void* stream);

/* ------------------------------------------------------------------------- */
/* CPE heads of the DQN step: DQNTrainerBaseLightning._calculate_cpes           */
/* (reagent/training/dqn_trainer_base.py:332-452), masked_softmax                 */
/* (reagent/core/torch_utils.py:62-73).  The reward network and the CPE q-network  */
/* are plain MLPs (rb200_mlp_forward / rb200_mlp_backward / rb200_mlp_wgrad); this  */
/* entry computes both losses and d loss / d output of both networks.              */
/* loss[0] = reward loss, loss[1] = CPE q-value loss.                               */
/* ------------------------------------------------------------------------- */
typedef struct rb200_cpe_args {
  int32_t batch, num_actions, num_metrics;   /* B, A, M = len(metrics_to_score) */
  const float* next_scores;        /* [B,A] q_network(next_state) (detached) */
  const float* mask;               /* [B,A] possible_next_actions_mask (maxq) | next_action, or NULL */
  float temperature;               /* rl.temperature */
  const float* action;             /* [B,A] logged action (argmax = index) */
  const float* metrics_reward;     /* [B,M] cat(reward, extras.metrics) */
  const float* discount_src;       /* [B] or NULL */
  float gamma;
  int32_t discount_mode;           /* RB200_DISCOUNT_* */
  const float* not_terminal;       /* [B] */
  const float* reward_est;         /* [B, M*A] reward_network(state) */
  const float* qcpe;               /* [B, M*A] q_network_cpe(state) */
  const float* qcpe_target_next;   /* [B, M*A] q_network_cpe_target(next_state) */
  int32_t loss_kind;               /* RB200_LOSS_* (rl.q_network_loss) for the CPE q-network */
  float* dz_reward;                /* [B, M*A] */
  float* dz_qcpe;                  /* [B, M*A] */
  float* propensities_next;        /* [B,A] or NULL */
  float* loss_partials;            /* [2 * ceil(B/256)] */
  float* loss;                     /* [2] */
  uint32_t* tile_counter;          /* [1] zero-initialised, self-resetting */
} rb200_cpe_args_t;
int rb200_cpe_heads(const rb200_cpe_args_t* args, void* stream);

/* ------------------------------------------------------------------------- */
/* Loss heads of ParametricDQNTrainer and C51Trainer (rb200_heads.cu); the networks */
/* around them run on rb200_mlp_forward / rb200_linear_forward / *_backward / wgrad. */
/*   rb200_pdqn_head: reagent/training/parametric_dqn_trainer.py:109-173 (TD target    */
/*     from the tiled possible next actions or the SARSA value, mse | huber, dL/dq)     */
/*   rb200_c51_head:  reagent/training/c51_trainer.py:98-173 (log-softmax over atoms,  */
/*     masked arg max of expected values, categorical projection, cross entropy,       */
/*     dL/dlogits); reagent/models/categorical_dqn.py:28-35                             */
/* ------------------------------------------------------------------------- */
typedef struct rb200_pdqn_args {
  int32_t batch, max_num_action;   /* M tiled next actions per row; 0 = SARSA */
  const float* next_q;             /* [B*M] q_network(tiled s', a') (double-Q) or NULL */
  const float* next_q_target;      /* [B*M] (maxq) or [B] (SARSA: q_target(s', next_action)) */
  const float* mask;               /* [B,M] possible_next_actions_mask or NULL */
  const float* reward;             /* [B] */
  const float* not_terminal;       /* [B] */
  const float* discount_src;       /* [B] or NULL */
  float gamma;
  int32_t discount_mode, double_q, loss_kind;
  const float* q_values;           /* [B] q_network(state, action) */
  float* dz;                       /* [B] d loss / d q */
  float* td_target;                /* [B] or NULL */
  float* loss_partials;            /* [ceil(B/256)] */
  float* loss;                     /* [1] */
  uint32_t* tile_counter;
} rb200_pdqn_args_t;
int rb200_pdqn_head(const rb200_pdqn_args_t* args, void* stream);

typedef struct rb200_c51_args {
  int32_t batch, num_actions, num_atoms;
  const float* logits_next_online; /* [B, A*N] distributional_network(next_state), online (double-Q) or NULL */
  const float* logits_next_target; /* [B, A*N] target network */
  const float* logits_cur;         /* [B, A*N] online network on state */
  const float* action;             /* [B,A] */
  const float* next_action;        /* [B,A] (SARSA) or NULL */
  const float* possible_next_actions_mask; /* [B,A] or NULL */
  const float* reward;             /* [B] */
  const float* not_terminal;       /* [B] */
  const float* discount_src;       /* [B] or NULL: gamma ** discount_src */
  const float* reward_boost;       /* [A] or NULL */
  const float* support;            /* [N] torch.linspace(qmin, qmax, N) */
  float gamma, qmin, qmax, scale_support;
  int32_t double_q, maxq;
  float* dz_logits;                /* [B, A*N] */
  float* all_q_values;             /* [B,A] or NULL */
  int32_t* next_action_idx;        /* [B] or NULL */
  float* loss_partials;            /* [B] per-row cross entropy, unweighted */
  float* loss;                     /* [1] */
  uint32_t* tile_counter;
  const float* sample_weight;      /* [B] or NULL: loss = mean(w * loss_row), dz_logits row scaled by w */
} rb200_c51_args_t;
int rb200_c51_head(const rb200_c51_args_t* args, void* stream);

/* Loss head of BehavioralCloningTrainer (rb200_heads.cu),                          */
/* reagent/training/behavioral_cloning_trainer.py:38-66, one warp per row:           */
/*   z = logits + (-1e10) * (1 - mask)   (FullyConnectedDQN.forward, models/dqn.py)  */
/*   y = first arg max of the label row  (each row's own logged action)              */
/*   loss = mean_b -log_softmax(z)[y],   dz = (softmax(z) - onehot(y)) / B            */
/* 1 <= num_actions <= 1024.  dz NULL: loss only.  Deterministic (fixed-order mean),  */
/* no allocation (graph-capturable); loss_partials holds                              */
/* ceil(B / RB200_BC_ROWS_PER_BLOCK) floats.                                          */
#define RB200_BC_ROWS_PER_BLOCK 8
typedef struct rb200_bc_xent_args {
  int32_t batch, num_actions;
  const float* logits;             /* [B,A] bc_net scores, unmasked */
  const float* labels;             /* [B,A] one-hot logged action */
  const float* mask;               /* [B,A] possible_actions_mask (1 = possible) */
  float* dz;                       /* [B,A] d loss / d logits, or NULL */
  float* loss_partials;
  float* loss;                     /* [1] */
  uint32_t* tile_counter;          /* [1] zero-initialised, self-resetting */
} rb200_bc_xent_args_t;
int rb200_bc_xent_head(const rb200_bc_xent_args_t* args, void* stream);

/* Loss head of SlateQTrainer (rb200_slateq.cu), reagent/training/slate_q_trainer.py:       */
/* 199-276, one warp per row.  Per row b it forms the next slate (next_action[b], or with  */
/* maxq the first slate_size candidates of q_next * docs_value in (score desc, index asc)  */
/* order), weights the target network's values of that slate by the docs value            */
/* (softmax(value * mask) over the slate with single_selection, value * mask without),     */
/* divides by min(sum(mask), slate_size) of the current or next candidate mask without     */
/* single_selection, and writes target = reward + discount * (next_q * not_terminal) with  */
/* discount = gamma ** (time_diff / time_scale) when time_diff is given, else gamma.  The  */
/* loss is mse(q_cur, target) over the reward_mask entries (single_selection) or all B*K   */
/* entries; dz = d loss / d q_cur.  A terminal row's next slate is candidate 0 everywhere, */
/* and in SARSA those rows of next_action are zeroed in place, as the reference does.     */
/* With single_selection a one-CTA pass first counts the reward_mask entries (an integer, */
/* so the count and the gradient scale 1 / count do not depend on the order); an empty    */
/* mask gives a NaN loss and dz = 0.  Indices follow torch's indexing: one in [-C, 0)     */
/* means C + index; one outside [-C, C) (the reference's IndexError) is never read: the   */
/* row uses candidate 0 instead and status[0] is set to 1 (sticky).                       */
/* Limits: 1 <= C <= RB200_SLATEQ_MAX_CANDIDATES, 1 <= K, K_next <= RB200_SLATEQ_MAX_SLATE, */
/* 1 <= slate_size <= min(C, RB200_SLATEQ_MAX_SLATE) (one slate entry per lane); beyond   */
/* them RB200_E_INVALID.                                                                   */
#define RB200_SLATEQ_MAX_CANDIDATES 1024
#define RB200_SLATEQ_MAX_SLATE 32
#define RB200_SLATEQ_ROWS_PER_BLOCK 8
#define RB200_SLATEQ_NORM_CURRENT 0 /* NORM_BY_CURRENT_SLATE_SIZE */
#define RB200_SLATEQ_NORM_NEXT 1    /* NORM_BY_NEXT_SLATE_SIZE */
typedef struct rb200_slateq_args {
  int32_t batch, num_candidates;   /* B, C */
  int32_t slate_width;             /* K = action.shape[1] */
  int32_t next_width;              /* K_next = next_action.shape[1] (SARSA); ignored with maxq */
  int32_t slate_size, maxq, single_selection, norm_method;
  const float* q_cur;              /* [B*K] q_network(state, docs[b, action]) */
  const float* q_next;             /* [B*C] q_network_target(next_state, every next candidate) */
  const float* next_value;         /* [B*C] next candidate_docs.value */
  const float* next_mask;          /* [B*C] next candidate_docs.mask */
  const float* cur_mask;           /* [B*C] current candidate_docs.mask (NORM_CURRENT) */
  int64_t* next_action;            /* [B*K_next] (SARSA, terminal rows zeroed) or NULL (maxq) */
  const int64_t* action;           /* [B*K] current slate, range-checked only; or NULL */
  const float* reward;             /* [B*K] */
  const float* reward_mask;        /* [B*K] (single_selection) */
  const float* not_terminal;       /* [B] */
  const float* time_diff;          /* [B] or NULL */
  float gamma, time_scale;
  float* dz;                       /* [B*K] d loss / d q_cur */
  float* target;                   /* [B*K] or NULL */
  int32_t* mask_count;             /* [1] scratch (single_selection) */
  int32_t* status;                 /* [1] sticky: 1 = an index outside [0, C) */
  float* loss_partials;            /* [ceil(B / RB200_SLATEQ_ROWS_PER_BLOCK)] */
  float* loss;                     /* [1] */
  uint32_t* tile_counter;          /* [1] zero-initialised, self-resetting */
} rb200_slateq_args_t;
int rb200_slateq_head(const rb200_slateq_args_t* args, void* stream);

/* Loss heads of DiscreteCRRTrainer (rb200_crr.cu), reagent/training/                 */
/* discrete_crr_trainer.py, one warp per row, 1 <= num_actions <= 1024.  The actor's    */
/* logits are FullyConnectedActor.forward's output (reagent/models/actor.py:90-110):    */
/*   l = actor_out                            without exploration noise (noise NULL)    */
/*   l = clamp(actor_out + noise, -1, 1)      with it; `noise` is the draw, scaled      */
/* Both heads are deterministic (fixed-order means) and allocate nothing                */
/* (graph-capturable); loss_partials holds 2 * ceil(B / RB200_CRR_ROWS_PER_BLOCK)       */
/* floats.                                                                              */
/* critic head: compute_target_q_values + compute_td_loss (:198-218, :304-326)          */
/*   r  = reward + sum_a action * reward_boost              (boost_rewards)             */
/*   V' = sum_a softmax(l')_a * q1_target(s')_a, min with q2's when q2 is given         */
/*   y  = r + gamma * V' * not_terminal                                                 */
/*   loss[c] = mean_b (q_c(s, a) - y)^2,  q_c(s, a) = sum_a q_c * action                */
/*   dz_qc = 2 * (q_c(s, a) - y) / B * action               (d loss[c] / d q_c)         */
#define RB200_CRR_ROWS_PER_BLOCK 16
typedef struct rb200_crr_critic_args {
  int32_t batch, num_actions;
  const float* actor_next;         /* [B,A] actor (or target actor) output on next_state, before noise */
  const float* noise_next;         /* [B,A] or NULL */
  const float* q1_target_next;     /* [B,A] q1_network_target(next_state) */
  const float* q2_target_next;     /* [B,A], with q2 only */
  const float* q1;                 /* [B,A] q1_network(state) */
  const float* q2;                 /* [B,A] q2_network(state) or NULL: single critic */
  const float* action;             /* [B,A] one-hot logged action */
  const float* reward;             /* [B] */
  const float* reward_boost;       /* [A] or NULL */
  const float* not_terminal;       /* [B] */
  float gamma;
  float* td_target;                /* [B] y */
  float* q1_selected;              /* [B] q1(s, a) */
  float* q2_selected;              /* [B], with q2 only */
  float* dz_q1;                    /* [B,A] */
  float* dz_q2;                    /* [B,A], with q2 only */
  float* loss_partials;
  float* loss;                     /* [2]: q1 loss, q2 loss (0 without q2) */
  uint32_t* tile_counter;          /* [1] zero-initialised, self-resetting */
} rb200_crr_critic_args_t;
int rb200_crr_critic_head(const rb200_crr_critic_args_t* args, void* stream);

/* actor head: compute_actor_loss (:220-288), a = first arg max of the action row       */
/*   pi = softmax(l),  V = sum_a pi_a * q1_a,  weight = clamp(exp((q1[a] - V) * inv_beta), */
/*   0, max_weight)  (a constant of the gradient),  log_pi = log_softmax(l)[a]          */
/*   loss[0] = mean_b(-log_pi * weight)                      actor_loss_without_reg     */
/*   loss[1] = loss[0] + entropy_coeff * mean_b(ratio * log_pi) when entropy_coeff > 0,  */
/*             ratio = clip(pi[a] / action_probability, 1e-4, clip_limit)               */
/*   dz = d loss[1] / d z for the PRE-activation z of the actor's last layer            */
/*        (actor_out = act(z)), which is what rb200_mlp_backward / rb200_mlp_wgrad take: */
/*        the gradient flows through log_pi and through the ratio where it is not        */
/*        clipped, is zero where actor_out + noise lies outside [-1, 1] (noise given),   */
/*        and is multiplied by act'(z) computed from actor_out.                          */
typedef struct rb200_crr_actor_args {
  int32_t batch, num_actions;
  const float* actor_out;          /* [B,A] actor output on state, before noise */
  const float* noise;              /* [B,A] or NULL */
  const float* q1;                 /* [B,A] q1_network(state), after q1's update */
  const float* action;             /* [B,A] one-hot logged action */
  const float* action_probability; /* [B] logged propensities; required iff entropy_coeff > 0 */
  float inv_beta, max_weight, entropy_coeff, clip_limit;
  int32_t action_activation;       /* RB200_ACT_* of the actor's last layer */
  float* weight;                   /* [B] or NULL */
  float* dz;                       /* [B,A], or NULL: losses only */
  float* loss_partials;
  float* loss;                     /* [2] */
  uint32_t* tile_counter;          /* [1] zero-initialised, self-resetting */
} rb200_crr_actor_args_t;
int rb200_crr_actor_head(const rb200_crr_actor_args_t* args, void* stream);

/* Policy gradient (rb200_pg.cu): ReinforceTrainer and PPOTrainer,                     */
/* reagent/training/reinforce_trainer.py and ppo_trainer.py.  A batch is packed: the    */
/* rows of n_traj trajectories one after another, trajectory t at rows                  */
/* [offsets[t], offsets[t + 1]).                                                        */
/* rb200_pg_returns, per trajectory (utils.py discounted_returns and whiten):           */
/*   r = min(reward, reward_clip)    (upper bound only)                                 */
/*   gamma != 0: running = r_t + gamma * running from the last row back, each op        */
/*               rounded to fp32 in the reference's order (bit-identical returns)       */
/*   norm: WHITEN (x - mean) / (std + EPS), WHITEN_NO_MEAN x / (std + EPS),              */
/*         SUBTRACT_MEAN x - mean; std is the population std, mean/var in double        */
/*   offset_clamp_min: max(x, 0)                                                        */
/* One warp per trajectory, any length.  Allocates nothing (graph-capturable).          */
#define RB200_PG_NORM_NONE 0
#define RB200_PG_NORM_WHITEN 1
#define RB200_PG_NORM_WHITEN_NO_MEAN 2
#define RB200_PG_NORM_SUBTRACT_MEAN 3
#define RB200_PG_WHITEN_EPS 2.220446049250313e-16 /* np.finfo(float).eps */
typedef struct rb200_pg_returns_args {
  int32_t n_traj;
  const int32_t* offsets;          /* [n_traj + 1] */
  const float* reward;             /* [R] */
  float reward_clip, gamma;
  int32_t norm;                    /* RB200_PG_NORM_* */
  int32_t offset_clamp_min;
  float* returns;                  /* [R] */
} rb200_pg_returns_args_t;
int rb200_pg_returns(const rb200_pg_returns_args_t* args, void* stream);

/* rb200_pg_head, one warp per row, 1 <= num_actions <= 1024:                           */
/*   x = (scores + (-1e10) * (1 - mask)) / temperature,  a = first arg max of action     */
/*   log_pi = log_softmax(x)[a]                                                          */
/*   advantage: RETURNS   adv = returns                                                  */
/*              BASELINE  adv = returns - value,              value target y = returns    */
/*              TD        y = min(reward, reward_clip) + gamma * nt * V',  adv = y - value, */
/*                        then max(adv, 0) with offset_clamp_min.  V' = next_value, or    */
/*                        without it the next row's value (0 after a trajectory's last    */
/*                        row); nt = not_terminal, or without it 0 on a last row, else 1  */
/*   REINFORCE: loss[0] = -sum adv * elig, elig = log_pi, or with logged_log_prob         */
/*              exp(min(log_pi - logged, log_clip_param)) (gradient 0 where it clamps)    */
/*   PPO:       loss[0] = -sum min(adv * rho, adv * clamp(rho, ppo_clip_lo, ppo_clip_hi)) */
/*              - entropy_weight * sum_rows H(softmax(x)),  rho = exp(log_pi - logged)    */
/*   loss[1] = value_scale * sum (value - y)^2,  dz_value = 2 * value_scale * (value - y) */
/*   dz = d loss[0] / d scores (the 1/temperature included; the mask adds nothing)       */
/* Sums in a fixed order (deterministic); allocates nothing.                             */
#define RB200_PG_ROWS_PER_BLOCK 8
#define RB200_PG_LOSS_REINFORCE 0
#define RB200_PG_LOSS_PPO 1
#define RB200_PG_ADV_RETURNS 0
#define RB200_PG_ADV_BASELINE 1
#define RB200_PG_ADV_TD 2
typedef struct rb200_pg_head_args {
  int32_t rows, num_actions, n_traj;
  const int32_t* offsets;          /* [n_traj + 1] */
  const float* scores;             /* [R,A] policy net output, before the mask */
  const float* mask;               /* [R,A] possible_actions_mask or NULL */
  const float* action;             /* [R,A] one-hot logged action */
  const float* logged_log_prob;    /* [R]: PPO; off-policy REINFORCE; else NULL */
  const float* returns;            /* [R] rb200_pg_returns output (RETURNS, BASELINE) */
  const float* value;              /* [R] V(state) (BASELINE, TD) or NULL */
  const float* next_value;         /* [R] V(next_state) or NULL (TD) */
  const float* reward;             /* [R] (TD) */
  const float* not_terminal;       /* [R] or NULL (TD) */
  float temperature, gamma, reward_clip, log_clip_param, entropy_weight;
  float ppo_clip_lo, ppo_clip_hi;  /* float(1 - eps), float(1 + eps), rounded from double */
  float value_scale;               /* 1/T: MSELoss(mean) of one trajectory; 1: MSELoss(sum) */
  int32_t loss_kind;               /* RB200_PG_LOSS_* */
  int32_t advantage_kind;          /* RB200_PG_ADV_* */
  int32_t offset_clamp_min;        /* TD advantage only */
  float* advantage_out;            /* [R] or NULL */
  float* dz;                       /* [R,A] or NULL */
  float* dz_value;                 /* [R] or NULL */
  float* loss_partials;            /* 2 * ceil(R / RB200_PG_ROWS_PER_BLOCK) */
  float* loss;                     /* [2]: policy loss, value loss */
  uint32_t* tile_counter;          /* [1] zero-initialised, self-resetting */
} rb200_pg_head_args_t;
int rb200_pg_head(const rb200_pg_head_args_t* args, void* stream);

/* ------------------------------------------------------------------------- */
/* QR-DQN (reagent/training/qrdqn_trainer.py:108-194).  The [hidden -> A*N] head  */
/* is too wide for a row tile, so it runs as 2-D tiled launches:                   */
/*   rb200_linear_forward      out = act(in . W^T + b), any N     (nn.Linear fwd) */
/*   rb200_linear_backward_dx  dz_prev = (dz . W) * act'(h_prev)  (autograd)      */
/*   rb200_mlp_backward        dZ chain of the layers below a given last-layer dz */
/*   rb200_qrdqn_head          mean over atoms, masked argmax, target             */
/*       distribution, pairwise quantile-Huber loss (:152-155, :217-218) and      */
/*       d loss / d head output, one CTA per row, nothing (N,B,N)-sized in HBM.   */
/* ------------------------------------------------------------------------- */
typedef struct rb200_qrdqn_args {
  int32_t batch, num_actions, num_atoms;
  const float* q_next_online;  /* [B, A*N] q_network(next_state)  (double-Q) or NULL */
  const float* q_next_target;  /* [B, A*N] q_network_target(next_state) */
  const float* q_cur;          /* [B, A*N] q_network(state) */
  const float* action;         /* [B, A] */
  const float* next_action;    /* [B, A] (SARSA) or NULL */
  const float* possible_next_actions_mask; /* [B, A] or NULL */
  const float* reward;         /* [B] */
  const float* not_terminal;   /* [B] */
  const float* discount_src;   /* [B] or NULL: gamma ** discount_src */
  const float* reward_boost;   /* [A] or NULL */
  float gamma;
  int32_t double_q, maxq;
  float* dz_head;              /* [B, A*N] d loss / d head output */
  float* all_q_values;         /* [B, A] mean over atoms of q(s), or NULL */
  int32_t* next_action_idx;    /* [B] or NULL */
  float* loss_partials;        /* [B] per-row quantile-Huber sum over the N*N pairs, unweighted */
  float* loss;                 /* [1] */
  uint32_t* tile_counter;      /* [1] zero-initialised, self-resetting */
  const float* sample_weight;  /* [B] or NULL: loss = mean(w * loss_row), dz_head row scaled by w */
} rb200_qrdqn_args_t;

int rb200_linear_forward(const float* W, const float* b, int32_t act, int32_t K, int32_t N,
                         const float* in, int32_t batch, float* out, void* stream);
/* wgmma (kind tf32, 3xTF32) implementation of rb200_linear_forward, taken
 * automatically for batch >= 128 and N >= 128 */
int rb200_linear_forward_tc(const float* W, const float* b, int32_t act, int32_t K, int32_t N,
                            const float* in, int32_t batch, float* out, void* stream);
int rb200_linear_backward_dx(const float* W, int32_t K, int32_t N, const float* dz,
                             const float* h_prev, int32_t act_prev, int32_t batch, float* out,
                             void* stream);
/* wgmma implementation of rb200_linear_backward_dx for a wide layer (the contraction runs
 * over the N out-features: split-K slices of the tensor-core GEMM, added in a fixed order).
 * _scratch_bytes returns 0 when the shape is not taken by this path (N < 1024, batch < 256 or
 * K / N not multiples of 4): call rb200_linear_backward_dx then.  Replaces the same autograd
 * step (torch.nn.functional.linear backward w.r.t. input, reagent/training/qrdqn_trainer.py:
 * 108-194 via reagent_lightning_module.py:108-133). */
int64_t rb200_linear_backward_dx_tc_scratch_bytes(int32_t K, int32_t N, int32_t batch);
int rb200_linear_backward_dx_tc(const float* W, int32_t K, int32_t N, const float* dz,
                                const float* h_prev, int32_t act_prev, int32_t batch, float* out,
                                void* scratch, int64_t scratch_bytes, void* stream);
int rb200_mlp_backward(const rb200_mlp_t* net, const float* dz_last, int32_t batch,
                       const rb200_net_ws_t* ws, void* stream);
int rb200_qrdqn_head(const rb200_qrdqn_args_t* args, void* stream);

/* ------------------------------------------------------------------------- */
/* Fused SAC / TD3 updates over row tiles.                                      */
/* critic step: replaces SACTrainer.train_step_gen's first section              */
/*   (reagent/training/sac_trainer.py:214-248: actor(s') + get_log_prob, target */
/*   critics, min, entropy term, target, q1/q2 MSE) or TD3Trainer's             */
/*   (reagent/training/td3_trainer.py:138-178), plus autograd's backward through*/
/*   q1 / q2.  loss[0] = q1 loss, loss[1] = q2 loss.                            */
/* actor step: replaces sac_trainer.py:254-322 (actor loss, alpha loss) or      */
/*   td3_trainer.py:181-187, plus the backward through the frozen critics into  */
/*   the actor (reagent/models/actor.py:169-261 for the Gaussian head).         */
/*   loss[0] = actor loss, loss[1] = alpha loss; alpha_grad[0] = d/d log_alpha. */
/* `noise_*` are the N(0,1) draws of torch.randn_like in the reference          */
/* (actor.py:217, td3_trainer.py:141), supplied by the caller.                  */
/* ------------------------------------------------------------------------- */
#define RB200_ALGO_SAC 0
#define RB200_ALGO_TD3 1
typedef struct rb200_ac_args {
  int32_t batch;
  int32_t algo;
  const float* state;        /* [B,S] */
  const float* action;       /* [B,A] (critic step) */
  const float* next_state;   /* [B,S] (critic step) */
  const float* reward;       /* [B] */
  const float* not_terminal; /* [B] */
  const float* noise_next;   /* [B,A] critic step */
  const float* noise_cur;    /* [B,A] SAC actor step */
  float gamma;
  const float* alpha;        /* [1] SAC entropy temperature (device) */
  const float* log_alpha;    /* [1] SAC (actor step: alpha loss value) or NULL */
  float target_entropy;
  int32_t backprop_through_log_prob;
  float noise_variance, noise_clip; /* TD3 */
  /* outputs */
  float* loss_partials;      /* [2 * num tiles] */
  float* loss;               /* [2] */
  uint32_t* tile_counter;    /* [1] zero-initialised, self-resetting */
  float* alpha_grad;         /* [1] or NULL */
  float* td_target;          /* [B] or NULL */
  float* next_action_out;    /* [B,A] or NULL: a' (critic step) / pi(s) (actor step) */
  float* log_prob_out;       /* [B] or NULL (unclamped sum of log-probs) */
  float* q1_value;           /* [B] or NULL */
  float* q2_value;           /* [B] or NULL */
  /* SAC state-value network V(s) (sac_trainer.py:109-113, :214-217, :254-283, :329-343);
     ahead of the prioritized-replay pair, which stays last */
  const rb200_mlp_t* value_target; /* critic step: non-NULL -> target r + gamma*V'(s')*not_terminal,
                                      no actor forward on s', no noise_next, no q targets */
  const rb200_mlp_t* value_net;    /* actor step with CRR: the current V [S -> 1] */
  float* min_q_out;          /* [B] or NULL: actor step writes min_c q_c(s, pi(s)); the value
                                step reads it (and log_prob_out) for its target */
  int32_t crr_mode;          /* RB200_CRR_*: actor loss mean(-clamp(log_prob) * w(advantage)) */
  float crr_threshold;       /* RB200_CRR_INDICATOR: w = (advantage >= threshold) */
  float crr_beta;            /* RB200_CRR_EXPONENT: w = exp(advantage / beta) ... */
  float crr_clamp;           /* ... clamped to [0, crr_clamp] when crr_clamp > 0 */
  int32_t logged_action_uniform_prior; /* value step: target min_q (1) or
                                          min_q - alpha * clamp(log_prob) (0) */
  /* prioritized replay (critic step only; the actor step ignores both) */
  const float* sample_weight; /* [B] or NULL: critic losses mean(w * d^2), dz row scaled by w */
  float* td_error_out;       /* [B] or NULL: max over critics of |q_c - td_target| */
} rb200_ac_args_t;
#define RB200_CRR_NONE 0
#define RB200_CRR_INDICATOR 1
#define RB200_CRR_EXPONENT 2

int rb200_ac_critic_step(const rb200_mlp_t* actor, const rb200_mlp_t* q1, const rb200_mlp_t* q2,
                         const rb200_mlp_t* q1_target, const rb200_mlp_t* q2_target,
                         const rb200_ac_args_t* args, const rb200_net_ws_t* ws_q1,
                         const rb200_net_ws_t* ws_q2, void* stream);
int rb200_ac_actor_step(const rb200_mlp_t* actor, const rb200_mlp_t* q1, const rb200_mlp_t* q2,
                        const rb200_ac_args_t* args, const rb200_net_ws_t* ws_actor,
                        const rb200_net_ws_t* ws_q1, const rb200_net_ws_t* ws_q2, void* stream);
/* value step (SAC with a value network, after the alpha step): V(s) against min_q_out, or    */
/*   min_q_out - alpha * clamp(log_prob_out) with the post-update alpha; MSE loss -> loss[0],  */
/*   dZ chain of the value network into ws_value (weight gradients: rb200_mlp_wgrad).          */
int rb200_ac_value_step(const rb200_mlp_t* value, const rb200_ac_args_t* args,
                        const rb200_net_ws_t* ws_value, void* stream);

/* ------------------------------------------------------------------------- */
/* Weight gradients: dW_l = dZ_l^T . A_{l-1}, db_l = sum_b dZ_l, split over    */
/* the batch; partial s lands at gpart + s*n_params (arena layout), on mma.sync */
/* 3xTF32 tiles (rb200_optim.cu).                                               */
/* Replaces autograd's Linear backward (torch) reached from                    */
/* loss.backward() in the Lightning loop (reagent_lightning_module.py:108-133).*/
/* ------------------------------------------------------------------------- */
/* batch splits for rb200_mlp_wgrad: one per 256 rows, between 1 and 64 */
int rb200_wgrad_splits(int batch);
int rb200_mlp_wgrad(const rb200_mlp_t* net, const float* net_input, int32_t batch,
                    const rb200_net_ws_t* ws, float* gpart, int32_t splits, void* stream);
/* g[i] = sum_s gpart[s*P + i]  (fixed order; feeds all-reduce / .grad views) */
int rb200_grad_reduce(const float* gpart, int32_t splits, int64_t n, float* g, void* stream);

/* ------------------------------------------------------------------------- */
/* K3: fused Adam + soft target update over flat arenas.                        */
/* Replaces torch.optim.Adam.step / AdamW.step (reagent/optimizer/optimizer.py: */
/* 64-85, uninferrable_optimizers.py:23-33, 70-78) and SoftUpdate.step          */
/* (reagent/optimizer/soft_update.py:47-71) in this order per element:          */
/* Adam on the source, then target = tau*new_source + (1-tau)*target.           */
/* `step` is a device int64 counter incremented by the kernel (graph friendly). */
/* ------------------------------------------------------------------------- */
typedef struct rb200_adam_args {
  float* params;          /* [n] */
  const float* grad;      /* [splits, n] partials, summed in order */
  int32_t splits;
  int64_t n;
  float* exp_avg;         /* [n] */
  float* exp_avg_sq;      /* [n] */
  int64_t* step;          /* [1] device */
  uint32_t* block_counter;/* [1] zero-initialised scratch, self-resetting */
  double lr, beta1, beta2, eps, weight_decay;
  float grad_scale;       /* multiplies the summed gradient (1/world for DP) */
  float* target;          /* [n] or NULL: fused Polyak update */
  float tau;
  float one_minus_tau;    /* float(1.0 - tau) computed in double on the host */
  float* exp_out;         /* [n] or NULL: exp(new param) (SAC: entropy_temperature =
                             log_alpha.exp(), sac_trainer.py:322) */
  /* Optional: also write the hi/lo tensor-core weight images of the UPDATED parameters (and of
   * the updated target) for the next rb200_dqn_td_step_tc, which can then be called with
   * weights_packed = 1 -- the work of rb200_dqn_tc_pack without its launch.  tc_net describes
   * the network whose arena `params` is (tc_net->params == params); needs `target`. */
  const rb200_mlp_t* tc_net;   /* NULL: no packing */
  void* tc_pack_ws;            /* the scratch buffer of rb200_dqn_td_step_tc */
  int64_t tc_pack_ws_bytes;
  int32_t tc_do_backward;      /* also the transposed images of the backward */
  /* Optional: data-parallel gradient exchange FUSED into this launch (dp_world > 1), replacing
   * rb200_grad_reduce + an NCCL all-reduce + this kernel by one kernel per rank.  Every rank
   * launches the same grid; block b of every rank (1) sums its slice of its own split-K
   * partials, (2) PUSHES the slice into every peer's receive buffer with peer-to-peer stores
   * over NVLink and raises a per-block flag there, (3) waits for the W-1 flags of its own
   * slice, (4) adds the W slices in rank order -- every rank computes the bit-identical global
   * gradient -- scales by grad_scale (1/W) and runs Adam / Polyak / packing as above.
   * dp_recv[r] / dp_flags[r] are DEVICE arrays of W peer-mapped pointers (rb200_dp_ipc_open):
   *   recv  of rank r: float    [2][W][dp_stride]      (parity of the step, source rank)
   *   flags of rank r: uint32_t [2][W][dp_max_blocks]  zero-initialised once
   * Two parities suffice: a rank cannot finish step k+1 before every peer has finished step k. */
  int32_t dp_world, dp_rank;
  float* const* dp_recv;
  uint32_t* const* dp_flags;
  int64_t dp_stride;           /* >= n */
  int32_t dp_max_blocks;       /* >= the grid this call launches (rb200_adam_blocks(n)) */
  /* Optional: torch.optim.AdamW / AMSGrad (torch/optim/adam.py, _single_tensor_adam).  All zero
   * is Adam as above.
   *   decoupled_weight_decay = 1: p = p * float(1 - lr*weight_decay) before the moment updates,
   *     in place of the coupled g += weight_decay * p.
   *   amsgrad = 1: max_exp_avg_sq = maximum(max_exp_avg_sq, exp_avg_sq) (NaN propagates, as
   *     torch.maximum), and the step's denominator is built from it instead of exp_avg_sq. */
  int32_t decoupled_weight_decay;  /* 0 or 1 */
  int32_t amsgrad;                 /* 0 or 1 */
  float* max_exp_avg_sq;           /* [n]; needed when amsgrad = 1 */
} rb200_adam_args_t;
int rb200_adam_blocks(int64_t n);
int rb200_adam_soft_update(const rb200_adam_args_t* a, void* stream);
/* stand-alone Polyak update (SoftUpdate.step when not fused) */
int rb200_soft_update(float* target, const float* source, int64_t n, float tau,
                      float one_minus_tau, void* stream);


/* ------------------------------------------------------------------------- */
/* K1: fused replay sampling over device-resident storage.                     */
/* Replaces SumTree.stratified_sample/sample (reagent/replay_memory/sum_tree.py:93-153),*/
/* ReplayBuffer.sample_index_batch / sample_transition_batch                   */
/* (circular_replay_buffer.py:589-706, :741-774), PrioritizedReplayBuffer's    */
/* sampling_probabilities (prioritized_replay_buffer.py:116-147), the dense    */
/* Preprocessor on state/next_state (preprocessing/preprocessor.py:115-170) and*/
/* the InputMakers (gym/preprocessors/trainer_preprocessor.py:72-227).         */
/* Random numbers come from the HOST (bit-exact index parity): `query` are the */
/* stratified uniforms of SumTree.stratified_sample, `ranks` torch.randint's   */
/* draws; rare invalid-index retries are resolved on the host and passed as    */
/* overrides (see reagent_b200/replay_memory/prioritized_replay_buffer.py).    */
/* ------------------------------------------------------------------------- */
#define RB200_SAMPLE_PRIORITIZED 0
#define RB200_SAMPLE_UNIFORM 1
#define RB200_SAMPLE_GIVEN 2
#define RB200_VALID_BLOCK 256
#define RB200_MAX_GATHER_SPECS 12

typedef struct rb200_gather_spec {
  const void* src;     /* [capacity, row_bytes] */
  void* dst;           /* [batch, row_bytes]    */
  int32_t row_bytes;
  int32_t which;       /* 0: sampled index, 1: next index */
} rb200_gather_spec_t;

typedef struct rb200_sample_args {
  int32_t batch, capacity, update_horizon, mode;
  int32_t timeline_next;              /* next index = i+1 instead of i+steps */
  /* index sources */
  const double* tree;                 /* fp64 heap: level l at [2^l-1, 2^(l+1)-1) */
  int32_t tree_depth;
  const double* query;                /* [B] in [0,1) */
  const int32_t* override_pos;        /* [n_override] batch positions */
  const int64_t* override_idx;        /* [n_override] replacement indices */
  int32_t n_override;
  const int64_t* ranks;               /* [B] rank among valid slots */
  const uint8_t* valid;               /* [capacity] */
  const int32_t* valid_block_offsets; /* [n_valid_blocks+1] */
  int32_t n_valid_blocks;
  const int64_t* indices_in;          /* [B] */
  /* storage */
  const uint8_t* terminal;            /* [capacity] */
  const float* reward;                /* [capacity] */
  const float* decays;                /* [update_horizon] gamma**k as f32 */
  const float* obs;                   /* [capacity, obs_dim] or NULL */
  int32_t obs_dim, obs_out_dim;
  const rb200_feature_col_t* cols;    /* NULL: raw copy */
  const float* quantiles;
  float* state;                       /* [B, obs_out_dim] */
  float* next_state;
  /* discrete action (int64 scalar per slot) */
  const int64_t* action_i64;
  int32_t num_actions;
  int64_t* action_out_i64;            /* [B] */
  int64_t* next_action_out_i64;       /* [B] */
  float* action_onehot;               /* [B, num_actions] */
  float* next_action_onehot;          /* zeroed on terminal rows */
  /* continuous action (f32 row per slot) */
  const float* action_f32;
  int32_t action_dim;
  float* action_out_raw;              /* [B, action_dim] */
  float* next_action_out_raw;
  float* action_rescaled;             /* [B, action_dim] rescaled to [train_low, train_high] */
  float* next_action_rescaled;        /* zeroed on terminal rows */
  const float* action_low;            /* [action_dim] */
  const float* action_high;
  float train_low, train_high;
  /* scalar outputs, all [B] */
  float* reward_out;
  float* next_reward_out;
  uint8_t* terminal_out;
  float* not_terminal_out;
  int64_t* indices_out;
  int64_t* step_out;
  float* step_f32_out;
  float* sampling_prob_out;
  int32_t n_specs;
  rb200_gather_spec_t specs[RB200_MAX_GATHER_SPECS];
} rb200_sample_args_t;

int rb200_replay_sample(const rb200_sample_args_t* args, void* stream);
/* validity bitmap -> per-256-slot counts and exclusive offsets (uniform sampling index);
 * counts [ceil(cap/256)], offsets [ceil(cap/256)+1] */
int rb200_valid_index_build(const uint8_t* valid, int64_t capacity, int32_t* counts,
                            int32_t* offsets, void* stream);

/* ------------------------------------------------------------------------- */
/* Device-resident replay bookkeeping (rb200_replay_dev.cu): the online loop "add a      */
/* transition -> draw a prioritized minibatch -> train" without host work per step.     */
/*   rb200_replay_add_device  n consecutive ReplayBuffer.add() calls, stack_size == 1    */
/*       (circular_replay_buffer.py:468-547; validity :430-438; PER priority ->          */
/*       SumTree.set, prioritized_replay_buffer.py:62-84) from device staging rows        */
/*   rb200_sumtree_set_device PrioritizedReplayBuffer.set_priority: SumTree.set for a     */
/*       batch applied IN ORDER (sum_tree.py:164-189), fp64, bit-equal to the host heap   */
/*   rb200_per_draw_indices   sample_index_batch of the prioritized buffer                */
/*       (prioritized_replay_buffer.py:86-115): B stratified random.uniform draws from a  */
/*       DEVICE copy of CPython's MT19937 state (624 words + position, as                 */
/*       random.getstate()[1] lays them out), the tree descents, and the sequential       */
/*       non-stratified retries of invalid hits with the shared attempt budget.           */
/*   rb200_per_weights        importance weights of drawn indices for prioritized replay:  */
/*       w_i = (p_min / p_i) ** beta_t over their fp64 leaves p_i (p_min: smallest nonzero */
/*       leaf of the batch; a zero leaf gets w = 0), beta_t = min(1, beta0 + (1 - beta0) * */
/*       t / beta_updates) with t = *step (the optimizer's device step counter).  w_out    */
/*       [n] fp32, w64_out [n] fp64 or NULL.                                               */
/*   rb200_per_priority_update  TD-error priorities written back IN ORDER:                */
/*       p_i = ((double)|q_selected_i - td_target_i| + eps) ** alpha -> p_out [n], then    */
/*       SumTree.set(idx_i, p_i) for i = 0..n-1 as rb200_sumtree_set_device.  A priority   */
/*       that is not finite applies none of them and sets status 3.                        */
/*   rb200_per_priority_update_rows  the same write-back from per-row losses (the         */
/*       distributional heads, which have no scalar TD error):                             */
/*       p_i = ((double)|row_loss_i| / divisor + eps) ** alpha, divisor > 0 and finite      */
/*       (N*N for the QR-DQN head's loss_partials, 1 for C51's).                           */
/*   rb200_per_priority_exchange  the data-parallel write-back's first half: this rank's   */
/*       n_local priorities (the two formulas above, the same fp64 arithmetic) gathered    */
/*       into the whole B_global-long vector on every rank (rb200_per_exchange_args_t).    */
/*   rb200_per_priority_apply  its second half: SumTree.set(idx_i, val_i) in order, as     */
/*       rb200_sumtree_set_device but with the PER rule: a value that is not finite       */
/*       applies none of them and sets status 3.  Every rank applies the same vector, so   */
/*       every rank reaches the same tree, max_recorded and status.                        */
/* status words are sticky error flags the host wrapper turns into the reference's        */
/* exceptions: 1 = "Max sample attempts", 2 = negative priority, 3 = non-finite PER       */
/* priority (a non-finite TD error or row loss).                                          */
/* ------------------------------------------------------------------------- */
typedef struct rb200_replay_dev {
  int64_t* state;             /* [4] device: add_count, transitions in the current episode,
                                 number of valid indices, sticky error */
  int32_t capacity, update_horizon;
  uint8_t* valid;             /* [capacity] */
  uint8_t* terminal;          /* [capacity] */
  float* reward;              /* [capacity] */
  double* tree;               /* fp64 heap (level l at [2^l-1, 2^(l+1)-1)) or NULL */
  int32_t tree_depth;
  double* max_priority;       /* [1] SumTree.max_recorded_priority or NULL */
} rb200_replay_dev_t;

typedef struct rb200_add_args {
  rb200_replay_dev_t rb;
  int32_t n;                          /* transitions in this call, <= 1024 */
  const uint8_t* terminal_in;         /* [n] */
  const float* reward_in;             /* [n] */
  const double* priority_in;          /* [n] or NULL */
  int32_t n_rows;                     /* other keys: src = staging [n,row_bytes], dst = store */
  rb200_gather_spec_t rows[RB200_MAX_GATHER_SPECS];
  int32_t priority_from_max;          /* 1: a NaN priority_in means *rb.max_priority (PER) */
} rb200_add_args_t;

typedef struct rb200_per_draw_args {
  uint32_t* mt_state;         /* [625] device, updated in place */
  int32_t batch;
  const double* lo;           /* [B] np.linspace(0,1,B+1)[:-1] */
  const double* hi;           /* [B] np.linspace(0,1,B+1)[1:]  */
  const double* tree;
  int32_t tree_depth;
  const uint8_t* valid;       /* [capacity] */
  int32_t max_attempts;
  int64_t* indices_out;       /* [B] */
  double* queries_out;        /* [B] or NULL */
  int32_t* status;            /* [2]: sticky error, retries used by this call */
} rb200_per_draw_args_t;

int rb200_replay_add_device(const rb200_add_args_t* args, void* stream);
int rb200_sumtree_set_device(double* tree, int32_t depth, const int64_t* idx, const double* val,
                             int32_t n, double* max_recorded, int32_t* status, void* stream);
int rb200_per_draw_indices(const rb200_per_draw_args_t* args, void* stream);
int rb200_per_weights(const double* tree, int32_t depth, const int64_t* idx, int32_t n,
                      const int64_t* step, double beta0, double beta_updates, float* w_out,
                      double* w64_out, void* stream);
int rb200_per_priority_update(double* tree, int32_t depth, const int64_t* idx,
                              const float* td_target, const float* q_selected, int32_t n,
                              double alpha, double eps, double* p_out, double* max_recorded,
                              int32_t* status, void* stream);
int rb200_per_priority_update_rows(double* tree, int32_t depth, const int64_t* idx,
                                   const float* row_loss, int32_t n, double divisor, double alpha,
                                   double eps, double* p_out, double* max_recorded,
                                   int32_t* status, void* stream);

/* Priority exchange of a data-parallel prioritized update over NVLink peer memory, the
 * pattern of rb200_adam_args_t.dp_*.  Rank `rank` of `world` holds rows [row0, row0 + n_local)
 * of the B_global-long update.  One launch (1) computes their priorities from row_loss
 * (p = (|row_loss| / divisor + eps) ** alpha) or, with row_loss NULL, from td_target and
 * q_selected (p = (|q_selected - td_target| + eps) ** alpha), bit-identical to
 * rb200_per_priority_update[_rows]; (2) stores them at [row0, row0 + n_local) of parity
 * (epoch & 1) of every rank's receive buffer; (3) issues one system-scope fence and raises
 * its flag at every peer with the new epoch; (4) waits for the world - 1 peer flags
 * (acquire loads, 4 s bound: a lost peer fails the step, never hangs) and (5) copies the
 * gathered vector to out [B_global].
 *   recv[r]  of rank r: double   [2][B_global]  (parity of the epoch)
 *   flags[r] of rank r: uint32_t [2][world]     (parity, source rank), zero-initialised once
 * recv / flags are DEVICE arrays of world peer-mapped pointers; epoch is this rank's [1]
 * device counter, zero-initialised once and advanced by every call.  Two parities suffice:
 * a rank cannot start exchange e + 1 before every peer has started exchange e.  With
 * world == 1 recv, flags and epoch may be NULL and the priorities go straight to out. */
typedef struct rb200_per_exchange_args {
  const float* td_target;     /* [n_local] */
  const float* q_selected;    /* [n_local] */
  const float* row_loss;      /* [n_local] or NULL */
  double divisor;             /* > 0 and finite when row_loss is given */
  double alpha, eps;
  int32_t n_local, row0, B_global;
  int32_t world, rank;        /* world <= 256 */
  double* const* recv;
  uint32_t* const* flags;
  uint32_t* epoch;
  double* out;                /* [B_global] */
} rb200_per_exchange_args_t;
int rb200_per_priority_exchange(const rb200_per_exchange_args_t* args, void* stream);
int rb200_per_priority_apply(double* tree, int32_t depth, const int64_t* idx, const double* val,
                             int32_t n, double* max_recorded, int32_t* status, void* stream);

/* ------------------------------------------------------------------------- */
/* MDN-RNN (reagent/models/mdn_rnn.py, reagent/training/world_model/mdnrnn_trainer.py):  */
/* an nn.LSTM over cat(action, state) and a mixture-density head gmm_linear on every     */
/* step's top hidden state.  Three launches per update, then Adam:                      */
/*   rb200_mdnrnn_forward   per row tile, every step and layer (h / c in shared memory), */
/*                          the head, the outputs, and (with targets) the three losses   */
/*                          and dL/d(gmm_outs); with `acts` the gate activations too.    */
/*   rb200_mdnrnn_backward  BPTT per row tile: dGates[l, t] into `dgates`.               */
/*   rb200_mdnrnn_wgrad     split-K weight gradients of every LSTM layer and of the head */
/*                          into `gpart` ([splits, n_params], the arena's layout).        */
/* Layouts (dense fp32, time-major): state/next_state [T,B,S], action [T,B,A],           */
/* reward/not_terminal [T,B], out [T,B,NG] with NG = (2S+1)G + 2 = mus (G*S) | sigmas     */
/* (G*S, exp applied) | logpi (G) | reward | not_terminal; hs / cs [L, T+1, B, H] with    */
/* slot 0 = the zero initial state (written by the forward); xin [T,B,A+S];              */
/* acts / dgates [L,T,B,4H] (i, f, g, o); dy [T,B,NG].                                    */
/* Limits: H <= 128, L <= 4, G <= 32, A + S <= 256, NG <= 1024; anything past them is     */
/* refused with RB200_E_INVALID before a launch.                                          */
/* ------------------------------------------------------------------------- */
#define RB200_MDNRNN_MAX_HIDDEN 128
#define RB200_MDNRNN_MAX_LAYERS 4
#define RB200_MDNRNN_MAX_GAUSSIANS 32
#define RB200_MDNRNN_MAX_INPUT 256
#define RB200_MDNRNN_MAX_OUT 1024
#define RB200_MDNRNN_ROWS_PER_BLOCK 16 /* loss_partials holds 3 * ceil(B / 16) floats */
typedef struct rb200_mdnrnn_args {
  int32_t seq_len, batch, state_dim, action_dim, hidden, layers, gaussians;
  const float* params;                           /* the arena */
  int64_t n_params;
  int64_t w_ih_off[RB200_MDNRNN_MAX_LAYERS], w_hh_off[RB200_MDNRNN_MAX_LAYERS];
  int64_t b_ih_off[RB200_MDNRNN_MAX_LAYERS], b_hh_off[RB200_MDNRNN_MAX_LAYERS];
  int64_t w_gmm_off, b_gmm_off;
  const float* state;
  const float* action;
  /* targets: all three or none (no loss) */
  const float* next_state;
  const float* reward;
  const float* not_terminal;
  float next_state_weight, not_terminal_weight, reward_weight;
  float gmm_divisor;                             /* loss = gmm / gmm_divisor + bce + mse */
  int32_t fit_only_one_next_step;                /* loss on the last step only           */
  float* out;                                    /* or NULL                              */
  float* hs;
  float* cs;
  /* training: all or none */
  float* xin;
  float* acts;
  float* dgates;
  float* dy;
  /* loss (with targets) */
  float* loss_partials;
  uint32_t* tile_counter;
  float* loss;                                   /* [4]: gmm, bce, mse, loss */
  /* weight gradients */
  float* gpart;
  int32_t splits;
} rb200_mdnrnn_args_t;
/* 0 if the shape is within the limits above, else RB200_E_INVALID (text via last_error) */
int rb200_mdnrnn_check_shape(int32_t state_dim, int32_t action_dim, int32_t hidden,
                             int32_t layers, int32_t gaussians);
int rb200_mdnrnn_forward(const rb200_mdnrnn_args_t* args, void* stream);
int rb200_mdnrnn_backward(const rb200_mdnrnn_args_t* args, void* stream);
int rb200_mdnrnn_wgrad(const rb200_mdnrnn_args_t* args, void* stream);

/* World-model evaluation (reagent/evaluation/world_model_evaluator.py):                  */
/*   rb200_mdnrnn_eval         the loss of num_variants perturbed copies of one batch in one  */
/*                             launch, grid [ceil(B / 16), V].  Variant v replaces columns     */
/*                             [col_begin[v], col_end[v]) of x = cat(action, state) by         */
/*                             fill[fill_off[v] ...] at every step and row (an empty range     */
/*                             keeps x); variant perm_variant (or -1) reads action row perm[b] */
/*                             (int64 [B]) for row b.  Targets are never changed.  `net` gives */
/*                             the shape, arena, inputs, targets, loss weights, gmm_divisor   */
/*                             and fit_only_one_next_step; its outputs, workspace and loss     */
/*                             buffers are not read.  Writes loss [V][4] (gmm, bce, mse, loss) */
/*                             -- each variant's the bits rb200_mdnrnn_forward gives on the    */
/*                             batch with its replacement made -- and, when mus is not NULL,   */
/*                             the means mus [V][T][B][G*S].  loss_partials holds              */
/*                             V * 3 * ceil(B / 16) floats, tile_counter V zeros.  A perm      */
/*                             value outside [0, B) makes that variant's results NaN.          */
/*   rb200_mdnrnn_fill_values  per feature group of x's columns (rows = T * B): a width-1     */
/*                             group's column mean (fp64 sum, rounded once); a wider (enum)    */
/*                             group's one-hot at the first column whose column sum equals the */
/*                             lower median of the group's column sums.  Into fill[column].   */
/*   rb200_mdnrnn_sensitivity  per group of state columns: the mean over (rows, G) of the sum  */
/*                             over the group's columns of |mus1 - mus0| (mus [rows, G, S]).   */
/* Groups: num_groups >= 1, group g is [group_begin[g], group_begin[g + 1]), boundaries       */
/* strictly increasing inside [0, width].  Limits: the MDN-RNN limits, and                   */
/* 1 <= num_variants <= 1 + action_dim + state_dim (<= 257).                                 */
#define RB200_MDNRNN_EVAL_MAX_VARIANTS (RB200_MDNRNN_MAX_INPUT + 1)
typedef struct rb200_mdnrnn_eval_args {
  rb200_mdnrnn_args_t net;
  int32_t num_variants;
  int32_t col_begin[RB200_MDNRNN_EVAL_MAX_VARIANTS];
  int32_t col_end[RB200_MDNRNN_EVAL_MAX_VARIANTS];
  int32_t fill_off[RB200_MDNRNN_EVAL_MAX_VARIANTS];
  const float* fill;
  int32_t fill_len;                              /* floats in fill */
  int32_t perm_variant;
  const int64_t* perm;
  float* mus;                                    /* or NULL */
  float* loss_partials;
  uint32_t* tile_counter;
  float* loss;
} rb200_mdnrnn_eval_args_t;
typedef struct rb200_mdnrnn_fill_args {
  int32_t rows, action_dim, state_dim;
  const float* action;                           /* [rows, action_dim] */
  const float* state;                            /* [rows, state_dim] */
  int32_t num_groups;
  int32_t group_begin[RB200_MDNRNN_MAX_INPUT + 1];  /* columns of x, width action_dim + state_dim */
  float* fill;                                   /* [action_dim + state_dim] */
} rb200_mdnrnn_fill_args_t;
typedef struct rb200_mdnrnn_sensitivity_args {
  int32_t rows, state_dim, gaussians;
  const float* mus0;
  const float* mus1;
  int32_t num_groups;
  int32_t group_begin[RB200_MDNRNN_MAX_INPUT + 1];  /* state columns, width state_dim */
  float* out;                                    /* [num_groups] */
} rb200_mdnrnn_sensitivity_args_t;
int rb200_mdnrnn_eval(const rb200_mdnrnn_eval_args_t* args, void* stream);
int rb200_mdnrnn_fill_values(const rb200_mdnrnn_fill_args_t* args, void* stream);
int rb200_mdnrnn_sensitivity(const rb200_mdnrnn_sensitivity_args_t* args, void* stream);

/* ------------------------------------------------------------------------- */
/* Cross-entropy-method planner (reagent/models/cem_planner.py): one launch of          */
/* rb200_cem_rollout per CEM iteration.  CTA (j, m) of the grid [ceil(P / 16), K] takes  */
/* the j-th group of 16 trajectories that drew world model m (model_idx), carries them   */
/* through all `horizon` steps -- each a T = 1 MDN-RNN forward from h = c = 0, so W_hh   */
/* drops out and c' = i * g -- samples mixture / next state / terminal from the noise,   */
/* and writes each trajectory's fp64 value.  The last CTA to finish reduces:             */
/*   continuous: elites (the num_elites largest values, ties to the larger index),       */
/*     mean / var update in fp64, `done` = 1 once max(var) <= epsilon;                   */
/*   discrete: first-action tally, nanargmax into action_out / one_hot.                  */
/* A launch that finds `done` set returns at once, so a plan needs no host sync.         */
/* Noise (dense, per plan): model_idx int32 [iters, P]; action_idx int32 [P, horizon]    */
/* (discrete); truncnorm fp64 [iters, P, horizon * A] (continuous); step_noise fp32      */
/* [iters, P, horizon, S + 2] = mixture uniform | S standard normals | Bernoulli uniform. */
/* `net` carries the shape and arena offsets (identical for every model); its params,    */
/* seq_len and batch are not read.                                                        */
/* Limits: the MDN-RNN limits, P <= 1024, K <= 8, horizon * A <= 4096,                    */
/* 1 <= num_elites <= P, horizon >= 1.                                                    */
/* ------------------------------------------------------------------------- */
#define RB200_CEM_MAX_MODELS 8
#define RB200_CEM_MAX_POPULATION 1024
#define RB200_CEM_MAX_PLAN 4096 /* horizon * action_dim */
#define RB200_CEM_ROWS_PER_BLOCK 16
typedef struct rb200_cem_args {
  rb200_mdnrnn_args_t net;
  int32_t num_models;
  const float* params[RB200_CEM_MAX_MODELS]; /* arena of each world model */
  int32_t population, horizon, iters, num_elites;
  int32_t discrete, terminal_effective;
  int32_t iter;                              /* the iteration this launch runs */
  double alpha, epsilon;
  const float* state;                        /* [S] */
  const float* discount;                     /* [horizon] fp32(gamma ** j) */
  const double* lower;                       /* [horizon * A] tiled bounds (continuous) */
  const double* upper;
  const int32_t* model_idx;
  const int32_t* action_idx;
  const double* truncnorm;
  const float* step_noise;
  double* mean;                              /* [horizon * A], read and updated */
  double* var;
  double* values;                            /* [iters, P] */
  int32_t* elites;                           /* [iters, num_elites], ascending value */
  double* mean_hist;                         /* [iters, horizon * A] after each update */
  double* var_hist;
  int32_t* done;
  int32_t* n_iters;
  int64_t* action_out;                       /* discrete: [1] */
  float* one_hot;                            /* discrete: [A] */
  uint32_t* counter;                         /* 0 between launches */
  float* dump;                               /* or NULL: iteration 0's per-step input and */
                                             /* head outputs, [P, horizon, A + S + NG]    */
} rb200_cem_args_t;
int rb200_cem_check_shape(int32_t state_dim, int32_t action_dim, int32_t hidden, int32_t layers,
                          int32_t gaussians, int32_t population, int32_t num_models,
                          int32_t horizon, int32_t num_elites);
int rb200_cem_rollout(const rb200_cem_args_t* args, void* stream);

/* ------------------------------------------------------------------------- */
/* Seq2Reward (reagent/models/seq2reward_model.py, reagent/training/world_model/         */
/* seq2reward_trainer.py, compress_model_trainer.py): an nn.LSTM over the one-hot action  */
/* sequence whose initial h of every layer is map_linear(state[0]) (c = 0), and a width-1 */
/* head lstm_linear on the top h of step valid_step - 1.  Per update:                     */
/*   rb200_seq2reward_forward   per 16-row tile: h0, every step and layer (h / c in       */
/*                              shared memory), acc_reward; with `reward` the target       */
/*                              cumsum(reward * discount)[valid - 1] (fp64 sum, rounded    */
/*                              once), the MSE (`loss`) and dy; with `step_labels` the     */
/*                              one-hot [B, multi_steps] of valid - 1.                     */
/*   rb200_seq2reward_backward  BPTT per row tile: dGates into `dgates`, and dh0 = the sum  */
/*                              over layers of dL/dh_{-1} (the map_linear output gradient). */
/*   rb200_seq2reward_wgrad     split-K weight gradients of every layer and lstm_linear     */
/*                              over T*B rows, then map_linear over B rows, into `gpart`.   */
/* valid_step (int64 [B], or NULL = T) is clamped to [1, T] by the kernels; callers check  */
/* its range.  No k-chunk rotation (see tile_linear_fwd): a row's outputs are the same in  */
/* whichever CTA computes it, which makes the plan bit-identical to the forward.           */
/* Layouts (dense fp32): state [B, S] (the sequence's first state), action [T, B, A],     */
/* reward [T, B], discount [T] = fp32(gamma ** t), acc_reward / target [B],               */
/* dy [T, B] = dL/dacc_reward on step valid - 1, else 0; hs / cs [L, T+1, B, H] with slot  */
/* 0 = the initial state; acts / dgates [L, T, B, 4H] (i, f, g, o); dh0 [B, H].            */
/* Limits: H <= 128, L <= 4 (the MDN-RNN limits), 1 <= S <= 256, 1 <= A <= 16,             */
/* 1 <= multi_steps <= 16, A ** multi_steps <= 65536, and the forward's tile within the    */
/* 227 KiB of shared memory of one CTA: 4 * (2 * 9216 + 16 * (round_up4(max(S, A)) + 4 +   */
/* (2L + 1)(round_up4(H) + 4) + 2 (round_up4(4H) + 4) + 1)) + 64 bytes, so L 4 with        */
/* H 128 takes S <= 252 (every other H, L takes S 256).  Anything else is refused before   */
/* any launch.                                                                              */
/* ------------------------------------------------------------------------- */
#define RB200_SEQ2REWARD_MAX_STATE 256
#define RB200_SEQ2REWARD_MAX_ACTIONS 16
#define RB200_SEQ2REWARD_MAX_STEPS 16
#define RB200_SEQ2REWARD_MAX_PERMUTATIONS 65536 /* num_action ** multi_steps */
#define RB200_SEQ2REWARD_PLAN_BUDGET_BYTES 268435456 /* plan workspace cap (256 MiB) */
#define RB200_SEQ2REWARD_ROWS_PER_BLOCK 16 /* loss_partials holds ceil(B / 16) floats */
typedef struct rb200_seq2reward_args {
  int32_t seq_len, batch, state_dim, action_dim, hidden, layers;
  const float* params;                           /* the arena */
  int64_t n_params;
  int64_t w_ih_off[RB200_MDNRNN_MAX_LAYERS], w_hh_off[RB200_MDNRNN_MAX_LAYERS];
  int64_t b_ih_off[RB200_MDNRNN_MAX_LAYERS], b_hh_off[RB200_MDNRNN_MAX_LAYERS];
  int64_t w_lin_off, b_lin_off;                  /* lstm_linear [1, H], [1] */
  int64_t w_map_off, b_map_off;                  /* map_linear [H, S], [H] */
  const float* state;
  const float* action;
  const int64_t* valid_step;                     /* or NULL */
  float* acc_reward;
  /* target and loss: reward, discount, target, loss_partials, tile_counter, loss, or none */
  const float* reward;
  const float* discount;
  float* target;
  float* loss_partials;
  uint32_t* tile_counter;
  float* loss;                                   /* [1] */
  float* step_labels;                            /* [B, multi_steps] or NULL */
  int32_t multi_steps;
  /* training (needs the target): hs, cs, acts, dy; the backward adds dgates and dh0 */
  float* hs;
  float* cs;
  float* acts;
  float* dy;
  float* dgates;
  float* dh0;
  /* weight gradients */
  float* gpart;
  int32_t splits;
} rb200_seq2reward_args_t;
/* rb200_seq2reward_plan: get_Q over the prefix tree of the action sequences.  q[b, a] is   */
/* the max of lstm_linear(h_top) over the A ** (k-1) sequences of length k that start with */
/* a; q_all[b, j-1, a] the same max over the sequences of length j, for j = 1..k.  Level j */
/* (one launch per level and state chunk) carries its B * A ** j nodes one LSTM step from  */
/* their parents: node i's children are i * A + a, the input is the one-hot of a.  Level j */
/* < k stores node i's h / c ([L, 2, H] per node) at row i * A ** (k-1-j) of `workspace`;  */
/* child 0 takes its parent's row, so a CTA holds every child of its parents (16 / A       */
/* parents, 16 / A * A rows).  Level k stores nothing.  Peak workspace = Bc * A ** (k-1) * */
/* L * 2 * H * 4 bytes for a chunk of Bc states: the call chunks the batch to what         */
/* `workspace_bytes` holds (rb200_seq2reward_plan_workspace_bytes gives the size for a     */
/* batch, at most RB200_SEQ2REWARD_PLAN_BUDGET_BYTES).  The maxima are taken by atomicMax  */
/* on order-preserving integer images in `qbits` [B, k, A] (order-free, so deterministic). */
typedef struct rb200_seq2reward_plan_args {
  rb200_seq2reward_args_t net;                   /* shape and arena; its seq_len, batch,   */
                                                 /* state, action and buffers are not read */
  int32_t batch, multi_steps;                    /* num_action is net.action_dim           */
  const float* state;                            /* [B, S] */
  float* q;                                      /* [B, A] */
  float* q_all;                                  /* [B, k, A] or NULL */
  uint32_t* qbits;                               /* [B, k, A] */
  float* workspace;
  int64_t workspace_bytes;
} rb200_seq2reward_plan_args_t;
/* CompressModelTrainer's head: loss = mean((out - q) ** 2) over B * A, dout = dL/dout (or */
/* NULL), accuracy = mean(argmax q == argmax out), first maximum on ties.  out / q [B, A]; */
/* loss_partials holds 2 * ceil(B / 256) floats; out_loss [2] = loss, accuracy.           */
typedef struct rb200_seq2reward_compress_args {
  int32_t batch, num_action;
  const float* out;
  const float* q;
  float* dout;
  float* loss_partials;
  uint32_t* tile_counter;
  float* out_loss;
} rb200_seq2reward_compress_args_t;
/* 0 if the shape is within the limits above, else RB200_E_INVALID (text via last_error) */
int rb200_seq2reward_check_shape(int32_t state_dim, int32_t action_dim, int32_t hidden,
                                 int32_t layers, int32_t multi_steps);
int rb200_seq2reward_forward(const rb200_seq2reward_args_t* args, void* stream);
int rb200_seq2reward_backward(const rb200_seq2reward_args_t* args, void* stream);
int rb200_seq2reward_wgrad(const rb200_seq2reward_args_t* args, void* stream);
int64_t rb200_seq2reward_plan_workspace_bytes(int32_t batch, int32_t action_dim,
                                              int32_t multi_steps, int32_t hidden, int32_t layers);
int rb200_seq2reward_plan(const rb200_seq2reward_plan_args_t* args, void* stream);
int rb200_seq2reward_compress_head(const rb200_seq2reward_compress_args_t* args, void* stream);

/* ------------------------------------------------------------------------- */
/* Seq2Slate transformer (reagent/models/seq2slate.py, rb200_seq2slate.cu): embedders, L    */
/* post-norm encoder layers, then the decoder (AUTOREGRESSIVE: L - 1 TransformerDecoderLayers */
/* and the head-averaged cross-attention weights of the last one; FRECHET_SORT: a masked      */
/* softmax of encoder_scorer(memory)).  One CTA carries one slate through all of it; the      */
/* decoder runs one position per step on cached self-attention keys / values, which is exact  */
/* because position t depends only on positions <= t and on tgt_in_idx[0..t].               */
/*   rb200_seq2slate_forward  decode FORCED (teacher forcing on tgt_in_idx / tgt_in_seq):    */
/*                            probs [B, T, N+2], log_probs = log(clamp(probs, 1e-40)) and    */
/*                            seq_log_prob [B] = log(clamp(prod_t probs[t, tgt_out_idx[t]],  */
/*                            1e-40)); each output may be NULL (one must be given).           */
/*   rb200_seq2slate_rank     decode GREEDY (first maximal index at every step) or SAMPLE     */
/*                            (the first symbol whose running sum of probabilities exceeds    */
/*                            noise[b, t] * their total, in candidate order): ranked_idx      */
/*                            [B, T], probs (the ranked per-symbol probabilities, or NULL)    */
/*                            and seq_prob [B] = clamp(prod, 1e-40).  FRECHET_SORT GREEDY is  */
/*                            the argsort of the first step's probabilities (ties: lowest     */
/*                            index first) with one-hot probs and seq_prob 1.                 */
/* Indices count the padding and start symbols (candidate i is symbol i + 2); the decoder's   */
/* first input in rank mode is the start symbol 1, whose features are zeros.                  */
/* off[] holds the offsets in `params` of the reference's parameters() in order: per encoder  */
/* layer 12 (in_proj w/b, out_proj w/b, linear1 w/b, linear2 w/b, norm1 w/b, norm2 w/b),     */
/* encoder_scorer w/b, per decoder layer 18 (self_attn in/out, multihead_attn in/out, linear1, */
/* linear2, norm1..3, each w/b), pos_embed w/b, state_embedder w/b, candidate_embedder w/b.    */
/* Layouts (dense fp32 unless noted): state [B, S], src_seq [B, N, C], tgt_in_idx /           */
/* tgt_out_idx / ranked_idx int64 [B, T], tgt_in_seq [B, T, C], noise [B, T].                 */
/* Limits: 1 <= S, C <= 256, 2 <= dim_model <= 128 divisible by num_heads, 1 <=               */
/* state_embed_dim < dim_model, dim_feedforward <= 512, 1 <= layers <= 4, 1 <= N <= 64 and    */
/* 1 <= T <= N.  Each CTA loops over slates with a workspace slice of about 4 * (N(4d +       */
/* max(3d, FFN)) + 2 L T d) bytes: in shared memory when that is at most 200 KiB (as many CTAs */
/* as fit on the device), else in `workspace`, which then holds                               */
/* rb200_seq2slate_workspace_bytes(args) for min(B, RB200_SEQ2SLATE_MAX_CTAS) CTAs (the size */
/* is 0, and `workspace` may be NULL, on the shared-memory path).  Anything else is refused  */
/* before any launch.                                                                         */
/* ------------------------------------------------------------------------- */
#define RB200_SEQ2SLATE_MAX_CANDIDATES 64
#define RB200_SEQ2SLATE_MAX_DIM_MODEL 128
#define RB200_SEQ2SLATE_MAX_FEEDFORWARD 512
#define RB200_SEQ2SLATE_MAX_LAYERS 4
#define RB200_SEQ2SLATE_MAX_INPUT 256
#define RB200_SEQ2SLATE_MAX_PARAMS (30 * RB200_SEQ2SLATE_MAX_LAYERS + 8)
#define RB200_SEQ2SLATE_MAX_CTAS 1056 /* 8 per SM of an H100 SXM */
#define RB200_SEQ2SLATE_ARCH_AUTOREGRESSIVE 0
#define RB200_SEQ2SLATE_ARCH_FRECHET_SORT 1
#define RB200_SEQ2SLATE_DECODE_FORCED 0
#define RB200_SEQ2SLATE_DECODE_GREEDY 1
#define RB200_SEQ2SLATE_DECODE_SAMPLE 2
typedef struct rb200_seq2slate_args {
  int32_t batch, src_len, tgt_len, state_dim, candidate_dim, state_embed_dim;
  int32_t dim_model, num_heads, dim_feedforward, layers, arch, decode;
  const float* params;                           /* the arena */
  int64_t n_params;
  int64_t off[RB200_SEQ2SLATE_MAX_PARAMS];
  const float* state;
  const float* src_seq;
  const int64_t* tgt_in_idx;                     /* FORCED */
  const int64_t* tgt_out_idx;                    /* FORCED */
  const float* tgt_in_seq;                       /* FORCED, AUTOREGRESSIVE */
  const float* noise;                            /* SAMPLE: uniforms in [0, 1) */
  float* probs;                                  /* [B, T, N + 2] or NULL */
  float* log_probs;                              /* FORCED: [B, T, N + 2] or NULL */
  float* seq_log_prob;                           /* FORCED: [B] or NULL */
  int64_t* ranked_idx;                           /* rank */
  float* seq_prob;                               /* rank: [B] */
  float* workspace;
  int64_t workspace_bytes;
} rb200_seq2slate_args_t;
/* 0 if the model shape is within the limits above, else RB200_E_INVALID (text via last_error) */
int rb200_seq2slate_check_shape(int32_t state_dim, int32_t candidate_dim, int32_t state_embed_dim,
                                int32_t dim_model, int32_t num_heads, int32_t dim_feedforward,
                                int32_t layers, int32_t max_src_seq_len, int32_t max_tgt_seq_len);
int64_t rb200_seq2slate_workspace_bytes(const rb200_seq2slate_args_t* args);
/* CTAs a launch of args runs, each looping over slates b, b + ctas, ... (on the shared-memory */
/* path as many as fit on the current device at once), or a negative RB200_E_* code           */
int rb200_seq2slate_ctas(const rb200_seq2slate_args_t* args);
int rb200_seq2slate_forward(const rb200_seq2slate_args_t* args, void* stream);
int rb200_seq2slate_rank(const rb200_seq2slate_args_t* args, void* stream);

/* ------------------------------------------------------------------------- */
/* Counterfactual policy evaluation (rb200_ope.cu), reagent/evaluation/*.py.  Every input is */
/* a dense row-major device array of the page's N rows; episodes are runs of equal mdp_id */
/* in a page sorted by (mdp_id, sequence_number, row).  ep_off[E+1] are their row offsets. */
/*   rb200_ope_page          per-row fields of EvaluationDataPage.create_from_tensors_dqn  */
/*   rb200_ope_episode_marks episode starts + validate()'s sequence / run checks           */
/*   rb200_ope_logged_values compute_values_for_mdps, column 0 of [N, C]                     */
/*   rb200_ope_sdr           SequentialDoublyRobustEstimator's per-episode value and return */
/*   rb200_ope_dr_rows       DoublyRobustEstimator's DM, IPS and DR rows                     */
/*   rb200_ope_boot_means    bootstrap sample means, from given int32 indices or in-kernel  */
/*                           Philox draws (idx == NULL)                                     */
/*   rb200_ope_wsdr_rows     WSDR per-row cumulative importance weights, V(s), Q(s, a_log)  */
/*   rb200_ope_seg_sum       fixed-order sums of segments (perm: row order, or NULL)        */
/*   rb200_ope_wsdr_returns  normalised weights -> every j-step return per trajectory      */
/*   rb200_ope_cov           np.cov of [J, T] rows, ddof 1                                   */
/* fp64 = 1 selects float64 weights (the padded trajectories of the reference), 0 float32.  */
/* ------------------------------------------------------------------------- */
#define RB200_OPE_MAX_J 32
int rb200_ope_page(int32_t n, int32_t num_actions, int32_t num_metrics, const float* q,
                   const float* reward_out, const float* qcpe_out, const float* mask,
                   const float* action, const float* reward, const float* reward_boost,
                   float temperature, float* boosted_reward, float* propensities,
                   int64_t* eval_action_idx, float* model_reward_logged,
                   float* model_metrics_logged, float* model_metrics_values_logged, void* stream);
int rb200_ope_episode_marks(int32_t n, const int64_t* mdp_id, const int64_t* seq,
                            uint8_t* is_start, int32_t* flags, void* stream);
/* step_discount[r] = (float)pow(gamma, seq[r+1] - seq[r]), computed by the host's libm pow */
int rb200_ope_logged_values(int32_t num_episodes, const int32_t* ep_off,
                            const float* step_discount, int32_t cols, const float* x, float* out,
                            void* stream);
int rb200_ope_sdr(int32_t num_episodes, const int32_t* ep_off, int32_t num_actions,
                  const float* propensities, const float* model_values, const float* action_mask,
                  const float* logged_reward, const float* logged_propensity, float gamma,
                  float* episode_dr, float* episode_value, void* stream);
int rb200_ope_dr_rows(int32_t n, int32_t num_actions, const float* propensities,
                      const float* model_rewards, const float* action_mask,
                      const float* logged_reward, const float* model_reward_logged,
                      const float* logged_propensity, float* dm, float* ips, float* dr,
                      void* stream);
int rb200_ope_boot_means(const float* data, int32_t n, const int32_t* idx, int32_t samples,
                         int32_t sample_size, int64_t seed, int64_t offset, double* means,
                         void* stream);
int rb200_ope_wsdr_rows(int32_t num_episodes, const int32_t* ep_off, int32_t num_actions,
                        int32_t fp64, const float* propensities, const float* model_values,
                        const float* action_mask, const float* logged_propensity, void* weight,
                        void* state_value, void* q_logged, void* stream);
int rb200_ope_seg_sum(int32_t fp64, const void* x, const int64_t* perm, const int64_t* seg_off,
                      int32_t num_segments, void* out, void* stream);
int rb200_ope_wsdr_returns(int32_t num_episodes, const int32_t* ep_off, int32_t fp64,
                           const void* weight, const void* state_value, const void* q_logged,
                           const float* logged_reward, const double* discounts, int32_t max_len,
                           const void* col_sum, int32_t num_j, const int32_t* j_steps,
                           int32_t num_subsets, const int32_t* subset_off, const void* subset_col_sum,
                           double* ret, double* subset_ret, double* episode_value, void* stream);
int rb200_ope_cov(const double* x, int32_t rows, int32_t cols, double* cov, void* stream);

/* ------------------------------------------------------------------------- */
/* Peer-memory plumbing of the fused data-parallel step (one process per GPU).  The    */
/* reference has no collective on this path (docs/distributed.rst:12-22 states the     */
/* intent: synchronous data parallelism with a gradient all-reduce).                   */
/*   rb200_dp_alloc      cudaMalloc'ed, zero-filled, IPC-exportable device buffer      */
/*   rb200_dp_ipc_handle 64-byte handle of such a buffer (cudaIpcGetMemHandle)          */
/*   rb200_dp_ipc_open   map a peer process's buffer into this one (enables peer access)*/
/* ------------------------------------------------------------------------- */
#define RB200_IPC_HANDLE_BYTES 64
int rb200_dp_alloc(int64_t bytes, void** out_ptr);
int rb200_dp_free(void* ptr);
int rb200_dp_ipc_handle(void* ptr, unsigned char* handle_out_host);
int rb200_dp_ipc_open(const unsigned char* handle_host, void** out_ptr);
int rb200_dp_ipc_close(void* ptr);

/* ---- host-side helpers (plain C, no CUDA; pointers are HOST memory) -------- */
/* MT19937 with CPython's exact stream: fills out[i] = lo[i] + (hi[i]-lo[i])*random()
 * (random.uniform, Lib/random.py) or random() itself when lo/hi are NULL.
 * state624 + *index are CPython's random.getstate()[1] (624 words + position). */
void rb200_mt19937_uniform_host(uint32_t* state624, int32_t* index, const double* lo_host,
                                const double* hi_host, double* out_host, int64_t n);
/* SumTree.set for a batch, sequentially, on a host fp64 heap (sum_tree.py:164-189).
 * Returns -1 if a value is negative (nothing after it is applied). */
int rb200_sumtree_set_host(double* tree_host, int32_t depth, const int64_t* idx_host,
                           const double* val_host, int64_t n, double* max_recorded_host);
/* Validity bookkeeping of n consecutive ReplayBuffer.add() calls, stack_size == 1
 * (circular_replay_buffer.py:468-522).  state = {add_count, episode length, num valid}. */
void rb200_replay_add_batch_host(const uint8_t* terminal_in_host, int64_t n, int64_t capacity,
                                 int32_t update_horizon, uint8_t* valid_host,
                                 uint8_t* terminal_store_host, int64_t* state_host);
/* SumTree.sample(query) on the host heap (sum_tree.py:93-131). */
int64_t rb200_sumtree_sample_host(const double* tree_host, int32_t depth, double query);
/* the same walk for queries[pos[0..n)] -> out[0..n) (PER retry check of one stratified draw) */
void rb200_sumtree_sample_many_host(const double* tree_host, int32_t depth, const double* queries,
                                    const int64_t* pos, int64_t n, int64_t* out);

#ifdef __cplusplus
}
#endif
#endif /* REAGENT_B200_H_ */
