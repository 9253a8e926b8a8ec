/*
 * gops_b200.h -- C ABI of libgops_b200.so: the H100 (sm_90a) implementation of GOPS's batched
 * model-rollout + ADP-update hot path.
 *
 * The reference (GOPS) has no FFI: its boundary for this path is the Python plugin API
 * (gops/algorithm/{fhadp,infadp}.py, gops/apprfunc/mlp.py, gops/env/.../env_model/*_model.py,
 * gops/env/wrapper/*.py assembled by gops/create_pkg/create_env_model.py:104-126).  The Python
 * classes in gops_b200/ mirror that API and call the entry points below through ctypes.  Every
 * entry point names the reference code it replaces.
 *
 * Conventions
 *   - all data pointers are DEVICE pointers owned by the caller (plain float32 / int32 arrays);
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on that stream;
 *   - return value 0 = ok; non-zero = error, message available from gops_b200_last_error();
 *   - a plan is bound to the device that was current at creation; one plan per host thread.
 *   - parameter vectors are the torch `parameters()` order of an `mlp()` Sequential, flattened:
 *     W1[h][in], b1[h], W2[h][h], b2[h], W3[out][h], b3[out]      (gops/apprfunc/mlp.py:36-41)
 */
#ifndef GOPS_B200_H
#define GOPS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GOPS_B200_ABI_VERSION 4   /* 2: plan_desc.open_loop, mlpnet_*, plan_set_path, launch_count; 3: peer_*; 4: veh_detour, batch.surr */
#define GOPS_B200_MAX_ACT 4   /* action dims supported by the fused kernels            */
#define GOPS_B200_MAX_LQ_N 8  /* pyth_lq state dim upper bound (configs ship n <= 6)   */

/* algorithm kinds ------------------------------------------------------------------------- */
enum {
  GOPS_ALG_FHADP = 0,        /* FHADP._compute_loss_policy        gops/algorithm/fhadp.py:113-125  */
  GOPS_ALG_INFADP_POLICY = 1,/* INFADP.__compute_loss_policy      gops/algorithm/infadp.py:188-213 */
  GOPS_ALG_INFADP_VALUE = 2  /* INFADP.__compute_loss_v           gops/algorithm/infadp.py:159-186 */
};

/* env-model kinds --------------------------------------------------------------------------- */
enum {
  GOPS_MODEL_IDPENDULUM = 0,      /* env_ocp/env_model/pyth_idpendulum_model.py:199-216           */
  GOPS_MODEL_LQ = 1,              /* env_ocp/resources/lq_base.py:343-354                         */
  GOPS_MODEL_VEH3DOFCONTI = 2,    /* env_ocp/env_model/pyth_veh3dofconti_model.py:91-145          */
  GOPS_MODEL_VEH3DOF_TRACKING = 3,/* env_gen_ocp/env_model/veh3dof_tracking_model.py:11-102       */
  GOPS_MODEL_MOBILEROBOT = 4      /* env_ocp/env_model/pyth_mobilerobot_model.py:61-195: state == obs (13), 2 actions,
                                     one constraint, obstacle noise (gops_b200_plan_set_model_io)                 */
};

/* activations                      gops/utils/common_utils.py:26-55 ------------------------- */
enum {
  GOPS_ACT_RELU = 0, GOPS_ACT_ELU = 1, GOPS_ACT_GELU = 2, GOPS_ACT_SELU = 3,
  GOPS_ACT_SIGMOID = 4, GOPS_ACT_TANH = 5, GOPS_ACT_LINEAR = 6
};

/* One `mlp()` network with two hidden layers of equal width. */
typedef struct gops_b200_mlp_desc {
  int32_t in_dim;      /* observation features (without the time column)                          */
  int32_t time_input;  /* 1 = FiniteHorizonPolicy: a column virtual_t is appended (mlp.py:103-111) */
  int32_t hidden;      /* hidden width: 64 or 256 (two equal hidden layers)                           */
  int32_t out_dim;     /* act_dim for policies, 1 for StateValue                                   */
  int32_t hidden_act;  /* GOPS_ACT_*                                                               */
  int32_t out_act;     /* GOPS_ACT_* (reference default "linear")                                  */
} gops_b200_mlp_desc;

/* Reference-trajectory generator constants, env_ocp/resources/ref_traj_data.py:19-37.  Doubles: the
 * reference forms derived constants (e.g. -A/omega) as python floats before touching fp32 tensors. */
typedef struct gops_b200_reftraj {
  double sine_A, sine_omega, sine_phi;
  double dl_t1, dl_t2, dl_t3, dl_t4, dl_y1, dl_y2;
  double tri_A, tri_T;
  double circ_r;
  double sp_A, sp_omega, sp_phi, sp_b, sp_const;
} gops_b200_reftraj;

typedef struct gops_b200_plan_desc {
  int32_t alg;          /* GOPS_ALG_*                                                            */
  int32_t model;        /* GOPS_MODEL_*                                                          */
  int32_t horizon;      /* FHADP pre_horizon / INFADP forward_step                               */
  float gamma;
  gops_b200_mlp_desc policy;
  gops_b200_mlp_desc value;  /* INFADP only (v and v_target share the shape)                     */

  /* wrapper chain, gops/create_pkg/create_env_model.py:104-126 */
  int32_t action_scale;      /* ScaleActionModel   wrapper/scale_action.py:75-83                 */
  int32_t clip_action;       /* ClipActionModel    wrapper/clip_action.py:27-40                  */
  int32_t clip_obs;          /* ClipObservationModel wrapper/clip_observation.py:27-44           */
  int32_t mask_at_done;      /* MaskAtDoneModel    wrapper/mask_at_done.py:26-40                 */
  int32_t reward_shaping;    /* ShapingRewardModel wrapper/shaping_reward.py:77-88               */
  float reward_shift, reward_scale;
  int32_t obs_scaling;       /* ScaleObservationModel wrapper/scale_observation.py:104-116       */
  const float* obs_scale;    /* HOST arrays of obs_dim floats (copied at plan creation) or NULL   */
  const float* obs_shift;
  int32_t repeat_num;        /* ActionRepeatModel wrapper/action_repeat.py:71-87 (0 = absent);   */
  int32_t sum_reward;        /*   state==obs models only                                         */
  float min_action[GOPS_B200_MAX_ACT], max_action[GOPS_B200_MAX_ACT];
  float act_low[GOPS_B200_MAX_ACT], act_high[GOPS_B200_MAX_ACT];         /* model action bounds  */
  float pol_act_low[GOPS_B200_MAX_ACT], pol_act_high[GOPS_B200_MAX_ACT]; /* policy tanh limits   */
  float obs_low[GOPS_B200_MAX_LQ_N], obs_high[GOPS_B200_MAX_LQ_N];       /* state==obs models    */

  /* pyth_lq: x' = inv_IA (B u dt + x), r = rs*(rsh - (sum Q x^2 + sum R u^2))  lq_base.py:89-141 */
  int32_t lq_n, lq_m;
  float lq_inv_IA[GOPS_B200_MAX_LQ_N * GOPS_B200_MAX_LQ_N]; /* row-major n x n                   */
  float lq_B[GOPS_B200_MAX_LQ_N * GOPS_B200_MAX_ACT];       /* row-major n x m                   */
  float lq_Q[GOPS_B200_MAX_LQ_N], lq_R[GOPS_B200_MAX_ACT];
  float lq_dt, lq_reward_scale, lq_reward_shift;

  /* vehicle models */
  int32_t veh_pre_horizon;   /* P: obs_dim = 6 + 4 P                                             */
  gops_b200_reftraj reftraj;
  /* FHADP2 (gops/algorithm/fhadp2.py:98-121): open-loop policy.  1 = `policy` is a FiniteHorizonFullPolicy
   * (mlp.py:114-145): ONE evaluation on obs_0 emits all `horizon` actions, policy.out_dim = act_dim * horizon (<= 256),
   * no time input; alg must be GOPS_ALG_FHADP.  Runs on the layer-wise wgmma path. */
  int32_t open_loop;
  /* pyth_veh3dofconti_errcstr (env_ocp/env_model/pyth_veh3dofconti_errcstr_model.py:19-55): the vehicle model that also
   * returns info["constraint"] = (|y_err| - y_error_tol, |u_err| - u_error_tol) of the incoming observation. */
  int32_t veh_errcstr;
  float veh_y_error_tol, veh_u_error_tol;
  /* env_gen_ocp veh3dof_tracking_detour (1; env_gen_ocp/env_model/veh3dof_tracking_detour_model.py:13-176) or
   * veh3dof_tracking_surrcstr (2; veh3dof_tracking_surrcstr_model.py:13-181): model must be GOPS_MODEL_VEH3DOF_TRACKING;
   * obs_dim = 6 + 4 P + 4 (one surrounding vehicle), info["constraint"] = the bicircle collision constraint of the
   * incoming state.  FHADP and its constrained variants, on the layer-wise wgmma path. */
  int32_t veh_detour;
  float veh_length, veh_width;
} gops_b200_plan_desc;

/* Per-call inputs (one replay batch shard).  Unused pointers are NULL. */
typedef struct gops_b200_batch {
  int64_t batch;             /* samples on this device                                           */
  const float* obs;          /* [batch][obs_dim]   data["obs"]                                   */
  const float* done;         /* [batch]            data["done"] (float32, replay_buffer.py:103)   */
  const float* state;        /* [batch][6]         veh: info["state"] / State.robot_state        */
  const float* ref_points;   /* [batch][P+1][4]    veh3dofconti info["ref_points"]               */
  const float* path_num;     /* [batch]            float32 as stored by the replay buffer        */
  const float* u_num;        /* [batch]                                                           */
  const float* ref_time;     /* [batch]                                                           */
  const float* reference;    /* [batch][ref_len][4] veh3dof_tracking ContextState.reference      */
  int32_t ref_t;             /* veh3dof_tracking ContextState.t (shared python int)              */
  int32_t ref_len;           /* veh3dof_tracking: points per sample in `reference`               */
  const float* surr;         /* [batch][surr_len][1][5] veh3dof_tracking_detour ContextState.constraint (x, y, phi, u, delta) */
  int32_t surr_len;          /* predictions per sample in `surr` (>= ref_t + horizon + 1)        */
} gops_b200_batch;

typedef struct gops_b200_plan gops_b200_plan;

int gops_b200_version(void);
const char* gops_b200_last_error(void);
/* Number of CUDA kernels this library has launched in this process so far (all plans, all devices): bench.py reports
 * the difference over its timed region as `gpu_launches`. */
int64_t gops_b200_launch_count(void);

/* Plan = compiled shape/constant bundle + device scratch (weight staging blob, rollout tape,
 * per-CTA gradient partials). */
int gops_b200_plan_create(const gops_b200_plan_desc* desc, gops_b200_plan** out);
int gops_b200_plan_destroy(gops_b200_plan* plan);
/* Re-derive the discount table fp32(gamma ** k), k = 0..horizon, from the python double (the
 * reference multiplies fp32 rewards by the python float `gamma ** step`, fhadp.py:121). */
int gops_b200_plan_set_gamma(gops_b200_plan* plan, double gamma);
/* Measurement aids (bench.py): CUDA events recorded on the launch stream around the fused rollout
 * kernel only; last_kernel_ms synchronises on the stop event.  launch_info: grid, block, tile S,
 * dynamic shared memory bytes of the last rollout launch. */
int gops_b200_plan_enable_timing(gops_b200_plan* plan, int enable);
int gops_b200_plan_last_kernel_ms(gops_b200_plan* plan, float* ms);
int gops_b200_plan_launch_info(const gops_b200_plan* plan, int32_t* out4);
/* Kernel path of the fused rollout.  AUTO (default) picks per launch: wgmma (BF16x3) where the nets are
 * 64-wide with <= 16 inputs, the mma.sync (3xTF32) / FFMA kernels elsewhere.  A plan option instead of an environment
 * switch so that a test can state AND assert which kernel ran (the env var GOPS_B200_ROLLOUT=tc|mma still overrides
 * for A/B runs from the shell).  last_path: path of the most recent rollout launch of this plan (GOPS_PATH_*). */
#define GOPS_PATH_AUTO 0
#define GOPS_PATH_MMA 1
#define GOPS_PATH_TC 2
int gops_b200_plan_set_path(gops_b200_plan* plan, int path);
int gops_b200_plan_last_path(const gops_b200_plan* plan);
/* Constrained FHADP variants on a constraint-providing env model (plan_desc.veh_errcstr):
 *   mode 1  exterior penalty   loss = -mean(v_r) + coef * mean(sum_k g^k sum_i max(c_i, 0)^2)     fhadp_exterior.py:55-70
 *   mode 2  Lagrangian         loss = -mean(v_r) + coef * mean(sum_k g^k sum_i max(c_i, 0))       fhadp_lagrangian.py:59-71
 *   mode 3  interior point     loss = -mean(v_r) + mean(feasible * sum_k g^k sum_i log(-min(c_i,0) + 1e-8)) / coef
 *                                     + coef * mean(~feasible * sum_k g^k sum_i max(c_i,0)^2)     fhadp_interior.py:55-84
 * coef = penalty / multiplier of the CURRENT update (the algorithms anneal it on the host).  scalars_out of
 * rollout_grad then carries [0] total loss, [1] the exterior / linear constraint term (mean), [2] #done, [3] #feasible.
 *   mode 4  SPIL (gops/algorithm/spil.py) on the mma.sync kernel only (coef unused), on pyth_veh3dofconti_errcstr (two
 *           constraints of the incoming observation) and pyth_mobilerobot (one constraint of the raw next state, done
 *           samples included; scalars_out [3] is then 0 and w_c1 unused):
 *     INFADP_VALUE plan  spil.py:182-212: loss_v = mean((v(o) - R)^2), R = sum_k g^k r_k + g^n v_target(o_n) WITHOUT the
 *                        (~d) mask; scalars_out = [0] loss_v, [1] mean v(o), [2] / [3] number of trajectories whose
 *                        constraint 0 / 1 stayed <= 0 on every step (the safe counts the controller turns into safe_prob).
 *     FHADP plan         spil.py:214-255 (DetermPolicy, no terminal value): loss = -mean(w_r R + sum_i w_c,i prod_k
 *                        Phi(c_k,i)), Phi(y) = 1.07 / (1 + 0.0315 exp(clamp(y / 0.07, -10, 5))); [w_r, w_c0, w_c1] are
 *                        read from the device pointer of plan_set_spil_weights; scalars_out = [0] loss, [1] mean R,
 *                        [2] / [3] mean Phi product of constraint 0 / 1.
 * The wgmma and layer-wise rollout paths do not have mode 4: it is refused on plans that can take them. */
int gops_b200_plan_set_constraint(gops_b200_plan* plan, int mode, float coef);
/* SPIL policy pass: DEVICE pointer to float[3] = [w_r, w_c0, w_c1] (written by gops_b200_spil_controller), read by every
 * later rollout_grad of this plan.  The pointer must stay valid while the plan uses it. */
int gops_b200_plan_set_spil_weights(gops_b200_plan* plan, const float* weights);
/* Models with noise and constraints (GOPS_MODEL_MOBILEROBOT): DEVICE pointers read / written by later calls of this
 * plan, which must stay valid while the plan uses them.
 *   noise:          the model's standard-deviation-scaled draws float32(normal(0, (0.03, 0.02))) of the obstacle's (v, w),
 *                   [horizon][batch][2] for rollout_grad / rollout_trace, [batch][2] for model_step (required on this model)
 *   constraint_out: [batch][1] info["constraint"] of model_step (0.89 - obstacle distance of the raw next state), or NULL */
int gops_b200_plan_set_model_io(gops_b200_plan* plan, const float* noise, float* constraint_out);
/* SPIL's PI multiplier controller (spil.py:257-270), one launch on `stream`, no host sync.  tail: DEVICE float[4] scalars of
 * the value pass (after the gradient exchange, so slots 2 / 3 hold the global safe counts); batch_global: the global batch
 * size.  safe_prob = float32(count) / float32(batch); state: DEVICE double[6] = [delta_i(2), safe_prob_pre(2), lam(2)],
 * updated in place; weights: DEVICE float[3] = [w_r, w_c0, w_c1] = float32 of 1 / (1 + sum lam), lam / (1 + sum lam). */
int gops_b200_spil_controller(const float* tail, int64_t batch_global, double kp, double ki, double kd,
                              double chance_thre0, double chance_thre1, double* state, float* weights, void* stream);
/* number of float32 parameters of the policy (which=0) / value (which=1) network */
int64_t gops_b200_plan_param_count(const gops_b200_plan* plan, int which);

/*
 * Fused rollout + loss + gradient.  Replaces, per call:
 *   FHADP._compute_gradient        fhadp.py:104-111   (alg = GOPS_ALG_FHADP; grads of policy)
 *   INFADP.__compute_gradient      infadp.py:135-157  (policy branch / value branch)
 * including policy/value forward (mlp.py), the wrapper chain and envmodel.forward.
 *   policy_params / value_params / vtarget_params: flat fp32 parameter vectors (see top).
 *   inv_batch_global: 1 / B_global (so multi-GPU shards sum to the global mean).
 *   grad_out: flat gradient of the network being updated (policy for FHADP/INFADP_POLICY,
 *             value for INFADP_VALUE), overwritten.
 *   scalars_out[4]: [0] loss (already scaled by inv_batch_global, summed over this shard),
 *                   [1] sum_b v(o_b) * inv_batch_global (INFADP_VALUE: critic avg value),
 *                   [2] number of samples done at the end of the rollout, [3] reserved.
 */
int gops_b200_rollout_grad(gops_b200_plan* plan, const gops_b200_batch* batch,
                           const float* policy_params, const float* value_params,
                           const float* vtarget_params, float inv_batch_global,
                           float* grad_out, float* scalars_out, void* stream);

/* torch.optim.Adam (no weight decay, no amsgrad) over a flat vector; `step` is 1-based.
 * Replaces policy_optimizer.step() fhadp.py:89 / optimizer_dict[..].step() infadp.py:123-124. */
int gops_b200_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                        int64_t n, int32_t step, double lr, double beta1, double beta2, double eps,
                        void* stream);

/* p_targ = (1 - tau) * p_targ + tau * p          infadp.py:126-133 */
int gops_b200_polyak(float* target, const float* src, float tau, int64_t n, void* stream);

/* Batched policy inference: act_out[b] = policy(obs[b], virtual_t).  Replaces
 * DetermPolicy.forward mlp.py:73-77 / FiniteHorizonPolicy.forward mlp.py:103-111. */
int gops_b200_policy_forward(gops_b200_plan* plan, const float* policy_params, const float* obs,
                             int64_t batch, float virtual_t, float* act_out, void* stream);

/* Batched state-value inference (StateValue.forward mlp.py:327-329). */
int gops_b200_value_forward(gops_b200_plan* plan, const float* value_params, const float* obs,
                            int64_t batch, float* v_out, void* stream);

/* Plan-free batched MLP inference.  act_low/act_high are HOST pointers (out_dim floats) holding the
 * policy's act_{low,high}_lim buffers; pass NULL for a raw (StateValue) output. */
int gops_b200_mlp_forward(const gops_b200_mlp_desc* net, const float* params, const float* obs,
                          int64_t batch, float virtual_t, const float* act_low, const float* act_high,
                          float* out, void* stream);

/* One step of the wrapped env model with explicit actions: replaces envmodel.forward(obs, action,
 * done, info) of the chain built by create_env_model.py:104-126.  `action` is [batch][act_dim] in
 * the policy's (scaled) action space.  next_state / next_ref_points / next_ref_time receive the
 * advanced `info` entries of the vehicle models (may be NULL for the other models). */
int gops_b200_model_step(gops_b200_plan* plan, const gops_b200_batch* batch, const float* action,
                         float* next_obs, float* reward, float* next_done, float* next_state,
                         float* next_ref_points, float* next_ref_time, void* stream);

/* Debug / parity aid: run the no-grad rollout and dump per-step tensors
 * obs_out[H][batch][obs_dim], act_out[H][batch][act_dim] (policy output), rew_out[H][batch],
 * done_out[H][batch] (as float).  Any output pointer may be NULL. */
int gops_b200_rollout_trace(gops_b200_plan* plan, const gops_b200_batch* batch,
                            const float* policy_params, float* obs_out, float* act_out,
                            float* rew_out, float* done_out, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Layer-wise MLP on the tensor cores (wgmma, BF16x3): a trainable `mlp()` network of 1..8 Linear layers with
 * widths <= 256, one hidden activation and a linear output -- reference gops/apprfunc/mlp.py:36-41 evaluated and
 * differentiated layer by layer.  It is the path of the networks the fused rollout kernels do not cover:
 * [256,256] policies (FHADP veh3dof_tracking), the [256,256,256] nets of DSAC (mlp.py:149-221, 271-296) and the
 * open-loop FiniteHorizonFullPolicy of FHADP2 (mlp.py:114-145).
 *   params: flat fp32 vector in torch parameters() order (W0, b0, W1, b1, ...), as everywhere in this header.
 *   pack:   split the weights into bf16 planes once per parameter update (forward and transposed images).
 *   forward(slot, train): y = net(x); with train != 0 the hidden activations and their derivatives are kept in `slot`
 *           (x itself is NOT copied: it must stay valid until the matching backward).
 *   backward(slot): given dL/dy of that forward pass, overwrite or accumulate the flat gradient (grad_flat may be NULL)
 *           and / or write dL/dx (dx may be NULL).  Deterministic (fixed-order reductions).
 */
typedef struct gops_b200_mlpnet gops_b200_mlpnet;
int gops_b200_mlpnet_create(const int32_t* sizes, int32_t n_sizes, int32_t hidden_act, int64_t max_batch,
                            int32_t slots, gops_b200_mlpnet** out);
int gops_b200_mlpnet_destroy(gops_b200_mlpnet* net);
int64_t gops_b200_mlpnet_param_count(const gops_b200_mlpnet* net);
int gops_b200_mlpnet_pack(gops_b200_mlpnet* net, const float* params, void* stream);
int gops_b200_mlpnet_forward(gops_b200_mlpnet* net, const float* x, int32_t ldx, int64_t batch, int32_t slot,
                             int32_t train, float* y, int32_t ldy, void* stream);
int gops_b200_mlpnet_backward(gops_b200_mlpnet* net, const float* dy, int32_t lddy, int64_t batch, int32_t slot,
                              float* grad_flat, int32_t accumulate, float* dx, int32_t lddx, void* stream);
/* Rollouts (one forward / backward pass per horizon step, one slot per step): keep_deltas(1) makes every backward pass
 * (called with grad_flat = NULL) leave its per-layer deltas in its slot; wgrad_slots then contracts the weight
 * gradients over all `nslots` passes at once (x / dy: input and output adjoint of slot0; slot s of them starts
 * x_stride / dy_stride rows further). */
/* Paired passes (twin critics): two handles created with identical sizes, activation, max_batch and slots, both packed,
 * evaluated on ONE shared input x.  Every forward GEMM, dgrad GEMM, weight-gradient contraction, column sum and
 * reduction runs both networks in one launch (blockIdx.z selects the network), so a pair issues as many launches as one
 * single-network pass.  Per network the arithmetic is that of mlpnet_forward / mlpnet_backward (same tiles, same
 * reduction order: bit-identical results); each network keeps its own activations in `slot`.  y_a / y_b share ldy,
 * dy_a / dy_b share lddy, dx_a / dx_b share lddx; grad_a / grad_b and dx_a / dx_b are both set or both NULL.  A
 * mismatched pair returns an error. */
int gops_b200_mlpnet_pair_forward(gops_b200_mlpnet* net_a, gops_b200_mlpnet* net_b, const float* x, int32_t ldx,
                                  int64_t batch, int32_t slot, int32_t train, float* y_a, float* y_b, int32_t ldy,
                                  void* stream);
int gops_b200_mlpnet_pair_backward(gops_b200_mlpnet* net_a, gops_b200_mlpnet* net_b, const float* dy_a, const float* dy_b,
                                   int32_t lddy, int64_t batch, int32_t slot, float* grad_a, float* grad_b,
                                   int32_t accumulate, float* dx_a, float* dx_b, int32_t lddx, void* stream);
int gops_b200_mlpnet_keep_deltas(gops_b200_mlpnet* net, int32_t enable);
int gops_b200_mlpnet_wgrad_slots(gops_b200_mlpnet* net, int32_t slot0, int32_t nslots, int64_t batch, const float* x,
                                 int32_t ldx, int64_t x_stride, const float* dy, int32_t lddy, int64_t dy_stride,
                                 float* grad_flat, int32_t accumulate, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * DSAC (gops/algorithm/dsac.py:155-290): the elementwise half of the update, each with its hand-derived gradient.
 * The network evaluations between them are gops_b200_mlpnet_* calls.  Device pointers, asynchronous on `stream`.
 *
 * sample:   StochaPolicy head (mlp.py:203-221, "mlp_shared") + TanhGaussDistribution.rsample
 *           (act_distribution_type.py:37-50).  logits [B][2A] raw policy-net outputs (mean | log_std), eps [B][A]
 *           standard-normal noise.  act [B][A], logp [B].  If qin != NULL the critic input row [obs | act] is written
 *           (ldq floats per row).  stats (optional, [2B]): tanh(mean_0) and std_0 per sample (tb scalars).
 * sample_backward: d loss / d logits given d loss / d act (columns act_col0.. of a [B][ldda] matrix, e.g. the
 *           critic's input gradient) and the coefficient of sum_b logp_b in the loss.
 * q_loss:   dsac.py:219-262 (clipped TD target, bound / unbound form): gradient w.r.t. the critic output [B][2] and
 *           out3 = {loss, mean q, mean q_std}.  z_next: standard-normal noise of the target critic sample.
 * policy_loss: dsac.py:264-275: out5 = {loss, entropy, mean(logp + target_entropy), mean tanh(mean_0), mean std_0}. */
int gops_b200_dsac_sample(const float* logits, const float* eps, int64_t batch, int32_t act_dim, float min_log_std,
                          float max_log_std, const float* act_half, const float* act_mid, float* act, float* logp,
                          const float* obs, int32_t obs_dim, float* qin, int32_t ldq, float* stats, void* stream);
int gops_b200_dsac_sample_backward(const float* logits, const float* eps, int64_t batch, int32_t act_dim,
                                   float min_log_std, float max_log_std, const float* act_half, const float* d_act,
                                   int32_t ldda, int32_t act_col0, float logp_coeff, float* d_logits, void* stream);
int gops_b200_dsac_q_loss(const float* q_out, const float* q_next_out, const float* z_next, const float* logp_next,
                          const float* rew, const float* done, int64_t batch, float gamma, float alpha, int32_t bound,
                          float* d_q_out, float* out3, void* stream);
int gops_b200_dsac_policy_loss(const float* q_out, const float* logp_new, int64_t batch, float alpha,
                               float target_entropy, float* d_q_out, float* out5, const float* stats, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * DSAC-T (gops/algorithm/dsact.py:162-329): the elementwise half of the twin-critic update.  The critic evaluations
 * between them are gops_b200_mlpnet_pair_* calls; action sampling is gops_b200_dsac_sample.
 *
 * q_loss:   dsact.py:229-313.  q1_out / q2_out: critic outputs [B][2] (mean | raw std) at (obs, act); q1_next_out /
 *           q2_next_out: target-critic outputs at (obs2, act2); z1_next / z2_next: standard-normal noise of the two
 *           target samples.  mean_std: DEVICE float[2], the running means of the critics' std, updated in place
 *           ((1 - tau_b) m + tau_b mean(std), or seeded with mean(std) where bit i of mean_std_unset is set) before the
 *           loss uses them.  Writes d loss / d (mean, raw std) of both critics and out9 = {loss_q, mean q1, mean q2, mean std1,
 *           mean std2, min std1, min std2, mean_std1, mean_std2}.
 * policy_loss: dsact.py:315-329 on the critic outputs at (obs, new_act): mean(alpha logp - min(q1, q2)).  d_q1_out /
 *           d_q2_out get -1/B on the mean of the smaller critic (half each on a tie), zero elsewhere; out5 as
 *           gops_b200_dsac_policy_loss.
 * sample_backward: gops_b200_dsac_sample_backward with d loss / d act = d_act_1 + d_act_2 (the two critics' input
 *           gradients, same ldda). */
int gops_b200_dsact_q_loss(const float* q1_out, const float* q2_out, const float* q1_next_out, const float* q2_next_out,
                           const float* z1_next, const float* z2_next, const float* logp_next, const float* rew,
                           const float* done, int64_t batch, float gamma, float alpha, double tau_b, float* mean_std,
                           int32_t mean_std_unset, float* d_q1_out, float* d_q2_out, float* out9, void* stream);
int gops_b200_dsact_policy_loss(const float* q1_out, const float* q2_out, const float* logp_new, int64_t batch,
                                float alpha, float target_entropy, float* d_q1_out, float* d_q2_out, float* out5,
                                const float* stats, void* stream);
int gops_b200_dsact_sample_backward(const float* logits, const float* eps, int64_t batch, int32_t act_dim,
                                    float min_log_std, float max_log_std, const float* act_half, const float* d_act_1,
                                    const float* d_act_2, int32_t ldda, int32_t act_col0, float logp_coeff,
                                    float* d_logits, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * SAC (gops/algorithm/sac.py:159-241): every loss of one update in one launch, after three paired forwards of the
 * twin ActionValue critics ([B] outputs each) with the pre-update weights: q1_out / q2_out at (obs, act), q1_new_out /
 * q2_new_out at (obs, new_act), q1_next_out / q2_next_out (target critics) at (obs2, next_act).
 *   y = rew + (1 - done) gamma (min(q1', q2') - alpha logp_next);  d_q{1,2}_out = 2 (q_i - y) / B
 *   actor mean(alpha logp_new - min(q1, q2)) at new_act: d_q{1,2}_new_out = -1/B to the smaller critic, -1/(2B) to
 *   each on a tie, 0 to the other
 *   out6 = {loss_q1 + loss_q2, mean q1, mean q2, actor loss, entropy -mean(logp_new),
 *           d loss_alpha / d log_alpha = -mean(logp_new + target_entropy)}
 * The action gradient through both critics is gops_b200_dsact_sample_backward with logp_coeff alpha / B. */
int gops_b200_sac_losses(const float* q1_out, const float* q2_out, const float* q1_new_out, const float* q2_new_out,
                         const float* q1_next_out, const float* q2_next_out, const float* logp_new,
                         const float* logp_next, const float* rew, const float* done, int64_t batch, float gamma,
                         float alpha, float target_entropy, float* d_q1_out, float* d_q2_out, float* d_q1_new_out,
                         float* d_q2_new_out, float* out6, void* stream);

/* ---- data-parallel gradient exchange over NVLink peer memory, fused with Adam (peer.cu) ---------------------------
 * Replaces the gradient hand-over between replicas of the reference's synchronous trainer
 * (gops/trainer/off_sync_trainer.py:97-120: workers' get_remote_update_info -> remote_update with the averaged
 * gradient) and the optimizer step behind it (fhadp.py:89, infadp.py:123-124): ONE kernel per rank pushes its flat
 * [gradient | loss | ...] vector into every peer's exchange region, waits for the peers' sequence flags, sums in rank
 * order (bit-identical on all ranks) and applies Adam.  One object per rank; regions are shared with cudaIpc handles
 * (one process per GPU: _export on every rank, exchange the 64-byte handles, _connect) or wired directly when the
 * ranks live in one process (_local_base / _connect_local).  All ranks must issue the same sequence of calls. */
#define GOPS_B200_IPC_HANDLE_BYTES 64
typedef struct gops_b200_peer gops_b200_peer;
int gops_b200_peer_create(int32_t world, int32_t rank, int64_t max_floats, gops_b200_peer** out);
int gops_b200_peer_destroy(gops_b200_peer* peer);
int gops_b200_peer_region_bytes(const gops_b200_peer* peer, int64_t* bytes);
int gops_b200_peer_export(gops_b200_peer* peer, void* handle64);
int gops_b200_peer_connect(gops_b200_peer* peer, const void* handles /* world x 64 bytes, rank order */);
int gops_b200_peer_local_base(gops_b200_peer* peer, void** base);
int gops_b200_peer_connect_local(gops_b200_peer* peer, void* const* bases /* world pointers, rank order */);
/* buf[0..n) <- sum over ranks (in place).  params != NULL: Adam over the first nparam entries with the summed gradient,
 * arguments as gops_b200_adam_step.  A peer that does not arrive within 60 s poisons buf with NaN and sets _error. */
int gops_b200_peer_allreduce(gops_b200_peer* peer, float* buf, int64_t n, float* params, float* exp_avg,
                             float* exp_avg_sq, int64_t nparam, int32_t step, double lr, double beta1, double beta2,
                             double eps, void* stream);
int gops_b200_peer_error(gops_b200_peer* peer, int32_t* err);

/* RPI (relaxed policy iteration, gops/algorithm/rpi.py) on pyth_oscillatorconti with a StateValue MLP [2 -> 64 -> 64 -> 1]
 * (hidden activation act: relu / elu / gelu / selu / sigmoid / tanh).  Parameter vectors are the value net's flat
 * parameters (4417 floats).  gamma_atte: the H-infinity attenuation of the model (the wrapped action bounds are
 * [-5, 5] and [-1/gamma_atte, 1/gamma_atte]).
 *
 * ApproxContainer.action_and_adversary (rpi.py:90-103) and the model's best_act / worst_adv
 * (pyth_oscillatorconti_model.py:772-815): act_out[b] = raw (a, w) = (-0.5 x0 p1, 0.5 / gamma_atte^2 x1 p1), p = dV/dx of
 * the target net at obs[b]; any batch. */
int gops_b200_rpi_policy(const float* target_params, int32_t act, double gamma_atte, const float* obs, int64_t batch,
                         float* act_out, void* stream);
/* RPI.__compute_loss / __calculate_hamiltonian (rpi.py:218-287) once: loss = mean_b |c + dV/dx . f| of the wrapped model
 * at (obs[b], act_in[b] = raw (a, w)); grad_out[4417] = d loss / d params, loss_out[1].  batch: a multiple of 64;
 * scratch: gops_b200_rpi_scratch_floats(batch) floats. */
int gops_b200_rpi_loss_grad(const float* params, int32_t act, double gamma_atte, const float* obs, const float* act_in,
                            int64_t batch, float* scratch, float* grad_out, float* loss_out, void* stream);
int64_t gops_b200_rpi_scratch_floats(int64_t batch);
/* One Newton iteration, RPI.local_update (rpi.py:174-215) with RPI.sample (:289-327), in ONE launch of a thread-block
 * cluster of batch / 64 CTAs (batch a multiple of 64, at most 512; threshold0/1: the model's state_threshold): H_before at set_state, then per inner step sample,
 * loss and gradient, cluster reduction, Adam (arguments as gops_b200_adam_step, steps step0 + 1, step0 + 2, ...) and
 * H_after, until H_after <= 0.88 H_before or max_steps steps; then target <- params.
 *   state [batch][2] sampler states, counter [1] the model's step_per_episode, both updated; max_step [batch];
 *   draws [rows][batch][2] reset() draws: row 0 is set_state, row n the reset draw of inner step n;
 *   out [8]: [0] steps n, [1] loss of the last step, [2] H_before, [3] H_after, [4] 1 if the loop stopped because the
 *   draws ran out; trace: NULL or [max_steps][2] (loss, H_after) per inner step. */
int gops_b200_rpi_newton(float* params, float* target, float* exp_avg, float* exp_avg_sq, int64_t step0, double lr,
                         double beta1, double beta2, double eps, int32_t act, double gamma_atte, double threshold0, double threshold1,
                         float* state, const int32_t* max_step, int32_t* counter, const float* draws, int32_t rows,
                         int32_t max_steps, int64_t batch, float* out, float* trace, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GOPS_B200_H */
