"""ctypes binding of libgops_b200.so (C ABI in include/gops_b200.h).

There is no CPU fallback: if the shared library is missing or a call fails, a RuntimeError is
raised.  Build it with `python -c "import __graft_entry__ as g; g.build()"` (nvcc, sm_90a).
"""
import ctypes as C
import os

MAX_ACT = 4
MAX_LQ_N = 8

ALG_FHADP, ALG_INFADP_POLICY, ALG_INFADP_VALUE = 0, 1, 2
MODEL_IDPENDULUM, MODEL_LQ, MODEL_VEH3DOFCONTI, MODEL_VEH3DOF_TRACKING, MODEL_MOBILEROBOT = 0, 1, 2, 3, 4
PATH_AUTO, PATH_MMA, PATH_TC = 0, 1, 2
PATH_NAMES = {0: "none", 1: "mma", 2: "tc"}
ACT_IDS = {"relu": 0, "elu": 1, "gelu": 2, "selu": 3, "sigmoid": 4, "tanh": 5, "linear": 6}

LIB_PATH = os.environ.get("GOPS_B200_LIB") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libgops_b200.so")   # override: A/B runs of two builds


class MlpDesc(C.Structure):
    _fields_ = [("in_dim", C.c_int32), ("time_input", C.c_int32), ("hidden", C.c_int32),
                ("out_dim", C.c_int32), ("hidden_act", C.c_int32), ("out_act", C.c_int32)]


class RefTraj(C.Structure):
    _fields_ = [(n, C.c_double) for n in (
        "sine_A", "sine_omega", "sine_phi", "dl_t1", "dl_t2", "dl_t3", "dl_t4", "dl_y1", "dl_y2",
        "tri_A", "tri_T", "circ_r", "sp_A", "sp_omega", "sp_phi", "sp_b", "sp_const")]


class PlanDesc(C.Structure):
    _fields_ = [
        ("alg", C.c_int32), ("model", C.c_int32), ("horizon", C.c_int32), ("gamma", C.c_float),
        ("policy", MlpDesc), ("value", MlpDesc),
        ("action_scale", C.c_int32), ("clip_action", C.c_int32), ("clip_obs", C.c_int32),
        ("mask_at_done", C.c_int32), ("reward_shaping", C.c_int32),
        ("reward_shift", C.c_float), ("reward_scale", C.c_float),
        ("obs_scaling", C.c_int32), ("obs_scale", C.POINTER(C.c_float)), ("obs_shift", C.POINTER(C.c_float)),
        ("repeat_num", C.c_int32), ("sum_reward", C.c_int32),
        ("min_action", C.c_float * MAX_ACT), ("max_action", C.c_float * MAX_ACT),
        ("act_low", C.c_float * MAX_ACT), ("act_high", C.c_float * MAX_ACT),
        ("pol_act_low", C.c_float * MAX_ACT), ("pol_act_high", C.c_float * MAX_ACT),
        ("obs_low", C.c_float * MAX_LQ_N), ("obs_high", C.c_float * MAX_LQ_N),
        ("lq_n", C.c_int32), ("lq_m", C.c_int32),
        ("lq_inv_IA", C.c_float * (MAX_LQ_N * MAX_LQ_N)), ("lq_B", C.c_float * (MAX_LQ_N * MAX_ACT)),
        ("lq_Q", C.c_float * MAX_LQ_N), ("lq_R", C.c_float * MAX_ACT),
        ("lq_dt", C.c_float), ("lq_reward_scale", C.c_float), ("lq_reward_shift", C.c_float),
        ("veh_pre_horizon", C.c_int32), ("reftraj", RefTraj),
        ("open_loop", C.c_int32),
        ("veh_errcstr", C.c_int32), ("veh_y_error_tol", C.c_float), ("veh_u_error_tol", C.c_float),
        ("veh_detour", C.c_int32), ("veh_length", C.c_float), ("veh_width", C.c_float),
    ]


class Batch(C.Structure):
    _fields_ = [("batch", C.c_int64), ("obs", C.c_void_p), ("done", C.c_void_p), ("state", C.c_void_p),
                ("ref_points", C.c_void_p), ("path_num", C.c_void_p), ("u_num", C.c_void_p),
                ("ref_time", C.c_void_p), ("reference", C.c_void_p), ("ref_t", C.c_int32), ("ref_len", C.c_int32),
                ("surr", C.c_void_p), ("surr_len", C.c_int32)]


# name -> (restype, argtypes); the parity test `test_abi_symbols` checks these against the header
PROTOTYPES = {
    "gops_b200_version": (C.c_int, []),
    "gops_b200_last_error": (C.c_char_p, []),
    "gops_b200_launch_count": (C.c_int64, []),
    "gops_b200_plan_create": (C.c_int, [C.POINTER(PlanDesc), C.POINTER(C.c_void_p)]),
    "gops_b200_plan_destroy": (C.c_int, [C.c_void_p]),
    "gops_b200_plan_set_gamma": (C.c_int, [C.c_void_p, C.c_double]),
    "gops_b200_plan_enable_timing": (C.c_int, [C.c_void_p, C.c_int]),
    "gops_b200_plan_last_kernel_ms": (C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
    "gops_b200_plan_launch_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "gops_b200_plan_set_path": (C.c_int, [C.c_void_p, C.c_int]),
    "gops_b200_plan_last_path": (C.c_int, [C.c_void_p]),
    "gops_b200_plan_set_constraint": (C.c_int, [C.c_void_p, C.c_int, C.c_float]),
    "gops_b200_plan_set_spil_weights": (C.c_int, [C.c_void_p, C.c_void_p]),
    "gops_b200_plan_set_model_io": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_spil_controller": (C.c_int, [C.c_void_p, C.c_int64, C.c_double, C.c_double, C.c_double, C.c_double,
                                            C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_plan_param_count": (C.c_int64, [C.c_void_p, C.c_int]),
    "gops_b200_rollout_grad": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_adam_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                      C.c_double, C.c_double, C.c_double, C.c_double, C.c_void_p]),
    "gops_b200_polyak": (C.c_int, [C.c_void_p, C.c_void_p, C.c_float, C.c_int64, C.c_void_p]),
    "gops_b200_policy_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float,
                                           C.c_void_p, C.c_void_p]),
    "gops_b200_value_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "gops_b200_mlp_forward": (C.c_int, [C.POINTER(MlpDesc), C.c_void_p, C.c_void_p, C.c_int64, C.c_float,
                                        C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p, C.c_void_p]),
    "gops_b200_rollout_trace": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_model_step": (C.c_int, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_mlpnet_create": (C.c_int, [C.POINTER(C.c_int32), C.c_int32, C.c_int32, C.c_int64, C.c_int32,
                                          C.POINTER(C.c_void_p)]),
    "gops_b200_mlpnet_destroy": (C.c_int, [C.c_void_p]),
    "gops_b200_mlpnet_param_count": (C.c_int64, [C.c_void_p]),
    "gops_b200_mlpnet_pack": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_mlpnet_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_int32,
                                           C.c_void_p, C.c_int32, C.c_void_p]),
    "gops_b200_mlpnet_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_void_p,
                                            C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "gops_b200_mlpnet_pair_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_int32,
                                                C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "gops_b200_mlpnet_pair_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64,
                                                 C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                                 C.c_int32, C.c_void_p]),
    "gops_b200_mlpnet_keep_deltas": (C.c_int, [C.c_void_p, C.c_int32]),
    "gops_b200_mlpnet_wgrad_slots": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_int32,
                                               C.c_int64, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_int32,
                                               C.c_void_p]),
    "gops_b200_dsac_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_float, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                        C.c_void_p, C.c_void_p]),
    "gops_b200_dsac_sample_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_float,
                                                 C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_void_p,
                                                 C.c_void_p]),
    "gops_b200_dsac_q_loss": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int64, C.c_float, C.c_float, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_dsac_policy_loss": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_dsact_q_loss": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float, C.c_double,
                                         C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_dsact_policy_loss": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_dsact_sample_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_float, C.c_float,
                                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_float,
                                                  C.c_void_p, C.c_void_p]),
    "gops_b200_sac_losses": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_float,
                                       C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    "gops_b200_peer_create": (C.c_int, [C.c_int32, C.c_int32, C.c_int64, C.POINTER(C.c_void_p)]),
    "gops_b200_peer_destroy": (C.c_int, [C.c_void_p]),
    "gops_b200_peer_region_bytes": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64)]),
    "gops_b200_peer_export": (C.c_int, [C.c_void_p, C.c_void_p]),
    "gops_b200_peer_connect": (C.c_int, [C.c_void_p, C.c_void_p]),
    "gops_b200_peer_local_base": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "gops_b200_peer_connect_local": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "gops_b200_peer_allreduce": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                           C.c_int32, C.c_double, C.c_double, C.c_double, C.c_double, C.c_void_p]),
    "gops_b200_peer_error": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "gops_b200_rpi_policy": (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "gops_b200_rpi_loss_grad": (C.c_int, [C.c_void_p, C.c_int32, C.c_double, C.c_void_p, C.c_void_p, C.c_int64,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "gops_b200_rpi_scratch_floats": (C.c_int64, [C.c_int64]),
    "gops_b200_rpi_newton": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_double, C.c_double,
                                       C.c_double, C.c_double, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
}

_lib = None


def lib():
    """Load the shared library once; raise loudly if it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"gops_b200: native library not found at {LIB_PATH}; build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(handle, name)      # AttributeError if the .so is stale
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


def check(rc):
    if rc != 0:
        raise RuntimeError("gops_b200: " + lib().gops_b200_last_error().decode())


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
