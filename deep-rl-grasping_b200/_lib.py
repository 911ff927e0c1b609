"""ctypes binding of libb200grasp.so (the C ABI in include/b200grasp.h).

The product path has NO CPU fallback: if the shared library is missing this raises, and if it
loads on a machine without an sm_90 (Hopper) GPU ``b2g_sac_create`` fails with B2G_ECUDA.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200grasp.so")

B2G_PREC_FP32_SIMT, B2G_PREC_BF16X3, B2G_PREC_BF16 = 0, 1, 2
B2G_EINVAL, B2G_ECUDA, B2G_ESTATE = -1, -2, -3

#: every symbol include/b200grasp.h declares (tests check the .so exports each of them)
SYMBOLS = [
    "b2g_last_error", "b2g_version", "b2g_nccl_unique_id", "b2g_sac_create", "b2g_sac_destroy", "b2g_sac_dp_export", "b2g_sac_dp_connect", "b2g_debug_dp_stamps", "b2g_debug_compact_host", "b2g_sync",
    "b2g_sac_create2", "b2g_sac_create3", "b2g_param_count", "b2g_param_info", "b2g_get_param", "b2g_set_param", "b2g_get_grad", "b2g_get_adam",
    "b2g_reset_optimizer", "b2g_replay_add", "b2g_replay_size", "b2g_replay_get", "b2g_replay_info", "b2g_get_last_batch", "b2g_set_norm_stats", "b2g_sac_step",
    "b2g_sac_step_async", "b2g_sac_step_explicit", "b2g_sac_step_host_pipelined", "b2g_sac_pipeline_flush", "b2g_sac_act", "b2g_launches_per_step", "b2g_last_step_ms",
    "b2g_profile_step", "b2g_sac_state_save", "b2g_sac_state_load",
    "b2g_sac_observe_act", "b2g_sac_observe_add", "b2g_obs_rms_set", "b2g_obs_rms_get", "b2g_upload_bytes",
    "b2g_bdq_create", "b2g_bdq_destroy", "b2g_bdq_param_count", "b2g_bdq_param_info", "b2g_bdq_get_param", "b2g_bdq_set_param",
    "b2g_bdq_get_grad", "b2g_bdq_replay_add", "b2g_bdq_replay_size", "b2g_bdq_set_norm_stats", "b2g_bdq_step",
    "b2g_bdq_step_explicit", "b2g_bdq_act", "b2g_bdq_set_per_beta", "b2g_bdq_get_last_per", "b2g_bdq_state_save", "b2g_bdq_state_load",
    "b2g_bdq_observe_act", "b2g_bdq_observe_add", "b2g_bdq_obs_rms_set", "b2g_bdq_obs_rms_get", "b2g_bdq_upload_bytes",
    "b2g_bdq_create2", "b2g_bdq_replay_info", "b2g_bdq_replay_get", "b2g_dqn_create2", "b2g_dqn_replay_info", "b2g_dqn_replay_get",
    "b2g_transition_replay_bytes",
    "b2g_dqn_create", "b2g_dqn_destroy", "b2g_dqn_param_count", "b2g_dqn_param_info", "b2g_dqn_get_param", "b2g_dqn_set_param",
    "b2g_dqn_get_grad", "b2g_dqn_replay_add", "b2g_dqn_replay_size", "b2g_dqn_set_norm_stats", "b2g_dqn_step",
    "b2g_dqn_step_explicit", "b2g_dqn_set_per_beta", "b2g_dqn_get_last_per", "b2g_dqn_update_target", "b2g_dqn_act",
    "b2g_dqn_state_save", "b2g_dqn_state_load",
    "b2g_dqn_observe_act", "b2g_dqn_observe_add", "b2g_dqn_act_raw", "b2g_dqn_obs_rms_set", "b2g_dqn_obs_rms_get",
    "b2g_dqn_upload_bytes", "b2g_dqn_set_obs_encoder",
    "b2g_ppo_create", "b2g_ppo_destroy", "b2g_ppo_param_count", "b2g_ppo_param_info", "b2g_ppo_get_param", "b2g_ppo_set_param",
    "b2g_ppo_get_grad", "b2g_ppo_rollout_act", "b2g_ppo_rollout_reward", "b2g_ppo_rollout_reset", "b2g_ppo_rollout_get",
    "b2g_ppo_update", "b2g_ppo_train_step_explicit", "b2g_ppo_act", "b2g_ppo_get_step", "b2g_ppo_state_save", "b2g_ppo_state_load",
    "b2g_trpo_create", "b2g_trpo_destroy", "b2g_trpo_param_count", "b2g_trpo_param_info", "b2g_trpo_get_param", "b2g_trpo_set_param",
    "b2g_trpo_get_grad", "b2g_trpo_rollout_act", "b2g_trpo_rollout_reward", "b2g_trpo_rollout_reset", "b2g_trpo_rollout_get",
    "b2g_trpo_update", "b2g_trpo_fvp", "b2g_trpo_step_explicit", "b2g_trpo_act", "b2g_trpo_get_step", "b2g_trpo_state_save",
    "b2g_trpo_state_load",
    "b2g_ppo_obs_rms_set", "b2g_ppo_obs_rms_get", "b2g_ppo_upload_bytes", "b2g_ppo_set_norm_stats", "b2g_ppo_set_obs_encoder",
    "b2g_ppo_observe_act", "b2g_ppo_act_raw", "b2g_trpo_obs_rms_set", "b2g_trpo_obs_rms_get", "b2g_trpo_upload_bytes",
    "b2g_trpo_set_norm_stats", "b2g_trpo_set_obs_encoder", "b2g_trpo_observe_act", "b2g_trpo_act_raw",
    "b2g_encoder_create", "b2g_encoder_destroy", "b2g_encoder_n_layers", "b2g_encoder_layer_shape", "b2g_encoder_set_weights",
    "b2g_encoder_encode", "b2g_encoder_create2", "b2g_debug_encoder_layers", "b2g_sac_set_obs_encoder", "b2g_bdq_set_obs_encoder", "b2g_debug_gemm", "b2g_debug_tensor_info", "b2g_debug_tensor", "b2g_debug_gg_simt", "b2g_debug_gg_tc",
    "b2g_debug_ppo_tensor_info", "b2g_debug_ppo_tensor", "b2g_debug_trpo_tensor_info", "b2g_debug_trpo_tensor",
    "b2g_debug_trpo_cg",
    "b2g_autoencoder_create", "b2g_autoencoder_destroy", "b2g_autoencoder_n_layers", "b2g_autoencoder_layer_shape",
    "b2g_autoencoder_set_weights", "b2g_autoencoder_get_weights", "b2g_autoencoder_get_grad", "b2g_autoencoder_reset_optimizer",
    "b2g_autoencoder_set_dataset", "b2g_autoencoder_train_epoch", "b2g_autoencoder_evaluate", "b2g_autoencoder_predict",
    "b2g_autoencoder_step", "b2g_autoencoder_create2", "b2g_debug_autoencoder_tensor", "b2g_debug_autoencoder_tensor_numel",
    "b2g_sac_metrics_log", "b2g_sac_metrics_drain", "b2g_bdq_metrics_log", "b2g_bdq_metrics_drain",
    "b2g_dqn_metrics_log", "b2g_dqn_metrics_drain",
]

#: columns of one per-step metrics-log row (B2G_*_LOG_COLS in include/b200grasp.h), by handle kind
LOG_COLS = {
    "sac": ("policy_loss", "qf1_loss", "qf2_loss", "value_loss", "ent_coef_loss", "entropy", "ent_coef", "learning_rate"),
    "bdq": ("loss", "mean_q", "grad_norm", "learning_rate"),
    "dqn": ("loss", "mean_q", "mean_abs_td", "grad_norm", "n_clipped", "learning_rate"),
}

ENC_MAX_LAYERS = 8


class EncoderCfg(C.Structure):
    _fields_ = [
        ("height", C.c_int32), ("width", C.c_int32), ("channels", C.c_int32), ("n_layers", C.c_int32),
        ("filters", C.c_int32 * ENC_MAX_LAYERS), ("kernel", C.c_int32 * ENC_MAX_LAYERS), ("strides", C.c_int32 * ENC_MAX_LAYERS),
        ("encoding_dim", C.c_int32), ("alpha", C.c_float), ("max_batch", C.c_int32), ("device", C.c_int32),
    ]


class BdqCfg(C.Structure):
    _fields_ = [
        ("obs_dim", C.c_int32), ("n_branches", C.c_int32), ("n_bins", C.c_int32), ("trunk0", C.c_int32), ("trunk1", C.c_int32),
        ("branch_hidden", C.c_int32), ("batch", C.c_int32), ("buffer_capacity", C.c_int64), ("gamma", C.c_float),
        ("target_update_freq", C.c_int32), ("trunk_grad_rescale", C.c_int32), ("seed", C.c_uint64), ("device", C.c_int32),
        ("rank", C.c_int32), ("nranks", C.c_int32), ("nccl_id", C.c_void_p), ("nccl_lib", C.c_char_p),
        ("prioritized_replay", C.c_int32), ("per_alpha", C.c_float), ("per_eps", C.c_float),
    ]


class BdqMetrics(C.Structure):
    _fields_ = [("loss", C.c_float), ("mean_q", C.c_float), ("grad_norm", C.c_float), ("n_updates", C.c_int64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class DqnCfg(C.Structure):
    _fields_ = [
        ("obs_dim", C.c_int32), ("n_actions", C.c_int32), ("hidden0", C.c_int32), ("hidden1", C.c_int32), ("batch", C.c_int32),
        ("buffer_capacity", C.c_int64), ("gamma", C.c_float), ("seed", C.c_uint64), ("device", C.c_int32),
        ("prioritized_replay", C.c_int32), ("per_alpha", C.c_float), ("per_eps", C.c_float),
    ]


class DqnMetrics(C.Structure):
    _fields_ = [("loss", C.c_float), ("mean_q", C.c_float), ("mean_abs_td", C.c_float), ("grad_norm", C.c_float),
                ("n_clipped", C.c_int32), ("n_updates", C.c_int64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class PpoCfg(C.Structure):
    _fields_ = [
        ("obs_dim", C.c_int32), ("n_actions", C.c_int32), ("hidden0", C.c_int32), ("hidden1", C.c_int32), ("n_envs", C.c_int32),
        ("n_steps", C.c_int32), ("nminibatches", C.c_int32), ("noptepochs", C.c_int32), ("gamma", C.c_float), ("lam", C.c_float),
        ("ent_coef", C.c_float), ("vf_coef", C.c_float), ("max_grad_norm", C.c_float), ("seed", C.c_uint64), ("device", C.c_int32),
    ]


class PpoMetrics(C.Structure):
    _fields_ = [("policy_loss", C.c_float), ("value_loss", C.c_float), ("entropy", C.c_float), ("approxkl", C.c_float),
                ("clipfrac", C.c_float), ("grad_norm", C.c_float), ("n_updates", C.c_int64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class TrpoCfg(C.Structure):
    _fields_ = [
        ("obs_dim", C.c_int32), ("n_actions", C.c_int32), ("hidden0", C.c_int32), ("hidden1", C.c_int32),
        ("timesteps_per_batch", C.c_int32), ("cg_iters", C.c_int32), ("vf_iters", C.c_int32), ("gamma", C.c_float), ("lam", C.c_float),
        ("max_kl", C.c_float), ("cg_damping", C.c_float), ("entcoeff", C.c_float), ("vf_stepsize", C.c_float), ("seed", C.c_uint64),
        ("device", C.c_int32),
    ]


class TrpoMetrics(C.Structure):
    _fields_ = [("optimgain", C.c_float), ("meankl", C.c_float), ("entbonus", C.c_float), ("surrgain", C.c_float), ("entropy", C.c_float),
                ("optimgain_after", C.c_float), ("meankl_after", C.c_float), ("entbonus_after", C.c_float),
                ("surrgain_after", C.c_float), ("entropy_after", C.c_float), ("grad_sq", C.c_float), ("shs", C.c_float),
                ("expected_improve", C.c_float), ("vf_loss", C.c_float), ("cg_iters", C.c_int32), ("accepted", C.c_int32),
                ("n_iterations", C.c_int64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class SacCfg(C.Structure):
    _fields_ = [
        ("obs_h", C.c_int32), ("obs_w", C.c_int32), ("obs_c", C.c_int32), ("obs_dim", C.c_int32),
        ("n_act", C.c_int32), ("hidden", C.c_int32), ("batch", C.c_int32), ("buffer_capacity", C.c_int64),
        ("gamma", C.c_float), ("tau", C.c_float), ("target_entropy", C.c_float), ("seed", C.c_uint64),
        ("precision", C.c_int32), ("device", C.c_int32), ("rank", C.c_int32), ("nranks", C.c_int32),
        ("nccl_id", C.c_void_p), ("nccl_lib", C.c_char_p),
    ]


class ReplayCfg(C.Structure):
    _fields_ = [("frame_capacity", C.c_int64), ("u8_plane_mask", C.c_uint32)]


#: b2g_sac_net_cfg.extractor: the CNN policy's feature extractor (include/b200grasp.h)
B2G_CNN_AUGMENTED, B2G_CNN_NATURE = 0, 1
EXTRACTORS = {"augmented": B2G_CNN_AUGMENTED, "nature_cnn": B2G_CNN_NATURE}


class SacNetCfg(C.Structure):
    _fields_ = [("extractor", C.c_int32)]


class SacMetrics(C.Structure):
    _fields_ = [(n, C.c_float) for n in (
        "policy_loss", "qf1_loss", "qf2_loss", "value_loss", "ent_coef_loss", "entropy", "ent_coef",
        "grad_norm_pi", "grad_norm_values", "grad_ent", "mean_q1", "mean_q2", "mean_v", "mean_logp")] + \
        [("n_updates", C.c_int64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


#: the gather-GEMM flags b2g_debug_gg_simt accepts (B2G_GG_* in include/b200grasp.h)
GG = dict(A_RVEC=1 << 0, B_RVEC=1 << 1, EPI_BIAS_RELU=1 << 2, EPI_MASK=1 << 3, EPI_ATOMIC=1 << 4, COLSUM=1 << 5,
          EPI_BIAS=1 << 10, EPI_SCALE=1 << 11, A_SCALAR=1 << 12, EPI_BIAS_LRELU=1 << 13, EPI_LRELU_GRAD=1 << 15,
          EPI_BIAS_TANH=1 << 16, EPI_TANH_GRAD=1 << 17)
#: the plane-producer flags of the wgmma engine that b2g_debug_gg_tc accepts besides A_RVEC .. COLSUM
GG_TC = dict(PLANES=1 << 6, A_ALIGN4=1 << 7, MN_MAJOR=1 << 9, A_ROWLANES=1 << 14)


class GgProblem(C.Structure):
    """b2g_debug_gg_problem: arena offsets (-1 = none), extents, flags, splitR and alpha of one gg_simt problem."""
    _fields_ = [(n, C.c_int64) for n in ("A", "B", "C", "bias", "mask", "colsum", "aM", "aR", "bR", "bN", "cM", "cN", "kM", "kN",
                                          "C_hi", "C_lo")] + \
        [(n, C.c_int32) for n in ("M", "N", "R", "flags", "splitR")] + [("alpha", C.c_float)]


class GgTcProblem(C.Structure):
    """b2g_debug_gg_tc_problem: arena offsets (-1 = none), extents, flags and splitR of one gg_tc problem."""
    _fields_ = [(n, C.c_int64) for n in ("A", "B", "C", "bias", "mask", "colsum", "aM", "aR", "bR", "bN", "cM", "cN", "kM", "kN",
                                          "bR_p", "bN_p", "A_hi", "A_lo", "B_hi", "B_lo", "C_hi", "C_lo")] + \
        [(n, C.c_int32) for n in ("M", "N", "R", "flags", "splitR")]


class B2GError(RuntimeError):
    def __init__(self, msg, code=None):
        super().__init__(msg)
        self.code = code


_lib = None


def load():
    """Loads libb200grasp.so (building it is ``__graft_entry__.build()`` / ``build.sh``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B2GError(f"{LIB_PATH} is missing: run ./build.sh (there is no CPU fallback for the learner path)")
    lib = C.CDLL(LIB_PATH)
    fp, dp, vp = C.POINTER(C.c_float), C.POINTER(C.c_double), C.c_void_p
    lib.b2g_last_error.restype = C.c_char_p
    lib.b2g_nccl_unique_id.argtypes = [vp, C.c_char_p]
    lib.b2g_sac_create.argtypes = [C.POINTER(SacCfg), C.POINTER(vp)]
    lib.b2g_sac_create2.argtypes = [C.POINTER(SacCfg), C.POINTER(ReplayCfg), C.POINTER(vp)]
    lib.b2g_sac_create3.argtypes = [C.POINTER(SacCfg), C.POINTER(ReplayCfg), C.POINTER(SacNetCfg), C.POINTER(vp)]
    i64p = C.POINTER(C.c_int64)
    lib.b2g_replay_info.argtypes = [vp, i64p, i64p, i64p, i64p, i64p, i64p]
    lib.b2g_sac_destroy.argtypes = [vp]
    lib.b2g_sac_dp_export.argtypes = [vp, vp]
    lib.b2g_sac_dp_connect.argtypes = [vp, vp, C.c_int]
    lib.b2g_debug_dp_stamps.argtypes = [vp, C.POINTER(C.c_longlong)]
    lib.b2g_debug_compact_host.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.b2g_sync.argtypes = [vp]
    lib.b2g_param_count.argtypes = [vp]
    lib.b2g_param_info.argtypes = [vp, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                   C.POINTER(C.c_int64)]
    for f in ("b2g_get_param", "b2g_set_param", "b2g_get_grad"):
        getattr(lib, f).argtypes = [vp, C.c_char_p, fp, C.c_size_t]
    lib.b2g_get_adam.argtypes = [vp, C.c_char_p, fp, fp, C.c_size_t]
    lib.b2g_reset_optimizer.argtypes = [vp]
    lib.b2g_replay_add.argtypes = [vp, fp, fp, fp, fp, fp, C.c_int64]
    lib.b2g_replay_size.argtypes = [vp]
    lib.b2g_replay_size.restype = C.c_int64
    lib.b2g_replay_get.argtypes = [vp, C.c_int64, fp, fp, fp, fp, fp]
    lib.b2g_get_last_batch.argtypes = [vp, C.POINTER(C.c_int32), fp, fp, fp]
    lib.b2g_set_norm_stats.argtypes = [vp, dp, dp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, C.c_int]
    lib.b2g_sac_step.argtypes = [vp, C.c_int, C.c_float, C.POINTER(SacMetrics)]
    lib.b2g_sac_step_async.argtypes = [vp, C.c_int, C.c_float]
    lib.b2g_sac_step_explicit.argtypes = [vp, fp, fp, fp, fp, fp, fp, C.c_float, C.c_int, C.POINTER(SacMetrics), fp, fp]
    lib.b2g_sac_step_host_pipelined.argtypes = [vp, fp, fp, fp, fp, fp, fp, C.c_float, C.POINTER(SacMetrics), C.POINTER(C.c_int)]
    lib.b2g_sac_pipeline_flush.argtypes = [vp, C.POINTER(SacMetrics)]
    lib.b2g_sac_act.argtypes = [vp, fp, C.c_int, C.c_int, fp]
    lib.b2g_sac_observe_act.argtypes = [vp, fp, C.c_int, C.c_int, C.c_int, fp]
    lib.b2g_sac_observe_add.argtypes = [vp, fp, fp, fp, fp, fp, C.c_int, C.c_int]
    lib.b2g_obs_rms_set.argtypes = [vp, dp, dp, C.c_double]
    lib.b2g_obs_rms_get.argtypes = [vp, dp, dp, dp]
    lib.b2g_upload_bytes.argtypes = [vp, i64p, i64p]
    lib.b2g_launches_per_step.argtypes = [vp]
    lib.b2g_last_step_ms.argtypes = [vp]
    lib.b2g_last_step_ms.restype = C.c_float
    lib.b2g_profile_step.argtypes = [vp, C.c_float, C.POINTER(C.c_char_p), fp, C.c_int]
    lib.b2g_sac_state_save.argtypes = lib.b2g_sac_state_load.argtypes = [vp, C.c_char_p]
    for p in ("bdq", "dqn", "ppo", "trpo"):  # the handle, named-parameter and training-state calls the learners share
        for f in ("destroy", "param_count"):
            getattr(lib, f"b2g_{p}_{f}").argtypes = [vp]
        getattr(lib, f"b2g_{p}_param_info").argtypes = [vp, C.c_int, C.c_char_p, C.c_size_t, i64p, i64p, C.POINTER(C.c_int32)]
        for f in ("get_param", "set_param", "get_grad"):
            getattr(lib, f"b2g_{p}_{f}").argtypes = [vp, C.c_char_p, fp, C.c_size_t]
        for f in ("state_save", "state_load"):
            getattr(lib, f"b2g_{p}_{f}").argtypes = [vp, C.c_char_p]
    for p in ("sac", "bdq", "dqn"):          # the per-step metrics ring of the replay learners
        getattr(lib, f"b2g_{p}_metrics_log").argtypes = [vp, C.c_int]
        getattr(lib, f"b2g_{p}_metrics_drain").argtypes = [vp, fp, C.c_int, i64p, C.POINTER(C.c_int), i64p]
    for p in ("bdq", "dqn"):                 # and the transition replay of the two Q learners
        getattr(lib, f"b2g_{p}_replay_add").argtypes = [vp, fp, fp, fp, fp, fp, C.c_int64]
        getattr(lib, f"b2g_{p}_replay_size").argtypes = [vp]
        getattr(lib, f"b2g_{p}_replay_size").restype = C.c_int64
        getattr(lib, f"b2g_{p}_set_norm_stats").argtypes = [vp, dp, dp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, C.c_int]
        getattr(lib, f"b2g_{p}_set_per_beta").argtypes = [vp, C.c_float]
        getattr(lib, f"b2g_{p}_get_last_per").argtypes = [vp, C.POINTER(C.c_int32), fp, fp]
        getattr(lib, f"b2g_{p}_replay_info").argtypes = [vp, i64p, i64p, i64p, i64p, i64p, i64p]
        getattr(lib, f"b2g_{p}_replay_get").argtypes = [vp, C.c_int64, fp, fp, fp, fp, fp, C.POINTER(C.c_int32)]
    lib.b2g_bdq_create2.argtypes = [C.POINTER(BdqCfg), C.POINTER(ReplayCfg), C.POINTER(vp)]
    lib.b2g_dqn_create2.argtypes = [C.POINTER(DqnCfg), C.POINTER(ReplayCfg), C.POINTER(vp)]
    lib.b2g_transition_replay_bytes.argtypes = [C.c_int64, C.c_int, C.c_int, C.c_int64]
    lib.b2g_transition_replay_bytes.restype = C.c_int64
    lib.b2g_bdq_create.argtypes = [C.POINTER(BdqCfg), C.POINTER(vp)]
    lib.b2g_bdq_step.argtypes = [vp, C.c_int, C.c_float, C.POINTER(BdqMetrics)]
    lib.b2g_bdq_step_explicit.argtypes = [vp, fp, fp, fp, fp, fp, fp, C.c_float, C.c_int, C.POINTER(BdqMetrics), fp]
    lib.b2g_bdq_act.argtypes = [vp, fp, C.c_int, C.POINTER(C.c_int32)]
    lib.b2g_bdq_observe_act.argtypes = [vp, fp, C.c_int, C.c_int, C.c_float, C.POINTER(C.c_int32)]
    lib.b2g_bdq_observe_add.argtypes = [vp, fp, fp, fp, fp, fp, C.c_int, C.c_int]
    lib.b2g_bdq_obs_rms_set.argtypes = [vp, dp, dp, C.c_double]
    lib.b2g_bdq_obs_rms_get.argtypes = [vp, dp, dp, dp]
    lib.b2g_bdq_upload_bytes.argtypes = [vp, i64p, i64p]
    lib.b2g_dqn_create.argtypes = [C.POINTER(DqnCfg), C.POINTER(vp)]
    lib.b2g_dqn_step.argtypes = [vp, C.c_int, C.c_float, C.POINTER(DqnMetrics)]
    lib.b2g_dqn_step_explicit.argtypes = [vp, fp, fp, fp, fp, fp, fp, C.c_float, C.c_int, C.POINTER(DqnMetrics), fp]
    lib.b2g_dqn_update_target.argtypes = [vp]
    lib.b2g_dqn_act.argtypes = lib.b2g_dqn_act_raw.argtypes = [vp, fp, C.c_int, C.POINTER(C.c_int32), fp]
    lib.b2g_dqn_observe_act.argtypes = [vp, fp, C.c_int, C.c_int, C.c_float, C.POINTER(C.c_int32)]
    lib.b2g_dqn_observe_add.argtypes = [vp, fp, fp, fp, fp, fp, C.c_int, C.c_int]
    lib.b2g_dqn_obs_rms_set.argtypes = [vp, dp, dp, C.c_double]
    lib.b2g_dqn_obs_rms_get.argtypes = [vp, dp, dp, dp]
    lib.b2g_dqn_upload_bytes.argtypes = [vp, i64p, i64p]
    lib.b2g_dqn_set_obs_encoder.argtypes = [vp, vp, C.c_int]
    lib.b2g_ppo_create.argtypes = [C.POINTER(PpoCfg), C.POINTER(vp)]
    lib.b2g_ppo_rollout_act.argtypes = [vp, fp, fp]
    lib.b2g_ppo_rollout_reward.argtypes = [vp, fp, fp]
    lib.b2g_ppo_rollout_reset.argtypes = [vp]
    lib.b2g_ppo_rollout_get.argtypes = [vp, fp, fp, fp, fp, fp]
    lib.b2g_ppo_update.argtypes = [vp, fp, C.POINTER(C.c_int32), C.c_float, C.c_float, C.c_float, C.POINTER(PpoMetrics)]
    lib.b2g_ppo_train_step_explicit.argtypes = [vp, fp, fp, fp, fp, fp, C.c_float, C.c_float, C.c_float, C.c_int, C.POINTER(PpoMetrics)]
    lib.b2g_ppo_act.argtypes = [vp, fp, C.c_int, C.c_int, fp, fp, fp]
    lib.b2g_ppo_get_step.argtypes = [vp, i64p, i64p, C.POINTER(C.c_int32)]
    lib.b2g_trpo_create.argtypes = [C.POINTER(TrpoCfg), C.POINTER(vp)]
    lib.b2g_trpo_rollout_act.argtypes = [vp, fp, fp]
    lib.b2g_trpo_rollout_reward.argtypes = [vp, C.c_float, C.c_float]
    lib.b2g_trpo_rollout_reset.argtypes = [vp]
    lib.b2g_trpo_rollout_get.argtypes = [vp, fp, fp, fp, fp]
    lib.b2g_trpo_update.argtypes = [vp, fp, C.POINTER(C.c_int32), C.POINTER(TrpoMetrics)]
    lib.b2g_trpo_fvp.argtypes = [vp, fp, fp, fp]
    lib.b2g_trpo_step_explicit.argtypes = [vp, fp, fp, fp, fp, C.POINTER(C.c_int32), C.POINTER(TrpoMetrics), fp, fp, fp]
    lib.b2g_trpo_act.argtypes = [vp, fp, C.c_int, C.c_int, fp, fp]
    lib.b2g_trpo_get_step.argtypes = [vp, i64p, i64p, C.POINTER(C.c_int32)]
    for p in ("ppo", "trpo"):                # VecNormalize's obs_rms on the device and the observe path of the two
        getattr(lib, f"b2g_{p}_obs_rms_set").argtypes = [vp, dp, dp, C.c_double]
        getattr(lib, f"b2g_{p}_obs_rms_get").argtypes = [vp, dp, dp, dp]
        getattr(lib, f"b2g_{p}_upload_bytes").argtypes = [vp, i64p, i64p]
        getattr(lib, f"b2g_{p}_set_norm_stats").argtypes = [vp, C.c_double, C.c_double, C.c_int]
        getattr(lib, f"b2g_{p}_set_obs_encoder").argtypes = [vp, vp, C.c_int]
        getattr(lib, f"b2g_{p}_observe_act").argtypes = [vp, fp, C.c_int, C.c_int, fp]
    lib.b2g_ppo_act_raw.argtypes = [vp, fp, C.c_int, C.c_int, fp, fp, fp]
    lib.b2g_trpo_act_raw.argtypes = [vp, fp, C.c_int, C.c_int, fp, fp]
    lib.b2g_encoder_create.argtypes = [C.POINTER(EncoderCfg), C.POINTER(vp)]
    lib.b2g_encoder_destroy.argtypes = [vp]
    lib.b2g_encoder_n_layers.argtypes = [vp]
    lib.b2g_encoder_layer_shape.argtypes = [vp, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    lib.b2g_encoder_set_weights.argtypes = [vp, C.c_int, fp, C.c_size_t, fp, C.c_size_t]
    lib.b2g_encoder_encode.argtypes = [vp, fp, C.c_int, fp]
    lib.b2g_encoder_create2.argtypes = [C.POINTER(EncoderCfg), C.c_int32, C.POINTER(vp)]
    lib.b2g_debug_encoder_layers.argtypes = [vp, fp, C.c_int, fp, C.c_int64]
    lib.b2g_sac_set_obs_encoder.argtypes = [vp, vp, C.c_int]
    lib.b2g_bdq_set_obs_encoder.argtypes = [vp, vp, C.c_int]
    lib.b2g_autoencoder_create.argtypes = [C.POINTER(EncoderCfg), C.POINTER(vp)]
    lib.b2g_autoencoder_create2.argtypes = [C.POINTER(EncoderCfg), C.c_int32, C.POINTER(vp)]
    lib.b2g_debug_autoencoder_tensor.argtypes = [vp, C.c_int, C.c_int, fp, C.c_int64, C.POINTER(C.c_int32)]
    lib.b2g_debug_autoencoder_tensor_numel.argtypes = [vp, C.c_int, C.c_int]
    lib.b2g_debug_autoencoder_tensor_numel.restype = C.c_int64
    lib.b2g_autoencoder_destroy.argtypes = [vp]
    lib.b2g_autoencoder_n_layers.argtypes = [vp]
    lib.b2g_autoencoder_layer_shape.argtypes = [vp, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    for f in ("b2g_autoencoder_set_weights", "b2g_autoencoder_get_weights", "b2g_autoencoder_get_grad"):
        getattr(lib, f).argtypes = [vp, C.c_int, fp, C.c_size_t, fp, C.c_size_t]
    lib.b2g_autoencoder_reset_optimizer.argtypes = [vp]
    lib.b2g_autoencoder_set_dataset.argtypes = [vp, fp, fp, C.c_int64]
    lib.b2g_autoencoder_train_epoch.argtypes = [vp, C.POINTER(C.c_int32), C.c_int64, C.c_int, C.c_float, dp]
    lib.b2g_autoencoder_evaluate.argtypes = [vp, C.c_int64, C.c_int64, dp]
    lib.b2g_autoencoder_predict.argtypes = [vp, fp, C.c_int, fp]
    lib.b2g_autoencoder_step.argtypes = [vp, fp, fp, C.c_int, C.c_float, C.c_int, dp]
    lib.b2g_debug_gemm.argtypes = [C.c_int, C.c_int, C.c_int, fp, fp, fp, C.c_int, C.c_int]
    lib.b2g_debug_tensor_info.argtypes = [vp, C.c_char_p, i64p, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    lib.b2g_debug_tensor.argtypes = [vp, C.c_char_p, C.c_int, vp, C.c_size_t]
    for k in ("ppo", "trpo"):
        getattr(lib, f"b2g_debug_{k}_tensor_info").argtypes = [vp, C.c_char_p, i64p, C.POINTER(C.c_int32)]
        getattr(lib, f"b2g_debug_{k}_tensor").argtypes = [vp, C.c_char_p, vp, C.c_size_t]
    lib.b2g_debug_trpo_cg.argtypes = [vp, fp, fp, fp, C.c_int, fp]
    lib.b2g_debug_gg_simt.argtypes = [C.c_int, C.POINTER(GgProblem), C.c_int, fp, C.c_int64, dp, C.c_int64, C.POINTER(C.c_uint16),
                                      C.c_int64, C.POINTER(C.c_int32), C.c_int64]
    lib.b2g_debug_gg_tc.argtypes = [C.c_int, C.POINTER(GgTcProblem), C.c_int, fp, C.c_int64, C.POINTER(C.c_uint16), C.c_int64,
                                    C.POINTER(C.c_int32), C.c_int64]
    _lib = lib
    return lib


def check(rc: int):
    if rc < 0:
        raise B2GError(f"libb200grasp error {rc}: {load().b2g_last_error().decode(errors='replace')}", rc)
    return rc


def default_nccl_lib():
    """Prefer the NCCL bundled with torch (2.28.9) over the system one (2.27.3)."""
    try:
        import importlib.util
        spec = importlib.util.find_spec("nvidia.nccl")
        if spec and spec.submodule_search_locations:
            p = os.path.join(list(spec.submodule_search_locations)[0], "lib", "libnccl.so.2")
            if os.path.exists(p):
                return p
    except Exception:
        pass
    return None
