"""ctypes binding of the C-ABI declared in include/xtb200.h.

This is the stub a reference maintainer would add (INTEGRATION.md shows it in full): plain
pointers and sizes, no torch types.  Loading fails loudly when the CUDA library is missing --
the product path has no CPU fallback."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("XTB_LIB_PATH") or os.path.join(HERE, "lib", "libxtb200.so")   # override: experiment builds (scripts/)

XTB_MAX_LAYERS = 16
CONV, DENSE, DUELING, LOGSTD = 0, 1, 2, 3
# enum xtb_act: the keys of the reference's ACTIVATION_MAP plus linear / None
ACT = {None: 0, "linear": 0, "relu": 1, "tanh": 2, "sigmoid": 3, "softsign": 4, "softplus": 5, "leaky_relu": 6, "elu": 7,
       "selu": 8, "swish": 9, "gelu": 10}
CLIP_NONE, CLIP_GLOBAL_NORM, CLIP_PER_TENSOR = 0, 1, 2
PER_NONFINITE, PER_BAD_INDEX, PER_EMPTY = 1, 2, 4     # xtb_per status bits
MZR_BAD_PRIORITY, MZR_REMAPPED, MZR_BAD_INDEX = 1, 2, 4   # xtb_muzero_replay status bits


class LayerDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("src", C.c_int32), ("act", C.c_int32), ("k", C.c_int32),
                ("stride", C.c_int32), ("cout", C.c_int32), ("pad_same", C.c_int32)]


class NetDesc(C.Structure):
    _fields_ = [("input_u8", C.c_int32), ("scale", C.c_float), ("in_h", C.c_int32), ("in_w", C.c_int32),
                ("in_c", C.c_int32), ("n_layers", C.c_int32), ("layers", LayerDesc * XTB_MAX_LAYERS)]


class LayerPlan(C.Structure):
    _fields_ = [("kind", C.c_int32), ("tc", C.c_int32), ("s2d", C.c_int32), ("w_res", C.c_int32), ("n_fwd", C.c_int32),
                ("n_dg", C.c_int32), ("R", C.c_int32), ("fwd_stages", C.c_int32), ("dg_stages", C.c_int32),
                ("dg_empty_units", C.c_int32), ("k_slices", C.c_int32)]


class PpoHyper(C.Structure):
    _fields_ = [("clip_ratio", C.c_float), ("ent_coef", C.c_float), ("vf_clip", C.c_float),
                ("critic_coef", C.c_float)]


class PpoRollout(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("action", C.c_void_p), ("old_logp", C.c_void_p), ("adv", C.c_void_p),
                ("old_v", C.c_void_p), ("target_v", C.c_void_p)]


class ImpalaTraj(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("behav_prob", C.c_void_p), ("action_mat", C.c_void_p), ("reward", C.c_void_p),
                ("done", C.c_void_p)]


class MuzeroDesc(C.Structure):
    _fields_ = [("unroll", C.c_int32), ("rep_h", C.c_int32), ("dyn_h", C.c_int32), ("dyn_r", C.c_int32), ("pred_p", C.c_int32),
                ("pred_v", C.c_int32), ("value_min", C.c_float), ("value_max", C.c_float), ("reward_min", C.c_float),
                ("reward_max", C.c_float)]


class MuzeroBatch(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("action", C.c_void_p), ("target_value", C.c_void_p), ("target_reward", C.c_void_p),
                ("target_policy", C.c_void_p), ("unroll", C.c_int32)]


class MuzeroReplaySlot(C.Structure):
    _fields_ = [("off", C.c_int64), ("len", C.c_int32), ("live", C.c_int32)]


class MuzeroReplayBatch(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("action", C.c_void_p), ("target_value", C.c_void_p), ("target_reward", C.c_void_p),
                ("target_policy", C.c_void_p)]


class QmixDesc(C.Structure):
    _fields_ = [("batch", C.c_int32), ("episode_limit", C.c_int32), ("n_agents", C.c_int32), ("use_double_q", C.c_int32),
                ("gamma", C.c_float), ("gru_off", C.c_longlong), ("act_envs", C.c_int32)]


class QmixBatch(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("seq_len", C.c_void_p), ("avail", C.c_void_p), ("actions", C.c_void_p), ("state", C.c_void_p),
                ("next_state", C.c_void_p), ("reward", C.c_void_p), ("terminated", C.c_void_p), ("mask", C.c_void_p)]


class SccDesc(C.Structure):
    _fields_ = [("batch", C.c_int32), ("episode_limit", C.c_int32), ("n_agents", C.c_int32), ("n_groups", C.c_int32),
                ("group", C.c_int32 * 8), ("channel_merge", C.c_int32), ("mc_sample_times", C.c_int32), ("gamma", C.c_float),
                ("gru_off", C.c_longlong), ("head_off", C.c_longlong), ("act_envs", C.c_int32)]


class SccBatch(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("raw_obs", C.c_void_p), ("seq_len", C.c_void_p), ("actions", C.c_void_p), ("reward", C.c_void_p),
                ("terminated", C.c_void_p), ("mask", C.c_void_p), ("subsets", C.c_void_p)]


class EpisodeBatch(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("raw_obs", C.c_void_p), ("seq_len", C.c_void_p), ("avail", C.c_void_p), ("actions", C.c_void_p),
                ("state", C.c_void_p), ("next_state", C.c_void_p), ("reward", C.c_void_p), ("terminated", C.c_void_p),
                ("mask", C.c_void_p)]


class InfoflowDesc(C.Structure):
    _fields_ = [("user_dim", C.c_int32), ("item_dim", C.c_int32), ("emb_dim", C.c_int32), ("vocab", C.c_int32), ("batch", C.c_int32),
                ("last_act", C.c_int32), ("gamma", C.c_double), ("gru_off", C.c_longlong), ("gru1_off", C.c_longlong),
                ("head_off", C.c_longlong), ("table", C.c_void_p)]


class InfoflowBatch(C.Structure):
    _fields_ = [("user", C.c_void_p), ("click", C.c_void_p), ("noclick", C.c_void_p), ("item", C.c_void_p), ("next_user", C.c_void_p),
                ("next_click", C.c_void_p), ("next_noclick", C.c_void_p), ("cand_off", C.c_void_p), ("cand_item", C.c_void_p),
                ("reward", C.c_void_p), ("done", C.c_void_p), ("label", C.c_void_p), ("n_cand", C.c_int32), ("cand_cap", C.c_int32)]


_P = C.c_void_p
_SIGS = {
    "xtb_version": (C.c_int, []),
    "xtb_last_error": (C.c_char_p, []),
    "xtb_launch_count": (C.c_longlong, []),
    "xtb_graph_replay_count": (C.c_longlong, []),
    "xtb_graph_capture_count": (C.c_longlong, []),
    "xtb_net_create": (C.c_int, [C.POINTER(NetDesc), C.c_int, C.POINTER(_P)]),
    "xtb_net_destroy": (None, [_P]),
    "xtb_net_param_count": (C.c_longlong, [_P]),
    "xtb_net_layer_params": (C.c_int, [_P, C.c_int, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong),
                                       C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "xtb_net_layer_plan": (C.c_int, [_P, C.c_int, C.POINTER(LayerPlan)]),
    "xtb_net_tensor_size": (C.c_int, [_P, C.c_int]),
    "xtb_net_workspace_bytes": (C.c_size_t, [_P]),
    "xtb_net_bind": (C.c_int, [_P, _P, _P, _P, C.c_size_t]),
    "xtb_net_bind_stream": (C.c_int, [_P, _P, _P, _P, C.c_size_t, _P]),
    "xtb_net_sync_weights": (C.c_int, [_P, _P]),
    "xtb_net_tensor": (_P, [_P, C.c_int]),
    "xtb_net_tensor_grad": (_P, [_P, C.c_int]),
    "xtb_net_forward": (C.c_int, [_P, _P, _P, _P, C.c_int, _P]),
    "xtb_net_backward": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(C.c_int32), C.c_int, _P]),
    "xtb_categorical_sample": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "xtb_argmax": (C.c_int, [_P, C.c_int, C.c_int, _P, _P]),
    "xtb_gae": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, _P, _P, _P, _P]),
    "xtb_ppo_loss_grad": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.POINTER(PpoHyper),
                                    C.c_float, _P, _P, _P, _P]),
    "xtb_vtrace_loss_grad": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float,
                                       _P, _P, _P, _P, _P, _P]),
    "xtb_dqn_loss_grad": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_float,
                                    _P, _P, _P, _P]),
    "xtb_dqn_td_loss_grad": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float,
                                      _P, _P, _P, _P, _P, _P]),
    "xtb_nstep_returns": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_float, _P, _P, _P, _P, _P]),
    "xtb_impala_train": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, _P, C.c_int, _P]),
    "xtb_dqn_train": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_float, C.c_float, C.c_int, _P, _P, _P,
                               C.c_int, _P]),
    "xtb_dqn_train_weighted": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_float, C.c_float, C.c_int, _P, _P,
                                        _P, _P, _P, C.c_int, _P]),
    "xtb_per_create": (C.c_int, [C.c_int, C.c_double, C.c_double, C.c_uint64, C.POINTER(_P)]),
    "xtb_per_destroy": (None, [_P]),
    "xtb_per_add": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "xtb_per_sample": (C.c_int, [_P, C.c_int, C.c_double, _P, _P, _P, _P]),
    "xtb_per_update": (C.c_int, [_P, _P, _P, C.c_int, _P]),
    "xtb_per_state": (C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_int),
                                C.POINTER(C.c_ulonglong), _P, _P]),
    "xtb_dqn_per_train": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_float, C.c_float, C.c_double, C.c_int,
                                   _P, _P, _P, _P, _P, _P, _P, C.c_int, _P]),
    "xtb_mse_loss_grad": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_float, _P, _P, _P]),
    "xtb_softmax": (C.c_int, [_P, C.c_int, C.c_int, _P, _P]),
    "xtb_impala_keras_loss_grad": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float,
                                             _P, _P, _P, _P]),
    "xtb_impala_keras_fit": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, _P,
                                       C.c_int, _P]),
    "xtb_impala_keras_train": (C.c_int, [_P, _P, C.POINTER(ImpalaTraj), C.c_int, C.c_int, C.c_int, C.c_int, _P, _P,
                                         C.c_float, C.c_float, C.c_int, C.c_int, _P, _P, _P, C.c_int, _P]),
    "xtb_adam_create": (C.c_int, [C.c_longlong, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int,
                                  C.c_float, C.POINTER(C.c_longlong), C.c_int, _P, _P, C.POINTER(_P)]),
    "xtb_adam_destroy": (None, [_P]),
    "xtb_adam_step": (C.c_int, [_P, _P, _P, C.c_float, _P]),
    "xtb_adam_step_net": (C.c_int, [_P, _P, C.c_float, _P]),
    "xtb_adam_grad_norm": (_P, [_P]),
    "xtb_adam_set_lr": (C.c_int, [_P, C.c_float]),
    "xtb_adam_set_decay": (C.c_int, [_P, C.c_float]),
    "xtb_opt_use_rmsprop": (C.c_int, [_P, _P, C.c_float, C.c_float]),
    "xtb_opt_use_rmsprop_plain": (C.c_int, [_P, C.c_float, C.c_float]),
    "xtb_ppo_train": (C.c_int, [_P, _P, C.POINTER(PpoRollout), C.c_int, C.c_int, C.c_int, _P, C.POINTER(PpoHyper),
                                C.c_int, C.c_int, C.c_int, _P, C.c_int, _P]),
    "xtb_ppo_rollout_infer": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, _P, _P, _P, _P,
                                        C.c_int, _P]),
    "xtb_ppo_predict_host": (C.c_int, [_P, _P, C.c_size_t, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint64, _P, _P, _P, _P,
                                       C.c_int, _P]),
    "xtb_ppo_heads_plan": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "xtb_dqn_heads_plan": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "xtb_diag_gaussian_sample": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "xtb_ppo_gauss_loss_grad": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, C.POINTER(PpoHyper), C.c_float,
                                          _P, _P, _P, _P, _P]),
    "xtb_muzero_create": (C.c_int, [_P, _P, _P, C.POINTER(MuzeroDesc), C.c_int, C.POINTER(_P)]),
    "xtb_muzero_destroy": (None, [_P]),
    "xtb_muzero_train": (C.c_int, [_P, _P, C.POINTER(MuzeroBatch), C.c_int, C.c_float, _P, _P, C.c_int, _P]),
    "xtb_muzero_initial_inference": (C.c_int, [_P, _P, C.c_int, _P, _P, _P, C.c_int, _P]),
    "xtb_muzero_recurrent_inference": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, _P, C.c_int, _P]),
    "xtb_muzero_tree_create": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(_P)]),
    "xtb_muzero_tree_destroy": (None, [_P]),
    "xtb_muzero_search": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, C.c_double, C.c_double, C.c_double, C.c_double, _P, _P,
                                    C.c_int, _P]),
    "xtb_muzero_replay_create": (C.c_int, [C.c_int, C.c_longlong, C.c_int, C.c_longlong, C.c_int, C.c_int, C.POINTER(_P)]),
    "xtb_muzero_replay_destroy": (None, [_P]),
    "xtb_muzero_replay_add": (C.c_int, [_P, _P, C.c_int, C.c_longlong, C.c_int, C.c_int, _P, _P, _P, _P, _P, C.c_int, _P, _P]),
    "xtb_muzero_replay_sample": (C.c_int, [_P, C.c_int, _P, _P, _P, C.POINTER(MuzeroReplayBatch), _P]),
    "xtb_muzero_replay_update": (C.c_int, [_P, C.c_int, _P, _P, _P, _P]),
    "xtb_muzero_replay_train": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, C.POINTER(MuzeroReplayBatch), C.c_float, _P, _P,
                                          C.c_int, _P]),
    "xtb_muzero_replay_state": (C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), _P, _P, _P]),
    "xtb_qmix_create": (C.c_int, [_P, _P, _P, C.POINTER(QmixDesc), C.POINTER(_P)]),
    "xtb_qmix_destroy": (None, [_P]),
    "xtb_qmix_train": (C.c_int, [_P, _P, _P, C.POINTER(QmixBatch), _P, C.c_int, _P]),
    "xtb_qmix_infer": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, _P]),
    "xtb_qmix_act": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, C.c_uint64, _P, _P, _P, _P, C.c_int, _P]),
    "xtb_scc_create": (C.c_int, [_P, _P, C.POINTER(_P), C.POINTER(SccDesc), C.POINTER(_P)]),
    "xtb_scc_destroy": (None, [_P]),
    "xtb_scc_train": (C.c_int, [_P, _P, _P, _P, C.POINTER(SccBatch), _P, C.c_int, _P]),
    "xtb_scc_infer": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, _P]),
    "xtb_scc_act": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, C.c_uint64, _P, _P, _P, _P, C.c_int, _P]),
    "xtb_scc_critic": (C.c_int, [_P, _P, C.c_int, _P, C.c_int, _P]),
    "xtb_episode_replay_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "xtb_episode_replay_destroy": (None, [_P]),
    "xtb_episode_replay_row_bytes": (C.c_longlong, [_P]),
    "xtb_episode_replay_add": (C.c_int, [_P, C.c_int, _P, C.c_longlong, _P]),
    "xtb_episode_replay_gather": (C.c_int, [_P, C.c_int, _P, C.POINTER(EpisodeBatch), _P, _P]),
    "xtb_qmix_replay_train": (C.c_int, [_P, _P, _P, _P, C.c_int, _P, C.POINTER(QmixBatch), _P, _P, C.c_int, _P]),
    "xtb_scc_replay_train": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, _P, C.POINTER(SccBatch), _P, _P, C.c_int, _P]),
    "xtb_infoflow_create": (C.c_int, [C.POINTER(InfoflowDesc), C.POINTER(_P)]),
    "xtb_infoflow_destroy": (None, [_P]),
    "xtb_infoflow_train": (C.c_int, [_P, _P, _P, C.POINTER(InfoflowBatch), _P, _P, C.c_int, _P]),
    "xtb_infoflow_predict": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, _P, C.c_int, _P]),
    "xtb_net_backward_input": (C.c_int, [_P, _P, _P, C.c_int, C.POINTER(C.c_int32), C.c_int, _P, _P]),
    "xtb_comm_unique_id": (C.c_int, [C.c_char_p, _P]),
    "xtb_comm_create": (C.c_int, [C.c_char_p, _P, C.c_int, C.c_int, C.POINTER(_P)]),
    "xtb_comm_destroy": (None, [_P]),
    "xtb_comm_world": (C.c_int, [_P]),
    "xtb_set_grad_comm": (C.c_int, [_P]),
    "xtb_comm_allreduce": (C.c_int, [_P, _P, C.c_longlong, _P]),
    "xtb_net_bench_layer": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, C.c_int, _P]),
    "xtb_set_fuse_heads": (C.c_int, [C.c_int]),
    "xtb_set_tc_mode": (C.c_int, [C.c_int]),
    "xtb_get_tc_mode": (C.c_int, []),
    "xtb_tc_gemm_test": (C.c_int, [C.c_int, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_int, _P]),
    "xtb_pinned_alloc": (_P, [C.c_size_t]),
    "xtb_pinned_free": (None, [_P]),
    "xtb_copy_h2d": (C.c_int, [_P, _P, C.c_size_t, _P]),
    "xtb_copy_h2d_staged": (C.c_int, [_P, _P, C.c_size_t, _P]),
    "xtb_copy_d2h": (C.c_int, [_P, _P, C.c_size_t, _P]),
    "xtb_stream_sync": (C.c_int, [_P]),
}

EXPORTED = tuple(_SIGS)
_lib = None


def lib():
    """Load libxtb200.so (once).  Raises if the CUDA library has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "xingtian_b200: CUDA library %s is missing -- run `python -m xingtian_b200.build` "
                "(there is no CPU fallback)" % LIB_PATH)
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(handle, name)   # AttributeError if a declared symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(rc):
    if rc != 0:
        raise RuntimeError("xtb200 error %d: %s" % (rc, lib().xtb_last_error().decode()))
