"""ctypes binding of the C ABI declared in ``include/irbpp.h``.

There is deliberately no fallback: if ``lib/libirbpp.so`` is missing this raises, and if no CUDA
device is present ``irbpp_create`` fails with ``IRBPP_ECUDA``."""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("IRBPP_LIB") or os.path.join(HERE, "lib", "libirbpp.so")   # IRBPP_LIB: build-variant experiments

c_i32, c_i64, c_f64 = ctypes.c_int32, ctypes.c_int64, ctypes.c_double
c_void_p, c_char_p = ctypes.c_void_p, ctypes.c_char_p

IRBPP_OK, IRBPP_EINVAL, IRBPP_ECUDA, IRBPP_ESTATE, IRBPP_EDEVICE = 0, -1, -2, -3, -4
ABI_VERSION = 2


class IrbppConfig(ctypes.Structure):
    _fields_ = [("num_envs", c_i32), ("num_rotations", c_i32), ("selected_action", c_i32),
                ("buffer_size", c_i32), ("bin_dimension", c_f64 * 3), ("resolution_act", c_f64),
                ("resolution_h", c_f64), ("resolution_z", c_f64), ("device", c_i32), ("approx_legacy", c_i32)]


class IrbppStepResult(ctypes.Structure):
    _fields_ = [("reward", c_void_p), ("done", c_void_p), ("valid", c_void_p), ("error", c_void_p),
                ("counter", c_void_p), ("ep_len", c_void_p), ("ratio", c_void_p), ("ep_reward", c_void_p)]


# The arrays irbpp_step_result points at, in the order of the library's result block, with their element types
RESULT_FIELDS = tuple((name, np.dtype(t)) for name, t in (
    ("ratio", np.float64), ("ep_reward", np.float64), ("reward", np.float32), ("counter", np.int32), ("ep_len", np.int32),
    ("done", np.uint8), ("valid", np.uint8), ("error", np.uint8)))


class IrbppReplayMemory(ctypes.Structure):
    _fields_ = [("num_memories", c_i32), ("capacity", c_i32), ("obs_len", c_i32), ("states", c_void_p),
                ("timesteps", c_void_p), ("actions", c_void_p), ("rewards", c_void_p), ("nonterminals", c_void_p),
                ("tree", c_void_p), ("state", c_void_p)]


class IrbppReplayBatch(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in ("tree_idx", "states", "actions", "returns", "next_states", "nonterminals",
                                         "weights", "attempts", "error")]


class IrbppDqnWeights(ctypes.Structure):
    """``irbpp_dqn_weights``: device pointers of the location network's effective weights, then the LeakyReLU slope."""
    _fields_ = [(n, c_void_p) for n in ("conv1_w", "conv1_b", "conv2_w", "conv2_b", "conv3_w", "conv3_b", "cand1_w",
                                         "cand1_b", "cand2_w", "cand2_b", "proj1_w", "proj1_b", "proj2_w", "proj2_b",
                                         "fc_h_v_w", "fc_h_v_b", "fc_z_v_w", "fc_z_v_b", "fc_h_a_w", "fc_h_a_b",
                                         "fc_z_a_w", "fc_z_a_b")] + [("negative_slope", ctypes.c_float)]


class IrbppDqnOrderWeights(ctypes.Structure):
    """``irbpp_dqn_order_weights``: device pointers of the order network's effective weights, then the LeakyReLU slope."""
    _fields_ = [(n, c_void_p) for n in ("conv1_w", "conv1_b", "conv2_w", "conv2_b", "conv3_w", "conv3_b", "gat1_w",
                                         "gat1_b", "gat2_w", "gat2_b", "wq", "wk", "wv", "wo_w", "wo_b", "ff1_w", "ff1_b",
                                         "ff2_w", "ff2_b", "fc_h_v_w", "fc_h_v_b", "fc_z_v_w", "fc_z_v_b", "fc_h_a_w",
                                         "fc_h_a_b", "fc_z_a_w", "fc_z_a_b")] + [("negative_slope", ctypes.c_float)]


class IrbppDqnGrads(ctypes.Structure):
    """``irbpp_dqn_grads``: device pointers of the gradients of the location network's row-section tensors."""
    _fields_ = [(n, c_void_p) for n in ("cand1_w", "cand1_b", "cand2_w", "cand2_b", "proj1_w", "proj1_b", "proj2_w",
                                         "proj2_b", "fc_h_v_w", "fc_h_v_b", "fc_z_v_w", "fc_z_v_b", "fc_h_a_w", "fc_h_a_b",
                                         "fc_z_a_w", "fc_z_a_b")]


class IrbppDqnOrderGrads(ctypes.Structure):
    """``irbpp_dqn_order_grads``: device pointers of the gradients of the order network's tensors after the convolutions."""
    _fields_ = [(n, c_void_p) for n in ("gat1_w", "gat1_b", "gat2_w", "gat2_b", "wq", "wk", "wv", "wo_w", "wo_b", "ff1_w",
                                         "ff1_b", "ff2_w", "ff2_b", "fc_h_v_w", "fc_h_v_b", "fc_z_v_w", "fc_z_v_b",
                                         "fc_h_a_w", "fc_h_a_b", "fc_z_a_w", "fc_z_a_b")]


class IrbppHeightEncoderWeights(ctypes.Structure):
    """``irbpp_height_encoder_weights``: device pointers of the height encoder's six tensors, then the LeakyReLU slope."""
    _fields_ = [(n, c_void_p) for n in ("conv1_w", "conv1_b", "conv2_w", "conv2_b", "conv3_w", "conv3_b")] + \
        [("negative_slope", ctypes.c_float)]


class IrbppHeightEncoderGrads(ctypes.Structure):
    """``irbpp_height_encoder_grads``: device pointers of the gradients of the height encoder's six tensors."""
    _fields_ = [(n, c_void_p) for n in ("conv1_w", "conv1_b", "conv2_w", "conv2_b", "conv3_w", "conv3_b")]


# symbol -> (restype, argtypes); every symbol of include/irbpp.h appears here (checked by the tests)
SIGNATURES = {
    "irbpp_abi_version": (c_i32, []),
    "irbpp_create": (c_i32, [ctypes.POINTER(IrbppConfig), ctypes.POINTER(c_void_p)]),
    "irbpp_destroy": (c_i32, [c_void_p]),
    "irbpp_last_error": (c_char_p, [c_void_p]),
    "irbpp_obs_len": (c_i32, [c_void_p, ctypes.POINTER(c_i32), ctypes.POINTER(c_i32), ctypes.POINTER(c_i32)]),
    "irbpp_load_shapes": (c_i32, [c_void_p, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64]),
    "irbpp_set_sequences": (c_i32, [c_void_p, c_void_p, c_i32]),
    "irbpp_set_item_rng": (c_i32, [c_void_p, ctypes.c_uint64]),
    "irbpp_set_item_groups": (c_i32, [c_void_p, ctypes.c_uint64, c_i32, c_void_p, c_void_p]),
    "irbpp_set_trajectories": (c_i32, [c_void_p, c_void_p, c_void_p, c_i32, c_i32, c_i32]),
    "irbpp_reset": (c_i32, [c_void_p, c_void_p, c_void_p, c_void_p]),
    "irbpp_step_async": (c_i32, [c_void_p, c_void_p, c_i32, c_void_p, c_void_p]),
    "irbpp_step_wait": (c_i32, [c_void_p, ctypes.POINTER(IrbppStepResult)]),
    "irbpp_step_wait_device": (c_i32, [c_void_p, ctypes.POINTER(IrbppStepResult)]),
    "irbpp_device_results": (c_i32, [c_void_p, ctypes.POINTER(IrbppStepResult)]),
    "irbpp_get_action_candidates": (c_i32, [c_void_p, c_void_p, c_i32, c_void_p, c_void_p]),
    "irbpp_get_all_possible_observation": (c_i32, [c_void_p, c_void_p, c_void_p]),
    "irbpp_heuristic_actions": (c_i32, [c_void_p, c_i32, c_i32, c_void_p, c_void_p, c_i32, c_void_p]),
    "irbpp_step_poses_async": (c_i32, [c_void_p, c_void_p, c_i32, c_void_p, c_void_p]),
    "irbpp_debug_state": (c_i32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "irbpp_debug_set_heightmap": (c_i32, [c_void_p, c_void_p]),
    "irbpp_debug_scan": (c_i32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "irbpp_debug_hulls": (c_i32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "irbpp_launch_count": (c_i64, [c_void_p]),
    "irbpp_packed_obs_bytes": (c_i32, [c_i32]),
    "irbpp_pack_observations": (c_i32, [c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p]),
    "irbpp_unpack_observations": (c_i32, [c_void_p, c_i32, c_i32, c_void_p, c_i64, c_void_p]),
    "irbpp_sample_point_clouds": (c_i32, [c_void_p, c_i32, c_i32, c_void_p, c_i64, c_i32, c_void_p, c_i32, ctypes.c_uint64,
                                          ctypes.c_uint64, c_i32, c_void_p, c_void_p, c_void_p]),
    "irbpp_shape_features": (c_i32, [c_void_p, c_i32, c_i32, c_void_p, c_i64, c_i32, c_void_p, c_i32, ctypes.c_uint64,
                                     ctypes.c_uint64, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_float,
                                     c_void_p, c_void_p, c_void_p]),
    "irbpp_debug_phase_cycles": (c_i32, [c_void_p, c_i32, c_void_p]),
    "irbpp_dqn_scratch_bytes": (c_i64, [c_i32, c_i32]),
    "irbpp_dqn_act": (c_i32, [ctypes.POINTER(IrbppDqnWeights), c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_i32,
                              c_void_p, c_i64, c_i64, c_void_p, c_void_p, c_void_p, c_i64, c_void_p]),
    "irbpp_dqn_order_scratch_bytes": (c_i64, [c_i32, c_i32, c_i32]),
    "irbpp_dqn_order_act": (c_i32, [ctypes.POINTER(IrbppDqnOrderWeights), c_void_p, c_i64, c_i32, c_i32, c_void_p, c_i32,
                                    c_void_p, c_i32, c_void_p, c_i64, c_i64, c_void_p, c_void_p, c_void_p, c_i64, c_void_p]),
    "irbpp_dqn_target": (c_i32, [ctypes.POINTER(IrbppDqnWeights), c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_i32,
                                 c_void_p, c_void_p, c_void_p, c_f64, c_f64, c_f64, c_void_p, c_void_p, c_void_p, c_i64,
                                 c_void_p]),
    "irbpp_dqn_order_target": (c_i32, [ctypes.POINTER(IrbppDqnOrderWeights), c_void_p, c_i64, c_i32, c_i32, c_void_p, c_i32,
                                       c_void_p, c_i32, c_void_p, c_void_p, c_void_p, c_f64, c_f64, c_f64, c_void_p,
                                       c_void_p, c_void_p, c_i64, c_void_p]),
    "irbpp_dqn_log_prob_scratch_bytes": (c_i64, [c_i32, c_i32]),
    "irbpp_dqn_log_prob": (c_i32, [ctypes.POINTER(IrbppDqnWeights), c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p,
                                   c_void_p, c_i32, c_void_p, c_void_p, c_i64, c_void_p]),
    "irbpp_dqn_log_prob_backward": (c_i32, [ctypes.POINTER(IrbppDqnWeights), c_void_p, c_i64, c_i32, c_i32, c_void_p,
                                            c_void_p, c_void_p, c_i32, c_void_p, ctypes.POINTER(IrbppDqnGrads), c_void_p,
                                            c_void_p, c_void_p, c_i64, c_void_p]),
    "irbpp_dqn_order_log_prob_scratch_bytes": (c_i64, [c_i32, c_i32, c_i32]),
    "irbpp_dqn_order_log_prob": (c_i32, [ctypes.POINTER(IrbppDqnOrderWeights), c_void_p, c_i64, c_i32, c_i32, c_void_p,
                                         c_i32, c_void_p, c_void_p, c_i32, c_void_p, c_void_p, c_i64, c_void_p]),
    "irbpp_dqn_order_log_prob_backward": (c_i32, [ctypes.POINTER(IrbppDqnOrderWeights), c_void_p, c_i64, c_i32, c_i32,
                                                  c_void_p, c_i32, c_void_p, c_void_p, c_i32, c_void_p,
                                                  ctypes.POINTER(IrbppDqnOrderGrads), c_void_p, c_void_p, c_void_p, c_i64,
                                                  c_void_p]),
    "irbpp_height_encoder_scratch_bytes": (c_i64, [c_i32]),
    "irbpp_height_encoder_forward": (c_i32, [ctypes.POINTER(IrbppHeightEncoderWeights), c_void_p, c_i64, c_i32, c_void_p,
                                             c_void_p]),
    "irbpp_height_encoder_backward": (c_i32, [ctypes.POINTER(IrbppHeightEncoderWeights), c_void_p, c_i64, c_i32, c_void_p,
                                              ctypes.POINTER(IrbppHeightEncoderGrads), c_void_p, c_i64, c_void_p]),
    "irbpp_replay_init": (c_i32, [ctypes.POINTER(IrbppReplayMemory), c_void_p]),
    "irbpp_replay_append": (c_i32, [ctypes.POINTER(IrbppReplayMemory), c_void_p, c_i64, c_void_p, c_void_p, c_void_p,
                                    c_void_p, ctypes.c_float, c_void_p]),
    "irbpp_replay_sample": (c_i32, [ctypes.POINTER(IrbppReplayMemory), c_void_p, c_i32, c_i32, c_i32, c_f64, c_f64, c_i32,
                                    ctypes.c_uint64, ctypes.c_uint64, c_void_p, ctypes.POINTER(IrbppReplayBatch),
                                    c_void_p, c_void_p]),
    "irbpp_replay_update_priorities": (c_i32, [ctypes.POINTER(IrbppReplayMemory), c_void_p, c_void_p, c_void_p, c_i32,
                                               c_f64, c_void_p, c_void_p]),
}

_LIB = None


class IrbppError(RuntimeError):
    def __init__(self, code, message):
        RuntimeError.__init__(self, "irbpp error %d: %s" % (code, message))
        self.code = code


def load():
    """Load ``libirbpp.so`` (built by ``irbpp_b200.build``); fails loudly when it is missing."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("CUDA library %s not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the library does not export the symbol
        fn.restype = res
        fn.argtypes = args
    if lib.irbpp_abi_version() != ABI_VERSION:
        raise RuntimeError("libirbpp ABI %d != binding %d" % (lib.irbpp_abi_version(), ABI_VERSION))
    _LIB = lib
    return lib


def check(lib, handle, rc):
    if rc != IRBPP_OK:
        msg = lib.irbpp_last_error(handle)
        raise IrbppError(rc, msg.decode() if msg else "?")
