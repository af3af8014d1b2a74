"""ctypes binding of include/tdmpc2_b200.h (the stub INTEGRATION.md refers to).

Loading fails loudly: there is no CPU or eager-PyTorch fallback for the planner.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TDMPC2_B200_LIB") or os.path.join(HERE, "libtdmpc2_b200.so")
MAX_ENC_LAYERS = 8
ENGINE_TCGEN05, ENGINE_SIMT = 0, 1     # tdmpc2_engine
Q_ALL, Q_MIN, Q_AVG = 0, 1, 2   # tdmpc2_q_return
ABI_VERSION = 9            # TDMPC2_B200_ABI_VERSION of include/tdmpc2_b200.h this binding was written against

# every symbol include/tdmpc2_b200.h declares
SYMBOLS = [
    "tdmpc2_abi_version", "tdmpc2_last_error", "tdmpc2_planner_create", "tdmpc2_planner_destroy",
    "tdmpc2_planner_packed_bytes", "tdmpc2_planner_workspace_bytes", "tdmpc2_planner_bind",
    "tdmpc2_planner_set_engine", "tdmpc2_planner_set_passes", "tdmpc2_pack_weights", "tdmpc2_plan_prologue",
    "tdmpc2_pixel_encoder_create", "tdmpc2_pixel_encoder_destroy", "tdmpc2_pixel_encoder_workspace_bytes", "tdmpc2_pixel_encode", "tdmpc2_plan_iter", "tdmpc2_plan_iter_rng", "tdmpc2_debug_rng",
    "tdmpc2_plan_epilogue", "tdmpc2_plan_get_state", "tdmpc2_estimate_value", "tdmpc2_debug_layer",
    "tdmpc2_planner_layer_count", "tdmpc2_planner_launch_count", "tdmpc2_planner_set_profile",
    "tdmpc2_planner_target_q_bytes", "tdmpc2_planner_bind_target_q", "tdmpc2_pack_target_q",
    "tdmpc2_wm_encode", "tdmpc2_wm_next", "tdmpc2_wm_reward", "tdmpc2_wm_termination", "tdmpc2_wm_pi", "tdmpc2_wm_q",
    "tdmpc2_td_target", "tdmpc2_pi_loss_tape_bytes", "tdmpc2_pi_loss_workspace_bytes", "tdmpc2_pi_loss_forward",
    "tdmpc2_pi_loss_backward", "tdmpc2_wm_loss_tape_bytes", "tdmpc2_wm_loss_workspace_bytes", "tdmpc2_wm_loss_forward",
    "tdmpc2_wm_loss_backward", "tdmpc2_pixel_encode_tape_bytes",
    "tdmpc2_pixel_backward_workspace_bytes", "tdmpc2_pixel_encode_backward", "tdmpc2_buffer_sample",
    "tdmpc2_model_file_open", "tdmpc2_model_file_close", "tdmpc2_model_file_dims", "tdmpc2_model_file_device_bytes",
    "tdmpc2_model_file_upload", "tdmpc2_plan_draws", "tdmpc2_act_scratch_bytes", "tdmpc2_act",
]


class Dims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "num_envs", "num_samples", "num_pi_trajs", "num_elites", "horizon", "iterations", "obs_dim",
        "action_dim", "latent_dim", "mlp_dim", "enc_dim", "num_enc_layers", "task_dim", "num_tasks",
        "num_q", "num_bins", "simnorm_dim", "episodic")] + [(n, C.c_float) for n in (
        "temperature", "min_std", "max_std", "log_std_min", "log_std_dif")]


class Linear(C.Structure):
    _fields_ = [("weight", C.c_void_p), ("bias", C.c_void_p), ("ln_weight", C.c_void_p), ("ln_bias", C.c_void_p)]


class Weights(C.Structure):
    _fields_ = [("num_enc", C.c_int32), ("enc", Linear * MAX_ENC_LAYERS), ("dynamics", Linear * 3),
                ("reward", Linear * 3), ("pi", Linear * 3), ("qs", Linear * 3),
                ("task_emb", C.c_void_p), ("action_masks", C.c_void_p), ("discount_pow", C.c_void_p),
                ("bins", C.c_void_p), ("termination", Linear * 3)]


class PixelDims(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("in_channels", "num_channels", "simnorm_dim")]


class ConvWeights(C.Structure):
    _fields_ = [("weight", C.c_void_p * 4), ("bias", C.c_void_p * 4)]


class ConvGrads(C.Structure):       # tdmpc2_conv_grads: .grad of _encoder.rgb.{2,4,6,8}.{weight,bias}
    _fields_ = [("weight", C.c_void_p * 4), ("bias", C.c_void_p * 4)]


class PiGrads(C.Structure):
    _fields_ = [("weight", C.c_void_p * 3), ("bias", C.c_void_p * 3), ("ln_weight", C.c_void_p * 2),
                ("ln_bias", C.c_void_p * 2), ("task_emb", C.c_void_p)]


class LinearGrad(C.Structure):
    _fields_ = [("weight", C.c_void_p), ("bias", C.c_void_p), ("ln_weight", C.c_void_p), ("ln_bias", C.c_void_p)]


class WmGrads(C.Structure):
    _fields_ = [("num_enc", C.c_int32), ("enc", LinearGrad * MAX_ENC_LAYERS), ("dynamics", LinearGrad * 3),
                ("reward", LinearGrad * 3), ("termination", LinearGrad * 3), ("qs", LinearGrad * 3), ("task_emb", C.c_void_p)]


class WmLossCoefs(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("consistency", "reward", "value", "termination", "rho", "vmin", "vmax", "bin_size")]


class BufferField(C.Structure):    # tdmpc2_buffer_field: one field of a Buffer.sample gather
    _fields_ = [("storage", C.c_void_p), ("out", C.c_void_p), ("row_bytes", C.c_int64), ("first_step", C.c_int32),
                ("steps", C.c_int32), ("host", C.c_int32)]


class ActArgs(C.Structure):       # tdmpc2_act_args
    _fields_ = [("obs", C.c_void_p), ("frames", C.c_void_p), ("task", C.c_void_p), ("t0", C.c_void_p), ("eval_mode", C.c_int32),
                ("rng_state", C.c_void_p), ("prev_mean", C.c_void_p), ("action_out", C.c_void_p), ("grid_base", C.c_void_p)]


class CabiError(RuntimeError):
    pass


_lib = None


def load():
    """dlopen the library and type its entry points.  Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise CabiError(
            f"{LIB_PATH} is missing: build it with `python -m tdmpc2_b200.build` "
            "(the planner has no CPU / PyTorch fallback)")
    lib = C.CDLL(LIB_PATH)
    for s in SYMBOLS:
        if not hasattr(lib, s):
            raise CabiError(f"{LIB_PATH} does not export {s}")
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    lib.tdmpc2_abi_version.restype = C.c_int
    if lib.tdmpc2_abi_version() != ABI_VERSION:
        raise CabiError(f"{LIB_PATH} has ABI version {lib.tdmpc2_abi_version()}, this binding needs {ABI_VERSION}: rebuild it")
    lib.tdmpc2_last_error.restype = C.c_char_p
    lib.tdmpc2_planner_create.argtypes = [C.POINTER(Dims), C.POINTER(vp)]
    lib.tdmpc2_planner_destroy.argtypes = [vp]
    lib.tdmpc2_planner_destroy.restype = None
    lib.tdmpc2_planner_packed_bytes.argtypes = [vp, C.POINTER(C.c_size_t)]
    lib.tdmpc2_planner_workspace_bytes.argtypes = [vp, C.POINTER(C.c_size_t)]
    lib.tdmpc2_planner_bind.argtypes = [vp, vp, vp]
    lib.tdmpc2_planner_set_engine.argtypes = [vp, C.c_int]
    lib.tdmpc2_planner_set_passes.argtypes = [vp, C.c_int]
    lib.tdmpc2_pack_weights.argtypes = [vp, C.POINTER(Weights), vp]
    lib.tdmpc2_plan_prologue.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.tdmpc2_pixel_encoder_create.argtypes = [C.POINTER(PixelDims), C.POINTER(vp)]
    lib.tdmpc2_pixel_encoder_destroy.argtypes = [vp]
    lib.tdmpc2_pixel_encoder_destroy.restype = None
    lib.tdmpc2_pixel_encoder_workspace_bytes.argtypes = [vp, C.POINTER(C.c_size_t)]
    lib.tdmpc2_pixel_encode.argtypes = [vp, vp, C.POINTER(ConvWeights), vp, vp, vp, i64, vp, vp, vp]
    lib.tdmpc2_plan_iter.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.tdmpc2_plan_iter_rng.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp]
    lib.tdmpc2_debug_rng.argtypes = [vp, C.c_uint32, C.c_uint64, C.c_int, vp, vp]
    lib.tdmpc2_plan_epilogue.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.tdmpc2_plan_get_state.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.tdmpc2_estimate_value.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    lib.tdmpc2_debug_layer.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, vp, vp]
    lib.tdmpc2_planner_layer_count.argtypes = [vp]
    lib.tdmpc2_planner_set_profile.argtypes = [vp, vp]
    lib.tdmpc2_planner_launch_count.argtypes = [vp]
    lib.tdmpc2_planner_launch_count.restype = i64
    lib.tdmpc2_planner_target_q_bytes.argtypes = [vp, C.POINTER(C.c_size_t)]
    lib.tdmpc2_planner_bind_target_q.argtypes = [vp, vp]
    lib.tdmpc2_pack_target_q.argtypes = [vp, C.POINTER(Linear), vp]
    lib.tdmpc2_wm_encode.argtypes = [vp, vp, vp, C.c_int, vp, vp]
    lib.tdmpc2_wm_next.argtypes = [vp, vp, vp, vp, C.c_int, vp, vp]
    lib.tdmpc2_wm_reward.argtypes = [vp, vp, vp, vp, C.c_int, vp, vp]
    lib.tdmpc2_wm_termination.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp]
    lib.tdmpc2_wm_pi.argtypes = [vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]
    lib.tdmpc2_wm_q.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    lib.tdmpc2_td_target.argtypes = [vp, vp, vp, vp, vp, vp, vp, C.c_int, vp, vp]
    lib.tdmpc2_pi_loss_tape_bytes.argtypes = [vp, C.c_int, C.POINTER(C.c_size_t)]
    lib.tdmpc2_pi_loss_workspace_bytes.argtypes = [vp, C.c_int, C.POINTER(C.c_size_t)]
    lib.tdmpc2_pi_loss_forward.argtypes = [vp, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]
    lib.tdmpc2_pi_loss_backward.argtypes = [vp, C.POINTER(Weights), vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, vp, C.c_float,
                                            C.c_float, C.POINTER(PiGrads), vp, vp]
    lib.tdmpc2_wm_loss_tape_bytes.argtypes = [vp, C.c_int, C.c_int, C.POINTER(C.c_size_t)]
    lib.tdmpc2_wm_loss_workspace_bytes.argtypes = [vp, C.c_int, C.c_int, C.POINTER(C.c_size_t)]
    lib.tdmpc2_wm_loss_forward.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp]
    lib.tdmpc2_wm_loss_backward.argtypes = [vp, C.POINTER(Weights), vp, vp, vp, vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp,
                                            vp, vp, C.POINTER(WmLossCoefs), C.POINTER(WmGrads), vp, vp, vp]
    lib.tdmpc2_pixel_encode_tape_bytes.argtypes = [vp, i64, C.POINTER(C.c_size_t)]
    lib.tdmpc2_pixel_backward_workspace_bytes.argtypes = [vp, i64, C.POINTER(C.c_size_t)]
    lib.tdmpc2_pixel_encode_backward.argtypes = [vp, C.POINTER(ConvWeights), vp, vp, vp, i64, vp, vp, vp, C.POINTER(ConvGrads),
                                                 vp, vp]
    lib.tdmpc2_buffer_sample.argtypes = [C.POINTER(BufferField), C.c_int, i64, vp, vp, i64, vp, vp, C.c_int, C.c_int, vp]
    lib.tdmpc2_model_file_open.argtypes = [C.c_char_p, C.POINTER(vp)]
    lib.tdmpc2_model_file_close.argtypes = [vp]
    lib.tdmpc2_model_file_close.restype = None
    lib.tdmpc2_model_file_dims.argtypes = [vp, C.POINTER(Dims), C.POINTER(PixelDims), C.POINTER(i32)]
    lib.tdmpc2_model_file_device_bytes.argtypes = [vp, C.POINTER(Dims), C.POINTER(C.c_size_t)]
    lib.tdmpc2_model_file_upload.argtypes = [vp, C.POINTER(Dims), vp, C.POINTER(Weights), C.POINTER(ConvWeights), C.POINTER(vp), vp]
    lib.tdmpc2_plan_draws.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp, vp, vp]
    lib.tdmpc2_act_scratch_bytes.argtypes = [vp, vp, C.POINTER(C.c_size_t)]
    lib.tdmpc2_act.argtypes = [vp, vp, vp, C.POINTER(ConvWeights), C.POINTER(ActArgs), vp, vp]
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        msg = load().tdmpc2_last_error()
        raise CabiError(f"tdmpc2_b200 C-ABI call failed ({rc}): {msg.decode() if msg else '?'}")
