"""ctypes binding of libb200seg.so (the C ABI declared in include/b200seg.h).

The library is the product: if it is missing or the device is not sm_90 every op raises — there is no
PyTorch/CPU fallback anywhere in this package (SURVEY.md §8b "Errors")."""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_int64, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200seg.so")

F32, F16 = 0, 1
ALGO_AUTO, ALGO_DIRECT, ALGO_TC = 0, 1, 2
ACT_NONE, ACT_RELU, ACT_LRELU = 0, 1, 2

P = c_void_p
I = c_int
L = c_int64
F = c_float

# name -> argtypes (restype is int unless listed in _RESTYPES); mirrors include/b200seg.h 1:1
_PROTOS = {
    "b200seg_version": [],
    "b200seg_strerror": [I],
    "b200seg_last_cuda_error": [],
    "b200seg_check_device": [],
    "b200seg_dice_ce_fwd": [P, I, L, L, L, P, I, P, I, L, I, F, F, P, P, P],
    "b200seg_dice_ce_bwd": [P, I, L, L, L, P, I, P, I, L, I, F, F, P, P, P, P],
    "b200seg_instnorm_stats": [P, I, I, I, I, L, I, P, P],
    "b200seg_instnorm_apply": [P, I, I, I, P, F, I, P, I, I, I, L, I, P],
    "b200seg_instnorm_bwd_reduce": [P, I, I, P, I, I, I, P, F, I, P, I, I, P, I, L, I, P],
    "b200seg_instnorm_bwd_apply": [P, I, I, P, I, I, I, P, P, F, P, I, I, P, I, I, I, L, I, P],
    "b200seg_pack_weight": [P, I, I, I, P, I, I, I, I, I, P],
    "b200seg_pack_chunk_elems": [],
    "b200seg_pack_tile_ci": [I],
    "b200seg_pack_weights_multi": [P, P, I, P],
    "b200seg_conv3d_algo": [I, I, I, I, I, I, I],
    "b200seg_conv3d_fwd": [P, I, I, P, F, I, P, P, P, I, I, P, I, I, P, P, I, I, P, F, I,
                           I, I, I, I, I, I, I, I, I, I, I, P],
    "b200seg_conv3d_wgrad_workspace": [I, I, I, I, I, I, I, I, I, I, I, I, I, I, I, I, I],
    "b200seg_conv3d_wgrad": [P, I, I, P, F, I, P, I, I, P, P, I, I, I, I, I, I, I, I, I, I, I, P, ctypes.c_size_t, P],
    "b200seg_conv3d_fwd_pc": [P, I, I, P, I, P, P, P, I, I, P, I, I, P, I, I, I, I, I, I, I, I, I, I, I, P],
    "b200seg_conv3d_wgrad_pc_workspace": [I, I, I, I, I, I, I, I, I, I, I, I, I, I, I, I, I],
    "b200seg_conv3d_wgrad_pc": [P, I, I, P, I, P, I, I, P, P, I, I, I, I, I, I, I, I, I, I, I, P, ctypes.c_size_t, P],
    "b200seg_batchnorm_fwd_fold": [P, I, I, c_double, P, P, P, P, P, F, F, I, P, P, P],
    "b200seg_batchnorm_apply": [P, I, I, I, P, I, P, I, I, L, I, P],
    "b200seg_batchnorm_bwd_reduce": [P, I, I, P, I, I, I, P, I, P, L, I, P, P],
    "b200seg_batchnorm_bwd_fold": [P, c_double, P, P, I, I, P, P, P, P],
    "b200seg_batchnorm_bwd_apply": [P, I, I, P, I, I, I, P, I, P, P, I, I, P, I, I, L, I, P],
    "b200seg_maxpool3d_fwd": [P, I, I, P, I, I, P, P, I, I, I, I, I, I, I, I, I, P],
    "b200seg_maxpool3d_bwd": [P, I, I, P, P, I, I, I, I, I, I, I, I, I, I, I, P],
    "b200seg_upsample_trilinear_fwd": [P, I, I, P, I, I, P, I, I, I, I, I, I, I, I, I, P],
    "b200seg_upsample_trilinear_bwd": [P, I, I, P, I, I, I, I, I, I, I, I, I, I, I, I, P],
    "b200seg_copy_channels": [P, I, I, I, P, I, I, I, I, L, I, P],
    "b200seg_dwconv3d_fwd": [P, I, I, P, F, I, P, I, P, I, I, P, I, I, I, I, I, I, I, I, I, P],
    "b200seg_dwconv3d_wgrad": [P, I, I, P, F, I, P, I, I, P, I, I, I, I, I, I, I, I, I, I, P],
    "b200seg_space_to_depth": [P, P, I, I, I, I, I, I, I, I, I, I, P],
    "b200seg_mapgen_workspace": [I, L, I, I],
    "b200seg_mapgen_fwd": [P, I, I, P, I, I, P, P, P, I, L, I, I, I, P],
    "b200seg_mapgen_bwd": [P, I, I, P, I, I, P, P, P, P, I, I, P, I, I, I, I, L, I, I, I, P],
    "b200seg_se_gate_fwd": [P, L, P, P, P, P, P, P, P, I, I, I, P],
    "b200seg_se_gate_bwd": [P, P, P, P, P, P, P, P, P, P, P, I, I, I, P],
    "b200seg_channel_scale_fwd": [P, P, P, I, L, I, I, P],
    "b200seg_channel_scale_bwd_workspace": [I, L, I],
    "b200seg_channel_scale_bwd_reduce": [P, P, P, P, I, L, I, I, P],
    "b200seg_channel_scale_bwd_apply": [P, P, P, P, I, L, I, I, P],
    "b200seg_layernorm_fwd": [P, P, P, P, P, I, I, F, I, P],
    "b200seg_layernorm_bwd": [P, P, P, P, P, P, P, I, I, I, P],
    "b200seg_gelu": [P, P, P, L, I, P],
    "b200seg_mhsa": [P, P, P, P, I, I, I, I, F, I, P],
    "b200seg_resblock_out_fwd": [P, I, P, P, I, I, P, F, I, P, I, I, L, I, I, P],
    "b200seg_resblock_out_bwd_reduce": [P, I, P, I, P, I, P, P, I, I, P, F, I, P, P, I, L, I, I, P],
    "b200seg_window_attn_workspace": [I, I, I, I, I, P],
    "b200seg_window_attn_fwd": [P, P, P, P, P, I, I, I, I, I, I, P, P, I, P],
    "b200seg_window_attn_bwd": [P, P, P, P, P, P, P, P, P, P, I, I, I, I, I, I, P, P, I, P],
    "b200seg_swin_merge": [P, P, I, I, I, I, I, I, I, I, P],
    "b200seg_attention_fwd": [P, P, P, I, I, I, I, I, P],
    "b200seg_attention_bwd": [P, P, P, P, P, P, I, I, I, I, I, P],
    "b200seg_optim_chunk_elems": [],
    "b200seg_grads_nonfinite": [P, P, I, P, P],
    "b200seg_adamw_ema_step": [P, P, I, F, F, F, F, F, F, P, P, P, P],
    "b200seg_softmax_accumulate": [P, I, L, L, L, P, P, I, I, I, I, I, I, I, I, I, I, I, P],
    "b200seg_normalize_argmax": [P, P, P, I, I, L, P],
    "b200seg_dice_metric": [P, I, P, I, L, I, P, P],
    "b200seg_surface_distance_workspace": [I, I, I, I],
    "b200seg_surface_distance": [P, I, P, I, I, I, I, I, c_double, c_double, c_double, c_double, P, P, P, P,
                                 ctypes.c_size_t, P],
    "b200seg_aug_resample": [P, P, I, I, P, P, P, P, P, P, I, P, P, I, P, I, P],
    "b200seg_aug_pointwise": [P, P, I, L, I, P, P, P, P, P, ctypes.c_uint64, P],
    "b200seg_aug_gaussian_blur": [P, P, I, I, I, I, P, I, P, I, P],
    "b200seg_attn_gate_fwd": [P, I, P, P, I, I, F, P, P, P, I, I, P, I, L, I, I, I, P],
    "b200seg_attn_gate_bwd": [P, I, I, P, I, I, P, I, P, P, P, F, P, P, P, P, P, I, L, I, I, I, P],
    "b200seg_biattn_workspace": [I, L, I, I],
    "b200seg_biattn_fwd": [P, I, I, P, I, I, P, I, P, I, I, P, I, I, P, I, I, P, P, I, L, I, I, I, F, I, P],
    "b200seg_biattn_bwd": [P, I, I, P, I, I, P, I, P, I, I, P, I, I, P, P, I, I, P, I, I, P, I, I, P, I, I,
                           P, I, P, I, I, P, I, L, I, I, I, F, I, P],
}
_RESTYPES = {"b200seg_strerror": c_char_p, "b200seg_last_cuda_error": c_char_p,
             "b200seg_conv3d_wgrad_workspace": ctypes.c_size_t, "b200seg_conv3d_wgrad_pc_workspace": ctypes.c_size_t, "b200seg_biattn_workspace": ctypes.c_size_t,
             "b200seg_mapgen_workspace": ctypes.c_size_t,
             "b200seg_channel_scale_bwd_workspace": ctypes.c_size_t, "b200seg_window_attn_workspace": ctypes.c_size_t,
             "b200seg_surface_distance_workspace": ctypes.c_size_t}

EXPORTED_SYMBOLS = tuple(_PROTOS)

_lib = None


class B200SegError(RuntimeError):
    pass


def load():
    """Load the shared library (once). Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200SegError(
                "libb200seg.so not found at %s — run `python __graft_entry__.py build` "
                "(there is no fallback path)" % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, argtypes in _PROTOS.items():
            fn = getattr(lib, name)
            fn.argtypes = argtypes
            fn.restype = _RESTYPES.get(name, c_int)
        _lib = lib
    return _lib


def check(rc, what):
    if rc != 0:
        lib = load()
        msg = lib.b200seg_strerror(rc).decode()
        if rc == -3:
            msg += " (" + lib.b200seg_last_cuda_error().decode() + ")"
        raise B200SegError("%s failed: %s" % (what, msg))


# kernels launched per entry point (dice fwd = reduce + finalize; its memset is not ours)
_KERNELS = {"b200seg_dice_ce_fwd": 2, "b200seg_biattn_fwd": 2, "b200seg_window_attn_bwd": 2, "b200seg_attention_bwd": 3, "b200seg_adamw_ema_step": 2, "b200seg_biattn_bwd": 2,
            "b200seg_mapgen_fwd": 2, "b200seg_channel_scale_bwd_reduce": 2, "b200seg_attn_gate_fwd": 2, "b200seg_attn_gate_bwd": 2}
launch_count = 0


def call(name, *args):
    """Invoke an int-returning entry point and raise on a non-zero code."""
    global launch_count
    check(getattr(load(), name)(*args), name)
    launch_count += _KERNELS.get(name, 1)
