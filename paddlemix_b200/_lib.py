"""ctypes binding of libb200mix.so (the C ABI declared in include/b200mix.h).

This is the only way the Python host code reaches the device. There is no fallback: if the shared library is
missing, importing this module raises, and every entry point returns B200MIX_ERR_NO_DEVICE without an sm_90 GPU.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200MIX_LIB selects an alternative build of the same library (A/B kernel experiments); never a different backend
LIB_PATH = os.environ.get("B200MIX_LIB") or os.path.join(_HERE, "libb200mix.so")


class B200MixError(RuntimeError):
    pass


class Epilogue(Structure):
    """Mirror of `b200mix_epilogue` (include/b200mix.h)."""

    _fields_ = [
        ("bias", c_void_p),
        ("row_add", c_void_p),
        ("row_gate", c_void_p),
        ("ld_row", c_int64),
        ("rows_per_group", c_int64),
        ("residual", c_void_p),
        ("ldr", c_int64),
        ("act", c_int32),
        ("glu", c_int32),
        ("out_fp32", c_int32),
        ("out_scale", c_float),
        ("residual_row_mod", c_int64),
        ("stats_out", c_void_p),
        ("ln_stats", c_void_p),
        ("ln_colsum", c_void_p),
        ("ln_rms", c_int32),
        ("ln_eps", c_float),
    ]


ACT_NONE, ACT_SILU, ACT_GELU_ERF, ACT_GELU_TANH, ACT_QUICK_GELU = 0, 1, 2, 3, 4
GLU_NONE, GLU_GEGLU, GLU_SWIGLU = 0, 1, 2

# name -> argtypes; every function returns int except the two string getters.
SIGNATURES = {
    "b200mix_init": [c_int],
    "b200mix_num_sms": [],
    "b200mix_zero_bytes": [c_void_p, c_int64, c_void_p],
    "b200mix_nccl_load": [c_char_p],
    "b200mix_nccl_version": [],
    "b200mix_nccl_unique_id": [c_void_p],
    "b200mix_comm_init": [POINTER(c_void_p), c_int32, c_int32, c_void_p],
    "b200mix_allgather_latents": [c_void_p, c_void_p, c_void_p, c_int64, c_void_p],
    "b200mix_comm_destroy": [c_void_p],
    "b200mix_linear": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int64,
                       POINTER(Epilogue), c_void_p],
    "b200mix_linear_batched": [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int64,
                               c_int64, c_int64, POINTER(Epilogue), c_int64, c_void_p],
    "b200mix_patchify": [c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int32, c_void_p],
    "b200mix_unpatchify": [c_void_p, c_void_p, c_int32, c_int64, c_int64, c_int64, c_int64, c_int32, c_void_p],
    "b200mix_conv3x3": [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int32,
                        POINTER(Epilogue), c_void_p],
    "b200mix_conv3x3_up2x": [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64,
                             POINTER(Epilogue), c_void_p],
    "b200mix_conv3x3_small_cin": [c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64,
                                  c_int64, c_void_p],
    "b200mix_sdpa": [c_void_p, c_void_p, c_void_p, c_void_p] + [c_int64] * 6 + [c_int64] * 12 +
                    [c_float, c_int32, c_void_p, c_int32, c_void_p, c_void_p, c_int32, c_int64, c_int64, c_int64, c_void_p],
    "b200mix_groupnorm_nhwc": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
                               c_int64, c_int64, c_int32, c_float, c_int32, c_void_p],
    "b200mix_layernorm": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                          c_int64, c_int64, c_int64, c_int64, c_float, c_int32, c_void_p],
    "b200mix_softmax_rows": [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_float, c_void_p],
    "b200mix_timestep_embedding": [c_void_p, c_void_p, c_int32, c_int64, c_int64, c_int64, c_int64, c_int32, c_float,
                                   c_float, c_float, c_void_p],
    "b200mix_activation": [c_void_p, c_void_p, c_int64, c_int32, c_int32, c_int32, c_void_p],
    "b200mix_upsample_nearest2x_nhwc": [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p],
    "b200mix_concat_channels": [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p],
    "b200mix_nchw_to_nhwc": [c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int64, c_int64, c_void_p],
    "b200mix_nhwc_to_nchw": [c_void_p, c_void_p, c_int32, c_int64, c_int64, c_int64, c_int64, c_void_p],
    "b200mix_add_residual_nhwc": [c_void_p, c_void_p, c_int32, c_int32, c_void_p, c_int64, c_int64, c_int64, c_int64,
                                  c_void_p],
    "b200mix_ddim_step": [c_void_p, c_void_p, c_int32, c_float, c_void_p, c_void_p, c_int64, c_float, c_float,
                          c_float, c_float, c_void_p],
    "b200mix_ddim_step_ex": [c_void_p, c_void_p, c_int32, c_float, c_void_p, c_void_p, c_int64, c_float, c_float,
                             c_float, c_float, c_int32, c_float, c_void_p],
    "b200mix_lcm_step": [c_void_p, c_void_p, c_int32, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float,
                         c_float, c_float, c_float, c_float, c_float, c_int32, c_float, c_void_p],
    "b200mix_cfg_rescale_ratio": [c_void_p, c_void_p, c_int32, c_float, c_void_p, c_int64, c_int64, c_void_p],
    "b200mix_cfg_combine": [c_void_p, c_void_p, c_int32, c_float, c_void_p, c_float, c_int64, c_void_p, c_int64, c_void_p],
    "b200mix_euler_step": [c_void_p, c_void_p, c_int32, c_float, c_void_p, c_void_p, c_int64, c_float, c_float,
                           c_void_p],
    "b200mix_scale_model_input": [c_void_p, c_void_p, c_int64, c_float, c_void_p],
    "b200mix_dpmpp_2m_step": [c_void_p, c_void_p, c_int32, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_float,
                              c_float, c_float, c_float, c_float, c_float, c_void_p],
    "b200mix_gather_rows": [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p],
    "b200mix_scatter_rows": [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p],
    "b200mix_broadcast_add": [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p],
    "b200mix_head_rmsnorm_inplace": [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_float, c_void_p],
    "b200mix_small_attention": [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64,
                                c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_float, c_void_p],
    "b200mix_patchify3d": [c_void_p, c_int32, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int32, c_void_p],
    "b200mix_unpatchify3d": [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_int32, c_void_p],
    "b200mix_cast": [c_void_p, c_void_p, c_int64, c_int32, c_int32, c_void_p],
    "b200mix_rope_inplace": [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p],
    "b200mix_decode_rope_cache": [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p, c_void_p],
}
STRING_GETTERS = ("b200mix_last_error", "b200mix_version")


def _load():
    if not os.path.exists(LIB_PATH):
        raise B200MixError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(b200mix has no CPU / PyTorch fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = c_int
    for name in STRING_GETTERS:
        getattr(lib, name).restype = c_char_p
        getattr(lib, name).argtypes = []
    lib.b200mix_debug_force_bn.argtypes = [c_int]
    lib.b200mix_debug_force_bn.restype = None
    lib.b200mix_debug_attn_bn64.argtypes = [c_int]
    lib.b200mix_debug_attn_bn64.restype = None
    lib.b200mix_debug_gemm_pair.argtypes = [c_int]
    lib.b200mix_debug_gemm_pair.restype = None
    lib.b200mix_debug_ln_register_only.argtypes = [c_int]
    lib.b200mix_debug_ln_register_only.restype = None
    return lib


lib = _load()


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib.b200mix_last_error().decode("utf-8", "replace")
        raise B200MixError(f"{what} failed with status {rc}: {msg}")
