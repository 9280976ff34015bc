"""ctypes binding of liblb200.so (C ABI declared in include/lb200.h).

The product path has NO fallback: if the shared library is missing or a call
fails, an exception is raised.  PyTorch is only used by callers for device
memory and streams; nothing here takes or returns torch types except through
``.data_ptr()`` integers.
"""
import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblb200.so")

c_void_p, c_int, c_int64, c_float, c_double, c_size_t = (
    ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_double, ctypes.c_size_t)

class GemmDesc(ctypes.Structure):
    """lb_gemm_desc of include/lb200.h."""
    _fields_ = [("a0", c_void_p), ("a0_ld", c_int64), ("a0_c", ctypes.c_int32),
                ("a1", c_void_p), ("a1_ld", c_int64), ("a1_c", ctypes.c_int32),
                ("B", ctypes.c_int32), ("H", ctypes.c_int32), ("W", ctypes.c_int32),
                ("taps", ctypes.c_int32),
                ("w", c_void_p), ("w_ld", c_int64),
                ("N", ctypes.c_int32),
                ("bias", c_void_p),
                ("bias2", c_void_p), ("bias2_ld", c_int64),
                ("res", c_void_p), ("res_ld", c_int64),
                ("out", c_void_p), ("out_ld", c_int64),
                ("mode", ctypes.c_int32),
                ("ln_stats", c_void_p), ("ln_parts", ctypes.c_int32),
                ("ln_csum", c_void_p), ("ln_bias", c_void_p), ("ln_eps", c_float),
                ("stats_out", c_void_p), ("stats_parts", ctypes.c_int32)]


class AttnDesc(ctypes.Structure):
    """lb_attn_desc of include/lb200.h."""
    _fields_ = [("q", c_void_p), ("q_ld", c_int64), ("q_col0", ctypes.c_int32),
                ("k", c_void_p), ("k_ld", c_int64), ("k_col0", ctypes.c_int32),
                ("v", c_void_p), ("v_ld", c_int64), ("v_col0", ctypes.c_int32),
                ("out", c_void_p), ("out_ld", c_int64),
                ("B", ctypes.c_int32), ("heads", ctypes.c_int32), ("Sq", ctypes.c_int32), ("Skv", ctypes.c_int32),
                ("head_dim", ctypes.c_int32), ("scale", c_float)]


c_int32 = ctypes.c_int32


class _NormOp(ctypes.Structure):
    _fields_ = [("x", c_void_p), ("ld_x", c_int64), ("rows", c_int64), ("B", c_int32), ("C", c_int32),
                ("groups", c_int32), ("silu", c_int32), ("eps", c_float), ("gamma", c_void_p), ("beta", c_void_p),
                ("out", c_void_p), ("ld_out", c_int64), ("workspace", c_void_p)]


class _EmbedOp(ctypes.Structure):
    _fields_ = [("text_embeds", c_void_p), ("time_ids", c_void_p), ("B", c_int32), ("dim_t", c_int32),
                ("pooled", c_int32), ("dim_a", c_int32), ("temb_in", c_void_p), ("add_in", c_void_p)]


class _LinOp(ctypes.Structure):
    _fields_ = [("x", c_void_p), ("ldx", c_int64), ("M", c_int32), ("K", c_int32), ("w", c_void_p), ("ldw", c_int64),
                ("bias", c_void_p), ("addend", c_void_p), ("ldadd", c_int64), ("act_in", c_int32),
                ("act_out", c_int32), ("out", c_void_p), ("ldo", c_int64), ("N", c_int32)]


class _ConvOp(ctypes.Structure):
    _fields_ = [("x", c_void_p), ("ld_x", c_int64), ("B", c_int32), ("Cin", c_int32), ("H", c_int32), ("W", c_int32),
                ("w", c_void_p), ("bias", c_void_p), ("Cout", c_int32), ("out", c_void_p), ("ld_out", c_int64),
                ("act", c_int32), ("in_scale", c_float)]


class _ResampleOp(ctypes.Structure):
    _fields_ = [("x", c_void_p), ("ld_x", c_int64), ("B", c_int32), ("H", c_int32), ("W", c_int32), ("C", c_int32),
                ("out", c_void_p), ("ld_out", c_int64), ("Ho", c_int32), ("Wo", c_int32)]


class _AuxOp(ctypes.Structure):
    _fields_ = [("x", c_void_p), ("ld_x", c_int64), ("w", c_void_p), ("bias", c_void_p), ("out", c_void_p),
                ("ld_out", c_int64), ("n", c_int64), ("B", c_int32), ("C", c_int32)]


class _PatchOp(ctypes.Structure):
    _fields_ = [("x", c_void_p), ("ld_x", c_int64), ("H", c_int32), ("W", c_int32), ("C", c_int32), ("k", c_int32),
                ("stride", c_int32), ("pad", c_int32), ("out", c_void_p), ("ld_out", c_int64), ("f", c_float * 6)]


class _OpUnion(ctypes.Union):
    _fields_ = [("gemm", GemmDesc), ("attn", AttnDesc), ("norm", _NormOp), ("embed", _EmbedOp), ("lin", _LinOp),
                ("conv", _ConvOp), ("resample", _ResampleOp), ("aux", _AuxOp), ("patch", _PatchOp)]


class Op(ctypes.Structure):
    """lb_op of include/lb200.h."""
    _fields_ = [("kind", c_int32), ("dtype", c_int32), ("u", _OpUnion)]


GEMM_STATIC_W = 0x100     # lb_gemm_desc.mode flag (include/lb200.h: LB_GEMM_STATIC_W)
GEMM_RELU = 0x200         # LB_GEMM_RELU
GEMM_TILE_BOX = 0x400     # LB_GEMM_TILE_BOX: force the pixel-box M tiling
GEMM_TILE_RUNS = 0x800    # LB_GEMM_TILE_RUNS: force the pixel-run M tiling
GEMM_BF16 = 0x1000        # LB_GEMM_BF16: bf16 operands, bias, residual and output
GEMM_OUT_F16 = 0x2000     # LB_GEMM_OUT_F16 (with GEMM_BF16): fp16 output
GEMM_D2S2 = 0x4000        # LB_GEMM_D2S2: nearest-2x upsample + 3x3 conv as one GEMM, depth-to-space store
DTYPE_F16, DTYPE_BF16 = 0, 1    # LB_DTYPE_F16 / LB_DTYPE_BF16: lb_op.dtype and the trailing dtype arguments
(OP_GEMM, OP_ATTENTION, OP_GROUPNORM, OP_LAYERNORM, OP_EMBED_INPUTS, OP_LINEAR_SMALL, OP_CONV_IN, OP_CONV_OUT,
 OP_UPSAMPLE_NEAREST, OP_IM2COL_S2, OP_LATENT_PREP, OP_SOFTMAX_ROWS, OP_POSTPROCESS_U8, OP_LPIPS_IM2COL_U8, OP_IM2COL,
 OP_MAXPOOL3S2, OP_NHWC_TO_NCHW) = range(1, 18)
CONV_IN_PLAIN, CONV_IN_TINY_VAE = 0, 1     # lb_conv_in's act


# name -> (restype, argtypes); mirrors include/lb200.h one to one
SIGNATURES = {
    "lb_abi_version": (c_int, []),
    "lb_last_error": (ctypes.c_char_p, []),
    "lb_ctx_create": (c_int, [c_int, ctypes.POINTER(c_void_p)]),
    "lb_ctx_destroy": (c_int, [c_void_p]),
    "lb_ctx_sm_count": (c_int, [c_void_p]),
    "lb_slerp_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "lb_slerp_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int64,
                              c_int, c_double, c_void_p, c_void_p, c_void_p]),
    "lb_lerp": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_double, c_void_p]),
    "lb_scale_model_input": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_float, c_void_p]),
    "lb_cfg_euler_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int,
                                  c_float, c_float, c_float, c_float, c_void_p, c_int, c_float, c_void_p]),
    "lb_gemm": (c_int, [c_void_p, ctypes.POINTER(GemmDesc), c_void_p]),
    "lb_gemm_stats_parts": (c_int, [c_void_p, ctypes.POINTER(GemmDesc)]),
    "lb_ctx_error_flag": (c_int, [c_void_p, ctypes.POINTER(c_int)]),
    "lb_program_create": (c_int, [c_void_p, ctypes.POINTER(Op), c_int64, ctypes.POINTER(c_void_p)]),
    "lb_program_run": (c_int, [c_void_p, c_float, c_void_p]),
    "lb_program_num_launches": (c_int64, [c_void_p]),
    "lb_program_is_graph": (c_int, [c_void_p]),
    "lb_program_run_kinds": (c_int, [c_void_p, c_float, ctypes.c_uint32, c_void_p]),
    "lb_program_count_kinds": (c_int64, [c_void_p, ctypes.c_uint32]),
    "lb_program_destroy": (c_int, [c_void_p]),
    "lb_attention": (c_int, [c_void_p, ctypes.POINTER(AttnDesc), c_void_p]),
    "lb_groupnorm_workspace_bytes": (c_size_t, [c_void_p, c_int, c_int, c_int]),
    "lb_groupnorm": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float,
                             c_int, c_void_p, c_int64, c_void_p, c_void_p, c_int]),
    "lb_layernorm": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p, c_void_p, c_float, c_void_p,
                             c_int64, c_void_p]),
    "lb_embed_inputs": (c_int, [c_void_p, c_float, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                c_void_p, c_void_p]),
    "lb_linear_small": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_int64, c_void_p, c_void_p,
                                c_int64, c_int, c_int, c_void_p, c_int64, c_int, c_void_p]),
    "lb_conv_in": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                           c_int64, c_int, c_float, c_void_p, c_int]),
    "lb_conv_out": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                            c_void_p, c_void_p]),
    "lb_upsample_nearest": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_int64, c_int,
                                    c_int, c_void_p, c_int]),
    "lb_im2col_s2": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "lb_latent_prep": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                               c_int]),
    "lb_softmax_rows": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p, c_int64, c_void_p, c_int]),
    "lb_postprocess_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_int]),
    "lb_nhwc_to_nchw": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int64, c_void_p, c_void_p, c_int]),
    "lb_lpips_im2col_u8": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_float),
                                   ctypes.POINTER(c_float), c_void_p, c_int64, c_void_p]),
    "lb_im2col": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "lb_maxpool3s2": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_int64, c_void_p]),
    "lb_lpips_tap_workspace_bytes": (c_size_t, [c_void_p]),
    "lb_lpips_tap": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p, c_int, c_void_p,
                             c_void_p, c_void_p]),
    "lb_frames_lerp_u8": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                  c_void_p]),
}

_lib = None
_lock = threading.Lock()
_ctx = {}


class LB200Error(RuntimeError):
    pass


def load():
    """Load liblb200.so (once).  Raises LB200Error if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise LB200Error(
                f"{LIB_PATH} not found: build it with `python -m latentblending_b200.build` "
                "(there is no CPU or PyTorch fallback for the CUDA hot path)")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)       # AttributeError if the .so lacks a declared symbol
            fn.restype = res
            fn.argtypes = args
        if lib.lb_abi_version() != 3:
            raise LB200Error("liblb200.so ABI version mismatch")
        _lib = lib
    return _lib


def check(status, what):
    if status != 0:
        msg = load().lb_last_error()
        raise LB200Error(f"{what} failed ({status}): {msg.decode() if msg else '?'}")


def ctx(device_index=0):
    """The per-device context handle (created on first use)."""
    lib = load()
    if device_index not in _ctx:
        h = c_void_p()
        check(lib.lb_ctx_create(int(device_index), ctypes.byref(h)), "lb_ctx_create")
        _ctx[device_index] = h
    return _ctx[device_index]


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)
