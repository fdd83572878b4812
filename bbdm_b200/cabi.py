"""ctypes binding of include/bbdm_b200.h (the C-ABI drop-in boundary).

Loading fails LOUDLY: if ``libbbdm_b200.so`` is missing the product path raises -- there is no
eager/PyTorch fallback for the kernels.  ``python -m bbdm_b200.build`` (or
``__graft_entry__.build()``) compiles it in-tree for sm_90a.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import gc
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# BBDM_LIB selects another in-tree build of the same sources (A/B experiments, tools/); the product default is fixed
LIB_PATH = os.environ.get("BBDM_LIB") or os.path.join(_HERE, "libbbdm_b200.so")

ABI_VERSION = 11
OBJ = {"grad": 0, "noise": 1, "ysubx": 2}
RESAMPLE_NONE, RESAMPLE_UP2, RESAMPLE_DOWN2 = 0, 1, 2
RES_NONE, RES_SAME, RES_UP2, RES_DOWN2 = 0, 1, 2, 3
GN_MAX_SLICES = 64
ATTN_HEAD_DIM_RULE = "multiples of 8 up to 128"
ATTN_TC_HEAD_DIMS = (64, 128)            # head sizes bbdm_attention_tc (wgmma) takes; bbdm_attention_split takes the rest
LN_MAX_C = 2048                          # bbdm_layernorm_split / _bwd: C even, <= this


def attn_head_dim_ok(d):
    """True for the head sizes the attention kernels are built for: a multiple of 8 (each head's columns stay
    16-byte aligned in the bf16 operand planes) up to 128 (the flash backward's tiles fit in shared memory)."""
    return d % 8 == 0 and 8 <= d <= 128


def attn_head_dims(be):
    """The attention head sizes backend ``be`` runs natively, as (ok, rule): ok(d) is True for the multiples of 8 up to
    its attn_max_head_dim (128 when it declares none; 256 for CudaBackend) and rule names them for error messages."""
    top = getattr(be, "attn_max_head_dim", 128)
    return (lambda d: d % 8 == 0 and 8 <= d <= top), f"multiples of 8 up to {top}"


def attn_gemm_route(be, d):
    """True when backend ``be`` runs attention heads of width d as GEMMs around a materialised row softmax (one image
    and head at a time): d is above its attn_max_head_dim and it declares attn_gemm_route."""
    return bool(getattr(be, "attn_gemm_route", False)) and d > getattr(be, "attn_max_head_dim", 128)


def attn_pad_route(be, d):
    """True when backend ``be`` runs attention heads of width d on its attention kernels at d rounded up to 8 (the
    heads repacked by prep(heads=...)): d is not a multiple of 8, at most its
    attn_max_head_dim, and it declares attn_pad_heads."""
    return bool(getattr(be, "attn_pad_heads", False)) and d % 8 != 0 and 0 < d <= getattr(be, "attn_max_head_dim", 128)


def pad_heads_width(d):
    """Width dp of a head of width d on the padded-head route: d rounded up to 8."""
    return -(-d // 8) * 8


def pad_heads_scale(d):
    """(dp/d)^(1/4): the factor the padded-head route folds into q and k, so that the kernels' softmax scale dp^-1/2
    (planes) or (dp^-1/4)^2 (fp32 qkv) becomes the reference's d^-1/2."""
    return (pad_heads_width(d) / d) ** 0.25


def gemm_heads_pad(d):
    """Width of a head's zero-padded q/k/v/o slices on the GEMM route: d rounded up to 32 (the channel multiple of the
    tensor-core GEMMs)."""
    return -(-d // 32) * 32


@contextlib.contextmanager
def collector_paused():
    """Collect the dead reference cycles now and keep Python's cycle collector off until the block ends; wraps every
    CUDA-graph capture.  A collection inside a capture can destroy CUDA objects held by dead cycles (a discarded
    model's graphs and their memory pools), and those calls invalidate the capture."""
    was = gc.isenabled()
    gc.collect()
    gc.disable()
    try:
        yield
    finally:
        if was:
            gc.enable()


def layernorm_bwd_workspace(rows, C):
    """floats of bbdm_layernorm_bwd's workspace: one [2, C] partial per 64 rows"""
    return -(-rows // 64) * 2 * C

# every symbol include/bbdm_b200.h declares (tests check the library exports all of them)
SYMBOLS = [
    "bbdm_abi_version", "bbdm_last_error", "bbdm_device_info", "bbdm_check_device_fault",
    "bbdm_bridge_q_sample", "bbdm_bridge_p_sample", "bbdm_bridge_p_sample_dev", "bbdm_nchw_to_nhwc_cat", "bbdm_nhwc_to_nchw",
    "bbdm_gather_rows", "bbdm_linear_f32", "bbdm_gn_stats", "bbdm_prep_operand",
    "bbdm_pack_weight_split", "bbdm_pack_weight_split_padded", "bbdm_pack_weight_split_taps", "bbdm_pack_weight_split_dgrad",
    "bbdm_pack_weight_f32", "bbdm_conv_umma", "bbdm_conv_direct",
    "bbdm_attention", "bbdm_attention_split", "bbdm_attention_tc", "bbdm_conv_umma_geometry", "bbdm_gn_finalize_partials",
    "bbdm_split_grad", "bbdm_conv_wgrad_workspace", "bbdm_conv_wgrad", "bbdm_gn_bwd_reduce", "bbdm_gn_bwd_apply",
    "bbdm_conv_wgrad_direct", "bbdm_attention_bwd", "bbdm_conv_direct_pad", "bbdm_softmax_rows_split", "bbdm_softmax_rows_bwd", "bbdm_vq_nearest", "bbdm_s2d_split", "bbdm_pack_weight_split_both",
    "bbdm_wino_geometry", "bbdm_wino_input", "bbdm_wino_output", "bbdm_wino_pack_weight",
    "bbdm_wino6_geometry", "bbdm_wino6_input", "bbdm_wino6_output", "bbdm_wino6_pack_weight",
    "bbdm_optim_chunk_elems", "bbdm_adam_multi", "bbdm_adam_multi_dev", "bbdm_ema_multi", "bbdm_denorm_to_uint8",
    "bbdm_layernorm_split", "bbdm_geglu_split", "bbdm_attention_cross", "bbdm_conv_stem", "bbdm_spatial_rescale",
    "bbdm_layernorm_bwd", "bbdm_geglu_bwd", "bbdm_attention_cross_bwd",
    "bbdm_attention_pad_heads", "bbdm_attention_unpad_heads",
]


class PSampleCoef(C.Structure):
    _fields_ = [("m_t", C.c_float), ("one_minus_m_t", C.c_float), ("sqrt_var_t", C.c_float),
                ("m_nt", C.c_float), ("one_minus_m_nt", C.c_float), ("c_xt", C.c_float),
                ("sigma_t", C.c_float)]


class PrepArgs(C.Structure):
    _fields_ = [("src1", C.c_void_p), ("c1", C.c_int), ("src2", C.c_void_p), ("c2", C.c_int),
                ("B", C.c_int), ("Hs", C.c_int), ("Ws", C.c_int), ("groups", C.c_int),
                ("mean", C.c_void_p), ("rstd", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
                ("film_scale", C.c_void_p), ("film_shift", C.c_void_p), ("film_stride", C.c_int64),
                ("silu", C.c_int), ("resample", C.c_int),
                ("act_f32", C.c_void_p), ("act_hi", C.c_void_p), ("act_lo", C.c_void_p),
                ("raw_f32", C.c_void_p), ("raw_hi", C.c_void_p), ("raw_lo", C.c_void_p)]


class ConvArgs(C.Structure):
    _fields_ = [("B", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("Cin", C.c_int), ("Cout", C.c_int), ("taps", C.c_int),
                ("a_hi", C.c_void_p), ("a_lo", C.c_void_p), ("w_hi", C.c_void_p), ("w_lo", C.c_void_p),
                ("bias", C.c_void_p),
                ("Cin2", C.c_int),
                ("a2_hi", C.c_void_p), ("a2_lo", C.c_void_p), ("w2_hi", C.c_void_p), ("w2_lo", C.c_void_p),
                ("bias2", C.c_void_p),
                ("residual", C.c_void_p), ("res_mode", C.c_int),
                ("out", C.c_void_p), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p),
                ("passes", C.c_int), ("out_nchw_channels", C.c_int), ("upsample2x", C.c_int),
                ("stats_partial", C.c_void_p), ("weights_per_image", C.c_int), ("operand_f16", C.c_int),
                ("window_origin", C.c_int)]


class WinoInputArgs(C.Structure):
    _fields_ = [("src1", C.c_void_p), ("c1", C.c_int), ("src2", C.c_void_p), ("c2", C.c_int),
                ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("groups", C.c_int),
                ("mean", C.c_void_p), ("rstd", C.c_void_p), ("gamma", C.c_void_p), ("beta", C.c_void_p),
                ("film_scale", C.c_void_p), ("film_shift", C.c_void_p), ("film_stride", C.c_int64),
                ("silu", C.c_int),
                ("v_hi", C.c_void_p), ("v_lo", C.c_void_p), ("raw_hi", C.c_void_p), ("raw_lo", C.c_void_p),
                ("act_hi", C.c_void_p), ("act_lo", C.c_void_p), ("down2", C.c_int)]


class WinoOutputArgs(C.Structure):
    _fields_ = [("m", C.c_void_p), ("inv_wscale", C.c_void_p), ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cout", C.c_int),
                ("bias", C.c_void_p), ("residual", C.c_void_p), ("res_mode", C.c_int),
                ("out", C.c_void_p), ("stats_partial", C.c_void_p), ("up2_phases", C.c_int)]


class BbdmError(RuntimeError):
    pass


_lib = None


def load():
    """dlopen the C-ABI library and declare prototypes.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise BbdmError(
            f"{LIB_PATH} not found: build the sm_90a kernels first (python -m bbdm_b200.build). "
            "bbdm_b200 has no PyTorch/CPU fallback for its kernels.")
    lib = C.CDLL(LIB_PATH)
    vp, i, i64, f = C.c_void_p, C.c_int, C.c_int64, C.c_float
    lib.bbdm_abi_version.restype = i
    lib.bbdm_last_error.restype = C.c_char_p
    lib.bbdm_device_info.argtypes = [C.POINTER(i)] * 3
    lib.bbdm_check_device_fault.argtypes = [vp, C.POINTER(C.c_ulonglong)]
    lib.bbdm_bridge_q_sample.argtypes = [vp, vp, vp, vp, vp, vp, i, i, vp, vp, i, i64, vp]
    lib.bbdm_bridge_p_sample.argtypes = [vp, vp, vp, vp, PSampleCoef, i, i, i, vp, vp, i64, vp]
    lib.bbdm_bridge_p_sample_dev.argtypes = [vp, vp, vp, vp, vp, i, i, i, vp, vp, i64, vp]
    lib.bbdm_nchw_to_nhwc_cat.argtypes = [vp, i, vp, i, i, i, i, vp, vp]
    lib.bbdm_nhwc_to_nchw.argtypes = [vp, i, i, i, i, vp, vp]
    lib.bbdm_gather_rows.argtypes = [vp, i, i, vp, i, vp, vp]
    lib.bbdm_linear_f32.argtypes = [vp, vp, vp, vp, i, i, i, i, i, vp]
    lib.bbdm_gn_stats.argtypes = [vp, i, vp, i, i, i, i, i, f, vp, vp, vp, vp]
    lib.bbdm_prep_operand.argtypes = [C.POINTER(PrepArgs), vp]
    lib.bbdm_pack_weight_split.argtypes = [vp, i, i, i, vp, vp, vp]
    lib.bbdm_pack_weight_split_padded.argtypes = [vp, i, i, i, i, vp, vp, vp]
    lib.bbdm_pack_weight_split_dgrad.argtypes = [vp, i, i, i, vp, vp, vp]
    lib.bbdm_pack_weight_split_taps.argtypes = [vp, i, i, i, vp, vp, vp]
    lib.bbdm_pack_weight_f32.argtypes = [vp, i, i, i, vp, vp]
    lib.bbdm_conv_umma.argtypes = [C.POINTER(ConvArgs), vp]
    lib.bbdm_conv_direct.argtypes = [vp, vp, vp, vp, vp, i, i, i, i, i, i, i, vp]
    lib.bbdm_conv_stem.argtypes = [vp, vp, vp, vp, i, i, i, i, i, vp, vp]
    lib.bbdm_attention.argtypes = [vp, i, i, i, i, i, vp, vp, vp, vp]
    lib.bbdm_conv_umma_geometry.argtypes = [i, i, C.POINTER(i), C.POINTER(i), C.POINTER(i), C.POINTER(i)]
    lib.bbdm_gn_finalize_partials.argtypes = [vp, i, i, vp, i, i, i, i, i, f, vp, vp, vp]
    lib.bbdm_split_grad.argtypes = [vp, i64, i, vp, vp, vp, vp, i64, vp, vp, vp]
    lib.bbdm_conv_wgrad_workspace.argtypes = [i, i, i, i, i, i, C.POINTER(i), C.POINTER(i64)]
    lib.bbdm_conv_wgrad.argtypes = [vp, vp, i64, vp, vp, i, i, i, i, i, i, i, vp, vp, vp]
    lib.bbdm_conv_wgrad_direct.argtypes = [vp, vp, i, i, i, i, i, i, vp, vp, i64, vp]
    lib.bbdm_gn_bwd_reduce.argtypes = [vp, vp, i, i, i, i, i, vp, vp, vp, vp, vp, vp, i64, i, vp, vp, vp]
    lib.bbdm_gn_bwd_apply.argtypes = [vp, vp, i, i, i, i, i, vp, vp, vp, vp, vp, vp, i64, i, vp, vp, vp, vp]
    lib.bbdm_attention_split.argtypes = [vp, vp, i, i, i, i, i, vp, vp, vp, vp]
    lib.bbdm_attention_tc.argtypes = [vp, vp, i, i, i, i, i, vp, vp, vp, vp]
    lib.bbdm_attention_bwd.argtypes = [vp, vp, vp, i, i, i, i, i, vp, vp, vp, vp]
    lib.bbdm_conv_direct_pad.argtypes = [vp, vp, vp, vp, vp, i, i, i, i, i, i, i, i, i, vp]
    lib.bbdm_softmax_rows_split.argtypes = [vp, i64, i64, i64, C.c_float, vp, vp, vp]
    lib.bbdm_softmax_rows_bwd.argtypes = [vp, vp, i64, i64, i64, C.c_float, vp, vp, vp]
    lib.bbdm_vq_nearest.argtypes = [vp, vp, i64, i, i, vp, vp, vp]
    lib.bbdm_s2d_split.argtypes = [vp, i, i, i, i, vp, vp, vp]
    lib.bbdm_pack_weight_split_both.argtypes = [vp, i, i, i, vp, vp, vp, vp, vp]
    lib.bbdm_wino_geometry.argtypes = [i, i, i, C.POINTER(i), C.POINTER(i), C.POINTER(i64), C.POINTER(i)]
    lib.bbdm_wino_input.argtypes = [C.POINTER(WinoInputArgs), vp]
    lib.bbdm_wino_output.argtypes = [C.POINTER(WinoOutputArgs), vp]
    lib.bbdm_wino_pack_weight.argtypes = [vp, i, i, i, vp, vp, vp, vp]
    lib.bbdm_wino6_geometry.argtypes = lib.bbdm_wino_geometry.argtypes
    lib.bbdm_wino6_input.argtypes = lib.bbdm_wino_input.argtypes
    lib.bbdm_wino6_output.argtypes = lib.bbdm_wino_output.argtypes
    lib.bbdm_wino6_pack_weight.argtypes = lib.bbdm_wino_pack_weight.argtypes
    lib.bbdm_denorm_to_uint8.argtypes = [vp, i, i, i, i, i, vp, vp]
    lib.bbdm_spatial_rescale.argtypes = [vp, i, i, i, i, i, vp, vp, i, vp, vp]
    lib.bbdm_layernorm_split.argtypes = [vp, i64, i, vp, vp, f, vp, vp, vp, vp]
    lib.bbdm_geglu_split.argtypes = [vp, i64, i, vp, vp, vp, vp]
    lib.bbdm_attention_cross.argtypes = [vp, vp, vp, vp, i, i, i, i, i, vp, vp, vp, vp]
    lib.bbdm_layernorm_bwd.argtypes = [vp, vp, i64, i, vp, f, vp, vp, vp, vp, vp]
    lib.bbdm_geglu_bwd.argtypes = [vp, vp, i64, i, vp, vp]
    lib.bbdm_attention_cross_bwd.argtypes = [vp, vp, vp, vp, i, i, i, i, i, vp, vp, vp, vp, vp]
    lib.bbdm_attention_pad_heads.argtypes = [vp, i64, i, i, i, i, f, f, f, vp, vp, vp, vp]
    lib.bbdm_attention_unpad_heads.argtypes = lib.bbdm_attention_pad_heads.argtypes
    lib.bbdm_optim_chunk_elems.argtypes = []
    lib.bbdm_adam_multi.argtypes = [vp, vp, vp, vp, vp, vp, i, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double,
                                     C.c_double, i64, vp, C.c_double, vp]
    lib.bbdm_adam_multi_dev.argtypes = [vp, vp, vp, vp, vp, vp, i, vp, vp, vp, vp, C.c_double, C.c_double, C.c_double,
                                         C.c_double, vp, C.c_double, vp]
    lib.bbdm_ema_multi.argtypes = [vp, vp, vp, vp, vp, i, vp, C.c_double, i, vp]
    for s in SYMBOLS:
        fn = getattr(lib, s)
        if s not in ("bbdm_last_error",):
            fn.restype = i
    if lib.bbdm_abi_version() != ABI_VERSION:
        raise BbdmError(f"libbbdm_b200.so ABI {lib.bbdm_abi_version()} != binding ABI {ABI_VERSION}")
    _lib = lib
    return lib


def check(rc: int):
    if rc != 0:
        raise BbdmError(f"bbdm_b200 C-ABI call failed ({rc}): {load().bbdm_last_error().decode()}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream():
    """torch's current stream of the CURRENT device; CudaBackend methods make the tensors' device current first."""
    return torch.cuda.current_stream().cuda_stream


def _device_guarded(fn):
    """Run a backend method with the device of its first CUDA tensor argument current.  The reference's
    single-GPU launcher (main.py --gpu_ids N) moves the model to cuda:N without torch.cuda.set_device, so the
    process default stays device 0: kernels, TMA descriptors, stream and SM-count lookups must all follow the
    tensors, not the default."""
    import functools

    @functools.wraps(fn)
    def wrapper(self, *args, **kw):
        dev = None
        for a in args:
            if isinstance(a, torch.Tensor) and a.is_cuda:
                dev = a.device.index
                break
        if dev is None:
            for a in kw.values():
                if isinstance(a, torch.Tensor) and a.is_cuda:
                    dev = a.device.index
                    break
        if dev is None or dev == torch.cuda.current_device():
            return fn(self, *args, **kw)
        with torch.cuda.device(dev):
            return fn(self, *args, **kw)
    return wrapper


def _guard_all(cls):
    for name, fn in list(vars(cls).items()):
        if callable(fn) and not name.startswith("_") and name not in ("empty", "conv_geometry", "wgrad_workspace", "wino_geometry", "optim_chunk_elems"):
            setattr(cls, name, _device_guarded(fn))
    return cls


# launch counter: every successful C-ABI compute call == >=1 kernel launch of OUR kernels
LAUNCHES = {"n": 0}


def _req(t, dtype=torch.float32):
    assert t.is_cuda and t.is_contiguous() and t.dtype == dtype, (t.device, t.dtype, t.is_contiguous())
    return t


def _pitch(hi_t, lo_t, rows, cols):
    """Row pitch (elements) of a pair of transposed [rows, cols] planes whose rows may be padded."""
    assert hi_t.is_cuda and tuple(hi_t.shape) == (rows, cols) and hi_t.stride(1) == 1, (hi_t.shape, hi_t.stride())
    assert lo_t.shape == hi_t.shape and lo_t.stride() == hi_t.stride(), (hi_t.stride(), lo_t.stride())
    return hi_t.stride(0)


@_guard_all
class CudaBackend:
    """The one product backend: each method is one C-ABI entry point on torch's current stream.
    (tests/ substitute an oracle-backed emulation with the same method set to check the host
    logic on CPU; the product never does.)"""

    name = "sm_90a"
    requires_cuda = True
    # wino_pack_weight / wino_output take inv_wscale: per-tensor power-of-two scales of the Winograd weight planes
    # (a backend without it packs at the fixed 2^8, and the engines call it without a scale)
    wino_tensor_scale = True
    # Winograd output tile sizes: F(4x4,3x3) and F(6x6,3x3) (the wino_* methods' tile argument)
    wino_tiles = (4, 6)
    # conv_umma / conv_wgrad take window_origin: the 2x2 window of taps = 4 at rows/cols -1..0 as well as 0..1 (the
    # UNet's stride-2 conv on a space-to-depth operand and the adjoints of it and of the nearest-2x conv)
    window_origin = True
    # conv_umma / conv_wgrad take channel counts that are multiples of 32 (a backend without this attribute: 64)
    conv_channel_multiple = 32
    # attention / _split / _cross / _bwd / _cross_bwd take head sizes that are multiples of 8 up to this (a backend
    # without this attribute: 128); attention_tc takes 64 and 128 only
    attn_max_head_dim = 256
    # heads wider than attn_max_head_dim run as two conv_umma GEMMs per (image, head) around softmax_rows_split, and
    # train through softmax_rows_split(grad=...), conv_umma and conv_wgrad (a backend without this attribute: not at all)
    attn_gemm_route = True
    # heads up to attn_max_head_dim whose width is not a multiple of 8 run on the attention kernels at the width rounded
    # up to 8, repacked by prep(heads=...) (a backend without this attribute: not at all)
    attn_pad_heads = True

    def __init__(self):
        self.lib = load()

    # -- memory ------------------------------------------------------------------------------
    def empty(self, shape, dtype, device):
        try:
            return torch.empty(shape, dtype=dtype, device=device)
        except torch.OutOfMemoryError:
            # a model and its executor refer to each other, so the buffer pools of a dropped model go back to the
            # allocator only when the cycle collector runs: run it, then try once more
            gc.collect()
            return torch.empty(shape, dtype=dtype, device=device)

    # -- bridge --------------------------------------------------------------------------------
    def q_sample(self, x0, y, noise, t, m_t, var_t, objective, xt_out, obj_out):
        B = x0.shape[0]
        n = x0.numel() // B
        for z in (x0, y, noise, m_t, var_t, xt_out, obj_out):
            _req(z)
        _req(t, torch.int64)
        check(self.lib.bbdm_bridge_q_sample(ptr(x0), ptr(y), ptr(noise), ptr(t), ptr(m_t), ptr(var_t),
                                            m_t.numel(), OBJ[objective], ptr(xt_out), ptr(obj_out), B, n,
                                            stream()))
        LAUNCHES["n"] += 1

    def p_sample(self, x_t, y, eps, noise, coef, objective, clip, is_last, x_out, x0_out):
        for z in (x_t, y, eps, x_out):
            _req(z)
        c = PSampleCoef(*[float(v) for v in coef])
        check(self.lib.bbdm_bridge_p_sample(ptr(x_t), ptr(y), ptr(eps), ptr(noise), c, OBJ[objective],
                                            int(clip), int(is_last), ptr(x_out), ptr(x0_out), x_t.numel(),
                                            stream()))
        LAUNCHES["n"] += 1

    def p_sample_dev(self, x_t, y, eps, noise, coef_dev, objective, clip, is_last, x_out, x0_out):
        for z in (x_t, y, eps, x_out, coef_dev):
            _req(z)
        check(self.lib.bbdm_bridge_p_sample_dev(ptr(x_t), ptr(y), ptr(eps), ptr(noise), ptr(coef_dev),
                                                OBJ[objective], int(clip), int(is_last), ptr(x_out), ptr(x0_out),
                                                x_t.numel(), stream()))
        LAUNCHES["n"] += 1

    # -- layout / dense ----------------------------------------------------------------------
    def nchw_to_nhwc_cat(self, x, ctx, out):
        B, c1, H, W = x.shape
        c2 = 0 if ctx is None else ctx.shape[1]
        check(self.lib.bbdm_nchw_to_nhwc_cat(ptr(_req(x)), c1, ptr(ctx), c2, B, H, W, ptr(_req(out)), stream()))
        LAUNCHES["n"] += 1

    def nhwc_to_nchw(self, src, out):
        B, H, W, Cc = src.shape
        check(self.lib.bbdm_nhwc_to_nchw(ptr(_req(src)), B, H, W, Cc, ptr(_req(out)), stream()))
        LAUNCHES["n"] += 1

    def gather_rows(self, table, idx, out):
        check(self.lib.bbdm_gather_rows(ptr(_req(table)), table.shape[0], table.shape[1],
                                        ptr(_req(idx, torch.int64)), idx.numel(), ptr(_req(out)), stream()))
        LAUNCHES["n"] += 1

    def linear(self, x, w, bias, out, act_in=False, act_out=False):
        B, K = x.shape
        N = w.shape[0]
        check(self.lib.bbdm_linear_f32(ptr(_req(x)), ptr(_req(w)), ptr(bias), ptr(_req(out)), B, K, N,
                                       int(act_in), int(act_out), stream()))
        LAUNCHES["n"] += (B + 7) // 8

    # -- group norm / prep ---------------------------------------------------------------------
    def gn_stats(self, src1, src2, groups, eps, mean, rstd, workspace):
        B, H, W, c1 = src1.shape
        c2 = 0 if src2 is None else src2.shape[3]
        check(self.lib.bbdm_gn_stats(ptr(_req(src1)), c1, ptr(src2), c2, B, H, W, groups, eps,
                                     ptr(_req(mean)), ptr(_req(rstd)), ptr(workspace), stream()))
        LAUNCHES["n"] += 2

    def prep(self, src1, src2, *, groups=32, mean=None, rstd=None, gamma=None, beta=None,
             film_scale=None, film_shift=None, film_stride=0, silu=True, resample=RESAMPLE_NONE,
             act_f32=None, act_hi=None, act_lo=None, raw_f32=None, raw_hi=None, raw_lo=None, heads=None):
        """heads: (n, scales, order) for the padded-head attention route -- the raw outputs then take src1's attention
        heads re-laid to their own head width (bbdm_attention_pad_heads / _unpad_heads) instead of a plain copy.  src1
        and the outputs hold len(scales) * n groups of columns, d wide on one side and d rounded up to 8 on the other;
        columns past d are zero, and tensor t's groups are multiplied by scales[t] (order 0: the tensors of one head
        together, the legacy qkv layout; order 1: all heads of one tensor together)."""
        if heads is not None:
            assert src2 is None and mean is None and act_f32 is None and act_hi is None and resample == RESAMPLE_NONE
            self._repack_heads(src1, *heads, raw_f32, raw_hi, raw_lo)
            return
        B, Hs, Ws, c1 = src1.shape
        a = PrepArgs(ptr(_req(src1)), c1, ptr(src2), 0 if src2 is None else src2.shape[3], B, Hs, Ws, groups,
                     ptr(mean), ptr(rstd), ptr(gamma), ptr(beta), ptr(film_scale), ptr(film_shift),
                     film_stride, int(silu), resample, ptr(act_f32), ptr(act_hi), ptr(act_lo),
                     ptr(raw_f32), ptr(raw_hi), ptr(raw_lo))
        check(self.lib.bbdm_prep_operand(C.byref(a), stream()))
        LAUNCHES["n"] += 1

    def _repack_heads(self, src, n, scales, order, out_f32, out_hi, out_lo):
        tensors = len(scales)
        out = out_f32 if out_f32 is not None else out_hi
        ws, wo = src.shape[-1] // (tensors * n), out.shape[-1] // (tensors * n)
        d, pad = min(ws, wo), wo >= ws
        assert ws * tensors * n == src.shape[-1] and wo * tensors * n == out.shape[-1], (src.shape, out.shape, n, scales)
        assert max(ws, wo) == pad_heads_width(d), (src.shape, out.shape)
        rows = src.numel() // src.shape[-1]
        for o, dt in ((out_f32, torch.float32), (out_hi, torch.bfloat16), (out_lo, torch.bfloat16)):
            if o is not None:
                assert o.numel() // o.shape[-1] == rows, (o.shape, src.shape)
                _req(o, dt)
        fn = self.lib.bbdm_attention_pad_heads if pad else self.lib.bbdm_attention_unpad_heads
        s = [float(x) for x in scales] + [1.0] * (3 - tensors)
        check(fn(ptr(_req(src)), rows, n, tensors, d, order, *s, ptr(out_f32), ptr(out_hi), ptr(out_lo), stream()))
        LAUNCHES["n"] += 1

    # -- convolutions --------------------------------------------------------------------------
    def pack_weight_split(self, w, hi, lo):
        """w [Cout,Cin,k,k] -> hi/lo [k*k, Cout_pad, Cin] bf16 (Cout_pad >= Cout; padding rows pre-zeroed)."""
        Cout, Cin, k = w.shape[0], w.shape[1], (w.shape[2] if w.dim() > 2 else 1)
        check(self.lib.bbdm_pack_weight_split_padded(ptr(_req(w)), Cout, Cin, k, hi.shape[1], ptr(hi), ptr(lo),
                                                     stream()))
        LAUNCHES["n"] += 1

    def pack_weight_split_dgrad(self, w, hi, lo):
        """w [Cout,Cin,k,k] -> hi/lo [k*k, Cin, Cout] bf16: flipped kernel, swapped channels."""
        Cout, Cin, k = w.shape[0], w.shape[1], w.shape[2]
        check(self.lib.bbdm_pack_weight_split_dgrad(ptr(_req(w)), Cout, Cin, k, ptr(hi), ptr(lo), stream()))
        LAUNCHES["n"] += 1

    def pack_weight_split_both(self, w, f_hi, f_lo, d_hi=None, d_lo=None):
        """forward planes [k*k, Cout, Cin] and (optionally) data-gradient planes [k*k, Cin, Cout] in one pass."""
        Cout, Cin, k = w.shape[0], w.shape[1], w.shape[2]
        check(self.lib.bbdm_pack_weight_split_both(ptr(_req(w)), Cout, Cin, k, ptr(f_hi), ptr(f_lo), ptr(d_hi), ptr(d_lo),
                                                   stream()))
        LAUNCHES["n"] += 1

    def pack_weight_split_taps(self, w, hi, lo):
        """w [Cout,Cin,taps] (any tap count) -> hi/lo [taps, Cout, Cin] bf16."""
        Cout, Cin, taps = w.shape
        check(self.lib.bbdm_pack_weight_split_taps(ptr(_req(w)), Cout, Cin, taps, ptr(hi), ptr(lo), stream()))
        LAUNCHES["n"] += 1

    def pack_weight_f32(self, w, out):
        Cout, Cin, k = w.shape[0], w.shape[1], (w.shape[2] if w.dim() > 2 else 1)
        check(self.lib.bbdm_pack_weight_f32(ptr(_req(w)), Cout, Cin, k, ptr(_req(out)), stream()))
        LAUNCHES["n"] += 1

    def conv_umma(self, *, B, H, W, Cin, Cout, taps, a_hi, a_lo, w_hi, w_lo, bias=None, Cin2=0,
                  a2_hi=None, a2_lo=None, w2_hi=None, w2_lo=None, bias2=None, residual=None,
                  res_mode=RES_NONE, out=None, out_hi=None, out_lo=None, passes=3, out_nchw_channels=0,
                  stats_partial=None, upsample2x=False, weights_per_image=False, operand_f16=False, window_origin=0):
        """window_origin (taps 4): 0 = 2x2 window at rows/cols 0..1, -1 = rows/cols -1..0."""
        a = ConvArgs(B, H, W, Cin, Cout, taps, ptr(a_hi), ptr(a_lo), ptr(w_hi), ptr(w_lo), ptr(bias),
                     Cin2, ptr(a2_hi), ptr(a2_lo), ptr(w2_hi), ptr(w2_lo), ptr(bias2),
                     ptr(residual), res_mode, ptr(out), ptr(out_hi), ptr(out_lo), passes, out_nchw_channels,
                     int(upsample2x), ptr(stats_partial), int(weights_per_image), int(operand_f16), int(window_origin))
        check(self.lib.bbdm_conv_umma(C.byref(a), stream()))
        LAUNCHES["n"] += 1

    def conv_geometry(self, H, W):
        """(TW, TH, TB, rows_per_image) of the tensor-core conv for an HxW output."""
        v = [C.c_int(0) for _ in range(4)]
        check(self.lib.bbdm_conv_umma_geometry(H, W, *[C.byref(z) for z in v]))
        return tuple(z.value for z in v)

    # -- Winograd F(4x4,3x3) / F(6x6,3x3) path ------------------------------------------------------
    def _wino(self, name, tile):
        assert tile in self.wino_tiles, tile
        return getattr(self.lib, f"bbdm_wino{'' if tile == 4 else tile}_{name}")

    def wino_geometry(self, B, H, W, tile=4):
        """(tiles_h, tiles_w, tiles_total, eligible); F(6,3): tiles_total padded to a multiple of 16."""
        th, tw, el, tot = C.c_int(0), C.c_int(0), C.c_int(0), C.c_int64(0)
        check(self._wino("geometry", tile)(B, H, W, C.byref(th), C.byref(tw), C.byref(tot), C.byref(el)))
        return th.value, tw.value, tot.value, bool(el.value)

    def wino_input(self, src1, src2, *, groups=32, mean=None, rstd=None, gamma=None, beta=None, film_scale=None,
                   film_shift=None, film_stride=0, silu=True, v_hi, v_lo, raw_hi=None, raw_lo=None, act_hi=None,
                   act_lo=None, tile=4, down2=False):
        """down2 (tile 6): transform the 2x2 average pool of the activated input (the conv runs on the H/2 x W/2
        map)."""
        B, H, W, c1 = src1.shape
        a = WinoInputArgs(ptr(_req(src1)), c1, ptr(src2), 0 if src2 is None else src2.shape[3], B, H, W, groups,
                          ptr(mean), ptr(rstd), ptr(gamma), ptr(beta), ptr(film_scale), ptr(film_shift), film_stride,
                          int(silu), ptr(_req(v_hi, torch.float16)), ptr(_req(v_lo, torch.float16)),
                          ptr(raw_hi), ptr(raw_lo), ptr(act_hi), ptr(act_lo), int(down2))
        check(self._wino("input", tile)(C.byref(a), stream()))
        LAUNCHES["n"] += 1

    def wino_output(self, m, *, B, H, W, Cout, bias=None, residual=None, res_mode=RES_NONE, out, stats_partial=None,
                    inv_wscale=None, tile=4, up2_phases=False):
        """inv_wscale: the [1] fp32 device tensor wino_pack_weight wrote for the weight planes of this GEMM (None:
        planes packed at the fixed 2^8).  up2_phases (tile 6): m holds the 4*Cout phase-major channels of a nearest-2x
        + 3x3 conv run on the HxW map; out is [B, 2H, 2W, Cout]."""
        a = WinoOutputArgs(ptr(_req(m)), None if inv_wscale is None else ptr(_req(inv_wscale)), B, H, W, Cout, ptr(bias), ptr(residual), res_mode, ptr(_req(out)),
                           ptr(stats_partial), int(up2_phases))
        check(self._wino("output", tile)(C.byref(a), stream()))
        LAUNCHES["n"] += 1

    def wino_pack_weight(self, w, u_hi, u_lo, dgrad=False, inv_wscale=None, tile=4):
        """w [Cout,Cin,3,3] fp32 -> u_hi/u_lo fp16 [(tile+2)^2, Cout, Cin] (s * G w G^T); dgrad: [.., Cin, Cout] of
        the flipped / channel-swapped kernel.  inv_wscale [1] fp32 on the device: s is the per-tensor power of two
        and 1/s is written there (pass it to wino_output); None: the fixed s = 2^8."""
        Cout, Cin = w.shape[0], w.shape[1]
        check(self._wino("pack_weight", tile)(ptr(_req(w)), Cout, Cin, int(dgrad), ptr(_req(u_hi, torch.float16)),
                                              ptr(_req(u_lo, torch.float16)),
                                              None if inv_wscale is None else ptr(_req(inv_wscale)), stream()))
        LAUNCHES["n"] += 1

    # -- SpatialTransformer pieces --------------------------------------------------------------------------
    def layernorm_split(self, x, gamma, beta, eps, out_f32=None, out_hi=None, out_lo=None):
        Cc = x.shape[-1]
        check(self.lib.bbdm_layernorm_split(ptr(_req(x)), x.numel() // Cc, Cc, ptr(_req(gamma)), ptr(_req(beta)), eps,
                                            ptr(out_f32), ptr(out_hi), ptr(out_lo), stream()))
        LAUNCHES["n"] += 1

    def geglu_split(self, u, out_f32=None, out_hi=None, out_lo=None):
        N2 = u.shape[-1]
        check(self.lib.bbdm_geglu_split(ptr(_req(u)), u.numel() // N2, N2 // 2, ptr(out_f32), ptr(out_hi), ptr(out_lo),
                                        stream()))
        LAUNCHES["n"] += 1

    def attention_cross(self, q_hi, q_lo, kv_hi, kv_lo, heads, out_f32=None, out_hi=None, out_lo=None):
        B, Tq, Cc = q_hi.shape
        Tkv = kv_hi.shape[1]
        check(self.lib.bbdm_attention_cross(ptr(_req(q_hi, torch.bfloat16)), ptr(_req(q_lo, torch.bfloat16)),
                                            ptr(_req(kv_hi, torch.bfloat16)), ptr(_req(kv_lo, torch.bfloat16)), B, Tq, Tkv,
                                            Cc, heads, ptr(out_f32), ptr(out_hi), ptr(out_lo), stream()))
        LAUNCHES["n"] += 1

    def layernorm_bwd(self, x, dy, gamma, eps, dx, dgamma, dbeta, workspace):
        """workspace: layernorm_bwd_workspace(rows, C) floats."""
        Cc = x.shape[-1]
        check(self.lib.bbdm_layernorm_bwd(ptr(_req(x)), ptr(_req(dy)), x.numel() // Cc, Cc, ptr(_req(gamma)), eps,
                                          ptr(_req(dx)), ptr(_req(dgamma)), ptr(_req(dbeta)), ptr(_req(workspace)),
                                          stream()))
        LAUNCHES["n"] += 2

    def geglu_bwd(self, u, dy, du):
        N2 = u.shape[-1]
        check(self.lib.bbdm_geglu_bwd(ptr(_req(u)), ptr(_req(dy)), u.numel() // N2, N2 // 2, ptr(_req(du)), stream()))
        LAUNCHES["n"] += 1

    def attention_cross_bwd(self, q, kv, out, dout, heads, dq, dkv, lse, delta):
        B, Tq, Cc = q.shape
        check(self.lib.bbdm_attention_cross_bwd(ptr(_req(q)), ptr(_req(kv)), ptr(_req(out)), ptr(_req(dout)), B, Tq,
                                                kv.shape[1], Cc, heads, ptr(_req(dq)), ptr(_req(dkv)), ptr(_req(lse)),
                                                ptr(_req(delta)), stream()))
        LAUNCHES["n"] += 2

    # -- sample_to_eval output path ------------------------------------------------------------------------
    def denorm_to_uint8(self, images, to_normal, out):
        B, Cc, H, W = images.shape
        check(self.lib.bbdm_denorm_to_uint8(ptr(_req(images)), B, Cc, H, W, int(to_normal), ptr(_req(out, torch.uint8)),
                                            stream()))
        LAUNCHES["n"] += 1

    def spatial_rescale(self, src, n_stages, weight, bias, out):
        """src [B,C,H,W] -> n_stages x bilinear(0.5) -> optional 1x1 map (weight [Cout,C], bias) -> out NCHW."""
        B, Cc, H, W = src.shape
        cout = 0 if weight is None else int(weight.shape[0])
        check(self.lib.bbdm_spatial_rescale(ptr(_req(src)), B, Cc, H, W, int(n_stages),
                                            ptr(None if weight is None else _req(weight)),
                                            ptr(None if bias is None else _req(bias)), cout, ptr(_req(out)), stream()))
        LAUNCHES["n"] += 1

    # -- multi-tensor optimizer / EMA -----------------------------------------------------------------------
    def optim_chunk_elems(self):
        return int(self.lib.bbdm_optim_chunk_elems())

    def adam_multi(self, tab, exp_avg, exp_avg_sq, *, lr, beta1, beta2, eps, weight_decay, step, ema_shadow=None,
                   ema_decay=0.0):
        """tab: bbdm_b200.optim.TensorTable (device pointer / size / chunk arrays of the parameter list)."""
        check(self.lib.bbdm_adam_multi(ptr(tab.params), ptr(tab.grads), ptr(tab.numel), ptr(tab.offsets),
                                       ptr(tab.chunk_tensor), ptr(tab.chunk_index), tab.n_chunks, ptr(_req(exp_avg)),
                                       ptr(_req(exp_avg_sq)), lr, beta1, beta2, eps, weight_decay, int(step),
                                       ptr(ema_shadow), float(ema_decay), stream()))
        LAUNCHES["n"] += 1

    def adam_multi_dev(self, tab, exp_avg, exp_avg_sq, *, step, lr, beta1, beta2, eps, weight_decay, ema_shadow=None,
                       ema_decay=0.0):
        """Capturable form: step (fp32 [] tensor, incremented here on the device) and lr (fp64 [] tensor) are read
        from device memory."""
        check(self.lib.bbdm_adam_multi_dev(ptr(tab.params), ptr(tab.grads), ptr(tab.numel), ptr(tab.offsets),
                                           ptr(tab.chunk_tensor), ptr(tab.chunk_index), tab.n_chunks, ptr(_req(exp_avg)),
                                           ptr(_req(exp_avg_sq)), ptr(_req(step)), ptr(_req(lr, torch.float64)),
                                           beta1, beta2, eps, weight_decay, ptr(ema_shadow), float(ema_decay), stream()))
        LAUNCHES["n"] += 2

    def ema_multi(self, tab, shadow, decay, with_decay=True):
        check(self.lib.bbdm_ema_multi(ptr(tab.params), ptr(tab.numel), ptr(tab.offsets), ptr(tab.chunk_tensor),
                                      ptr(tab.chunk_index), tab.n_chunks, ptr(_req(shadow)), float(decay), int(with_decay),
                                      stream()))
        LAUNCHES["n"] += 1

    def gn_finalize_partials(self, part1, rows1, part2, rows2, B, hw, groups, eps, mean, rstd):
        c1 = part1.shape[1]
        c2 = 0 if part2 is None else part2.shape[1]
        check(self.lib.bbdm_gn_finalize_partials(ptr(_req(part1)), c1, rows1, ptr(part2), c2, rows2, B, hw, groups,
                                                 eps, ptr(_req(mean)), ptr(_req(rstd)), stream()))
        LAUNCHES["n"] += 1

    # -- training gradients -----------------------------------------------------------------------
    def split_grad(self, src, hi, lo, hi_t, lo_t, colsum=None, workspace=None):
        """hi_t / lo_t: [C, P], rows possibly padded (train._transposed_planes)."""
        P, Cc = src.numel() // src.shape[-1], src.shape[-1]
        ld = _pitch(hi_t, lo_t, Cc, P)
        check(self.lib.bbdm_split_grad(ptr(_req(src)), P, Cc, ptr(hi), ptr(lo), ptr(hi_t), ptr(lo_t), ld, ptr(colsum),
                                       ptr(workspace), stream()))
        LAUNCHES["n"] += 1 + (colsum is not None)

    def wgrad_workspace(self, B, H, W, Cin, Cout, taps):
        sp, fl = C.c_int(0), C.c_int64(0)
        check(self.lib.bbdm_conv_wgrad_workspace(B, H, W, Cin, Cout, taps, C.byref(sp), C.byref(fl)))
        return sp.value, fl.value

    def conv_wgrad(self, g_hi_t, g_lo_t, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, workspace, window_origin=0):
        """taps 1, 9, or 4 with window_origin 0 / -1 (dw [Cout, Cin, 2, 2])."""
        ld = _pitch(g_hi_t, g_lo_t, Cout, B * H * W)
        check(self.lib.bbdm_conv_wgrad(ptr(g_hi_t), ptr(g_lo_t), ld, ptr(a_hi), ptr(a_lo), B, H, W, Cin, Cout, taps,
                                       int(window_origin), ptr(_req(dw)), ptr(_req(workspace)), stream()))
        LAUNCHES["n"] += 2

    def conv_wgrad_direct(self, dy, x, k, dw, workspace):
        B, H, W, Cin = x.shape
        Cout = dy.shape[3]
        check(self.lib.bbdm_conv_wgrad_direct(ptr(_req(dy)), ptr(_req(x)), B, H, W, Cin, Cout, k, ptr(_req(dw)),
                                              ptr(_req(workspace)), workspace.numel(), stream()))
        LAUNCHES["n"] += 2

    def gn_bwd_reduce(self, x, da, groups, mean, rstd, gamma, beta, fscale, fshift, fstride, silu, a12, ws):
        B, H, W, Cc = x.shape
        check(self.lib.bbdm_gn_bwd_reduce(ptr(_req(x)), ptr(_req(da)), B, H, W, Cc, groups, ptr(mean), ptr(rstd),
                                          ptr(gamma), ptr(beta), ptr(fscale), ptr(fshift), fstride, int(silu),
                                          ptr(_req(a12)), ptr(_req(ws)), stream()))
        LAUNCHES["n"] += 2

    def gn_bwd_apply(self, x, da, groups, mean, rstd, gamma, beta, fscale, fshift, fstride, silu, s1, s2, dx):
        B, H, W, Cc = x.shape
        check(self.lib.bbdm_gn_bwd_apply(ptr(_req(x)), ptr(_req(da)), B, H, W, Cc, groups, ptr(mean), ptr(rstd),
                                         ptr(gamma), ptr(beta), ptr(fscale), ptr(fshift), fstride, int(silu),
                                         ptr(_req(s1)), ptr(_req(s2)), ptr(_req(dx)), stream()))
        LAUNCHES["n"] += 1

    def conv_direct(self, src, w_packed, bias, residual, out, Cout, k, stride=1):
        B, H, W, Cin = src.shape
        check(self.lib.bbdm_conv_direct(ptr(_req(src)), ptr(_req(w_packed)), ptr(bias), ptr(residual),
                                        ptr(_req(out)), B, H, W, Cin, Cout, k, stride, stream()))
        LAUNCHES["n"] += 1

    def conv_stem(self, src, w_packed, bias, out, Cout, stats_partial=None):
        B, H, W, Cin = src.shape
        check(self.lib.bbdm_conv_stem(ptr(_req(src)), ptr(_req(w_packed)), ptr(bias), ptr(_req(out)), B, H, W, Cin, Cout,
                                      ptr(stats_partial), stream()))
        LAUNCHES["n"] += 1

    # -- attention -------------------------------------------------------------------------------
    def attention(self, qkv, heads, order, out_f32=None, out_hi=None, out_lo=None):
        B, T, C3 = qkv.shape
        check(self.lib.bbdm_attention(ptr(_req(qkv)), B, T, C3 // 3, heads, order, ptr(out_f32),
                                      ptr(out_hi), ptr(out_lo), stream()))
        LAUNCHES["n"] += 1

    def attention_split(self, qkv_hi, qkv_lo, heads, order, out_f32=None, out_hi=None, out_lo=None):
        B, T, C3 = qkv_hi.shape
        check(self.lib.bbdm_attention_split(ptr(_req(qkv_hi, torch.bfloat16)), ptr(_req(qkv_lo, torch.bfloat16)),
                                            B, T, C3 // 3, heads, order, ptr(out_f32), ptr(out_hi), ptr(out_lo),
                                            stream()))
        LAUNCHES["n"] += 1

    def attention_tc(self, qkv_hi, qkv_lo, heads, order, out_f32=None, out_hi=None, out_lo=None):
        B, T, C3 = qkv_hi.shape
        check(self.lib.bbdm_attention_tc(ptr(_req(qkv_hi, torch.bfloat16)), ptr(_req(qkv_lo, torch.bfloat16)),
                                         B, T, C3 // 3, heads, order, ptr(out_f32), ptr(out_hi), ptr(out_lo), stream()))
        LAUNCHES["n"] += 1

    def attention_bwd(self, qkv, out, dout, heads, order, dqkv, lse, delta):
        B, T, C3 = qkv.shape
        check(self.lib.bbdm_attention_bwd(ptr(_req(qkv)), ptr(_req(out)), ptr(_req(dout)), B, T, C3 // 3, heads, order,
                                          ptr(_req(dqkv)), ptr(_req(lse)), ptr(_req(delta)), stream()))
        LAUNCHES["n"] += 2

    def conv_direct_pad(self, src, w_packed, bias, residual, out, cout, k, stride, pad_lo, pad_hi):
        B, H, W, Cin = src.shape
        check(self.lib.bbdm_conv_direct_pad(ptr(_req(src)), ptr(_req(w_packed)), ptr(bias), ptr(residual), ptr(_req(out)),
                                            B, H, W, Cin, cout, k, stride, pad_lo, pad_hi, stream()))
        LAUNCHES["n"] += 1

    def softmax_rows_split(self, src, scale, out_hi, out_lo, valid_cols=None, grad=None):
        """The planes of p = softmax(scale * src) per row.  valid_cols: the columns of each row the softmax covers (None:
        all); the planes are zero in the rest.  grad: dL/dp of the same shape -- the planes then hold the backward's
        score gradient scale * p * (grad - sum_j p_j grad_j) instead of p (bbdm_softmax_rows_bwd)."""
        rows, cols = src.numel() // src.shape[-1], src.shape[-1]
        v = cols if valid_cols is None else int(valid_cols)
        if grad is not None:
            assert grad.shape == src.shape, (grad.shape, src.shape)
            check(self.lib.bbdm_softmax_rows_bwd(ptr(_req(src)), ptr(_req(grad)), rows, cols, v, float(scale),
                                                 ptr(_req(out_hi, torch.bfloat16)), ptr(_req(out_lo, torch.bfloat16)),
                                                 stream()))
        else:
            check(self.lib.bbdm_softmax_rows_split(ptr(_req(src)), rows, cols, v, float(scale),
                                                   ptr(_req(out_hi, torch.bfloat16)), ptr(_req(out_lo, torch.bfloat16)),
                                                   stream()))
        LAUNCHES["n"] += 1

    def s2d_split(self, src, out_hi, out_lo):
        B, H, W, Cc = src.shape
        check(self.lib.bbdm_s2d_split(ptr(_req(src)), B, H, W, Cc, ptr(_req(out_hi, torch.bfloat16)),
                                      ptr(_req(out_lo, torch.bfloat16)), stream()))
        LAUNCHES["n"] += 1

    def vq_nearest(self, z, codebook, z_q, indices):
        n, d = z.numel() // z.shape[-1], z.shape[-1]
        check(self.lib.bbdm_vq_nearest(ptr(_req(z)), ptr(_req(codebook)), n, codebook.shape[0], d, ptr(_req(z_q)),
                                       ptr(_req(indices, torch.int64)), stream()))
        LAUNCHES["n"] += 1

    def check_fault(self, device=None):
        """Raise if a kernel on ``device`` (default: the current device) set the device fault word."""
        w = C.c_ulonglong(0)
        if device is not None and torch.device(device).index not in (None, torch.cuda.current_device()):
            with torch.cuda.device(device):
                check(self.lib.bbdm_check_device_fault(stream(), C.byref(w)))
            return
        check(self.lib.bbdm_check_device_fault(stream(), C.byref(w)))
