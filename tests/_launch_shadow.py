"""TEST-ONLY: a shadow backend that checks every kernel launch of the UNet executor against an fp64 recomputation of
that launch, from copies of the tensors the launch read.

``Shadow`` wraps a backend (cabi.CudaBackend, or the CPU emulation to test the checker itself) the way the Recorder of
tests/test_launch_trace_host.py wraps the emulation: every launching method is bound to its signature, the tensors it
reads are cloned, the real launch runs, the device is synchronized and its fault word read, and then

- every input that is not also an output must be bit-unchanged (an out-of-bounds write into a neighbouring pool buffer
  that the launch reads shows here);
- every output is compared with a float64 recomputation from the clones, on the tensors' own device.  The deviation is
  taken per image: the max over images of max|got - want| / max|want| within the image, so one wrong image of a batch
  cannot hide behind the others.

The Winograd chains are paired by buffer identity (wino_input's V planes -> the position GEMMs' A operand, the GEMMs'
output -> wino_output's M) and checked stage by stage and as a whole, against the fp64 conv of the fp64 activation with
the module's fp32 weight; ``register_engine`` maps each cache entry's U planes to its module weight.

The training Functions of bbdm_b200/train.py and FusedAdam are checked the same way: the backward kernels against fp64
autograd of the operation they implement, from the launch's own inputs (GroupNorm statistics, split planes, the forward
output attention_bwd reads); the weight packers bit for bit; adam_multi per parameter tensor against an fp64
torch.optim.Adam step from the pre-launch parameters, gradients and moments, which it reads through the TensorTable's
pointer arrays rather than tensor arguments.  Training packs its Winograd weight planes on the fly, so
wino_pack_weight itself maps the U planes to the weight they hold (for the data gradient the flipped, channel-swapped
kernel), and the output transform that consumes them takes the entry out again.

The sampling and VQGAN launches are checked the same way: the bridge update (p_sample, and p_sample_dev with its
coefficients read from the device before the launch) and the uint8 output path bit for bit against the reference's
fp32 expressions, the space-to-depth split bit for bit, the SpatialRescaler, the padded direct conv, the row softmax and
the nearest-code search against fp64.  Inside a CUDA-graph capture the shadow only runs each launch and lists it in
``captured``: a capture records work for later replays, so nothing may be copied, synchronised or read there.

Bounds are those of the single-kernel GPU tests, measured on an H100 with synthetic operands; each names its source.
A launch whose output goes beyond its bound is a finding, not a bound to raise.
"""
import collections
import inspect
import math

import torch
import torch.nn.functional as F

from oracle import bbdm_oracle as O
from test_launch_trace_host import NOT_LAUNCHES

F64 = torch.float64

# what each launching method writes; a method not listed is an error (a new launch kind must get a reference)
OUTPUTS = {
    "nchw_to_nhwc_cat": ("out",), "nhwc_to_nchw": ("out",), "gather_rows": ("out",), "linear": ("out",),
    "gn_stats": ("mean", "rstd", "workspace"), "gn_finalize_partials": ("mean", "rstd"),
    "prep": ("act_f32", "act_hi", "act_lo", "raw_f32", "raw_hi", "raw_lo"),
    "pack_weight_split": ("hi", "lo"), "pack_weight_split_taps": ("hi", "lo"), "pack_weight_f32": ("out",),
    "wino_pack_weight": ("u_hi", "u_lo", "inv_wscale"),
    "conv_umma": ("out", "out_hi", "out_lo", "stats_partial"), "conv_direct": ("out",),
    "conv_stem": ("out", "stats_partial"),
    "wino_input": ("v_hi", "v_lo", "raw_hi", "raw_lo", "act_hi", "act_lo"), "wino_output": ("out", "stats_partial"),
    "attention": ("out_f32", "out_hi", "out_lo"), "attention_split": ("out_f32", "out_hi", "out_lo"),
    "attention_tc": ("out_f32", "out_hi", "out_lo"),
    # training: bridge, gradient operands, backward kernels, optimizer
    "q_sample": ("xt_out", "obj_out"),
    "split_grad": ("hi", "lo", "hi_t", "lo_t", "colsum", "workspace"),
    "pack_weight_split_both": ("f_hi", "f_lo", "d_hi", "d_lo"), "pack_weight_split_dgrad": ("hi", "lo"),
    "conv_wgrad": ("dw", "workspace"), "conv_wgrad_direct": ("dw", "workspace"),
    "gn_bwd_reduce": ("a12", "ws"), "gn_bwd_apply": ("dx",),
    "attention_bwd": ("dqkv", "lse", "delta"),
    "attention_cross": ("out_f32", "out_hi", "out_lo"), "attention_cross_bwd": ("dq", "dkv", "lse", "delta"),
    "layernorm_split": ("out_f32", "out_hi", "out_lo"), "layernorm_bwd": ("dx", "dgamma", "dbeta", "workspace"),
    "geglu_split": ("out_f32", "out_hi", "out_lo"), "geglu_bwd": ("du",),
    "adam_multi": ("exp_avg", "exp_avg_sq", "ema_shadow"), "ema_multi": ("shadow",),
    # the capturable Adam step also increments its device step counter
    "adam_multi_dev": ("exp_avg", "exp_avg_sq", "ema_shadow", "step"),
    # sampling: the bridge update, the SpatialRescaler condition, the uint8 output path
    "p_sample": ("x_out", "x0_out"), "p_sample_dev": ("x_out", "x0_out"), "spatial_rescale": ("out",),
    "denorm_to_uint8": ("out",),
    # VQGAN ends (and the UNet's tensor-core Downsample operand)
    "s2d_split": ("out_hi", "out_lo"), "conv_direct_pad": ("out",), "softmax_rows_split": ("out_hi", "out_lo"),
    "vq_nearest": ("z_q", "indices"),
}
# launches that read (and adam_multi writes) the parameters of a TensorTable instead of tensor arguments
TABLE_LAUNCHES = ("adam_multi", "adam_multi_dev", "ema_multi")

# a split-bf16 pair carries 16 bits: 2^-17 = 7.6e-6 of the element (test_gpu_winograd.py::test_wino_input_production_layouts)
PAIR = 8e-6
BOUNDS = {
    "exact": 0.0,
    "linear": 2e-6,             # test_gpu_kernels.py::test_gather_and_linear
    "gn_stats": 2e-6,           # test_gpu_kernels.py::test_gn_stats
    "gn_finalize": 3e-6,        # test_gpu_kernels.py::test_conv_umma_fused_groupnorm_statistics
    "prep_act": 5e-6,           # test_gpu_kernels.py::test_prep_operand (act_f32)
    "prep_act_planes": 5e-6 + PAIR,
    "prep_raw": 1e-6,           # test_gpu_kernels.py::test_prep_operand (raw_f32)
    "prep_raw_planes": 1e-6 + PAIR,
    "conv_direct": 3e-6,        # test_gpu_kernels.py::test_conv_direct
    "conv_stem": 2e-6,          # test_gpu_kernels.py::test_conv_stem_equals_conv_direct_and_fuses_gn_partials
    "conv_umma": 6e-6,          # test_gpu_kernels.py::test_conv_umma (fp64 evaluation of the same split products)
    "conv_umma_planes": 6e-6 + PAIR,
    "stats": 1e-5,              # test_gpu_winograd6.py::test_wino6_chain_vs_fp64_conv (GroupNorm partial sums)
    "attention": 2e-5,          # test_gpu_kernels.py::test_attention_tc / test_attention_split / test_attention
    "attention_planes": 2e-5 + PAIR,
    "wino_v6": 1e-6,            # test_gpu_winograd6.py::test_wino6_input_transform_exact_positions
    "wino_v4": 2e-6,            # test_gpu_winograd.py::test_wino_input_production_layouts
    "wino_act_planes": PAIR,    # test_gpu_winograd.py::test_wino_input_production_layouts (act planes)
    "wino_m": 3e-6,             # test_gpu_winograd.py::test_wino_conv_chain_vs_fp64_conv (position GEMMs)
    # tools/host_check_wino6_output.cu (run by test_wino6_output_host.py) holds the output transform to 2e-6 of max|Y|
    # with random M.  In the model M is far larger than Y (the transform cancels), and the fp32 evaluation's error
    # scales with |A^T| |M| |A|: measured up to 3.7e-6 on an H100 80GB HBM3 (cfg2 at B = 16 and cfg4 at B = 64, the
    # 64x64 F(6,3) wide-input conv1s), while the same launches stay within the chain bound against the independent
    # fp64 conv (1.84e-5 and 1.34e-5).
    "wino_y": 5e-6,
    "chain6": 2e-5,             # test_gpu_winograd6.py CHAIN_BOUND
    "chain4": 1.6e-5,           # test_gpu_winograd.py CHAIN_BOUND_BIASED
    # The training data gradient's F(4,3) chain (identity input transform of the power-of-two normalised dY, flipped
    # weight planes), per image.  CHAIN_BOUND_BIASED was measured on forward chains, whole tensor.  The dgrad chains of
    # the cfg3 training step at B = 32 reach 1.63e-5 on an H100 80GB HBM3 (700 W; the 32x32 512-channel convs) with
    # every stage within its own bound (V 3.6e-7, position GEMMs 1.5e-6, output transform 2.4e-6), and the CPU
    # emulation, whose transforms are exact fp64, reaches 1.65e-5 on the same kind of operands
    # (test_train_shadow_host.py): the F(4,3) deviation of 22-bit fp16-pair planes on data-gradient operands.
    "chain4_dgrad": 2e-5,
    "pack_wino6": 1e-6,         # test_gpu_winograd6.py::test_wino6_pack_weight
    "pack_wino4": 2e-7,         # test_gpu_winograd.py::test_wino_pack_weight
    "up_phase": 2.0 ** -16,     # test_gpu_kernels.py::test_conv_umma_fused_upsample: the taps are summed in fp32, then split
    # training
    "colsum": 1e-6,             # test_gpu_training.py::test_split_grad
    "conv_wgrad": 2e-5,         # test_gpu_training.py::test_conv_wgrad (whole tensor)
    "conv_wgrad_direct": 2e-6,  # test_gpu_training.py::test_small_conv_function_gradients
    "gn_bwd": 2e-6,             # test_gpu_training.py::test_gn_bwd_kernels
    "attention_bwd": 2e-5,      # test_gpu_training.py::test_attention_bwd_kernel
    "attention_cross": 2e-5,    # test_gpu_kernels.py::test_attention_cross
    "attention_cross_bwd": 2e-5,  # test_gpu_transformer_training.py::test_attention_cross_bwd_kernel
    "layernorm": 2e-6,          # test_gpu_kernels.py::test_layernorm_split
    "layernorm_planes": 2e-6 + PAIR,
    "layernorm_bwd": 2e-6,      # test_gpu_transformer_training.py::test_layernorm_bwd_kernel
    "geglu": 2e-6,              # test_gpu_kernels.py::test_geglu_split
    "geglu_planes": 2e-6 + PAIR,
    "geglu_bwd": 2e-6,          # test_gpu_transformer_training.py::test_geglu_bwd_kernel
    # adam_multi / ema_multi, per parameter tensor.  No single-kernel test bounds these at this granularity
    # (test_optim_host.py compares parameters after several steps).  The moments and the EMA shadow are one fp32
    # multiply-add of the previous value: a few 2^-24 of the tensor's largest element.  The update dp is counted
    # beyond the half-ulp of the fp32 parameter that has to hold it (see _ref_adam_multi).
    "adam_dp": 1e-5,
    "adam_moments": 1e-6,
    "ema": 1e-6,
    # sampling and VQGAN ends
    "conv_direct_pad": 2e-6,    # test_gpu_vqgan.py::test_conv_direct_pad
    "softmax": 2e-5,            # test_gpu_vqgan.py::test_softmax_rows_split
    "vq_distance": 1e-5,        # test_gpu_vqgan.py::test_vq_nearest (chosen vs minimum distance; the top-2 gap)
    "spatial_rescale": 1e-6,    # test_gpu_kernels.py::test_spatial_rescale
}

# Winograd matrices, interpolation points 0, +-1, +-2 (F(4,3)) and 0, +-1, +-2, +-1/2 (F(6,3))
BT = {4: [[4, 0, -5, 0, 1, 0], [0, -4, -4, 1, 1, 0], [0, 4, -4, -1, 1, 0], [0, -2, -1, 2, 1, 0], [0, 2, -1, -2, 1, 0],
          [0, 4, 0, -5, 0, 1]],
      6: [[1, 0, -21 / 4, 0, 21 / 4, 0, -1, 0], [0, 1, 1, -17 / 4, -17 / 4, 1, 1, 0], [0, -1, 1, 17 / 4, -17 / 4, -1, 1, 0],
          [0, 1 / 2, 1 / 4, -5 / 2, -5 / 4, 2, 1, 0], [0, -1 / 2, 1 / 4, 5 / 2, -5 / 4, -2, 1, 0],
          [0, 2, 4, -5 / 2, -5, 1 / 2, 1, 0], [0, -2, 4, 5 / 2, -5, -1 / 2, 1, 0], [0, -1, 0, 21 / 4, 0, -21 / 4, 0, 1]]}
G = {4: [[1 / 4, 0, 0], [-1 / 6, -1 / 6, -1 / 6], [-1 / 6, 1 / 6, -1 / 6], [1 / 24, 1 / 12, 1 / 6],
         [1 / 24, -1 / 12, 1 / 6], [0, 0, 1]],
     6: [[1, 0, 0], [-2 / 9, -2 / 9, -2 / 9], [-2 / 9, 2 / 9, -2 / 9], [1 / 90, 1 / 45, 2 / 45], [1 / 90, -1 / 45, 2 / 45],
         [32 / 45, 16 / 45, 8 / 45], [32 / 45, -16 / 45, 8 / 45], [0, 0, 1]]}
AT = {4: [[1, 1, 1, 1, 1, 0], [0, 1, -1, 2, -2, 0], [0, 1, 1, 4, 4, 0], [0, 1, -1, 8, -8, 1]],
      6: [[1, 1, 1, 1, 1, 1, 1, 0], [0, 1, -1, 2, -2, 1 / 2, -1 / 2, 0], [0, 1, 1, 4, 4, 1 / 4, 1 / 4, 0],
          [0, 1, -1, 8, -8, 1 / 8, -1 / 8, 0], [0, 1, 1, 16, 16, 1 / 16, 1 / 16, 0],
          [0, 1, -1, 32, -32, 1 / 32, -1 / 32, 1]]}


def _mat(table, tile, dev):
    return torch.tensor(table[tile], dtype=F64, device=dev)


# ------------------------------------------------------------------------------------------------ metrics
def image_devs(got, want):
    """Per image (dim 0): max|got - want| / max|want|; NaN counts as infinitely wrong."""
    n = got.shape[0]
    g, w = got.reshape(n, -1).to(F64), want.reshape(n, -1).to(F64)
    d = (g - w).abs().amax(1) / w.abs().amax(1).clamp_min(1e-30)
    return torch.nan_to_num(d, nan=math.inf)


def image_equal(got, want):
    """Per image: 0 where got is bit-identical to want, else inf."""
    n = got.shape[0]
    same = (got.reshape(n, -1) == want.reshape(n, -1)).all(1)
    return torch.where(same, 0.0, math.inf).to(F64)


def _words(t):
    b = t.contiguous().view(-1).view(torch.uint8)
    return b.view(torch.int32) if b.numel() % 4 == 0 else b


def bits_equal(a, b):
    if a.shape != b.shape:
        return False
    wa, wb = _words(a), _words(b)
    step = 1 << 26                     # no full-size temporaries next to the executor's multi-GB buffers
    return all(torch.equal(wa[i:i + step], wb[i:i + step]) for i in range(0, wa.numel(), step))


# inputs of at least this size (the F(6,3) V planes and wide concat inputs at 256x256, batch 16) are not copied: two
# checksums of their bytes, taken before and after the launch, stand in for the copy, and the references read them in
# place
BIG = 1 << 30


def fingerprint(t):
    """(sum of the 32-bit words, position-weighted sum) of t's bytes, chunked."""
    w = _words(t)
    s1 = s2 = 0
    step = 1 << 26
    for i in range(0, w.numel(), step):
        x = w[i:i + step].to(torch.int64)
        s1 += int(x.sum())
        s2 += int((x * (torch.arange(x.numel(), device=x.device) % 65521 + i % 65521 + 1)).sum())
    return s1, s2


def split_bf16(x):
    """x (fp32) -> (hi, lo) bf16 with hi = bf16(x), lo = bf16(x - hi)."""
    h = x.to(torch.bfloat16)
    return h, (x - h.float()).to(torch.bfloat16)


def pair_well_formed(hi, lo):
    """Per image: 0 where hi is bf16(hi + lo) (a split pair, not two arbitrary halves), else inf."""
    v = hi.float() + lo.float()
    r = v.to(torch.bfloat16).float()
    ok = (r == hi.float()) | ((r - hi.float()).abs() == 2 * lo.float().abs())
    n = hi.shape[0]
    return torch.where(ok.reshape(n, -1).all(1), 0.0, math.inf).to(F64)


def planes(hi, lo):
    return hi.to(F64) + lo.to(F64)


def chunks(n, per_item_bytes, dev):
    """Slices of range(n) whose fp64 working set stays under a few GB (references must not exhaust the device)."""
    limit = (2 << 30) if torch.device(dev).type == "cuda" else (1 << 30)
    step = max(1, int(limit // max(1, per_item_bytes)))
    for b0 in range(0, n, step):
        yield slice(b0, min(n, b0 + step))


# ------------------------------------------------------------------------------------------------ fp64 operations
def tap_conv(ap, taps, H, W):
    """sum over (dy, dx, w [Cout, C]) of ap[:, dy:dy+H, dx:dx+W] @ w^T; ap [n, Hp, Wp, C] fp64 -> [n, H, W, Cout]."""
    n, C = ap.shape[0], ap.shape[3]
    out = None
    for dy, dx, w in taps:
        t = ap[:, dy:dy + H, dx:dx + W].reshape(n * H * W, C) @ w.t()
        out = t if out is None else out.add_(t)
    return out.view(n, H, W, -1)


def conv3x3(a, w):
    """'same' 3x3 conv of NHWC a (fp64) with OIHW w (fp64)."""
    n, H, W, _ = a.shape
    ap = F.pad(a, (0, 0, 1, 1, 1, 1))
    return tap_conv(ap, [(ky, kx, w[:, :, ky, kx]) for ky in range(3) for kx in range(3)], H, W)


def up2(a):
    return a.repeat_interleave(2, 1).repeat_interleave(2, 2)


def pool2(a):
    n, H, W, C = a.shape
    return a[:, :H // 2 * 2, :W // 2 * 2].reshape(n, H // 2, 2, W // 2, 2, C).mean((2, 4))


def add_residual(o, res, mode):
    """o [n, Ho, Wo, C] fp64 + the residual of the C ABI's res_mode (1 same, 2 nearest-up of half size, 3 2x2 average
    of double size)."""
    if mode == 0 or res is None:
        return o
    r = res.to(F64)
    return o + {1: lambda: r, 2: lambda: up2(r), 3: lambda: pool2(r)}[mode]()


def gn_act(x, a, sl):
    """The prep / wino_input activation of images sl in fp64: GroupNorm affine (+FiLM) (+SiLU), or x itself without
    statistics.  a: the launch's cloned arguments."""
    xb = x[sl].to(F64)
    if a.get("mean") is None:
        return xb
    f = lambda t: None if t is None else t[sl].to(F64)
    return O.op_gn_act(xb, f(a["mean"]), f(a["rstd"]), a["gamma"].to(F64), a["beta"].to(F64), f(a.get("film_scale")),
                       f(a.get("film_shift")), bool(a.get("silu", True)), 0)


def cat(a, b):
    return a if b is None else torch.cat([a, b], 3)


def up_phase_reference(w):
    """fp64 phase taps [16, Cout, Cin] of nearest-2x + the 3x3 conv w, from the definition: output pixel 2y+a reads
    upsampled row 2y+a+ky-1, i.e. source row y + (a+ky-1)//2, which is tap r = (a+ky-1)//2 + 1 - a of phase a."""
    w = w.to(F64)
    out = torch.zeros(16, w.shape[0], w.shape[1], dtype=F64, device=w.device)
    for a in range(2):
        for b in range(2):
            for ky in range(3):
                for kx in range(3):
                    r, c = (a + ky - 1) // 2 + 1 - a, (b + kx - 1) // 2 + 1 - b
                    out[(2 * a + b) * 4 + 2 * r + c] += w[:, :, ky, kx]
    return out


def space_to_depth(x):
    """NHWC [n, H, W, C] -> [n, H/2, W/2, 4C]: channel (a*2 + b)*C + c of pixel (i, j) is pixel (2i + a, 2j + b)."""
    n, H, W, C = x.shape
    return x.reshape(n, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(n, H // 2, W // 2, 4 * C)


def s2d_tap_reference(w, origin):
    """fp64 2x2 taps [4, Cout, 4*Cin] of a 3x3 stride-2 conv w on the space-to-depth operand, from the definition:
    output pixel i reads input row 2i + k - pad_lo (pad_lo 1 for padding 1, 0 for the VQGAN's (0, 1) padding), which
    is phase a of operand row i + o for 2o + a = k - pad_lo; tap r = o - origin of the window at origin."""
    w = w.to(F64)
    co, ci = w.shape[0], w.shape[1]
    out = torch.zeros(4, co, 4, ci, dtype=F64, device=w.device)
    pad_lo = -origin            # origin -1: padding (1, 1), the UNet Downsample; origin 0: padding (0, 1)
    for ky in range(3):
        for kx in range(3):
            (oy, a), (ox, b) = divmod(ky - pad_lo, 2), divmod(kx - pad_lo, 2)
            out[(oy - origin) * 2 + (ox - origin), :, a * 2 + b] = w[:, :, ky, kx]
    return out.reshape(4, co, 4 * ci)


def attention_ref(qkv, heads, order, sl_img):
    """fp64 softmax attention of images sl_img of qkv [B, T, 3C] (fp64), head by head -> [n, T, C]."""
    B, T, C3 = qkv.shape
    C = C3 // 3
    d = C // heads
    out = torch.empty(qkv[sl_img].shape[0], T, C, dtype=F64, device=qkv.device)
    for i, b in enumerate(range(*sl_img.indices(B))):
        for h in range(heads):
            if order:      # new order: q | k | v, each heads x d
                q, k, v = (qkv[b, :, j * C + h * d:j * C + (h + 1) * d] for j in range(3))
            else:          # legacy order: per head q, k, v of d channels each
                q, k, v = (qkv[b, :, h * 3 * d + j * d:h * 3 * d + (j + 1) * d] for j in range(3))
            s = torch.softmax((q @ k.t()) / math.sqrt(d), dim=-1)
            out[i, :, h * d:(h + 1) * d] = s @ v
    return out


def _capturing():
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


# ------------------------------------------------------------------------------------------------ the shadow
Check = collections.namedtuple("Check", "launch method form what dev bound shapes")


class Shadow:
    def __init__(self, be, bounds=None):
        """bounds: entries of BOUNDS to replace (the CPU emulation's chain)."""
        self.be = be
        self.bounds = dict(BOUNDS, **(bounds or {}))
        self.checks, self.launches = [], []
        self.captured = []                # methods launched inside a CUDA-graph capture: run, not checked
        self.mutate = {}                  # launch index -> fn(bound arguments): perturbs an output after the launch
        self._wino_in, self._wino_m = {}, {}
        self._weights = {}                # U planes' data_ptr -> (module weight [Cout, Cin, 3, 3], up2_phases, name)
        self._packed = {}                 # U planes' data_ptr -> (weight clone, dgrad) of an on-the-fly pack
        self._dgrad_w = set()             # data_ptrs of data-gradient split planes not yet read by a conv

    # -- bookkeeping -------------------------------------------------------------------------------------------
    def register_engine(self, eng):
        """Map every Winograd cache entry's U planes to the module weight they were packed from (plain convs, tile 4 and
        6, and the phase-stacked '#up6' entries of the up-ResBlock conv1s), and check the up-phase tap stacks against the
        module weights, and the stride-2 convs' 2x2 tap stacks (space-to-depth operand) likewise.  The UNet executor
        keeps its modules on eng.unet, the VQGAN executor on eng.vq."""
        root = eng.vq if hasattr(eng, "vq") else eng.unet
        for name, ent in eng._w.items():
            if not isinstance(ent, dict):
                continue
            mod = name[:-len("#up6")] if name.endswith("#up6") else name
            if "u_hi" in ent:
                w = root.get_submodule(mod).weight.detach()
                self._weights[ent["u_hi"].data_ptr()] = (w, name.endswith("#up6"), name)
                self._packed.pop(ent["u_hi"].data_ptr(), None)
            if "up_hi" in ent:
                w = root.get_submodule(mod).weight.detach()
                d = image_devs(planes(ent["up_hi"], ent["up_lo"])[None], up_phase_reference(w)[None])
                self._record(-1, "pack_weight_split_taps", "up-phase stack", "phase taps vs module weight", d,
                             self.bounds["up_phase"], [tuple(ent["up_hi"].shape)])
            for key, origin in (("s2_hi", -1), ("ds_hi", 0)):     # UNet Downsample / VQGAN Downsample
                if key in ent:
                    w = root.get_submodule(mod).weight.detach()
                    got = planes(ent[key], ent[key[:2] + "_lo"])
                    d = image_devs(got[None], s2d_tap_reference(w, origin)[None])
                    self._record(-1, "pack_weight_split_taps", f"s2d stack origin {origin}",
                                 "s2d taps vs module weight", d, PAIR, [tuple(got.shape)])

    def _record(self, idx, method, form, what, devs, bound, shapes):
        dev = float(devs.max()) if isinstance(devs, torch.Tensor) and devs.numel() else float(devs)
        self.checks.append(Check(idx, method, form, what, dev, bound, shapes))

    def failures(self):
        return [c for c in self.checks if not c.dev <= c.bound]

    def flagged_launches(self):
        return sorted({c.launch for c in self.failures()})

    def families(self):
        """{(method, what): (checks, worst deviation, bound)}"""
        fam = {}
        for c in self.checks:
            k = (c.method, c.what)
            n, worst, _ = fam.get(k, (0, 0.0, c.bound))
            fam[k] = (n + 1, max(worst, c.dev), c.bound)
        return fam

    def table(self, title):
        lines = [f"{title}: {len(self.launches)} launches, {len(self.checks)} checks",
                 "  launches per method: " + ", ".join(f"{m} {n}" for m, n in
                                                       sorted(collections.Counter(m for m, _ in self.launches).items()))]
        if self.captured:
            lines.append("  captured, not checked: " + ", ".join(f"{m} {n}" for m, n in
                                                                 sorted(collections.Counter(self.captured).items())))
        for (m, what), (n, worst, bound) in sorted(self.families().items()):
            lines.append(f"  {m:22s} {what:34s} {n:5d}  worst {worst:.2e}  bound {bound:.1e}")
        return "\n".join(lines)

    def forms(self):
        return collections.Counter(self.launches)

    # -- the wrapper -------------------------------------------------------------------------------------------
    def __getattr__(self, name):
        attr = getattr(self.be, name)
        if name in NOT_LAUNCHES or name == "check_fault" or not callable(attr):
            return attr
        if name not in OUTPUTS:
            raise NotImplementedError(f"no fp64 reference for launch {name}")
        sig = inspect.signature(attr)

        def launch(*args, **kwargs):
            if _capturing():
                # a stream capture records the launch for later replays: no copy, synchronisation or fault-word read
                # may run inside it, and its outputs do not exist yet
                self.captured.append(name)
                return attr(*args, **kwargs)
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            a = dict(bound.arguments)
            outs = {k for k in OUTPUTS[name] if isinstance(a.get(k), torch.Tensor)}
            out_ptrs = {a[k].untyped_storage().data_ptr() for k in outs}
            ins = {k: v for k, v in a.items() if isinstance(v, torch.Tensor) and k not in outs}
            big = {k for k, v in ins.items() if v.numel() * v.element_size() >= BIG}
            clones = {k: v.clone() for k, v in ins.items() if k not in big}
            prints = {k: fingerprint(ins[k]) for k in big}
            pre = {k: a[k].clone() for k in outs} if name in ("pack_weight_split",) + TABLE_LAUNCHES else {}
            tab = a.get("tab") if name in TABLE_LAUNCHES else None
            if tab is not None:         # what the launch reads through the table's pointer arrays
                pre["params"] = [p.detach().clone() for p in tab.tensors]
                pre["grads"] = [None if p.grad is None else p.grad.clone() for p in tab.tensors]
            r = attr(*args, **kwargs)
            dev = next((v.device for v in a.values() if isinstance(v, torch.Tensor)), None) or tab.device
            if dev.type == "cuda":
                torch.cuda.synchronize(dev)
            self.be.check_fault()
            idx = len(self.launches)
            form = self._form(name, a)
            if idx in self.mutate:
                self.mutate[idx](a)
            self.launches.append((name, form))
            shapes = [tuple(v.shape) for v in a.values() if isinstance(v, torch.Tensor)]
            for k, v in ins.items():
                if v.untyped_storage().data_ptr() not in out_ptrs:
                    same = fingerprint(v) == prints[k] if k in big else bits_equal(v, clones[k])
                    self._record(idx, name, form, "inputs unchanged", 0.0 if same else math.inf, 0.0,
                                 [(k, tuple(v.shape))])
            if tab is not None:         # adam_multi(_dev) reads the gradients, ema_multi the parameters
                adam = name != "ema_multi"
                read = [p.grad for p in tab.tensors] if adam else [p.detach() for p in tab.tensors]
                want = pre["grads"] if adam else pre["params"]
                same = all((g is None) == (w is None) and (g is None or bits_equal(g, w)) for g, w in zip(read, want))
                self._record(idx, name, form, "inputs unchanged", 0.0 if same else math.inf, 0.0,
                             [("tab", len(tab.tensors))])
            c = dict(a, **clones)            # the launch's arguments, inputs replaced by their clones
            c["_prints"] = prints
            getattr(self, "_ref_" + name)(idx, form, shapes, c, a, pre)
            del c, clones
            if dev.type == "cuda":
                torch.cuda.empty_cache()     # the references' multi-GB temporaries must not fragment the executor's pool
            return r
        return launch

    def _form(self, name, a):
        f = []
        if name == "conv_umma":
            if a["weights_per_image"]:
                return "position GEMMs"
            f.append(f"taps {a['taps']}")
            if a.get("window_origin", 0):
                f.append(f"origin {a['window_origin']}")
            if a["w_hi"].data_ptr() in self._dgrad_w:        # a training data gradient (each plane set is read once)
                self._dgrad_w.discard(a["w_hi"].data_ptr())
                f.append("dgrad")
            f += [t for t, on in (("upsample2x", a["upsample2x"]), ("fused 1x1", a["Cin2"]),
                                  ("NCHW head", a["out_nchw_channels"]), ("split out", a["out_hi"] is not None),
                                  ("stats", a["stats_partial"] is not None)) if on]
            if a["res_mode"]:
                f.append(f"res {a['res_mode']}")
            if a["Cin"] >= 4096:           # the VQGAN AttnBlock's O = P V: K = T = 4096 positive products
                f.append("long K")
        elif name in ("wino_input", "wino_output", "wino_pack_weight"):
            f.append(f"F({a.get('tile', 4)},3)")
            if name == "wino_pack_weight" and a["dgrad"]:
                f.append("dgrad")
            if name == "wino_input":
                f += [t for t, on in (("two-source", a["src2"] is not None), ("raw planes", a["raw_hi"] is not None),
                                      ("act planes", a["act_hi"] is not None), ("down2", a.get("down2")),
                                      ("identity", a["mean"] is None)) if on]
            elif name == "wino_output":
                if a.get("up2_phases"):
                    f.append("up2_phases")
                if a["res_mode"]:
                    f.append(f"res {a['res_mode']}")
        elif name == "prep":
            f.append("gn" if a["mean"] is not None else "raw")
            f += [t for t, on in (("two-source", a["src2"] is not None), ("film", a["film_scale"] is not None),
                                  (f"resample {a['resample']}", a["resample"])) if on]
        elif name == "split_grad":
            f += [t for t, on in (("planes", a["hi"] is not None), ("colsum", a["colsum"] is not None)) if on]
        elif name == "conv_wgrad":
            f.append(f"taps {a['taps']}")
            if a["taps"] == 4:
                f.append(f"origin {a.get('window_origin', 0)}")
        elif name == "conv_wgrad_direct":
            f.append(f"taps {a['k'] ** 2}")
            if a["x"].shape[3] * a["dy"].shape[3] > 1024:
                f.append("beyond 1024 channel pairs")
        elif name in ("gn_bwd_reduce", "gn_bwd_apply"):
            f += [t for t, on in (("film", a["fscale"] is not None), ("no act", not a["silu"])) if on]
        elif name == "attention_bwd":
            f.append(f"order {a['order']}")
        elif name in ("adam_multi", "adam_multi_dev"):
            # adam_multi_dev increments its step counter first: the form names the step it takes, as adam_multi's
            f.append(f"step {a['step'] if name == 'adam_multi' else int(a['step'].item())}")
            if a["ema_shadow"] is not None:
                f.append("ema")
        elif name in ("p_sample", "p_sample_dev"):
            f += [t for t, on in (("last" if a["is_last"] else "not last", True), ("clip", a["clip"])) if on]
        elif name == "conv_direct_pad":
            f.append(f"k {a['k']} stride {a['stride']} pad ({a['pad_lo']}, {a['pad_hi']})")
        elif name == "softmax_rows_split":
            f.append(f"{a['src'].shape[-1]} columns")
        elif name == "spatial_rescale":
            f.append(f"{a['n_stages']} stages")
            if a["weight"] is not None:
                f.append("1x1 map")
        elif name == "denorm_to_uint8" and a["to_normal"]:
            f.append("to_normal")
        return " ".join(f)

    # -- references: layout / dense ----------------------------------------------------------------------------
    def _ref_nchw_to_nhwc_cat(self, idx, form, shapes, c, a, pre):
        want = torch.cat([c["x"], c["ctx"]], 1) if c["ctx"] is not None else c["x"]
        self._record(idx, "nchw_to_nhwc_cat", form, "copy", image_equal(a["out"], want.permute(0, 2, 3, 1)),
                     0.0, shapes)

    def _ref_nhwc_to_nchw(self, idx, form, shapes, c, a, pre):
        self._record(idx, "nhwc_to_nchw", form, "copy", image_equal(a["out"], c["src"].permute(0, 3, 1, 2)), 0.0,
                     shapes)

    def _ref_gather_rows(self, idx, form, shapes, c, a, pre):
        self._record(idx, "gather_rows", form, "copy", image_equal(a["out"], c["table"][c["idx"]]), 0.0, shapes)

    def _ref_linear(self, idx, form, shapes, c, a, pre):
        z = c["x"].to(F64)
        z = F.silu(z) if c["act_in"] else z
        z = z @ c["w"].to(F64).t() + (0 if c["bias"] is None else c["bias"].to(F64))
        z = F.silu(z) if c["act_out"] else z
        self._record(idx, "linear", form, "out", image_devs(a["out"], z), self.bounds["linear"], shapes)

    # -- group norm / prep -------------------------------------------------------------------------------------
    def _check_stats(self, idx, method, form, shapes, mean, rstd, m_want, r_want, bound):
        """mean in units of the group's standard deviation (what (x - mean) * rstd sees), rstd relative; per image."""
        dm = ((mean.to(F64) - m_want).abs() * r_want).amax(1)
        self._record(idx, method, form, "mean", torch.nan_to_num(dm, nan=math.inf), bound, shapes)
        self._record(idx, method, form, "rstd", image_devs(rstd, r_want), bound, shapes)

    @staticmethod
    def _moments(s, sq, n, eps):
        m = s / n
        return m, 1.0 / torch.sqrt((sq / n - m * m).clamp_min(0) + eps)

    def _ref_gn_stats(self, idx, form, shapes, c, a, pre):
        x = cat(c["src1"], c["src2"])
        B, H, W, C = x.shape
        g = c["groups"]
        ms, rs = [], []
        for sl in chunks(B, H * W * C * 8, x.device):
            xg = x[sl].to(F64).reshape(-1, H * W, g, C // g)
            ms.append(xg.mean((1, 3)))
            rs.append(1.0 / torch.sqrt(xg.var((1, 3), unbiased=False) + c["eps"]))
        self._check_stats(idx, "gn_stats", form, shapes, a["mean"], a["rstd"], torch.cat(ms), torch.cat(rs),
                          self.bounds["gn_stats"])

    def _ref_gn_finalize_partials(self, idx, form, shapes, c, a, pre):
        B, g = c["B"], c["groups"]
        s = [c["part1"].to(F64).view(B, c["rows1"], -1, 2).sum(1)]
        if c["part2"] is not None:
            s.append(c["part2"].to(F64).view(B, c["rows2"], -1, 2).sum(1))
        s = torch.cat(s, 1)
        C = s.shape[1]
        sg = s.view(B, g, C // g, 2).sum(2)
        m, r = self._moments(sg[..., 0], sg[..., 1], c["hw"] * (C // g), c["eps"])
        self._check_stats(idx, "gn_finalize_partials", form, shapes, a["mean"], a["rstd"], m, r,
                          self.bounds["gn_finalize"])

    def _ref_prep(self, idx, form, shapes, c, a, pre):
        x = cat(c["src1"], c["src2"])
        B, H, W, C = x.shape
        res = c["resample"]
        dv = collections.defaultdict(list)
        for sl in chunks(B, H * W * C * 8 * 8, x.device):
            if c["mean"] is not None:
                act = O.op_resample(gn_act(x, c, sl), res)
                if a["act_f32"] is not None:
                    dv["act_f32"].append(image_devs(a["act_f32"][sl], act))
                if a["act_hi"] is not None:
                    dv["act planes"].append(image_devs(planes(a["act_hi"][sl], a["act_lo"][sl]), act))
                    dv["act planes split"].append(self._split_of(a["act_hi"][sl], a["act_lo"][sl], a["act_f32"], sl))
            if a["raw_f32"] is not None or a["raw_hi"] is not None:
                raw = O.op_resample(x[sl].to(F64), res)
                if a["raw_f32"] is not None:
                    dv["raw_f32"].append(image_devs(a["raw_f32"][sl], raw))
                if a["raw_hi"] is not None:
                    dv["raw planes"].append(image_devs(planes(a["raw_hi"][sl], a["raw_lo"][sl]), raw))
                    dv["raw planes split"].append(self._split_of(a["raw_hi"][sl], a["raw_lo"][sl], a["raw_f32"], sl))
        bound = {"act_f32": self.bounds["prep_act"], "act planes": self.bounds["prep_act_planes"], "raw_f32": self.bounds["prep_raw"],
                 "raw planes": self.bounds["prep_raw_planes"]}
        for what, devs in dv.items():
            self._record(idx, "prep", form, what, torch.cat(devs), bound.get(what, 0.0), shapes)

    @staticmethod
    def _split_of(hi, lo, f32, sl):
        """The planes are bf16(v), bf16(v - hi) of the launch's own fp32 output v where it writes one, else a well-formed
        pair."""
        if f32 is None:
            return pair_well_formed(hi, lo)
        h, l = split_bf16(f32[sl])
        return torch.maximum(image_equal(hi, h), image_equal(lo, l))

    # -- weight packing ----------------------------------------------------------------------------------------
    def _ref_pack_weight_split(self, idx, form, shapes, c, a, pre):
        w = c["w"]
        while w.dim() < 4:
            w = w.unsqueeze(-1)
        cout, cin, k = w.shape[0], w.shape[1], w.shape[2]
        h, l = split_bf16(w.permute(2, 3, 0, 1).reshape(k * k, cout, cin).contiguous())
        want_hi, want_lo = pre["hi"].clone(), pre["lo"].clone()       # padding rows beyond Cout: left as they were
        want_hi[:, :cout], want_lo[:, :cout] = h, l
        ok = bits_equal(a["hi"], want_hi) and bits_equal(a["lo"], want_lo)
        self._record(idx, "pack_weight_split", form, "split planes", 0.0 if ok else math.inf, 0.0, shapes)

    def _ref_pack_weight_split_taps(self, idx, form, shapes, c, a, pre):
        h, l = split_bf16(c["w"].permute(2, 0, 1).contiguous())
        ok = bits_equal(a["hi"], h) and bits_equal(a["lo"], l)
        self._record(idx, "pack_weight_split_taps", form, "split planes", 0.0 if ok else math.inf, 0.0, shapes)

    def _ref_pack_weight_f32(self, idx, form, shapes, c, a, pre):
        w = c["w"]
        while w.dim() < 4:
            w = w.unsqueeze(-1)
        k = w.shape[2]
        ok = bits_equal(a["out"], w.permute(2, 3, 1, 0).reshape(k * k, w.shape[1], w.shape[0]).contiguous())
        self._record(idx, "pack_weight_f32", form, "fp32 planes", 0.0 if ok else math.inf, 0.0, shapes)

    def _ref_wino_pack_weight(self, idx, form, shapes, c, a, pre):
        t = c.get("tile", 4)
        w = c["w"].to(F64)
        if c["dgrad"]:
            w = w.flip(2, 3).transpose(0, 1)
        s = 256.0
        if a["inv_wscale"] is not None:
            inv = float(a["inv_wscale"].item())
            pow2 = inv > 0 and math.frexp(inv)[0] == 0.5
            self._record(idx, "wino_pack_weight", form, "scale is a power of two", 0.0 if pow2 else math.inf, 0.0,
                         shapes)
            s = 1.0 / inv
        g = _mat(G, t, w.device)
        U = torch.einsum("ij,kcjl,ml->imkc", g, w, g).reshape(a["u_hi"].shape) * s
        self._record(idx, "wino_pack_weight", form, f"U planes F({t},3)", image_devs(planes(a["u_hi"], a["u_lo"])[None],
                                                                                   U[None]),
                     self.bounds[f"pack_wino{t}"], shapes)
        # the weight the chain through these planes computes with (register_engine's entries take precedence)
        self._packed[a["u_hi"].data_ptr()] = (c["w"], bool(c["dgrad"]))

    # -- convolutions ------------------------------------------------------------------------------------------
    def _stats_check(self, idx, method, form, shapes, out, part, B):
        """GroupNorm partial sums: the rows of each image summed against the fp64 sums of the launch's own output (the
        consumer, gn_finalize_partials, reads only these per-image sums)."""
        rows = part.shape[0] // B
        got = part.to(F64).view(B, rows, -1, 2).sum(1)
        devs = []
        for sl in chunks(B, out[0].numel() * 8 * 2, out.device):
            o = out[sl].to(F64).reshape(out[sl].shape[0], -1, out.shape[-1])
            want = torch.stack([o.sum(1), (o * o).sum(1)], -1)
            g = got[sl]
            devs.append(torch.maximum(image_devs(g[..., 0], want[..., 0]), image_devs(g[..., 1], want[..., 1])))
        self._record(idx, method, form, "GroupNorm partial sums", torch.cat(devs), self.bounds["stats"], shapes)

    def _ref_conv_umma(self, idx, form, shapes, c, a, pre):
        if c["weights_per_image"]:
            return self._ref_position_gemms(idx, form, shapes, c, a)
        B, H, W, Cin, Cout, taps = c["B"], c["H"], c["W"], c["Cin"], c["Cout"], c["taps"]
        f = 2 if c["upsample2x"] else 1
        Ho, Wo = f * H, f * W
        wh, wl = c["w_hi"].to(F64), c["w_lo"].to(F64)
        if c["upsample2x"]:
            # 4 output phases x 2x2 taps on the low-res operand: phase (pa, pb), tap (r, s) reads source row y + r - 1 + pa
            assert taps == 4
            tap_of = lambda w: [[(r + pa, s + pb, w[(2 * pa + pb) * 4 + 2 * r + s]) for r in range(2) for s in range(2)]
                                for pa in range(2) for pb in range(2)]
        elif taps == 9:
            tap_of = lambda w: [[(ky, kx, w[3 * ky + kx]) for ky in range(3) for kx in range(3)]]
        elif taps == 4:     # 2x2 window at rows / columns o..o+1 (window_origin o = 0 or -1), zero padding outside
            o0 = 1 + c.get("window_origin", 0)
            tap_of = lambda w: [[(o0 + r, o0 + s, w[2 * r + s]) for r in range(2) for s in range(2)]]
        else:
            assert taps == 1
            tap_of = lambda w: [[(1, 1, w[0])]]
        passes = c["passes"]
        res = c["residual"]
        if res is not None:
            rs = {1: (Ho, Wo), 2: (Ho // 2, Wo // 2), 3: (2 * Ho, 2 * Wo)}[c["res_mode"]]
            res = res.reshape(B, rs[0], rs[1], Cout)
        a_hi, a_lo = c["a_hi"].reshape(B, H, W, Cin), c["a_lo"].reshape(B, H, W, Cin)
        dv = collections.defaultdict(list)
        nchw = c["out_nchw_channels"]
        for sl in chunks(B, (H + 2) * (W + 2) * Cin * 8 * 4 + Ho * Wo * Cout * 8 * 2, a_hi.device):
            ah = F.pad(a_hi[sl].to(F64), (0, 0, 1, 1, 1, 1))
            av = ah + F.pad(a_lo[sl].to(F64), (0, 0, 1, 1, 1, 1))
            # split products A_hi W_hi + A_lo W_hi + A_hi W_lo (passes 3), or A_hi W_hi (passes 1), in fp64
            phases = []
            for tl_h, tl_l in zip(tap_of(wh), tap_of(wl)):
                o = tap_conv(av if passes == 3 else ah, tl_h, H, W)
                if passes == 3:
                    o = o.add_(tap_conv(ah, tl_l, H, W))
                phases.append(o)
            if c["upsample2x"]:
                o = torch.empty(phases[0].shape[0], Ho, Wo, Cout, dtype=F64, device=ah.device)
                for ph, p in enumerate(phases):
                    o[:, ph >> 1::2, ph & 1::2] = p
            else:
                o = phases[0]
            if c["Cin2"]:
                a2h = c["a2_hi"].reshape(B, H, W, -1)[sl].to(F64)
                a2v = a2h + c["a2_lo"].reshape(B, H, W, -1)[sl].to(F64)
                w2h, w2l = c["w2_hi"][0].to(F64), c["w2_lo"][0].to(F64)
                n = a2h.shape[0]
                o2 = (a2v if passes == 3 else a2h).reshape(-1, c["Cin2"]) @ w2h.t()
                if passes == 3:
                    o2 += a2h.reshape(-1, c["Cin2"]) @ w2l.t()
                o = o + o2.view(n, H, W, Cout)
                if c["bias2"] is not None:
                    o = o + c["bias2"].to(F64)
            if c["bias"] is not None:
                o = o + c["bias"].to(F64)
            o = add_residual(o, None if res is None else res[sl], c["res_mode"])
            if nchw:
                dv["out"].append(image_devs(a["out"][sl], o[..., :nchw].permute(0, 3, 1, 2)))
            elif a["out"] is not None:
                dv["out"].append(image_devs(a["out"][sl].reshape(o.shape), o))
            if a["out_hi"] is not None:
                hi, lo = a["out_hi"][sl].reshape(o.shape), a["out_lo"][sl].reshape(o.shape)
                if a["out"] is None:
                    dv["out planes"].append(image_devs(planes(hi, lo), o))
                dv["out planes split"].append(self._split_of(hi, lo, None if a["out"] is None else
                                                             a["out"].reshape(B, Ho, Wo, Cout), sl))
        bound = {"out": self.bounds["conv_umma"], "out planes": self.bounds["conv_umma_planes"]}
        for what, devs in dv.items():
            self._record(idx, "conv_umma", form, what, torch.cat(devs), bound.get(what, 0.0), shapes)
        if a["stats_partial"] is not None:
            self._stats_check(idx, "conv_umma", form, shapes, a["out"].reshape(B, Ho, Wo, Cout), a["stats_partial"], B)

    def _ref_position_gemms(self, idx, form, shapes, c, a):
        P, Cout = c["B"], c["Cout"]
        V = c["a_hi"].reshape(P, -1, c["Cin"])
        Vl = c["a_lo"].reshape(P, -1, c["Cin"])
        m = a["out"].reshape(P, -1, Cout)
        devs = []
        for sl in chunks(P, V.shape[1] * (c["Cin"] + Cout) * 8 * 2, V.device):
            want = torch.bmm(planes(V[sl], Vl[sl]), planes(c["w_hi"][sl], c["w_lo"][sl]).transpose(1, 2))
            devs.append(image_devs(m[sl], want))
        self._record(idx, "conv_umma", form, "Winograd M (per position)", torch.cat(devs), self.bounds["wino_m"], shapes)
        src = self._wino_in.pop(a["a_hi"].data_ptr(), None)
        self._wino_m[a["out"].data_ptr()] = dict(launch=idx, input=src, u=a["w_hi"].data_ptr())

    def _ref_conv_direct(self, idx, form, shapes, c, a, pre):
        src, k, cout, stride = c["src"], c["k"], c["Cout"], c["stride"]
        w = c["w_packed"].reshape(k, k, src.shape[3], cout).permute(3, 2, 0, 1).to(F64)
        devs = []
        for sl in chunks(src.shape[0], src[0].numel() * 8 * 4, src.device):
            o = F.conv2d(src[sl].to(F64).permute(0, 3, 1, 2), w, None if c["bias"] is None else c["bias"].to(F64),
                         stride=stride, padding=k // 2).permute(0, 2, 3, 1)
            if c["residual"] is not None:
                o = o + c["residual"][sl].to(F64)
            devs.append(image_devs(a["out"][sl], o))
        self._record(idx, "conv_direct", form, "out", torch.cat(devs), self.bounds["conv_direct"], shapes)

    def _ref_conv_stem(self, idx, form, shapes, c, a, pre):
        src, cout = c["src"], c["Cout"]
        B, H, W, cin = src.shape
        w = c["w_packed"].reshape(3, 3, cin, cout).permute(3, 2, 0, 1).to(F64)
        devs = []
        for sl in chunks(B, H * W * (cin + cout) * 8 * 2, src.device):
            o = F.conv2d(src[sl].to(F64).permute(0, 3, 1, 2), w, None if c["bias"] is None else c["bias"].to(F64),
                         padding=1).permute(0, 2, 3, 1)
            devs.append(image_devs(a["out"][sl], o))
        self._record(idx, "conv_stem", form, "out", torch.cat(devs), self.bounds["conv_stem"], shapes)
        if a["stats_partial"] is not None:
            self._stats_check(idx, "conv_stem", form, shapes, a["out"], a["stats_partial"], B)

    # -- Winograd ----------------------------------------------------------------------------------------------
    def _wino_act(self, rec, sl):
        """fp64 input of the 3x3 conv of a wino_input launch (activation, 2x2-pooled for down2), images sl."""
        c = rec["args"]
        act = gn_act(cat(c["src1"], c["src2"]), c, sl)
        return pool2(act) if c.get("down2") else act

    @staticmethod
    def _inputs_intact(rec):
        """Whether the inputs of a wino_input launch that the shadow did not copy still hold what that launch read (the
        whole-chain check reads them at the output transform)."""
        return all(fingerprint(rec["args"][k]) == p for k, p in rec["args"]["_prints"].items())

    def _ref_wino_input(self, idx, form, shapes, c, a, pre):
        t = c.get("tile", 4)
        x = cat(c["src1"], c["src2"])
        B, Hs, Ws, C = x.shape
        rec = dict(launch=idx, args=c, tile=t)
        H, W = (Hs // 2, Ws // 2) if c.get("down2") else (Hs, Ws)
        th, tw = -(-H // t), -(-W // t)
        npos = (t + 2) ** 2
        bt = _mat(BT, t, x.device)
        vh, vl = a["v_hi"], a["v_lo"]
        dv = collections.defaultdict(list)
        for sl in chunks(B, Hs * Ws * C * 8 * 3 + npos * th * tw * C * 8 * 3, x.device):
            act = self._wino_act(rec, sl)
            n = act.shape[0]
            pad = (0, 0, 1, t * tw + 1 - W, 1, t * th + 1 - H)
            tiles = F.pad(act, pad).unfold(1, t + 2, t).unfold(2, t + 2, t)          # [n, th, tw, C, t+2, t+2]
            V = torch.einsum("ij,nxycjk,lk->nilxyc", bt, tiles, bt).reshape(n, npos, th * tw, C)
            rows = slice(sl.start * th * tw, sl.stop * th * tw)
            got = planes(vh[:, rows], vl[:, rows]).reshape(npos, n, th * tw, C).transpose(0, 1)
            dv[f"V F({t},3)"].append(image_devs(got, V))
            if c["raw_hi"] is not None:
                h, l = split_bf16(x[sl].float())
                dv["raw planes (bit-exact split)"].append(torch.maximum(image_equal(a["raw_hi"][sl], h),
                                                                        image_equal(a["raw_lo"][sl], l)))
            if c["act_hi"] is not None:
                dv["act planes"].append(image_devs(planes(a["act_hi"][sl], a["act_lo"][sl]), gn_act(x, c, sl)))
                dv["act planes split"].append(pair_well_formed(a["act_hi"][sl], a["act_lo"][sl]))
        bound = {f"V F({t},3)": self.bounds[f"wino_v{t}"], "act planes": self.bounds["wino_act_planes"]}
        for what, devs in dv.items():
            self._record(idx, "wino_input", form, what, torch.cat(devs), bound.get(what, 0.0), shapes)
        zero = bool((vh[:, B * th * tw:] == 0).all()) and bool((vl[:, B * th * tw:] == 0).all())
        self._record(idx, "wino_input", form, "GEMM padding rows zero", 0.0 if zero else math.inf, 0.0, shapes)
        self._wino_in[vh.data_ptr()] = rec

    def _ref_wino_output(self, idx, form, shapes, c, a, pre):
        t, B, H, W, Cout = c.get("tile", 4), c["B"], c["H"], c["W"], c["Cout"]
        up = c.get("up2_phases", False)
        th, tw = -(-H // t), -(-W // t)
        ncols = 4 * Cout if up else Cout
        inv = 1.0 / 256.0 if c["inv_wscale"] is None else float(c["inv_wscale"].item())
        at = _mat(AT, t, c["m"].device)
        f = 2 if up else 1
        Ho, Wo = f * H, f * W
        res = c["residual"]
        if res is not None:
            rs = {1: (Ho, Wo), 2: (Ho // 2, Wo // 2), 3: (2 * Ho, 2 * Wo)}[c["res_mode"]]
            res = res.reshape(B, rs[0], rs[1], Cout)
        bias = 0.0 if c["bias"] is None else c["bias"].to(F64)
        chain = self._wino_m.pop(a["m"].data_ptr(), None)
        src = None if chain is None else chain["input"]
        wt = None if chain is None else self._weights.get(chain["u"])
        packed = None if chain is None else self._packed.pop(chain["u"], None)     # a freed address must not pair again
        dgrad = False
        if wt is None and packed is not None:
            w, dgrad = packed
            wt = (w.to(F64).flip(2, 3).transpose(0, 1) if dgrad else w, False, "packed with the launch")
        whole = f"chain F({t},3){' dgrad' if dgrad else ''} vs fp64 conv"
        out = a["out"]
        dv = collections.defaultdict(list)
        M = c["m"].reshape((t + 2) ** 2, -1, ncols)
        for sl in chunks(B, th * tw * (t + 2) ** 2 * ncols * 8 * 3 + Ho * Wo * Cout * 8 * 4, out.device):
            n = out[sl].shape[0]
            Mb = M[:, sl.start * th * tw:sl.stop * th * tw].to(F64).reshape(t + 2, t + 2, n, th, tw, ncols)
            Y = torch.einsum("ij,jlnxyc,ml->nxiymc", at, Mb, at) * inv
            y = Y.reshape(n, t * th, t * tw, ncols)[:, :H, :W]
            if up:     # phase-major channels -> output pixel (2y + ph // 2, 2x + ph % 2)
                yy = torch.empty(n, Ho, Wo, Cout, dtype=F64, device=y.device)
                for ph in range(4):
                    yy[:, ph >> 1::2, ph & 1::2] = y[..., ph * Cout:(ph + 1) * Cout]
                y = yy
            r = None if res is None else res[sl]
            dv["Y = A^T M A / s"].append(image_devs(out[sl], add_residual(y + bias, r, c["res_mode"])))
            if src is not None and wt is not None and self._inputs_intact(src):
                act = self._wino_act(src, sl)
                w, w_up, _ = wt
                want = conv3x3(up2(act) if w_up else act, w.to(act.device, F64)) + bias
                dv[whole].append(image_devs(out[sl], add_residual(want, r, c["res_mode"])))
        if chain is None or src is None or wt is None or not self._inputs_intact(src):
            # an output transform whose GEMM, input transform or weight the shadow did not see cannot be checked whole
            dv[whole].append(torch.tensor([math.inf], dtype=F64))
        bound = {"Y = A^T M A / s": self.bounds["wino_y"], whole: self.bounds[f"chain{t}{'_dgrad' if dgrad else ''}"]}
        for what, devs in dv.items():
            self._record(idx, "wino_output", form, what, torch.cat([d.cpu() for d in devs]), bound[what], shapes)
        if a["stats_partial"] is not None:
            self._stats_check(idx, "wino_output", form, shapes, out, a["stats_partial"], B)

    # -- attention ---------------------------------------------------------------------------------------------
    def _attention(self, idx, name, form, shapes, qkv, c, a):
        B, T, C3 = qkv.shape
        dv = collections.defaultdict(list)
        for sl in chunks(B, T * T * 8 * 2 + T * C3 * 8, qkv.device):
            o = attention_ref(qkv[sl].to(F64) if qkv.dtype != F64 else qkv[sl], c["heads"], c["order"],
                              slice(0, qkv[sl].shape[0]))
            if a["out_f32"] is not None:
                dv["out"].append(image_devs(a["out_f32"][sl], o))
            if a["out_hi"] is not None:
                if a["out_f32"] is None:
                    dv["out planes"].append(image_devs(planes(a["out_hi"][sl], a["out_lo"][sl]), o))
                dv["out planes split"].append(self._split_of(a["out_hi"][sl], a["out_lo"][sl], a["out_f32"], sl))
        bound = {"out": self.bounds["attention"], "out planes": self.bounds["attention_planes"]}
        for what, devs in dv.items():
            self._record(idx, name, form, what, torch.cat(devs), bound.get(what, 0.0), shapes)

    def _ref_attention(self, idx, form, shapes, c, a, pre):
        self._attention(idx, "attention", form, shapes, c["qkv"], c, a)

    def _ref_attention_split(self, idx, form, shapes, c, a, pre):
        self._attention(idx, "attention_split", form, shapes, planes(c["qkv_hi"], c["qkv_lo"]), c, a)

    def _ref_attention_tc(self, idx, form, shapes, c, a, pre):
        self._attention(idx, "attention_tc", form, shapes, planes(c["qkv_hi"], c["qkv_lo"]), c, a)

    # -- training: bridge, gradient operands, weight packing -----------------------------------------------------
    def _ref_q_sample(self, idx, form, shapes, c, a, pre):
        """The oracle's expression on the CPU, as test_gpu_kernels.py::test_q_sample_bit_exact holds the kernel to."""
        cpu = lambda k: c[k].cpu()
        xt, obj = O.q_sample({"m_t": cpu("m_t"), "variance_t": cpu("var_t")}, cpu("x0"), cpu("y"), cpu("t"),
                             cpu("noise"), c["objective"])
        for what, got, want in (("x_t", a["xt_out"], xt), ("objective", a["obj_out"], obj)):
            self._record(idx, "q_sample", form, what, image_equal(got.cpu(), want), 0.0, shapes)

    def _ref_split_grad(self, idx, form, shapes, c, a, pre):
        src = c["src"]
        h, l = split_bf16(src.reshape(-1, src.shape[-1]))
        if a["hi"] is not None:
            self._record(idx, "split_grad", form, "planes (bit-exact split)",
                         torch.maximum(image_equal(a["hi"], h.reshape(a["hi"].shape)),
                                       image_equal(a["lo"], l.reshape(a["lo"].shape))), 0.0, shapes)
        if a["hi_t"] is not None:
            ok = bits_equal(a["hi_t"], h.t().contiguous()) and bits_equal(a["lo_t"], l.t().contiguous())
            self._record(idx, "split_grad", form, "transposed planes (bit-exact)", 0.0 if ok else math.inf, 0.0, shapes)
        if a["colsum"] is not None:
            want = src.reshape(-1, src.shape[-1]).to(F64).sum(0)
            self._record(idx, "split_grad", form, "column sums", image_devs(a["colsum"][None], want[None]),
                         self.bounds["colsum"], shapes)

    @staticmethod
    def _dgrad_layout(w):
        """[Cout, Cin, k, k] -> [k*k, Cin, Cout]: the kernel flipped, the channels swapped."""
        k = w.shape[2]
        return w.flip(2, 3).permute(2, 3, 1, 0).reshape(k * k, w.shape[1], w.shape[0]).contiguous()

    def _ref_pack_weight_split_both(self, idx, form, shapes, c, a, pre):
        w = c["w"]
        k = w.shape[2]
        ok = True
        if a["f_hi"] is not None:
            h, l = split_bf16(w.permute(2, 3, 0, 1).reshape(k * k, w.shape[0], w.shape[1]).contiguous())
            ok = bits_equal(a["f_hi"], h) and bits_equal(a["f_lo"], l)
        if a["d_hi"] is not None:
            h, l = split_bf16(self._dgrad_layout(w))
            ok = ok and bits_equal(a["d_hi"], h) and bits_equal(a["d_lo"], l)
            self._dgrad_w.add(a["d_hi"].data_ptr())
        self._record(idx, "pack_weight_split_both", form, "split planes", 0.0 if ok else math.inf, 0.0, shapes)

    def _ref_pack_weight_split_dgrad(self, idx, form, shapes, c, a, pre):
        h, l = split_bf16(self._dgrad_layout(c["w"]))
        ok = bits_equal(a["hi"], h) and bits_equal(a["lo"], l)
        self._dgrad_w.add(a["hi"].data_ptr())
        self._record(idx, "pack_weight_split_dgrad", form, "split planes", 0.0 if ok else math.inf, 0.0, shapes)

    # -- training: weight gradients ------------------------------------------------------------------------------
    @staticmethod
    def _wgrad64(act, grad_rows, k, origin=None):
        """fp64 weight gradient [Cout, Cin, k, k] of a stride-1 conv whose window starts at offset origin (default
        -(k // 2), the 'same' conv): dw[:, :, ky, kx] = sum over pixels p of dY[p] act[p + origin + (ky, kx)]^T, zero
        outside the map.  act [B, H, W, Cin] (any dtype), grad_rows fn(slice of images) -> [Cout, n*H*W] fp64, summed
        over image chunks."""
        B, H, W, Cin = act.shape
        o = -(k // 2) if origin is None else origin
        p = max(-o, k - 1 + o)
        dw = None
        for sl in chunks(B, (H + 2 * p) * (W + 2 * p) * Cin * 8 * 2, act.device):
            ap = F.pad(act[sl].to(F64), (0, 0, p, p, p, p))
            g = grad_rows(sl)
            if dw is None:
                dw = torch.zeros(g.shape[0], Cin, k, k, dtype=F64, device=act.device)
            for ky in range(k):
                for kx in range(k):
                    y0, x0 = p + o + ky, p + o + kx
                    dw[:, :, ky, kx] += g @ ap[:, y0:y0 + H, x0:x0 + W].reshape(-1, Cin)
        return dw

    def _ref_conv_wgrad(self, idx, form, shapes, c, a, pre):
        B, H, W, Cin, Cout, taps = c["B"], c["H"], c["W"], c["Cin"], c["Cout"], c["taps"]
        act = planes(c["a_hi"], c["a_lo"]).reshape(B, H, W, Cin)
        gh, gl = c["g_hi_t"].reshape(Cout, -1), c["g_lo_t"].reshape(Cout, -1)
        rows = lambda sl: planes(gh[:, sl.start * H * W:sl.stop * H * W], gl[:, sl.start * H * W:sl.stop * H * W])
        if taps == 4:       # the 2x2 window at rows / columns o..o+1, o = window_origin
            want = self._wgrad64(act, rows, 2, c.get("window_origin", 0))
        else:
            want = self._wgrad64(act, rows, 3 if taps == 9 else 1)
        self._record(idx, "conv_wgrad", form, "dW", image_devs(a["dw"][None], want[None]), self.bounds["conv_wgrad"],
                     shapes)

    def _ref_conv_wgrad_direct(self, idx, form, shapes, c, a, pre):
        dy = c["dy"]
        B, H, W, Cout = dy.shape
        rows = lambda sl: dy[sl].to(F64).reshape(-1, Cout).t()
        want = self._wgrad64(c["x"], rows, c["k"])
        self._record(idx, "conv_wgrad_direct", form, "dW", image_devs(a["dw"][None], want[None]),
                     self.bounds["conv_wgrad_direct"], shapes)

    # -- training: GroupNorm (+FiLM) (+SiLU) backward ------------------------------------------------------------
    @staticmethod
    def _gn_bwd_terms(c, sl):
        """fp64 (x_hat, dz, rstd, 1 + scale) of images sl, from the fp32 statistics the launch got."""
        x = c["x"][sl].to(F64)
        C, G = x.shape[3], c["groups"]
        e = lambda t: t[sl].to(F64).repeat_interleave(C // G, 1)[:, None, None, :]
        r = e(c["rstd"])
        xh = (x - e(c["mean"])) * r
        f1 = f0 = None
        if c["fscale"] is not None:
            f1 = 1.0 + c["fscale"][sl, :C].to(F64)[:, None, None, :]
            f0 = c["fshift"][sl, :C].to(F64)[:, None, None, :]
        z = c["gamma"].to(F64) * xh + c["beta"].to(F64)
        if f1 is not None:
            z = z * f1 + f0
        da = c["da"][sl].to(F64)
        if c["silu"]:
            sg = torch.sigmoid(z)
            da = da * sg * (1 + z * (1 - sg))
        return xh, da, r, (1.0 if f1 is None else f1)

    def _ref_gn_bwd_reduce(self, idx, form, shapes, c, a, pre):
        B, H, W, C = c["x"].shape
        dv = collections.defaultdict(list)
        for sl in chunks(B, H * W * C * 8 * 6, c["x"].device):
            xh, dz, _, _ = self._gn_bwd_terms(c, sl)
            dv["sum dz"].append(image_devs(a["a12"][sl, :, 0], dz.sum((1, 2))))
            dv["sum dz*x_hat"].append(image_devs(a["a12"][sl, :, 1], (dz * xh).sum((1, 2))))
        for what, devs in dv.items():
            self._record(idx, "gn_bwd_reduce", form, what, torch.cat(devs), self.bounds["gn_bwd"], shapes)

    def _ref_gn_bwd_apply(self, idx, form, shapes, c, a, pre):
        B, H, W, C = c["x"].shape
        G = c["groups"]
        n = H * W * (C // G)
        devs = []
        for sl in chunks(B, H * W * C * 8 * 6, c["x"].device):
            xh, dz, r, f1 = self._gn_bwd_terms(c, sl)
            e = lambda t: t[sl].to(F64).repeat_interleave(C // G, 1)[:, None, None, :]
            want = r * (dz * c["gamma"].to(F64) * f1 - (e(c["s1"]) + xh * e(c["s2"])) / n)
            devs.append(image_devs(a["dx"][sl], want))
        self._record(idx, "gn_bwd_apply", form, "dx", torch.cat(devs), self.bounds["gn_bwd"], shapes)

    # -- training: attention backward, SpatialTransformer pieces -------------------------------------------------
    @staticmethod
    def _attention64(qkv, heads, order):
        """softmax(q k^T / sqrt(d)) v of qkv [n, T, 3C] (fp64, differentiable) -> [n, T, C]."""
        n, T, C3 = qkv.shape
        d = C3 // 3 // heads
        if order:
            q, k, v = qkv.view(n, T, 3, heads, d).unbind(2)
        else:
            q, k, v = qkv.view(n, T, heads, 3, d).unbind(3)
        s = torch.softmax(torch.einsum("nthd,nshd->nhts", q, k) / math.sqrt(d), dim=-1)
        return torch.einsum("nhts,nshd->nthd", s, v).reshape(n, T, C3 // 3)

    @staticmethod
    def _cross64(q, kv, heads):
        """softmax(q k^T / sqrt(d)) v for queries q [n, Tq, C] and k|v kv [n, Tkv, 2C] (fp64) -> [n, Tq, C]."""
        n, Tq, C = q.shape
        d = C // heads
        sp = lambda t: t.reshape(n, t.shape[1], heads, d)
        s = torch.softmax(torch.einsum("nthd,nshd->nhts", sp(q), sp(kv[..., :C])) / math.sqrt(d), dim=-1)
        return torch.einsum("nhts,nshd->nthd", s, sp(kv[..., C:])).reshape(n, Tq, C)

    def _ref_attention_bwd(self, idx, form, shapes, c, a, pre):
        qkv = c["qkv"]
        B, T, C3 = qkv.shape
        devs = []
        for sl in chunks(B, c["heads"] * T * T * 8 * 4 + T * C3 * 8 * 4, qkv.device):
            q = qkv[sl].to(F64).requires_grad_(True)
            with torch.enable_grad():
                self._attention64(q, c["heads"], c["order"]).backward(c["dout"][sl].to(F64))
            devs.append(image_devs(a["dqkv"][sl], q.grad))
        self._record(idx, "attention_bwd", form, "dqkv", torch.cat(devs), self.bounds["attention_bwd"], shapes)

    def _ref_attention_cross(self, idx, form, shapes, c, a, pre):
        q, kv = planes(c["q_hi"], c["q_lo"]), planes(c["kv_hi"], c["kv_lo"])
        B, Tq, _ = q.shape
        dv = collections.defaultdict(list)
        for sl in chunks(B, c["heads"] * Tq * kv.shape[1] * 8 * 3, q.device):
            o = self._cross64(q[sl], kv[sl], c["heads"])
            self._rows_out(dv, a, sl, o)
        self._record_rows(idx, "attention_cross", form, shapes, dv, "attention_cross")

    def _ref_attention_cross_bwd(self, idx, form, shapes, c, a, pre):
        B, Tq, _ = c["q"].shape
        Tkv = c["kv"].shape[1]
        dq, dkv = [], []
        for sl in chunks(B, c["heads"] * Tq * Tkv * 8 * 4, c["q"].device):
            q, kv = c["q"][sl].to(F64).requires_grad_(True), c["kv"][sl].to(F64).requires_grad_(True)
            with torch.enable_grad():
                self._cross64(q, kv, c["heads"]).backward(c["dout"][sl].to(F64))
            dq.append(image_devs(a["dq"][sl], q.grad))
            dkv.append(image_devs(a["dkv"][sl], kv.grad))
        for what, devs in (("dq", dq), ("dkv", dkv)):
            self._record(idx, "attention_cross_bwd", form, what, torch.cat(devs), self.bounds["attention_cross_bwd"],
                         shapes)

    def _rows_out(self, dv, a, sl, want):
        """Row outputs (out_f32 and / or split planes) of images sl against want."""
        shp = lambda t: t[sl].reshape(want.shape)
        if a["out_f32"] is not None:
            dv["out"].append(image_devs(shp(a["out_f32"]), want))
        if a["out_hi"] is not None:
            hi, lo = shp(a["out_hi"]), shp(a["out_lo"])
            if a["out_f32"] is None:
                dv["out planes"].append(image_devs(planes(hi, lo), want))
            dv["out planes split"].append(self._split_of(hi, lo, None if a["out_f32"] is None else
                                                         a["out_f32"].reshape(a["out_f32"].shape[0], *want.shape[1:]),
                                                         sl))

    def _record_rows(self, idx, method, form, shapes, dv, key):
        bound = {"out": self.bounds[key], "out planes": self.bounds.get(key + "_planes", self.bounds[key] + PAIR)}
        for what, devs in dv.items():
            self._record(idx, method, form, what, torch.cat(devs), bound.get(what, 0.0), shapes)

    def _ref_layernorm_split(self, idx, form, shapes, c, a, pre):
        x = c["x"]
        C = x.shape[-1]
        dv = collections.defaultdict(list)
        for sl in chunks(x.shape[0], x[0].numel() * 8 * 3, x.device):
            want = F.layer_norm(x[sl].to(F64), (C,), c["gamma"].to(F64), c["beta"].to(F64), c["eps"])
            self._rows_out(dv, a, sl, want)
        self._record_rows(idx, "layernorm_split", form, shapes, dv, "layernorm")

    def _ref_layernorm_bwd(self, idx, form, shapes, c, a, pre):
        x = c["x"]
        C = x.shape[-1]
        dx = []
        dg = torch.zeros(C, dtype=F64, device=x.device)
        db = torch.zeros_like(dg)
        for sl in chunks(x.shape[0], x[0].numel() * 8 * 4, x.device):
            xd = x[sl].to(F64).requires_grad_(True)
            gd = c["gamma"].to(F64).requires_grad_(True)
            bd = torch.zeros_like(gd, requires_grad=True)
            with torch.enable_grad():
                F.layer_norm(xd, (C,), gd, bd, c["eps"]).backward(c["dy"][sl].to(F64))
            dx.append(image_devs(a["dx"][sl], xd.grad))
            dg += gd.grad
            db += bd.grad
        b = self.bounds["layernorm_bwd"]
        self._record(idx, "layernorm_bwd", form, "dx", torch.cat(dx), b, shapes)
        self._record(idx, "layernorm_bwd", form, "dgamma", image_devs(a["dgamma"][None], dg[None]), b, shapes)
        self._record(idx, "layernorm_bwd", form, "dbeta", image_devs(a["dbeta"][None], db[None]), b, shapes)

    @staticmethod
    def _geglu64(u):
        v, g = u.chunk(2, dim=-1)
        return v * F.gelu(g)

    def _ref_geglu_split(self, idx, form, shapes, c, a, pre):
        u = c["u"]
        dv = collections.defaultdict(list)
        for sl in chunks(u.shape[0], u[0].numel() * 8 * 3, u.device):
            self._rows_out(dv, a, sl, self._geglu64(u[sl].to(F64)))
        self._record_rows(idx, "geglu_split", form, shapes, dv, "geglu")

    def _ref_geglu_bwd(self, idx, form, shapes, c, a, pre):
        u = c["u"]
        devs = []
        for sl in chunks(u.shape[0], u[0].numel() * 8 * 4, u.device):
            ud = u[sl].to(F64).requires_grad_(True)
            with torch.enable_grad():
                self._geglu64(ud).backward(c["dy"][sl].to(F64))
            devs.append(image_devs(a["du"][sl], ud.grad))
        self._record(idx, "geglu_bwd", form, "du", torch.cat(devs), self.bounds["geglu_bwd"], shapes)

    # -- optimizer -----------------------------------------------------------------------------------------------
    def _ref_adam_multi(self, idx, form, shapes, c, a, pre):
        self._adam(idx, "adam_multi", form, shapes, c, a, pre, c["lr"], c["step"])

    def _ref_adam_multi_dev(self, idx, form, shapes, c, a, pre):
        """The capturable step: lr and the step counter are device scalars, read here as they stood before the launch;
        the launch takes step + 1 and leaves exactly that in the counter."""
        s0 = float(pre["step"].item())
        self._record(idx, "adam_multi_dev", form, "step counter + 1", 0.0 if float(a["step"].item()) == s0 + 1 else
                     math.inf, 0.0, shapes)
        self._adam(idx, "adam_multi_dev", form, shapes, c, a, pre, float(c["lr"].item()), int(s0) + 1)

    def _adam(self, idx, method, form, shapes, c, a, pre, lr, step):
        """Per parameter tensor: one fp64 torch.optim.Adam step from the pre-launch parameter, gradient and moments
        (state step = step - 1).

        The update dp = p_new - p_old is compared with the fp64 update, relative to the tensor's largest |dp|.  The
        fp32 parameter cannot hold p_old + dp closer than half its own spacing (at lr 1e-4 that is up to 6e-4 of dp for
        parameters near 1), so what counts is the distance beyond that half-ulp: a kernel that evaluates the update
        exactly scores 0, and one whose update is wrong by more than the parameter's fp32 resolution shows."""
        tab = a["tab"]
        dp, mo, ema = [], [], []
        for i, p in enumerate(tab.tensors):
            g = pre["grads"][i]
            if g is None:
                continue
            o, n = tab.offsets_host[i], tab.numel_host[i]
            p0 = pre["params"][i]
            q = torch.nn.Parameter(p0.to(F64))
            q.grad = g.to(F64)
            ref = torch.optim.Adam([q], lr=lr, betas=(c["beta1"], c["beta2"]), eps=c["eps"],
                                   weight_decay=c["weight_decay"], foreach=False)
            ref.state[q] = {"step": torch.tensor(float(step - 1)),
                            "exp_avg": pre["exp_avg"][o:o + n].view(p.shape).to(F64),
                            "exp_avg_sq": pre["exp_avg_sq"][o:o + n].view(p.shape).to(F64)}
            ref.step()
            p1 = p.detach()
            want = q.detach() - p0.to(F64)
            spacing = (torch.nextafter(p1.abs(), torch.full_like(p1, math.inf)) - p1.abs()).to(F64)
            beyond = ((p1.to(F64) - q.detach()).abs() - 0.5 * spacing).clamp_min(0)
            d = beyond.max() / want.abs().max().clamp_min(1e-30)
            dp.append(torch.nan_to_num(d, nan=math.inf).reshape(1))
            st = ref.state[q]
            mo.append(torch.maximum(image_devs(a["exp_avg"][o:o + n][None], st["exp_avg"].reshape(1, -1)),
                                    image_devs(a["exp_avg_sq"][o:o + n][None], st["exp_avg_sq"].reshape(1, -1))))
            if a["ema_shadow"] is not None:
                s0 = pre["ema_shadow"][o:o + n].to(F64)
                w = (1.0 - c["ema_decay"]) * p1.reshape(-1).to(F64) + c["ema_decay"] * s0
                ema.append(image_devs(a["ema_shadow"][o:o + n][None], w[None]))
        self._record(idx, method, form, "dp beyond fp32 resolution", torch.cat(dp), self.bounds["adam_dp"], shapes)
        self._record(idx, method, form, "exp_avg, exp_avg_sq", torch.cat(mo), self.bounds["adam_moments"], shapes)
        if ema:
            self._record(idx, method, form, "EMA shadow", torch.cat(ema), self.bounds["ema"], shapes)

    def _ref_ema_multi(self, idx, form, shapes, c, a, pre):
        tab = a["tab"]
        devs = []
        for i, p0 in enumerate(pre["params"]):
            o, n = tab.offsets_host[i], tab.numel_host[i]
            w = p0.reshape(-1).to(F64)
            if c["with_decay"]:
                w = (1.0 - c["decay"]) * w + c["decay"] * pre["shadow"][o:o + n].to(F64)
            devs.append(image_devs(a["shadow"][o:o + n][None], w[None]))
        self._record(idx, "ema_multi", form, "EMA shadow", torch.cat(devs), self.bounds["ema"], shapes)

    # -- sampling: bridge update, condition, output path ---------------------------------------------------------
    def _p_sample(self, idx, method, form, shapes, c, a, coef):
        """The reference's update (oracle.p_sample_update, BrownianBridgeModel.py:174-201) evaluated with fp32 torch
        ops on the CPU from the launch's seven step coefficients (schedule.step_coefficients), as
        test_gpu_kernels.py::test_p_sample_update_bit_exact holds the kernel to it: bit for bit."""
        m_t, om_t, sq, m_nt, om_nt, c_xt, sigma = (torch.tensor(float(v), dtype=torch.float32) for v in coef)
        x_t, y, eps = (c[k].cpu().float() for k in ("x_t", "y", "eps"))
        x0 = {"grad": lambda: x_t - eps, "noise": lambda: (x_t - m_t * y - sq * eps) / om_t,
              "ysubx": lambda: y - eps}[c["objective"]]()
        if c["clip"]:
            x0 = x0.clamp(-1.0, 1.0)
        if c["is_last"]:
            x1 = x0
        else:
            x1 = om_nt * x0 + m_nt * y + c_xt * (x_t - om_t * x0 - m_t * y) + sigma * c["noise"].cpu().float()
        outs = [("x_{t-1}", a["x_out"], x1)] + ([("x0", a["x0_out"], x0)] if a["x0_out"] is not None else [])
        for what, got, want in outs:
            self._record(idx, method, form, what, image_equal(got.cpu(), want), 0.0, shapes)

    def _ref_p_sample(self, idx, form, shapes, c, a, pre):
        self._p_sample(idx, "p_sample", form, shapes, c, a, c["coef"])

    def _ref_p_sample_dev(self, idx, form, shapes, c, a, pre):
        self._p_sample(idx, "p_sample_dev", form, shapes, c, a, c["coef_dev"].cpu().tolist())   # pre-launch clone

    def _ref_spatial_rescale(self, idx, form, shapes, c, a, pre):
        """n_stages bilinear x0.5 interpolations (align_corners False: the mean of each 2x2 block, an odd last row /
        column dropped), then the optional 1x1 map, in fp64."""
        x = c["src"].to(F64)
        for _ in range(c["n_stages"]):
            H, W = x.shape[2] // 2 * 2, x.shape[3] // 2 * 2
            x = x[:, :, :H, :W].reshape(x.shape[0], x.shape[1], H // 2, 2, W // 2, 2).mean((3, 5))
        if c["weight"] is not None:
            x = torch.einsum("oc,bchw->bohw", c["weight"].to(F64), x)
            if c["bias"] is not None:
                x = x + c["bias"].to(F64).view(1, -1, 1, 1)
        self._record(idx, "spatial_rescale", form, "out", image_devs(a["out"], x), self.bounds["spatial_rescale"],
                     shapes)

    def _ref_denorm_to_uint8(self, idx, form, shapes, c, a, pre):
        """runners/utils.py:67-74 of the reference, on the CPU in fp32, as the byte-exact single-kernel test."""
        x = c["images"].cpu().float()
        if c["to_normal"]:
            x = x.mul(0.5).add(0.5).clamp(0, 1.)
        want = x.mul(255).add(0.5).clamp(0, 255).permute(0, 2, 3, 1).to(torch.uint8)
        self._record(idx, "denorm_to_uint8", form, "bytes", image_equal(a["out"].cpu(), want), 0.0, shapes)

    # -- VQGAN ends and the space-to-depth operand ---------------------------------------------------------------
    def _ref_s2d_split(self, idx, form, shapes, c, a, pre):
        h, l = split_bf16(space_to_depth(c["src"]))
        self._record(idx, "s2d_split", form, "planes (bit-exact split)",
                     torch.maximum(image_equal(a["out_hi"], h), image_equal(a["out_lo"], l)), 0.0, shapes)

    def _ref_conv_direct_pad(self, idx, form, shapes, c, a, pre):
        src, k, cout = c["src"], c["k"], c["cout"]
        w = c["w_packed"].reshape(k, k, src.shape[3], cout).permute(3, 2, 0, 1).to(F64)
        p = (c["pad_lo"], c["pad_hi"])
        devs = []
        for sl in chunks(src.shape[0], src[0].numel() * 8 * 4, src.device):
            x = F.pad(src[sl].to(F64).permute(0, 3, 1, 2), p + p)
            o = F.conv2d(x, w, None if c["bias"] is None else c["bias"].to(F64), stride=c["stride"]).permute(0, 2, 3, 1)
            if c["residual"] is not None:
                o = o + c["residual"][sl].to(F64)
            devs.append(image_devs(a["out"][sl], o))
        self._record(idx, "conv_direct_pad", form, "out", torch.cat(devs), self.bounds["conv_direct_pad"], shapes)

    def _ref_softmax_rows_split(self, idx, form, shapes, c, a, pre):
        """Per row: fp64 softmax(scale * s) against hi + lo, and hi, lo a split pair."""
        s = c["src"]
        n = s.shape[-1]
        hi, lo = a["out_hi"].reshape(-1, n), a["out_lo"].reshape(-1, n)
        want = torch.softmax(s.reshape(-1, n).to(F64) * c["scale"], dim=-1)
        self._record(idx, "softmax_rows_split", form, "rows hi + lo", image_devs(planes(hi, lo), want),
                     self.bounds["softmax"], shapes)
        self._record(idx, "softmax_rows_split", form, "rows split", pair_well_formed(hi, lo), 0.0, shapes)

    def _ref_vq_nearest(self, idx, form, shapes, c, a, pre):
        """Per image: the chosen code's fp64 squared distance within fp32 noise of the fp64 minimum, the index equal to
        the fp64 argmin wherever the top-2 gap is clear of that noise, and z_q = z + (e - z) (the reference's
        straight-through expression) bit for bit.  Distances are in units of 1 + |z|^2 + |e|^2, the magnitude of the
        terms an fp32 evaluation sums."""
        z, cb = c["z"], c["codebook"]
        B, D = z.shape[0], cb.shape[1]
        zf = z.reshape(B, -1, D)
        idx_got = a["indices"].reshape(B, -1)
        cb64 = cb.to(F64)
        gap_dev, idx_dev, zq_dev = [], [], []
        for b in range(B):
            for r0 in range(0, zf.shape[1], 4096):
                zr = zf[b, r0:r0 + 4096].to(F64)
                d = torch.cdist(zr, cb64) ** 2
                top = d.topk(2, dim=1, largest=False)
                chosen = a["indices"].reshape(B, -1)[b, r0:r0 + 4096]
                ok_range = bool(((chosen >= 0) & (chosen < cb.shape[0])).all())
                ci = chosen.clamp(0, cb.shape[0] - 1)
                scale = 1.0 + (zr * zr).sum(1) + (cb64[ci] * cb64[ci]).sum(1)
                excess = (d.gather(1, ci[:, None])[:, 0] - top.values[:, 0]) / scale
                gap_dev.append(float(excess.max()) if ok_range else math.inf)
                clear = (top.values[:, 1] - top.values[:, 0]) / scale > self.bounds["vq_distance"]
                idx_dev.append(0.0 if ok_range and torch.equal(chosen[clear], top.indices[clear, 0]) else math.inf)
                zr32 = zf[b, r0:r0 + 4096]
                e = cb[ci]
                want = zr32 + (e - zr32)
                got = a["z_q"].reshape(B, -1, D)[b, r0:r0 + 4096]
                zq_dev.append(0.0 if torch.equal(got, want) else math.inf)
        per = lambda v: torch.tensor(v, dtype=F64).reshape(B, -1).amax(1)
        self._record(idx, "vq_nearest", form, "chosen distance - minimum", per(gap_dev), self.bounds["vq_distance"],
                     shapes)
        self._record(idx, "vq_nearest", form, "index where the top-2 gap is clear", per(idx_dev), 0.0, shapes)
        self._record(idx, "vq_nearest", form, "z_q = z + (e - z) (bit-exact)", per(zq_dev), 0.0, shapes)


# ------------------------------------------------------------------------------------------------ coverage
# (method, features that one launch's form must all have, features it must not have).  What the cfg2 routing issues: the
# F(6,3) forms -- plain, two-source with the raw planes of a fused 1x1 skip, the down-ResBlock's pooled conv1, the
# up-ResBlock's phase-stacked conv1, each residual mode -- and the direct tensor-core forms.  Its up-ResBlocks all take
# the phase-stacked F(6,3) conv, so the fused nearest-2x direct conv (UPSAMPLE_FORMS) is required of cfg1 and cfg3-5.
CFG2_FORMS = [
    ("wino_input", ("F(6,3)",), ("two-source", "down2", "raw planes")),
    ("wino_input", ("F(6,3)", "two-source", "raw planes"), ()),
    ("wino_input", ("F(6,3)", "down2"), ()),
    ("wino_output", ("F(6,3)", "up2_phases"), ()),
    ("wino_output", ("F(6,3)",), ("res", "up2_phases")),
    ("wino_output", ("F(6,3)", "res 1"), ()),
    ("wino_output", ("F(6,3)", "res 2"), ()),
    ("wino_output", ("F(6,3)", "res 3"), ()),
    ("conv_umma", ("position GEMMs",), ()),
    ("conv_umma", ("fused 1x1",), ()),
    ("conv_umma", ("NCHW head",), ()),
    ("conv_umma", ("split out",), ()),
    ("conv_umma", ("taps 9", "res 1"), ()),
    ("conv_umma", ("taps 9", "res 3"), ()),
    ("attention_tc", (), ()),
    ("conv_stem", (), ()),
]
UPSAMPLE_FORMS = [("conv_umma", ("upsample2x",), ())]
F43_FORMS = [("wino_input", ("F(4,3)",), ()), ("wino_output", ("F(4,3)",), ())]
# What one training micro-step of the LBBDM-f4 UNet at batch 32 issues (q_sample, forward, backward, two FusedAdam
# steps): the F(4,3) training forward (act planes for the weight gradient, fused residual) and data-gradient chain
# (identity input transform of dY, flipped weight planes), the direct tensor-core forward and data gradient, the
# resampling operand passes, the gradient split with and without the planes of a direct data gradient, the weight
# gradients, the GroupNorm backward with and without FiLM and without activation (the attention block's qkv), the
# attention backward, and Adam's first two steps.  (Every conv of the cfg3 UNet has a bias: the split without column
# sums comes with the transformer's bias-free projections.)
TRAIN_FORMS = [
    ("q_sample", (), ()),
    ("wino_input", ("F(4,3)", "act planes"), ()),
    ("wino_output", ("F(4,3)", "res 1"), ()),
    ("wino_input", ("F(4,3)", "identity"), ()),
    ("wino_pack_weight", ("F(4,3)", "dgrad"), ()),
    ("conv_umma", ("taps 9",), ("dgrad",)),
    ("conv_umma", ("taps 9", "dgrad"), ()),
    ("conv_umma", ("taps 1",), ()),
    ("prep", ("resample 1",), ()),
    ("prep", ("resample 2",), ()),
    ("split_grad", ("planes", "colsum"), ()),
    ("split_grad", ("colsum",), ("planes",)),
    ("conv_wgrad", ("taps 9",), ()),
    ("conv_wgrad", ("taps 1",), ()),
    ("conv_direct", (), ()),
    ("conv_wgrad_direct", (), ()),
    ("gn_bwd_reduce", ("film",), ()),
    ("gn_bwd_apply", ("film",), ()),
    ("gn_bwd_apply", (), ("film", "no act")),
    ("gn_bwd_apply", ("no act",), ()),
    ("attention_tc", (), ()),
    ("attention_bwd", (), ()),
    ("adam_multi", ("step 1",), ()),
    ("adam_multi", ("step 2",), ()),
]
# ... and with SpatialTransformers: LayerNorm and GEGLU operand passes and their backward, cross-attention and its
# backward, the k|v projection of the 3-channel context (3 x 2C channel pairs) on the direct weight gradient
ST_TRAIN_FORMS = TRAIN_FORMS + [
    ("layernorm_split", (), ()), ("layernorm_bwd", (), ()), ("geglu_split", (), ()), ("geglu_bwd", (), ()),
    ("attention_cross", (), ()), ("attention_cross_bwd", (), ()),
    ("conv_wgrad_direct", ("beyond 1024 channel pairs",), ()), ("split_grad", (), ("colsum",)),
]


def missing_forms(shadow, required):
    """The entries of required that no launch of the shadow matched."""
    return [r for r in required if not any(m == r[0] and all(f in form for f in r[1]) and
                                           not any(f in form for f in r[2]) for m, form in shadow.launches)]
