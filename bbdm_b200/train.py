"""Training path: the ResBlock convolutions (96 % of the training FLOPs) as an autograd Function
over the wgmma kernels -- forward (bbdm_conv_umma), data gradient (bbdm_conv_umma with the
flipped/transposed weights) and weight gradient (bbdm_conv_wgrad), all split-bf16 x3 with fp32
accumulation (fp32-class accuracy, like the reference's fp32 autograd).

Tensors cross the Function boundary as ordinary NCHW-shaped torch tensors in channels_last
memory format, i.e. physically the NHWC layout the kernels use: no layout copies when the
surrounding ops keep channels_last.  GroupNorm+SiLU+FiLM(+resampling) in front of a conv and the
attention core have their own Functions below.

Replaces the autograd of nn.Conv2d inside ResBlock (reference openaimodel.py:207,233,244) for
``loss.backward()`` (runners/BaseRunner.py:412); gradients land in the same nn.Parameter.grad, so
DDP's bucketed NCCL allreduce works unchanged.
"""
from __future__ import annotations

import contextlib
import threading

import torch
import torch.utils.checkpoint

from . import cabi, convs
from .weights import (stride2_dgrad_weights, stride2_fold_wgrad, stride2_s2d_weights, upsample_dgrad_weights,
                      upsample_fold_wgrad, upsample_phase_weights)

_BACKEND = None

# Winograd F(4x4,3x3) for the forward and data-gradient 3x3 convolutions of the training graph (csrc/winograd.cu;
# same eligibility rule as the sampling engines).  The weight gradient stays the direct wgmma GEMM.
WINO_TRAIN = convs.WINOGRAD_TRAIN
WINO_MIN_C = convs.WINO_MIN_C
WINO_MIN_TILES = convs.WINO_MIN_TILES

_WARNED = set()


def _library_path(what, x):
    """A CUDA training call whose shape the native kernels do not take runs on stock PyTorch (library) kernels: valid
    results, but not this library's path -- say so once per shape instead of falling back silently."""
    if x.is_cuda:
        key = (what, tuple(x.shape))
        if key not in _WARNED:
            _WARNED.add(key)
            import warnings
            warnings.warn(f"bbdm_b200.train: {what} with input {tuple(x.shape)} runs on stock PyTorch kernels "
                          "(shape outside the tensor-core kernels' envelope)", stacklevel=3)


def _wino_ok(be, B, H, W, Cin, Cout, k):
    return bool(WINO_TRAIN and k == 3 and hasattr(be, "wino_geometry")
                and convs.winograd_ok(be.wino_geometry(B, H, W), Cin, Cout, WINO_MIN_C, WINO_MIN_TILES))


# Trimmed recompute of checkpointed blocks: the recompute reuses the GroupNorm statistics of the original forward and,
# in a ResBlock's tail (unread_outputs), skips the convolutions whose outputs nothing in the backward reads.  False
# recomputes the whole block; both give bit-identical gradients (the tests compare them).
RECOMPUTE_TRIM = True

_TLS = threading.local()       # .block: the _BlockRun of the checkpointed block running on this thread; .unread


class _BlockRun:
    """One checkpointed block call: the GroupNorm (mean, rstd) pairs its forward computed, in order, for its recompute."""

    def __init__(self):
        self.stats, self.recompute, self.next = [], False, 0


@contextlib.contextmanager
def _running(run, recompute):
    prev = getattr(_TLS, "block", None)
    _TLS.block, run.recompute, run.next = run, recompute, 0
    try:
        yield
    finally:
        _TLS.block = prev


def _block_contexts():
    """checkpoint's context_fn: the same _BlockRun around the forward and around the recompute."""
    run = _BlockRun()
    return _running(run, False), _running(run, True)


def _trimmed_recompute():
    run = getattr(_TLS, "block", None)
    return run if RECOMPUTE_TRIM and run is not None and run.recompute else None


@contextlib.contextmanager
def unread_outputs():
    """Around a block's tail whose convolution outputs only feed the block's output: in a trimmed recompute those
    convolutions write their backward's operand planes and launch no GEMM (the output tensors stay unwritten)."""
    prev = getattr(_TLS, "unread", False)
    _TLS.unread = _trimmed_recompute() is not None
    try:
        yield
    finally:
        _TLS.unread = prev


def _unread():
    return getattr(_TLS, "unread", False)


def _unwritten(shape, dev):
    """The output of a convolution skipped under unread_outputs: the right shape, no storage behind it."""
    return torch.empty((1,) * len(shape), dtype=torch.float32, device=dev).expand(*shape)


def checkpointed(block, fn, *args):
    """fn(*args), the forward of a UNet block; with block.use_checkpoint on and autograd recording, only the arguments are
    kept and fn runs again in the backward (non-reentrant torch.utils.checkpoint, so torch.autograd.grad -- the graph
    capture's warm-up and DDP -- works).  The recompute issues the forward's own launches on the same operands, minus
    what RECOMPUTE_TRIM drops: the gradients are bit-identical to the plain graph's.  The RNG state is stashed only where
    a Dropout of p > 0 is active, so that the recompute draws the forward's masks; reading the generator state is not
    allowed inside a CUDA graph capture, which such a block never reaches (train_graph.fallback_reason)."""
    if not (block.use_checkpoint and torch.is_grad_enabled()):
        return fn(*args)
    dropout = any(isinstance(m, torch.nn.Dropout) and m.p > 0 and m.training for m in block.modules())
    return torch.utils.checkpoint.checkpoint(fn, *args, use_reentrant=False, preserve_rng_state=dropout,
                                             context_fn=_block_contexts)


def backend():
    global _BACKEND
    if _BACKEND is None:
        _BACKEND = cabi.CudaBackend()
    return _BACKEND


def set_backend(b):
    """tests/ inject their oracle-backed emulation here to check this module's host logic (gradient formulas,
    adjoints, tensor plumbing) on CPU; the product only ever uses cabi.CudaBackend."""
    global _BACKEND
    _BACKEND = b


def _on_device(x: torch.Tensor) -> bool:
    return x.is_cuda or (_BACKEND is not None and not getattr(_BACKEND, "requires_cuda", True))


def _tc_ok(x: torch.Tensor, cin: int, cout: int) -> bool:
    """Operands the tensor-core fwd/dgrad/wgrad kernels take: fp32 [B, C, H, W] on the device and the shapes of
    convs.tensor_core_ok at the backend's channel multiple (any map size and batch).  The backend is consulted only for
    an operand on the device: a CPU call never loads the library."""
    if not _on_device(x) or x.dtype != torch.float32 or x.dim() != 4:
        return False
    return convs.tensor_core_ok(cin, cout, x.shape[3], convs.channel_multiple(backend()))


def native_ok(conv: torch.nn.Conv2d, x: torch.Tensor) -> bool:
    """Convolutions the tensor-core fwd/dgrad/wgrad kernels take."""
    k = conv.kernel_size
    return (k in ((1, 1), (3, 3)) and conv.stride == (1, 1) and conv.padding == (k[0] // 2, k[0] // 2)
            and conv.groups == 1 and conv.dilation == (1, 1) and _tc_ok(x, conv.in_channels, conv.out_channels))


def _transposed_planes(C, P, dev):
    """Split planes (hi, lo) of dY^T for bbdm_split_grad / bbdm_conv_wgrad: [C, P] views of [C, P rounded up to 8]
    buffers -- the weight-gradient kernel reads the rows through a TMA map, whose row pitch must be a multiple of 16
    bytes.  The padding columns are never read (the map ends at P)."""
    ld = -(-P // 8) * 8
    return tuple(torch.empty((C, ld), dtype=torch.bfloat16, device=dev)[:, :P] for _ in range(2))


def _nhwc(x):
    """NCHW-shaped tensor -> contiguous NHWC view (copy only if x is not channels_last already)."""
    return x.contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1)


def _pack_weights(be, weight, need_dgrad):
    """(w_hi, w_lo, wd_hi, wd_lo): forward planes and, if the input needs a gradient, the data-gradient planes
    (flipped kernel, channels swapped) from the same single pass over the weight."""
    Cout, Cin, k, _ = weight.shape
    dev = weight.device
    w_hi = torch.empty((k * k, Cout, Cin), dtype=torch.bfloat16, device=dev)
    w_lo = torch.empty_like(w_hi)
    wd_hi = wd_lo = None
    if need_dgrad:
        wd_hi = torch.empty((k * k, Cin, Cout), dtype=torch.bfloat16, device=dev)
        wd_lo = torch.empty_like(wd_hi)
    be.pack_weight_split_both(weight.detach().contiguous(), w_hi, w_lo, wd_hi, wd_lo)
    return w_hi, w_lo, wd_hi, wd_lo


class Conv2dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        be = backend()
        B, Cin, H, W = x.shape
        Cout, _, k, _ = weight.shape
        dev = x.device
        xn = _nhwc(x.detach())
        a_hi = torch.empty((B, H, W, Cin), dtype=torch.bfloat16, device=dev)
        a_lo = torch.empty_like(a_hi)
        be.prep(xn, None, raw_hi=a_hi, raw_lo=a_lo)                      # operand split (one HBM pass)
        w_hi, w_lo, wd_hi, wd_lo = _pack_weights(be, weight, ctx.needs_input_grad[0])
        if _unread():
            out = _unwritten((B, H, W, Cout), dev)
        else:
            out = torch.empty((B, H, W, Cout), dtype=torch.float32, device=dev)
            be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=k * k, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo,
                         bias=None if bias is None else bias.detach(), out=out, passes=3)
        ctx.save_for_backward(a_hi, a_lo, weight, wd_hi, wd_lo)
        ctx.has_bias = bias is not None
        ctx.shape = (B, H, W, Cin, Cout, k)
        return out.permute(0, 3, 1, 2)                                   # NCHW shape, channels_last strides

    @staticmethod
    def backward(ctx, dy):
        a_hi, a_lo, weight, wd_hi, wd_lo = ctx.saved_tensors
        dxn, dw, dbias = _conv_backward(backend(), ctx.shape, a_hi, a_lo, weight, dy, ctx.needs_input_grad[0],
                                        ctx.needs_input_grad[1], ctx.has_bias and ctx.needs_input_grad[2],
                                        wd=(wd_hi, wd_lo))
        return (None if dxn is None else dxn.permute(0, 3, 1, 2)), dw, dbias


def _conv_backward(be, ctx_shape, a_hi, a_lo, weight, dy, need_dx, need_dw, need_db, wd=(None, None)):
    """Shared by both Functions: (dA or dX as NHWC fp32, dW, dbias) of the tensor-core conv."""
    B, H, W, Cin, Cout, k = ctx_shape
    dev = dy.device
    P = B * H * W
    dyn = _nhwc(dy)
    g_hi = g_lo = None
    wino_dx = need_dx and _wino_ok(be, B, H, W, Cout, Cin, k)
    if need_dx and not wino_dx:
        g_hi = torch.empty((B, H, W, Cout), dtype=torch.bfloat16, device=dev)
        g_lo = torch.empty_like(g_hi)
    gt_hi, gt_lo = _transposed_planes(Cout, P, dev)
    dbias = ws_b = None
    if need_db:
        dbias = torch.empty((Cout,), dtype=torch.float32, device=dev)
        ws_b = torch.empty(((P + 63) // 64) * Cout, dtype=torch.float32, device=dev)
    be.split_grad(dyn, g_hi, g_lo, gt_hi, gt_lo, dbias, ws_b)
    dxn = None
    if wino_dx:
        # data gradient = conv of dY with the flipped, channel-swapped kernel -- on the Winograd path.
        # Its operand planes are fp16 pairs (5 exponent bits): loss gradients (1e-4 ... 1e-8) would sit in fp16's
        # subnormal range and lose their mantissa (measured: 4e-3 per layer on the LBBDM-f4 UNet).  dY is therefore
        # normalised by a power of two that puts its largest element into [16, 32) -- the range the forward path's
        # activations live in -- and the result is scaled back; both scalings are exact, and the scale stays on the
        # device (no host synchronisation).
        amax = dyn.abs().amax().clamp_min(2.0 ** -100)
        scale = torch.exp2(4.0 - torch.floor(torch.log2(amax)))
        dxn = convs.wino_conv(be, convs.FreshBuffers(dev), be.wino_geometry(B, H, W), (dyn * scale).contiguous(), None,
                              cout=Cin, weight=weight, dgrad=True, silu=False)
        dxn.mul_(1.0 / scale)
    elif need_dx:
        # data gradient = the same conv with the kernel flipped and Cin/Cout swapped
        wd_hi, wd_lo = wd
        if wd_hi is None:
            wd_hi = torch.empty((k * k, Cin, Cout), dtype=torch.bfloat16, device=dev)
            wd_lo = torch.empty_like(wd_hi)
            be.pack_weight_split_dgrad(weight.detach().contiguous(), wd_hi, wd_lo)
        dxn = torch.empty((B, H, W, Cin), dtype=torch.float32, device=dev)
        be.conv_umma(B=B, H=H, W=W, Cin=Cout, Cout=Cin, taps=k * k, a_hi=g_hi, a_lo=g_lo, w_hi=wd_hi, w_lo=wd_lo,
                     out=dxn, passes=3)
    dw = None
    if need_dw:
        _, fl = be.wgrad_workspace(B, H, W, Cin, Cout, k * k)
        ws = torch.empty((fl,), dtype=torch.float32, device=dev)
        dw = torch.empty((Cout, Cin, k, k), dtype=torch.float32, device=dev)
        be.conv_wgrad(gt_hi, gt_lo, a_hi, a_lo, B, H, W, Cin, Cout, k * k, dw, ws)
    return dxn, dw, dbias


def _pack_taps(be, w, dev):
    """w [Cout', Cin', taps] fp32 -> split planes [taps][Cout'][Cin']."""
    hi = torch.empty((w.shape[2], w.shape[0], w.shape[1]), dtype=torch.bfloat16, device=dev)
    lo = torch.empty_like(hi)
    be.pack_weight_split_taps(w, hi, lo)
    return hi, lo


def _split_dy(be, dyn, need_dx, need_db):
    """dY [B, H, W, C] fp32 (contiguous) -> split planes (g_hi, g_lo) [B, H, W, C] if need_dx, the transposed planes
    (gt_hi, gt_lo) [C][P] of the weight-gradient GEMM, and the column sums [C] if need_db."""
    B, H, W, Cc = dyn.shape
    P, dev = B * H * W, dyn.device
    g_hi = g_lo = dsum = ws = None
    if need_dx:
        g_hi = torch.empty(dyn.shape, dtype=torch.bfloat16, device=dev)
        g_lo = torch.empty_like(g_hi)
    gt_hi, gt_lo = _transposed_planes(Cc, P, dev)
    if need_db:
        dsum = torch.empty((Cc,), dtype=torch.float32, device=dev)
        ws = torch.empty(((P + 63) // 64) * Cc, dtype=torch.float32, device=dev)
    be.split_grad(dyn, g_hi, g_lo, gt_hi, gt_lo, dsum, ws)
    return g_hi, g_lo, gt_hi, gt_lo, dsum


def _wgrad(be, gt_hi, gt_lo, a_hi, a_lo, B, H, W, Cin, Cout, taps, window_origin=0):
    """conv_wgrad into a fresh [Cout, Cin, k, k] tensor (k = 2 for taps 4)."""
    dev = gt_hi.device
    _, fl = be.wgrad_workspace(B, H, W, Cin, Cout, taps)
    ws = torch.empty((fl,), dtype=torch.float32, device=dev)
    k = {1: 1, 4: 2, 9: 3}[taps]
    dw = torch.empty((Cout, Cin, k, k), dtype=torch.float32, device=dev)
    be.conv_wgrad(gt_hi, gt_lo, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, ws, window_origin=window_origin)
    return dw


class Stride2Conv2dFn(torch.autograd.Function):
    """3x3 conv, stride 2, padding 1 (the UNet Downsample, openaimodel.py:137-163) on the tensor cores.  With the
    space-to-depth operand x' (bbdm_s2d_split: 4*Cin phase-major channels on the H/2 x W/2 grid) it is a 2x2-tap conv
    whose window sits at rows/cols -1..0 (weights.stride2_s2d_weights):
      forward          conv_umma, taps 4, window_origin -1, over x'
      data gradient    the transposed, tap-flipped 2x2 conv over dY (window_origin 0) gives dx', depth-to-space dx
      weight gradient  conv_wgrad, taps 4, window_origin -1, over (x', dY), folded back to [Cout][Cin][3][3]
      bias gradient    the column sums of dY (bbdm_split_grad)
    x: [B, Cin, H, W] with H, W even -> [B, Cout, H/2, W/2] (channels_last strides)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        be = backend()
        B, Cin, H, W = x.shape
        Cout = weight.shape[0]
        Ho, Wo = H // 2, W // 2
        dev = x.device
        xn = _nhwc(x.detach()).contiguous()
        a_hi = torch.empty((B, Ho, Wo, 4 * Cin), dtype=torch.bfloat16, device=dev)
        a_lo = torch.empty_like(a_hi)
        be.s2d_split(xn, a_hi, a_lo)
        w_hi, w_lo = _pack_taps(be, stride2_s2d_weights(weight.detach()), dev)
        out = torch.empty((B, Ho, Wo, Cout), dtype=torch.float32, device=dev)
        be.conv_umma(B=B, H=Ho, W=Wo, Cin=4 * Cin, Cout=Cout, taps=4, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo,
                     bias=None if bias is None else bias.detach(), out=out, passes=3, window_origin=-1)
        ctx.save_for_backward(a_hi, a_lo, weight)
        ctx.has_bias = bias is not None
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dy):
        be = backend()
        a_hi, a_lo, weight = ctx.saved_tensors
        B, Ho, Wo, Cin4 = a_hi.shape
        Cin, Cout = Cin4 // 4, weight.shape[0]
        dev = dy.device
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        need_db = ctx.has_bias and ctx.needs_input_grad[2]
        g_hi, g_lo, gt_hi, gt_lo, db = _split_dy(be, _nhwc(dy).contiguous(), need_dx, need_db)
        dx = dw = None
        if need_dx:
            wd_hi, wd_lo = _pack_taps(be, stride2_dgrad_weights(weight.detach()), dev)
            dxs = torch.empty((B, Ho, Wo, Cin4), dtype=torch.float32, device=dev)
            be.conv_umma(B=B, H=Ho, W=Wo, Cin=Cout, Cout=Cin4, taps=4, a_hi=g_hi, a_lo=g_lo, w_hi=wd_hi, w_lo=wd_lo,
                         out=dxs, passes=3)
            # depth-to-space: channel (a*2 + b)*Cin + ci of pixel (i, j) -> pixel (2i + a, 2j + b)
            dxn = dxs.view(B, Ho, Wo, 2, 2, Cin).permute(0, 1, 3, 2, 4, 5).reshape(B, 2 * Ho, 2 * Wo, Cin)
            dx = dxn.permute(0, 3, 1, 2)
        if need_dw:
            dw = stride2_fold_wgrad(_wgrad(be, gt_hi, gt_lo, a_hi, a_lo, B, Ho, Wo, Cin4, Cout, 4, window_origin=-1))
        return dx, dw, db


class Up2Conv2dFn(torch.autograd.Function):
    """Nearest-2x upsample followed by a 3x3 'same' conv (the UNet Upsample, openaimodel.py:93-121) on the tensor
    cores, never materialising the upsampled tensor:
      forward          the fused 4-phase conv (conv_umma upsample2x, weights.upsample_phase_weights) on x
      data gradient    a stride-1 3x3 conv on the low-res grid over dY' = space-to-depth(dY) (4*Cout channels)
      weight gradient  conv_wgrad, taps 9, over (x, dY'), folded back to [Cout][Cin][3][3]
      bias gradient    the column sums of dY' summed over the 4 phases
    (weights.upsample_dgrad_weights / upsample_fold_wgrad).  x: [B, Cin, H, W] -> [B, Cout, 2H, 2W]."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        be = backend()
        B, Cin, H, W = x.shape
        Cout = weight.shape[0]
        dev = x.device
        xn = _nhwc(x.detach())
        a_hi = torch.empty((B, H, W, Cin), dtype=torch.bfloat16, device=dev)
        a_lo = torch.empty_like(a_hi)
        be.prep(xn, None, raw_hi=a_hi, raw_lo=a_lo)
        w_hi, w_lo = _pack_taps(be, upsample_phase_weights(weight.detach()), dev)
        out = torch.empty((B, 2 * H, 2 * W, Cout), dtype=torch.float32, device=dev)
        be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=4, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo,
                     bias=None if bias is None else bias.detach(), out=out, passes=3, upsample2x=True)
        ctx.save_for_backward(a_hi, a_lo, weight)
        ctx.has_bias = bias is not None
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dy):
        be = backend()
        a_hi, a_lo, weight = ctx.saved_tensors
        B, H, W, Cin = a_hi.shape
        Cout = weight.shape[0]
        dev = dy.device
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        need_db = ctx.has_bias and ctx.needs_input_grad[2]
        # space-to-depth of dY: pixel (2i + a, 2j + b), channel co -> pixel (i, j), channel (a*2 + b)*Cout + co
        dys = _nhwc(dy).reshape(B, H, 2, W, 2, Cout).permute(0, 1, 3, 2, 4, 5).reshape(B, H, W, 4 * Cout)
        g_hi, g_lo, gt_hi, gt_lo, db4 = _split_dy(be, dys.contiguous(), need_dx, need_db)
        dx = dw = db = None
        if need_dx:
            wd_hi, wd_lo = _pack_taps(be, upsample_dgrad_weights(weight.detach()), dev)
            dxn = torch.empty((B, H, W, Cin), dtype=torch.float32, device=dev)
            be.conv_umma(B=B, H=H, W=W, Cin=4 * Cout, Cout=Cin, taps=9, a_hi=g_hi, a_lo=g_lo, w_hi=wd_hi, w_lo=wd_lo,
                         out=dxn, passes=3)
            dx = dxn.permute(0, 3, 1, 2)
        if need_dw:
            dw = upsample_fold_wgrad(_wgrad(be, gt_hi, gt_lo, a_hi, a_lo, B, H, W, Cin, 4 * Cout, 9))
        if need_db:
            db = db4.view(4, Cout).sum(0)
        return dx, dw, db


def _resample_ok(x, cin, cout):
    """Operand checks shared by the resampling convs: a backend with the 2x2 window origin, fp32 [B, C, H, W] on the
    device."""
    return (_on_device(x) and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == cin
            and getattr(backend(), "window_origin", False))


def downsample_conv(conv: torch.nn.Conv2d, x: torch.Tensor, enabled: bool = True):
    """The Downsample's 3x3 stride-2 padding-1 conv on Stride2Conv2dFn, or None where the kernels do not take the
    shape (Cin, Cout multiples of the backend's channel multiple, H and W even, and a half-resolution grid at least 4
    wide)."""
    if not (enabled and _resample_ok(x, conv.in_channels, conv.out_channels)):
        return None
    B, Cin, H, W = x.shape
    mult = convs.channel_multiple(backend())
    if Cin % mult or H % 2 or W % 2 or not convs.tensor_core_ok(4 * Cin, conv.out_channels, W // 2, mult):
        return None
    return Stride2Conv2dFn.apply(x, conv.weight, conv.bias)


def upsample_conv(conv: torch.nn.Conv2d, x: torch.Tensor, enabled: bool = True):
    """conv(nearest-2x(x)) of the Upsample on Up2Conv2dFn, or None where the kernels do not take the shape (Cin, Cout
    multiples of the backend's channel multiple and a low-res grid at least 4 wide)."""
    if not (enabled and _resample_ok(x, conv.in_channels, conv.out_channels)):
        return None
    B, Cin, H, W = x.shape
    if not convs.tensor_core_ok(Cin, conv.out_channels, W, convs.channel_multiple(backend())):
        return None
    return Up2Conv2dFn.apply(x, conv.weight, conv.bias)


class GNActConv2dFn(torch.autograd.Function):
    """conv( silu( GroupNorm32(x) * (1 + scale) + shift ) ) fused: the forward is the sampling path's
    stats + prep + wgmma conv; the backward adds the two-pass GroupNorm/SiLU/FiLM gradient kernels."""

    @staticmethod
    def forward(ctx, x, gamma, beta, scale, shift, weight, bias, resample=0, residual=None, act=True, eps=1e-5):
        """resample: 0 none, 1 nearest-2x up, 2 2x2 average pool -- applied between SiLU and the conv
        (ResBlock(up/down), openaimodel.py:259-264).  eps: the GroupNorm's (1e-5 in GroupNorm32, 1e-6 in
        SpatialTransformer.norm)."""
        be = backend()
        B, Cin, Hs, Ws = x.shape
        H, W = (Hs * 2, Ws * 2) if resample == 1 else ((Hs // 2, Ws // 2) if resample == 2 else (Hs, Ws))
        Cout, _, k, _ = weight.shape
        dev = x.device
        xn = _nhwc(x.detach())
        run = getattr(_TLS, "block", None)
        if _trimmed_recompute() is not None:      # the statistics the block's forward reduced, in the same order
            mean, rstd = run.stats[run.next]
            run.next += 1
        else:
            mean = torch.empty((B, 32), dtype=torch.float32, device=dev)
            rstd = torch.empty_like(mean)
            ws = torch.empty((B * 32 * cabi.GN_MAX_SLICES * 2,), dtype=torch.float64, device=dev)
            be.gn_stats(xn, None, 32, eps, mean, rstd, ws)
            if run is not None and not run.recompute:
                run.stats.append((mean, rstd))
        unread = _unread()
        fs = fh = None
        if scale is not None:
            fs, fh = scale.detach().contiguous().float(), shift.detach().contiguous().float()
        a_hi = torch.empty((B, H, W, Cin), dtype=torch.bfloat16, device=dev)
        a_lo = torch.empty_like(a_hi)
        rn = None if residual is None or unread else _nhwc(residual.detach())      # + skip(x), fused in the epilogue
        if resample == 0 and _wino_ok(be, B, H, W, Cin, Cout, k) and unread:
            # a trimmed recompute of the Winograd route: only the activated planes (prep computes them bit for bit as
            # the input transform does)
            be.prep(xn, None, groups=32, mean=mean, rstd=rstd, gamma=gamma.detach(), beta=beta.detach(), film_scale=fs,
                    film_shift=fh, film_stride=0 if fs is None else fs.shape[1], silu=act, act_hi=a_hi, act_lo=a_lo)
            out = _unwritten((B, H, W, Cout), dev)
            wd_hi = wd_lo = None
        elif resample == 0 and _wino_ok(be, B, H, W, Cin, Cout, k):
            # Winograd forward; the input transform also writes the activated split planes the weight gradient needs
            out = convs.wino_conv(be, convs.FreshBuffers(dev), be.wino_geometry(B, H, W), xn.contiguous(), None,
                                  cout=Cout, weight=weight, bias=None if bias is None else bias.detach(),
                                  residual=None if rn is None else rn.contiguous(),
                                  res_mode=cabi.RES_NONE if rn is None else cabi.RES_SAME, groups=32, mean=mean,
                                  rstd=rstd, gamma=gamma.detach(), beta=beta.detach(), film_scale=fs, film_shift=fh,
                                  film_stride=0 if fs is None else fs.shape[1], silu=act, act_hi=a_hi, act_lo=a_lo)
            wd_hi = wd_lo = None              # the backward re-derives what it needs (Winograd dgrad planes)
        else:
            be.prep(xn, None, groups=32, mean=mean, rstd=rstd, gamma=gamma.detach(), beta=beta.detach(), film_scale=fs,
                    film_shift=fh, film_stride=0 if fs is None else fs.shape[1], silu=act, resample=resample,
                    act_hi=a_hi, act_lo=a_lo)
            w_hi, w_lo, wd_hi, wd_lo = _pack_weights(be, weight, True)
            if unread:
                out = _unwritten((B, H, W, Cout), dev)
            else:
                out = torch.empty((B, H, W, Cout), dtype=torch.float32, device=dev)
                be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=k * k, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi,
                             w_lo=w_lo, bias=None if bias is None else bias.detach(), residual=rn,
                             res_mode=cabi.RES_NONE if rn is None else cabi.RES_SAME, out=out, passes=3)
        ctx.save_for_backward(xn, mean, rstd, gamma, beta, fs, fh, a_hi, a_lo, weight, wd_hi, wd_lo)
        ctx.has_bias = bias is not None
        ctx.shape = (B, H, W, Cin, Cout, k)
        ctx.resample = resample
        ctx.has_res = residual is not None
        ctx.act = act
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dy):
        be = backend()
        xn, mean, rstd, gamma, beta, fs, fh, a_hi, a_lo, weight, wd_hi, wd_lo = ctx.saved_tensors
        B, H, W, Cin, Cout, k = ctx.shape
        dev = dy.device
        da, dw, dbias = _conv_backward(be, ctx.shape, a_hi, a_lo, weight, dy, True, ctx.needs_input_grad[5],
                                       ctx.has_bias and ctx.needs_input_grad[6], wd=(wd_hi, wd_lo))
        if ctx.resample == 1:        # adjoint of nearest-2x: sum the four children
            da = da.view(B, H // 2, 2, W // 2, 2, Cin).sum(dim=(2, 4)).contiguous()
        elif ctx.resample == 2:      # adjoint of the 2x2 mean: a quarter to each of the four parents
            da = (0.25 * da).repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).contiguous()
        H, W = xn.shape[1], xn.shape[2]
        g, b_ = gamma.detach(), beta.detach()
        fstride = 0 if fs is None else fs.shape[1]
        a12 = torch.empty((B, Cin, 2), dtype=torch.float32, device=dev)
        ws = torch.empty((B * 64 * Cin * 2,), dtype=torch.float32, device=dev)
        be.gn_bwd_reduce(xn, da, 32, mean, rstd, g, b_, fs, fh, fstride, ctx.act, a12, ws)
        a1, a2 = a12[..., 0], a12[..., 1]                                  # [B, C]
        f1 = (1.0 + fs) if fs is not None else torch.ones_like(a1)
        dgamma = (f1 * a2).sum(0)
        dbeta = (f1 * a1).sum(0)
        dscale = dshift = None
        if fs is not None:
            dshift = a1
            dscale = g * a2 + b_ * a1
        gf = g * f1                                                       # [B, C]
        s1 = (gf * a1).view(B, 32, Cin // 32).sum(2).contiguous()
        s2 = (gf * a2).view(B, 32, Cin // 32).sum(2).contiguous()
        dxn = torch.empty((B, H, W, Cin), dtype=torch.float32, device=dev)
        be.gn_bwd_apply(xn, da, 32, mean, rstd, g, b_, fs, fh, fstride, ctx.act, s1, s2, dxn)
        return (dxn.permute(0, 3, 1, 2), dgamma, dbeta, dscale, dshift, dw, dbias, None, (dy if ctx.has_res else None),
                None, None)


def gn_act_conv2d(norm, conv, x, scale=None, shift=None, enabled=True, resample=0, residual=None, act=True):
    """conv(resample(silu(norm(x) * (1 + scale) + shift))) [+ residual] -- fused tensor-core path when the
    shape qualifies (the residual add then happens in the conv epilogue)."""
    B, _, Hs, Ws = x.shape
    H, W = (Hs * 2, Ws * 2) if resample == 1 else ((Hs // 2, Ws // 2) if resample == 2 else (Hs, Ws))
    probe = x if resample == 0 else x.new_empty((B, x.shape[1], H, W))       # shape check at the conv's resolution
    if enabled and native_ok(conv, probe) and x.shape[1] % 32 == 0 and x.shape[1] <= 4096 and \
            (resample != 2 or (Hs % 2 == 0 and Ws % 2 == 0)):
        sc = None if scale is None else scale.reshape(scale.shape[0], -1)
        sh = None if shift is None else shift.reshape(shift.shape[0], -1)
        return GNActConv2dFn.apply(x, norm.weight, norm.bias, sc, sh, conv.weight, conv.bias, resample, residual, act,
                                   norm.eps)
    if enabled:
        _library_path("GroupNorm+activation+conv", x)
    h = norm(x)
    if scale is not None:
        h = h * (1 + scale) + shift
    if act:
        h = torch.nn.functional.silu(h)
    if resample == 1:
        h = torch.nn.functional.interpolate(h, scale_factor=2, mode="nearest")
    elif resample == 2:
        h = torch.nn.functional.avg_pool2d(h, 2)
    h = conv2d(conv, h, enabled)
    return h if residual is None else residual + h


class SmallConv2dFn(torch.autograd.Function):
    """The UNet stem / head (3..32 channels on one side): exact fp32 on CUDA cores -- forward and data
    gradient through bbdm_conv_direct, weight gradient through bbdm_conv_wgrad_direct."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        be = backend()
        B, Cin, H, W = x.shape
        Cout, _, k, _ = weight.shape
        dev = x.device
        xn = _nhwc(x.detach()).contiguous()
        wp = torch.empty((k * k, Cin, Cout), dtype=torch.float32, device=dev)
        be.pack_weight_f32(weight.detach().contiguous(), wp)
        out = torch.empty((B, H, W, Cout), dtype=torch.float32, device=dev)
        be.conv_direct(xn, wp, None if bias is None else bias.detach(), None, out, Cout, k, 1)
        ctx.save_for_backward(xn, weight)
        ctx.has_bias = bias is not None
        ctx.k = k
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dy):
        be = backend()
        xn, weight = ctx.saved_tensors
        k = ctx.k
        B, H, W, Cin = xn.shape
        Cout = weight.shape[0]
        dev = dy.device
        dyn = _nhwc(dy).contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            wd = weight.detach().flip(2, 3).transpose(0, 1).contiguous()          # [Cin, Cout, k, k]
            wdp = torch.empty((k * k, Cout, Cin), dtype=torch.float32, device=dev)
            be.pack_weight_f32(wd, wdp)
            dxn = torch.empty((B, H, W, Cin), dtype=torch.float32, device=dev)
            be.conv_direct(dyn, wdp, None, None, dxn, Cin, k, 1)
            dx = dxn.permute(0, 3, 1, 2)
        if ctx.needs_input_grad[1]:
            n = k * k * Cin * Cout
            ws = torch.empty((2048 * n,), dtype=torch.float32, device=dev)
            dw = torch.empty((Cout, Cin, k, k), dtype=torch.float32, device=dev)
            be.conv_wgrad_direct(dyn, xn, k, dw, ws)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dyn.sum(dim=(0, 1, 2))
        return dx, dw, db


def small_ok(conv: torch.nn.Conv2d, x: torch.Tensor) -> bool:
    k = conv.kernel_size
    return (_on_device(x) and x.dtype == torch.float32 and x.dim() == 4 and k in ((1, 1), (3, 3))
            and conv.stride == (1, 1) and conv.padding == (k[0] // 2, k[0] // 2) and conv.groups == 1
            and conv.dilation == (1, 1) and conv.in_channels * conv.out_channels <= 1024
            and min(conv.in_channels, conv.out_channels) <= 32)


def conv1x1(conv1d: torch.nn.Conv1d, x4: torch.Tensor, enabled: bool = True):
    """nn.Conv1d(k=1) of AttentionBlock (qkv / proj_out, openaimodel.py:307,315) applied to a [B,C,H,W]
    tensor as a 1x1 convolution on the tensor-core autograd path; returns [B,Cout,H,W] or None if the
    shape does not qualify (caller falls back to the module)."""
    if not (enabled and conv1d.kernel_size == (1,) and _tc_ok(x4, x4.shape[1], conv1d.out_channels)):
        return None
    return Conv2dFn.apply(x4, conv1d.weight.unsqueeze(-1), conv1d.bias)


def _gemm_heads(be, q, k, v, grid, dout=None, grads=None):
    """Attention heads wider than the flash kernels take, one (image, head) at a time as tensor-core GEMMs around the
    materialised row softmax (UNetEngine's route in sampling).  q [B, T, heads, d], k / v [B, Tkv, heads, d]: fp32 views
    of the saved inputs; grid = (H, W) of the queries (T = H * W).  Each head's slices are copied into zero-padded
    [T, d32] / [Tkvp, d32] tensors (d32 = d rounded up to 32, Tkvp = Tkv rounded up to 64), and the scratch covers one
    image-head: no [B * heads, T, Tkv] tensor exists.
      forward (dout None): out [B, T, heads, d] = softmax(Q K^T d^-1/2) V, through KernelExecutor._attention_gemm.
      backward: writes dq, dk, dv into grads (views of q's, k's and v's shapes) for dout [B, T, heads, d].  S = Q K^T
      and dP = dO V^T are recomputed (conv_umma); softmax_rows_split gives the planes of P and, with grad=dP, of dS;
      dQ = dS K (conv_umma); dK^T = Q^T dS and dV^T = dO^T P are weight gradients over the query pixels (conv_wgrad,
      taps 1), so only Q and dO need transposed planes, never a [Tkv, T] matrix."""
    from .engine import KernelExecutor
    B, T, heads, d = q.shape
    tkv = k.shape[1]
    H, W = grid
    dev = q.device
    d32, tkvp = cabi.gemm_heads_pad(d), -(-tkv // 64) * 64
    scale = float(d ** -0.5)
    bf = torch.bfloat16
    zeros = lambda *shape: torch.zeros(shape, dtype=torch.float32, device=dev)
    planes = lambda *shape: torch.empty((2,) + shape, dtype=bf, device=dev)
    qp, kp, vp = zeros(1, H, W, d32), zeros(tkvp, d32), zeros(tkvp, d32)
    q_pl, k_pl, kt_pl = planes(1, H, W, d32), planes(1, tkvp, d32), planes(1, d32, tkvp)
    s = torch.empty((1, H, W, tkvp), dtype=torch.float32, device=dev)
    ex = KernelExecutor(be)
    out = None
    if dout is None:
        out = torch.empty((B, T, heads, d), dtype=torch.float32, device=dev)
        vt_pl = torch.zeros((2, 1, d32, tkvp), dtype=bf, device=dev)
        p_pl, o = planes(1, H, W, tkvp), torch.empty((1, H, W, d32), dtype=torch.float32, device=dev)
    else:
        dq, dk, dv = grads
        v_pl, vt_pl = planes(1, tkvp, d32), planes(1, d32, tkvp)
        dop, do_pl = zeros(1, H, W, d32), planes(1, H, W, d32)
        qt_pl, dot_pl = _transposed_planes(d32, T, dev), _transposed_planes(d32, T, dev)
        dp = torch.empty_like(s)
        p_pl, ds_pl = planes(1, H, W, tkvp), planes(1, H, W, tkvp)
        dqo = torch.empty((1, H, W, d32), dtype=torch.float32, device=dev)
        dkw, dvw = (torch.empty((d32, tkvp, 1, 1), dtype=torch.float32, device=dev) for _ in range(2))
        ws = torch.empty((be.wgrad_workspace(1, H, W, tkvp, d32, 1)[1],), dtype=torch.float32, device=dev)
    masked = {} if tkv == tkvp else dict(valid_cols=tkv)
    for b in range(B):
        for h in range(heads):
            qp[..., :d].copy_(q[b, :, h].view(H, W, d))
            kp[:tkv, :d].copy_(k[b, :, h])
            vp[:tkv, :d].copy_(v[b, :, h])
            be.split_grad(kp, k_pl[0], k_pl[1], kt_pl[0, 0], kt_pl[1, 0])
            if dout is None:
                be.prep(qp, None, raw_hi=q_pl[0], raw_lo=q_pl[1])
                ex._attention_gemm((q_pl[0], q_pl[1]), (k_pl[0], k_pl[1]), (vt_pl[0], vt_pl[1]), vp[:tkv], grid, tkv,
                                   scale, s, (p_pl[0], p_pl[1]), out_f32=o)
                out[b, :, h].copy_(o.view(T, d32)[:, :d])
                continue
            be.split_grad(qp.view(T, d32), q_pl[0].view(T, d32), q_pl[1].view(T, d32), *qt_pl)
            be.split_grad(vp, v_pl[0], v_pl[1], vt_pl[0, 0], vt_pl[1, 0])
            dop[..., :d].copy_(dout[b, :, h].view(H, W, d))
            be.split_grad(dop.view(T, d32), do_pl[0].view(T, d32), do_pl[1].view(T, d32), *dot_pl)
            be.conv_umma(B=1, H=H, W=W, Cin=d32, Cout=tkvp, taps=1, a_hi=q_pl[0], a_lo=q_pl[1], w_hi=k_pl[0],
                         w_lo=k_pl[1], out=s, passes=3)
            be.conv_umma(B=1, H=H, W=W, Cin=d32, Cout=tkvp, taps=1, a_hi=do_pl[0], a_lo=do_pl[1], w_hi=v_pl[0],
                         w_lo=v_pl[1], out=dp, passes=3)
            s2, dp2 = s.view(T, tkvp), dp.view(T, tkvp)
            be.softmax_rows_split(s2, scale, p_pl[0].view(T, tkvp), p_pl[1].view(T, tkvp), **masked)
            be.softmax_rows_split(s2, scale, ds_pl[0].view(T, tkvp), ds_pl[1].view(T, tkvp), grad=dp2, **masked)
            be.conv_umma(B=1, H=H, W=W, Cin=tkvp, Cout=d32, taps=1, a_hi=ds_pl[0], a_lo=ds_pl[1], w_hi=kt_pl[0],
                         w_lo=kt_pl[1], out=dqo, passes=3)
            be.conv_wgrad(*qt_pl, ds_pl[0], ds_pl[1], 1, H, W, tkvp, d32, 1, dkw, ws)
            be.conv_wgrad(*dot_pl, p_pl[0], p_pl[1], 1, H, W, tkvp, d32, 1, dvw, ws)
            dq[b, :, h].copy_(dqo.view(T, d32)[:, :d])
            dk[b, :, h].copy_(dkw.view(d32, tkvp)[:d, :tkv].t())
            dv[b, :, h].copy_(dvw.view(d32, tkvp)[:d, :tkv].t())
    return out


def _qkv_heads(t, heads, order):
    """q, k, v views [B, T, heads, d] of an NHWC qkv tensor [B, H, W, 3C]: order 1 puts head h's q, k, v at channels
    h*d, C + h*d, 2C + h*d; order 0 (legacy) at 3hd, 3hd + d, 3hd + 2d."""
    B, H, W, C3 = t.shape
    d = C3 // 3 // heads
    v = t.view(B, H * W, 3, heads, d) if order else t.view(B, H * W, heads, 3, d).transpose(2, 3)
    return v[:, :, 0], v[:, :, 1], v[:, :, 2]


def _pad_heads(be, t, heads, scales, order, planes=False):
    """fp32 [..., G*dp] copy of an fp32 NHWC tensor t [..., G*d] on the padded-head route (prep(heads=...): each
    head's columns zero-filled from d to dp = d rounded up to 8, tensor i of len(scales) scaled by scales[i]), and with
    planes also its split planes; returns (fp32, hi, lo)."""
    d = t.shape[-1] // (len(scales) * heads)
    shape = t.shape[:-1] + (len(scales) * heads * cabi.pad_heads_width(d),)
    f = torch.empty(shape, dtype=torch.float32, device=t.device)
    hi = lo = None
    if planes:
        hi, lo = torch.empty(shape, dtype=torch.bfloat16, device=t.device), torch.empty(shape, dtype=torch.bfloat16, device=t.device)
    be.prep(t, None, raw_f32=f, raw_hi=hi, raw_lo=lo, heads=(heads, scales, order))
    return f, hi, lo


def _unpad_heads(be, t, heads, scales, order, d):
    """fp32 [..., G*d] of a padded [..., G*dp] tensor (prep(heads=...)), tensor i scaled by scales[i]."""
    out = torch.empty(t.shape[:-1] + (len(scales) * heads * d,), dtype=torch.float32, device=t.device)
    be.prep(t, None, raw_f32=out, heads=(heads, scales, order))
    return out


class AttentionCoreFn(torch.autograd.Function):
    """softmax((q s)(k s)^T) v per head (QKVAttentionLegacy / QKVAttention, openaimodel.py:350-413) on a
    [B,3C,H,W] qkv tensor -> [B,C,H,W].  Forward: the sampling path's attention kernels (wgmma for
    head_dim 64 and 128, the fp32-qkv mma.sync kernel for the other multiples of 8 up to the backend's
    attn_max_head_dim, 256 on CudaBackend; a width d that is not a multiple of 8 runs at d rounded up to 8 with the
    heads repacked, _pad_heads); backward: bbdm_attention_bwd (flash-style recompute, exact fp32) -- the T x T matrix
    is never stored, which also replaces the reference's checkpoint() around the block (openaimodel.py:318)."""

    @staticmethod
    def forward(ctx, qkv, heads, order):
        be = backend()
        B, C3, H, W = qkv.shape
        Cc, T = C3 // 3, H * W
        d = Cc // heads
        dev = qkv.device
        qn = _nhwc(qkv.detach()).contiguous()
        ctx.heads, ctx.order = heads, order
        ctx.pad = cabi.attn_pad_route(be, d)
        if cabi.attn_gemm_route(be, d):
            out = _gemm_heads(be, *_qkv_heads(qn, heads, order), (H, W)).view(B, T, Cc)
            ctx.save_for_backward(qn, out)
            return out.view(B, H, W, Cc).permute(0, 3, 1, 2)
        q_hi = q_lo = None
        dk = cabi.pad_heads_width(d) if ctx.pad else d           # the head width the kernels run
        if ctx.pad:
            # q and k scaled by (dp/d)^(1/4): the kernels' dp^-1/4 pre-scaling then gives the reference's d^-1/2
            c = cabi.pad_heads_scale(d)
            qn, q_hi, q_lo = _pad_heads(be, qn, heads, (c, c, 1.0), order, planes=dk in cabi.ATTN_TC_HEAD_DIMS)
            C3 = qn.shape[-1]
        out = torch.empty((B, T, C3 // 3), dtype=torch.float32, device=dev)
        if dk in cabi.ATTN_TC_HEAD_DIMS:
            if q_hi is None:
                q_hi = torch.empty((B, H, W, C3), dtype=torch.bfloat16, device=dev)
                q_lo = torch.empty_like(q_hi)
                be.prep(qn, None, raw_hi=q_hi, raw_lo=q_lo)
            be.attention_tc(q_hi.view(B, T, C3), q_lo.view(B, T, C3), heads, order, out, None, None)
        else:
            be.attention(qn.view(B, T, C3), heads, order, out, None, None)
        ctx.save_for_backward(qn, out)
        if ctx.pad:
            out = _unpad_heads(be, out, heads, (1.0,), 0, d)
        return out.view(B, H, W, Cc).permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dout):
        be = backend()
        qn, out = ctx.saved_tensors
        B, H, W, C3 = qn.shape
        T = H * W
        dev = dout.device
        don = _nhwc(dout).contiguous()
        if cabi.attn_gemm_route(be, C3 // 3 // ctx.heads):
            dqkv = torch.empty_like(qn)
            _gemm_heads(be, *_qkv_heads(qn, ctx.heads, ctx.order), (H, W), dout=don.view(B, T, ctx.heads, -1),
                        grads=_qkv_heads(dqkv, ctx.heads, ctx.order))
            return dqkv.permute(0, 3, 1, 2), None, None
        if ctx.pad:       # qn and out are the padded forward's; dout comes compact
            don = _pad_heads(be, don, ctx.heads, (1.0,), 0)[0]
        dqkv = torch.empty_like(qn)
        lse = torch.empty((B * ctx.heads * T,), dtype=torch.float32, device=dev)
        delta = torch.empty_like(lse)
        be.attention_bwd(qn.view(B, T, C3), out, don.view(B, T, C3 // 3), ctx.heads, ctx.order,
                         dqkv.view(B, T, C3), lse, delta)
        if ctx.pad:       # d(c q) / dq = c: dq = c dq', dk = c dk', dv unchanged
            d = dout.shape[1] // ctx.heads
            c = cabi.pad_heads_scale(d)
            dqkv = _unpad_heads(be, dqkv, ctx.heads, (c, c, 1.0), ctx.order, d)
        return dqkv.permute(0, 3, 1, 2), None, None


def attention_core(qkv4: torch.Tensor, heads: int, new_order: bool, enabled: bool = True):
    """[B,3C,H,W] -> [B,C,H,W] or None when the native kernels do not take the shape."""
    B, C3, H, W = qkv4.shape
    hd = C3 // 3 // heads
    if not (enabled and _on_device(qkv4) and qkv4.dtype == torch.float32
            and (cabi.attn_head_dims(backend())[0](hd) or cabi.attn_pad_route(backend(), hd)
                 or (cabi.attn_gemm_route(backend(), hd) and W >= 4))
            and (C3 // 3) % 4 == 0 and B * heads <= 65535):
        return None
    return AttentionCoreFn.apply(qkv4, heads, 1 if new_order else 0)


class LayerNormLinearFn(torch.autograd.Function):
    """Linear(LayerNorm(x)) of a SpatialTransformer block (norm1/2/3 followed by to_q / q|k|v / ff.net.0.proj) over
    the [B, C, H, W] token grid: LayerNorm writes the 1x1 conv's split operand planes directly (bbdm_layernorm_split);
    the backward is the conv backward followed by bbdm_layernorm_bwd.  weight: [Cout, C, 1, 1]."""

    @staticmethod
    def forward(ctx, x, gamma, beta, weight, bias, eps):
        be = backend()
        B, Cin, H, W = x.shape
        Cout = weight.shape[0]
        dev = x.device
        xn = _nhwc(x.detach()).contiguous()
        a_hi = torch.empty((B, H, W, Cin), dtype=torch.bfloat16, device=dev)
        a_lo = torch.empty_like(a_hi)
        be.layernorm_split(xn, gamma.detach(), beta.detach(), eps, out_hi=a_hi, out_lo=a_lo)
        w_hi, w_lo, wd_hi, wd_lo = _pack_weights(be, weight, True)
        out = torch.empty((B, H, W, Cout), dtype=torch.float32, device=dev)
        be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=1, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo,
                     bias=None if bias is None else bias.detach(), out=out, passes=3)
        ctx.save_for_backward(xn, gamma, a_hi, a_lo, weight, wd_hi, wd_lo)
        ctx.has_bias = bias is not None
        ctx.shape = (B, H, W, Cin, Cout, 1)
        ctx.eps = eps
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dy):
        be = backend()
        xn, gamma, a_hi, a_lo, weight, wd_hi, wd_lo = ctx.saved_tensors
        da, dw, dbias = _conv_backward(be, ctx.shape, a_hi, a_lo, weight, dy, True, ctx.needs_input_grad[3],
                                       ctx.has_bias and ctx.needs_input_grad[4], wd=(wd_hi, wd_lo))
        Cin = xn.shape[3]
        dev = dy.device
        dxn = torch.empty_like(xn)
        dgamma = torch.empty((Cin,), dtype=torch.float32, device=dev)
        dbeta = torch.empty_like(dgamma)
        ws = torch.empty((cabi.layernorm_bwd_workspace(xn.numel() // Cin, Cin),), dtype=torch.float32, device=dev)
        be.layernorm_bwd(xn, da, gamma.detach(), ctx.eps, dxn, dgamma, dbeta, ws)
        return dxn.permute(0, 3, 1, 2), dgamma, dbeta, dw, dbias, None


class GEGLULinearFn(torch.autograd.Function):
    """Linear(a * gelu(g)) for u = [a | g] (FeedForward(glu=True): GEGLU then ff.net.2) over the [B, 2N, H, W] token
    grid: the gate writes the 1x1 conv's split operand planes directly (bbdm_geglu_split); the backward is the conv
    backward followed by bbdm_geglu_bwd.  weight: [Cout, N, 1, 1]."""

    @staticmethod
    def forward(ctx, u, weight, bias):
        be = backend()
        B, N2, H, W = u.shape
        Cout = weight.shape[0]
        dev = u.device
        un = _nhwc(u.detach()).contiguous()
        g_hi = torch.empty((B, H, W, N2 // 2), dtype=torch.bfloat16, device=dev)
        g_lo = torch.empty_like(g_hi)
        be.geglu_split(un, out_hi=g_hi, out_lo=g_lo)
        w_hi, w_lo, wd_hi, wd_lo = _pack_weights(be, weight, True)
        out = torch.empty((B, H, W, Cout), dtype=torch.float32, device=dev)
        be.conv_umma(B=B, H=H, W=W, Cin=N2 // 2, Cout=Cout, taps=1, a_hi=g_hi, a_lo=g_lo, w_hi=w_hi, w_lo=w_lo,
                     bias=None if bias is None else bias.detach(), out=out, passes=3)
        ctx.save_for_backward(un, g_hi, g_lo, weight, wd_hi, wd_lo)
        ctx.has_bias = bias is not None
        ctx.shape = (B, H, W, N2 // 2, Cout, 1)
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dy):
        be = backend()
        un, g_hi, g_lo, weight, wd_hi, wd_lo = ctx.saved_tensors
        dg, dw, dbias = _conv_backward(be, ctx.shape, g_hi, g_lo, weight, dy, True, ctx.needs_input_grad[1],
                                       ctx.has_bias and ctx.needs_input_grad[2], wd=(wd_hi, wd_lo))
        du = torch.empty_like(un)
        be.geglu_bwd(un, dg, du)
        return du.permute(0, 3, 1, 2), dw, dbias


class CrossAttentionCoreFn(torch.autograd.Function):
    """softmax(q k^T D^-1/2) v per head (CrossAttention, attention.py:166-192) for queries q [B, C, H, W] and keys|values
    kv [B, 2C, Hc, Wc] (k = channels [0, C), v = [C, 2C)) -> [B, C, H, W].  Forward: bbdm_attention_cross; backward:
    bbdm_attention_cross_bwd (flash-style recompute, exact fp32): no Tq x Tkv tensor is stored, which also replaces
    the reference's checkpoint() around the transformer block.  A head width d that is not a multiple of 8 runs at d
    rounded up to 8 with the heads repacked (_pad_heads)."""

    @staticmethod
    def forward(ctx, q, kv, heads):
        be = backend()
        B, Cc, H, W = q.shape
        Tq, Tkv = H * W, kv.shape[2] * kv.shape[3]
        dev = q.device
        qn, kvn = _nhwc(q.detach()).contiguous(), _nhwc(kv.detach()).contiguous()
        ctx.heads = heads
        if cabi.attn_gemm_route(be, Cc // heads):
            kv5 = kvn.view(B, Tkv, 2, heads, -1)
            out = _gemm_heads(be, qn.view(B, Tq, heads, -1), kv5[:, :, 0], kv5[:, :, 1], (H, W)).view(B, Tq, Cc)
            ctx.save_for_backward(qn, kvn, out)
            return out.view(B, H, W, Cc).permute(0, 3, 1, 2)
        d = Cc // heads
        ctx.pad = cabi.attn_pad_route(be, d)
        if ctx.pad:
            # heads at d rounded up to 8, q and k scaled by (dp/d)^(1/4): the kernel's dp^-1/2 becomes d^-1/2
            c = cabi.pad_heads_scale(d)
            qn, q_hi, q_lo = _pad_heads(be, qn, heads, (c,), 1, planes=True)
            kvn, kv_hi, kv_lo = _pad_heads(be, kvn, heads, (c, 1.0), 1, planes=True)
        else:
            planes = []
            for t in (qn, kvn):
                hi = torch.empty(t.shape, dtype=torch.bfloat16, device=dev)
                lo = torch.empty_like(hi)
                be.prep(t, None, raw_hi=hi, raw_lo=lo)
                planes += [hi, lo]
            q_hi, q_lo, kv_hi, kv_lo = planes
        Ck = qn.shape[-1]
        out = torch.empty((B, Tq, Ck), dtype=torch.float32, device=dev)
        be.attention_cross(q_hi.view(B, Tq, Ck), q_lo.view(B, Tq, Ck), kv_hi.view(B, Tkv, 2 * Ck),
                           kv_lo.view(B, Tkv, 2 * Ck), heads, out_f32=out)
        ctx.save_for_backward(qn, kvn, out)
        if ctx.pad:
            out = _unpad_heads(be, out, heads, (1.0,), 0, d)
        return out.view(B, H, W, Cc).permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dout):
        be = backend()
        qn, kvn, out = ctx.saved_tensors
        B, H, W, Cc = qn.shape
        Tq, Tkv = H * W, kvn.shape[1] * kvn.shape[2]
        dev = dout.device
        don = _nhwc(dout).contiguous()
        dq, dkv = torch.empty_like(qn), torch.empty_like(kvn)
        if cabi.attn_gemm_route(be, Cc // ctx.heads):
            kv5, dkv5 = kvn.view(B, Tkv, 2, ctx.heads, -1), dkv.view(B, Tkv, 2, ctx.heads, -1)
            _gemm_heads(be, qn.view(B, Tq, ctx.heads, -1), kv5[:, :, 0], kv5[:, :, 1], (H, W),
                        dout=don.view(B, Tq, ctx.heads, -1), grads=(dq.view(B, Tq, ctx.heads, -1), dkv5[:, :, 0],
                                                                    dkv5[:, :, 1]))
            return dq.permute(0, 3, 1, 2), dkv.permute(0, 3, 1, 2), None
        if ctx.pad:       # qn, kvn and out are the padded forward's; dout comes compact
            don = _pad_heads(be, don, ctx.heads, (1.0,), 0)[0]
        lse = torch.empty((B * ctx.heads * Tq,), dtype=torch.float32, device=dev)
        delta = torch.empty_like(lse)
        be.attention_cross_bwd(qn.view(B, Tq, Cc), kvn.view(B, Tkv, 2 * Cc), out, don.view(B, Tq, Cc), ctx.heads,
                               dq.view(B, Tq, Cc), dkv.view(B, Tkv, 2 * Cc), lse, delta)
        if ctx.pad:       # dq = c dq', dk = c dk', dv unchanged
            d = dout.shape[1] // ctx.heads
            c = cabi.pad_heads_scale(d)
            dq = _unpad_heads(be, dq, ctx.heads, (c,), 0, d)
            dkv = _unpad_heads(be, dkv, ctx.heads, (c, 1.0), 1, d)
        return dq.permute(0, 3, 1, 2), dkv.permute(0, 3, 1, 2), None


def gn_conv1x1(norm, conv1d: torch.nn.Conv1d, x4: torch.Tensor, enabled: bool = True):
    """conv1d_k1(GroupNorm32(x)) of AttentionBlock (openaimodel.py:307,321) fused like gn_act_conv2d, without
    the activation; None if the shape does not qualify."""
    if not (enabled and conv1d.kernel_size == (1,) and _tc_ok(x4, x4.shape[1], conv1d.out_channels)
            and x4.shape[1] <= 4096):
        return None
    return GNActConv2dFn.apply(x4, norm.weight, norm.bias, None, None, conv1d.weight.unsqueeze(-1), conv1d.bias,
                               0, None, False, norm.eps)


def conv2d(conv: torch.nn.Conv2d, x: torch.Tensor, enabled: bool = True) -> torch.Tensor:
    """nn.Conv2d call with the tensor-core autograd path when the shape qualifies."""
    if enabled and native_ok(conv, x):
        return Conv2dFn.apply(x, conv.weight, conv.bias)
    if enabled and small_ok(conv, x):
        return SmallConv2dFn.apply(x, conv.weight, conv.bias)
    if enabled:
        _library_path(f"Conv2d {conv.in_channels}->{conv.out_channels} k{conv.kernel_size[0]}", x)
    return conv(x)
