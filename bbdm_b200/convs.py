"""Convolution decisions shared by the UNet and VQGAN executors (engine.py, vqgan_engine.py) and the training
Functions (train.py): which convs run on the tensor cores, when a 3x3 conv takes the Winograd path, the Winograd launch sequence itself, and the packed
weight planes the executors cache.

A leaf module (torch, cabi and the torch-only weights helper): train.py is imported by unet.py, which engine.py
imports, so the shared code cannot live in engine.py.
"""
from __future__ import annotations

import os

import torch

from . import cabi
from .weights import stride2_s2d_weights, upsample_phase_weights

# Winograd F(4x4,3x3) for the stride-1 3x3 convs with at least WINO_MIN_C input and output channels (parity mode only;
# below that the transform traffic outweighs the 4x MAC saving).  BBDM_WINOGRAD=0 disables it in the sampling
# executors, BBDM_WINOGRAD_TRAIN=0 for the training forward and data gradient (the weight gradient is always direct).
# These are the defaults: each executor copies them into its wino / wino_min_c / wino_min_tiles attributes, and
# train.py into its WINO_TRAIN / WINO_MIN_C / WINO_MIN_TILES, which is where a caller overrides them.
WINOGRAD = os.environ.get("BBDM_WINOGRAD", "1") != "0"
WINOGRAD_TRAIN = os.environ.get("BBDM_WINOGRAD_TRAIN", "1") != "0"
WINO_MIN_C = int(os.environ.get("BBDM_WINO_MIN_C", "256"))
# ... and at least this many 4x4 tiles per launch: below it the 36 position GEMMs have too few M tiles each
# (measured: cfg1, 256 tiles, graph replay 3.9 -> 4.4 ms with Winograd; cfg3, 2048 tiles, 20.2 -> 17.1 ms)
WINO_MIN_TILES = int(os.environ.get("BBDM_WINO_MIN_TILES", "512"))


def channel_multiple(be):
    """The channel multiple the backend's tensor-core convolutions take (its conv_channel_multiple; 64 when it does not
    declare one)."""
    return getattr(be, "conv_channel_multiple", 64)


def tensor_core_ok(cin, cout, w, multiple=64):
    """Convolutions the tensor-core kernels take, in sampling (bbdm_conv_umma) and in training (its data gradient and
    bbdm_conv_wgrad): channel counts that are multiples of ``multiple`` (channel_multiple of the backend: 32 for
    CudaBackend) and a map at least 4 pixels wide.  Any height and batch: the forward covers ragged map edges with
    zero-filled tile boxes, the weight gradient reads its 64-pixel K blocks in TMA im2col mode wherever they wrap across
    rows and images."""
    return cin % multiple == 0 and cout % multiple == 0 and w >= 4


def wino_channels_ok(cin, cout, min_c, tile=4):
    """The channel half of the Winograd rule (the executors apply it when they pack the weight planes).

    F(6x6,3x3) (the UNet sampling executor on its large maps) also takes a conv with cin >= 256 and cout >= 128: it
    issues about 0.2x the direct kernel's MACs and pays for them with the V / M round trip through HBM, which the
    wide-input convs win.  Measured in isolation at the cfg2 shapes (B=16, tools/time_wino.py --f63-conv1, H100 80GB
    HBM3 at 700 W; GroupNorm-SiLU operand pass + direct conv against the F(6,3) chain): 640 -> 128 at 256x256
    10.8 -> 6.9 ms, 256 -> 128 at 256x256 3.8 -> 3.4 ms (both with the raw planes of the fused 1x1 skip).  128 -> 512 at
    128x128 (1.6 -> 1.9 ms: the M round trip of 512 outputs outweighs the MACs 128 inputs save) and 128 -> 128 lose and
    stay direct."""
    if cin % 64 or cout % 64:
        return False
    if min(cin, cout) >= min_c:
        return True
    return tile == 6 and cin >= 256 and cout >= 128


def wino_tile(H, W):
    """Output tile size of the sampling executor's Winograd convs at an HxW map: 6 (F(6x6,3x3), 64 transform
    positions per 6x6 tile, edge tiles zero-padded) where its position-GEMM MACs are at most 0.9x those of F(4x4,3x3)
    (36 positions per 4x4 tile): 48x48 and larger maps (0.84x at 64x64 and 128x128, 0.80x at 256x256), else 4
    (32x32: 1.11x)."""
    f6 = 64 * (-(-H // 6)) * (-(-W // 6))
    f4 = 36 * (H / 4) * (W / 4)
    return 6 if f6 <= 0.9 * f4 else 4


def winograd_ok(geometry, cin, cout, min_c, min_tiles, tile=4):
    """Whether a stride-1 3x3 conv of cin -> cout channels takes the Winograd path; geometry is the backend's
    wino_geometry(B, H, W, tile).  The size clauses count output pixels of the tile grid (tile^2 per tile), so they mean
    the same at both tile sizes: at >= 128 F(4,3) tiles' worth of pixels per image always (the choice must not depend
    on the batch size there: batch-size independent, bit-identical results at the pixel resolutions); smaller maps
    only when the whole batch has min_tiles F(4,3) tiles' worth."""
    th, tw, tiles, ok = geometry
    px = tile * tile
    return bool(ok and wino_channels_ok(cin, cout, min_c, tile) and
                (th * tw * px >= 128 * 16 or tiles * px >= min_tiles * 16))


class FreshBuffers:
    """The engines' pool interface over plain allocations (training: the buffers live as long as autograd keeps
    them)."""

    def __init__(self, device):
        self.device = device

    def get(self, shape, dtype=torch.float32):
        return torch.empty(shape, dtype=dtype, device=self.device)

    def put(self, *ts):
        pass


def wino_conv(be, pool, geometry, src1, src2, *, cout, planes=None, weight=None, dgrad=False, bias=None,
              residual=None, res_mode=cabi.RES_NONE, stats=False, tile=4, up2_phases=False, down2=False, **transform):
    """3x3 conv of cat(src1, src2) (NHWC fp32) on the Winograd path: input transform (``transform`` are the
    wino_input arguments: GroupNorm affine + FiLM + SiLU, or identity with silu=False; raw_* / act_* side outputs) ->
    (tile+2)^2 position GEMMs in one wgmma launch -> output transform (+ bias, + residual, + GroupNorm partial sums if
    stats).  tile: 4 (F(4x4,3x3)) or 6 (F(6x6,3x3)); geometry is the backend's wino_geometry for that tile.

    planes = (u_hi, u_lo, u_inv) packed beforehand (WeightPacker.winograd, same tile), or weight [Cout, Cin, 3, 3] to
    pack here (dgrad: the flipped, channel-swapped kernel).  pool: the executors' _Pool or FreshBuffers.

    up2_phases (tile 6, planes of WeightPacker.up_phase_winograd): nearest-2x upsample of the activated input, then the
    3x3 conv -- run on the input's own map as a 3x3 conv with 4*cout phase-major outputs, whose output transform
    interleaves the phases into the [B, 2H, 2W, cout] result (bias [cout], no residual).

    down2 (tile 6): the conv's input is the 2x2 average pool of the activated input; it runs on the H/2 x W/2 map, which
    geometry describes."""
    B, H, W, c1 = src1.shape
    cin = c1 + (0 if src2 is None else src2.shape[3])
    th, _, mtot, _ = geometry
    npos = (tile + 2) ** 2
    tkw = {} if tile == 4 else dict(tile=tile)
    assert not up2_phases or (tile == 6 and planes is not None and residual is None)
    assert not down2 or (tile == 6 and not up2_phases)
    if down2:
        H, W = H // 2, W // 2
        transform["down2"] = True
    ncols = 4 * cout if up2_phases else cout            # output channels of the position GEMMs
    v_hi, v_lo = pool.get((npos, mtot, cin), torch.float16), pool.get((npos, mtot, cin), torch.float16)
    be.wino_input(src1, src2, v_hi=v_hi, v_lo=v_lo, **transform, **tkw)
    if planes is None:
        u_hi, u_lo = pool.get((npos, cout, cin), torch.float16), pool.get((npos, cout, cin), torch.float16)
        # per-tensor scale of the planes: 1/s stays on the device (no host synchronisation)
        u_inv = pool.get((1,)) if getattr(be, "wino_tensor_scale", False) else None
        be.wino_pack_weight(weight.detach().contiguous(), u_hi, u_lo, dgrad=dgrad,
                            **({} if u_inv is None else dict(inv_wscale=u_inv)), **tkw)
    else:
        u_hi, u_lo, u_inv = planes
        assert u_hi.shape[0] == npos, (u_hi.shape, tile)
    m = pool.get((npos, mtot, ncols))
    be.conv_umma(B=npos, H=mtot // 16, W=16, Cin=cin, Cout=ncols, taps=1, a_hi=v_hi, a_lo=v_lo, w_hi=u_hi, w_lo=u_lo,
                 out=m, passes=3, weights_per_image=True, operand_f16=True)
    pool.put(v_hi, v_lo)
    f = 2 if up2_phases else 1
    rows = 4 * th if up2_phases else th                 # GroupNorm partial-sum rows per image
    out = pool.get((B, f * H, f * W, cout))
    part = pool.get((B * rows, cout, 2)) if stats else None
    if up2_phases:
        tkw["up2_phases"] = True
    be.wino_output(m, B=B, H=H, W=W, Cout=cout, bias=bias, residual=residual, res_mode=res_mode, out=out,
                   stats_partial=part, **({} if u_inv is None else dict(inv_wscale=u_inv)), **tkw)
    pool.put(m)
    if part is not None:
        out._gn = (part, rows)
    return out


class WeightPacker:
    """Packs conv weights into the cache entries the executors read.  Buffers of the previous cache (``old``) are
    re-packed in place when name, field, shape and device match: no reallocation of the planes when EMA weights are
    swapped in and out, and every address a captured CUDA graph holds stays valid.

    An entry has cout, cin, k, bias, f32 [k*k][Cin][Cout], and split-bf16 hi/lo [k*k][Cout][Cin] when both channel
    counts are multiples of ``multiple`` (the executor's tensor-core channel multiple).  The caller decides which convs also get a zero-padded head (padded_head), Winograd
    planes (winograd), the fused nearest-2x phase planes (up_phase) or the space-to-depth planes of a stride-2 conv
    (stride2)."""

    def __init__(self, be, device, old=None, multiple=64):
        self.be, self.device, self.old, self.w = be, device, old or {}, {}
        self.multiple = multiple

    def _buf(self, name, field, shape, dtype):
        ent = self.old.get(name)
        t = ent.get(field) if isinstance(ent, dict) else None
        if t is not None and tuple(t.shape) == tuple(shape) and t.device == self.device:
            return t
        return self.be.empty(tuple(shape), dtype, self.device)

    def conv(self, name, weight, bias, padded_head=False):
        """weight [Cout, Cin, k, k] (or Conv1d [Cout, Cin, 1] / Linear [out, in]).  padded_head: a 3x3 conv with
        Cout < 64 (an image head) gets planes zero-padded to one 64-wide N tile, for the NCHW-storing epilogue."""
        be, wt = self.be, weight.detach()
        while wt.dim() < 4:
            wt = wt.unsqueeze(-1)
        wt = wt.contiguous()
        cout, cin, k = wt.shape[0], wt.shape[1], wt.shape[2]
        ent = {"cout": cout, "cin": cin, "k": k, "bias": None if bias is None else bias.detach()}
        m = self.multiple
        if cin % m == 0 and cout % m == 0 and k in (1, 3):
            ent["hi"] = self._buf(name, "hi", (k * k, cout, cin), torch.bfloat16)
            ent["lo"] = self._buf(name, "lo", (k * k, cout, cin), torch.bfloat16)
            be.pack_weight_split(wt, ent["hi"], ent["lo"])
        elif padded_head and cin % m == 0 and cout < 64 and k == 3:
            prev = self.old[name].get("hi_pad") if isinstance(self.old.get(name), dict) else None
            hi = self._buf(name, "hi_pad", (k * k, 64, cin), torch.bfloat16)
            lo = self._buf(name, "lo_pad", (k * k, 64, cin), torch.bfloat16)
            bp = self._buf(name, "bias_pad", (64,), torch.float32)
            if hi is not prev:                   # freshly allocated: the padding rows must be zeroed
                hi.zero_()
                lo.zero_()
            bp.zero_()
            if bias is not None:
                bp[:cout].copy_(bias.detach())
            be.pack_weight_split(wt, hi, lo)
            ent["hi_pad"], ent["lo_pad"], ent["bias_pad"] = hi, lo, bp
        ent["f32"] = self._buf(name, "f32", (k * k, cin, cout), torch.float32)
        be.pack_weight_f32(wt, ent["f32"])
        self.w[name] = ent
        return ent

    def winograd(self, name, weight, tile=4):
        """Winograd-domain planes U = s G g G^T of the packed 3x3 conv ``name`` for F(tile x tile, 3x3), fp16 hi/lo
        [(tile+2)^2][Cout][Cin], and 1/s (per-tensor power of two) as a device scalar beside them: a stable address for
        graph replay.  ent["u_tile"] records the tile size."""
        ent = self.w[name]
        npos = (tile + 2) ** 2
        ent["u_hi"] = self._buf(name, "u_hi", (npos, ent["cout"], ent["cin"]), torch.float16)
        ent["u_lo"] = self._buf(name, "u_lo", (npos, ent["cout"], ent["cin"]), torch.float16)
        ent["u_tile"] = tile
        skw = {} if tile == 4 else dict(tile=tile)
        if getattr(self.be, "wino_tensor_scale", False):
            ent["u_inv"] = skw["inv_wscale"] = self._buf(name, "u_inv", (1,), torch.float32)
        self.be.wino_pack_weight(weight.detach().contiguous(), ent["u_hi"], ent["u_lo"], **skw)

    def up_phase(self, name, weight):
        """The 16 phase taps of nearest-2x + the packed 3x3 conv ``name`` (4 output phases x 2x2 taps on the low-res
        operand)."""
        ent = self.w[name]
        ent["up_hi"] = self._buf(name, "up_hi", (16, ent["cout"], ent["cin"]), torch.bfloat16)
        ent["up_lo"] = self._buf(name, "up_lo", (16, ent["cout"], ent["cin"]), torch.bfloat16)
        self.be.pack_weight_split_taps(upsample_phase_weights(weight.detach()), ent["up_hi"], ent["up_lo"])

    def stride2(self, name, weight):
        """The 3x3 stride-2 padding-1 conv ``name`` (UNet Downsample) as a 2x2-tap conv on the space-to-depth operand
        (bbdm_s2d_split): planes [4][Cout][4*Cin], window at rows/cols -1..0 (conv_umma window_origin -1)."""
        ent = self.w[name]
        ent["s2_hi"] = self._buf(name, "s2_hi", (4, ent["cout"], 4 * ent["cin"]), torch.bfloat16)
        ent["s2_lo"] = self._buf(name, "s2_lo", (4, ent["cout"], 4 * ent["cin"]), torch.bfloat16)
        self.be.pack_weight_split_taps(stride2_s2d_weights(weight.detach()), ent["s2_hi"], ent["s2_lo"])

    def up_phase_winograd(self, name, weight):
        """F(6x6,3x3) planes of nearest-2x + the packed 3x3 conv ``name`` as one 3x3 conv on the low-res map with
        4*Cout outputs, phase-major (phase = 2a + b of output pixel (2y+a, 2x+b)): each phase's 2x2 taps sit in the
        3x3 window at rows a..a+1, columns b..b+1.  A conv entry of its own, ``name + "#up6"`` (cout = 4*Cout),
        that ent["up6"] refers to, for convs.wino_conv(up2_phases=True)."""
        ent = self.w[name]
        cout, cin = ent["cout"], ent["cin"]
        pw = upsample_phase_weights(weight.detach()).view(cout, cin, 2, 2, 2, 2)      # [o, i, a, b, r, c]
        w3 = torch.zeros(2, 2, cout, cin, 3, 3, dtype=pw.dtype, device=pw.device)
        for a in range(2):
            for b in range(2):
                w3[a, b, :, :, a:a + 2, b:b + 2] = pw[:, :, a, b]
        ent["up6"] = self.w[name + "#up6"] = {"cout": 4 * cout, "cin": cin, "k": 3}
        self.winograd(name + "#up6", w3.view(4 * cout, cin, 3, 3), tile=6)
