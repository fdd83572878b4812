"""UNet executor over the C-ABI kernels.

Walks the reference-shaped module tree (bbdm_b200.unet) and issues one C-ABI call per fused
step.  Data layout inside the UNet: NHWC fp32 activations in HBM; every tensor-core conv reads
its A operand as a split-bf16 plane pair produced by the one-pass ``prep`` kernel
(GroupNorm-affine + FiLM + SiLU + up/down-sampling + concat, fused) and writes fp32 NHWC with
bias / 1x1-skip / residual fused in its epilogue.  See README.md, section "Kernels".

The executor is written against a *backend* object (``cabi.CudaBackend`` -- the only product
backend).  tests/ inject an oracle-backed emulation of the same method set to verify this host
logic (block wiring, concat order, FiLM offsets, skip modes) on CPU; the product never does.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import cabi, convs
from .transformer import SpatialTransformer
from .unet import (AttentionBlock, Downsample, ResBlock, TimestepEmbedSequential, UNetModel,
                   Upsample, timestep_embedding)

GN_GROUPS = 32
GN_EPS = 1e-5


def resample_to_res(resample):
    return {cabi.RESAMPLE_NONE: cabi.RES_SAME, cabi.RESAMPLE_UP2: cabi.RES_UP2,
            cabi.RESAMPLE_DOWN2: cabi.RES_DOWN2}[resample]


class _Pool:
    """Shape-keyed free lists.  The forward pass is the same acquire/release sequence every
    call, so after the first call no allocation happens and every intermediate keeps a stable
    address (required for CUDA-graph replay, avoids allocator traffic)."""

    _serial = 0

    def __init__(self, backend, device):
        self.be, self.device, self.free = backend, device, {}
        self.padded = {}
        self.bytes = 0
        _Pool._serial += 1
        self.serial = _Pool._serial          # identity of this set of buffers (captured graphs key on it)

    def get(self, shape, dtype=torch.float32):
        key = (tuple(shape), dtype)
        lst = self.free.get(key)
        if lst:
            return lst.pop()
        t = self.be.empty(tuple(shape), dtype, self.device)
        self.bytes += t.numel() * t.element_size()
        return t

    def zero_padded(self, tag, shape, dtype=torch.float32):
        """The buffer `tag` of this shape, zeroed once when allocated and never put on the free lists: for operands
        whose users all write the same leading rows or columns and rely on the rest staying zero from call to call."""
        key = (tag, tuple(shape), dtype)
        t = self.padded.get(key)
        if t is None:
            t = self.padded[key] = self.be.empty(tuple(shape), dtype, self.device).zero_()
            self.bytes += t.numel() * t.element_size()
        return t

    def put(self, *ts):
        for t in ts:
            if t is not None:
                gn = t.__dict__.pop("_gn", None)      # fused GroupNorm partial sums travel with the tensor
                if gn is not None:
                    self.put(gn[0])
                self.free.setdefault((tuple(t.shape), t.dtype), []).append(t)


class KernelExecutor:
    """What every executor over the C-ABI kernels shares: the backend, the precision mode, the buffer
    pools, GroupNorm statistics (fused partials or a stats pass), the convolution dispatch, and the
    ResBlock flow, image head and resampling built on it."""

    gn_eps = GN_EPS

    def __init__(self, backend=None, precision: str = "split3"):
        self.be = backend if backend is not None else cabi.CudaBackend()
        assert precision in ("split3", "bf16")
        self.passes = 3 if precision == "split3" else 1
        self.precision = precision
        self._pools = {}
        self._gn_ws = None
        self._geom_cache = {}
        # Winograd F(4x4,3x3) convs (parity mode only); the thresholds per executor, defaults from convs
        self.wino = precision == "split3" and convs.WINOGRAD
        self.wino_min_c, self.wino_min_tiles = convs.WINO_MIN_C, convs.WINO_MIN_TILES
        self._wino_geom = {}

    def _umma_ok(self, cin, cout, w):
        return convs.tensor_core_ok(cin, cout, w)

    # ------------------------------------------------------------------------------ helpers
    def _pool(self, device, shape_key=None):
        """Intermediate-buffer pool for one (device, input shape).  At most two shapes stay resident (the
        steady batch and e.g. a smaller last batch of sample_to_eval); older pools are dropped so a
        long-lived model does not accumulate HBM across shape changes."""
        key = (device, shape_key)
        p = self._pools.pop(key, None)
        if p is None:
            p = _Pool(self.be, device)
            while len(self._pools) >= 2:
                self._pools.pop(next(iter(self._pools)))       # evict least recently used
        self._pools[key] = p                                   # (re)insert as most recent
        return p

    def pool_serial(self, device, shape_key):
        return self._pool(device, shape_key).serial

    def pool_bytes(self):
        return sum(p.bytes for p in self._pools.values())

    def _stats(self, pool, src1, src2, eps=None):
        eps = self.gn_eps if eps is None else eps
        B = src1.shape[0]
        mean, rstd = pool.get((B, GN_GROUPS)), pool.get((B, GN_GROUPS))
        g1 = getattr(src1, "_gn", None)
        g2 = None if src2 is None else getattr(src2, "_gn", None)
        if g1 is not None and (src2 is None or g2 is not None):
            # both tensors came out of the tensor-core conv: its epilogue already reduced them
            self.be.gn_finalize_partials(g1[0], g1[1], None if g2 is None else g2[0], 0 if g2 is None else g2[1],
                                         B, src1.shape[1] * src1.shape[2], GN_GROUPS, eps, mean, rstd)
            return mean, rstd
        if self._gn_ws is None or self._gn_ws.numel() < B * GN_GROUPS * cabi.GN_MAX_SLICES * 2 \
                or self._gn_ws.device != src1.device:
            self._gn_ws = self.be.empty((B * GN_GROUPS * cabi.GN_MAX_SLICES * 2,), torch.float64, src1.device)
        self.be.gn_stats(src1, src2, GN_GROUPS, eps, mean, rstd, self._gn_ws)
        return mean, rstd

    def _conv(self, pool, ent, *, a_f32=None, a_hi=None, a_lo=None, shape, bias=None, residual=None,
              res_mode=cabi.RES_NONE, second=None, out_split=False, want_f32=True, stride=1, out=None,
              stats=False, planes=None, taps=None, upsample2x=False, window_origin=0):
        """One convolution.  shape = (B,H,W) of the INPUT; returns (out_f32, out_hi, out_lo).  On the tensor-core
        path planes = (w_hi, w_lo) [taps][Cout][Cin] replaces the entry's hi/lo (e.g. its up-phase planes),
        upsample2x runs the fused nearest-2x conv (output at twice the input's resolution), and window_origin -1 puts
        a 4-tap conv's 2x2 window at rows/cols -1..0."""
        B, H, W = shape
        bias = ent["bias"] if bias is None else bias
        if a_hi is not None:
            w_hi, w_lo = (ent["hi"], ent["lo"]) if planes is None else planes
            taps = ent["k"] ** 2 if taps is None else taps
            cout, cin = w_hi.shape[1], w_hi.shape[2]
            f = 2 if upsample2x else 1
            oshape = (B, f * H, f * W, cout)
            if out is None:
                out = pool.get(oshape) if want_f32 else None
            oh = ol = None
            if out_split:
                oh, ol = pool.get(oshape, torch.bfloat16), pool.get(oshape, torch.bfloat16)
            kw = {} if not window_origin else dict(window_origin=window_origin)
            if second is not None:
                e2, r_hi, r_lo = second
                kw.update(Cin2=e2["cin"], a2_hi=r_hi, a2_lo=r_lo, w2_hi=e2["hi"], w2_lo=e2["lo"], bias2=e2["bias"])
            part = None
            if stats and out is not None:
                rows = f * f * self._geom(H, W)
                if rows:
                    part = pool.get((B * rows, cout, 2))
            self.be.conv_umma(B=B, H=H, W=W, Cin=cin, Cout=cout, taps=taps, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi,
                              w_lo=w_lo, bias=bias, residual=residual, res_mode=res_mode, out=out, out_hi=oh,
                              out_lo=ol, passes=self.passes, stats_partial=part, upsample2x=upsample2x, **kw)
            if part is not None:
                out._gn = (part, rows)
            return out, oh, ol
        assert second is None and res_mode in (cabi.RES_NONE, cabi.RES_SAME) and not out_split
        cout, k = ent["cout"], ent["k"]
        Ho, Wo = (H + stride - 1) // stride, (W + stride - 1) // stride
        if out is None:
            out = pool.get((B, Ho, Wo, cout))
        self.be.conv_direct(a_f32, ent["f32"], bias, residual, out, cout, k, stride)
        return out, None, None

    def _gn_act(self, pool, x, norm, umma, silu=True, eps=None):
        """GroupNorm (+ SiLU) of x as a conv operand: (a_f32, a_hi, a_lo)."""
        mean, rstd = self._stats(pool, x, None, eps=eps)
        a_f32 = a_hi = a_lo = None
        if umma:
            a_hi, a_lo = pool.get(x.shape, torch.bfloat16), pool.get(x.shape, torch.bfloat16)
        else:
            a_f32 = pool.get(x.shape)
        self.be.prep(x, None, groups=GN_GROUPS, mean=mean, rstd=rstd, gamma=norm.weight.detach(),
                     beta=norm.bias.detach(), silu=silu, resample=cabi.RESAMPLE_NONE, act_f32=a_f32, act_hi=a_hi,
                     act_lo=a_lo)
        pool.put(mean, rstd)
        return a_f32, a_hi, a_lo

    def _conv_plain(self, pool, ent, x, **kw):
        """Conv of an fp32 NHWC tensor with no normalisation in front: on the tensor-core path from x's split planes,
        else the fp32 direct conv.  kw: further _conv arguments."""
        B, H, W, _ = x.shape
        if "hi" in ent and W >= 4:
            hi, lo = pool.get(x.shape, torch.bfloat16), pool.get(x.shape, torch.bfloat16)
            self.be.prep(x, None, raw_hi=hi, raw_lo=lo)
            out, _, _ = self._conv(pool, ent, a_hi=hi, a_lo=lo, shape=(B, H, W), **kw)
            pool.put(hi, lo)
            return out
        out, _, _ = self._conv(pool, ent, a_f32=x, shape=(B, H, W), **kw)
        return out

    def _head(self, pool, h, norm, ent, out=None):
        """GroupNorm -> SiLU -> 3x3 conv of the last feature map h, which goes back to the pool here: the NHWC result,
        or into the NCHW tensor out.  A head with Cout < 64 that has padded planes runs on the tensor-core path with
        its N tile zero-padded to 64 couts, and the epilogue stores the real ones into out directly."""
        B, H, W, _ = h.shape
        if out is not None and "hi_pad" in ent and W >= 4:
            _, a_hi, a_lo = self._gn_act(pool, h, norm, True)
            self.be.conv_umma(B=B, H=H, W=W, Cin=ent["cin"], Cout=64, taps=9, a_hi=a_hi, a_lo=a_lo,
                              w_hi=ent["hi_pad"], w_lo=ent["lo_pad"], bias=ent["bias_pad"], out=out,
                              passes=self.passes, out_nchw_channels=out.shape[1])
            pool.put(a_hi, a_lo, h)
            return out
        a_f32, a_hi, a_lo = self._gn_act(pool, h, norm, "hi" in ent and W >= 4)
        pool.put(h)
        y, _, _ = self._conv(pool, ent, a_f32=a_f32, a_hi=a_hi, a_lo=a_lo, shape=(B, H, W))
        pool.put(a_f32, a_hi, a_lo)
        if out is None:
            return y
        self.be.nhwc_to_nchw(y, out)
        pool.put(y)
        return out

    def _upsample(self, pool, x, ent):
        """Nearest-2x of x, then the 3x3 conv ent unless it is None: the fused 4-phase conv on x itself where the entry has
        up-phase planes, else the direct conv of an upsampled fp32 copy."""
        B, H, W, Cc = x.shape
        if ent is not None and "up_hi" in ent and W >= 4:
            return self._conv_plain(pool, ent, x, planes=(ent["up_hi"], ent["up_lo"]), taps=4, upsample2x=True,
                                    stats=True)
        up = pool.get((B, 2 * H, 2 * W, Cc))
        self.be.prep(x, None, resample=cabi.RESAMPLE_UP2, raw_f32=up)
        if ent is None:
            return up
        out, _, _ = self._conv(pool, ent, a_f32=up, shape=(B, 2 * H, 2 * W))
        pool.put(up)
        return out

    def _avg_pool2(self, pool, x):
        """2x2 average pool of x."""
        B, H, W, Cc = x.shape
        out = pool.get((B, H // 2, W // 2, Cc))
        self.be.prep(x, None, resample=cabi.RESAMPLE_DOWN2, raw_f32=out)
        return out

    def _skip_residual(self, pool, es, src1, id_mode, r_f32, r_hi, r_lo, shape):
        """The ResBlock skip path as conv2's residual: (residual, res_mode, skip output to release).  The skip conv es
        runs on the raw input's split planes (tensor-core GEMM) or its fp32 copy; without a skip conv the residual is
        the raw fp32 input if prep wrote one, else src1 itself, resampled by conv2's epilogue (id_mode)."""
        if es is not None:
            skip, _, _ = self._conv(pool, es, a_f32=r_f32, a_hi=r_hi, a_lo=r_lo, shape=shape)
            return skip, cabi.RES_SAME, skip
        if r_f32 is not None:
            return r_f32, cabi.RES_SAME, None
        return src1, id_mode, None

    def _resblock_flow(self, pool, src1, src2, norm1, norm2, e1, e2, es, resample=cabi.RESAMPLE_NONE, film=None,
                       bias1=None):
        """ResBlock on cat(src1, src2): GN -> SiLU -> (up/down) -> conv1 (e1), GN (+FiLM) -> SiLU -> conv2 (e2), + the
        skip conv es (None: identity skip).  Conditioning, if any: film = (scale, shift) views [B, Cout] of conv2's
        FiLM rows, or bias1 = per-sample conv1 bias rows [B, Cout] that replace conv1's bias."""
        be = self.be
        B, Hs, Ws, c1 = src1.shape
        c2 = 0 if src2 is None else src2.shape[3]
        cin, cout = c1 + c2, e1["cout"]
        H, W = {cabi.RESAMPLE_NONE: (Hs, Ws), cabi.RESAMPLE_UP2: (Hs * 2, Ws * 2),
                cabi.RESAMPLE_DOWN2: (Hs // 2, Ws // 2)}[resample]
        shape, shp = (B, H, W), (B, H, W, cin)
        umma1 = self._umma_ok(cin, cout, W)
        umma2 = self._umma_ok(cout, cout, W)
        # a 1x1 skip conv rides as extra K-blocks of conv2 (or, before a Winograd conv2, as its own GEMM) on the raw
        # input's split planes; any other skip that is not plain src1 needs the raw (resampled / concatenated) input
        fuse_skip = es is not None and umma1 and umma2 and es["k"] == 1
        need_raw_f32 = (es is not None and not fuse_skip) or \
                       (es is None and (src2 is not None or (resample != cabi.RESAMPLE_NONE and not umma2)))
        r_f32 = r_hi = r_lo = None

        # ---- conv1: GN -> SiLU -> (up/down) -> conv3x3 ---------------------------------------------------------
        mean, rstd = self._stats(pool, src1, src2)
        gkw = dict(groups=GN_GROUPS, mean=mean, rstd=rstd, gamma=norm1.weight.detach(), beta=norm1.bias.detach(),
                   silu=True)
        # the up-phase and Winograd convs add conv1's own bias: not taken with per-sample bias rows
        up_phase = resample == cabi.RESAMPLE_UP2 and umma1 and "up_hi" in e1 and Ws >= 4 and bias1 is None \
            and not need_raw_f32 and not fuse_skip
        if up_phase and self.wino and "up6" in e1 and c1 % 64 == 0:
            # ... on a low-res map of 48x48 or more: the phase-stacked conv on F(6x6,3x3) tiles of the low-res map;
            # GroupNorm + SiLU are pointwise, so the input transform applies them before the (implicit) upsample
            u = e1["up6"]
            h1 = convs.wino_conv(be, pool, self._wino_geometry(B, Hs, Ws, 6), src1, src2, cout=cout,
                                 planes=(u["u_hi"], u["u_lo"], u.get("u_inv")), bias=e1["bias"], stats=True, tile=6,
                                 up2_phases=True, **gkw)
            pool.put(mean, rstd)
        elif up_phase:
            # up-ResBlock on the tensor-core path: never materialise the upsampled activation -- the conv runs as
            # 4 output phases x 2x2 taps on the low-res operand (2.25x fewer MACs)
            a_hi, a_lo = pool.get((B, Hs, Ws, cin), torch.bfloat16), pool.get((B, Hs, Ws, cin), torch.bfloat16)
            be.prep(src1, src2, **gkw, resample=cabi.RESAMPLE_NONE, act_hi=a_hi, act_lo=a_lo)
            pool.put(mean, rstd)
            h1, _, _ = self._conv(pool, e1, a_hi=a_hi, a_lo=a_lo, shape=(B, Hs, Ws), planes=(e1["up_hi"], e1["up_lo"]),
                                  taps=4, upsample2x=True, stats=True)
            pool.put(a_hi, a_lo)
        elif umma1 and not need_raw_f32 and bias1 is None and (
                resample == cabi.RESAMPLE_NONE or (resample == cabi.RESAMPLE_DOWN2 and e1.get("u_tile") == 6
                                                   and not fuse_skip)) and self._wino_ok(e1, B, H, W, c1):
            # Winograd conv1; the raw split planes for a fused 1x1 skip come out of the same input pass.  A
            # down-ResBlock's conv1 (F(6,3) only) takes the 2x2 pool of the activated input inside the input transform
            if fuse_skip:
                r_hi, r_lo = pool.get(shp, torch.bfloat16), pool.get(shp, torch.bfloat16)
            h1 = self._wino_conv(pool, e1, src1, src2, **gkw, raw_hi=r_hi, raw_lo=r_lo,
                                 down2=resample == cabi.RESAMPLE_DOWN2)
            pool.put(mean, rstd)
        else:
            a_f32 = a_hi = a_lo = None
            if umma1:
                a_hi, a_lo = pool.get(shp, torch.bfloat16), pool.get(shp, torch.bfloat16)
            else:
                a_f32 = pool.get(shp)
            if fuse_skip:
                r_hi, r_lo = pool.get(shp, torch.bfloat16), pool.get(shp, torch.bfloat16)
            if need_raw_f32:
                r_f32 = pool.get(shp)
            be.prep(src1, src2, **gkw, resample=resample, act_f32=a_f32, act_hi=a_hi, act_lo=a_lo,
                    raw_f32=r_f32, raw_hi=r_hi, raw_lo=r_lo)
            pool.put(mean, rstd)
            if bias1 is None:
                h1, _, _ = self._conv(pool, e1, a_f32=a_f32, a_hi=a_hi, a_lo=a_lo, shape=shape, stats=True)
            else:
                h1 = pool.get((B, H, W, cout))
                for b in range(B):
                    sl = lambda z: None if z is None else z[b:b + 1]
                    self._conv(pool, e1, a_f32=sl(a_f32), a_hi=sl(a_hi), a_lo=sl(a_lo), shape=(1, H, W),
                               bias=bias1[b], out=h1[b:b + 1])
            pool.put(a_f32, a_hi, a_lo)

        # ---- conv2: GN (+FiLM) -> SiLU -> conv3x3 (+skip) ------------------------------------------------------
        mean, rstd = self._stats(pool, h1, None)
        gkw = dict(groups=GN_GROUPS, mean=mean, rstd=rstd, gamma=norm2.weight.detach(), beta=norm2.bias.detach(),
                   silu=True)
        if film is not None:
            scale, shift = film
            gkw.update(film_scale=scale, film_shift=shift, film_stride=scale.stride(0))
        id_mode = resample_to_res(resample)
        if umma2 and self._wino_ok(e2, B, H, W):
            # Winograd conv2: the 1x1 skip (if any) runs as its own tensor-core GEMM and enters as the residual
            residual, res_mode, skip_out = self._skip_residual(pool, es, src1, id_mode, r_f32, r_hi, r_lo, shape)
            out = self._wino_conv(pool, e2, h1, None, **gkw, residual=residual, res_mode=res_mode)
            pool.put(mean, rstd, h1)
        else:
            b_f32 = b_hi = b_lo = None
            if umma2:
                b_hi, b_lo = pool.get((B, H, W, cout), torch.bfloat16), pool.get((B, H, W, cout), torch.bfloat16)
            else:
                b_f32 = pool.get((B, H, W, cout))
            be.prep(h1, None, **gkw, resample=cabi.RESAMPLE_NONE, act_f32=b_f32, act_hi=b_hi, act_lo=b_lo)
            pool.put(mean, rstd, h1)
            if fuse_skip:
                second, residual, res_mode, skip_out = (es, r_hi, r_lo), None, cabi.RES_NONE, None
            else:
                second = None
                residual, res_mode, skip_out = self._skip_residual(pool, es, src1, id_mode, r_f32, r_hi, r_lo, shape)
            out, _, _ = self._conv(pool, e2, a_f32=b_f32, a_hi=b_hi, a_lo=b_lo, shape=shape, residual=residual,
                                   res_mode=res_mode, second=second, stats=True)
            pool.put(b_f32, b_hi, b_lo)
        pool.put(r_f32, r_hi, r_lo, skip_out)
        return out

    def _attention_gemm(self, q, k, vt, v, shape, tkv, scale, s, p, out_f32=None, out_hi=None, out_lo=None,
                        write_k=None):
        """softmax(scale Q K^T) V of one image and one head as two tensor-core GEMMs around the row softmax; the key axis
        is padded to Tkvp, a multiple of 64, and the softmax covers its first tkv columns.
          q         (hi, lo) [1, H, W, d] query planes, shape = (H, W): T = H * W queries; d a multiple of 32
          k         (hi, lo) [1, Tkvp, d] key planes, zero in rows tkv..Tkvp-1 (the weights of S = Q K^T); write_k, if
                    given, writes their first tkv rows first
          vt, v     (hi, lo) [1, d, Tkvp] planes that receive V^T from the fp32 values v [tkv, d] (split_grad), zero
                    in columns tkv..Tkvp-1
          s, p      scratch: fp32 [1, H, W, Tkvp] scores and the (hi, lo) planes of P
          out_*     O = P V [1, H, W, d] as fp32 and / or split planes"""
        be = self.be
        H, W = shape
        T, tkvp, d = H * W, k[0].shape[1], k[0].shape[2]
        if write_k is not None:
            write_k()
        be.split_grad(v, None, None, vt[0][0, :, :tkv], vt[1][0, :, :tkv])
        be.conv_umma(B=1, H=H, W=W, Cin=d, Cout=tkvp, taps=1, a_hi=q[0], a_lo=q[1], w_hi=k[0], w_lo=k[1], out=s,
                     passes=self.passes)
        masked = {} if tkv == tkvp else dict(valid_cols=tkv)
        be.softmax_rows_split(s.view(T, tkvp), scale, p[0].view(T, tkvp), p[1].view(T, tkvp), **masked)
        be.conv_umma(B=1, H=H, W=W, Cin=tkvp, Cout=d, taps=1, a_hi=p[0], a_lo=p[1], w_hi=vt[0], w_lo=vt[1],
                     out=out_f32, out_hi=out_hi, out_lo=out_lo, passes=self.passes)

    def _attention_padded(self, pool, heads, d, srcs, order, planes, out_f32=None, out_hi=None, out_lo=None):
        """Attention whose heads are d wide, d not a multiple of 8, on the kernels at dp = d rounded up to 8.  srcs:
        (qkv,) fp32 [B, H, W, 3C] in the qkv order ``order``, or (q, kv) fp32 [B, H, W, C] and [B, Hc, Wc, 2C] for
        cross-attention.  prep(heads=...) lays every head out dp wide (zeros past d) with (dp/d)^(1/4) folded into
        q and k -- as split planes for the tensor-core kernels (planes) or fp32 for the fp32-qkv one -- the kernel runs
        at dp, and prep(heads=...) writes the [B, H, W, C] output back d wide into out_f32 and/or out_hi / out_lo."""
        be = self.be
        B, H, W = srcs[0].shape[:3]
        T, dp, c = H * W, cabi.pad_heads_width(d), cabi.pad_heads_scale(d)
        cp = heads * dp
        scales = ((c, c, 1.0),) if len(srcs) == 1 else ((c,), (c, 1.0))
        bufs, ops = [], []            # the padded operands, and their [B, tokens, width] views the kernels take
        for src, sc in zip(srcs, scales):
            shape = src.shape[:3] + (len(sc) * cp,)
            if planes:
                t = pool.get(shape, torch.bfloat16), pool.get(shape, torch.bfloat16)
                be.prep(src, None, raw_hi=t[0], raw_lo=t[1], heads=(heads, sc, order))
            else:
                t = (pool.get(shape),)
                be.prep(src, None, raw_f32=t[0], heads=(heads, sc, order))
            bufs += t
            ops += [u.view(shape[0], -1, shape[3]) for u in t]
        o = pool.get((B, H, W, cp))
        if len(srcs) == 2:
            be.attention_cross(*ops, heads, o.view(B, T, cp), None, None)
        elif planes:
            attn = be.attention_tc if dp in cabi.ATTN_TC_HEAD_DIMS else be.attention_split
            attn(*ops, heads, order, o.view(B, T, cp), None, None)
        else:
            be.attention(*ops, heads, order, o.view(B, T, cp), None, None)
        pool.put(*bufs)
        be.prep(o, None, raw_f32=out_f32, raw_hi=out_hi, raw_lo=out_lo, heads=(heads, (1.0,), 0))
        pool.put(o)

    def _geom(self, H, W):
        key = (H, W)
        r = self._geom_cache.get(key)
        if r is None:
            r = self._geom_cache[key] = self.be.conv_geometry(H, W)[3]
        return r


    # ---- Winograd F(4x4,3x3) path (csrc/winograd.cu) ----------------------------------------------------------
    def _wino_geometry(self, B, H, W, tile=4):
        key = (B, H, W, tile)
        g = self._wino_geom.get(key)
        if g is None:
            g = self._wino_geom[key] = self.be.wino_geometry(B, H, W, **({} if tile == 4 else dict(tile=tile)))
        return g

    def _wino_ok(self, ent, B, H, W, c1=None):
        """c1: channels of the first tensor of a concatenated input -- the F(6,3) input transform takes 64-channel
        chunks inside each tensor (cin % 64 == 0 alone does not give that)."""
        if not (self.wino and "u_hi" in ent):
            return False
        tile = ent["u_tile"]
        if tile == 6 and c1 is not None and c1 % 64:
            return False
        return convs.winograd_ok(self._wino_geometry(B, H, W, tile), ent["cin"], ent["cout"], self.wino_min_c,
                                 self.wino_min_tiles, tile)

    def _wino_ready(self, ent, tile=4):
        """Whether refresh_weights gives the packed conv ent Winograd planes of that tile size."""
        return self.wino and "hi" in ent and ent["k"] == 3 and convs.wino_channels_ok(ent["cin"], ent["cout"],
                                                                                     self.wino_min_c, tile)

    def _wino_conv(self, pool, ent, src1, src2, *, residual=None, res_mode=cabi.RES_NONE, down2=False, **transform):
        """GroupNorm-affine(+FiLM)+SiLU (-> 2x2 average pool if down2) -> 3x3 conv (+bias, +residual, GN partial sums)
        of cat(src1, src2) on the Winograd path with the entry's planes; transform: the wino_input arguments (groups,
        mean, rstd, ...)."""
        B, H, W, _ = src1.shape
        f = 2 if down2 else 1
        tile = ent["u_tile"]
        return convs.wino_conv(self.be, pool, self._wino_geometry(B, H // f, W // f, tile), src1, src2,
                               cout=ent["cout"], planes=(ent["u_hi"], ent["u_lo"], ent.get("u_inv")), bias=ent["bias"],
                               residual=residual, res_mode=res_mode, stats=True, tile=tile, down2=down2, **transform)


class UNetEngine(KernelExecutor):
    def __init__(self, unet: UNetModel, backend=None, precision: str = "split3"):
        super().__init__(backend, precision)
        # channel multiple of the tensor-core convs and GEMMs (32 on CudaBackend); Winograd keeps 64 (convs.wino_*)
        self.conv_multiple = convs.channel_multiple(self.be)
        self.unet = unet
        self._wkey = None
        self._w = {}
        self._table = None
        self.num_timesteps = 1000
        self.generation = 0          # bumps whenever cache/parameter ADDRESSES change (graphs key on it)

    def _umma_ok(self, cin, cout, w):
        return convs.tensor_core_ok(cin, cout, w, self.conv_multiple)

    # ------------------------------------------------------------------------------ weights
    def _params_key(self):
        return tuple((p.data_ptr(), p._version) for p in self.unet.parameters())

    @staticmethod
    def _ptrs(key):
        return None if key is None else tuple(k[0] for k in key)

    def refresh_weights(self, force=False):
        """(Re)derive the packed weight caches if any parameter changed (optimizer step, EMA
        swap, load_state_dict).  The nn.Parameters themselves stay OIHW fp32."""
        key = self._params_key()
        if not force and key == self._wkey:
            return
        be, u = self.be, self.unet
        dev = next(u.parameters()).device
        # Derived caches are re-packed into the EXISTING buffers whenever name, shape and device match (no
        # reallocation of the ~5 GB of planes when the runner swaps EMA weights in and out for validation /
        # sampling, runners/base/EMA.py:31-43).  Same parameter storage (in-place optimizer update): every address a
        # captured CUDA graph holds stays valid; changed storage (EMA .data swap, load_state_dict): biases / norm
        # affines are read through the parameters' own addresses, so graphs are re-captured (generation bump).
        old = self._w or {}
        if self._ptrs(key) != self._ptrs(self._wkey) or not self._w:
            self.generation += 1
        packer = convs.WeightPacker(be, dev, old, multiple=self.conv_multiple)
        w = packer.w
        mult = self.conv_multiple

        film_w, film_b, off = [], [], 0
        for name, m in u.named_modules():
            if isinstance(m, (nn.Conv2d, nn.Conv1d)):
                # out.2 is the UNet head (Cout = 3..16): zero-padded to one 64-wide N tile of the tensor-core conv
                packer.conv(name, m.weight, m.bias, padded_head=(name == "out.2"))
            if isinstance(m, ResBlock):
                lin = m.emb_layers[1]
                n = lin.weight.shape[0]
                assert n % 4 == 0
                b = lin.bias.detach()
                if not m.use_scale_shift_norm:
                    # h + emb_out happens before out_layers' GroupNorm: fold conv1's bias into the
                    # per-sample vector so conv1 can take it as its (per-sample) bias directly
                    b = b + m.in_layers[2].bias.detach()
                film_w.append(lin.weight.detach())
                film_b.append(b)
                w[name + "#film"] = (off, n)
                off += n
        for name, m in u.named_modules():
            if isinstance(m, SpatialTransformer):
                # every nn.Linear of the transformer blocks as a 1x1 "conv" over the token grid; q|k|v of the
                # self-attention (and k|v of the cross-attention) concatenated into one GEMM each
                for j, blk in enumerate(m.transformer_blocks):
                    pre = f"{name}.transformer_blocks.{j}"
                    a1, a2 = blk.attn1, blk.attn2
                    packer.conv(pre + ".attn1.qkv", torch.cat([a1.to_q.weight, a1.to_k.weight, a1.to_v.weight], 0), None)
                    packer.conv(pre + ".attn1.to_out.0", a1.to_out[0].weight, a1.to_out[0].bias)
                    packer.conv(pre + ".attn2.to_q", a2.to_q.weight, None)
                    packer.conv(pre + ".attn2.to_kv", torch.cat([a2.to_k.weight, a2.to_v.weight], 0), None)
                    packer.conv(pre + ".attn2.to_out.0", a2.to_out[0].weight, a2.to_out[0].bias)
                    packer.conv(pre + ".ff.net.0.proj", blk.ff.net[0].proj.weight, blk.ff.net[0].proj.bias)
                    packer.conv(pre + ".ff.net.2", blk.ff.net[2].weight, blk.ff.net[2].bias)
                    if cabi.attn_gemm_route(be, m.d_head):
                        for a in ("attn1", "attn2"):
                            at = getattr(blk, a)
                            self._pack_gemm_heads(packer, f"{pre}.{a}", m.n_heads, m.d_head, at.to_q.weight,
                                                  at.to_k.weight, at.to_v.weight, None, None, None,
                                                  at.to_out[0].weight, at.to_out[0].bias)
            if isinstance(m, AttentionBlock) and cabi.attn_gemm_route(be, m.channels // m.num_heads):
                C, heads = m.channels, m.num_heads
                d = C // heads
                wq, bq = m.qkv.weight.detach()[:, :, 0], m.qkv.bias.detach()
                if m.new_order:          # q, k, v of head h at channels h*d, C + h*d, 2C + h*d
                    rows = lambda j: torch.cat([torch.arange(j * C + h * d, j * C + (h + 1) * d) for h in range(heads)])
                else:                    # legacy: head h's q, k, v at 3hd, 3hd + d, 3hd + 2d
                    rows = lambda j: torch.cat([torch.arange(3 * h * d + j * d, 3 * h * d + (j + 1) * d)
                                                for h in range(heads)])
                r = [rows(j).to(wq.device) for j in range(3)]
                self._pack_gemm_heads(packer, name, heads, d, wq[r[0]], wq[r[1]], wq[r[2]], bq[r[0]], bq[r[1]],
                                      bq[r[2]], m.proj_out.weight.detach()[:, :, 0], m.proj_out.bias)
        sizes = self._resblock_sizes()
        for name, m in u.named_modules():
            # Winograd planes for the stride-1 3x3 convs of the scale-shift ResBlocks: F(6x6,3x3) for the convs that
            # run on a large map at the UNet's image_size (convs.wino_tile), else F(4x4,3x3); a forward at another
            # size runs the form that is packed.  A down-ResBlock's conv1 only on F(6,3), whose input transform pools
            # its input; an up-ResBlock's conv1 gets the phase planes below instead
            if isinstance(m, ResBlock) and m.use_scale_shift_norm:
                hw = sizes[name]
                tile = convs.wino_tile(hw, hw) if 6 in getattr(be, "wino_tiles", (4,)) else 4
                for cname, conv, direct in ((name + ".in_layers.2", m.in_layers[2], m.up or (m.down and tile != 6)),
                                            (name + ".out_layers.3", m.out_layers[3], False)):
                    if not direct and self._wino_ready(w[cname], tile):
                        packer.winograd(cname, conv.weight, tile)
        for name, m in u.named_modules():
            if isinstance(m, ResBlock) and m.up and m.channels % mult == 0 and m.out_channels % mult == 0:
                # up-ResBlock in_layers conv: 16 phase taps of the fused nearest-2x + 3x3 conv; on a low-res map that
                # takes F(6,3) also its phase-stacked F(6,3) planes (4*Cout outputs: 2.1x fewer tensor-core MACs
                # than the 16 phase taps at 64x64 and 128x128, edge tiles included; Winograd needs multiples of 64)
                packer.up_phase(name + ".in_layers.2", m.in_layers[2].weight)
                low = sizes[name] // 2
                if self.wino and 6 in getattr(be, "wino_tiles", (4,)) and convs.wino_tile(low, low) == 6 \
                        and m.channels % 64 == 0 and m.out_channels % 64 == 0:
                    packer.up_phase_winograd(name + ".in_layers.2", m.in_layers[2].weight)
        if getattr(be, "window_origin", False):
            for name, m in u.named_modules():
                if isinstance(m, Downsample) and m.use_conv and m.channels % mult == 0 and m.out_channels % mult == 0:
                    # Downsample conv: 2x2 taps on the space-to-depth operand instead of the fp32 stride-2 kernel
                    packer.stride2(name + ".op", m.op.weight)
        if old and old.get("film_n") == off and old["film_w"].device == dev:
            w["film_w"], w["film_b"] = old["film_w"], old["film_b"]
            torch.cat(film_w, 0, out=w["film_w"])
            torch.cat(film_b, 0, out=w["film_b"])
        else:
            w["film_w"] = torch.cat(film_w, 0).contiguous()
            w["film_b"] = torch.cat(film_b, 0).contiguous()
        w["film_n"] = off
        self._w = w
        self._wkey = key

    @staticmethod
    def _pack_gemm_heads(packer, pre, heads, d, wq, wk, wv, bq, bk, bv, wo, bo):
        """Per-head 1x1 conv entries of an attention whose heads run on the GEMM route: pre.q{h} / .k{h} / .v{h} from
        rows h*d.. of wq / wk / wv ([heads*d, Cin]) and biases, their outputs zero-padded to d32 = d rounded up to 32
        (zero weights and zero bias); pre.o{h} from columns h*d.. of the output projection wo ([Cout, heads*d]), zero
        columns past d, with the bias bo on head 0 only (the later heads add to head 0's result)."""
        d32 = cabi.gemm_heads_pad(d)

        def padded(name, field, shape, src, into):
            t = packer._buf(name, field, shape, torch.float32)     # reused across refreshes: the bias keeps its address
            t.zero_()
            into(t).copy_(src)
            return t

        for h in range(heads):
            sl = slice(h * d, (h + 1) * d)
            for j, (wt, bt) in enumerate(((wq, bq), (wk, bk), (wv, bv))):
                name = f"{pre}.{'qkv'[j]}{h}"
                w = padded(name, "w_src", (d32, wt.shape[1]), wt.detach()[sl], lambda t: t[:d])
                b = None if bt is None else padded(name, "b_src", (d32,), bt.detach()[sl], lambda t: t[:d])
                ent = packer.conv(name, w, b)
                ent["w_src"], ent["b_src"] = w, b
            name = f"{pre}.o{h}"
            w = padded(name, "w_src", (wo.shape[0], d32), wo.detach()[:, sl], lambda t: t[:, :d])
            packer.conv(name, w, None if h else bo)["w_src"] = w

    def _resblock_sizes(self):
        """{ResBlock name: side of the map its convs write} at the UNet's nominal image_size (the input side)."""
        u, side, out = self.unet, int(self.unet.image_size), {}
        for prefix, blocks in (("input_blocks", u.input_blocks), ("middle_block", [u.middle_block]),
                               ("output_blocks", u.output_blocks)):
            for i, block in enumerate(blocks):
                for j, layer in enumerate(block):
                    if isinstance(layer, Downsample) or (isinstance(layer, ResBlock) and layer.down):
                        side //= 2
                    elif isinstance(layer, Upsample) or (isinstance(layer, ResBlock) and layer.up):
                        side *= 2
                    if isinstance(layer, ResBlock):
                        out[f"{prefix}.{j}" if prefix == "middle_block" else f"{prefix}.{i}.{j}"] = side
        return out

    def _embedding_table(self, dev):
        """Rows 0..T-1 of the sinusoidal embedding (host-built with the reference's own expression,
        util.py:151-171: indexing is exact).  T follows the owning bridge model (``unet.num_timesteps``, set by
        BrownianBridgeModel.__init__) and is re-checked on every forward, outside the weight-key early return; an
        index >= T sets the device fault word in bbdm_gather_rows (the reference computes the embedding for any
        t, but its schedule gather raises for t >= T long before)."""
        want = max(self.num_timesteps, int(getattr(self.unet, "num_timesteps", 0) or 0))
        if self._table is None or self._table.shape[0] < want or self._table.device != dev:
            self.num_timesteps = want
            if self._table is not None:
                self.generation += 1      # table address changes: captured graphs must be rebuilt
            tab = timestep_embedding(torch.arange(want), self.unet.model_channels)
            self._table = tab.to(dev).contiguous()
        return self._table

    # ------------------------------------------------------------------------------ blocks
    def _resblock(self, pool, name, m: ResBlock, src1, src2, film):
        w = self._w
        assert src1.shape[3] + (0 if src2 is None else src2.shape[3]) == m.channels
        resample = cabi.RESAMPLE_UP2 if m.up else (cabi.RESAMPLE_DOWN2 if m.down else cabi.RESAMPLE_NONE)
        foff, fn = w[name + "#film"]
        rows = film[:, foff:foff + fn]
        # scale-shift: emb_out = [scale | shift] of out_layers' GroupNorm; else conv1's bias + emb_out per sample
        cond = dict(film=rows.chunk(2, dim=1)) if m.use_scale_shift_norm else dict(bias1=rows)
        es = w[name + ".skip_connection"] if isinstance(m.skip_connection, nn.Conv2d) else None
        return self._resblock_flow(pool, src1, src2, m.in_layers[0], m.out_layers[0], w[name + ".in_layers.2"],
                                   w[name + ".out_layers.3"], es, resample, **cond)

    def _attention(self, pool, name, m: AttentionBlock, x):
        be, w = self.be, self._w
        B, H, W, Cc = x.shape
        T = H * W
        eq, ep = w[name + ".qkv"], w[name + ".proj_out"]
        heads = m.num_heads
        hd = Cc // heads
        head_dim_ok, rule = cabi.attn_head_dims(be)
        umma = self._umma_ok(Cc, Cc, W)
        if cabi.attn_gemm_route(be, hd) and umma:
            _, a_hi, a_lo = self._gn_act(pool, x, m.norm, True, silu=False)
            out = self._attention_heads_gemm(pool, name, heads, hd, (a_hi, a_lo), None, (B, H, W), x)
            pool.put(a_hi, a_lo)
            return out
        pad = cabi.attn_pad_route(be, hd)
        if not (head_dim_ok(hd) or pad):
            raise NotImplementedError(f"attention head_dim {hd}: the sm_90a kernels take {rule}")
        a_f32, a_hi, a_lo = self._gn_act(pool, x, m.norm, umma, silu=False)
        # qkv 1x1: on the tensor-core path its epilogue writes the split planes the attention core reads (fp32 for the
        # padded-head route, which repacks it)
        qkv, q_hi, q_lo = self._conv(pool, eq, a_f32=a_f32, a_hi=a_hi, a_lo=a_lo, shape=(B, H, W),
                                     out_split=umma and not pad, want_f32=pad or not umma)
        pool.put(a_f32, a_hi, a_lo)
        o_f32 = o_hi = o_lo = None
        order = 1 if m.new_order else 0
        if pad:
            if umma:
                o_hi, o_lo = pool.get(x.shape, torch.bfloat16), pool.get(x.shape, torch.bfloat16)
            else:
                o_f32 = pool.get(x.shape)
            self._attention_padded(pool, heads, hd, (qkv,), order, umma, o_f32, o_hi, o_lo)
        elif umma:
            o_hi, o_lo = pool.get(x.shape, torch.bfloat16), pool.get(x.shape, torch.bfloat16)
            # head_dim 64 (all templates) or 128: warp-specialised wgmma kernel; any other size (up to 256): the
            # mma.sync one
            attn = be.attention_tc if hd in cabi.ATTN_TC_HEAD_DIMS else be.attention_split
            attn(q_hi.view(B, T, 3 * Cc), q_lo.view(B, T, 3 * Cc), heads, order,
                 None, o_hi.view(B, T, Cc), o_lo.view(B, T, Cc))
        else:
            o_f32 = pool.get(x.shape)
            be.attention(qkv.view(B, T, 3 * Cc), heads, order, o_f32.view(B, T, Cc), None, None)
        pool.put(qkv, q_hi, q_lo)
        out, _, _ = self._conv(pool, ep, a_f32=o_f32, a_hi=o_hi, a_lo=o_lo, shape=(B, H, W),
                               residual=x, res_mode=cabi.RES_SAME, stats=True)
        pool.put(o_f32, o_hi, o_lo)
        return out

    def _attention_heads_gemm(self, pool, pre, heads, d, a, ctx, shape, residual, stats=True):
        """Multi-head attention whose heads are wider than the flash kernels take, and its output projection: per head
        the q/k/v 1x1 convs of its padded slices (pre.q{h}, .k{h}, .v{h}: d32 = d rounded up to 32 outputs), per image
        the GEMM-composed core (_attention_gemm), then the head's slice of the output projection (pre.o{h}) added to the
        running result.  a: (hi, lo) [B, H, W, Cin] planes the projections read; ctx: fp32 [B, Hc, Wc, Cc] context the k
        and v projections read instead (fp32 direct conv: few channels), or None; residual: fp32 [B, H, W, Cout] the
        first head's projection adds.  Scratch is one image-head's [T, Tkvp] scores and P planes.  Returns the fp32
        output, with the GroupNorm partial sums of its last conv if stats."""
        be, w = self.be, self._w
        B, H, W = shape
        T = H * W
        bf = torch.bfloat16
        d32 = cabi.gemm_heads_pad(d)
        kv_shape = shape if ctx is None else tuple(ctx.shape[:3])
        tkv = kv_shape[1] * kv_shape[2]
        tkvp = -(-tkv // 64) * 64
        k_pl = pool.zero_padded(("gemm heads K", tkv), (2, tkvp, d32), bf)
        vt_pl = pool.zero_padded(("gemm heads V^T", tkv), (2, d32, tkvp), bf)
        s = pool.get((1, H, W, tkvp))
        p = pool.get((1, H, W, tkvp), bf), pool.get((1, H, W, tkvp), bf)
        scale = float(d ** -0.5)
        out = residual
        for h in range(heads):
            eq, ek, ev = w[f"{pre}.q{h}"], w[f"{pre}.k{h}"], w[f"{pre}.v{h}"]
            _, q_hi, q_lo = self._conv(pool, eq, a_hi=a[0], a_lo=a[1], shape=shape, out_split=True, want_f32=False)
            k = None
            if ctx is None:
                v, _, _ = self._conv(pool, ev, a_hi=a[0], a_lo=a[1], shape=shape)
            else:
                k, _, _ = self._conv(pool, ek, a_f32=ctx, shape=kv_shape)
                v, _, _ = self._conv(pool, ev, a_f32=ctx, shape=kv_shape)
            o_hi, o_lo = pool.get((B, H, W, d32), bf), pool.get((B, H, W, d32), bf)
            k_rows = (k_pl[0, :tkv].view(1, *kv_shape[1:], d32), k_pl[1, :tkv].view(1, *kv_shape[1:], d32))
            for b in range(B):
                if ctx is None:      # K of this image straight into the padded planes (its k 1x1 conv's epilogue)
                    write_k = lambda b=b: be.conv_umma(
                        B=1, H=H, W=W, Cin=ek["cin"], Cout=d32, taps=1, a_hi=a[0][b:b + 1], a_lo=a[1][b:b + 1],
                        w_hi=ek["hi"], w_lo=ek["lo"], bias=ek["bias"], out=None, out_hi=k_rows[0], out_lo=k_rows[1],
                        passes=self.passes)
                else:
                    write_k = lambda b=b: be.prep(k[b:b + 1], None, raw_hi=k_rows[0], raw_lo=k_rows[1])
                self._attention_gemm((q_hi[b:b + 1], q_lo[b:b + 1]), (k_pl[0:1], k_pl[1:2]), (vt_pl[0:1], vt_pl[1:2]),
                                     v[b].view(tkv, d32), (H, W), tkv, scale, s, p, out_hi=o_hi[b:b + 1],
                                     out_lo=o_lo[b:b + 1], write_k=write_k)
            pool.put(q_hi, q_lo, k, v)
            new, _, _ = self._conv(pool, w[f"{pre}.o{h}"], a_hi=o_hi, a_lo=o_lo, shape=shape, residual=out,
                                   res_mode=cabi.RES_SAME, stats=stats and h == heads - 1)
            pool.put(o_hi, o_lo)
            if out is not residual:
                pool.put(out)
            out = new
        pool.put(s, *p)
        return out

    def _stem(self, pool, ent, x):
        """A bare nn.Conv2d inside a block = the UNet stem (openaimodel.py:524): few input channels.  Dedicated kernel
        (weights in shared memory, GroupNorm partial sums of the output fused) when the shape fits, else the general
        fp32 kernel."""
        B, H, W, cin = x.shape
        cout = ent["cout"]
        if ent["k"] == 3 and cin <= 16 and cout % 32 == 0 and cout <= 128 and W % 32 == 0 and hasattr(self.be, "conv_stem"):
            out = pool.get((B, H, W, cout))
            part = pool.get((B * H, cout, 2))
            self.be.conv_stem(x, ent["f32"], ent["bias"], out, cout, stats_partial=part)
            out._gn = (part, H)
            return out
        out, _, _ = self._conv(pool, ent, a_f32=x, shape=(B, H, W))
        return out

    def _spatial_transformer(self, pool, name, m: SpatialTransformer, x, ctx):
        """GroupNorm(1e-6) -> proj_in -> [LN -> self-attention -> +, LN -> cross-attention(context) -> +,
        LN -> GEGLU feed-forward -> +] x depth -> proj_out -> + x   (reference attention.py:196-264).  Every Linear /
        1x1 conv is a wgmma GEMM over the token grid whose epilogue adds the residual; LayerNorm and GEGLU write the
        next GEMM's split operand planes directly."""
        be, w = self.be, self._w
        B, H, W, Cc = x.shape
        T, heads, d = H * W, m.n_heads, m.d_head
        inner = heads * d
        head_dim_ok, rule = cabi.attn_head_dims(be)
        gemm, pad = cabi.attn_gemm_route(be, d), cabi.attn_pad_route(be, d)
        if not (head_dim_ok(d) or gemm or pad):
            raise NotImplementedError(f"SpatialTransformer head_dim {d}: the sm_90a attention kernels take {rule}")
        if not self._umma_ok(Cc, inner, W):
            raise NotImplementedError(f"SpatialTransformer: channel counts must be multiples of {self.conv_multiple} "
                                      "(tensor-core GEMMs)")
        bf = torch.bfloat16
        tok = (B, H, W, inner)
        _, a_hi, a_lo = self._gn_act(pool, x, m.norm, True, silu=False, eps=m.norm.eps)
        h, _, _ = self._conv(pool, w[name + ".proj_in"], a_hi=a_hi, a_lo=a_lo, shape=(B, H, W))
        pool.put(a_hi, a_lo)

        def layernorm(ln, src):
            n_hi, n_lo = pool.get(tok, bf), pool.get(tok, bf)
            be.layernorm_split(src, ln.weight.detach(), ln.bias.detach(), ln.eps, out_hi=n_hi, out_lo=n_lo)
            return n_hi, n_lo

        def project_out(ent, o_hi, o_lo, res):
            new, _, _ = self._conv(pool, ent, a_hi=o_hi, a_lo=o_lo, shape=(B, H, W), residual=res, res_mode=cabi.RES_SAME)
            pool.put(o_hi, o_lo, res)
            return new

        def feed_forward(pre, blk, h):
            # ---- GEGLU feed-forward -----------------------------------------------------------------------------------
            if not blk.ff.glu:
                raise NotImplementedError("SpatialTransformer feed-forward without GEGLU")
            n_hi, n_lo = layernorm(blk.norm3, h)
            uu, _, _ = self._conv(pool, w[pre + ".ff.net.0.proj"], a_hi=n_hi, a_lo=n_lo, shape=(B, H, W))
            pool.put(n_hi, n_lo)
            ffi = uu.shape[3] // 2
            g_hi, g_lo = pool.get((B, H, W, ffi), bf), pool.get((B, H, W, ffi), bf)
            be.geglu_split(uu, out_hi=g_hi, out_lo=g_lo)
            pool.put(uu)
            return project_out(w[pre + ".ff.net.2"], g_hi, g_lo, h)

        for j, blk in enumerate(m.transformer_blocks):
            pre = f"{name}.transformer_blocks.{j}"
            # ---- self-attention ----------------------------------------------------------------------------------
            n_hi, n_lo = layernorm(blk.norm1, h)
            if gemm:
                # heads wider than the flash kernels take: per head GEMMs around the row softmax, to_out per head
                new = self._attention_heads_gemm(pool, pre + ".attn1", heads, d, (n_hi, n_lo), None, (B, H, W), h,
                                                 stats=False)
                pool.put(n_hi, n_lo, h)
                n_hi, n_lo = layernorm(blk.norm2, new)
                h = self._attention_heads_gemm(pool, pre + ".attn2", heads, d, (n_hi, n_lo), ctx, (B, H, W), new,
                                               stats=False)
                pool.put(n_hi, n_lo, new)
                h = feed_forward(pre, blk, h)
                continue
            if pad:
                # heads whose width is not a multiple of 8: the kernels at the width rounded up to 8, from fp32 q|k|v
                qkv, _, _ = self._conv(pool, w[pre + ".attn1.qkv"], a_hi=n_hi, a_lo=n_lo, shape=(B, H, W))
                pool.put(n_hi, n_lo)
                o_hi, o_lo = pool.get(tok, bf), pool.get(tok, bf)
                self._attention_padded(pool, heads, d, (qkv,), 1, True, out_hi=o_hi, out_lo=o_lo)
                pool.put(qkv)
                h = project_out(w[pre + ".attn1.to_out.0"], o_hi, o_lo, h)
                n_hi, n_lo = layernorm(blk.norm2, h)
                q, _, _ = self._conv(pool, w[pre + ".attn2.to_q"], a_hi=n_hi, a_lo=n_lo, shape=(B, H, W))
                ekv = w[pre + ".attn2.to_kv"]
                if ctx is None:
                    kv, _, _ = self._conv(pool, ekv, a_hi=n_hi, a_lo=n_lo, shape=(B, H, W))
                else:
                    kv, _, _ = self._conv(pool, ekv, a_f32=ctx, shape=tuple(ctx.shape[:3]))
                pool.put(n_hi, n_lo)
                o_hi, o_lo = pool.get(tok, bf), pool.get(tok, bf)
                self._attention_padded(pool, heads, d, (q, kv), 1, True, out_hi=o_hi, out_lo=o_lo)
                pool.put(q, kv)
                h = project_out(w[pre + ".attn2.to_out.0"], o_hi, o_lo, h)
                h = feed_forward(pre, blk, h)
                continue
            _, q_hi, q_lo = self._conv(pool, w[pre + ".attn1.qkv"], a_hi=n_hi, a_lo=n_lo, shape=(B, H, W), out_split=True,
                                       want_f32=False)
            pool.put(n_hi, n_lo)
            o_hi, o_lo = pool.get(tok, bf), pool.get(tok, bf)
            attn = be.attention_tc if d in cabi.ATTN_TC_HEAD_DIMS else be.attention_split
            attn(q_hi.view(B, T, 3 * inner), q_lo.view(B, T, 3 * inner), heads, 1, None, o_hi.view(B, T, inner),
                 o_lo.view(B, T, inner))
            pool.put(q_hi, q_lo)
            h = project_out(w[pre + ".attn1.to_out.0"], o_hi, o_lo, h)
            # ---- cross-attention over the conditioning tokens (or over h itself without a context) ------------------
            n_hi, n_lo = layernorm(blk.norm2, h)
            _, q_hi, q_lo = self._conv(pool, w[pre + ".attn2.to_q"], a_hi=n_hi, a_lo=n_lo, shape=(B, H, W), out_split=True,
                                       want_f32=False)
            ekv = w[pre + ".attn2.to_kv"]
            if ctx is None:
                _, kv_hi, kv_lo = self._conv(pool, ekv, a_hi=n_hi, a_lo=n_lo, shape=(B, H, W), out_split=True, want_f32=False)
                Tc = T
            else:
                Bc, Hc, Wc, _ = ctx.shape
                Tc = Hc * Wc
                kv, _, _ = self._conv(pool, ekv, a_f32=ctx, shape=(Bc, Hc, Wc))          # few context channels: fp32 direct
                kv_hi, kv_lo = pool.get(kv.shape, bf), pool.get(kv.shape, bf)
                be.prep(kv, None, resample=cabi.RESAMPLE_NONE, raw_hi=kv_hi, raw_lo=kv_lo)
                pool.put(kv)
            pool.put(n_hi, n_lo)
            o_hi, o_lo = pool.get(tok, bf), pool.get(tok, bf)
            be.attention_cross(q_hi.view(B, T, inner), q_lo.view(B, T, inner), kv_hi.view(B, Tc, 2 * inner),
                               kv_lo.view(B, Tc, 2 * inner), heads, None, o_hi.view(B, T, inner), o_lo.view(B, T, inner))
            pool.put(q_hi, q_lo, kv_hi, kv_lo)
            h = project_out(w[pre + ".attn2.to_out.0"], o_hi, o_lo, h)
            h = feed_forward(pre, blk, h)
        r_hi, r_lo = pool.get(tok, bf), pool.get(tok, bf)
        be.prep(h, None, resample=cabi.RESAMPLE_NONE, raw_hi=r_hi, raw_lo=r_lo)
        pool.put(h)
        out, _, _ = self._conv(pool, w[name + ".proj_out"], a_hi=r_hi, a_lo=r_lo, shape=(B, H, W), residual=x,
                               res_mode=cabi.RES_SAME, stats=True)
        pool.put(r_hi, r_lo)
        return out

    def _resample_layer(self, pool, name, m, x):
        if isinstance(m, Upsample):
            return self._upsample(pool, x, self._w[name + ".conv"] if m.use_conv else None)
        if not m.use_conv:
            return self._avg_pool2(pool, x)
        ent = self._w[name + ".op"]
        B, H, W, Cc = x.shape
        if "s2_hi" in ent and H % 2 == 0 and W % 2 == 0 and W // 2 >= 4:
            # stride-2 conv on the tensor cores: space-to-depth split, then the 2x2-tap conv at origin -1 on the
            # half-resolution grid, GroupNorm partial sums of the result in its epilogue
            hi = pool.get((B, H // 2, W // 2, 4 * Cc), torch.bfloat16)
            lo = pool.get((B, H // 2, W // 2, 4 * Cc), torch.bfloat16)
            self.be.s2d_split(x, hi, lo)
            out, _, _ = self._conv(pool, ent, a_hi=hi, a_lo=lo, shape=(B, H // 2, W // 2),
                                   planes=(ent["s2_hi"], ent["s2_lo"]), taps=4, stats=True, window_origin=-1)
            pool.put(hi, lo)
            return out
        out, _, _ = self._conv(pool, ent, a_f32=x, shape=x.shape[:3], stride=2)
        return out

    def _run_block(self, pool, prefix, block: TimestepEmbedSequential, h, skip, film, release_input):
        """h (+ skip, channel-concatenated behind it for the first layer) through one block.
        release_input: whether h/skip may go back to the pool once the first layer has consumed
        them (False while they are still referenced as saved skip tensors)."""
        cur, cur_skip, owned = h, skip, release_input
        for j, layer in enumerate(block):
            name = f"{prefix}.{j}"
            if isinstance(layer, ResBlock):
                new = self._resblock(pool, name, layer, cur, cur_skip, film)
            else:
                assert cur_skip is None, "a concatenated input is only consumed by a ResBlock"
                if isinstance(layer, AttentionBlock):
                    new = self._attention(pool, name, layer, cur)
                elif isinstance(layer, SpatialTransformer):
                    new = self._spatial_transformer(pool, name, layer, cur, self._ctx_nhwc)
                elif isinstance(layer, (Downsample, Upsample)):
                    new = self._resample_layer(pool, name, layer, cur)
                elif isinstance(layer, nn.Conv2d):
                    new = self._stem(pool, self._w[name], cur)
                else:
                    raise NotImplementedError(type(layer).__name__)
            if owned:
                pool.put(cur, cur_skip)
            cur, cur_skip, owned = new, None, True
        return cur

    # ------------------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, x, timesteps, context=None, assume_fresh_weights=False, out=None):
        u, be = self.unet, self.be
        if not assume_fresh_weights:
            self.refresh_weights()
        w = self._w
        dev = x.device
        x = x.contiguous().float()
        B, Cx, H, W = x.shape
        pool = self._pool(dev, (B, H, W))
        ctx = None
        if u.condition_key != "nocond":
            ctx = context.contiguous().float()
        t = timesteps.to(device=dev, dtype=torch.int64).contiguous()

        # ---- timestep embedding MLP + all FiLM projections (3 small fp32 GEMV launches) --------
        mc, ted = u.model_channels, u.model_channels * 4
        temb, e1, emb = pool.get((B, mc)), pool.get((B, ted)), pool.get((B, ted))
        film = pool.get((B, w["film_n"]))
        be.gather_rows(self._embedding_table(dev), t, temb)
        l0, l2 = u.time_embed[0], u.time_embed[2]
        be.linear(temb, l0.weight.detach(), l0.bias.detach(), e1, act_out=True)
        be.linear(e1, l2.weight.detach(), l2.bias.detach(), emb)
        be.linear(emb, w["film_w"], w["film_b"], film, act_in=True)
        pool.put(temb, e1)

        # ---- stem --------------------------------------------------------------------------------
        cin0 = Cx + (0 if ctx is None else ctx.shape[1])
        xin = pool.get((B, H, W, cin0))
        be.nchw_to_nhwc_cat(x, ctx, xin)
        self._ctx_nhwc = None
        if getattr(u, "use_spatial_transformer", False) and ctx is not None:
            # the transformers cross-attend to the same conditioning tensor (openaimodel.py:745-748), token-major
            self._ctx_nhwc = pool.get((B, ctx.shape[2], ctx.shape[3], ctx.shape[1]))
            be.nchw_to_nhwc_cat(ctx, None, self._ctx_nhwc)
        hs = []
        h = xin
        for i, block in enumerate(u.input_blocks):
            # block inputs after the stem are saved skip tensors (hs): not released here
            h = self._run_block(pool, f"input_blocks.{i}", block, h, None, film, release_input=(i == 0))
            hs.append(h)
        h = self._run_block(pool, "middle_block", u.middle_block, h, None, film, release_input=False)
        for i, block in enumerate(u.output_blocks):
            # h is the previous block's output, hs.pop() the matching skip: both die here
            h = self._run_block(pool, f"output_blocks.{i}", block, h, hs.pop(), film, release_input=True)

        # ---- head: GN -> SiLU -> conv3x3 -> NCHW ----------------------------------------------------
        if out is None:
            out = torch.empty((B, u.out_channels, H, W), dtype=torch.float32, device=dev)
        self._head(pool, h, u.out[0], w["out.2"], out)
        pool.put(emb, film, self._ctx_nhwc)
        self._ctx_nhwc = None
        return out
