"""SpatialTransformer / cross-attention conditioning -- parameter tree.

Same parameter names and shapes as the reference modules
(upstream model/BrownianBridge/base/modules/attention.py:36-264: GEGLU, FeedForward, CrossAttention,
BasicTransformerBlock, SpatialTransformer), so checkpoints, EMA and ``weights_init`` (which keys on the class
names ``Linear`` / ``Conv2d``) work unchanged.  No-grad CUDA calls are executed by
``bbdm_b200.engine.UNetEngine._spatial_transformer`` on the sm_90a kernels (GroupNorm + 1x1 projections and every
Linear on the wgmma GEMM, LayerNorm / GEGLU as fused operand-producing passes, self- and cross-attention on the flash
kernels).  ``SpatialTransformer.forward`` is the training / autograd graph: on the device it runs the autograd
Functions of ``bbdm_b200.train`` over the same kernels (each Linear a 1x1 ``Conv2dFn`` on the token grid,
LayerNorm->Linear and GEGLU->Linear fused, the attention cores with flash-style backward kernels); on CPU tensors,
shapes outside the kernels' envelope and with ``unet.NATIVE_TRAIN_CONV = False`` it runs the ``forward`` methods of
the modules below, in stock PyTorch ops.

Reference semantics kept: the UNet passes the SAME 4-D ``context`` tensor it concatenates to the input
(openaimodel.py:741-748) to every transformer, where it is flattened to ``b (h w) c`` (attention.py:171-172), so
``context_dim`` is its channel count and the cross-attention runs over all of its pixels.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import cabi, train


def _zero(m):
    for p in m.parameters():
        p.detach().zero_()
    return m


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)

    def forward(self, x):
        x, gate = self.proj(x).chunk(2, dim=-1)
        return x * F.gelu(gate)


class FeedForward(nn.Module):
    def __init__(self, dim, dim_out=None, mult=4, glu=False, dropout=0.0):
        super().__init__()
        inner = int(dim * mult)
        dim_out = dim if dim_out is None else dim_out
        project_in = GEGLU(dim, inner) if glu else nn.Sequential(nn.Linear(dim, inner), nn.GELU())
        self.glu = glu
        # indices 0 and 2 carry the parameters, like the reference's Sequential (attention.py:62-66)
        self.net = nn.Sequential(project_in, nn.Dropout(dropout), nn.Linear(inner, dim_out))

    def forward(self, x):
        return self.net(x)


class CrossAttention(nn.Module):
    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.0):
        super().__init__()
        inner = dim_head * heads
        context_dim = query_dim if context_dim is None else context_dim
        self.scale = dim_head ** -0.5
        self.heads, self.dim_head = heads, dim_head
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(context_dim, inner, bias=False)
        self.to_v = nn.Linear(context_dim, inner, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, query_dim), nn.Dropout(dropout))

    def forward(self, x, context=None):
        h = self.heads
        if context is not None:
            context = context.flatten(2).transpose(1, 2)          # 'b c h w -> b (h w) c'
        else:
            context = x
        q, k, v = self.to_q(x), self.to_k(context), self.to_v(context)
        b, n, _ = q.shape
        split = lambda t: t.reshape(b, t.shape[1], h, -1).permute(0, 2, 1, 3).reshape(b * h, t.shape[1], -1)
        q, k, v = split(q), split(k), split(v)
        attn = (torch.einsum("bid,bjd->bij", q, k) * self.scale).softmax(dim=-1)
        out = torch.einsum("bij,bjd->bid", attn, v)
        out = out.reshape(b, h, n, -1).permute(0, 2, 1, 3).reshape(b, n, -1)
        return self.to_out(out)


class BasicTransformerBlock(nn.Module):
    """checkpoint: recompute the block in the backward (the reference's default is on, attention.py:200-212; here it
    follows the UNet's use_checkpoint -- the native attention cores store no attention matrix either way)."""

    def __init__(self, dim, n_heads, d_head, dropout=0.0, context_dim=None, gated_ff=True, checkpoint=False):
        super().__init__()
        self.use_checkpoint = checkpoint
        self.attn1 = CrossAttention(query_dim=dim, heads=n_heads, dim_head=d_head, dropout=dropout)      # self-attention
        self.ff = FeedForward(dim, dropout=dropout, glu=gated_ff)
        self.attn2 = CrossAttention(query_dim=dim, context_dim=context_dim, heads=n_heads, dim_head=d_head,
                                    dropout=dropout)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(dim), nn.LayerNorm(dim), nn.LayerNorm(dim)

    def forward(self, x, context=None):
        # (the reference wraps this in its checkpoint(): same values)
        x = self.attn1(self.norm1(x)) + x
        x = self.attn2(self.norm2(x), context=context) + x
        return self.ff(self.norm3(x)) + x

    def forward_native(self, h, context=None):
        """forward() over the token grid h [B, C, H, W] (channels_last) on the autograd Functions of
        bbdm_b200.train; context: the 4-D conditioning [B, context_dim, Hc, Wc] or None."""
        a1, a2, ff = self.attn1, self.attn2, self.ff.net
        ln_linear = lambda ln, x, w, b=None: train.LayerNormLinearFn.apply(x, ln.weight, ln.bias, w, b, ln.eps)
        linear = lambda lin, x: train.Conv2dFn.apply(x, lin.weight[:, :, None, None], lin.bias)
        # q|k|v as one GEMM over the concatenated weights (autograd splits the gradient back): q at channels h*D,
        # k at C + h*D, v at 2C + h*D -- AttentionCoreFn's order 1; its (D^-1/4)^2 equals the D^-1/2 scale here
        qkv_w = lambda a: torch.cat([a.to_q.weight, a.to_k.weight, a.to_v.weight])[:, :, None, None]
        h = linear(a1.to_out[0], train.AttentionCoreFn.apply(ln_linear(self.norm1, h, qkv_w(a1)), a1.heads, 1)) + h
        if context is None:               # attn2 attends to its own input: self-attention
            o = train.AttentionCoreFn.apply(ln_linear(self.norm2, h, qkv_w(a2)), a2.heads, 1)
        else:
            # k|v of the few-channel context on the fp32 direct kernels (data gradient only if the context needs one)
            kv = train.SmallConv2dFn.apply(context, torch.cat([a2.to_k.weight, a2.to_v.weight])[:, :, None, None], None)
            o = train.CrossAttentionCoreFn.apply(ln_linear(self.norm2, h, a2.to_q.weight[:, :, None, None]), kv, a2.heads)
        h = linear(a2.to_out[0], o) + h
        u = ln_linear(self.norm3, h, ff[0].proj.weight[:, :, None, None], ff[0].proj.bias)
        return train.GEGLULinearFn.apply(u, ff[2].weight[:, :, None, None], ff[2].bias) + h


class SpatialTransformer(nn.Module):
    """GroupNorm(eps 1e-6) -> 1x1 proj_in -> depth x BasicTransformerBlock over 'b (h w) c' -> 1x1 proj_out -> + x
    (attention.py:218-264)."""

    def __init__(self, in_channels, n_heads, d_head, depth=1, dropout=0.0, context_dim=None, use_checkpoint=False):
        super().__init__()
        self.in_channels, self.n_heads, self.d_head, self.context_dim = in_channels, n_heads, d_head, context_dim
        inner = n_heads * d_head
        self.norm = nn.GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)
        self.proj_in = nn.Conv2d(in_channels, inner, kernel_size=1)
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(inner, n_heads, d_head, dropout=dropout, context_dim=context_dim,
                                   checkpoint=use_checkpoint) for _ in range(depth)])
        self.proj_out = _zero(nn.Conv2d(inner, in_channels, kernel_size=1))

    def _native_ok(self, x, context):
        """Shapes the training Functions' kernels take: tensor-core GEMM channel counts (proj_in's, in_channels ->
        inner, at the backend's channel multiple) and token grid, GroupNorm over 32 groups, LayerNorm width, attention
        head size (or a backend with the padded-head route for widths that are not a multiple of 8, or the GEMM route
        for heads wider than its attention kernels take), a few-channel fp32 context; no active dropout."""
        inner = self.n_heads * self.d_head
        be = train.backend()
        ok = (train.native_ok(self.proj_in, x) and self.in_channels % 32 == 0 and self.in_channels <= 4096
              and inner <= cabi.LN_MAX_C and (cabi.attn_head_dims(be)[0](self.d_head)
                                              or cabi.attn_pad_route(be, self.d_head)
                                              or cabi.attn_gemm_route(be, self.d_head))
              and x.shape[0] * self.n_heads <= 65535
              and not (self.training and any(m.p > 0 for m in self.modules() if isinstance(m, nn.Dropout))))
        if context is not None:
            ok = ok and (train._on_device(context) and context.dtype == torch.float32 and context.dim() == 4
                         and context.shape[0] == x.shape[0] and context.shape[1] <= 32)
        return ok

    def forward(self, x, context=None):
        from . import unet
        if unet.NATIVE_TRAIN_CONV:
            if self._native_ok(x, context):
                h = train.gn_act_conv2d(self.norm, self.proj_in, x, act=False)
                for blk in self.transformer_blocks:
                    h = train.checkpointed(blk, blk.forward_native, h, context)
                return train.conv2d(self.proj_out, h) + x
            train._library_path("SpatialTransformer", x)
        b, c, h, w = x.shape
        x_in = x
        x = self.proj_in(self.norm(x))
        x = x.flatten(2).transpose(1, 2)
        for blk in self.transformer_blocks:
            x = train.checkpointed(blk, blk, x, context)
        x = x.transpose(1, 2).reshape(b, -1, h, w)
        return self.proj_out(x) + x_in
