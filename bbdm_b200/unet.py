"""Denoising UNet -- parameter tree + dispatch.

The module tree reproduces the *parameter names and shapes* of the reference
``UNetModel`` (upstream model/BrownianBridge/base/modules/diffusionmodules/
openaimodel.py:416-703) so reference checkpoints, the EMA shadow dict
(runners/base/EMA.py:11-43) and ``weights_init`` (runners/utils.py:35-45, which keys on the
class names ``Conv2d`` / ``Linear``) work unchanged: every learnable tensor lives in a stock
``nn.Conv2d`` / ``nn.Conv1d`` / ``nn.Linear`` / ``nn.GroupNorm`` used purely as a parameter
container.

Execution:
  * no-grad CUDA calls (sampling, validation) go to :class:`bbdm_b200.engine.UNetEngine`,
    i.e. the hand-written sm_90a kernels behind the C ABI.  There is no CPU path: a CPU
    tensor raises.
  * calls that need autograd (training) run ``_forward_autograd``: an autograd graph over the same
    parameters whose nodes are the native kernels too (``bbdm_b200/train.py``: wgmma conv
    forward / data gradient / weight gradient, fused GroupNorm+FiLM+SiLU backward, flash-style
    attention backward); skip concats, residual adds, the time-embedding MLP and the loss stay
    stock tensor ops.  ``NATIVE_TRAIN_CONV = False`` runs the whole graph on library kernels.
    With ``UNetModel.train_graph`` on, that graph runs as two CUDA-graph replays (forward, backward;
    ``bbdm_b200/train_graph.py``).
"""
from __future__ import annotations

import math
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from .transformer import BasicTransformerBlock, SpatialTransformer
from .train import (attention_core as _attention_core, checkpointed as _checkpointed, conv1x1 as _conv1x1,
                    conv2d as _conv2d, downsample_conv as _downsample_conv, gn_act_conv2d as _gn_act_conv2d,
                    gn_conv1x1 as _gn_conv1x1, unread_outputs as _unread_outputs, upsample_conv as _upsample_conv)

# training path: ResBlock convolutions on the wgmma fwd / dgrad / wgrad kernels (bbdm_b200/train.py);
# set False to run the whole training graph on stock PyTorch kernels
NATIVE_TRAIN_CONV = True


class GroupNorm32(nn.GroupNorm):
    """GroupNorm(32, C), eps 1e-5, computed in fp32 (reference util.py:199-216)."""

    def forward(self, x):
        return super().forward(x.float()).type(x.dtype)


def zero_module(m):
    for p in m.parameters():
        p.detach().zero_()
    return m


def timestep_embedding(timesteps, dim, max_period=10000):
    """[cos | sin] sinusoidal embedding (reference util.py:151-171)."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(0, half, dtype=torch.float32) / half
                      ).to(device=timesteps.device)
    args = timesteps[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    return emb


class TimestepBlock(nn.Module):
    pass


class TimestepEmbedSequential(nn.Sequential, TimestepBlock):
    """Routes (x, emb) to TimestepBlocks and x to everything else (openaimodel.py:75-90)."""

    def forward(self, x, emb, context=None):
        for layer in self:
            if isinstance(layer, TimestepBlock):
                x = layer(x, emb)
            elif isinstance(layer, SpatialTransformer):
                x = layer(x, context)
            else:
                x = layer(x)
        return x


class Upsample(nn.Module):
    """nearest 2x (+ optional 3x3 conv) -- openaimodel.py:93-121."""

    def __init__(self, channels, use_conv, out_channels=None):
        super().__init__()
        self.channels, self.out_channels, self.use_conv = channels, out_channels or channels, use_conv
        if use_conv:
            self.conv = nn.Conv2d(self.channels, self.out_channels, 3, padding=1)

    def forward(self, x):
        if self.use_conv and NATIVE_TRAIN_CONV:
            # nearest-2x + conv as one tensor-core Function (no upsampled copy) where the shape qualifies
            y = _upsample_conv(self.conv, x)
            if y is not None:
                return y
        x = F.interpolate(x, scale_factor=2, mode="nearest")
        return self.conv(x) if self.use_conv else x


class Downsample(nn.Module):
    """stride-2 3x3 conv or 2x2 average pool -- openaimodel.py:137-163."""

    def __init__(self, channels, use_conv, out_channels=None):
        super().__init__()
        self.channels, self.out_channels, self.use_conv = channels, out_channels or channels, use_conv
        if use_conv:
            self.op = nn.Conv2d(self.channels, self.out_channels, 3, stride=2, padding=1)
        else:
            assert self.channels == self.out_channels
            self.op = nn.AvgPool2d(2, 2)

    def forward(self, x):
        if self.use_conv and NATIVE_TRAIN_CONV:
            y = _downsample_conv(self.op, x)          # stride-2 conv on the tensor cores where the shape qualifies
            if y is not None:
                return y
        return self.op(x)


class ResBlock(TimestepBlock):
    """GN-SiLU-[up/down]-conv3x3, FiLM/add of the timestep embedding, GN-SiLU-conv3x3, + skip
    (openaimodel.py:166-278)."""

    def __init__(self, channels, emb_channels, dropout, out_channels=None, use_conv=False,
                 use_scale_shift_norm=False, use_checkpoint=False, up=False, down=False):
        super().__init__()
        self.channels, self.out_channels = channels, out_channels or channels
        self.use_checkpoint = use_checkpoint
        self.use_scale_shift_norm, self.up, self.down = use_scale_shift_norm, up, down
        self.dropout = dropout
        self.in_layers = nn.Sequential(GroupNorm32(32, channels), nn.SiLU(),
                                       nn.Conv2d(channels, self.out_channels, 3, padding=1))
        self.emb_layers = nn.Sequential(
            nn.SiLU(),
            nn.Linear(emb_channels, 2 * self.out_channels if use_scale_shift_norm else self.out_channels))
        self.out_layers = nn.Sequential(
            GroupNorm32(32, self.out_channels), nn.SiLU(), nn.Dropout(p=dropout),
            zero_module(nn.Conv2d(self.out_channels, self.out_channels, 3, padding=1)))
        if self.out_channels == channels:
            self.skip_connection = nn.Identity()
        elif use_conv:
            self.skip_connection = nn.Conv2d(channels, self.out_channels, 3, padding=1)
        else:
            self.skip_connection = nn.Conv2d(channels, self.out_channels, 1)

    def forward(self, x, emb):
        """Training / autograd graph.  On CUDA the GN+SiLU(+FiLM)+conv chains run as fused autograd
        Functions over the tensor-core kernels (bbdm_b200/train.py) when shapes qualify.  With use_checkpoint the
        block keeps only its inputs and runs its forward again in the backward."""
        return _checkpointed(self, self._forward, x, emb)

    def _forward(self, x, emb):
        nat = NATIVE_TRAIN_CONV
        if self.up or self.down:
            h = _gn_act_conv2d(self.in_layers[0], self.in_layers[2], x, None, None, nat, resample=1 if self.up else 2)
            x = F.interpolate(x, scale_factor=2, mode="nearest") if self.up else F.avg_pool2d(x, 2)
        else:
            h = _gn_act_conv2d(self.in_layers[0], self.in_layers[2], x, None, None, nat)
        e = self.emb_layers(emb).type(h.dtype)[:, :, None, None]
        with _unread_outputs():       # a recompute needs none of the convolution outputs from here on
            skip_is_conv = isinstance(self.skip_connection, nn.Conv2d)
            if self.use_scale_shift_norm and self.dropout == 0:
                scale, shift = torch.chunk(e, 2, dim=1)
                # the skip path (identity or 1x1 conv of x) is added in the conv epilogue
                sk = _conv2d(self.skip_connection, x, nat) if skip_is_conv else x
                return _gn_act_conv2d(self.out_layers[0], self.out_layers[3], h, scale, shift, nat, residual=sk)
            else:
                if self.use_scale_shift_norm:
                    scale, shift = torch.chunk(e, 2, dim=1)
                    h = self.out_layers[0](h) * (1 + scale) + shift
                else:
                    h = self.out_layers[0](h + e)
                h = self.out_layers[2](self.out_layers[1](h))            # SiLU, Dropout
                h = _conv2d(self.out_layers[3], h, nat)
            if isinstance(self.skip_connection, nn.Conv2d):
                return _conv2d(self.skip_connection, x, nat) + h
            return x + h


class AttentionBlock(nn.Module):
    """GN -> qkv 1x1 -> multi-head softmax attention -> proj 1x1 -> +x (openaimodel.py:281-413)."""

    def __init__(self, channels, num_heads=1, num_head_channels=-1, use_checkpoint=False,
                 use_new_attention_order=False):
        super().__init__()
        self.channels = channels
        self.use_checkpoint = use_checkpoint
        if num_head_channels == -1:
            self.num_heads = num_heads
        else:
            assert channels % num_head_channels == 0, \
                f"q,k,v channels {channels} is not divisible by num_head_channels {num_head_channels}"
            self.num_heads = channels // num_head_channels
        self.new_order = use_new_attention_order
        self.norm = GroupNorm32(32, channels)
        self.qkv = nn.Conv1d(channels, channels * 3, 1)
        self.proj_out = zero_module(nn.Conv1d(channels, channels, 1))

    def forward(self, x):
        # Training forward.  The reference always wraps this in its CheckpointFunction (openaimodel.py:318); here the
        # native attention core never stores the T x T matrix, so the block is recomputed only with use_checkpoint.
        return _checkpointed(self, self._forward, x)

    def _forward(self, x):
        b, c, *spatial = x.shape
        nat = NATIVE_TRAIN_CONV and x.dim() == 4
        q4 = None
        if nat:                   # GroupNorm + qkv 1x1 on the tensor-core autograd path when the shape qualifies
            q4 = _gn_conv1x1(self.norm, self.qkv, x, True)
            if q4 is None:
                q4 = _conv1x1(self.qkv, self.norm(x), True)
        a4 = _attention_core(q4, self.num_heads, self.new_order) if q4 is not None else None
        if a4 is None:
            xf = x.reshape(b, c, -1)
            qkv = q4.reshape(b, 3 * c, -1) if q4 is not None else self.qkv(self.norm(xf))
            a = self._attention_torch(qkv)
            a4 = a.reshape(b, c, *spatial) if nat else None
        if a4 is not None:
            p4 = _conv1x1(self.proj_out, a4, True)
            if p4 is not None:
                return x + p4
            a = a4.reshape(b, c, -1)
        return (x.reshape(b, c, -1) + self.proj_out(a)).reshape(b, c, *spatial)

    def _attention_torch(self, qkv):
        """Stock-PyTorch attention core (CPU / shapes the native kernels do not take)."""
        bs, width, length = qkv.shape
        ch = width // (3 * self.num_heads)
        if self.new_order:
            q, k, v = (z.reshape(bs * self.num_heads, ch, length) for z in qkv.chunk(3, dim=1))
        else:
            q, k, v = qkv.reshape(bs * self.num_heads, ch * 3, length).split(ch, dim=1)
        scale = 1 / math.sqrt(math.sqrt(ch))
        w = torch.einsum("bct,bcs->bts", q * scale, k * scale)
        w = torch.softmax(w.float(), dim=-1).type(w.dtype)
        return torch.einsum("bts,bcs->bct", w, v).reshape(bs, -1, length)


class UNetModel(nn.Module):
    """Same constructor surface as the reference UNetModel (openaimodel.py:446-473); unknown
    template keys (conv_resample, dims, num_heads, context_dim, ...) are accepted alike."""

    # training forward and backward on CUDA-graph replays (bbdm_b200/train_graph.py); BBDM_TRAIN_GRAPH=1 turns it on
    # for every model, the attribute per class or instance
    train_graph = os.environ.get("BBDM_TRAIN_GRAPH", "0") != "0"

    def __init__(self, image_size, in_channels, model_channels, out_channels, num_res_blocks,
                 attention_resolutions, dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True,
                 dims=2, num_classes=None, use_checkpoint=False, use_fp16=False, num_heads=-1,
                 num_head_channels=-1, num_heads_upsample=-1, use_scale_shift_norm=False,
                 resblock_updown=False, use_new_attention_order=False,
                 use_spatial_transformer=False, transformer_depth=1, context_dim=None,
                 n_embed=None, legacy=True, condition_key="concat"):
        super().__init__()
        if use_spatial_transformer:
            assert context_dim is not None, "use_spatial_transformer needs context_dim (the conditioning's channel count)"
        if context_dim is not None:
            assert use_spatial_transformer, "context_dim is only used by the spatial transformer"
            if not isinstance(context_dim, int):
                context_dim = list(context_dim)
                if len(context_dim) != 1:
                    raise NotImplementedError("one context dimension per UNet is supported")
                context_dim = int(context_dim[0])
        self.use_spatial_transformer, self.context_dim = bool(use_spatial_transformer), context_dim
        if dims != 2 or num_classes is not None or n_embed is not None or use_fp16:
            raise NotImplementedError("only dims=2, unconditional-class, fp32 UNets are supported")
        if num_heads_upsample == -1:
            num_heads_upsample = num_heads
        if num_heads == -1:
            assert num_head_channels != -1, "Either num_heads or num_head_channels has to be set"
        if num_head_channels == -1:
            assert num_heads != -1, "Either num_heads or num_head_channels has to be set"
        self.image_size, self.in_channels, self.model_channels = image_size, in_channels, model_channels
        self.out_channels, self.num_res_blocks = out_channels, num_res_blocks
        self.attention_resolutions, self.dropout = attention_resolutions, dropout
        self.channel_mult, self.conv_resample = channel_mult, conv_resample
        self.num_heads, self.num_head_channels = num_heads, num_head_channels
        self.use_scale_shift_norm, self.resblock_updown = use_scale_shift_norm, resblock_updown
        self.condition_key = condition_key
        self.dtype = torch.float32

        ted = model_channels * 4
        self.time_embed = nn.Sequential(nn.Linear(model_channels, ted), nn.SiLU(), nn.Linear(ted, ted))

        def res(cin, cout, **kw):
            return ResBlock(cin, ted, dropout, out_channels=cout, use_scale_shift_norm=use_scale_shift_norm,
                            use_checkpoint=use_checkpoint, **kw)

        def attn(ch, heads):
            if use_spatial_transformer:
                # openaimodel.py:547-564 (legacy=True): heads follow num_head_channels when given, d_head = ch // heads
                n_heads = num_heads if num_head_channels == -1 else ch // num_head_channels
                return SpatialTransformer(ch, n_heads, ch // n_heads, depth=transformer_depth, context_dim=context_dim,
                                          use_checkpoint=use_checkpoint)
            return AttentionBlock(ch, num_heads=heads, num_head_channels=num_head_channels,
                                  use_checkpoint=use_checkpoint, use_new_attention_order=use_new_attention_order)

        self.input_blocks = nn.ModuleList(
            [TimestepEmbedSequential(nn.Conv2d(in_channels, model_channels, 3, padding=1))])
        chans = [model_channels]
        ch, ds = model_channels, 1
        for level, mult in enumerate(channel_mult):
            for _ in range(num_res_blocks):
                layers = [res(ch, mult * model_channels)]
                ch = mult * model_channels
                if ds in attention_resolutions:
                    layers.append(attn(ch, num_heads))
                self.input_blocks.append(TimestepEmbedSequential(*layers))
                chans.append(ch)
            if level != len(channel_mult) - 1:
                self.input_blocks.append(TimestepEmbedSequential(
                    res(ch, ch, down=True) if resblock_updown
                    else Downsample(ch, conv_resample, out_channels=ch)))
                chans.append(ch)
                ds *= 2
        self.middle_block = TimestepEmbedSequential(res(ch, ch), attn(ch, num_heads), res(ch, ch))
        self.output_blocks = nn.ModuleList([])
        for level, mult in list(enumerate(channel_mult))[::-1]:
            for i in range(num_res_blocks + 1):
                ich = chans.pop()
                layers = [res(ch + ich, model_channels * mult)]
                ch = model_channels * mult
                if ds in attention_resolutions:
                    layers.append(attn(ch, num_heads_upsample))
                if level and i == num_res_blocks:
                    layers.append(res(ch, ch, up=True) if resblock_updown
                                  else Upsample(ch, conv_resample, out_channels=ch))
                    ds //= 2
                self.output_blocks.append(TimestepEmbedSequential(*layers))
        self.out = nn.Sequential(GroupNorm32(32, ch), nn.SiLU(),
                                 zero_module(nn.Conv2d(model_channels, out_channels, 3, padding=1)))
        self.use_checkpoint = use_checkpoint
        self._engine = None

    @property
    def use_checkpoint(self):
        """Gradient checkpointing of the training graph: every ResBlock, AttentionBlock and transformer block keeps only
        its inputs in the forward and recomputes the rest in the backward (openaimodel.py:253-254, attention.py:211-212).
        Setting it sets the blocks' own switches; sampling ignores it."""
        return self._use_checkpoint

    @use_checkpoint.setter
    def use_checkpoint(self, on):
        self._use_checkpoint = bool(on)
        for m in self.modules():
            if isinstance(m, (ResBlock, AttentionBlock, BasicTransformerBlock)):
                m.use_checkpoint = bool(on)

    # ------------------------------------------------------------------------------ dispatch
    def engine(self):
        """The sm_90a executor for this parameter set (created on first use)."""
        if self._engine is None:
            from .engine import UNetEngine
            object.__setattr__(self, "_engine", UNetEngine(self))
        return self._engine

    def forward(self, x, timesteps=None, context=None, y=None, **kwargs):
        assert y is None, "must specify y if and only if the model is class-conditional"
        needs_grad = torch.is_grad_enabled() and (
            x.requires_grad or any(p.requires_grad for p in self.parameters()))
        if needs_grad:
            if self.train_graph and x.is_cuda:
                # the same graph on CUDA-graph replays (bbdm_b200/train_graph.py); None where it must run eagerly
                from . import train_graph
                emb = timestep_embedding(timesteps, self.model_channels)
                out = train_graph.forward(self, x, emb, context)
                return out if out is not None else self._forward_emb(x, emb, context)
            return self._forward_autograd(x, timesteps, context)
        eng = self.engine()       # raises if libbbdm_b200.so is not built
        if not x.is_cuda and getattr(eng.be, "requires_cuda", True):
            raise RuntimeError(
                "bbdm_b200: the denoising UNet inference path runs only on a CUDA sm_90a device "
                "(hand-written kernels behind libbbdm_b200.so); there is no CPU fallback.")
        return eng.forward(x, timesteps, context)

    def _forward_autograd(self, x, timesteps, context):
        """Training graph: plain PyTorch ops over the same parameters (openaimodel.py:721-759)."""
        return self._forward_emb(x, timestep_embedding(timesteps, self.model_channels), context)

    def _forward_emb(self, x, temb, context):
        """The training graph from the sinusoidal timestep embedding on (what train_graph captures: the embedding
        itself is computed from a host-side frequency table, which a CUDA graph cannot copy in)."""
        emb = self.time_embed(temb)
        if self.condition_key != "nocond":
            x = torch.cat([x, context], dim=1)
        h, hs = x, []
        ctx = context if self.use_spatial_transformer else None     # the transformers attend to the same 4-D context
        for i, m in enumerate(self.input_blocks):
            h = _conv2d(m[0], h, NATIVE_TRAIN_CONV) if i == 0 else m(h, emb, ctx)     # [0] is the stem conv
            hs.append(h)
        h = self.middle_block(h, emb, ctx)
        for m in self.output_blocks:
            h = m(torch.cat([h, hs.pop()], dim=1), emb, ctx)
        return _conv2d(self.out[2], self.out[1](self.out[0](h)), NATIVE_TRAIN_CONV)
