"""VQGAN encode / decode executor over the C-ABI kernels.

The latent models call the frozen autoencoder at both ends of the bridge loop and twice per training
sample (LatentBrownianBridgeModel.py:57-100 of the reference).  This executor walks the reference's own
``VQModel`` module tree (model/VQGAN/vqgan.py:30-88, model.py:342-537 -- the module stays the parameter
container, exactly like the UNet) and issues the same kernels as the UNet executor:

  ResnetBlock (model.py:76-138)   the UNet's ResBlock flow (KernelExecutor._resblock_flow) without conditioning,
                                  GN eps 1e-6: the 1x1 nin_shortcut rides as extra K-blocks of conv2, the identity
                                  skip as its residual
  AttnBlock   (model.py:140-192)  single head of width C: C <= 64 -> the flash kernels; C >= 128 -> per image two
                                  tensor-core GEMMs (S = Q K^T, O = P V) around bbdm_softmax_rows_split, the key axis
                                  zero-padded to a multiple of 64 and masked in the softmax at any other token count
  Downsample  (model.py:55-73)    zero-pad (0,1,0,1) + stride-2 conv = space-to-depth split + 2x2-tap wgmma conv
                                  (bbdm_conv_direct_pad for unaligned channel counts)
  Upsample    (model.py:38-53)    nearest-2x + conv3x3 = the fused 4-phase wgmma conv (no upsampled tensor)
  VectorQuantizer2 (quantize.py:271-312)  bbdm_vq_nearest

Inference only (the autoencoder is frozen and always called under no_grad).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import cabi, convs
from .engine import KernelExecutor


class VQGANEngine(KernelExecutor):
    gn_eps = 1e-6                      # model/VQGAN/model.py:34-35

    def __init__(self, vqmodel: nn.Module, backend=None, precision: str = "split3"):
        super().__init__(backend, precision)
        self.vq = vqmodel
        self._w = {}
        self._wkey = None

    # ------------------------------------------------------------------------------ weights
    def _params_key(self):
        return tuple((p.data_ptr(), p._version) for p in self.vq.parameters())

    def refresh_weights(self, force=False):
        key = self._params_key()
        if not force and key == self._wkey:
            return
        be = self.be
        dev = next(self.vq.parameters()).device
        packer = convs.WeightPacker(be, dev, self._w)
        w = packer.w

        def pack(name, wt, bias):
            # any 3x3 conv with Cout < 64 is an image head (Cout = 3): NCHW-storing padded planes
            ent = packer.conv(name, wt, bias, padded_head=True)
            if (name.endswith(".conv1") or name.endswith(".conv2")) and self._wino_ready(ent):
                packer.winograd(name, wt)          # ResnetBlock 3x3 convs, like the UNet's ResBlocks

        for name, m in self.vq.named_modules():
            if isinstance(m, nn.Conv2d) and not name.startswith("loss"):
                pack(name, m.weight, m.bias)
            if type(m).__name__ == "AttnBlock" and m.in_channels <= 64:
                # q | k | v as one 1x1 conv ("new order" layout of the flash kernels, one head)
                pack(name + ".qkv", torch.cat([m.q.weight, m.k.weight, m.v.weight], 0),
                     torch.cat([m.q.bias, m.k.bias, m.v.bias], 0))
        for name, m in self.vq.named_modules():          # second pass: the convs above are packed now
            if type(m).__name__ == "Upsample" and m.with_conv and "hi" in w.get(name + ".conv", {}):
                packer.up_phase(name + ".conv", m.conv.weight)
            if type(m).__name__ == "Downsample" and m.with_conv:
                # stride-2 3x3 conv on the zero-padded input == 2x2-tap conv over the space-to-depth tensor:
                # W2[tap=(ty,tx)][co][(a*2+b)*C + ci] = w[co][ci][2ty+a][2tx+b]  (zero where 2ty+a or 2tx+b = 3)
                cw = m.conv.weight.detach()
                co, ci = cw.shape[0], cw.shape[1]
                if co % 64 == 0 and (4 * ci) % 64 == 0:
                    w2 = torch.zeros((co, 4, ci, 4), dtype=torch.float32, device=dev)     # [co][a*2+b][ci][tap]
                    for ty in range(2):
                        for tx in range(2):
                            for a in range(2):
                                for b in range(2):
                                    if 2 * ty + a < 3 and 2 * tx + b < 3:
                                        w2[:, a * 2 + b, :, ty * 2 + tx] = cw[:, :, 2 * ty + a, 2 * tx + b]
                    ent = w[name + ".conv"]
                    ent["ds_hi"] = be.empty((4, co, 4 * ci), torch.bfloat16, dev)
                    ent["ds_lo"] = be.empty((4, co, 4 * ci), torch.bfloat16, dev)
                    be.pack_weight_split_taps(w2.reshape(co, 4 * ci, 4).contiguous(), ent["ds_hi"], ent["ds_lo"])
        self._w, self._wkey = w, key

    # ------------------------------------------------------------------------------ pieces
    def _resnet(self, pool, name, m, x):
        w = self._w
        es = w.get(name + ".nin_shortcut", w.get(name + ".conv_shortcut"))
        assert (es is None) == (m.in_channels == m.out_channels)
        return self._resblock_flow(pool, x, None, m.norm1, m.norm2, w[name + ".conv1"], w[name + ".conv2"], es)

    def _attn(self, pool, name, m, x):
        be, w = self.be, self._w
        B, H, W, Cc = x.shape
        T = H * W
        ep = w[name + ".proj_out"]
        umma = self._umma_ok(Cc, Cc, W)
        a_f32, a_hi, a_lo = self._gn_act(pool, x, m.norm, umma, silu=False)
        o_f32 = o_hi = o_lo = None
        if Cc in (16, 32, 64):
            # one head of width C: the flash kernel's scale D^-1/4 on q and on k is the reference's C^-1/2
            qkv, _, _ = self._conv(pool, w[name + ".qkv"], a_f32=a_f32, a_hi=a_hi, a_lo=a_lo, shape=(B, H, W))
            if umma:
                o_hi, o_lo = pool.get(x.shape, torch.bfloat16), pool.get(x.shape, torch.bfloat16)
            else:
                o_f32 = pool.get(x.shape)
            be.attention(qkv.view(B, T, 3 * Cc), 1, 1, None if o_f32 is None else o_f32.view(B, T, Cc),
                         None if o_hi is None else o_hi.view(B, T, Cc), None if o_lo is None else o_lo.view(B, T, Cc))
            pool.put(qkv)
        elif not umma:
            raise NotImplementedError(f"VQGAN AttnBlock with C={Cc} on a {H}x{W} map: the GEMM-composed attention "
                                      f"needs C % 64 == 0 and a map at least 4 wide")
        elif T % 64:
            o_hi, o_lo = self._attn_padded(pool, name, a_hi, a_lo, x.shape)
        else:
            _, q_hi, q_lo = self._conv(pool, w[name + ".q"], a_hi=a_hi, a_lo=a_lo, shape=(B, H, W), out_split=True,
                                       want_f32=False)
            _, k_hi, k_lo = self._conv(pool, w[name + ".k"], a_hi=a_hi, a_lo=a_lo, shape=(B, H, W), out_split=True,
                                       want_f32=False)
            v, _, _ = self._conv(pool, w[name + ".v"], a_hi=a_hi, a_lo=a_lo, shape=(B, H, W))
            vt_hi, vt_lo = pool.get((B, Cc, T), torch.bfloat16), pool.get((B, Cc, T), torch.bfloat16)
            o_hi, o_lo = pool.get(x.shape, torch.bfloat16), pool.get(x.shape, torch.bfloat16)
            s = pool.get((1, H, W, T))
            p_hi, p_lo = pool.get((1, H, W, T), torch.bfloat16), pool.get((1, H, W, T), torch.bfloat16)
            scale = float(int(Cc) ** (-0.5))
            for b in range(B):
                # S[t, s] = sum_c q[t, c] k[s, c]: the K planes of this image ARE a [Cout=T][Cin=C] weight; V^T planes
                # [C][T] are the K-major B operand of O = P V
                self._attention_gemm((q_hi[b:b + 1], q_lo[b:b + 1]), (k_hi[b].view(1, T, Cc), k_lo[b].view(1, T, Cc)),
                                     (vt_hi[b].view(1, Cc, T), vt_lo[b].view(1, Cc, T)), v[b].view(T, Cc), (H, W), T,
                                     scale, s, (p_hi, p_lo), out_hi=o_hi[b:b + 1], out_lo=o_lo[b:b + 1])
            pool.put(q_hi, q_lo, k_hi, k_lo, v, vt_hi, vt_lo, s, p_hi, p_lo)
        pool.put(a_f32, a_hi, a_lo)
        out, _, _ = self._conv(pool, ep, a_f32=o_f32, a_hi=o_hi, a_lo=o_lo, shape=(B, H, W), residual=x,
                               res_mode=cabi.RES_SAME, stats=True)
        pool.put(o_f32, o_hi, o_lo)
        return out

    def _attn_padded(self, pool, name, a_hi, a_lo, shape):
        """The GEMM-composed AttnBlock at a token count T that is not a multiple of 64: the key axis is padded to
        Tp = T rounded up to 64.  Each image's k 1x1 conv writes the first T rows of [Tp][C] K planes and its V^T the
        first T columns of [C][Tp] planes, both zero beyond; S = Q K^T then has Tp columns, the softmax covers the first
        T of them and writes zeros past them, and O = P V runs over K = Tp.  Returns O's split planes."""
        be, w = self.be, self._w
        B, H, W, Cc = shape
        T = H * W
        Tp = -(-T // 64) * 64
        bf16 = torch.bfloat16
        ek = w[name + ".k"]
        _, q_hi, q_lo = self._conv(pool, w[name + ".q"], a_hi=a_hi, a_lo=a_lo, shape=(B, H, W), out_split=True,
                                   want_f32=False)
        v, _, _ = self._conv(pool, w[name + ".v"], a_hi=a_hi, a_lo=a_lo, shape=(B, H, W))
        k_pl = pool.zero_padded(("attention K", T), (2, Tp, Cc), bf16)
        vt_pl = pool.zero_padded(("attention V^T", T), (2, Cc, Tp), bf16)
        o_hi, o_lo = pool.get(shape, bf16), pool.get(shape, bf16)
        s = pool.get((1, H, W, Tp))
        p_hi, p_lo = pool.get((1, H, W, Tp), bf16), pool.get((1, H, W, Tp), bf16)
        scale = float(int(Cc) ** (-0.5))
        for b in range(B):
            write_k = lambda b=b: be.conv_umma(
                B=1, H=H, W=W, Cin=Cc, Cout=Cc, taps=1, a_hi=a_hi[b:b + 1], a_lo=a_lo[b:b + 1], w_hi=ek["hi"],
                w_lo=ek["lo"], bias=ek["bias"], out=None, out_hi=k_pl[0, :T].view(1, H, W, Cc),
                out_lo=k_pl[1, :T].view(1, H, W, Cc), passes=self.passes)
            self._attention_gemm((q_hi[b:b + 1], q_lo[b:b + 1]), (k_pl[0:1], k_pl[1:2]), (vt_pl[0:1], vt_pl[1:2]),
                                 v[b].view(T, Cc), (H, W), T, scale, s, (p_hi, p_lo), out_hi=o_hi[b:b + 1],
                                 out_lo=o_lo[b:b + 1], write_k=write_k)
        pool.put(q_hi, q_lo, v, s, p_hi, p_lo)
        return o_hi, o_lo

    def _downsample(self, pool, name, m, x):
        B, H, W, Cc = x.shape
        if not m.with_conv:
            return self._avg_pool2(pool, x)
        ent = self._w[name + ".conv"]
        if "ds_hi" in ent and H % 2 == 0 and W % 2 == 0 and W // 2 >= 4:
            hi = pool.get((B, H // 2, W // 2, 4 * Cc), torch.bfloat16)
            lo = pool.get((B, H // 2, W // 2, 4 * Cc), torch.bfloat16)
            self.be.s2d_split(x, hi, lo)
            out, _, _ = self._conv(pool, ent, a_hi=hi, a_lo=lo, shape=(B, H // 2, W // 2),
                                   planes=(ent["ds_hi"], ent["ds_lo"]), taps=4, stats=True)
            pool.put(hi, lo)
            return out
        out = pool.get((B, (H + 1 - 3) // 2 + 1, (W + 1 - 3) // 2 + 1, Cc))
        self.be.conv_direct_pad(x, ent["f32"], ent["bias"], None, out, Cc, 3, 2, 0, 1)
        return out

    def _step(self, pool, h, fn, *args):
        new = fn(pool, *args, h)
        pool.put(h)
        return new

    def _mid(self, pool, prefix, mid, h):
        h = self._step(pool, h, self._resnet, prefix + ".block_1", mid.block_1)
        h = self._step(pool, h, self._attn, prefix + ".attn_1", mid.attn_1)
        return self._step(pool, h, self._resnet, prefix + ".block_2", mid.block_2)

    def _to_nhwc(self, pool, x):
        B, Cx, H, W = x.shape
        xin = pool.get((B, H, W, Cx))
        self.be.nchw_to_nhwc_cat(x.contiguous().float(), None, xin)
        return xin

    # ------------------------------------------------------------------------------ public
    # activation budget of one pass: 32 images of 256x256 (the cfg3 batch; ~25 GB of pooled NHWC tensors and operand
    # planes).  Larger batches / resolutions run in chunks of this many image pixels -- the ends are 2-13 % of a
    # sampled batch, so nothing is lost, and BASELINE configs[3] (64 x 512^2) would otherwise need > 180 GB.
    max_pixels_per_pass = 32 * 256 * 256

    def _chunks(self, n_images, image_pixels):
        per = max(1, self.max_pixels_per_pass // max(1, image_pixels))
        return [(i, min(n_images, i + per)) for i in range(0, n_images, per)]

    @torch.no_grad()
    def encode(self, x, quant_conv=True):
        """vqgan.encoder(x) [-> vqgan.quant_conv]   (LatentBrownianBridgeModel.py:73-82): NCHW in, NCHW out."""
        ch = self._chunks(x.shape[0], x.shape[2] * x.shape[3])
        if len(ch) == 1:
            return self._encode_pass(x, quant_conv)
        return torch.cat([self._encode_pass(x[a:b], quant_conv) for a, b in ch], 0)

    def _encode_pass(self, x, quant_conv=True):
        self.refresh_weights()
        enc, w = self.vq.encoder, self._w
        pool = self._pool(x.device, ("enc",) + tuple(x.shape))
        h = self._to_nhwc(pool, x)
        h = self._step(pool, h, lambda p, t: self._conv_plain(p, w["encoder.conv_in"], t))
        for i in range(enc.num_resolutions):
            lvl = enc.down[i]
            for j in range(enc.num_res_blocks):
                h = self._step(pool, h, self._resnet, f"encoder.down.{i}.block.{j}", lvl.block[j])
                if len(lvl.attn) > 0:
                    h = self._step(pool, h, self._attn, f"encoder.down.{i}.attn.{j}", lvl.attn[j])
            if i != enc.num_resolutions - 1:
                h = self._step(pool, h, self._downsample, f"encoder.down.{i}.downsample", lvl.downsample)
        h = self._mid(pool, "encoder.mid", enc.mid, h)
        y = self._head(pool, h, enc.norm_out, w["encoder.conv_out"])
        if quant_conv:
            y = self._step(pool, y, lambda p, t: self._conv_plain(p, w["quant_conv"], t))
        B, H, W, Cz = y.shape
        out = torch.empty((B, Cz, H, W), dtype=torch.float32, device=x.device)
        self.be.nhwc_to_nchw(y, out)
        pool.put(y)
        return out

    @torch.no_grad()
    def quantize(self, z_nhwc, pool):
        cb = self.vq.quantize.embedding.weight.detach()
        zq = pool.get(z_nhwc.shape)
        idx = pool.get(z_nhwc.shape[:3], torch.int64)
        self.be.vq_nearest(z_nhwc, cb, zq, idx)
        return zq, idx

    @torch.no_grad()
    def decode(self, z, quant_conv_first=False, return_indices=False):
        """[quant_conv ->] quantize -> post_quant_conv -> decoder   (LatentBrownianBridgeModel.py:84-100)."""
        f = 2 ** (self.vq.decoder.num_resolutions - 1)
        ch = self._chunks(z.shape[0], z.shape[2] * z.shape[3] * f * f)
        if len(ch) == 1:
            return self._decode_pass(z, quant_conv_first, return_indices)
        outs = [self._decode_pass(z[a:b], quant_conv_first, return_indices) for a, b in ch]
        if return_indices:
            return torch.cat([o[0] for o in outs], 0), torch.cat([o[1] for o in outs], 0)
        return torch.cat(outs, 0)

    def _decode_pass(self, z, quant_conv_first=False, return_indices=False):
        self.refresh_weights()
        dec, w = self.vq.decoder, self._w
        pool = self._pool(z.device, ("dec",) + tuple(z.shape))
        h = self._to_nhwc(pool, z)
        if quant_conv_first:
            h = self._step(pool, h, lambda p, t: self._conv_plain(p, w["quant_conv"], t))
        zq, idx = self.quantize(h, pool)
        pool.put(h)
        indices = idx.clone() if return_indices else None
        pool.put(idx)
        h = self._step(pool, zq, lambda p, t: self._conv_plain(p, w["post_quant_conv"], t))
        h = self._step(pool, h, lambda p, t: self._conv_plain(p, w["decoder.conv_in"], t))
        h = self._mid(pool, "decoder.mid", dec.mid, h)
        for i in reversed(range(dec.num_resolutions)):
            lvl = dec.up[i]
            for j in range(dec.num_res_blocks + 1):
                h = self._step(pool, h, self._resnet, f"decoder.up.{i}.block.{j}", lvl.block[j])
                if len(lvl.attn) > 0:
                    h = self._step(pool, h, self._attn, f"decoder.up.{i}.attn.{j}", lvl.attn[j])
            if i != 0:
                ent = w[f"decoder.up.{i}.upsample.conv"] if lvl.upsample.with_conv else None
                h = self._step(pool, h, lambda p, t: self._upsample(p, t, ent))
        ent = w["decoder.conv_out"]
        B, H, W, _ = h.shape
        out = torch.empty((B, ent["cout"], H, W), dtype=torch.float32, device=z.device)
        self._head(pool, h, dec.norm_out, ent, out)
        return (out, indices) if return_indices else out
