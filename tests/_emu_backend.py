"""TEST-ONLY emulation of cabi.CudaBackend on CPU tensors, built on the oracle's per-kernel
restatements.  It lets the not-gpu suite verify the engine's host logic (block wiring, FiLM
offsets, concat order, skip/residual modes, buffer lifetimes) without a GPU.  It lives under
tests/ and is never imported by the product."""
import math

import torch
import torch.nn.functional as F

from oracle import bbdm_oracle as O


class EmuBackend:
    name = "oracle-emulation (tests only)"
    requires_cuda = False
    wino_tensor_scale = True          # as CudaBackend: per-tensor Winograd weight scales

    def __init__(self):
        self.calls = []

    def empty(self, shape, dtype, device):
        # poison so that reading an unwritten / prematurely recycled buffer shows up as NaN
        t = torch.empty(shape, dtype=dtype, device="cpu")
        if dtype.is_floating_point:
            t.fill_(float("nan"))
        return t

    def _planes(self, hi, lo):
        return hi.float() + lo.float()

    def _write_split(self, x, hi, lo):
        h, l = O.bf16_split(x.float())
        hi.copy_(h.to(torch.bfloat16))
        lo.copy_(l.to(torch.bfloat16))
        assert not torch.isnan(hi.float()).any()

    # -- bridge ----------------------------------------------------------------------------------
    def q_sample(self, x0, y, noise, t, m_t, var_t, objective, xt_out, obj_out):
        self.calls.append("q_sample")
        xt, obj = O.q_sample({"m_t": m_t, "variance_t": var_t}, x0, y, t, noise, objective)
        xt_out.copy_(xt)
        obj_out.copy_(obj)

    def p_sample(self, x_t, y, eps, noise, coef, objective, clip, is_last, x_out, x0_out):
        self.calls.append("p_sample")
        m_t, om_t, sq, m_nt, om_nt, c_xt, sigma = [torch.tensor(float(v), dtype=torch.float32) for v in coef]
        if objective == "grad":
            x0 = x_t - eps
        elif objective == "noise":
            x0 = (x_t - m_t * y - sq * eps) / om_t
        else:
            x0 = y - eps
        if clip:
            x0 = x0.clamp(-1.0, 1.0)
        if x0_out is not None:
            x0_out.copy_(x0)
        if is_last:
            x_out.copy_(x0)
        else:
            mean = om_nt * x0 + m_nt * y + c_xt * (x_t - om_t * x0 - m_t * y)
            x_out.copy_(mean + sigma * noise)

    # -- layout / dense ----------------------------------------------------------------------------
    def nchw_to_nhwc_cat(self, x, ctx, out):
        self.calls.append("nchw_to_nhwc_cat")
        z = x if ctx is None else torch.cat([x, ctx], dim=1)
        out.copy_(z.permute(0, 2, 3, 1))

    def nhwc_to_nchw(self, src, out):
        self.calls.append("nhwc_to_nchw")
        assert not torch.isnan(src).any()
        out.copy_(src.permute(0, 3, 1, 2))

    def gather_rows(self, table, idx, out):
        self.calls.append("gather_rows")
        out.copy_(table[idx])

    def linear(self, x, w, bias, out, act_in=False, act_out=False):
        self.calls.append("linear")
        z = F.silu(x) if act_in else x
        z = F.linear(z, w, bias)
        out.copy_(F.silu(z) if act_out else z)

    # -- group norm / prep ---------------------------------------------------------------------------
    def gn_stats(self, src1, src2, groups, eps, mean, rstd, workspace):
        self.calls.append("gn_stats")
        x = src1 if src2 is None else torch.cat([src1, src2], dim=3)
        assert not torch.isnan(x).any()
        m, r = O.op_gn_stats(x, groups, eps)
        mean.copy_(m)
        rstd.copy_(r)

    def prep(self, src1, src2, *, groups=32, mean=None, rstd=None, gamma=None, beta=None,
             film_scale=None, film_shift=None, film_stride=0, silu=True, resample=0,
             act_f32=None, act_hi=None, act_lo=None, raw_f32=None, raw_hi=None, raw_lo=None):
        self.calls.append("prep")
        x = src1 if src2 is None else torch.cat([src1, src2], dim=3)
        assert not torch.isnan(x).any()
        if mean is not None:
            a = O.op_gn_act(x, mean, rstd, gamma, beta, film_scale, film_shift, silu, resample)
            if act_f32 is not None:
                act_f32.copy_(a)
            if act_hi is not None:
                self._write_split(a, act_hi, act_lo)
        if raw_f32 is not None or raw_hi is not None:
            r = O.op_resample(x, resample)
            if raw_f32 is not None:
                raw_f32.copy_(r)
            if raw_hi is not None:
                self._write_split(r, raw_hi, raw_lo)

    # -- convolutions ----------------------------------------------------------------------------------
    def pack_weight_split(self, w, hi, lo):
        self.calls.append("pack_weight_split")
        cout, cin, k = w.shape[0], w.shape[1], w.shape[2]
        self._write_split(w.permute(2, 3, 0, 1).reshape(k * k, cout, cin), hi[:, :cout], lo[:, :cout])

    def pack_weight_f32(self, w, out):
        self.calls.append("pack_weight_f32")
        cout, cin, k = w.shape[0], w.shape[1], w.shape[2]
        out.copy_(w.permute(2, 3, 1, 0).reshape(k * k, cin, cout))

    @staticmethod
    def _oihw_from_split(hi, lo, taps):
        k = 3 if taps == 9 else 1
        w = hi.float() + lo.float()                      # [taps, Cout, Cin]
        return w.reshape(k, k, w.shape[1], w.shape[2]).permute(2, 3, 0, 1).contiguous()

    def conv_umma(self, *, B, H, W, Cin, Cout, taps, a_hi, a_lo, w_hi, w_lo, bias=None, Cin2=0,
                  a2_hi=None, a2_lo=None, w2_hi=None, w2_lo=None, bias2=None, residual=None,
                  res_mode=0, out=None, out_hi=None, out_lo=None, passes=3, out_nchw_channels=0,
                  stats_partial=None, upsample2x=False, weights_per_image=False, operand_f16=False):
        self.calls.append("conv_umma")
        if weights_per_image:
            # B independent GEMMs: image b [H*W, Cin] x matrix b [Cout, Cin]^T
            assert taps == 1 and Cin2 == 0 and H * W >= 128 and operand_f16 == (a_hi.dtype == torch.float16)
            a = self._planes(a_hi, a_lo).reshape(B, H * W, Cin)
            w = self._planes(w_hi, w_lo).reshape(B, Cout, Cin)
            assert not torch.isnan(a).any() and not torch.isnan(w).any()
            out.copy_(torch.bmm(a, w.transpose(1, 2)).reshape(out.shape))
            return
        if upsample2x:
            return self._conv_up2(B, H, W, Cin, Cout, a_hi, a_lo, w_hi, w_lo, bias, residual, res_mode, out,
                                  stats_partial)
        assert Cin % 64 == 0 and Cout % 64 == 0 and Cin2 % 64 == 0 and W >= 4
        a = self._planes(a_hi, a_lo).reshape(B, H, W, Cin)
        assert not torch.isnan(a).any()
        if taps == 4:
            # 2x2 window at rows/cols (0..1), zero padding bottom/right
            w4 = (w_hi.float() + w_lo.float()).reshape(2, 2, Cout, Cin).permute(2, 3, 0, 1)
            o = F.conv2d(F.pad(a.permute(0, 3, 1, 2), (0, 1, 0, 1)), w4, bias).permute(0, 2, 3, 1)
        else:
            o = O.op_conv_nhwc(a, self._oihw_from_split(w_hi, w_lo, taps), bias)
        if Cin2:
            a2 = self._planes(a2_hi, a2_lo).reshape(B, H, W, Cin2)
            o = o + O.op_conv_nhwc(a2, self._oihw_from_split(w2_hi, w2_lo, 1), bias2)
        if res_mode == 1:
            o = o + residual.reshape(B, H, W, Cout)
        elif res_mode == 2:
            o = o + O.op_resample(residual.reshape(B, H // 2, W // 2, Cout), 1)
        elif res_mode == 3:
            o = o + O.op_resample(residual.reshape(B, H * 2, W * 2, Cout), 2)
        if stats_partial is not None:
            # same contract as the kernel: rows of per-channel (sum, sum sq); here all in row 0
            rows = stats_partial.shape[0] // B
            assert rows == self.conv_geometry(H, W)[3] and rows > 0
            sp = stats_partial.view(B, rows, Cout, 2)
            sp.zero_()
            sp[:, 0, :, 0] = o.reshape(B, -1, Cout).sum(1)
            sp[:, 0, :, 1] = (o.reshape(B, -1, Cout) ** 2).sum(1)
        if out_nchw_channels:
            out.copy_(o[..., :out_nchw_channels].permute(0, 3, 1, 2))
        elif out is not None:
            out.copy_(o.reshape(out.shape))
        if out_hi is not None:
            self._write_split(o.reshape(out_hi.shape), out_hi, out_lo)

    def _conv_up2(self, B, H, W, Cin, Cout, a_hi, a_lo, w_hi, w_lo, bias, residual, res_mode, out, stats_partial):
        """The kernel's phase formulation, literally: 4 phases x 2x2 taps on the low-res input."""
        a = self._planes(a_hi, a_lo).reshape(B, H, W, Cin)
        w = (w_hi.float() + w_lo.float())                     # [16, Cout, Cin]
        ap = F.pad(a, (0, 0, 1, 1, 1, 1))                     # zero pad H and W by 1
        o = torch.zeros(B, 2 * H, 2 * W, Cout)
        for ph in range(4):
            pa, pb = ph >> 1, ph & 1
            acc = torch.zeros(B, H, W, Cout)
            for t in range(4):
                r, c = t >> 1, t & 1
                dy = r if pa else r - 1
                dx = c if pb else c - 1
                src = ap[:, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W, :]
                acc = acc + src @ w[ph * 4 + t].T
            o[:, pa::2, pb::2, :] = acc
        if bias is not None:
            o = o + bias
        if res_mode == 1:
            o = o + residual.reshape(B, 2 * H, 2 * W, Cout)
        elif res_mode == 2:
            o = o + O.op_resample(residual.reshape(B, H, W, Cout), 1)
        if stats_partial is not None:
            rows = stats_partial.shape[0] // B
            assert rows == 4 * self.conv_geometry(H, W)[3] and rows > 0
            sp = stats_partial.view(B, rows, Cout, 2)
            sp.zero_()
            sp[:, 0, :, 0] = o.reshape(B, -1, Cout).sum(1)
            sp[:, 0, :, 1] = (o.reshape(B, -1, Cout) ** 2).sum(1)
        out.copy_(o)

    # -- Winograd F(4x4,3x3): the kernels' transform formulation, literally ---------------------------------
    _BT = torch.tensor([[4, 0, -5, 0, 1, 0], [0, -4, -4, 1, 1, 0], [0, 4, -4, -1, 1, 0],
                        [0, -2, -1, 2, 1, 0], [0, 2, -1, -2, 1, 0], [0, 4, 0, -5, 0, 1]], dtype=torch.float64)
    _G = torch.tensor([[1 / 4, 0, 0], [-1 / 6, -1 / 6, -1 / 6], [-1 / 6, 1 / 6, -1 / 6],
                       [1 / 24, 1 / 12, 1 / 6], [1 / 24, -1 / 12, 1 / 6], [0, 0, 1]], dtype=torch.float64)
    _AT = torch.tensor([[1, 1, 1, 1, 1, 0], [0, 1, -1, 2, -2, 0], [0, 1, 1, 4, 4, 0], [0, 1, -1, 8, -8, 1]],
                       dtype=torch.float64)

    def wino_geometry(self, B, H, W):
        th, tw = H // 4, W // 4
        tot = B * th * tw
        return th, tw, tot, (H % 4 == 0 and W % 4 == 0 and tot % 16 == 0 and tot >= 128)

    def _write_split_f16(self, x, hi, lo):
        h = x.float().to(torch.float16)
        hi.copy_(h)
        lo.copy_((x.float() - h.float()).to(torch.float16))

    def wino_input(self, src1, src2, *, groups=32, mean=None, rstd=None, gamma=None, beta=None, film_scale=None,
                   film_shift=None, film_stride=0, silu=True, v_hi, v_lo, raw_hi=None, raw_lo=None, act_hi=None,
                   act_lo=None):
        self.calls.append("wino_input")
        x = src1 if src2 is None else torch.cat([src1, src2], dim=3)
        assert not torch.isnan(x).any()
        B, H, W, C = x.shape
        if mean is None:
            assert not silu and film_scale is None
            a = x.float()
        else:
            a = O.op_gn_act(x, mean, rstd, gamma, beta, film_scale, film_shift, silu, 0)    # [B,H,W,C]
        if act_hi is not None:
            self._write_split(a, act_hi, act_lo)
        t = F.pad(a.permute(0, 3, 1, 2).double(), (1, 1, 1, 1)).unfold(2, 6, 4).unfold(3, 6, 4)   # [B,C,th,tw,6,6]
        V = torch.einsum("ij,bcxyjk,lk->ilbxyc", self._BT, t, self._BT)                      # [6,6,B,th,tw,C]
        self._write_split_f16(V.reshape(v_hi.shape), v_hi, v_lo)
        if raw_hi is not None:
            self._write_split(x, raw_hi, raw_lo)

    @staticmethod
    def _wino_wscale(w):
        """The kernel's per-tensor power of two: 2^(14 - ceil(log2 max|w|)), exponent clamped to +-100; 2^8 for 0."""
        m = float(w.abs().max())
        if m == 0.0:
            return 256.0
        f, e = math.frexp(m)                                   # m = f * 2^e, f in [0.5, 1)
        return 2.0 ** min(max(14 - (e - 1 if f == 0.5 else e), -100), 100)

    def wino_pack_weight(self, w, u_hi, u_lo, dgrad=False, inv_wscale=None):
        self.calls.append("wino_pack_weight")
        s = 256.0 if inv_wscale is None else self._wino_wscale(w)
        if inv_wscale is not None:
            inv_wscale.fill_(1.0 / s)
        if dgrad:
            w = w.flip(2, 3).transpose(0, 1)
        U = torch.einsum("ij,kcjl,ml->imkc", self._G, w.double(), self._G) * s               # [6,6,Cout,Cin]
        self._write_split_f16(U.reshape(u_hi.shape), u_hi, u_lo)

    def wino_output(self, m, *, B, H, W, Cout, bias=None, residual=None, res_mode=0, out, stats_partial=None,
                    inv_wscale=None):
        self.calls.append("wino_output")
        assert not torch.isnan(m).any()
        th, tw = H // 4, W // 4
        M = m.double().reshape(6, 6, B, th, tw, Cout)
        inv = 1.0 / 256.0 if inv_wscale is None else float(inv_wscale)
        Y = torch.einsum("ij,jlbxyc,ml->bxiymc", self._AT, M, self._AT) * inv               # [B,th,4,tw,4,Cout]
        o = Y.reshape(B, H, W, Cout).float()
        if bias is not None:
            o = o + bias
        if res_mode == 1:
            o = o + residual.reshape(B, H, W, Cout)
        elif res_mode == 2:
            o = o + O.op_resample(residual.reshape(B, H // 2, W // 2, Cout), 1)
        elif res_mode == 3:
            o = o + O.op_resample(residual.reshape(B, H * 2, W * 2, Cout), 2)
        if stats_partial is not None:
            assert stats_partial.shape[0] == B * th
            sp = stats_partial.view(B, th, Cout, 2)
            sp.zero_()
            sp[:, 0, :, 0] = o.reshape(B, -1, Cout).sum(1)
            sp[:, 0, :, 1] = (o.reshape(B, -1, Cout) ** 2).sum(1)
        out.copy_(o)

    # -- SpatialTransformer pieces ------------------------------------------------------------------------------
    def layernorm_split(self, x, gamma, beta, eps, out_f32=None, out_hi=None, out_lo=None):
        self.calls.append("layernorm_split")
        assert not torch.isnan(x).any()
        y = F.layer_norm(x, (x.shape[-1],), gamma, beta, eps)
        if out_f32 is not None:
            out_f32.copy_(y.reshape(out_f32.shape))
        if out_hi is not None:
            self._write_split(y.reshape(out_hi.shape), out_hi, out_lo)

    def geglu_split(self, u, out_f32=None, out_hi=None, out_lo=None):
        self.calls.append("geglu_split")
        assert not torch.isnan(u).any()
        a, g = u.chunk(2, dim=-1)
        y = a * F.gelu(g)
        if out_f32 is not None:
            out_f32.copy_(y.reshape(out_f32.shape))
        if out_hi is not None:
            self._write_split(y.reshape(out_hi.shape), out_hi, out_lo)

    def attention_cross(self, q_hi, q_lo, kv_hi, kv_lo, heads, out_f32=None, out_hi=None, out_lo=None):
        self.calls.append("attention_cross")
        q, kv = self._planes(q_hi, q_lo), self._planes(kv_hi, kv_lo)
        assert not torch.isnan(q).any() and not torch.isnan(kv).any()
        B, Tq, Cc = q.shape
        d = Cc // heads
        k, v = kv[..., :Cc], kv[..., Cc:]
        sp = lambda t: t.reshape(B, t.shape[1], heads, d).permute(0, 2, 1, 3)
        w = torch.softmax(torch.einsum("bhid,bhjd->bhij", sp(q), sp(k)) * d ** -0.5, dim=-1)
        o = torch.einsum("bhij,bhjd->bhid", w, sp(v)).permute(0, 2, 1, 3).reshape(B, Tq, Cc)
        if out_f32 is not None:
            out_f32.copy_(o)
        if out_hi is not None:
            self._write_split(o, out_hi, out_lo)

    def denorm_to_uint8(self, images, to_normal, out):
        self.calls.append("denorm_to_uint8")
        x = images.detach().clone()
        if to_normal:
            x = x.mul_(0.5).add_(0.5).clamp_(0, 1.)
        out.copy_(x.mul_(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 1).to(torch.uint8))

    def spatial_rescale(self, src, n_stages, weight, bias, out):
        self.calls.append("spatial_rescale")
        x = src.detach()
        for _ in range(n_stages):
            h2, w2 = x.shape[2] // 2, x.shape[3] // 2
            a, b = x[:, :, 0:2 * h2:2, 0:2 * w2:2], x[:, :, 0:2 * h2:2, 1:2 * w2:2]
            c, d = x[:, :, 1:2 * h2:2, 0:2 * w2:2], x[:, :, 1:2 * h2:2, 1:2 * w2:2]
            x = 0.5 * (0.5 * a + 0.5 * b) + 0.5 * (0.5 * c + 0.5 * d)
        if weight is not None:
            x = torch.einsum("oc,bchw->bohw", weight.detach(), x)
            if bias is not None:
                x = x + bias.detach().view(1, -1, 1, 1)
        out.copy_(x)

    # -- multi-tensor optimizer / EMA (flat state buffers) ----------------------------------------------------
    def optim_chunk_elems(self):
        return 4096

    def adam_multi(self, tab, exp_avg, exp_avg_sq, *, lr, beta1, beta2, eps, weight_decay, step, ema_shadow=None,
                   ema_decay=0.0):
        self.calls.append("adam_multi")
        bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
        for p, m, v, s in zip(tab.tensors, tab.views(exp_avg), tab.views(exp_avg_sq),
                              tab.views(ema_shadow) if ema_shadow is not None else [None] * len(tab.tensors)):
            if p.grad is None:
                continue
            g = p.grad + weight_decay * p.data if weight_decay else p.grad
            m.lerp_(g, 1.0 - beta1)
            v.mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
            denom = (v.sqrt() / (bc2 ** 0.5)).add_(eps)
            p.data.addcdiv_(m, denom, value=-(lr / bc1))
            if s is not None:
                s.copy_((1.0 - ema_decay) * p.data + ema_decay * s)

    def ema_multi(self, tab, shadow, decay, with_decay=True):
        self.calls.append("ema_multi")
        for p, s in zip(tab.tensors, tab.views(shadow)):
            s.copy_((1.0 - decay) * p.data + decay * s if with_decay else p.data)

    def pack_weight_split_taps(self, w, hi, lo):
        self.calls.append("pack_weight_split_taps")
        self._write_split(w.permute(2, 0, 1), hi, lo)

    def conv_geometry(self, H, W):
        p2f = lambda x: 1 << (x.bit_length() - 1)
        p2c = lambda x: 1 << (x - 1).bit_length()
        tw = min(16, p2f(W))
        th = min(128 // tw, p2c(H))
        tb = 128 // (tw * th)
        rows = 4 * (-(-W // tw)) * (-(-H // th)) if tb == 1 else 0
        return tw, th, tb, rows

    def gn_finalize_partials(self, part1, rows1, part2, rows2, B, hw, groups, eps, mean, rstd):
        self.calls.append("gn_finalize_partials")
        ch = [part1.view(B, rows1, -1, 2).double().sum(1)]
        if part2 is not None:
            ch.append(part2.view(B, rows2, -1, 2).double().sum(1))
        s = torch.cat(ch, dim=1)                               # [B, C, 2]
        assert not torch.isnan(s).any()
        C = s.shape[1]
        sg = s.view(B, groups, C // groups, 2).sum(2)
        n = hw * (C // groups)
        m = sg[..., 0] / n
        var = (sg[..., 1] / n - m * m).clamp_min(0)
        mean.copy_(m.float())
        rstd.copy_((1.0 / torch.sqrt(var + eps)).float())

    def conv_direct(self, src, w_packed, bias, residual, out, Cout, k, stride=1):
        self.calls.append("conv_direct")
        assert not torch.isnan(src).any()
        cin = src.shape[3]
        w = w_packed.reshape(k, k, cin, Cout).permute(3, 2, 0, 1)
        o = F.conv2d(src.permute(0, 3, 1, 2), w, bias, stride=stride, padding=k // 2).permute(0, 2, 3, 1)
        if residual is not None:
            o = o + residual
        out.copy_(o)

    def conv_stem(self, src, w_packed, bias, out, Cout, stats_partial=None):
        self.calls.append("conv_stem")
        B, H, W, cin = src.shape
        assert W % 32 == 0 and cin <= 16 and Cout % 32 == 0 and Cout <= 128
        w = w_packed.reshape(3, 3, cin, Cout).permute(3, 2, 0, 1)
        o = F.conv2d(src.permute(0, 3, 1, 2), w, bias, padding=1).permute(0, 2, 3, 1)
        out.copy_(o)
        if stats_partial is not None:
            sp = stats_partial.view(B, H, Cout, 2)
            sp[..., 0] = o.sum(2)
            sp[..., 1] = (o * o).sum(2)

    # -- attention ----------------------------------------------------------------------------------------
    def attention(self, qkv, heads, order, out_f32=None, out_hi=None, out_lo=None):
        self.calls.append("attention")
        o = O.op_attention_nhwc(qkv, heads, bool(order))
        if out_f32 is not None:
            out_f32.copy_(o)
        if out_hi is not None:
            self._write_split(o, out_hi, out_lo)

    def attention_split(self, qkv_hi, qkv_lo, heads, order, out_f32=None, out_hi=None, out_lo=None):
        self.calls.append("attention_split")
        self.attention(self._planes(qkv_hi, qkv_lo), heads, order, out_f32, out_hi, out_lo)

    def attention_tc(self, qkv_hi, qkv_lo, heads, order, out_f32=None, out_hi=None, out_lo=None):
        self.calls.append("attention_tc")
        assert qkv_hi.shape[2] // 3 // heads == 64
        self.attention(self._planes(qkv_hi, qkv_lo), heads, order, out_f32, out_hi, out_lo)

    # -- VQGAN ends ---------------------------------------------------------------------------------------
    def conv_direct_pad(self, src, w_packed, bias, residual, out, cout, k, stride, pad_lo, pad_hi):
        self.calls.append("conv_direct_pad")
        assert not torch.isnan(src).any()
        cin = src.shape[3]
        w = w_packed.reshape(k, k, cin, cout).permute(3, 2, 0, 1)
        x = F.pad(src.permute(0, 3, 1, 2), (pad_lo, pad_hi, pad_lo, pad_hi))
        o = F.conv2d(x, w, bias, stride=stride, padding=0).permute(0, 2, 3, 1)
        out.copy_(o if residual is None else o + residual)

    def softmax_rows_split(self, src, scale, out_hi, out_lo):
        self.calls.append("softmax_rows_split")
        assert not torch.isnan(src).any()
        self._write_split(torch.softmax(src.reshape(out_hi.shape) * scale, dim=-1), out_hi, out_lo)

    def s2d_split(self, src, out_hi, out_lo):
        self.calls.append("s2d_split")
        B, H, W, Cc = src.shape
        x = src.reshape(B, H // 2, 2, W // 2, 2, Cc).permute(0, 1, 3, 2, 4, 5).reshape(B, H // 2, W // 2, 4 * Cc)
        self._write_split(x, out_hi, out_lo)

    def vq_nearest(self, z, codebook, z_q, indices):
        self.calls.append("vq_nearest")
        flat = z.reshape(-1, codebook.shape[1])
        d = torch.sum(flat ** 2, dim=1, keepdim=True) + torch.sum(codebook ** 2, dim=1) - 2 * flat @ codebook.t()
        idx = torch.argmin(d, dim=1)
        z_q.copy_((flat + (codebook[idx] - flat)).reshape(z_q.shape))
        indices.copy_(idx.reshape(indices.shape))

    def split_grad(self, src, hi, lo, hi_t, lo_t, colsum=None, workspace=None):
        self.calls.append("split_grad")
        s2 = src.float().reshape(-1, src.shape[-1])
        h, l = O.bf16_split(s2)
        for dst, v in ((hi, h), (lo, l), (hi_t, h.t()), (lo_t, l.t())):
            if dst is not None:
                dst.copy_(v.reshape(dst.shape).to(torch.bfloat16))
        if colsum is not None:
            colsum.copy_(s2.double().sum(0).float())

    # -- training gradients (host logic of bbdm_b200/train.py on CPU) ---------------------------------------
    def pack_weight_split_dgrad(self, w, hi, lo):
        self.calls.append("pack_weight_split_dgrad")
        cout, cin, k = w.shape[0], w.shape[1], w.shape[2]
        self._write_split(w.flip(2, 3).permute(2, 3, 1, 0).reshape(k * k, cin, cout), hi, lo)

    def pack_weight_split_both(self, w, f_hi, f_lo, d_hi=None, d_lo=None):
        self.calls.append("pack_weight_split_both")
        if f_hi is not None:
            self.pack_weight_split(w, f_hi, f_lo)
        if d_hi is not None:
            self.pack_weight_split_dgrad(w, d_hi, d_lo)

    def wgrad_workspace(self, B, H, W, Cin, Cout, taps):
        return 1, 1

    @staticmethod
    def _wgrad(a_nhwc, g_nhwc, k):
        w = torch.zeros((g_nhwc.shape[3], a_nhwc.shape[3], k, k), dtype=torch.float64, requires_grad=True)
        with torch.enable_grad():
            F.conv2d(a_nhwc.double().permute(0, 3, 1, 2), w, padding=k // 2).backward(g_nhwc.double().permute(0, 3, 1, 2))
        return w.grad.float()

    def conv_wgrad(self, g_hi_t, g_lo_t, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, workspace):
        self.calls.append("conv_wgrad")
        g = self._planes(g_hi_t, g_lo_t).t().reshape(B, H, W, Cout)
        dw.copy_(self._wgrad(self._planes(a_hi, a_lo).reshape(B, H, W, Cin), g, 3 if taps == 9 else 1))

    def conv_wgrad_direct(self, dy, x, k, dw, workspace):
        self.calls.append("conv_wgrad_direct")
        dw.copy_(self._wgrad(x, dy, k))

    @staticmethod
    def _gn_bwd_terms(x, da, groups, mean, rstd, gamma, beta, fscale, fshift, silu):
        B, H, W, C = x.shape
        m = mean.repeat_interleave(C // groups, dim=1)[:, None, None, :]
        r = rstd.repeat_interleave(C // groups, dim=1)[:, None, None, :]
        xh = (x - m) * r
        f1 = 1.0 if fscale is None else (1.0 + fscale[:, None, None, :C])
        f0 = 0.0 if fscale is None else fshift[:, None, None, :C]
        z = (gamma * xh + beta) * f1 + f0
        if silu:
            sg = torch.sigmoid(z)
            dz = da * sg * (1 + z * (1 - sg))
        else:
            dz = da
        return xh, dz, r, f1

    def gn_bwd_reduce(self, x, da, groups, mean, rstd, gamma, beta, fscale, fshift, fstride, silu, a12, ws):
        self.calls.append("gn_bwd_reduce")
        xh, dz, _, _ = self._gn_bwd_terms(x, da, groups, mean, rstd, gamma, beta, fscale, fshift, silu)
        a12[..., 0] = dz.double().sum((1, 2)).float()
        a12[..., 1] = (dz * xh).double().sum((1, 2)).float()

    def gn_bwd_apply(self, x, da, groups, mean, rstd, gamma, beta, fscale, fshift, fstride, silu, s1, s2, dx):
        self.calls.append("gn_bwd_apply")
        B, H, W, C = x.shape
        xh, dz, r, f1 = self._gn_bwd_terms(x, da, groups, mean, rstd, gamma, beta, fscale, fshift, silu)
        n = H * W * (C // groups)
        e = lambda t: t.repeat_interleave(C // groups, dim=1)[:, None, None, :]
        dx.copy_(r * (dz * gamma * f1 - (e(s1) + xh * e(s2)) / n))

    def attention_bwd(self, qkv, out, dout, heads, order, dqkv, lse, delta):
        self.calls.append("attention_bwd")
        q = qkv.detach().double().requires_grad_(True)
        with torch.enable_grad():
            O.op_attention_nhwc(q, heads, bool(order)).backward(dout.double())
        dqkv.copy_(q.grad.float())

    def check_fault(self):
        pass
