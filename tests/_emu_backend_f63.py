"""TEST-ONLY: the oracle-backed emulation backend (tests/_emu_backend.py) with CudaBackend's Winograd F(6x6,3x3) forms
as well -- the wino_* methods' tile argument and the phase-stacked nearest-2x output form (up2_phases).  The base
class keeps CudaBackend's F(4,3) signatures unchanged (the pinned launch traces bind every argument)."""
import torch
import torch.nn.functional as F

from _emu_backend import EmuBackend
from oracle import bbdm_oracle as O

# F(6x6,3x3), interpolation points 0, +-1, +-2, +-1/2: the matrices the kernels apply
BT8 = torch.tensor([[1, 0, -5.25, 0, 5.25, 0, -1, 0], [0, 1, 1, -4.25, -4.25, 1, 1, 0],
                    [0, -1, 1, 4.25, -4.25, -1, 1, 0], [0, 0.5, 0.25, -2.5, -1.25, 2, 1, 0],
                    [0, -0.5, 0.25, 2.5, -1.25, -2, 1, 0], [0, 2, 4, -2.5, -5, 0.5, 1, 0],
                    [0, -2, 4, 2.5, -5, -0.5, 1, 0], [0, -1, 0, 5.25, 0, -5.25, 0, 1]], dtype=torch.float64)
G8 = torch.tensor([[1, 0, 0], [-2 / 9, -2 / 9, -2 / 9], [-2 / 9, 2 / 9, -2 / 9], [1 / 90, 1 / 45, 2 / 45],
                   [1 / 90, -1 / 45, 2 / 45], [32 / 45, 16 / 45, 8 / 45], [32 / 45, -16 / 45, 8 / 45], [0, 0, 1]],
                  dtype=torch.float64)
AT8 = torch.tensor([[1, 1, 1, 1, 1, 1, 1, 0], [0, 1, -1, 2, -2, 0.5, -0.5, 0], [0, 1, 1, 4, 4, 0.25, 0.25, 0],
                    [0, 1, -1, 8, -8, 0.125, -0.125, 0], [0, 1, 1, 16, 16, 0.0625, 0.0625, 0],
                    [0, 1, -1, 32, -32, 0.03125, -0.03125, 1]], dtype=torch.float64)


class EmuBackendF63(EmuBackend):
    wino_tiles = (4, 6)

    def wino_geometry(self, B, H, W, tile=4):
        if tile == 4:
            return super().wino_geometry(B, H, W)
        th, tw = -(-H // 6), -(-W // 6)
        return th, tw, max(128, -(-B * th * tw // 16) * 16), True

    def wino_input(self, src1, src2, *, groups=32, mean=None, rstd=None, gamma=None, beta=None, film_scale=None,
                   film_shift=None, film_stride=0, silu=True, v_hi, v_lo, raw_hi=None, raw_lo=None, act_hi=None,
                   act_lo=None, tile=4):
        kw = dict(groups=groups, mean=mean, rstd=rstd, gamma=gamma, beta=beta, film_scale=film_scale,
                  film_shift=film_shift, film_stride=film_stride, silu=silu, v_hi=v_hi, v_lo=v_lo, raw_hi=raw_hi,
                  raw_lo=raw_lo, act_hi=act_hi, act_lo=act_lo)
        if tile == 4:
            return super().wino_input(src1, src2, **kw)
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
        th, tw = -(-H // 6), -(-W // 6)
        pad = (1, 6 * tw + 1 - W, 1, 6 * th + 1 - H)                 # edge tiles read zeros past H, W
        t = F.pad(a.permute(0, 3, 1, 2).double(), pad).unfold(2, 8, 6).unfold(3, 8, 6)     # [B,C,th,tw,8,8]
        V = torch.einsum("ij,bcxyjk,lk->ilbxyc", BT8, t, BT8).reshape(64, B * th * tw, C)
        V = F.pad(V, (0, 0, 0, v_hi.shape[1] - V.shape[1]))           # zero rows up to tiles_total
        self._write_split_f16(V, v_hi, v_lo)
        if raw_hi is not None:
            self._write_split(x, raw_hi, raw_lo)

    def wino_pack_weight(self, w, u_hi, u_lo, dgrad=False, inv_wscale=None, tile=4):
        if tile == 4:
            return super().wino_pack_weight(w, u_hi, u_lo, dgrad=dgrad, inv_wscale=inv_wscale)
        self.calls.append("wino_pack_weight")
        s = 256.0 if inv_wscale is None else self._wino_wscale(w)
        if inv_wscale is not None:
            inv_wscale.fill_(1.0 / s)
        if dgrad:
            w = w.flip(2, 3).transpose(0, 1)
        U = torch.einsum("ij,kcjl,ml->imkc", G8, w.double(), G8) * s                       # [8,8,Cout,Cin]
        self._write_split_f16(U.reshape(u_hi.shape), u_hi, u_lo)

    def wino_output(self, m, *, B, H, W, Cout, bias=None, residual=None, res_mode=0, out, stats_partial=None,
                    inv_wscale=None, tile=4, up2_phases=False):
        """up2_phases: m holds 4*Cout phase-major channels on the HxW tile grid; out is [B, 2H, 2W, Cout]."""
        if tile == 4:
            assert not up2_phases
            return super().wino_output(m, B=B, H=H, W=W, Cout=Cout, bias=bias, residual=residual, res_mode=res_mode,
                                       out=out, stats_partial=stats_partial, inv_wscale=inv_wscale)
        self.calls.append("wino_output")
        th, tw = -(-H // 6), -(-W // 6)
        ncols = 4 * Cout if up2_phases else Cout
        M = m[:, :B * th * tw]
        assert not torch.isnan(M).any()
        M = M.double().reshape(8, 8, B, th, tw, ncols)
        inv = 1.0 / 256.0 if inv_wscale is None else float(inv_wscale)
        Y = torch.einsum("ij,jlbxyc,ml->bxiymc", AT8, M, AT8) * inv                       # [B,th,6,tw,6,ncols]
        o = Y.reshape(B, 6 * th, 6 * tw, ncols)[:, :H, :W].float()
        rows = th
        if up2_phases:
            assert res_mode == 0
            y = o
            o = torch.empty(B, 2 * H, 2 * W, Cout)
            for ph in range(4):
                o[:, ph >> 1::2, ph & 1::2] = y[..., ph * Cout:(ph + 1) * Cout]
            H, W, rows = 2 * H, 2 * W, 4 * th                 # the output map; partial-sum rows per image
        if bias is not None:
            o = o + bias
        if res_mode == 1:
            o = o + residual.reshape(B, H, W, Cout)
        elif res_mode == 2:
            o = o + O.op_resample(residual.reshape(B, H // 2, W // 2, Cout), 1)
        elif res_mode == 3:
            o = o + O.op_resample(residual.reshape(B, H * 2, W * 2, Cout), 2)
        if stats_partial is not None:
            # same contract as the kernel: rows of per-channel (sum, sum sq); here all in row 0
            assert stats_partial.shape[0] == B * rows
            sp = stats_partial.view(B, rows, Cout, 2)
            sp.zero_()
            sp[:, 0, :, 0] = o.reshape(B, -1, Cout).sum(1)
            sp[:, 0, :, 1] = (o.reshape(B, -1, Cout) ** 2).sum(1)
        out.copy_(o)
