"""TEST-ONLY: the emulation backend (tests/_emu_backend_ragged.py) with CudaBackend's channel multiple of 32
(conv_channel_multiple).  Its conv_umma / conv_wgrad zero-pad every channel count to a multiple of 64 and run the base
emulation, which is what the kernels compute: the TMA zero-fills the K blocks past Cin / Cin2, and the columns past
Cout are computed and not stored.  The base EmuBackend declares no multiple, so the executors keep the 64 rule on it
and its launch traces stay as they are."""
import torch
import torch.nn.functional as F

from _emu_backend_ragged import EmuBackendRagged


def _up64(c):
    return -(-c // 64) * 64


def _pad_last(t, c, cp):
    """[..., c] -> [N, cp], zeros past c."""
    return F.pad(t.reshape(-1, c), (0, cp - c))


def _pad_w(w, cout, cin, coutp, cinp):
    """[taps][Cout][Cin] -> [taps][Coutp][Cinp], zeros past the real channels."""
    return F.pad(w.reshape(-1, cout, cin), (0, cinp - cin, 0, coutp - cout))


class EmuBackendWidths(EmuBackendRagged):
    conv_channel_multiple = 32

    def conv_umma(self, *, B, H, W, Cin, Cout, taps, a_hi, a_lo, w_hi, w_lo, bias=None, Cin2=0, a2_hi=None,
                  a2_lo=None, w2_hi=None, w2_lo=None, bias2=None, residual=None, res_mode=0, out=None, out_hi=None,
                  out_lo=None, passes=3, out_nchw_channels=0, stats_partial=None, upsample2x=False,
                  weights_per_image=False, operand_f16=False, window_origin=0):
        assert Cin % 32 == 0 and Cout % 32 == 0 and Cin2 % 32 == 0
        kw = dict(B=B, H=H, W=W, taps=taps, passes=passes, out_nchw_channels=out_nchw_channels,
                  upsample2x=upsample2x, weights_per_image=weights_per_image, operand_f16=operand_f16,
                  res_mode=res_mode, **({} if not window_origin else dict(window_origin=window_origin)))
        cinp, coutp, cin2p = _up64(Cin), _up64(Cout), _up64(Cin2)
        if (cinp, coutp, cin2p) == (Cin, Cout, Cin2):
            return super().conv_umma(Cin=Cin, Cout=Cout, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo, bias=bias,
                                     Cin2=Cin2, a2_hi=a2_hi, a2_lo=a2_lo, w2_hi=w2_hi, w2_lo=w2_lo, bias2=bias2,
                                     residual=residual, out=out, out_hi=out_hi, out_lo=out_lo,
                                     stats_partial=stats_partial, **kw)
        assert not weights_per_image and (not out_nchw_channels or coutp == Cout)
        pa = lambda t: None if t is None else _pad_last(t, Cin, cinp)
        pw = lambda t: None if t is None else _pad_w(t, Cout, Cin, coutp, cinp)
        if Cin2:
            kw.update(Cin2=cin2p, a2_hi=_pad_last(a2_hi, Cin2, cin2p), a2_lo=_pad_last(a2_lo, Cin2, cin2p),
                      w2_hi=_pad_w(w2_hi, Cout, Cin2, coutp, cin2p), w2_lo=_pad_w(w2_lo, Cout, Cin2, coutp, cin2p),
                      bias2=None if bias2 is None else F.pad(bias2, (0, coutp - Cout)))
        po = pst = ph = pl = None
        if out is not None:
            po = out if out_nchw_channels else torch.empty(out.shape[:-1] + (coutp,))
        if out_hi is not None:
            ph = torch.empty(out_hi.shape[:-1] + (coutp,), dtype=out_hi.dtype)
            pl = torch.empty_like(ph)
        if stats_partial is not None:
            pst = torch.empty((stats_partial.shape[0], coutp, 2))
        super().conv_umma(Cin=cinp, Cout=coutp, a_hi=pa(a_hi), a_lo=pa(a_lo), w_hi=pw(w_hi), w_lo=pw(w_lo),
                          bias=None if bias is None else F.pad(bias, (0, coutp - Cout)),
                          residual=None if residual is None else _pad_last(residual, Cout, coutp),
                          out=po, out_hi=ph, out_lo=pl, stats_partial=pst, **kw)
        if out is not None and not out_nchw_channels:
            out.copy_(po[..., :Cout])
        if out_hi is not None:
            out_hi.copy_(ph[..., :Cout])
            out_lo.copy_(pl[..., :Cout])
        if stats_partial is not None:
            stats_partial.copy_(pst[:, :Cout])

    def conv_wgrad(self, g_hi_t, g_lo_t, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, workspace, window_origin=0):
        assert Cin % 32 == 0 and Cout % 32 == 0
        cinp, coutp = _up64(Cin), _up64(Cout)
        if (cinp, coutp) == (Cin, Cout):
            return super().conv_wgrad(g_hi_t, g_lo_t, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, workspace,
                                      window_origin=window_origin)
        pg = lambda g: F.pad(g, (0, 0, 0, coutp - Cout))
        pa = lambda a: _pad_last(a, Cin, cinp).reshape(B, H, W, cinp)
        pdw = torch.empty((coutp, cinp) + tuple(dw.shape[2:]))
        super().conv_wgrad(pg(g_hi_t), pg(g_lo_t), pa(a_hi), pa(a_lo), B, H, W, cinp, coutp, taps, pdw, workspace,
                           window_origin=window_origin)
        dw.copy_(pdw[:Cout, :Cin])
