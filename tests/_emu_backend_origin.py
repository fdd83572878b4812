"""TEST-ONLY: the F(6,3) emulation backend with the rest of CudaBackend's launch set that the executors reach only on a
backend that offers it: the 2x2 window origin of conv_umma / conv_wgrad (taps 4, window_origin 0 or -1: the UNet's
tensor-core Downsample and the adjoints of the resampling convs), the device-coefficient bridge update of the graphed
sampling step (p_sample_dev) and the capturable Adam step (adam_multi_dev).  The window-origin convs are defined in
fp64 from the definition, independently of bbdm_b200/weights.py."""
import torch
import torch.nn.functional as F

from _emu_backend_f63_pool import EmuBackendF63Pool


def _window_pad(origin):
    """F.pad of an NCHW map for a 2x2 window at rows / cols origin..origin+1 of each output pixel."""
    return (1, 0, 1, 0) if origin == -1 else (0, 1, 0, 1)


class EmuBackendOrigin(EmuBackendF63Pool):
    window_origin = True

    def conv_umma(self, *, B, H, W, Cin, Cout, taps, a_hi, a_lo, w_hi, w_lo, bias=None, Cin2=0, a2_hi=None, a2_lo=None,
                  w2_hi=None, w2_lo=None, bias2=None, residual=None, res_mode=0, out=None, out_hi=None, out_lo=None,
                  passes=3, out_nchw_channels=0, stats_partial=None, upsample2x=False, weights_per_image=False,
                  operand_f16=False, window_origin=0):
        if not window_origin:
            return super().conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=taps, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi,
                                     w_lo=w_lo, bias=bias, Cin2=Cin2, a2_hi=a2_hi, a2_lo=a2_lo, w2_hi=w2_hi,
                                     w2_lo=w2_lo, bias2=bias2, residual=residual, res_mode=res_mode, out=out,
                                     out_hi=out_hi, out_lo=out_lo, passes=passes, out_nchw_channels=out_nchw_channels,
                                     stats_partial=stats_partial, upsample2x=upsample2x,
                                     weights_per_image=weights_per_image, operand_f16=operand_f16)
        self.calls.append("conv_umma")
        assert taps == 4 and window_origin == -1 and not (upsample2x or weights_per_image or Cin2 or res_mode
                                                           or out_nchw_channels)
        a = self._planes(a_hi, a_lo).reshape(B, H, W, Cin).permute(0, 3, 1, 2).double()
        assert not torch.isnan(a).any()
        w4 = (w_hi.double() + w_lo.double()).reshape(2, 2, Cout, Cin).permute(2, 3, 0, 1)
        o = F.conv2d(F.pad(a, _window_pad(window_origin)), w4, None if bias is None else bias.double())
        o = o.permute(0, 2, 3, 1).float()
        if stats_partial is not None:       # the base emulation's contract: all partial sums in row 0 of each image
            sp = stats_partial.view(B, stats_partial.shape[0] // B, Cout, 2)
            sp.zero_()
            sp[:, 0, :, 0] = o.reshape(B, -1, Cout).sum(1)
            sp[:, 0, :, 1] = (o.reshape(B, -1, Cout) ** 2).sum(1)
        if out is not None:
            out.copy_(o.reshape(out.shape))
        if out_hi is not None:
            self._write_split(o.reshape(out_hi.shape), out_hi, out_lo)

    def conv_wgrad(self, g_hi_t, g_lo_t, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, workspace, window_origin=0):
        if taps != 4:
            assert window_origin == 0
            return super().conv_wgrad(g_hi_t, g_lo_t, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, workspace)
        self.calls.append("conv_wgrad")
        g = self._planes(g_hi_t, g_lo_t)[:, :B * H * W].double().reshape(Cout, B, H, W).permute(1, 0, 2, 3)
        a = self._planes(a_hi, a_lo).double().reshape(B, H, W, Cin).permute(0, 3, 1, 2)
        dw.copy_(torch.nn.grad.conv2d_weight(F.pad(a, _window_pad(window_origin)), (Cout, Cin, 2, 2), g))

    def p_sample_dev(self, x_t, y, eps, noise, coef_dev, objective, clip, is_last, x_out, x0_out):
        self.p_sample(x_t, y, eps, noise, coef_dev.tolist(), objective, clip, is_last, x_out, x0_out)
        self.calls[-1] = "p_sample_dev"

    def adam_multi_dev(self, tab, exp_avg, exp_avg_sq, *, step, lr, beta1, beta2, eps, weight_decay, ema_shadow=None,
                       ema_decay=0.0):
        step += 1
        self.adam_multi(tab, exp_avg, exp_avg_sq, lr=float(lr), beta1=beta1, beta2=beta2, eps=eps,
                        weight_decay=weight_decay, step=int(step), ema_shadow=ema_shadow, ema_decay=ema_decay)
        self.calls[-1] = "adam_multi_dev"
