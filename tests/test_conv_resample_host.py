"""Host checks of the resampling-conv formulations the tensor-core path uses (bbdm_b200/weights.py), in fp64 against
torch's own stride-2 conv, nearest-2x + conv and their autograd:

  * the UNet Downsample (3x3, stride 2, padding 1) = a 2x2-tap conv at window origin -1 on the space-to-depth operand;
    its data gradient = the transposed 2x2 conv at origin 0 over dY, then depth-to-space; its weight gradient = the
    origin -1 2x2 weight gradient folded back to 3x3;
  * the Upsample (nearest 2x + 3x3 conv): data gradient = a stride-1 3x3 conv over the space-to-depth of dY; weight
    gradient = the 3x3 weight gradient of (x, space-to-depth(dY)) folded over the phases.
"""
import pytest
import torch
import torch.nn.functional as F

from bbdm_b200 import weights as Wt


def s2d(t):
    """NCHW [B, C, H, W] -> [B, 4C, H/2, W/2], channel (a*2 + b)*C + c = pixel (2i + a, 2j + b) (bbdm_s2d_split)."""
    B, C, H, W = t.shape
    return t.view(B, C, H // 2, 2, W // 2, 2).permute(0, 3, 5, 1, 2, 4).reshape(B, 4 * C, H // 2, W // 2)


def d2s(t, C):
    B, _, h, w = t.shape
    return t.view(B, 2, 2, C, h, w).permute(0, 3, 4, 1, 5, 2).reshape(B, C, 2 * h, 2 * w)


def taps_conv(x, w, pad):
    """x NCHW, w [Cout, Cin, k*k] taps -> the valid conv of the padded x."""
    k = int(round(w.shape[2] ** 0.5))
    return F.conv2d(F.pad(x, pad), w.view(w.shape[0], w.shape[1], k, k))


def weight_grad(x, dy, k, pad):
    """sum_p dY[p] x[p + tap]^T for a k x k window over the padded x -> [Cout, Cin, k, k]."""
    return torch.nn.grad.conv2d_weight(F.pad(x, pad), (dy.shape[1], x.shape[1], k, k), dy)


@pytest.mark.parametrize("B,Cin,Cout,H,W", [(2, 3, 5, 8, 6), (1, 4, 4, 4, 10)])
def test_stride2_conv_as_window_origin_conv(B, Cin, Cout, H, W):
    g = torch.Generator().manual_seed(B * 100 + H)
    x = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64).requires_grad_(True)
    w = torch.randn(Cout, Cin, 3, 3, generator=g, dtype=torch.float64).requires_grad_(True)
    y = F.conv2d(x, w, stride=2, padding=1)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dy)
    xs = s2d(x.detach())
    assert torch.allclose(taps_conv(xs, Wt.stride2_s2d_weights(w.detach()), (1, 0, 1, 0)), y, atol=1e-12)
    dxs = taps_conv(dy, Wt.stride2_dgrad_weights(w.detach()), (0, 1, 0, 1))
    assert torch.allclose(d2s(dxs, Cin), x.grad, atol=1e-12)
    g4 = weight_grad(xs, dy, 2, (1, 0, 1, 0))
    assert torch.allclose(Wt.stride2_fold_wgrad(g4), w.grad, atol=1e-12)


@pytest.mark.parametrize("B,Cin,Cout,H,W", [(2, 3, 5, 4, 6), (1, 4, 2, 5, 3)])
def test_upsample_conv_gradients_on_the_low_res_grid(B, Cin, Cout, H, W):
    g = torch.Generator().manual_seed(B * 100 + H)
    x = torch.randn(B, Cin, H, W, generator=g, dtype=torch.float64).requires_grad_(True)
    w = torch.randn(Cout, Cin, 3, 3, generator=g, dtype=torch.float64).requires_grad_(True)
    y = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), w, padding=1)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dy)
    dys = s2d(dy)
    assert torch.allclose(taps_conv(dys, Wt.upsample_dgrad_weights(w.detach()), (1, 1, 1, 1)), x.grad, atol=1e-12)
    v = weight_grad(x.detach(), dys, 3, (1, 1, 1, 1))
    assert torch.allclose(Wt.upsample_fold_wgrad(v), w.grad, atol=1e-12)


def test_resampling_functions_need_a_backend_with_the_window_origin():
    """A backend without window_origin (the CPU emulation backend) keeps the modules on their stock path."""
    from bbdm_b200 import train

    class NoOrigin:
        requires_cuda = False

    old = train._BACKEND
    train.set_backend(NoOrigin())
    try:
        x = torch.zeros(2, 64, 16, 16)
        conv = torch.nn.Conv2d(64, 64, 3, stride=2, padding=1)
        assert train.downsample_conv(conv, x) is None
        assert train.upsample_conv(torch.nn.Conv2d(64, 64, 3, padding=1), x) is None
    finally:
        train.set_backend(old)
