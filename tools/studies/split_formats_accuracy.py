#!/usr/bin/env python
"""CPU study (no GPU), round 2: per-layer deviation of candidate tensor-core operand formats against the fp64 conv.

  bf16x3            : today's kernel (A_hi W_hi + A_lo W_hi + A_hi W_lo on split-bf16 planes)
  fp16x3            : same three products on split-fp16 planes (weights pre-scaled by 2^8 so W_lo stays normal)
  wino23_bf16x3     : Winograd F(2x2,3x3), split-bf16 operands            (round-1 study)
  wino23_fp16x3     : Winograd F(2x2,3x3), split-fp16 operands            (round-2 candidate)
  wino43_fp16x3     : Winograd F(4x4,3x3), split-fp16 operands
  fp16_fp8cross     : A_hi W_hi in fp16 + both cross terms as e4m3 x e4m3 products (2 tensor-pipe units instead of 3)
  fp16_mixedcross   : A_hi W_hi + A_lo W_hi in fp16, A_hi W_lo as e4m3 x e4m3 (2.5 units)
All products are evaluated in fp64 on the exactly representable planes (the tensor core's fp32 accumulation is
not modelled), transforms are rounded to fp32 where the kernels would round.
The fixed 2^8 weight scale fits the N(0, 0.02) weights studied here only: for smaller weights W_lo becomes an fp16
subnormal.  The Winograd kernels therefore scale per tensor, by 2^(14 - ceil(log2 max|w|)) (csrc/winograd.cu).
"""
import json

import torch
import torch.nn.functional as F

torch.manual_seed(0)
BT23 = torch.tensor([[1, 0, -1, 0], [0, 1, 1, 0], [0, -1, 1, 0], [0, 1, 0, -1]], dtype=torch.float64)
G23 = torch.tensor([[1, 0, 0], [.5, .5, .5], [.5, -.5, .5], [0, 0, 1]], dtype=torch.float64)
AT23 = torch.tensor([[1, 1, 1, 0], [0, 1, -1, -1]], dtype=torch.float64)
# F(4x4, 3x3), Lavin & Gray interpolation points 0, +-1, +-2
BT43 = torch.tensor([[4, 0, -5, 0, 1, 0], [0, -4, -4, 1, 1, 0], [0, 4, -4, -1, 1, 0],
                     [0, -2, -1, 2, 1, 0], [0, 2, -1, -2, 1, 0], [0, 4, 0, -5, 0, 1]], dtype=torch.float64)
G43 = torch.tensor([[1 / 4, 0, 0], [-1 / 6, -1 / 6, -1 / 6], [-1 / 6, 1 / 6, -1 / 6],
                    [1 / 24, 1 / 12, 1 / 6], [1 / 24, -1 / 12, 1 / 6], [0, 0, 1]], dtype=torch.float64)
AT43 = torch.tensor([[1, 1, 1, 1, 1, 0], [0, 1, -1, 2, -2, 0], [0, 1, 1, 4, 4, 0], [0, 1, -1, 8, -8, 1]],
                    dtype=torch.float64)


def split(x, dt):
    x = x.float()
    hi = x.to(dt).float()
    lo = (x - hi).to(dt).float()
    return hi.double(), lo.double()


def e4m3(x, scale):
    """x*scale rounded to e4m3 (saturating), returned unscaled in fp64."""
    y = (x.float() * scale).clamp(-448, 448).to(torch.float8_e4m3fn).float()
    return y.double() / scale


def pow2_scale(x, target):
    return 2.0 ** torch.floor(torch.log2(torch.tensor(target / float(x.abs().max())))).item()


def conv3(xh, xl, wh, wl):
    return F.conv2d(xh, wh, padding=1) + F.conv2d(xl, wh, padding=1) + F.conv2d(xh, wl, padding=1)


def direct(x, w, dt, wscale=1.0):
    xh, xl = split(x, dt)
    wh, wl = split(w * wscale, dt)
    return conv3(xh, xl, wh, wl) / wscale


def fp8cross(x, w, mixed):
    xh, xl = split(x, torch.float16)
    wh, wl = split(w * 256.0, torch.float16)
    xl_f = (x.float() - xh.float()).double()
    wl_f = (w.float() * 256.0 - wh.float()).double()
    out = F.conv2d(xh, wh, padding=1)
    # e4m3 planes with per-tensor power-of-two scales (top of the range at ~256)
    xh8 = e4m3(xh, pow2_scale(xh, 256.0))
    wl8 = e4m3(wl_f, pow2_scale(wl_f, 256.0))
    out = out + F.conv2d(xh8, wl8, padding=1)
    if mixed:
        out = out + F.conv2d(xl, wh, padding=1)
    else:
        xl8 = e4m3(xl_f, pow2_scale(xl_f, 256.0))
        wh8 = e4m3(wh, pow2_scale(wh, 256.0))
        out = out + F.conv2d(xl8, wh8, padding=1)
    return out / 256.0


def winograd(x, w, dt, BT, G, AT, m, wscale=1.0):
    B, C, H, W = x.shape
    K = w.shape[0]
    a = m + 2
    xp = F.pad(x.double(), (1, 1, 1, 1))
    t = xp.unfold(2, a, m).unfold(3, a, m)
    V = torch.einsum("ij,bcxyjk,lk->bcxyil", BT, t, BT).float()
    U = (torch.einsum("ij,kcjl,ml->kcim", G, w.double(), G) * wscale).float()
    Vh, Vl = split(V, dt)
    Uh, Ul = split(U, dt)
    M = sum(torch.einsum("bcxyil,kcil->bkxyil", p, q) for p, q in ((Vh, Uh), (Vl, Uh), (Vh, Ul))).float()
    Y = (torch.einsum("ij,bkxyjl,ml->bkxyim", AT, M.double(), AT) / wscale).float()
    th, tw = Y.shape[2], Y.shape[3]
    return Y.permute(0, 1, 2, 4, 3, 5).reshape(B, K, th * m, tw * m).double()


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def main():
    for C, K, HW in ((128, 128, 16), (512, 512, 8), (1024, 512, 8)):
        x = F.silu(torch.randn(2, C, HW, HW) * 1.0 + 0.1)
        w = torch.randn(K, C, 3, 3) * 0.02
        ref = F.conv2d(x.double(), w.double(), padding=1)
        row = {"Cin": C, "Cout": K, "HW": HW,
               "bf16x3": rel(direct(x, w, torch.bfloat16), ref),
               "fp16x3": rel(direct(x, w, torch.float16, 256.0), ref),
               "wino23_bf16x3": rel(winograd(x, w, torch.bfloat16, BT23, G23, AT23, 2), ref),
               "wino23_fp16x3": rel(winograd(x, w, torch.float16, BT23, G23, AT23, 2, 256.0), ref),
               "wino43_fp16x3": rel(winograd(x, w, torch.float16, BT43, G43, AT43, 4, 256.0), ref),
               "fp16_fp8cross": rel(fp8cross(x, w, False), ref),
               "fp16_mixedcross": rel(fp8cross(x, w, True), ref),
               "fp32_conv": rel(F.conv2d(x, w, padding=1).double(), ref)}
        print(json.dumps(row))


if __name__ == "__main__":
    main()
