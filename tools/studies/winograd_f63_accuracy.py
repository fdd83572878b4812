#!/usr/bin/env python
"""CPU study (no GPU): Winograd F(6x6,3x3) against F(4x4,3x3) and the direct split-bf16 x3 kernel, all against the fp64
direct convolution.

Emulates what csrc/winograd.cu + the wgmma position GEMMs compute: V = B^T d B in fp32, U = s G g G^T (fp64 -> fp32,
s the kernel's per-tensor power of two), both split into fp16 hi/lo planes; M = V_hi U_hi + V_lo U_hi + V_hi U_lo summed
exactly and rounded to fp32; Y = A^T M A / s in fp32.  Maps that do not divide into tiles are zero-padded, as the
kernels do.  The exact sum leaves out the tensor core's truncating accumulator between fp32 promotions, which the GPU
tests (tests/test_gpu_winograd.py, tests/test_gpu_winograd6.py) cover.

Transform matrices come from the Toom-Cook construction on the interpolation points: 0, +-1, +-2 for F(4,3) and
0, +-1, +-2, +-1/2 for F(6,3) (plus the point at infinity).
"""
import json

import numpy as np
import torch
import torch.nn.functional as F

torch.manual_seed(0)
POINTS = {4: [0, 1, -1, 2, -2], 6: [0, 1, -1, 2, -2, 0.5, -0.5]}


def toom(m, pts):
    """(A^T [m x n], G [n x 3], B^T [n x n]) of F(m, 3), n = m + 2."""
    r, n = 3, m + 2
    assert len(pts) == n - 1
    AT, G = np.zeros((m, n)), np.zeros((n, r))
    for j, p in enumerate(pts):
        AT[:, j] = [p ** i for i in range(m)]
        den = np.prod([p - q for q in pts if q != p])
        G[j] = [p ** k / den for k in range(r)]
    AT[m - 1, n - 1] = 1
    G[n - 1, r - 1] = 1
    # B^T from exactness: sum_j AT[i,j] G[j,k] BT[j,l] = [l == i+k]
    rows, rhs = [], []
    for i in range(m):
        for k in range(r):
            for l in range(n):
                row = np.zeros((n, n))
                row[:, l] = AT[i] * G[:, k]
                rows.append(row.ravel())
                rhs.append(1.0 if l == i + k else 0.0)
    BT = np.linalg.lstsq(np.array(rows), np.array(rhs), rcond=None)[0].reshape(n, n)
    BT[np.abs(BT) < 1e-12] = 0
    return [torch.tensor(x, dtype=torch.float64) for x in (AT, G, BT)]


def split16(x, s=1.0):
    x = (x * s).float()
    hi = x.half().float()
    lo = (x - hi).half().float()
    return hi.double(), lo.double()


def winograd(x, w, m):
    AT, G, BT = toom(m, POINTS[m])
    n = m + 2
    B, C, H, W = x.shape
    K = w.shape[0]
    th, tw = -(-H // m), -(-W // m)
    xp = F.pad(x.double(), (1, 1 + tw * m - W, 1, 1 + th * m - H))
    t = xp.unfold(2, n, m).unfold(3, n, m)                                        # [B, C, th, tw, n, n]
    V = torch.einsum("ij,bcxyjk,lk->bcxyil", BT.float(), t.float(), BT.float())    # fp32 input transform
    U = torch.einsum("ij,kcjl,ml->kcim", G, w.double(), G).float()
    s = 2.0 ** (14 - np.ceil(np.log2(float(w.abs().max()))))                    # the kernel's per-tensor scale
    Vh, Vl = split16(V)
    Uh, Ul = split16(U, s)
    M = sum(torch.einsum("bcxyil,kcil->bkxyil", a, b) for a, b in ((Vh, Uh), (Vl, Uh), (Vh, Ul))).float()
    Y = torch.einsum("ij,bkxyjl,ml->bkxyim", AT.float(), M, AT.float()) / s
    return Y.permute(0, 1, 2, 4, 3, 5).reshape(B, K, th * m, tw * m)[:, :, :H, :W].double()


def direct_bf16x3(x, w):
    def sp(z):
        z = z.float()
        hi = z.bfloat16().float()
        return hi.double(), (z - hi).bfloat16().double()
    xh, xl = sp(x)
    wh, wl = sp(w)
    return F.conv2d(xh, wh, padding=1) + F.conv2d(xl, wh, padding=1) + F.conv2d(xh, wl, padding=1)


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


def main():
    rows = []
    for C, K, HW, xs, wstd in ((512, 64, 24, 1.0, 0.02), (1024, 64, 18, 1.0, 0.02), (512, 64, 24, 3.0, 0.05),
                               (512, 64, 24, 1.0, 0.2)):
        x = F.silu(torch.randn(1, C, HW, HW, dtype=torch.float64) * xs + 0.1)  # post GN+SiLU-like
        w = torch.randn(K, C, 3, 3, dtype=torch.float64) * wstd
        ref = F.conv2d(x, w, padding=1)
        rows.append({"Cin": C, "Cout": K, "HW": HW, "act_scale": xs, "w_std": wstd,
                     "direct_bf16x3": rel(direct_bf16x3(x, w), ref),
                     "f43": rel(winograd(x, w, 4), ref), "f63": rel(winograd(x, w, 6), ref)})
        print(json.dumps(rows[-1]), flush=True)
    return rows


if __name__ == "__main__":
    main()
