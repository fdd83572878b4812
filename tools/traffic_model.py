#!/usr/bin/env python
"""Algorithmic bytes / FLOPs per kernel family for one UNet forward, from a shape-only dry run of
the engine (tensors on the 'meta' device, a recording backend)."""
import collections
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from bbdm_b200.engine import UNetEngine  # noqa: E402
from bbdm_b200.unet import UNetModel  # noqa: E402


def nbytes(*ts):
    return sum(t.numel() * t.element_size() for t in ts if t is not None)


class Rec:
    requires_cuda = False

    def __init__(self):
        self.b = collections.Counter()
        self.f = collections.Counter()
        self.n = collections.Counter()

    def empty(self, shape, dtype, device):
        return torch.empty(shape, dtype=dtype, device="meta")

    def _add(self, k, by, fl=0):
        self.b[k] += by
        self.f[k] += fl
        self.n[k] += 1

    def nchw_to_nhwc_cat(self, x, ctx, out): self._add("layout", nbytes(x, ctx, out))
    def nhwc_to_nchw(self, src, out): self._add("layout", nbytes(src, out))
    def gather_rows(self, table, idx, out): self._add("small", nbytes(out) * 2)
    def linear(self, x, w, bias, out, act_in=False, act_out=False): self._add("linear", nbytes(w, x, out), 2 * x.shape[0] * w.numel())
    def gn_stats(self, s1, s2, g, eps, mean, rstd, ws): self._add("gn_stats", nbytes(s1, s2))
    def gn_finalize_partials(self, p1, r1, p2, r2, B, hw, g, eps, mean, rstd): self._add("gn_finalize", nbytes(p1, p2))
    def conv_geometry(self, H, W):
        p2f = lambda x: 1 << (x.bit_length() - 1)
        p2c = lambda x: 1 << (x - 1).bit_length()
        tw = min(16, p2f(W)); th = min(128 // tw, p2c(H)); tb = 128 // (tw * th)
        return tw, th, tb, (4 * (-(-W // tw)) * (-(-H // th)) if tb == 1 else 0)
    def prep(self, s1, s2, **kw):
        outs = [kw.get(k) for k in ("act_f32", "act_hi", "act_lo", "raw_f32", "raw_hi", "raw_lo")]
        rd = nbytes(s1, s2) * (4 if kw.get("resample") == 1 else 1) // (1 if kw.get("resample") != 1 else 4)
        self._add("prep", rd + nbytes(*outs))
    def pack_weight_split(self, *a): pass
    def pack_weight_split_taps(self, *a): pass
    def pack_weight_f32(self, *a): pass
    def conv_umma(self, **kw):
        # FLOPs: 2x the MACs the kernel issues (split3 runs each product three times on the tensor pipe)
        B, H, W, Cin, Cout, taps = (kw[k] for k in ("B", "H", "W", "Cin", "Cout", "taps"))
        up = kw.get("upsample2x")
        fl = 2.0 * B * H * W * (4 if up else 1) * Cout * (taps * Cin + kw.get("Cin2", 0))
        by = nbytes(kw["a_hi"], kw["a_lo"], kw["w_hi"], kw["w_lo"], kw.get("a2_hi"), kw.get("a2_lo"), kw.get("out"),
                    kw.get("out_hi"), kw.get("out_lo"), kw.get("stats_partial"))
        if kw.get("res_mode"):
            by += nbytes(kw["residual"])
        fam = "wino_gemm" if kw.get("weights_per_image") else ("conv_umma_up2" if up else f"conv_umma_{taps}tap")
        self._add(fam, by, fl)
    # Winograd transforms (F(4x4,3x3) and F(6x6,3x3)) and their tile grids, as bbdm_wino*_geometry computes them
    wino_tiles = (4, 6)
    wino_tensor_scale = True
    def wino_geometry(self, B, H, W, tile=4):
        th, tw = -(-H // tile), -(-W // tile)
        tot = B * th * tw
        if tile == 6:
            return th, tw, max(128, -(-tot // 16) * 16), True
        return th, tw, tot, H % 4 == 0 and W % 4 == 0 and tot % 16 == 0 and tot >= 128
    def wino_pack_weight(self, *a, **kw): pass
    def wino_input(self, s1, s2, **kw):
        outs = [kw.get(k) for k in ("v_hi", "v_lo", "raw_hi", "raw_lo", "act_hi", "act_lo")]
        self._add("wino_input", nbytes(s1, s2, *outs))
    def wino_output(self, m, **kw):
        res = kw.get("residual") if kw.get("res_mode") else None
        self._add("wino_output", nbytes(m, res, kw["out"], kw.get("stats_partial")))
    def conv_direct(self, src, w, bias, res, out, Cout, k, stride=1):
        self._add("conv_direct", nbytes(src, w, res, out), 2.0 * out.numel() * src.shape[3] * k * k)
    def attention(self, qkv, heads, order, out_f32=None, out_hi=None, out_lo=None):
        B, T, C3 = qkv.shape
        self._add("attention", nbytes(qkv, out_f32, out_hi, out_lo), 4.0 * B * (C3 // 3) * T * T)
    def attention_split(self, qh, ql, heads, order, out_f32=None, out_hi=None, out_lo=None):
        B, T, C3 = qh.shape
        self._add("attention", nbytes(qh, ql, out_f32, out_hi, out_lo), 4.0 * B * (C3 // 3) * T * T)


Rec.attention_tc = Rec.attention_split


def main(cfg_name="cfg2"):
    cfg = bench.CONFIGS[cfg_name]
    unet = UNetModel(**cfg["unet"])
    rec = Rec()
    eng = UNetEngine(unet, backend=rec)
    B, C, S = cfg["batch"], cfg["channels"], cfg["size"]
    x = torch.empty((B, C, S, S), device="meta")
    t = torch.zeros((B,), dtype=torch.long)
    eng._table = torch.empty((1000, cfg["unet"]["model_channels"]), device="meta")
    orig_to = torch.Tensor.to
    eng.forward(x, torch.empty((B,), dtype=torch.long, device="meta"), x, out=torch.empty((B, cfg["unet"]["out_channels"], S, S), device="meta"))
    print(f"# {cfg_name}: algorithmic HBM bytes / FLOPs per UNet forward, by kernel family")
    print("family,launches,GB,TFLOP,ms_at_6501.9GBps")
    for k in sorted(rec.b, key=lambda k: -rec.b[k]):
        print(f"{k},{rec.n[k]},{rec.b[k] / 1e9:.3f},{rec.f[k] / 1e12:.3f},{rec.b[k] / 6501.9e9 * 1e3:.3f}")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "cfg2")
