#!/usr/bin/env python
"""Time the attention core at head sizes above 256 (the GEMM-composed route) against the stock-PyTorch core the
training graph ran before these sizes had a native route.  For each shape:

  native_fwd       train.AttentionCoreFn forward: per (image, head) S = Q K^T, bbdm_softmax_rows_split, O = P V
  native_fwd_bwd   + its backward: S and dP = dO V^T, the P and dS planes (bbdm_softmax_rows_split / _bwd), dQ = dS K,
                   dK / dV as weight gradients
  stock_fwd        the stock core (AttentionBlock._attention_torch), fp32, TF32 off
  stock_fwd_bwd    + its autograd backward

Each variant is warmed up, then the variants are timed in alternating rounds (CUDA events around --iters calls); the
median over rounds and the spread (min..max) are printed with the peak memory a forward + backward allocates above its
inputs, the card and its power limit.  One JSON line per (shape, variant) goes to stdout and, with --out, to a file.

    python tools/time_attention_gemm.py                         # the three default shapes
    python tools/time_attention_gemm.py --shapes 8,1024,1,1024  # B,T,heads,head_dim
"""
import argparse
import json
import os
import statistics
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bbdm_b200 import cabi, train  # noqa: E402
from bbdm_b200.unet import AttentionBlock  # noqa: E402
from time_attention_wide import peak_mib, power_limit, time_ms  # noqa: E402

DEFAULT_SHAPES = ["8,1024,1,1024", "8,256,2,512", "4,4096,1,512"]


def variants(B, T, heads, D):
    C = heads * D
    side = int(round(T ** 0.5))
    assert side * side == T, "T must be a square token grid"
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(B, 3 * C, side, side, device="cuda", generator=g)
    dout = 0.3 * torch.randn(B, C, side, side, device="cuda", generator=g)
    core = SimpleNamespace(num_heads=heads, new_order=False)

    def native(bwd):
        x = qkv.detach().requires_grad_(bwd)
        o = train.AttentionCoreFn.apply(x, heads, 0)
        if bwd:
            o.backward(dout)

    def stock(bwd):
        x = qkv.detach().view(B, 3 * C, T).requires_grad_(bwd)
        o = AttentionBlock._attention_torch(core, x)
        if bwd:
            o.backward(dout.view(B, C, T))

    return {"native_fwd": lambda: native(False), "native_fwd_bwd": lambda: native(True),
            "stock_fwd": lambda: stock(False), "stock_fwd_bwd": lambda: stock(True)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=DEFAULT_SHAPES, metavar="B,T,heads,D")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_attention_gemm.py needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    be = train.backend()
    card = f"{torch.cuda.get_device_name()} (power limit {power_limit()})"
    print(f"# {card}; median of {a.rounds} alternating rounds x {a.iters} calls, spread = min..max")
    lines = []
    for spec in a.shapes:
        B, T, heads, D = (int(z) for z in spec.split(","))
        if not cabi.attn_gemm_route(be, D):
            ap.error(f"head_dim {D} does not take the GEMM route (it must exceed {be.attn_max_head_dim})")
        fns = variants(B, T, heads, D)
        for fn in fns.values():
            for _ in range(a.warmup):
                fn()
        samples = {k: [] for k in fns}
        for _ in range(a.rounds):
            for k, fn in fns.items():
                samples[k].append(time_ms(fn, a.iters))
        peaks = {k: peak_mib(fns[k]) for k in ("native_fwd_bwd", "stock_fwd_bwd")}
        be.check_fault()
        what = f"B={B} T={T} {heads}x{D}"
        for k, s in samples.items():
            rec = dict(shape=what, variant=k, median_ms=round(statistics.median(s), 4), min_ms=round(min(s), 4),
                       max_ms=round(max(s), 4), card=card)
            if k in peaks:
                rec["peak_mib"] = round(peaks[k], 1)
            lines.append(json.dumps(rec))
            print(lines[-1], flush=True)
    if a.out:
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
