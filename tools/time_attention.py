#!/usr/bin/env python
"""Time the attention kernels alone with CUDA events, per head_dim at equal FLOPs.

    python tools/time_attention.py [--head-dims 64 128] [--B 16 --T 4096 --C 1024] [--kernels ...] [--out FILE]
    python tools/time_attention.py B T C heads          # one head layout, head_dim = C / heads

Default: the cfg2 middle-block shape (B=16, T=4096, C=1024) as 16 heads x 64 and as 8 heads x 128.  For each
head_dim it times the --kernels (default: bbdm_attention_tc with split-bf16 planes in and split planes out, and
bbdm_attention_bwd in exact fp32; also available: the mma.sync forwards bbdm_attention, fp32 qkv in and fp32 out, and
bbdm_attention_split, split planes in and out, and stock_fwd_bwd, the stock PyTorch attention core that training
runs on shapes the kernels do not take (AttentionBlock._attention_torch, fp32, forward and autograd backward through
the stored T x T matrix)), alternating the variants over rounds and reporting the median.  attention_tc takes
head_dim 64 and 128; attention, attention_split and attention_bwd take any multiple of 8 up to 128.
Algorithmic FLOPs: forward 4 B T^2 C (QK^T, PV), backward 10 B T^2 C (the five T x T x D products of
FlashAttention's backward), whatever the kernels recompute; stock_fwd_bwd counts both (14 B T^2 C).
One JSON line per (kernel, head_dim), each tagged with the card's name and power limit read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bbdm_b200 import cabi  # noqa: E402
from bbdm_b200.unet import AttentionBlock  # noqa: E402


def card():
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = r.stdout.strip() or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return info


def event_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("shape", type=int, nargs="*", metavar="B T C heads", help="time this one shape instead")
    ap.add_argument("--head-dims", type=int, nargs="+", default=[64, 128])
    ap.add_argument("--B", type=int, default=16)
    ap.add_argument("--T", type=int, default=4096)
    ap.add_argument("--C", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--fwd-iters", type=int, default=10)
    ap.add_argument("--bwd-iters", type=int, default=2)
    ap.add_argument("--kernels", nargs="+", default=["attention_tc", "attention_bwd"],
                    choices=["attention_tc", "attention_bwd", "attention", "attention_split", "stock_fwd_bwd"])
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    if a.shape:
        if len(a.shape) != 4 or a.shape[2] % a.shape[3]:
            ap.error("positional form: B T C heads, with C divisible by heads")
        a.B, a.T, a.C = a.shape[:3]
        a.head_dims = [a.shape[2] // a.shape[3]]
    for d in a.head_dims:
        head_dim_ok, rule = cabi.attn_head_dims(cabi.CudaBackend)
        if not head_dim_ok(d):
            ap.error(f"head_dim {d}: the kernels take {rule}")
        if "attention_tc" in a.kernels and d not in cabi.ATTN_TC_HEAD_DIMS:
            ap.error(f"attention_tc takes head_dim {cabi.ATTN_TC_HEAD_DIMS}, not {d}")
    assert torch.cuda.is_available(), "time_attention.py needs a GPU"
    B, T, C = a.B, a.T, a.C
    be = cabi.CudaBackend()
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(B, T, 3 * C, device="cuda", generator=g)
    hi = qkv.to(torch.bfloat16)
    lo = (qkv - hi.float()).to(torch.bfloat16)
    o_hi = torch.empty(B, T, C, dtype=torch.bfloat16, device="cuda")
    o_lo = torch.empty_like(o_hi)
    out = torch.empty(B, T, C, device="cuda")
    dout = torch.randn(B, T, C, device="cuda", generator=g)
    dqkv = torch.empty_like(qkv)
    qkv_bct = qkv.permute(0, 2, 1).contiguous()                    # the stock core's [B, 3C, T] layout

    def stock_fwd_bwd(heads):
        x = qkv_bct.detach().requires_grad_(True)
        AttentionBlock._attention_torch(SimpleNamespace(num_heads=heads, new_order=False), x).backward(
            dout.permute(0, 2, 1))

    runs = []                                                      # (kernel, head_dim, heads, fn, iters, flops)
    for d in a.head_dims:
        assert C % d == 0, (C, d)
        heads = C // d
        lse = torch.empty(B * heads * T, device="cuda")
        delta = torch.empty_like(lse)
        fns = {"attention_tc": (lambda h=heads: be.attention_tc(hi, lo, h, 0, None, o_hi, o_lo), a.fwd_iters, 4.0),
               "attention_bwd": (lambda h=heads, l=lse, dl=delta: be.attention_bwd(qkv, out, dout, h, 0, dqkv, l, dl),
                                 a.bwd_iters, 10.0),
               "attention": (lambda h=heads: be.attention(qkv, h, 0, out, None, None), a.fwd_iters, 4.0),
               "attention_split": (lambda h=heads: be.attention_split(hi, lo, h, 0, None, o_hi, o_lo), a.fwd_iters, 4.0),
               "stock_fwd_bwd": (lambda h=heads: stock_fwd_bwd(h), a.bwd_iters, 14.0)}
        if "attention_bwd" in a.kernels:
            be.attention(qkv, heads, 0, out, None, None)           # the forward output the backward is given
        for k in a.kernels:
            fns[k][0]()                                            # warm up every shape timed below
            runs.append((k, d, heads, *fns[k], []))
        torch.cuda.synchronize()
    info = card()
    for _ in range(a.rounds):                                      # alternate the variants
        for k, d, heads, fn, iters, fl, ms in runs:
            ms.append(event_ms(fn, iters))
    be.check_fault()

    lines = []
    for k, d, heads, fn, iters, fl, ms in runs:
        med = statistics.median(ms)
        lines.append(json.dumps({"kernel": k, "B": B, "T": T, "C": C, "heads": heads, "head_dim": d,
                                 "ms": round(med, 4), "ms_rounds": [round(x, 4) for x in ms],
                                 "algo_tflops": round(fl * B * T * T * C / med / 1e9, 2), **info}))
    for ln in lines:
        print(ln)
    if a.out:
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
