#!/usr/bin/env python
"""Time the attention core at head sizes above 128 against the stock-PyTorch core the training graph ran before these
sizes had kernels.  For each shape:

  native_fwd       bbdm_attention (fp32 qkv, the training forward; cross: bbdm_attention_cross on split planes)
  native_fwd_bwd   + bbdm_attention_bwd (cross: bbdm_attention_cross_bwd)
  stock_fwd        the stock core (AttentionBlock._attention_torch / the CrossAttention einsums), fp32, TF32 off
  stock_fwd_bwd    + its autograd backward

Each variant is warmed up, then the variants are timed in alternating rounds (CUDA events around --iters calls); the
median over rounds and the spread (min..max) are printed with the peak memory a forward + backward allocates above its
inputs, the card and its power limit.  One JSON line per (shape, variant) goes to stdout and, with --out, to a file.

    python tools/time_attention_wide.py                        # the four default shapes
    python tools/time_attention_wide.py --shapes 8,1024,4,256  # B,T,heads,head_dim[,Tkv for cross-attention]
"""
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

DEFAULT_SHAPES = ["8,1024,4,256", "8,1024,8,160", "8,256,8,192", "8,256,8,192,256", "4,4096,1,256"]


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def variants(be, B, T, heads, D, Tkv):
    """{name: (fn, inputs that the peak is measured above)} for one shape."""
    C = heads * D
    g = torch.Generator(device="cuda").manual_seed(0)
    dev = "cuda"
    lse = torch.empty(B * heads * T, device=dev)
    delta = torch.empty_like(lse)
    if Tkv is None:
        qkv = torch.randn(B, T, 3 * C, device=dev, generator=g)
        out = torch.empty(B, T, C, device=dev)
        dout = torch.randn(B, T, C, device=dev, generator=g)
        dqkv = torch.empty_like(qkv)
        qkv_bct = qkv.permute(0, 2, 1).contiguous()
        dout_bct = dout.permute(0, 2, 1).contiguous()
        core = SimpleNamespace(num_heads=heads, new_order=False)

        def native_fwd():
            be.attention(qkv, heads, 0, out, None, None)

        def native_fwd_bwd():
            be.attention(qkv, heads, 0, out, None, None)
            be.attention_bwd(qkv, out, dout, heads, 0, dqkv, lse, delta)

        def stock(bwd):
            x = qkv_bct.detach().requires_grad_(bwd)
            o = AttentionBlock._attention_torch(core, x)
            if bwd:
                o.backward(dout_bct)
    else:
        q = torch.randn(B, T, C, device=dev, generator=g)
        kv = torch.randn(B, Tkv, 2 * C, device=dev, generator=g)
        split = lambda t: (t.to(torch.bfloat16), (t - t.to(torch.bfloat16).float()).to(torch.bfloat16))
        (q_hi, q_lo), (kv_hi, kv_lo) = split(q), split(kv)
        out = torch.empty(B, T, C, device=dev)
        dout = torch.randn(B, T, C, device=dev, generator=g)
        dq, dkv = torch.empty_like(q), torch.empty_like(kv)

        def native_fwd():
            be.attention_cross(q_hi, q_lo, kv_hi, kv_lo, heads, out_f32=out)

        def native_fwd_bwd():
            be.attention_cross(q_hi, q_lo, kv_hi, kv_lo, heads, out_f32=out)
            be.attention_cross_bwd(q, kv, out, dout, heads, dq, dkv, lse, delta)

        def stock(bwd):      # CrossAttention.forward's core (transformer.py), batch*heads first
            qq, kk = q.detach().requires_grad_(bwd), kv.detach().requires_grad_(bwd)
            sp = lambda t, n: t.reshape(B, n, heads, D).permute(0, 2, 1, 3).reshape(B * heads, n, D)
            w = (torch.einsum("bid,bjd->bij", sp(qq, T), sp(kk[..., :C], Tkv)) * D ** -0.5).softmax(dim=-1)
            o = torch.einsum("bij,bjd->bid", w, sp(kk[..., C:], Tkv)).reshape(B, heads, T, D)
            if bwd:
                o.permute(0, 2, 1, 3).reshape(B, T, C).backward(dout)

    return {"native_fwd": native_fwd, "native_fwd_bwd": native_fwd_bwd,
            "stock_fwd": lambda: stock(False), "stock_fwd_bwd": lambda: stock(True)}


def time_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def peak_mib(fn):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=DEFAULT_SHAPES, metavar="B,T,heads,D[,Tkv]")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_attention_wide.py needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    ok, rule = cabi.attn_head_dims(cabi.CudaBackend)
    be = cabi.CudaBackend()
    card = f"{torch.cuda.get_device_name()} (power limit {power_limit()})"
    print(f"# {card}; median of {a.rounds} alternating rounds x {a.iters} calls, spread = min..max")
    lines = []
    for spec in a.shapes:
        v = [int(z) for z in spec.split(",")]
        B, T, heads, D = v[:4]
        Tkv = v[4] if len(v) > 4 else None
        if not ok(D):
            ap.error(f"head_dim {D}: the kernels take {rule}")
        fns = variants(be, B, T, heads, D, Tkv)
        for fn in fns.values():
            for _ in range(a.warmup):
                fn()
        samples = {k: [] for k in fns}
        for _ in range(a.rounds):
            for k, fn in fns.items():
                samples[k].append(time_ms(fn, a.iters))
        peaks = {k: peak_mib(fns[k]) for k in ("native_fwd_bwd", "stock_fwd_bwd")}
        be.check_fault()
        what = f"B={B} T={T} {heads}x{D}" + ("" if Tkv is None else f" cross Tkv={Tkv}")
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
