#!/usr/bin/env python
"""Time attention heads whose width is not a multiple of 8 (the padded-head route) against the stock-PyTorch core the
training graph ran before these widths had a native path.  For each shape (self-attention, legacy qkv order):

  native_fwd       AttentionCoreFn forward: the head repack (prep(heads=...)), the kernel at d rounded up to 8, the repack back
  native_fwd_bwd   + its backward: the repacks around bbdm_attention_bwd
  stock_fwd        the stock core (AttentionBlock._attention_torch), fp32, TF32 off
  stock_fwd_bwd    + its autograd backward

Each variant is warmed up, then the variants are timed in alternating rounds (CUDA events around --iters calls); the
median over rounds and the spread (min..max) are printed with the peak memory a forward + backward allocates above its
inputs, the card and its power limit.  With --unet, one sampling forward of a 224 x (1, 2, 3, 4) UNet whose heads are
sized by num_heads: 8 (widths 28, 56, 84, 112; attention at every level) is timed the same way.  One JSON line per
measurement goes to stdout and, with --out, to a file.

    python tools/time_attention_pad.py                        # the default shapes and the UNet
    python tools/time_attention_pad.py --shapes 8,1024,8,20   # B,T,heads,head_dim
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
from bbdm_b200 import cabi, train  # noqa: E402
from bbdm_b200.unet import AttentionBlock, UNetModel  # noqa: E402

DEFAULT_SHAPES = ["8,1024,8,20", "8,1024,8,84", "8,1024,8,28", "8,4096,8,12"]
UNET_224 = dict(image_size=32, in_channels=3, model_channels=224, out_channels=3, num_res_blocks=2,
                attention_resolutions=(1, 2, 4, 8), channel_mult=(1, 2, 3, 4), conv_resample=True, dims=2, num_heads=8,
                num_head_channels=-1, use_scale_shift_norm=True, resblock_updown=True, use_spatial_transformer=False,
                context_dim=None, condition_key="nocond")


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def variants(B, T, heads, D):
    C = heads * D
    g = torch.Generator(device="cuda").manual_seed(0)
    qkv = torch.randn(B, 3 * C, 1, T, device="cuda", generator=g)
    dout = torch.randn(B, C, 1, T, device="cuda", generator=g)
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


def run(fns, a, what, card, peaks=()):
    for fn in fns.values():
        for _ in range(a.warmup):
            fn()
    samples = {k: [] for k in fns}
    for _ in range(a.rounds):
        for k, fn in fns.items():
            samples[k].append(time_ms(fn, a.iters))
    pk = {k: peak_mib(fns[k]) for k in peaks}
    lines = []
    for k, s in samples.items():
        rec = dict(shape=what, variant=k, median_ms=round(statistics.median(s), 4), min_ms=round(min(s), 4),
                   max_ms=round(max(s), 4), card=card)
        if k in pk:
            rec["peak_mib"] = round(pk[k], 1)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
    return lines


def unet_forward(B):
    """One sampling forward of UNET_224 (seeded weights) at batch B on the native engine."""
    torch.manual_seed(0)
    net = UNetModel(**UNET_224).eval().cuda()
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(0.05 * torch.randn_like(p))
    S = UNET_224["image_size"]
    x = torch.randn(B, UNET_224["in_channels"], S, S, device="cuda")
    t = torch.randint(0, 1000, (B,), device="cuda")

    def fwd():
        with torch.no_grad():
            net(x, timesteps=t)
    return fwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", nargs="+", default=DEFAULT_SHAPES, metavar="B,T,heads,D")
    ap.add_argument("--unet", type=int, default=8, metavar="B", help="batch of the UNet forward (0: skip it)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_attention_pad.py needs a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    be = cabi.CudaBackend()
    card = f"{torch.cuda.get_device_name()} (power limit, max SM clock: {power_limit()})"
    print(f"# {card}; median of {a.rounds} alternating rounds x {a.iters} calls, spread = min..max")
    lines = []
    for spec in a.shapes:
        B, T, heads, D = (int(z) for z in spec.split(","))
        if not cabi.attn_pad_route(be, D):
            ap.error(f"head_dim {D}: not on the padded-head route (a multiple of 8, or wider than 256)")
        lines += run(variants(B, T, heads, D), a, f"B={B} T={T} {heads}x{D}", card,
                     peaks=("native_fwd_bwd", "stock_fwd_bwd"))
    if a.unet:
        lines += run({"native_sampling_forward": unet_forward(a.unet)}, a,
                     f"UNet 224x(1,2,3,4) num_heads 8, {UNET_224['image_size']}x{UNET_224['image_size']}, B={a.unet}",
                     card)
    be.check_fault()
    if a.out:
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
