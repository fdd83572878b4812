#!/usr/bin/env python
"""Per-launch time of bbdm_conv_wgrad (the weight-gradient GEMM and its split-K reduce) at the training shapes of the
benchmark UNets: the cfg3 levels at batch 32 and the cfg2 levels at batch 8 (3x3 C -> C and the wide-input 3x3
conv1s of each level, the attention levels' 1x1 qkv).  CUDA events around --iters launches after --warmup.

Prints one JSON line: per shape the mean ms, and a sha256 of the dW bytes (seeded operands), so two builds can be
compared for time and for bit-identical results.

    python tools/time_wgrad.py [--iters 50] [--warmup 5] [--shapes cfg3,cfg2]
"""
import hashlib
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bbdm_b200 import cabi, train  # noqa: E402

# name: (B, H, W, Cin, Cout, taps)
SHAPES = {
    "cfg3": [("64x64 3x3 128", 32, 64, 64, 128, 128, 9), ("32x32 3x3 512", 32, 32, 32, 512, 512, 9),
             ("32x32 3x3 128->512", 32, 32, 32, 128, 512, 9), ("16x16 3x3 1024", 32, 16, 16, 1024, 1024, 9),
             ("16x16 3x3 1536->1024", 32, 16, 16, 1536, 1024, 9), ("32x32 1x1 qkv 512", 32, 32, 32, 512, 1536, 1),
             ("16x16 1x1 qkv 1024", 32, 16, 16, 1024, 3072, 1)],
    "cfg2": [("256x256 3x3 128", 8, 256, 256, 128, 128, 9), ("128x128 3x3 512", 8, 128, 128, 512, 512, 9),
             ("128x128 3x3 128->512", 8, 128, 128, 128, 512, 9), ("64x64 3x3 1024", 8, 64, 64, 1024, 1024, 9),
             ("64x64 3x3 1536->1024", 8, 64, 64, 1536, 1024, 9)],
}


def _arg(flag, default):
    return type(default)(sys.argv[sys.argv.index(flag) + 1]) if flag in sys.argv else default


def time_shape(be, B, H, W, Cin, Cout, taps, iters, warmup):
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(B * 7 + H * 5 + Cin * 3 + Cout)
    P = B * H * W
    a_hi = torch.randn((B, H, W, Cin), device=dev, generator=g).to(torch.bfloat16)
    a_lo = (1e-3 * torch.randn((B, H, W, Cin), device=dev, generator=g)).to(torch.bfloat16)
    dy = 0.1 * torch.randn((P, Cout), device=dev, generator=g)
    gt_hi = torch.empty((Cout, P), dtype=torch.bfloat16, device=dev)
    gt_lo = torch.empty_like(gt_hi)
    be.split_grad(dy, None, None, gt_hi, gt_lo)
    _, fl = be.wgrad_workspace(B, H, W, Cin, Cout, taps)
    ws = torch.empty((fl,), dtype=torch.float32, device=dev)
    k = {1: 1, 9: 3}[taps]
    dw = torch.empty((Cout, Cin, k, k), dtype=torch.float32, device=dev)
    run = lambda: be.conv_wgrad(gt_hi, gt_lo, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, ws)
    for _ in range(warmup):
        run()
    torch.cuda.synchronize()
    digest = hashlib.sha256(dw.cpu().numpy().tobytes()).hexdigest()[:16]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    be.check_fault()
    ms = e0.elapsed_time(e1) / iters
    return {"ms": round(ms, 4), "tflops_3_products": round(2 * P * taps * Cin * Cout * 3 / ms / 1e9, 1), "dw_sha": digest}


if __name__ == "__main__":
    assert torch.cuda.is_available(), "time_wgrad needs a GPU"
    iters, warmup = _arg("--iters", 50), _arg("--warmup", 5)
    groups = _arg("--shapes", "cfg3,cfg2").split(",")
    be = train.backend()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": smi, "lib": cabi.LIB_PATH, "abi": cabi.ABI_VERSION, "rows": []}
    for grp in groups:
        for name, *shape in SHAPES[grp]:
            out["rows"].append({"config": grp, "shape": name, **time_shape(be, *shape, iters, warmup)})
    print(json.dumps(out))
