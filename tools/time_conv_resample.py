#!/usr/bin/env python
"""Time the UNet's standalone resampling convolutions (resblock_updown=False, conv_resample=True).

    python tools/time_conv_resample.py [--out FILE]

  sampling  the Downsample's 3x3 stride-2 conv: the fp32 SIMT kernel (bbdm_conv_direct, stride 2) against the
            tensor-core route the sampling executor takes (bbdm_s2d_split + bbdm_conv_umma taps 4, window origin -1,
            GroupNorm partial sums in the epilogue), at batch 16: 128 channels on 256x256 and 512 on 128x128 (the cfg2
            levels of a resblock_updown=False UNet), the 64x64 level, and small maps at batch 1 and 2.
  training  forward + backward of Stride2Conv2dFn / Up2Conv2dFn against the nn.Conv2d graph on cuDNN
            (F.interpolate + conv for the upsample), with cuDNN's TF32 on (PyTorch's default) and off.
Prints one JSON line per measurement and the GPU's name and power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bbdm_b200 import cabi, train  # noqa: E402
from bbdm_b200.weights import stride2_s2d_weights  # noqa: E402

# B, H (= W), C: the cfg2 levels, the 64x64 level, and small maps / batches (the smallest the route takes: W/2 = 4)
DOWN_SHAPES = [(16, 256, 128), (16, 128, 512), (16, 64, 128), (16, 64, 512), (16, 32, 512), (2, 32, 64), (2, 16, 128),
               (1, 8, 64), (1, 8, 512)]
TRAIN_SHAPES = [(8, 256, 128), (8, 128, 512), (8, 64, 512)]                                  # B, H of the input, C


def timeit(fn, n=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def time_downsample(be, dev, rows):
    bf = torch.bfloat16
    for B, H, C in DOWN_SHAPES:
        h = H // 2
        x = torch.randn(B, H, H, C, device=dev)
        w, b = 0.02 * torch.randn(C, C, 3, 3, device=dev), torch.zeros(C, device=dev)
        wf = torch.empty((9, C, C), device=dev)
        be.pack_weight_f32(w, wf)
        s_hi, s_lo = torch.empty((4, C, 4 * C), dtype=bf, device=dev), torch.empty((4, C, 4 * C), dtype=bf, device=dev)
        be.pack_weight_split_taps(stride2_s2d_weights(w), s_hi, s_lo)
        out_d, out_t = torch.empty((B, h, h, C), device=dev), torch.empty((B, h, h, C), device=dev)
        a_hi, a_lo = torch.empty((B, h, h, 4 * C), dtype=bf, device=dev), torch.empty((B, h, h, 4 * C), dtype=bf, device=dev)
        rows_pi = be.conv_geometry(h, h)[3]
        part = torch.empty((B * rows_pi, C, 2), device=dev) if rows_pi else None

        def simt():
            be.conv_direct(x, wf, b, None, out_d, C, 3, 2)

        def conv():
            be.conv_umma(B=B, H=h, W=h, Cin=4 * C, Cout=C, taps=4, a_hi=a_hi, a_lo=a_lo, w_hi=s_hi, w_lo=s_lo, bias=b,
                         out=out_t, passes=3, stats_partial=part, window_origin=-1)

        def tc():
            be.s2d_split(x, a_hi, a_lo)
            conv()

        t_simt, t_tc, t_split = timeit(simt, 5 if H >= 256 else 20), timeit(tc), timeit(lambda: be.s2d_split(x, a_hi, a_lo))
        rel = float((out_t - out_d).abs().max() / out_d.abs().max())
        r = dict(what="downsample_sampling", B=B, H=H, C=C, simt_ms=round(t_simt, 4), tc_ms=round(t_tc, 4),
                 s2d_split_ms=round(t_split, 4), speedup=round(t_simt / t_tc, 2), tc_vs_simt_rel_dev=rel)
        print(json.dumps(r), flush=True)
        rows.append(r)
        del x, out_d, out_t, a_hi, a_lo


def time_training(dev, rows):
    for kind in ("down", "up"):
        for B, H, C in TRAIN_SHAPES:
            if kind == "up":
                H //= 2                                           # low-res input of the upsample
            x = torch.randn(B, C, H, H, device=dev).contiguous(memory_format=torch.channels_last).requires_grad_(True)
            conv = torch.nn.Conv2d(C, C, 3, stride=2 if kind == "down" else 1, padding=1).to(dev)
            conv = conv.to(memory_format=torch.channels_last)
            fn = train.Stride2Conv2dFn if kind == "down" else train.Up2Conv2dFn
            with torch.no_grad():
                ho = H // 2 if kind == "down" else 2 * H
            gy = torch.randn(B, C, ho, ho, device=dev).contiguous(memory_format=torch.channels_last)

            def native():
                fn.apply(x, conv.weight, conv.bias).backward(gy)

            def library():
                y = conv(x) if kind == "down" else conv(F.interpolate(x, scale_factor=2, mode="nearest"))
                y.backward(gy)

            t_nat = timeit(native, 10)
            res = {}
            for tf32 in (True, False):
                torch.backends.cudnn.allow_tf32 = tf32
                res[tf32] = timeit(library, 10)
            torch.backends.cudnn.allow_tf32 = True
            r = dict(what=f"{kind}sample_training_fwd_bwd", B=B, H=H, C=C, native_ms=round(t_nat, 4),
                     cudnn_tf32_ms=round(res[True], 4), cudnn_fp32_ms=round(res[False], 4))
            print(json.dumps(r), flush=True)
            rows.append(r)
            del x, gy


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs an sm_90a GPU"
    dev = "cuda"
    be = cabi.CudaBackend()
    rows = [dict(gpu=gpu_info())]
    print(json.dumps(rows[0]), flush=True)
    time_downsample(be, dev, rows)
    time_training(dev, rows)
    be.check_fault()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
