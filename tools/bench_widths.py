#!/usr/bin/env python
"""Sampling and training steps of LDM-4-shaped UNets whose channel counts are multiples of 32 but not all of 64, on
CudaBackend (tensor-core convs at the multiple of 32) against the same model on the 64 rule (a CudaBackend subclass
that declares conv_channel_multiple = 64: the widths that miss it run on the fp32 direct conv in sampling and on stock
PyTorch in training).

    python tools/bench_widths.py [--widths 224,96,160] [--batch 8] [--steps 10] [--warmup 3]

The UNet: 64x64 latents (3 channels, unconditioned), channel_mult (1, 2, 3, 4), two ResBlocks per level, attention at
ds 8, 4 and 2 with num_head_channels 32.  Per width and routing: ms per eager UNet sampling forward (the executor,
UNetEngine.forward), ms per CUDA-graph replay of that forward, and ms per training step (q_sample + UNet forward + L1
loss + backward); host clock around --steps steps that end in a device synchronise.  The card name and power limit are
printed beside the times.
"""
import argparse
import os
import subprocess
import sys
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from bbdm_b200 import cabi, train  # noqa: E402
from bbdm_b200.engine import UNetEngine  # noqa: E402
from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel  # noqa: E402
from _recipe import bb_namespace, fill_state_dict, synth_images  # noqa: E402


class Rule64Backend(cabi.CudaBackend):
    """CudaBackend with the channel rule of the kernels before they took multiples of 32."""
    conv_channel_multiple = 64


def unet(width):
    return dict(image_size=64, in_channels=3, model_channels=width, out_channels=3, num_res_blocks=2,
                attention_resolutions=(8, 4, 2), channel_mult=(1, 2, 3, 4), conv_resample=True, dims=2, num_heads=8,
                num_head_channels=32, use_scale_shift_norm=True, resblock_updown=True, use_spatial_transformer=False,
                context_dim=None, condition_key="nocond")


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def run(width, be, batch, steps, warmup):
    net = BrownianBridgeModel(bb_namespace(unet(width)))
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(fill_state_dict(shapes, seed=1234))
    net = net.cuda()
    x = synth_images((batch, 3, 64, 64), 11).cuda()
    y = synth_images((batch, 3, 64, 64), 12).cuda()
    t = torch.randint(0, 1000, (batch,), generator=torch.Generator().manual_seed(5)).cuda()
    res = {}
    net.eval()
    eng = UNetEngine(net.denoise_fn, backend=be)
    out = torch.empty_like(x)
    res["sample_eager_ms"] = timed(lambda: eng.forward(x, t, out=out), steps, warmup)
    eng.refresh_weights()
    fwd = lambda: eng.forward(x, t, assume_fresh_weights=True, out=out)
    for _ in range(2):
        fwd()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fwd()
    res["sample_graph_ms"] = timed(g.replay, steps, warmup)
    del g, eng
    net.train()
    old = train._BACKEND
    train.set_backend(be)
    nz = torch.randn_like(x)
    opt = torch.optim.SGD(net.denoise_fn.parameters(), lr=0.0)

    def step():
        opt.zero_grad(set_to_none=True)
        loss, _ = net.p_losses(x, y, None, t, nz)
        loss.backward()
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            res["train_step_ms"] = timed(step, steps, warmup)
    finally:
        train.set_backend(old)
    del net, opt
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", default="224,96,160")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    print(f"card: {card()}")
    for w in (int(s) for s in a.widths.split(",")):
        for name, be in (("multiple of 32", cabi.CudaBackend()), ("64 rule", Rule64Backend())):
            r = run(w, be, a.batch, a.steps, a.warmup)
            print(f"model_channels {w}, batch {a.batch}, {name}: " + ", ".join(f"{k} {v:.2f}" for k, v in r.items()),
                  flush=True)


if __name__ == "__main__":
    main()
