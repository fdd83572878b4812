#!/usr/bin/env python
"""Eager against CUDA-graph-replayed training steps (UNetModel.train_graph, bbdm_b200/train_graph.py) at the UNet shapes
of the reference's training templates.  A step is q_sample + the UNet forward + L1 loss + backward + FusedAdam; the
VQGAN encodes of the latent models are not part of it (the latents are synthetic).

    python tools/bench_train_graph.py [--shapes f16,f8,f4,cfg2] [--steps 20] [--warmup 3] [--profile] [--checkpoint]
                                      [--whole-recompute] [--out FILE]

Per shape and mode: ms/step (host clock around --steps steps that end in a device synchronise), peak allocated and
reserved memory, and
whether the two modes' losses agree bit for bit over three steps from the same weights and seeds.  --checkpoint trains
with UNetModel.use_checkpoint on (every block recomputed in the backward); --whole-recompute recomputes the whole block
(train.RECOMPUTE_TRIM = False).  --profile adds, for
each mode, the summed device time of the kernels of one step (torch.profiler) -- set against the step time it says how
much of an eager step the GPU is idle, waiting for the host.  The card name, power limit and SM clocks of the run are
recorded with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel  # noqa: E402


def _unet(size, ch, attn, cond):
    """The template UNet (model_channels 128, channel_mult 1/4/8, two ResBlocks per level, 64-channel heads)."""
    return dict(image_size=size, in_channels=ch * (2 if cond else 1), model_channels=128, out_channels=ch,
                num_res_blocks=2, attention_resolutions=attn, channel_mult=(1, 4, 8), conv_resample=True, dims=2,
                num_heads=8, num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True,
                use_spatial_transformer=False, context_dim=None, condition_key="SpatialRescaler" if cond else "nocond")


# name -> (UNet, batch, channels of x / y, map size); configs/Template-LBBDM-f16/f8/f4.yaml and Template-BBDM.yaml
SHAPES = {
    "f16": (_unet(16, 8, (16, 8, 4), False), 8, 8, 16),
    "f8": (_unet(32, 4, (32, 16, 8), False), 8, 4, 32),
    "f4": (_unet(64, 3, (32, 16, 8), False), 8, 3, 64),
    "cfg2": (_unet(256, 3, (32, 16, 8), True), 8, 3, 256),
}


def _model(unet, graph, dev, checkpoint=False):
    torch.manual_seed(0)              # the constructor's own initialisation (biases, GroupNorm) as well as the weights
    net = BrownianBridgeModel(bench.namespace(unet, 200)).train()
    bench.init_weights(net.denoise_fn)
    net = net.to(dev)
    net.denoise_fn.train_graph = graph
    net.denoise_fn.use_checkpoint = checkpoint
    from bbdm_b200.optim import FusedAdam
    return net, FusedAdam(net.get_parameters(), lr=1e-4)


def _step(net, opt, x, y):
    opt.zero_grad(set_to_none=True)
    loss, _ = net(x, y)
    loss.backward()
    opt.step()
    return loss


def _kernel_ms(net, opt, x, y, dev):
    """Summed device time of the kernels (and device-side copies) one step issues."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        _step(net, opt, x, y)
        torch.cuda.synchronize(dev)
    tot = 0.0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            tot += e.device_time if hasattr(e, "device_time") else e.cuda_time
    return tot / 1000.0


def run_shape(name, steps, warmup, profile, dev, checkpoint=False):
    unet, B, C, S = SHAPES[name]
    x = bench.synth((B, C, S, S), 1).to(dev)
    y = bench.synth((B, C, S, S), 2).to(dev)
    from bbdm_b200 import train_graph
    from bbdm_b200 import train
    row = {"shape": name, "batch": B, "map": S, "channels": C, "use_checkpoint": checkpoint,
           "recompute_trim": train.RECOMPUTE_TRIM}
    losses = {}
    for mode, graph in (("eager", False), ("graph", True)):
        net, opt = _model(unet, graph, dev, checkpoint)
        # the parity check first: three steps from the initial weights under fixed seeds
        ls = []
        for s in range(3):
            torch.manual_seed(100 + s)
            ls.append(_step(net, opt, x, y).detach().clone())
        losses[mode] = torch.stack(ls)
        n_cap = train_graph.CAPTURES["n"]
        for _ in range(warmup):
            _step(net, opt, x, y)
        torch.cuda.synchronize(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        t0 = time.perf_counter()
        for _ in range(steps):
            _step(net, opt, x, y)
        torch.cuda.synchronize(dev)
        ms = (time.perf_counter() - t0) * 1000.0 / steps
        # reserved, not allocated: the graph's private pool holds its activations as cached (reserved) blocks
        row[mode] = {"ms_per_step": round(ms, 3), "peak_allocated_gb": round(torch.cuda.max_memory_allocated(dev) / 2**30, 3),
                     "peak_reserved_gb": round(torch.cuda.max_memory_reserved(dev) / 2**30, 3),
                     "captures_in_timed_window": train_graph.CAPTURES["n"] - n_cap}
        if profile:
            row[mode]["kernel_ms_per_step"] = round(_kernel_ms(net, opt, x, y, dev), 3)
        train_graph.release(net.denoise_fn)
        del net, opt
        torch.cuda.empty_cache()
    row["losses_bit_identical"] = bool(torch.equal(losses["eager"], losses["graph"]))
    row["speedup"] = round(row["eager"]["ms_per_step"] / row["graph"]["ms_per_step"], 3)
    return row


def gpu_info():
    try:
        q = "name,power.limit,clocks.sm,clocks.max.sm"
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "nvidia-smi: no output"
    except Exception as e:  # pragma: no cover - reported, not fatal
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="f16,f8,f4,cfg2")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--checkpoint", action="store_true")
    ap.add_argument("--whole-recompute", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_train_graph: needs a CUDA device")
    dev = torch.device("cuda", 0)
    from bbdm_b200 import train
    train.RECOMPUTE_TRIM = not a.whole_recompute
    rows = {"gpu_before": gpu_info(), "rows": []}
    for name in a.shapes.split(","):
        r = run_shape(name, a.steps, a.warmup, a.profile, dev, a.checkpoint)
        print(json.dumps(r), flush=True)
        rows["rows"].append(r)
    rows["gpu_after"] = gpu_info()
    print(json.dumps({"gpu_before": rows["gpu_before"], "gpu_after": rows["gpu_after"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
