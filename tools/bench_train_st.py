#!/usr/bin/env python
"""Training micro-step (q_sample + UNet forward + L1 loss + backward + FusedAdam) of a cross-attention-conditioned
BBDM, with the SpatialTransformer on the native kernels (``native``) and with the whole graph on stock PyTorch
kernels (``stock``, ``NATIVE_TRAIN_CONV = False``, fp32, TF32 off).  Prints the ms per micro-step and
``torch.cuda.max_memory_allocated()`` of both as one JSON line.

Config: the LBBDM-f4 UNet of bench.py's cfg3 (latent 64x64x3, batch 32) with ``use_spatial_transformer=True,
context_dim=3, condition_key="SpatialRescaler"`` (so in_channels 6: the latent and its 3-channel context).  With
attention_resolutions (32, 16, 8) read as downsample rates, as the reference UNet does, the one transformer is the
middle block's: 1024 channels, 16 heads of 64, 16x16 queries attending over the 4096 context pixels.  The model is
BrownianBridgeModel on latent-shaped tensors with y as the context (what the latent model's SpatialRescaler stage
hands the UNet, without the VQGAN encode).  A third arm, ``native_st_stock``, runs every other layer natively and only
the transformer on its stock graph, to attribute the difference to the transformer.

    python tools/bench_train_st.py [--steps 10] [--warmup 3] [--batch 32]
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import bbdm_b200.unet as U  # noqa: E402
from bbdm_b200.optim import FusedAdam  # noqa: E402
from bbdm_b200.transformer import SpatialTransformer  # noqa: E402
from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel  # noqa: E402

UNET = dict(bench.CONFIGS["cfg3"]["unet"], in_channels=6, use_spatial_transformer=True, context_dim=3,
            condition_key="SpatialRescaler")


def run(mode, B, steps, warmup):
    U.NATIVE_TRAIN_CONV = mode != "stock"
    st_native_ok = SpatialTransformer._native_ok
    if mode == "native_st_stock":
        SpatialTransformer._native_ok = lambda self, x, context: False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    net = BrownianBridgeModel(bench.namespace(UNET, 200)).train()
    bench.init_weights(net.denoise_fn)
    net = net.cuda()
    x, y = bench.synth((B, 3, 64, 64), 1).cuda(), bench.synth((B, 3, 64, 64), 2).cuda()
    opt = FusedAdam(net.get_parameters(), lr=1e-4)

    def step():
        opt.zero_grad(set_to_none=True)
        loss, _ = net(x, y)
        loss.backward()
        opt.step()
        return loss

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    SpatialTransformer._native_ok = st_native_ok
    return {"mode": mode, "ms_per_micro_step": e0.elapsed_time(e1) / steps,
            "max_mem_gb": torch.cuda.max_memory_allocated() / 1e9, "loss": float(loss.detach())}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_train_st needs a CUDA device"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    warnings.simplefilter("ignore")                    # the native_st_stock arm's library-path warnings
    rows = []
    for mode in ("native", "stock", "native_st_stock") * 2:    # alternated: the spread between repeats shows the noise
        gc.collect()
        torch.cuda.empty_cache()
        rows.append(run(mode, a.batch, a.steps, a.warmup))
    print(json.dumps({"config": f"LBBDM-f4 UNet + SpatialTransformer (context_dim 3), latent 64x64x3, batch {a.batch}",
                      "gpu": gpu, "what": "training micro-step incl. FusedAdam", "rows": rows}))
