#!/usr/bin/env python
"""Training micro-step (q_sample + UNet forward + L1 loss + backward) at the UNet shape of BASELINE
configs[2] (LBBDM-f4: latents [32,3,64,64] per rank, nocond) -- tensor-core conv autograd path
(bbdm_b200/train.py) vs the stock PyTorch graph in fp32 / TF32 / bf16-autocast.  VQGAN encodes are
outside this measurement (frozen reference module).

    python tools/bench_train.py cfg2 --size 224 --batch 8 --modes native,fp32,tf32 [--checkpoint]

--size / --batch train the config's UNet at another map size and batch (the FLOP count is scaled by pixels and batch).
--checkpoint sets UNetModel.use_checkpoint (every block recomputed in the backward); --whole-recompute with it recomputes
the whole block (train.RECOMPUTE_TRIM = False).  A mode that runs out of memory is reported as an error row.
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import bbdm_b200.unet as U  # noqa: E402
from bbdm_b200 import train  # noqa: E402
from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel  # noqa: E402


def run(mode, cfg, steps=3, warmup=2, ddp=False):
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    U.NATIVE_TRAIN_CONV = mode == "native"
    torch.backends.cudnn.allow_tf32 = mode == "tf32"
    torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
    torch.backends.cudnn.benchmark = True
    net = BrownianBridgeModel(bench.namespace(cfg["unet"], cfg["sample_step"])).train()
    bench.init_weights(net.denoise_fn)
    net.denoise_fn.use_checkpoint = "--checkpoint" in sys.argv
    train.RECOMPUTE_TRIM = "--whole-recompute" not in sys.argv
    net = net.to(dev)
    if mode == "bf16":
        net.denoise_fn.to(memory_format=torch.channels_last)
    B, C, S = cfg["batch"], cfg["channels"], cfg["size"]
    x = bench.synth((B, C, S, S), 1).to(dev)
    y = bench.synth((B, C, S, S), 2).to(dev)
    if mode == "native" and "--torch-adam" not in sys.argv:
        from bbdm_b200.optim import FusedAdam                      # one multi-tensor launch per optimizer step
        opt = FusedAdam(net.get_parameters(), lr=1e-4)
    else:
        opt = torch.optim.Adam(net.get_parameters(), lr=1e-4)
    model = net
    if ddp:      # exactly what runners/BaseRunner.py:76 does
        model = torch.nn.parallel.DistributedDataParallel(net, device_ids=[dev.index], output_device=dev.index)
        x = bench.synth((B, C, S, S), 10 + dev.index).to(dev)          # different data per rank

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "bf16"):
            loss, _ = model(x, y)
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
    ms = e0.elapsed_time(e1) / steps
    extra = {}
    if ddp:
        import torch.distributed as dist
        g = torch.cat([p.grad.flatten()[:1000] for p in net.get_parameters()][:20]).double()
        lo, hi = g.clone(), g.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        extra = {"ddp_world": dist.get_world_size(), "grads_identical_across_ranks": bool(torch.equal(lo, hi))}
    return {**extra, "mode": mode, "optimizer": type(opt).__name__, "use_checkpoint": net.denoise_fn.use_checkpoint,
            "recompute_trim": train.RECOMPUTE_TRIM,
            "ms_per_micro_step": ms, "micro_steps_per_s": 1e3 / ms, "loss": float(loss),
            "train_tflops_per_s": 3 * cfg["flops_per_step"] / ms / 1e9, "max_mem_gb": torch.cuda.max_memory_allocated() / 1e9,
            "max_reserved_gb": torch.cuda.max_memory_reserved() / 1e9}


def _arg(flag, default):
    return type(default)(sys.argv[sys.argv.index(flag) + 1]) if flag in sys.argv else default


def resized(cfg, size, batch):
    """cfg with the UNet trained at size x size, batch images (FLOPs scaled by the pixel count)."""
    f = (size / cfg["size"]) ** 2 * batch / cfg["batch"]
    return dict(cfg, unet=dict(cfg["unet"], image_size=size), size=size, batch=batch,
                flops_per_step=cfg["flops_per_step"] * f, name=f"{cfg['name']} -- trained at {size}x{size}, batch {batch}")


if __name__ == "__main__":
    name = sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith("--") else "cfg3"
    cfg = bench.CONFIGS[name]
    cfg = resized(cfg, _arg("--size", cfg["size"]), _arg("--batch", cfg["batch"]))
    if "--ddp" in sys.argv:
        import torch.distributed as dist
        dist.init_process_group("nccl")
        r = run("native", cfg, ddp=True)
        if dist.get_rank() == 0:
            print(json.dumps({"config": cfg["name"], "rows": [r]}))
        dist.barrier()
        dist.destroy_process_group()
        sys.exit(0)
    out = {"config": cfg["name"], "what": "UNet training micro-step incl. Adam; train_tflops = 3 x forward FLOPs / time", "rows": []}
    modes = ("native", "fp32", "tf32", "bf16")
    if "--modes" in sys.argv:
        modes = tuple(sys.argv[sys.argv.index("--modes") + 1].split(","))
    for mode in modes:
        try:
            out["rows"].append(run(mode, cfg))
        except Exception as e:  # noqa: BLE001
            out["rows"].append({"mode": mode, "error": repr(e)[:300]})
        torch.cuda.empty_cache()
    print(json.dumps(out))
