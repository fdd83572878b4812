#!/usr/bin/env python
"""Generate attention_mma.npz: outputs of the three mma.sync attention entry points (bbdm_attention on fp32 qkv,
bbdm_attention_split and bbdm_attention_cross on split bf16 planes) on seeded inputs, for a bit-for-bit replay by
test_gpu_kernels.py::test_attention_mma_bit_pinned.

    BBDM_LIB=<libbbdm_b200.so built from the commit to pin> python tests/golden/make_golden_attention_mma.py

Needs an H100.  The inputs are not stored: every case regenerates them from its seed on the CPU (inputs() below).
The cases cover head_dim 16/32/64/128, both qkv channel orders, query and key counts 1 / 100 / 257 (one partial
tile; one and three 128-query CTAs), a one-head C = 64 case like the VQGAN AttnBlocks, and fp32-only, hi/lo-only and
both output forms."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "attention_mma.npz")
# kind, head_dim, heads, order, T (cross-attention: query and key counts), outputs.  Two heads where the qkv channel
# orders must differ; the head_dim 64 / 128 cases with many rows run one head, which keeps the file small.
_TABLE = [
    ("attention", 16, 2, 0, 257, "f32"), ("attention", 16, 2, 1, 100, "hilo"),
    ("attention", 32, 2, 0, 100, "f32"), ("attention", 32, 2, 1, 1, "both"),
    ("attention", 64, 2, 0, 1, "both"), ("attention", 64, 2, 1, 1, "both"),
    ("attention", 64, 1, 1, 100, "hilo"),                                             # VQGAN AttnBlock, C = 64
    ("attention", 128, 2, 0, 1, "both"), ("attention", 128, 1, 1, 257, "f32"),
    ("attention_split", 16, 2, 0, 1, "both"), ("attention_split", 16, 2, 1, 257, "hilo"),
    ("attention_split", 32, 2, 0, 100, "f32"), ("attention_split", 32, 2, 1, 1, "both"),
    ("attention_split", 64, 1, 0, 100, "hilo"), ("attention_split", 64, 2, 1, 1, "both"),
    ("attention_split", 128, 2, 0, 1, "both"), ("attention_split", 128, 1, 1, 100, "f32"),
    ("attention_cross", 16, 2, None, (257, 100), "hilo"), ("attention_cross", 32, 2, None, (100, 1), "f32"),
    ("attention_cross", 64, 2, None, (1, 257), "both"), ("attention_cross", 128, 2, None, (1, 257), "f32"),
]


def _cases():
    cases = []
    for kind, D, heads, order, T, outs in _TABLE:
        c = dict(kind=kind, D=D, heads=heads, T=T, outs=outs, seed=100 + len(cases))
        if kind == "attention_cross":
            c["T"], c["Tkv"] = T
        else:
            c["order"] = order
        cases.append(c)
    return cases


CASES = _cases()


def _planes(x):
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def inputs(case):
    """CPU tensors of one case: (qkv,) fp32 for attention, (hi, lo) for attention_split, (q_hi, q_lo, kv_hi, kv_lo)
    for attention_cross."""
    g = torch.Generator().manual_seed(case["seed"])
    C = case["heads"] * case["D"]
    if case["kind"] == "attention_cross":
        q = 1.2 * torch.randn(1, case["T"], C, generator=g)
        kv = 1.2 * torch.randn(1, case["Tkv"], 2 * C, generator=g)
        return (*_planes(q), *_planes(kv))
    qkv = 1.2 * torch.randn(1, case["T"], 3 * C, generator=g)
    return (qkv,) if case["kind"] == "attention" else _planes(qkv)


def run(be, case):
    """Run one case on the GPU; returns the requested outputs as CPU tensors keyed 'f32', 'hi', 'lo'."""
    xs = [x.cuda() for x in inputs(case)]
    shape = (1, case["T"], case["heads"] * case["D"])
    out = torch.full(shape, float("nan"), device="cuda") if case["outs"] != "hilo" else None
    oh = torch.zeros(shape, dtype=torch.bfloat16, device="cuda") if case["outs"] != "f32" else None
    ol = torch.zeros_like(oh) if oh is not None else None
    if case["kind"] == "attention_cross":
        be.attention_cross(*xs, case["heads"], out_f32=out, out_hi=oh, out_lo=ol)
    else:
        getattr(be, case["kind"])(*xs, case["heads"], case["order"], out_f32=out, out_hi=oh, out_lo=ol)
    torch.cuda.synchronize()
    res = {} if out is None else {"f32": out.cpu()}
    if oh is not None:
        res.update(hi=oh.cpu(), lo=ol.cpu())
    return res


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from bbdm_b200 import cabi
    be = cabi.CudaBackend()
    arrays = {"cases": np.array(json.dumps(CASES))}
    for i, case in enumerate(CASES):
        for k, v in run(be, case).items():
            arrays[f"{i}_{k}"] = (v.view(torch.int16) if v.dtype == torch.bfloat16 else v).numpy()
    be.check_fault()
    np.savez(OUT, **arrays)
    print(f"wrote {OUT}: {len(CASES)} cases, {os.path.getsize(OUT)} bytes, from {cabi.LIB_PATH}")
