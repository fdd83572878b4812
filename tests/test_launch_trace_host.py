"""Every kernel launch the UNet and VQGAN executors and the training Functions issue, pinned.

A recorder wraps the oracle-backed emulation backend (tests/_emu_backend.py) and logs each launching call: the method
name and every argument bound to the method's signature (defaults filled in).  Tensors are logged as (shape, dtype,
stride, slot, storage offset), where slot numbers the distinct storages in order of first appearance; the recorder
keeps every logged tensor alive, so a freed address cannot come back as another tensor.  The slots therefore pin the
buffer pools' reuse pattern, which CUDA-graph replay depends on, and not only the launch sequence.

tests/golden/launch_traces.json holds the sha256, the call count and the per-method counts of each scenario's trace,
recorded from the executors before they were moved onto the shared code in bbdm_b200/convs.py; vqgan_vq_small and
vqgan_vq_tc_winograd were re-recorded when the VQGAN's ResnetBlocks moved onto the UNet's ResBlock flow (a raw fp32
input copy for an unfused 1x1 shortcut; the skip GEMM after conv2's GroupNorm statistics).  A change to the host code
that is meant to be a pure refactor must leave every trace unchanged.  On a mismatch the full trace is written to
the test's tmp_path, to be diffed against one dumped from the earlier code."""
import collections
import hashlib
import inspect
import json
import os

import numpy as np
import pytest
import torch

from _emu_backend import EmuBackend
from _hd128 import HD128_CONFIGS
from _recipe import UNET_CONFIGS, VQGAN_CONFIGS, fill_state_dict, vqgan_namespace, vqgan_state_dict

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FIXTURE = os.path.join(GOLD, "launch_traces.json")
NOT_LAUNCHES = {"empty", "conv_geometry", "wino_geometry", "wgrad_workspace", "optim_chunk_elems"}


class _Emu(EmuBackend):
    """The emulation with bbdm_attention_tc's head_dim 128 instance (the kernel takes 64 and 128)."""

    def attention_tc(self, qkv_hi, qkv_lo, heads, order, out_f32=None, out_hi=None, out_lo=None):
        self.calls.append("attention_tc")
        assert qkv_hi.shape[2] // 3 // heads in (64, 128)
        self.attention(self._planes(qkv_hi, qkv_lo), heads, order, out_f32, out_hi, out_lo)


class Recorder:
    def __init__(self):
        self.be = _Emu()
        self.trace, self._slots, self._alive = [], {}, []

    def _describe(self, v):
        if isinstance(v, torch.Tensor):
            key = v.untyped_storage().data_ptr()
            if key not in self._slots:
                self._slots[key] = len(self._slots)
            self._alive.append(v)
            return ["T", list(v.shape), str(v.dtype), list(v.stride()), self._slots[key], v.storage_offset()]
        if isinstance(v, bool) or v is None or isinstance(v, (int, str)):
            return v
        if isinstance(v, float):
            return float(f"{v:.12g}")
        if isinstance(v, (tuple, list)):
            return [self._describe(x) for x in v]
        return repr(v)

    def __getattr__(self, name):
        attr = getattr(self.be, name)
        if name in NOT_LAUNCHES or not callable(attr):
            return attr
        sig = inspect.signature(attr)

        def launch(*args, **kwargs):
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            self.trace.append([name, [[k, self._describe(v)] for k, v in bound.arguments.items()]])
            return attr(*args, **kwargs)
        return launch


def _golden(tag):
    return {k: torch.from_numpy(v) for k, v in np.load(os.path.join(GOLD, tag + ".npz")).items() if v.ndim}


def _unet(cfg, train=False):
    from bbdm_b200.unet import UNetModel
    net = UNetModel(**cfg)
    net.train(train)
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    net.load_state_dict(fill_state_dict(shapes, seed=1234))
    return net


def _unet_scenario(rec, tag, cfg, precision="split3", wino=None, refresh=False):
    from bbdm_b200.engine import UNetEngine
    g = _golden(tag)
    net = _unet(cfg)
    eng = UNetEngine(net, backend=rec, precision=precision)
    if wino is not None:
        eng.wino_min_c, eng.wino_min_tiles = wino
    ctx = None if net.condition_key == "nocond" else g["y"]
    for _ in range(2):
        eng.forward(g["x"], g["t"], ctx)
    if refresh:
        with torch.no_grad():
            for i, p in enumerate(net.parameters()):
                p.add_(1e-3 * (i % 7))                 # optimizer-style in-place update
        eng.refresh_weights()
        eng.forward(g["x"], g["t"], ctx)
        for p in net.parameters():
            p.data = p.data.clone()                    # EMA-style .data swap
        eng.refresh_weights()
        eng.forward(g["x"], g["t"], ctx)


def _vqgan_scenario(rec, name, wino=None):
    from bbdm_b200.vqgan import VQModel
    from bbdm_b200.vqgan_engine import VQGANEngine
    g = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}
    vq = VQModel(**vqgan_namespace(VQGAN_CONFIGS[name])).eval()
    vq.load_state_dict(vqgan_state_dict({k: tuple(v.shape) for k, v in vq.state_dict().items()}), strict=True)
    eng = VQGANEngine(vq, backend=rec)
    if wino is not None:
        eng.wino_min_c, eng.wino_min_tiles = wino
    eng.encode(g["x"], quant_conv=True)
    eng.decode(g["lat"], return_indices=True)


def _train_scenario(rec, monkeypatch, wino):
    import bbdm_b200.unet as U
    from bbdm_b200 import train
    if wino:
        monkeypatch.setattr(train, "WINO_MIN_C", 64)
        monkeypatch.setattr(train, "WINO_MIN_TILES", 16)
    g = _golden("mid_pixel")
    net = _unet(UNET_CONFIGS["mid_pixel"], train=True)
    monkeypatch.setattr(U, "NATIVE_TRAIN_CONV", True)
    train.set_backend(rec)
    try:
        out = net(g["x"], timesteps=g["t"], context=g["y"])
        gy = 1e-3 * torch.randn(out.shape, generator=torch.Generator().manual_seed(7))
        out.backward(gy)
    finally:
        train.set_backend(None)


SCENARIOS = {
    **{f"unet_{t}": (lambda rec, mp, t=t: _unet_scenario(rec, t, UNET_CONFIGS[t]))
       for t in ("tiny_pixel", "tiny_latent", "tiny_variant", "mid_pixel", "tiny_st")},
    "unet_mid_hd128": lambda rec, mp: _unet_scenario(rec, "mid_hd128", HD128_CONFIGS["mid_hd128"]),
    "unet_mid_pixel_winograd": lambda rec, mp: _unet_scenario(rec, "mid_pixel", UNET_CONFIGS["mid_pixel"], wino=(64, 128)),
    "unet_mid_pixel_bf16": lambda rec, mp: _unet_scenario(rec, "mid_pixel", UNET_CONFIGS["mid_pixel"], precision="bf16"),
    "unet_mid_pixel_refresh": lambda rec, mp: _unet_scenario(rec, "mid_pixel", UNET_CONFIGS["mid_pixel"], wino=(64, 128),
                                                             refresh=True),
    **{f"vqgan_{n}": (lambda rec, mp, n=n: _vqgan_scenario(rec, n)) for n in VQGAN_CONFIGS},
    "vqgan_vq_tc_winograd": lambda rec, mp: _vqgan_scenario(rec, "vq_tc", wino=(64, 32)),
    "train_mid_pixel": lambda rec, mp: _train_scenario(rec, mp, wino=False),
    "train_mid_pixel_winograd": lambda rec, mp: _train_scenario(rec, mp, wino=True),
}


def record(name, monkeypatch):
    torch.manual_seed(0)
    rec = Recorder()
    SCENARIOS[name](rec, monkeypatch)
    text = json.dumps(rec.trace, separators=(",", ":"))
    counts = collections.Counter(c[0] for c in rec.trace)
    return rec.trace, {"sha256": hashlib.sha256(text.encode()).hexdigest(), "calls": len(rec.trace),
                       "methods": dict(sorted(counts.items()))}


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_launch_trace_unchanged(name, monkeypatch, tmp_path):
    with open(FIXTURE) as f:
        want = json.load(f)[name]
    trace, got = record(name, monkeypatch)
    if got != want:
        path = tmp_path / f"{name}.trace.json"
        path.write_text("\n".join(json.dumps(c) for c in trace) + "\n")
        pytest.fail(f"{name}: launch trace changed (full trace in {path}): "
                    f"calls {got['calls']} vs {want['calls']}, methods {got['methods']} vs {want['methods']}")
