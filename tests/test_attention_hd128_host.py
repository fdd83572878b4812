"""Attention head_dim 128 (heads sized by num_heads, the reference UNetModel's default num_head_channels=-1) on CPU:
the oracle against the reference-generated fixtures, the sampling engine's wiring and the training Function's routing
through the oracle-backed backend emulation (tests/_emu_backend.py).  The kernels are checked by the -m gpu suite."""
import os

import numpy as np
import pytest
import torch

from _emu_backend import EmuBackend as _EmuBackend
from _hd128 import HD128_CONFIGS
from _recipe import fill_state_dict, rel_dev
from bbdm_b200.engine import UNetEngine
from bbdm_b200.unet import UNetModel
from oracle import bbdm_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TAGS = ["mid_hd128", "mid_st_hd128"]


class EmuBackend(_EmuBackend):
    """The emulation backend with bbdm_attention_tc's head_dim 128 instance (the kernel takes 64 and 128)."""

    def attention_tc(self, qkv_hi, qkv_lo, heads, order, out_f32=None, out_hi=None, out_lo=None):
        self.calls.append("attention_tc")
        assert qkv_hi.shape[2] // 3 // heads in (64, 128)
        self.attention(self._planes(qkv_hi, qkv_lo), heads, order, out_f32, out_hi, out_lo)


def build(cfg):
    net = UNetModel(**cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    net.load_state_dict(fill_state_dict(shapes, seed=1234))
    return net


def load(tag):
    return {k: torch.from_numpy(v) if v.ndim else v for k, v in np.load(os.path.join(GOLD, tag + ".npz")).items()}


def test_configs_have_head_dim_128():
    for tag in TAGS:
        net = UNetModel(**HD128_CONFIGS[tag])
        dims = {m.d_head if hasattr(m, "d_head") else m.channels // m.num_heads
                for m in net.modules() if type(m).__name__ in ("AttentionBlock", "SpatialTransformer")}
        assert dims == {128}, (tag, dims)


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_matches_hd128_reference_fixture(tag):
    """The oracle's attention at head_dim 128 (AttentionBlock, and SpatialTransformer self- and cross-attention)
    against the fixture of the unmodified reference."""
    g = load(tag)
    cfg = O.unet_cfg(**HD128_CONFIGS[tag])
    sd = build(HD128_CONFIGS[tag]).state_dict()
    bufs, steps = O.make_schedule()
    x, y, t = g["x"], g["y"], g["t"]
    assert rel_dev(O.unet_forward(sd, cfg, x, t, y), g["unet_out"]) < 2e-6
    for i in g["ps_ids"].tolist():
        o, _ = O.p_sample(sd, cfg, bufs, steps, i, g[f"ps{i}_xt"], y, y, g[f"ps{i}_noise"], prefix="")
        assert rel_dev(o, g[f"ps{i}_out"]) < 2e-6


@pytest.mark.parametrize("tag", TAGS)
def test_engine_wiring_hd128_matches_reference_fixture(tag):
    g = {k: v for k, v in load(tag).items() if isinstance(v, torch.Tensor)}
    net = build(HD128_CONFIGS[tag])
    be = EmuBackend()
    eng = UNetEngine(net, backend=be)
    out = eng.forward(g["x"], g["t"], g["y"])
    assert out.shape == g["unet_out"].shape and not torch.isnan(out).any()
    assert rel_dev(out, g["unet_out"]) < 6e-5
    assert "attention_tc" in be.calls and "attention_split" not in be.calls
    if tag == "mid_st_hd128":
        assert "attention_cross" in be.calls
    pool = eng._pool(g["x"].device, tuple(g["x"].shape[i] for i in (0, 2, 3)))
    nbytes = pool.bytes
    out2 = eng.forward(g["x"], g["t"], g["y"])
    assert pool.bytes == nbytes
    assert torch.equal(out, out2)


@pytest.mark.parametrize("tag", TAGS)
def test_engine_rejects_head_dim_256(tag):
    cfg = dict(HD128_CONFIGS[tag], num_heads=1)            # 256 channels / 1 head
    eng = UNetEngine(build(cfg), backend=EmuBackend())
    x = torch.zeros(1, cfg["out_channels"], 32, 32)       # concatenated with the 3-channel condition
    with pytest.raises(NotImplementedError, match="head_dim 256.*128"):
        eng.forward(x, torch.zeros(1, dtype=torch.long), torch.zeros(1, 3, 32, 32))


def test_attention_block_hd128_training_routes_through_native_function():
    """AttentionBlock(256, num_heads=2) training step: the attention core runs AttentionCoreFn (attention_tc forward,
    attention_bwd backward), and matches the stock-PyTorch graph of the same block."""
    import bbdm_b200.unet as U
    from bbdm_b200 import train
    be = EmuBackend()
    train.set_backend(be)
    try:
        blk = U.AttentionBlock(256, num_heads=2)
        gen = torch.Generator().manual_seed(40)
        with torch.no_grad():
            for p_ in blk.parameters():
                p_.copy_(0.05 * torch.randn(p_.shape, generator=gen))
            blk.norm.weight.add_(1.0)
        x = torch.randn((2, 256, 8, 8), generator=gen)
        gy = 0.2 * torch.randn((2, 256, 8, 8), generator=gen)
        res = {}
        for native in (True, False):
            U.NATIVE_TRAIN_CONV = native
            be.calls.clear()
            blk.zero_grad(set_to_none=True)
            xi = x.clone().requires_grad_(True)
            y = blk(xi)
            y.backward(gy)
            res[native] = (y.detach(), xi.grad, {n: p_.grad.clone() for n, p_ in blk.named_parameters()}, set(be.calls))
    finally:
        U.NATIVE_TRAIN_CONV = True
        train.set_backend(None)
    assert {"attention_tc", "attention_bwd"} <= res[True][3]
    assert rel_dev(res[True][0], res[False][0]) < 3e-5
    assert rel_dev(res[True][1], res[False][1]) < 1e-4
    for n in res[False][2]:
        assert rel_dev(res[True][2][n], res[False][2][n]) < 1e-4, n
