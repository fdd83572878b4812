"""Attention head sizes that are multiples of 8 but not 16/32/64/128 (heads sized by num_heads, the reference UNetModel's
default num_head_channels=-1) on CPU: the head-size rule, the oracle against the reference-generated fixtures, the
sampling engine's wiring and the training Functions' routing through the oracle-backed backend emulation
(tests/_emu_backend.py).  The kernels are checked by the -m gpu suite (tests/test_gpu_attention_head_dims.py)."""
import os

import numpy as np
import pytest
import torch

from _emu_backend import EmuBackend
from test_transformer_training_host import EmuBackend as TransformerEmuBackend
from _head_dims import HEAD_DIM_CONFIGS, HEAD_DIMS
from _recipe import fill_state_dict, rel_dev
from bbdm_b200 import cabi
from bbdm_b200.engine import UNetEngine
from bbdm_b200.unet import UNetModel
from oracle import bbdm_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TAGS = list(HEAD_DIM_CONFIGS)


def build(cfg):
    net = UNetModel(**cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    net.load_state_dict(fill_state_dict(shapes, seed=1234))
    return net


def load(tag):
    return {k: torch.from_numpy(v) if v.ndim else v for k, v in np.load(os.path.join(GOLD, tag + ".npz")).items()}


def test_head_dim_rule():
    assert [d for d in range(257) if cabi.attn_head_dim_ok(d)] == list(range(8, 129, 8))


@pytest.mark.parametrize("d,heads", [(4, 8), (12, 8), (20, 8), (136, 4), (256, 1)])
def test_engine_rejects_head_dims_outside_the_rule(d, heads):
    """A UNet whose attention heads are d wide raises on the first sampling forward, naming d and the rule."""
    assert not cabi.attn_head_dim_ok(d)
    cfg = dict(HEAD_DIM_CONFIGS["mid_hd96"], model_channels=d * heads, channel_mult=(1, 1, 1), num_heads=heads)
    eng = UNetEngine(build(cfg), backend=EmuBackend())
    x = torch.zeros(1, cfg["out_channels"], 32, 32)       # concatenated with the 3-channel condition
    with pytest.raises(NotImplementedError, match=f"head_dim {d}: .*multiples of 8 up to 128"):
        eng.forward(x, torch.zeros(1, dtype=torch.long), torch.zeros(1, 3, 32, 32))


def test_configs_have_the_head_dims():
    for tag in TAGS:
        net = UNetModel(**HEAD_DIM_CONFIGS[tag])
        dims = {m.d_head if hasattr(m, "d_head") else m.channels // m.num_heads
                for m in net.modules() if type(m).__name__ in ("AttentionBlock", "SpatialTransformer")}
        assert dims == {HEAD_DIMS[tag]}, (tag, dims)


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_matches_head_dim_reference_fixture(tag):
    g = load(tag)
    cfg = O.unet_cfg(**HEAD_DIM_CONFIGS[tag])
    sd = build(HEAD_DIM_CONFIGS[tag]).state_dict()
    bufs, steps = O.make_schedule()
    x, y, t = g["x"], g["y"], g["t"]
    assert rel_dev(O.unet_forward(sd, cfg, x, t, y), g["unet_out"]) < 2e-6
    for i in g["ps_ids"].tolist():
        o, _ = O.p_sample(sd, cfg, bufs, steps, i, g[f"ps{i}_xt"], y, y, g[f"ps{i}_noise"], prefix="")
        assert rel_dev(o, g[f"ps{i}_out"]) < 2e-6


@pytest.mark.parametrize("tag", TAGS)
def test_engine_wiring_matches_head_dim_reference_fixture(tag):
    """The engine runs these sizes on the mma.sync kernel (attention_split; cross-attention: attention_cross), never
    on the wgmma one."""
    g = {k: v for k, v in load(tag).items() if isinstance(v, torch.Tensor)}
    net = build(HEAD_DIM_CONFIGS[tag])
    be = EmuBackend()
    eng = UNetEngine(net, backend=be)
    out = eng.forward(g["x"], g["t"], g["y"])
    assert out.shape == g["unet_out"].shape and not torch.isnan(out).any()
    assert rel_dev(out, g["unet_out"]) < 6e-5
    assert "attention_split" in be.calls and "attention_tc" not in be.calls
    if "_st_" in tag:
        assert "attention_cross" in be.calls


def _train_pair(blk, x, gy, be, ctx=None):
    """(output, input grad, param grads, calls) of blk with the native training Functions and with the stock graph."""
    import bbdm_b200.unet as U
    from bbdm_b200 import train
    train.set_backend(be)
    res = {}
    try:
        for native in (True, False):
            U.NATIVE_TRAIN_CONV = native
            be.calls.clear()
            blk.zero_grad(set_to_none=True)
            xi = x.clone().requires_grad_(True)
            y = blk(xi) if ctx is None else blk(xi, ctx)
            y.backward(gy)
            res[native] = (y.detach(), xi.grad, {n: p_.grad.clone() for n, p_ in blk.named_parameters()}, set(be.calls))
    finally:
        U.NATIVE_TRAIN_CONV = True
        train.set_backend(None)
    return res


def _fill(blk, seed):
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p_ in blk.parameters():
            p_.copy_(0.05 * torch.randn(p_.shape, generator=gen))
    return gen


@pytest.mark.parametrize("new_order", [False, True])
def test_attention_block_hd48_trains_through_native_functions(new_order):
    """AttentionBlock(192, num_heads=4): head_dim 48 runs AttentionCoreFn (fp32-qkv mma.sync forward, flash backward)
    and matches the stock-PyTorch graph of the same block."""
    import bbdm_b200.unet as U
    blk = U.AttentionBlock(192, num_heads=4, use_new_attention_order=new_order)
    gen = _fill(blk, 41)
    with torch.no_grad():
        blk.norm.weight.add_(1.0)
    x = torch.randn((2, 192, 8, 8), generator=gen)
    gy = 0.2 * torch.randn((2, 192, 8, 8), generator=gen)
    res = _train_pair(blk, x, gy, EmuBackend())
    assert {"attention", "attention_bwd"} <= res[True][3] and "attention_tc" not in res[True][3]
    assert not res[False][3] & {"attention", "attention_bwd"}
    assert rel_dev(res[True][0], res[False][0]) < 3e-5
    assert rel_dev(res[True][1], res[False][1]) < 1e-4
    for n in res[False][2]:
        assert rel_dev(res[True][2][n], res[False][2][n]) < 1e-4, n


def test_transformer_dhead40_trains_through_native_functions():
    """SpatialTransformer(320, 8 heads of 40, context): self- and cross-attention run the native Functions
    (attention / attention_bwd, attention_cross / attention_cross_bwd) and match the stock graph."""
    from bbdm_b200.transformer import SpatialTransformer
    m = SpatialTransformer(320, 8, 40, context_dim=3)
    gen = _fill(m, 42)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, (torch.nn.LayerNorm, torch.nn.GroupNorm)):
                mod.weight.add_(1.0)
    x = torch.randn((2, 320, 8, 8), generator=gen)
    ctx = torch.randn((2, 3, 8, 8), generator=gen)
    gy = 0.2 * torch.randn((2, 320, 8, 8), generator=gen)
    res = _train_pair(m, x, gy, TransformerEmuBackend(), ctx)
    assert {"attention_bwd", "attention_cross", "attention_cross_bwd"} <= res[True][3]
    assert not res[False][3]
    assert rel_dev(res[True][0], res[False][0]) < 3e-5
    assert rel_dev(res[True][1], res[False][1]) < 1e-4
    for n in res[False][2]:
        assert rel_dev(res[True][2][n], res[False][2][n]) < 1e-4, n
