"""Attention heads wider than 128 channels (multiples of 8 up to 256) on CPU: the backend-declared head-size rule, the
oracle against the reference-generated fixtures, the sampling engine's wiring and the training Functions' routing
through the oracle-backed emulation with CudaBackend's limit (tests/_emu_backend_wide.py), and the unchanged 128 rule
on a backend that declares no limit.  The kernels are checked by the -m gpu suite
(tests/test_gpu_attention_wide_heads.py)."""
import pytest
import torch

from _emu_backend import EmuBackend
from _emu_backend_wide import EmuBackendWide
from _recipe import rel_dev
from _wide_heads import WIDE_HEAD_CONFIGS, WIDE_HEAD_DIMS
from bbdm_b200 import cabi
from bbdm_b200.engine import UNetEngine
from bbdm_b200.unet import UNetModel
from oracle import bbdm_oracle as O
from test_attention_head_dims_host import _fill, _train_pair, build, load

TAGS = list(WIDE_HEAD_CONFIGS)


def test_wide_head_dim_rule():
    """CudaBackend and the wide emulation take every multiple of 8 up to 256; a backend that declares no limit keeps
    the 128 rule (cabi.attn_head_dim_ok and its text)."""
    for be in (cabi.CudaBackend, EmuBackendWide()):
        ok, rule = cabi.attn_head_dims(be)
        assert [d for d in range(513) if ok(d)] == list(range(8, 257, 8))
        assert rule == "multiples of 8 up to 256"
    ok, rule = cabi.attn_head_dims(EmuBackend())
    assert [d for d in range(513) if ok(d)] == [d for d in range(513) if cabi.attn_head_dim_ok(d)]
    assert rule == cabi.ATTN_HEAD_DIM_RULE
    assert cabi.ATTN_TC_HEAD_DIMS == (64, 128)


def test_configs_have_the_head_dims():
    for tag in TAGS:
        net = UNetModel(**WIDE_HEAD_CONFIGS[tag])
        dims = {m.d_head if hasattr(m, "d_head") else m.channels // m.num_heads
                for m in net.modules() if type(m).__name__ in ("AttentionBlock", "SpatialTransformer")}
        assert dims == {WIDE_HEAD_DIMS[tag]}, (tag, dims)
        chans = {m.num_channels for m in net.modules() if isinstance(m, torch.nn.GroupNorm)}
        assert all(c % 32 == 0 for c in chans), (tag, chans)


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_matches_wide_head_reference_fixture(tag):
    g = load(tag)
    cfg = O.unet_cfg(**WIDE_HEAD_CONFIGS[tag])
    sd = build(WIDE_HEAD_CONFIGS[tag]).state_dict()
    bufs, steps = O.make_schedule()
    x, y, t = g["x"], g["y"], g["t"]
    assert rel_dev(O.unet_forward(sd, cfg, x, t, y), g["unet_out"]) < 2e-6
    for i in g["ps_ids"].tolist():
        o, _ = O.p_sample(sd, cfg, bufs, steps, i, g[f"ps{i}_xt"], y, y, g[f"ps{i}_noise"], prefix="")
        assert rel_dev(o, g[f"ps{i}_out"]) < 2e-6


@pytest.mark.parametrize("tag", TAGS)
def test_engine_wiring_matches_wide_head_reference_fixture(tag):
    """On a backend that declares attn_max_head_dim = 256 the engine runs these sizes on the mma.sync kernel
    (attention_split; cross-attention: attention_cross), never on the wgmma one."""
    g = {k: v for k, v in load(tag).items() if isinstance(v, torch.Tensor)}
    be = EmuBackendWide()
    eng = UNetEngine(build(WIDE_HEAD_CONFIGS[tag]), backend=be)
    out = eng.forward(g["x"], g["t"], g["y"])
    assert out.shape == g["unet_out"].shape and not torch.isnan(out).any()
    assert rel_dev(out, g["unet_out"]) < 6e-5
    assert "attention_split" in be.calls and "attention_tc" not in be.calls
    if "_st_" in tag:
        assert "attention_cross" in be.calls


@pytest.mark.parametrize("tag", TAGS)
def test_base_emulation_still_rejects_wide_heads(tag):
    """The same model on a backend that declares no limit raises on the first sampling forward with the 128 rule."""
    g = {k: v for k, v in load(tag).items() if isinstance(v, torch.Tensor)}
    eng = UNetEngine(build(WIDE_HEAD_CONFIGS[tag]), backend=EmuBackend())
    d = WIDE_HEAD_DIMS[tag]
    with pytest.raises(NotImplementedError, match=f"head_dim {d}: .*multiples of 8 up to 128"):
        eng.forward(g["x"], g["t"], g["y"])


@pytest.mark.parametrize("d,heads", [(288, 1), (512, 1)])
def test_engine_rejects_head_dims_outside_the_wide_rule(d, heads):
    """Heads wider than 256 still raise on the wide backend, naming its rule."""
    cfg = dict(WIDE_HEAD_CONFIGS["mid_hd256"], model_channels=d * heads, channel_mult=(1, 1, 1), num_heads=heads)
    eng = UNetEngine(build(cfg), backend=EmuBackendWide())
    x = torch.zeros(1, cfg["out_channels"], 32, 32)
    with pytest.raises(NotImplementedError, match=f"head_dim {d}: .*multiples of 8 up to 256"):
        eng.forward(x, torch.zeros(1, dtype=torch.long), torch.zeros(1, 3, 32, 32))


def _attention_block(channels, heads, new_order, seed):
    import bbdm_b200.unet as U
    blk = U.AttentionBlock(channels, num_heads=heads, use_new_attention_order=new_order)
    gen = _fill(blk, seed)
    with torch.no_grad():
        blk.norm.weight.add_(1.0)
    x = torch.randn((2, channels, 8, 8), generator=gen)
    gy = 0.2 * torch.randn((2, channels, 8, 8), generator=gen)
    return blk, x, gy


@pytest.mark.parametrize("channels,heads,new_order", [(256, 1, False), (544, 4, False), (544, 4, True)])
def test_attention_block_wide_heads_train_through_native_functions(channels, heads, new_order):
    """AttentionBlock with heads of 256 or 136: AttentionCoreFn (fp32-qkv mma.sync forward, flash backward) on the wide
    backend, matching the stock-PyTorch graph of the same block."""
    blk, x, gy = _attention_block(channels, heads, new_order, 43)
    res = _train_pair(blk, x, gy, EmuBackendWide())
    assert {"attention", "attention_bwd"} <= res[True][3] and "attention_tc" not in res[True][3]
    assert not res[False][3] & {"attention", "attention_bwd"}
    assert rel_dev(res[True][0], res[False][0]) < 3e-5
    assert rel_dev(res[True][1], res[False][1]) < 1e-4
    for n in res[False][2]:
        assert rel_dev(res[True][2][n], res[False][2][n]) < 1e-4, n


def test_attention_block_wide_heads_take_the_stock_core_without_a_declared_limit():
    """On a backend that declares no limit, a 256-wide head keeps training on the stock attention core."""
    blk, x, gy = _attention_block(256, 1, False, 44)
    res = _train_pair(blk, x, gy, EmuBackend())
    assert not res[True][3] & {"attention", "attention_split", "attention_tc", "attention_bwd"}
    assert rel_dev(res[True][1], res[False][1]) < 1e-4


def test_transformer_dhead160_trains_through_native_functions():
    """SpatialTransformer(320, 2 heads of 160, context): self- and cross-attention run the native Functions
    (attention / attention_bwd, attention_cross / attention_cross_bwd) and match the stock graph."""
    from bbdm_b200.transformer import SpatialTransformer
    m = SpatialTransformer(320, 2, 160, context_dim=3)
    gen = _fill(m, 45)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, (torch.nn.LayerNorm, torch.nn.GroupNorm)):
                mod.weight.add_(1.0)
    x = torch.randn((2, 320, 8, 8), generator=gen)
    ctx = torch.randn((2, 3, 8, 8), generator=gen)
    gy = 0.2 * torch.randn((2, 320, 8, 8), generator=gen)
    res = _train_pair(m, x, gy, EmuBackendWide(), ctx)
    assert {"attention_bwd", "attention_cross", "attention_cross_bwd"} <= res[True][3]
    assert "attention_tc" not in res[True][3]
    assert not res[False][3]
    assert rel_dev(res[True][0], res[False][0]) < 3e-5
    assert rel_dev(res[True][1], res[False][1]) < 1e-4
    for n in res[False][2]:
        assert rel_dev(res[True][2][n], res[False][2][n]) < 1e-4, n
