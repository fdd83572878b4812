"""Attention heads whose width is not a multiple of 8 on CPU: the padded-head route's predicate, the repack reference
at both qkv orders, the sampling engine's wiring against reference-generated fixtures and the training Functions'
routing through the oracle-backed emulation that declares the route (tests/_emu_backend_pad_heads.py), and the
unchanged behaviour of backends that do not declare it.  The kernels are checked by the -m gpu suite
(tests/test_gpu_attention_pad_heads.py)."""
import warnings

import pytest
import torch

from _emu_backend import EmuBackend
from _emu_backend_gemm_heads import EmuBackendGemmHeads
from _emu_backend_pad_heads import EmuBackendPadHeads, pad_heads_ref, unpad_heads_ref
from _emu_backend_wide import EmuBackendWide
from _pad_heads import PAD_HEAD_CONFIGS, PAD_HEAD_DIMS
from _recipe import rel_dev
from bbdm_b200 import cabi
from bbdm_b200.engine import UNetEngine
from bbdm_b200.unet import UNetModel
from oracle import bbdm_oracle as O
from test_attention_head_dims_host import _fill, _train_pair, build, load

TAGS = list(PAD_HEAD_CONFIGS)


def test_pad_route_predicate():
    """CudaBackend and the padded-head emulation take every width up to 256 natively (multiples of 8 on the kernels,
    the rest on the route); the older emulations declare no route; the rule's text is unchanged."""
    for be in (cabi.CudaBackend, EmuBackendPadHeads()):
        ok, rule = cabi.attn_head_dims(be)
        assert [d for d in range(1, 300) if ok(d) or cabi.attn_pad_route(be, d)] == list(range(1, 257))
        assert [d for d in range(1, 300) if cabi.attn_pad_route(be, d)] == [d for d in range(1, 257) if d % 8]
        assert rule == "multiples of 8 up to 256"
    for be in (EmuBackend(), EmuBackendWide(), EmuBackendGemmHeads()):
        assert not any(cabi.attn_pad_route(be, d) for d in range(1, 600))
    assert [cabi.pad_heads_width(d) for d in (4, 12, 20, 60, 124, 132, 252)] == [8, 16, 24, 64, 128, 136, 256]
    assert abs(cabi.pad_heads_scale(20) ** 4 - 24 / 20) < 1e-12


@pytest.mark.parametrize("order", [0, 1])
def test_repack_reference_scales_zero_fills_and_inverts(order):
    """qkv of 3 heads of 5 at both orders: q and k groups scaled, v not; zeros from 5 to 8; unpad with the inverse
    scales gives the source back, and the padded heads keep softmax(q k^T / sqrt(5)) v."""
    heads, d, c = 3, 5, cabi.pad_heads_scale(5)
    x = torch.randn(2, 7, 3 * heads * d, generator=torch.Generator().manual_seed(1))
    p = pad_heads_ref(x, heads, (c, c, 1.0), order)
    assert p.shape == (2, 7, 3 * heads * 8)
    g = p.view(2, 7, 3 * heads, 8)
    assert torch.equal(g[..., d:], torch.zeros_like(g[..., d:]))
    src = x.view(2, 7, 3 * heads, d)
    for i in range(3 * heads):
        t = i // heads if order else i % 3
        want = src[:, :, i] * torch.tensor(c if t < 2 else 1.0, dtype=torch.float32)
        assert torch.equal(g[..., i, :d], want), i
    back = unpad_heads_ref(p, heads, (1 / c, 1 / c, 1.0), order, d)
    assert rel_dev(back, x) < 1e-6
    # the oracle scales the padded heads by 8^-1/2; c^2 turns that into 5^-1/2
    o_ref = O.op_attention_nhwc(x.double(), heads, bool(order))
    o_pad = O.op_attention_nhwc(p.double(), heads, bool(order))
    assert rel_dev(unpad_heads_ref(o_pad.float(), heads, (1.0,), 0, d), o_ref.float()) < 1e-5


def test_configs_have_the_head_dims():
    for tag in TAGS:
        net = UNetModel(**PAD_HEAD_CONFIGS[tag])
        dims = {m.d_head if hasattr(m, "d_head") else m.channels // m.num_heads
                for m in net.modules() if type(m).__name__ in ("AttentionBlock", "SpatialTransformer")}
        assert dims == {PAD_HEAD_DIMS[tag]}, (tag, dims)
        chans = {m.num_channels for m in net.modules() if isinstance(m, torch.nn.GroupNorm)}
        assert all(c % 32 == 0 for c in chans), (tag, chans)


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_matches_pad_head_reference_fixture(tag):
    g = load(tag)
    cfg = O.unet_cfg(**PAD_HEAD_CONFIGS[tag])
    sd = build(PAD_HEAD_CONFIGS[tag]).state_dict()
    bufs, steps = O.make_schedule()
    x, y, t = g["x"], g["y"], g["t"]
    assert rel_dev(O.unet_forward(sd, cfg, x, t, y), g["unet_out"]) < 2e-6
    for i in g["ps_ids"].tolist():
        o, _ = O.p_sample(sd, cfg, bufs, steps, i, g[f"ps{i}_xt"], y, y, g[f"ps{i}_noise"], prefix="")
        assert rel_dev(o, g[f"ps{i}_out"]) < 2e-6


@pytest.mark.parametrize("tag", TAGS)
def test_engine_wiring_matches_pad_head_reference_fixture(tag):
    """On the emulation with the route the engine repacks every head to dp and runs the existing kernel there (its
    methods reject any width that is not a multiple of 8): wgmma at 64 and 128, mma.sync otherwise."""
    g = {k: v for k, v in load(tag).items() if isinstance(v, torch.Tensor)}
    be = EmuBackendPadHeads()
    eng = UNetEngine(build(PAD_HEAD_CONFIGS[tag]), backend=be)
    out = eng.forward(g["x"], g["t"], g["y"])
    assert out.shape == g["unet_out"].shape and not torch.isnan(out).any()
    assert rel_dev(out, g["unet_out"]) < 6e-5
    assert {"prep heads pad", "prep heads unpad"} <= set(be.calls)
    dp = cabi.pad_heads_width(PAD_HEAD_DIMS[tag])
    if "_st_" in tag:
        assert "attention_cross" in be.calls
    assert ("attention_tc" in be.calls) == (dp in cabi.ATTN_TC_HEAD_DIMS)


@pytest.mark.parametrize("tag", ["mid_hd20", "mid_st_hd36"])
@pytest.mark.parametrize("be_cls", [EmuBackend, EmuBackendWide])
def test_backends_without_the_route_still_raise(tag, be_cls):
    g = {k: v for k, v in load(tag).items() if isinstance(v, torch.Tensor)}
    eng = UNetEngine(build(PAD_HEAD_CONFIGS[tag]), backend=be_cls())
    with pytest.raises(NotImplementedError, match=f"head_dim {PAD_HEAD_DIMS[tag]}: .*multiples of 8 up to"):
        eng.forward(g["x"], g["t"], g["y"])


def _attention_block(channels, heads, new_order, seed):
    import bbdm_b200.unet as U
    blk = U.AttentionBlock(channels, num_heads=heads, use_new_attention_order=new_order)
    gen = _fill(blk, seed)
    with torch.no_grad():
        blk.norm.weight.add_(1.0)
    x = torch.randn((2, channels, 8, 8), generator=gen)
    gy = 0.2 * torch.randn((2, channels, 8, 8), generator=gen)
    return blk, x, gy


def _no_library_warning(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        r = fn()
    assert not [x for x in w if "library" in str(x.message).lower()], [str(x.message) for x in w]
    return r


@pytest.mark.parametrize("channels,heads,new_order", [(160, 8, False), (96, 8, True), (480, 8, False),
                                                      (1056, 8, True)])
def test_attention_block_pad_heads_train_through_native_functions(channels, heads, new_order):
    """AttentionBlock with heads of 20, 12, 60 or 132: AttentionCoreFn repacks to dp and runs the kernels there
    (wgmma forward at 64), matching the stock-PyTorch graph of the same block with no library-path warning."""
    blk, x, gy = _attention_block(channels, heads, new_order, 47)
    res = _no_library_warning(lambda: _train_pair(blk, x, gy, EmuBackendPadHeads()))
    calls = res[True][3]
    assert {"prep heads pad", "prep heads unpad", "attention_bwd"} <= calls
    assert ("attention_tc" in calls) == (cabi.pad_heads_width(channels // heads) in cabi.ATTN_TC_HEAD_DIMS)
    assert not res[False][3] & {"attention", "attention_bwd", "prep heads pad"}
    assert rel_dev(res[True][0], res[False][0]) < 3e-5
    assert rel_dev(res[True][1], res[False][1]) < 1e-4
    for n in res[False][2]:
        assert rel_dev(res[True][2][n], res[False][2][n]) < 1e-4, n


def test_attention_block_pad_heads_take_the_stock_core_without_the_route():
    blk, x, gy = _attention_block(160, 8, False, 48)
    res = _train_pair(blk, x, gy, EmuBackendWide())
    assert not res[True][3] & {"attention", "attention_split", "attention_tc", "attention_bwd"}
    assert rel_dev(res[True][1], res[False][1]) < 1e-4


@pytest.mark.parametrize("d", [20, 36])
def test_transformer_pad_heads_train_through_native_functions(d):
    """SpatialTransformer(8 heads of d, context): self- and cross-attention repack to dp and run the native Functions,
    matching the stock graph."""
    from bbdm_b200.transformer import SpatialTransformer
    C = 8 * d
    m = SpatialTransformer(C, 8, d, context_dim=3)
    gen = _fill(m, 49)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, (torch.nn.LayerNorm, torch.nn.GroupNorm)):
                mod.weight.add_(1.0)
    x = torch.randn((2, C, 8, 8), generator=gen)
    ctx = torch.randn((2, 3, 8, 8), generator=gen)
    gy = 0.2 * torch.randn((2, C, 8, 8), generator=gen)
    res = _no_library_warning(lambda: _train_pair(m, x, gy, EmuBackendPadHeads(), ctx))
    assert {"prep heads pad", "prep heads unpad", "attention_bwd", "attention_cross",
            "attention_cross_bwd"} <= res[True][3]
    assert not res[False][3]
    assert rel_dev(res[True][0], res[False][0]) < 3e-5
    assert rel_dev(res[True][1], res[False][1]) < 1e-4
    for n in res[False][2]:
        assert rel_dev(res[True][2][n], res[False][2][n]) < 1e-4, n


def test_shadow_checks_the_emulated_head_repacks():
    """The pad-heads launch shadow accepts the emulated sampling forward of a SpatialTransformer UNet on the route, checks
    both repack directions bit for bit, and flags exactly the repack whose output was perturbed."""
    from _launch_shadow_pad_heads import PadHeadsShadow
    g = {k: v for k, v in load("mid_st_hd20").items() if isinstance(v, torch.Tensor)}

    def run(mutate=None):
        sh = PadHeadsShadow(EmuBackendPadHeads())
        sh.mutate = mutate or {}
        eng = UNetEngine(build(PAD_HEAD_CONFIGS["mid_st_hd20"]), backend=sh)
        eng.forward(g["x"], g["t"], g["y"])
        return sh

    clean = run()
    assert not clean.failures(), clean.failures()[:5]
    whats = {c.what for c in clean.checks if c.method == "prep"}
    assert {"heads pad planes", "heads unpad planes"} <= whats, whats
    idx = next(i for i, (m, f) in enumerate(clean.launches) if m == "prep" and f.endswith("heads"))

    def flip(a):
        a["raw_hi"].view(-1)[-1:].view(torch.int16).bitwise_xor_(1)

    assert run({idx: flip}).flagged_launches() == [idx]
