"""Attention heads wider than 256 channels on CPU: the rule that sends them to the GEMM-composed route on a backend that
declares it (and nowhere else), the sampling engine's wiring against the reference-generated fixtures, routing (no
flash-attention launch sees such a head, no library-path warning in a training step) and the emulated training step
against the stock graph, through the oracle-backed emulation with CudaBackend's route (tests/_emu_backend_gemm_heads.py).
The kernels are checked by the -m gpu suite (tests/test_gpu_attention_gemm_heads.py)."""
import warnings

import pytest
import torch

from _emu_backend_gemm_heads import EmuBackendGemmHeads, softmax_rows_bwd64
from _emu_backend_wide import EmuBackendWide
from _gemm_heads import GEMM_HEAD_CONFIGS, GEMM_HEAD_DIMS
from _recipe import rel_dev
from bbdm_b200 import cabi
from bbdm_b200.engine import UNetEngine
from bbdm_b200.unet import UNetModel
from test_attention_head_dims_host import _fill, _train_pair, build, load

TAGS = list(GEMM_HEAD_CONFIGS)
FLASH = {"attention", "attention_split", "attention_tc", "attention_cross", "attention_bwd", "attention_cross_bwd"}


def test_gemm_route_rule():
    """CudaBackend and the route's emulation send every width above 256 to the route and nothing up to 256; backends
    without the attribute send nothing."""
    for be in (cabi.CudaBackend, EmuBackendGemmHeads()):
        assert [d for d in range(2049) if cabi.attn_gemm_route(be, d)] == list(range(257, 2049))
    for be in (EmuBackendWide(),):
        assert not any(cabi.attn_gemm_route(be, d) for d in range(2049))
    assert [cabi.gemm_heads_pad(d) for d in (264, 288, 336, 384, 512, 1000)] == [288, 288, 352, 384, 512, 1024]


def test_configs_have_the_head_dims():
    for tag in TAGS:
        net = UNetModel(**GEMM_HEAD_CONFIGS[tag])
        dims = {m.d_head if hasattr(m, "d_head") else m.channels // m.num_heads
                for m in net.modules() if type(m).__name__ in ("AttentionBlock", "SpatialTransformer")}
        assert dims == {GEMM_HEAD_DIMS[tag]}, (tag, dims)


@pytest.mark.parametrize("tag", TAGS)
def test_engine_wiring_matches_gemm_head_reference_fixture(tag):
    """The engine runs these heads as conv_umma GEMMs around softmax_rows_split (the emulation's flash methods reject
    them) and matches the reference's UNet output."""
    g = {k: v for k, v in load(tag).items() if isinstance(v, torch.Tensor)}
    be = EmuBackendGemmHeads()
    out = UNetEngine(build(GEMM_HEAD_CONFIGS[tag]), backend=be).forward(g["x"], g["t"], g["y"])
    assert out.shape == g["unet_out"].shape and not torch.isnan(out).any()
    assert rel_dev(out, g["unet_out"]) < 6e-5
    assert {"softmax_rows_split", "split_grad"} <= set(be.calls) and not set(be.calls) & FLASH


@pytest.mark.parametrize("tag", ["mid_hd512", "mid_st_hd384"])
def test_without_the_route_wide_heads_still_raise(tag):
    g = {k: v for k, v in load(tag).items() if isinstance(v, torch.Tensor)}
    eng = UNetEngine(build(GEMM_HEAD_CONFIGS[tag]), backend=EmuBackendWide())
    with pytest.raises(NotImplementedError, match=f"head_dim {GEMM_HEAD_DIMS[tag]}: .*multiples of 8 up to 256"):
        eng.forward(g["x"], g["t"], g["y"])


def test_softmax_rows_bwd_oracle_is_the_softmax_adjoint():
    g = torch.Generator().manual_seed(3)
    s, dp = torch.randn(5, 12, generator=g, dtype=torch.float64), torch.randn(5, 12, generator=g, dtype=torch.float64)
    x = s[:, :9].clone().requires_grad_(True)
    torch.softmax(0.3 * x, -1).backward(dp[:, :9])
    p, ds = softmax_rows_bwd64(s, dp, 0.3, 9)
    assert torch.allclose(ds[:, :9], x.grad) and not ds[:, 9:].any() and not p[:, 9:].any()


def _train(blk, x, gy, ctx=None):
    be = EmuBackendGemmHeads()
    with warnings.catch_warnings():
        warnings.simplefilter("error")          # a library-path warning fails the test
        res = _train_pair(blk, x, gy, be, ctx)
    assert be.softmax_grads > 0                 # the backward ran the score-gradient mode (the stock pass runs none)
    return res


def _check(res):
    assert {"softmax_rows_split", "conv_wgrad"} <= res[True][3]
    assert not res[True][3] & FLASH
    assert rel_dev(res[True][0], res[False][0]) < 3e-5
    assert rel_dev(res[True][1], res[False][1]) < 1e-4
    for n in res[False][2]:
        assert rel_dev(res[True][2][n], res[False][2][n]) < 1e-4, n


@pytest.mark.parametrize("channels,heads,new_order,side", [(512, 1, False, 8), (672, 2, True, 10), (672, 2, False, 10)])
def test_attention_block_trains_on_the_gemm_route(channels, heads, new_order, side):
    import bbdm_b200.unet as U
    blk = U.AttentionBlock(channels, num_heads=heads, use_new_attention_order=new_order)
    gen = _fill(blk, 43)
    with torch.no_grad():
        blk.norm.weight.add_(1.0)
    x = torch.randn((2, channels, side, side), generator=gen)
    gy = 0.2 * torch.randn((2, channels, side, side), generator=gen)
    _check(_train(blk, x, gy))


def test_transformer_dhead384_trains_on_the_gemm_route():
    """SpatialTransformer(768, 2 heads of 384) with a 5x5 context (Tkv = 25, masked): self- and cross-attention."""
    from bbdm_b200.transformer import SpatialTransformer
    m = SpatialTransformer(768, 2, 384, context_dim=3)
    gen = _fill(m, 45)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, (torch.nn.LayerNorm, torch.nn.GroupNorm)):
                mod.weight.add_(1.0)
    x = torch.randn((2, 768, 10, 10), generator=gen)
    ctx = torch.randn((2, 3, 5, 5), generator=gen)
    gy = 0.2 * torch.randn((2, 768, 10, 10), generator=gen)
    _check(_train(m, x, gy, ctx))
