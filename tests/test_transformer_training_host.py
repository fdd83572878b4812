"""SpatialTransformer training on CPU through the oracle-backed backend emulation: the autograd plumbing of the native
path (LayerNorm->Linear and GEGLU->Linear Functions, the q|k|v weight concat, the cross-attention Function, the
context's k|v projection and its gradient on / off) against the stock-PyTorch graph.  The kernels themselves are
checked by the -m gpu suite (tests/test_gpu_transformer_training.py)."""
import pytest
import torch
import torch.nn.functional as F

from _emu_backend import EmuBackend as _EmuBackend
from _recipe import rel_dev


class EmuBackend(_EmuBackend):
    """The emulation backend with the three SpatialTransformer backward entry points (fp64 autograd)."""

    def layernorm_bwd(self, x, dy, gamma, eps, dx, dgamma, dbeta, workspace):
        self.calls.append("layernorm_bwd")
        assert not torch.isnan(x).any() and not torch.isnan(dy).any()
        xd, gd = x.double().requires_grad_(True), gamma.double().requires_grad_(True)
        bd = torch.zeros_like(gd, requires_grad=True)
        with torch.enable_grad():
            F.layer_norm(xd, (x.shape[-1],), gd, bd, eps).backward(dy.double())
        dx.copy_(xd.grad)
        dgamma.copy_(gd.grad)
        dbeta.copy_(bd.grad)

    def geglu_bwd(self, u, dy, du):
        self.calls.append("geglu_bwd")
        ud = u.double().requires_grad_(True)
        with torch.enable_grad():
            a, g = ud.chunk(2, dim=-1)
            (a * F.gelu(g)).backward(dy.double())
        du.copy_(ud.grad)

    def attention_cross_bwd(self, q, kv, out, dout, heads, dq, dkv, lse, delta):
        self.calls.append("attention_cross_bwd")
        B, Tq, Cc = q.shape
        d = Cc // heads
        qd, kvd = q.double().requires_grad_(True), kv.double().requires_grad_(True)
        sp = lambda t: t.reshape(B, t.shape[1], heads, d).permute(0, 2, 1, 3)
        with torch.enable_grad():
            w = torch.softmax(torch.einsum("bhid,bhjd->bhij", sp(qd), sp(kvd[..., :Cc])) * d ** -0.5, dim=-1)
            o = torch.einsum("bhij,bhjd->bhid", w, sp(kvd[..., Cc:])).permute(0, 2, 1, 3).reshape(B, Tq, Cc)
            o.backward(dout.double())
        dq.copy_(qd.grad)
        dkv.copy_(kvd.grad)


def _transformer(context_dim, seed=3):
    from bbdm_b200.transformer import SpatialTransformer
    m = SpatialTransformer(64, 1, 64, context_dim=context_dim)
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in m.named_parameters():
            p.copy_(0.1 * torch.randn(p.shape, generator=gen) + (1.0 if "norm" in n and n.endswith("weight") else 0.0))
    return m


@pytest.fixture
def emu():
    from bbdm_b200 import train
    be = EmuBackend()
    train.set_backend(be)
    yield be
    train.set_backend(None)


def _run(m, x, ctx, gy, native, be):
    import bbdm_b200.unet as U
    U.NATIVE_TRAIN_CONV = native
    try:
        be.calls.clear()
        m.zero_grad(set_to_none=True)
        xi = x.clone().requires_grad_(True)
        ci = None if ctx is None else ctx[0].clone().requires_grad_(ctx[1])
        y = m(xi, ci)
        y.backward(gy)
    finally:
        U.NATIVE_TRAIN_CONV = True
    return (y.detach(), xi.grad, None if ci is None else ci.grad, {n: p.grad.clone() for n, p in m.named_parameters()},
            list(be.calls))


@pytest.mark.parametrize("context_grad", [True, False])
def test_cross_attention_transformer_native_graph_matches_stock(emu, context_grad):
    m = _transformer(3)
    gen = torch.Generator().manual_seed(4)
    x = torch.randn((2, 64, 8, 8), generator=gen).contiguous(memory_format=torch.channels_last)
    ctx = torch.randn((2, 3, 16, 16), generator=gen)
    gy = 0.2 * torch.randn((2, 64, 8, 8), generator=gen)
    nat = _run(m, x, (ctx, context_grad), gy, True, emu)
    ref = _run(m, x, (ctx, context_grad), gy, False, emu)
    calls = nat[4]
    assert {"layernorm_split", "layernorm_bwd", "geglu_split", "geglu_bwd", "attention_cross", "attention_cross_bwd",
            "attention_tc", "attention_bwd", "conv_wgrad_direct", "gn_bwd_apply"} <= set(calls), set(calls)
    assert not ref[4]                                     # the stock graph calls no kernel
    # the k|v projection runs bbdm_conv_direct once forward, and once more for the data gradient only if needed
    assert calls.count("conv_direct") == (2 if context_grad else 1)
    assert rel_dev(nat[0], ref[0]) < 3e-5
    assert rel_dev(nat[1], ref[1]) < 1e-4
    if context_grad:
        assert rel_dev(nat[2], ref[2]) < 1e-4
    else:
        assert nat[2] is None and ref[2] is None
    assert set(nat[3]) == set(ref[3])
    for n in ref[3]:
        assert rel_dev(nat[3][n], ref[3][n]) < 1e-4, (n, rel_dev(nat[3][n], ref[3][n]))


def test_transformer_without_context_runs_attn2_as_self_attention(emu):
    m = _transformer(None)
    gen = torch.Generator().manual_seed(5)
    x = torch.randn((2, 64, 8, 8), generator=gen).contiguous(memory_format=torch.channels_last)
    gy = 0.2 * torch.randn((2, 64, 8, 8), generator=gen)
    nat = _run(m, x, None, gy, True, emu)
    ref = _run(m, x, None, gy, False, emu)
    assert nat[4].count("attention_bwd") == 2 and "attention_cross" not in nat[4]
    assert rel_dev(nat[0], ref[0]) < 3e-5 and rel_dev(nat[1], ref[1]) < 1e-4
    for n in ref[3]:
        assert rel_dev(nat[3][n], ref[3][n]) < 1e-4, n


def test_shape_outside_the_kernels_takes_the_stock_graph(emu):
    """head_dim 48 is not a kernel instance: the transformer falls back to the stock graph (with the library-path
    warning on CUDA tensors) and no kernel runs."""
    from bbdm_b200.transformer import SpatialTransformer
    m = SpatialTransformer(96, 2, 48, context_dim=3)
    x = torch.randn((2, 96, 8, 8))
    m(x.requires_grad_(True), torch.randn((2, 3, 8, 8))).sum().backward()
    assert not emu.calls
