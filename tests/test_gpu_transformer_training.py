"""-m gpu: SpatialTransformer training on the native kernels -- the three backward kernels (LayerNorm, GEGLU,
cross-attention) against fp64 torch, the k|v projection's direct weight gradient beyond 1024 channel pairs, and
full training steps of transformer UNets against the stock-PyTorch graph and the unmodified reference's gradients
(tests/golden/st_grads.npz, tests/golden/make_golden_st_grads.py)."""
import os
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _hd128 import HD128_CONFIGS
from _recipe import bb_namespace, fill_state_dict, rel_dev

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(__file__), "golden")

# mid_st_hd128: 256 channels / 2 heads (head_dim 128); the _hd64 variant: 4 heads of 64.  Transformers at 8x8
# (T = 64, B = 2: 128 tokens), cross-attention over the 32x32 3-channel context (Tkv = 1024).
ST_CONFIGS = {"mid_st_hd128": HD128_CONFIGS["mid_st_hd128"],
              "mid_st_hd64": dict(HD128_CONFIGS["mid_st_hd128"], num_heads=4)}


def picked_gradients(unet):
    """The parameters whose gradients st_grads.npz stores: all of the middle block's transformer, the GroupNorm /
    LayerNorm affine parameters of every transformer, the stem, a ResBlock and the head."""
    keep = lambda n: n.startswith(("middle_block.1.", "input_blocks.0.0", "input_blocks.1.0.", "out.2")) or ".norm" in n
    return {n: p for n, p in unet.named_parameters() if keep(n)}


def fixture_rows(g):
    """The part of a gradient st_grads.npz stores: whole tensors up to 4096 elements, else 16 output rows spread evenly
    over the tensor (for ff.net.0.proj both the value and the gate half), which keeps the fixture small."""
    return g if g.numel() <= 4096 else g[:: max(1, g.shape[0] // 16)]


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).float()


@pytest.mark.parametrize("rows,C", [(100, 64), (1000, 256), (4097, 1280), (37, 2048)])
def test_layernorm_bwd_kernel(be, rows, C):
    """dx, dgamma, dbeta against fp64 autograd of F.layer_norm; two runs bit-identical (fixed-order column sums)."""
    from bbdm_b200 import cabi
    x = (rnd((rows, C), 1, 1.5) + 0.3).to(DEV)
    dy = rnd((rows, C), 2, 0.2).to(DEV)
    gamma, beta = (1 + 0.1 * rnd((C,), 3)).to(DEV), (0.1 * rnd((C,), 4)).to(DEV)
    runs = []
    for _ in range(2):
        dx = torch.full((rows, C), float("nan"), device=DEV)
        dg, db = torch.full((C,), float("nan"), device=DEV), torch.full((C,), float("nan"), device=DEV)
        ws = torch.full((cabi.layernorm_bwd_workspace(rows, C),), float("nan"), device=DEV)
        be.layernorm_bwd(x, dy, gamma, 1e-5, dx, dg, db, ws)
        runs.append((dx, dg, db))
    torch.cuda.synchronize()
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    xd, gd, bd = (t.double().requires_grad_(True) for t in (x, gamma, beta))
    F.layer_norm(xd, (C,), gd, bd, 1e-5).backward(dy.double())
    for name, got, want in (("dx", runs[0][0], xd.grad), ("dgamma", runs[0][1], gd.grad), ("dbeta", runs[0][2], bd.grad)):
        assert rel_dev(got, want) < 2e-6, (name, rel_dev(got, want))


@pytest.mark.parametrize("rows,N", [(128, 1024), (77, 64)])
def test_geglu_bwd_kernel(be, rows, N):
    """du = [dy*gelu(g) | dy*a*gelu'(g)] against fp64 autograd, with gates across [-9, 9] and near 0."""
    u = rnd((rows, 2 * N), 5, 2.0)
    g = u[:, N:]
    g[:, : N // 4] = torch.linspace(-9.0, 9.0, N // 4)               # |g| > 6: Phi saturates, phi underflows
    g[:, N // 4: N // 2] = torch.linspace(-1e-3, 1e-3, N // 4)     # g near 0
    u, dy = u.to(DEV), rnd((rows, N), 6, 0.3).to(DEV)
    du = torch.full_like(u, float("nan"))
    be.geglu_bwd(u, dy, du)
    ud = u.double().requires_grad_(True)
    a, gd = ud.chunk(2, dim=-1)
    (a * F.gelu(gd)).backward(dy.double())
    assert torch.isfinite(du).all()
    assert rel_dev(du, ud.grad) < 2e-6, rel_dev(du, ud.grad)


def _cross_ref(q, kv, heads):
    B, Tq, Cc = q.shape
    D = Cc // heads
    k, v = kv[..., :Cc], kv[..., Cc:]
    sp = lambda t: t.reshape(B, t.shape[1], heads, D).permute(0, 2, 1, 3)
    w = (torch.einsum("bhid,bhjd->bhij", sp(q), sp(k)) * D ** -0.5).softmax(-1)
    return torch.einsum("bhij,bhjd->bhid", w, sp(v)).permute(0, 2, 1, 3).reshape(B, Tq, Cc)


CROSS_BWD_CASES = [
    # B, Tq, Tkv, heads, D
    (2, 64, 1024, 2, 128),
    (2, 100, 1, 4, 64),        # one key: P = 1
    (1, 257, 100, 3, 32),      # ragged Tq and Tkv
    (2, 1, 300, 2, 16),        # one query
    (1, 128, 4096, 8, 64),
]


@pytest.mark.parametrize("case", CROSS_BWD_CASES)
def test_attention_cross_bwd_kernel(be, case):
    B, Tq, Tkv, heads, D = case
    Cc = heads * D
    q, kv = rnd((B, Tq, Cc), 7, 1.2), rnd((B, Tkv, 2 * Cc), 8, 1.2)
    dout = rnd((B, Tq, Cc), 9, 0.3)
    qd, kvd = q.double().requires_grad_(True), kv.double().requires_grad_(True)
    od = _cross_ref(qd, kvd, heads)
    od.backward(dout.double())
    dq, dkv = torch.full((B, Tq, Cc), float("nan"), device=DEV), torch.full((B, Tkv, 2 * Cc), float("nan"), device=DEV)
    lse, delta = torch.empty(B * heads * Tq, device=DEV), torch.empty(B * heads * Tq, device=DEV)
    be.attention_cross_bwd(q.to(DEV), kv.to(DEV), od.detach().float().to(DEV), dout.to(DEV), heads, dq, dkv, lse, delta)
    torch.cuda.synchronize()
    if Tkv == 1:      # one key: P = 1, dS = P (dP - delta) = 0 exactly, so dq is 0 up to rounding
        assert dq.abs().max() < 1e-6
    else:
        assert rel_dev(dq, qd.grad) < 2e-5, rel_dev(dq, qd.grad)
    assert rel_dev(dkv, kvd.grad) < 2e-5, rel_dev(dkv, kvd.grad)


def test_small_conv_wgrad_beyond_1024_pairs():
    """The k|v projection of a 3-channel context to 2 x 512 channels (3072 channel pairs): SmallConv2dFn's direct
    forward, data and weight gradients vs fp64."""
    from bbdm_b200.train import SmallConv2dFn
    x = rnd((2, 3, 32, 32), 10).to(DEV).requires_grad_(True)
    w = rnd((1024, 3, 1, 1), 11, 0.3).to(DEV).requires_grad_(True)
    gy = rnd((2, 1024, 32, 32), 12, 0.2).to(DEV)
    SmallConv2dFn.apply(x, w, None).backward(gy)
    xd, wd = x.detach().double().requires_grad_(True), w.detach().double().requires_grad_(True)
    F.conv2d(xd, wd).backward(gy.double())
    assert rel_dev(w.grad, wd.grad) < 2e-6 and rel_dev(x.grad, xd.grad) < 2e-6


class _Recorder:
    """cabi.CudaBackend with a log of the entry points called."""

    def __init__(self, inner):
        self.inner, self.calls = inner, set()

    def __getattr__(self, name):
        a = getattr(self.inner, name)
        if callable(a):
            def rec(*args, **kw):
                self.calls.add(name)
                return a(*args, **kw)
            return rec
        return a


def _st_model(tag):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    net = BrownianBridgeModel(bb_namespace(ST_CONFIGS[tag])).train()
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(fill_state_dict(shapes, seed=1234))
    return net.cuda()


@pytest.mark.parametrize("tag", list(ST_CONFIGS))
def test_transformer_training_step_native_matches_stock_and_reference(tag, monkeypatch):
    """One training step of a SpatialTransformer UNet: loss and every parameter gradient on the native path vs the
    stock-PyTorch graph (TF32 off) and vs the unmodified reference's CPU fp32 gradients; no layer runs on library
    kernels, and the transformer's native kernels ran."""
    import bbdm_b200.unet as U
    from bbdm_b200 import cabi, train
    g = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(GOLD, "mid_st_hd128.npz")).items() if v.ndim}
    net = _st_model(tag)
    x, y, t, nz = (g[k].cuda() for k in ("x", "y", "t", "q_noise"))
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    rec = _Recorder(cabi.CudaBackend())
    monkeypatch.setattr(train, "_BACKEND", rec)
    monkeypatch.setattr(train, "_WARNED", set())
    res = {}
    for native in (True, False):
        monkeypatch.setattr(U, "NATIVE_TRAIN_CONV", native)
        net.zero_grad(set_to_none=True)
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            loss, _ = net.p_losses(x, y, y, t, nz)
            loss.backward()
        res[native] = (float(loss), {n: p.grad.detach().clone() for n, p in net.denoise_fn.named_parameters()})
        if native:
            lib = [str(w.message) for w in caught if "stock PyTorch kernels" in str(w.message)]
            assert not lib, lib
    torch.cuda.synchronize()
    rec.inner.check_fault()
    assert {"layernorm_split", "layernorm_bwd", "geglu_split", "geglu_bwd", "attention_cross", "attention_cross_bwd",
            "attention_bwd", "conv_wgrad_direct"} <= rec.calls, rec.calls
    assert abs(res[True][0] - res[False][0]) < 1e-4 * abs(res[False][0])
    devs = {n: rel_dev(res[True][1][n], res[False][1][n]) for n in res[False][1]}
    worst = max(devs, key=devs.get)
    print(f"\n[{tag}] loss native {res[True][0]:.6f} stock {res[False][0]:.6f}; worst grad vs stock {worst} {devs[worst]:.3e}")
    assert devs[worst] < 3e-4
    gr = np.load(os.path.join(GOLD, "st_grads.npz"))
    ref_loss = float(gr[f"{tag}:loss"])
    assert abs(res[True][0] - ref_loss) < 2e-4 * abs(ref_loss)
    pre = f"{tag}:grad:"
    rdev = {k[len(pre):]: rel_dev(fixture_rows(res[True][1][k[len(pre):]]), torch.from_numpy(gr[k]))
            for k in gr.files if k.startswith(pre)}
    worst = max(rdev, key=rdev.get)
    print(f"[{tag}] vs reference gradient fixture: {len(rdev)} tensors, worst {worst} {rdev[worst]:.3e}")
    assert len(rdev) >= 30 and rdev[worst] < 3e-4


def test_context_gradient_reaches_spatial_rescaler(monkeypatch):
    """A trainable cond stage (SpatialRescaler with a channel map, as LatentBrownianBridgeModel optimises it) feeds the
    UNet's stem concat and every transformer's k|v projection: its weight gradient on the native path matches the
    stock graph."""
    import bbdm_b200.unet as U
    from bbdm_b200.cond import SpatialRescaler
    net = _st_model("mid_st_hd64").denoise_fn
    cond = SpatialRescaler(n_stages=1, in_channels=3, out_channels=3).cuda()
    with torch.no_grad():
        cond.channel_mapper.weight.copy_(torch.eye(3)[:, :, None, None] + 0.1 * rnd((3, 3, 1, 1), 13))
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    y64 = rnd((2, 3, 64, 64), 14).cuda()
    x = rnd((2, 3, 32, 32), 15).cuda()
    t = torch.tensor([17, 328], device=DEV)
    res = {}
    for native in (True, False):
        monkeypatch.setattr(U, "NATIVE_TRAIN_CONV", native)
        net.zero_grad(set_to_none=True)
        cond.zero_grad(set_to_none=True)
        out = net(x, timesteps=t, context=cond(y64))
        (out * rnd(tuple(out.shape), 16).cuda()).sum().backward()
        res[native] = cond.channel_mapper.weight.grad.clone()
    d = rel_dev(res[True], res[False])
    print(f"\n[context gradient] channel_mapper.weight.grad native vs stock rel dev {d:.3e}")
    assert d < 3e-4
