"""-m gpu: attention at the head sizes that are multiples of 8 but not 16/32/64/128 -- the mma.sync forwards, the
cross-attention core and both flash backwards against fp64 for every such size, the drop-in model against the
reference-generated fixtures (tests/golden/mid_hd*.npz, mid_st_hd*.npz), training steps against the stock graph, the
graphed and checkpointed steps against the eager one, and every launch of a sampling forward and a training step
against its fp64 recomputation."""
import contextlib
import gc
import os
import warnings

import numpy as np
import pytest
import torch

from _head_dims import HEAD_DIM_CONFIGS
from _launch_shadow import Shadow
from _recipe import bb_namespace, fill_state_dict, rel_dev, synth_images
from oracle import bbdm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL_PSAMPLE = 1e-4
NEW_DIMS = [8, 24, 40, 48, 56, 72, 80, 88, 96, 104, 112, 120]
SHAPES = [(1, 1, 2), (2, 100, 2), (1, 200, 3), (1, 1024, 2)]        # B, T, heads


def tol(T):
    """rel_dev bound against the exact result: max |error| over max |out|.  Over 1024 keys the near-uniform softmax
    averages the values down, so max |out| shrinks while the error does not (D = 8: 2.2e-5 and 2.7e-5 measured)."""
    return 3e-5 if T >= 1024 else 2e-5


@pytest.fixture(scope="module", autouse=True)
def _release_gpu_memory():
    """The models built here (a BrownianBridgeModel and its bridge reference each other) are freed only by the cycle
    collector: collect them and return their memory once the module is done, so that later full-size tests of the
    suite find the card as empty as without this module."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).float()


def nan_buffers(B, T, C):
    """fp32 and hi/lo outputs pre-filled with NaN: a column written wrongly or not at all shows up."""
    out = torch.full((B, T, C), float("nan"), device=DEV)
    oh = torch.full((B, T, C), float("nan"), dtype=torch.bfloat16, device=DEV)
    return out, oh, oh.clone()


def check_split(out, oh, ol):
    h, l = O.bf16_split(out.cpu())
    assert torch.equal(oh.float().cpu(), h) and torch.equal(ol.float().cpu(), l)


# ------------------------------------------------------------------------------------ forward kernels
@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("B,T,heads", SHAPES)
@pytest.mark.parametrize("D", NEW_DIMS)
def test_attention_split_head_dims(be, D, B, T, heads, order):
    """mma.sync attention on the pre-split planes at D padded to a multiple of 16."""
    C = heads * D
    qkv = rnd((B, T, 3 * C), 70 + D, 1.2)
    hi, lo = O.bf16_split(qkv)
    want = O.op_attention_nhwc((hi + lo).double(), heads, bool(order))
    out, oh, ol = nan_buffers(B, T, C)
    be.attention_split(hi.to(torch.bfloat16).to(DEV), lo.to(torch.bfloat16).to(DEV), heads, order,
                       out_f32=out, out_hi=oh, out_lo=ol)
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()
    assert rel_dev(out, want) < tol(T), rel_dev(out, want)
    assert rel_dev(out, O.op_attention_nhwc(qkv.double(), heads, bool(order))) < 5e-5
    check_split(out, oh, ol)


@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("B,T,heads", SHAPES)
@pytest.mark.parametrize("D", NEW_DIMS)
def test_attention_fp32_qkv_head_dims(be, D, B, T, heads, order):
    """The fp32-qkv form (K / V split in shared memory, padded chunk grid)."""
    C = heads * D
    qkv = rnd((B, T, 3 * C), 90 + D, 1.2)
    want = O.op_attention_nhwc(qkv.double(), heads, bool(order))
    out, oh, ol = nan_buffers(B, T, C)
    be.attention(qkv.to(DEV), heads, order, out_f32=out, out_hi=oh, out_lo=ol)
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()
    assert rel_dev(out, want) < tol(T), rel_dev(out, want)
    check_split(out, oh, ol)


def _cross_ref(q, kv, heads, D):
    B, Tq, C = q.shape
    sp = lambda t: t.reshape(B, t.shape[1], heads, D).permute(0, 2, 1, 3)
    w = torch.softmax(torch.einsum("bhid,bhjd->bhij", sp(q), sp(kv[..., :C])) * D ** -0.5, dim=-1)
    return torch.einsum("bhij,bhjd->bhid", w, sp(kv[..., C:])).permute(0, 2, 1, 3).reshape(B, Tq, C)


@pytest.mark.parametrize("D", NEW_DIMS)
def test_attention_cross_head_dims(be, D):
    B, Tq, Tkv, heads = 2, 100, 77, 2
    C = heads * D
    q, kv = rnd((B, Tq, C), 120 + D, 1.2), rnd((B, Tkv, 2 * C), 121 + D, 1.2)
    want = _cross_ref(q.double(), kv.double(), heads, D)
    planes = lambda t: tuple(z.to(torch.bfloat16).to(DEV) for z in O.bf16_split(t))
    q_hi, q_lo = planes(q)
    kv_hi, kv_lo = planes(kv)
    out, oh, ol = nan_buffers(B, Tq, C)
    be.attention_cross(q_hi, q_lo, kv_hi, kv_lo, heads, out_f32=out, out_hi=oh, out_lo=ol)
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()
    assert rel_dev(out, want) < 2e-5, rel_dev(out, want)
    check_split(out, oh, ol)


# ------------------------------------------------------------------------------------ backward kernels
@pytest.mark.parametrize("B,T,heads,order", [(2, 100, 2, 0), (1, 200, 3, 1), (1, 64, 1, 0)])
@pytest.mark.parametrize("D", NEW_DIMS)
def test_attention_bwd_head_dims(be, D, B, T, heads, order):
    Cc = heads * D
    qkv = rnd((B, T, 3 * Cc), 30 + D, 1.5)
    dout = rnd((B, T, Cc), 31 + D, 0.3)
    qd = qkv.double().requires_grad_(True)
    od = O.op_attention_nhwc(qd, heads, bool(order))
    od.backward(dout.double())
    dqkv = torch.full((B, T, 3 * Cc), float("nan"), device=DEV)
    lse, delta = torch.empty(B * heads * T, device=DEV), torch.empty(B * heads * T, device=DEV)
    be.attention_bwd(qkv.to(DEV), od.detach().float().to(DEV), dout.to(DEV), heads, order, dqkv, lse, delta)
    torch.cuda.synchronize()
    assert not torch.isnan(dqkv).any()
    assert rel_dev(dqkv, qd.grad) < 2e-5, rel_dev(dqkv, qd.grad)


@pytest.mark.parametrize("D", NEW_DIMS)
def test_attention_cross_bwd_head_dims(be, D):
    B, Tq, Tkv, heads = 2, 100, 77, 2
    C = heads * D
    q, kv = rnd((B, Tq, C), 130 + D, 1.2), rnd((B, Tkv, 2 * C), 131 + D, 1.2)
    dout = rnd((B, Tq, C), 132 + D, 0.3)
    qd, kvd = q.double().requires_grad_(True), kv.double().requires_grad_(True)
    od = _cross_ref(qd, kvd, heads, D)
    od.backward(dout.double())
    dq = torch.full((B, Tq, C), float("nan"), device=DEV)
    dkv = torch.full((B, Tkv, 2 * C), float("nan"), device=DEV)
    lse, delta = torch.empty(B * heads * Tq, device=DEV), torch.empty(B * heads * Tq, device=DEV)
    be.attention_cross_bwd(q.to(DEV), kv.to(DEV), od.detach().float().to(DEV), dout.to(DEV), heads, dq, dkv, lse,
                           delta)
    torch.cuda.synchronize()
    assert not torch.isnan(dq).any() and not torch.isnan(dkv).any()
    assert rel_dev(dq, qd.grad) < 2e-5, rel_dev(dq, qd.grad)
    assert rel_dev(dkv, kvd.grad) < 2e-5, rel_dev(dkv, kvd.grad)


# ------------------------------------------------------------------------------------ drop-in model
def build(u, train=False, **kw):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    net = BrownianBridgeModel(bb_namespace(u, **kw))
    net = net.train() if train else net.eval()
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(fill_state_dict(shapes, seed=1234))
    return net.to(DEV)


def load(tag):
    return {k: torch.from_numpy(v) if v.ndim else v for k, v in np.load(os.path.join(GOLD, tag + ".npz")).items()}


@pytest.mark.parametrize("tag", list(HEAD_DIM_CONFIGS))
def test_head_dim_model_matches_reference_fixture(tag):
    g = load(tag)
    net = build(HEAD_DIM_CONFIGS[tag])
    c = lambda z: z.cuda()
    x, y, t = c(g["x"]), c(g["y"]), c(g["t"])
    with torch.no_grad():
        out = net.denoise_fn(x, timesteps=t, context=y)
    d_unet = rel_dev(out, g["unet_out"])
    devs = {}
    for i in g["ps_ids"].tolist():
        for clip, key in ((False, f"ps{i}_out"), (True, f"ps{i}_out_clip")):
            o, _ = net.p_sample(c(g[f"ps{i}_xt"]), y, y, i, clip_denoised=clip, noise=c(g[f"ps{i}_noise"]))
            devs[(i, clip)] = rel_dev(o, g[key])
    net._bridge.backend().check_fault()
    print(f"\n[{tag}] unet rel dev {d_unet:.3e}; p_sample rel dev {devs}")
    assert d_unet < TOL_PSAMPLE
    assert max(devs.values()) < TOL_PSAMPLE


# ------------------------------------------------------------------------------------ training
class _Recorder:
    """Pass-through backend that records which entry points ran."""

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


def _step(net, inputs):
    """loss, {name: grad}, the library-path warnings of one training step."""
    from bbdm_b200 import train
    x, y, t, nz = inputs
    train._WARNED.clear()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        net.zero_grad(set_to_none=True)
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
    torch.cuda.synchronize()
    train.backend().check_fault()
    lib = {str(r.message) for r in rec if "stock PyTorch" in str(r.message)}
    return loss.detach().clone(), {n: p.grad.detach().clone() for n, p in net.denoise_fn.named_parameters()}, lib


def _fixture_inputs(tag):
    g = load(tag)
    return tuple(g[k].cuda() for k in ("x", "y", "t", "q_noise"))


@pytest.mark.parametrize("tag", ["mid_hd48", "mid_st_hd40"])
def test_head_dim_training_step_matches_stock_graph(tag, monkeypatch):
    """Loss and every parameter gradient of one training step on the native path against the stock-PyTorch graph
    (TF32 off); the attention cores ran on the native Functions and no layer took the library path.  The gradient
    bound is test_gpu_transformer_training.py's for the same comparison: the stock graph's own fp32 error is part of
    it (worst tensors measured 1.6e-4 at head_dim 48, 1.5e-4 at d_head 40)."""
    import bbdm_b200.unet as U
    from bbdm_b200 import cabi, train
    net = build(HEAD_DIM_CONFIGS[tag], train=True)
    inputs = _fixture_inputs(tag)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    rec = _Recorder(cabi.CudaBackend())
    monkeypatch.setattr(train, "_BACKEND", rec)
    res = {}
    for native in (True, False):
        monkeypatch.setattr(U, "NATIVE_TRAIN_CONV", native)
        res[native] = _step(net, inputs)
    assert not res[True][2], res[True][2]
    want = {"attention", "attention_bwd"} | ({"attention_cross", "attention_cross_bwd"} if "_st_" in tag else set())
    assert want <= rec.calls, want - rec.calls
    loss_n, loss_s = float(res[True][0]), float(res[False][0])
    devs = {n: rel_dev(res[True][1][n], res[False][1][n]) for n in res[False][1]}
    worst = max(devs, key=devs.get)
    print(f"\n[{tag}] loss native {loss_n:.7f} stock {loss_s:.7f}; worst grad vs stock {worst} {devs[worst]:.3e}")
    assert abs(loss_n - loss_s) < 1e-4 * abs(loss_s)
    assert devs[worst] < 3e-4


def _same(a, b, what):
    assert torch.equal(a[0], b[0]), (what, float(a[0]), float(b[0]))
    bad = [n for n in a[1] if not torch.equal(a[1][n], b[1][n])]
    assert not bad, (what, bad[:5])


def test_head_dim_graphed_and_checkpointed_steps_are_bit_identical():
    """mid_st_hd40: the use_checkpoint step and the graphed step reproduce the plain eager step bit for bit."""
    from bbdm_b200 import train_graph
    net = build(HEAD_DIM_CONFIGS["mid_st_hd40"], train=True)
    inputs = _fixture_inputs("mid_st_hd40")
    plain = _step(net, inputs)
    net.denoise_fn.use_checkpoint = True
    _same(plain, _step(net, inputs), "use_checkpoint")
    net.denoise_fn.use_checkpoint = False
    net.denoise_fn.train_graph = True
    n0 = train_graph.CAPTURES["n"]
    for _ in range(2):
        _same(plain, _step(net, inputs), "graphed")
    assert train_graph.CAPTURES["n"] - n0 == 1
    train_graph.release(net.denoise_fn)


# ------------------------------------------------------------------------------------ launch shadow
def test_head_dim_sampling_forward_every_launch_against_fp64():
    from bbdm_b200 import cabi
    from bbdm_b200.engine import UNetEngine
    from bbdm_b200.unet import UNetModel
    net = UNetModel(**HEAD_DIM_CONFIGS["mid_st_hd40"]).eval()
    net.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1234))
    net = net.cuda()
    sh = Shadow(cabi.CudaBackend())
    eng = UNetEngine(net, backend=sh)
    eng.refresh_weights()
    sh.register_engine(eng)
    B = 2
    x, y = synth_images((B, 3, 32, 32), 11).cuda(), synth_images((B, 3, 32, 32), 12).cuda()
    t = torch.tensor([0, 999], dtype=torch.long).cuda()
    out = eng.forward(x, t, y)
    assert torch.isfinite(out).all()
    fails = sh.failures()
    print(f"\n{sh.table('mid_st_hd40 sampling forward, 32x32, B=2')}")
    assert not fails, fails[:10]
    checked = {c.method for c in sh.checks}
    assert {"attention_split", "attention_cross"} <= checked, checked


@contextlib.contextmanager
def _shadowed(monkeypatch):
    from bbdm_b200 import cabi, train
    from bbdm_b200.bridge import BridgeOps
    sh = Shadow(cabi.CudaBackend())
    monkeypatch.setattr(BridgeOps, "backend_factory", staticmethod(lambda: sh))
    old = train._BACKEND
    train.set_backend(sh)
    try:
        yield sh
    finally:
        train.set_backend(old)


def test_head_dim_training_step_every_launch_against_fp64(monkeypatch):
    net = build(HEAD_DIM_CONFIGS["mid_hd48"], train=True)
    x, y, t, nz = _fixture_inputs("mid_hd48")
    with _shadowed(monkeypatch) as sh:
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
    torch.cuda.synchronize()
    fails = sh.failures()
    print(f"\n{sh.table('mid_hd48 training step, 32x32, B=2')}")
    assert torch.isfinite(loss)
    assert not fails, fails[:10]
    checked = {c.method for c in sh.checks}
    assert {"attention", "attention_bwd"} <= checked, checked
