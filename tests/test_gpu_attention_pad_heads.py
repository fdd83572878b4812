"""-m gpu: attention heads whose width d is not a multiple of 8 (the padded-head route) -- the repack kernels bit for bit
against torch, the route's sampling and training forms against fp64 (self- and cross-attention, forward and backward),
the drop-in models against the reference-generated fixtures (tests/golden/mid_hd4.npz ... mid_st_hd36.npz), training
steps against the stock graph, the graphed and checkpointed steps against the eager one, every launch of a sampling
forward and a training step under the fp64 shadow over the launch guard, and the memory of a T = 4096 training step."""
import contextlib
import gc
from types import SimpleNamespace

import pytest
import torch

from _emu_backend_pad_heads import pad_heads_ref, unpad_heads_ref
from _launch_guard import Guard, canaried, tail_untouched
from _launch_shadow import split_bf16
from _launch_shadow_pad_heads import PadHeadsShadow
from _pad_heads import PAD_HEAD_CONFIGS
from _recipe import fill_state_dict, rel_dev, synth_images
from test_gpu_attention_head_dims import _Recorder, _cross_ref, _fixture_inputs, _same, _step, build, load, rnd

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL_PSAMPLE = 1e-4
PAD_DIMS = [4, 12, 20, 60, 124, 132, 252]           # dp 8, 16, 24 (mma.sync), 64, 128 (wgmma), 136, 256 (wide)
SHAPES = [(2, 1, 3), (2, 100, 2), (1, 1024, 2)]       # B, T, heads
# The route's bound against fp64, forward and backward: the kernels' own bounds (test_gpu_attention_head_dims.py: 2e-5,
# 3e-5 over 1024 keys) are taken on operands of 8 or more nonzero columns per head; heads of 4 to 20 put fewer products
# into each output, and measured up to 3.4e-5 (forward, d 4, T 1024) and 5.7e-5 (cross-attention dq, d 4, T 1024) on
# an H100 80GB HBM3 (700 W).  The zero columns add exact zeros, so the kernels at dp see the values they would at d.
ROUTE_TOL = 6e-5


class _HeadsRecorder(_Recorder):
    """_Recorder that names prep's head repacks ('prep heads pad' / 'prep heads unpad')."""

    def prep(self, src1, src2, **kw):
        if kw.get("heads") is not None:
            out = kw["raw_f32"] if kw.get("raw_f32") is not None else kw["raw_hi"]
            self.calls.add("prep heads pad" if out.shape[-1] >= src1.shape[-1] else "prep heads unpad")
        else:
            self.calls.add("prep")
        return self.inner.prep(src1, src2, **kw)


def train_cfg(tag):
    """The training tests' variant of a fixture configuration: model_channels 64 and 16 heads (the same head width)."""
    return dict(PAD_HEAD_CONFIGS[tag], model_channels=64, num_heads=16)


@pytest.fixture(scope="module", autouse=True)
def _release_gpu_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


# ------------------------------------------------------------------------------------ repack kernels
@pytest.mark.parametrize("d", [1, 4, 5, 12, 20, 36, 60, 84, 124, 132, 252])
@pytest.mark.parametrize("scales,order", [((1.1, 1.1, 1.0), 0), ((1.1, 1.1, 1.0), 1), ((1.07,), 0), ((1.07, 1.0), 1),
                                          ((1.0,), 0)])
def test_pad_and_unpad_are_bit_exact(be, d, scales, order):
    """fp32 outputs equal torch's one fp32 multiply per element, zeros from d to dp; the planes are the split of the
    scaled values (bbdm_prep_operand's rounding); canary tails behind every output stay untouched."""
    from bbdm_b200 import cabi
    heads, rows = 3, 37
    G, dp = len(scales) * heads, cabi.pad_heads_width(d)
    x = rnd((rows, G * d), 300 + d, 2.0).to(DEV)
    (pf, pfb), (ph, phb), (pl, plb) = canaried((rows, G * dp)), canaried((rows, G * dp), torch.bfloat16), \
        canaried((rows, G * dp), torch.bfloat16)
    be.prep(x, None, raw_f32=pf, raw_hi=ph, raw_lo=pl, heads=(heads, scales, order))
    want = pad_heads_ref(x, heads, scales, order)
    h, l = split_bf16(want)
    torch.cuda.synchronize()
    assert torch.equal(pf, want) and torch.equal(ph, h) and torch.equal(pl, l)
    hp, lp = torch.empty_like(ph), torch.empty_like(pl)
    be.prep(want.view(1, 1, rows, G * dp), None, raw_hi=hp.view(1, 1, rows, -1), raw_lo=lp.view(1, 1, rows, -1))
    assert torch.equal(ph, hp) and torch.equal(pl, lp)
    (uf, ufb), (uh, uhb), (ul, ulb) = canaried((rows, G * d)), canaried((rows, G * d), torch.bfloat16), \
        canaried((rows, G * d), torch.bfloat16)
    src = rnd((rows, G * dp), 400 + d).to(DEV)
    be.prep(src, None, raw_f32=uf, raw_hi=uh, raw_lo=ul, heads=(heads, scales, order))
    want = unpad_heads_ref(src, heads, scales, order, d)
    h, l = split_bf16(want)
    torch.cuda.synchronize()
    assert torch.equal(uf, want) and torch.equal(uh, h) and torch.equal(ul, l)
    assert all(tail_untouched(b) for b in (pfb, phb, plb, ufb, uhb, ulb))


# ------------------------------------------------------------------------------------ the route against fp64
def _self_ref(qkv, heads, order):
    from oracle import bbdm_oracle as O
    return O.op_attention_nhwc(qkv.double(), heads, bool(order))


@pytest.mark.parametrize("B,T,heads", SHAPES)
@pytest.mark.parametrize("d", PAD_DIMS)
def test_sampling_route_against_fp64(be, d, B, T, heads):
    """KernelExecutor._attention_padded as the sampling engine runs it: self-attention from fp32 qkv into planes (both
    orders, the tensor-core kernels) and into fp32 (the fp32-qkv kernel), cross-attention from fp32 q and k|v."""
    from bbdm_b200.engine import KernelExecutor
    ex = KernelExecutor(be)
    pool = ex._pool(torch.device(DEV), ("pad heads test", d, B, T))
    C = heads * d
    for order, planes in ((0, True), (1, True), (1, False)):
        qkv = rnd((B, 1, T, 3 * C), 500 + d + order, 1.2).to(DEV)
        want = _self_ref(qkv.view(B, T, 3 * C), heads, order)
        oh, ol = torch.empty((B, 1, T, C), dtype=torch.bfloat16, device=DEV), \
            torch.empty((B, 1, T, C), dtype=torch.bfloat16, device=DEV)
        of = torch.full((B, 1, T, C), float("nan"), device=DEV)
        ex._attention_padded(pool, heads, d, (qkv,), order, planes, out_f32=of, out_hi=oh, out_lo=ol)
        torch.cuda.synchronize()
        dv = rel_dev(of.view(B, T, C), want)
        print(f" d {d} order {order} planes {planes}: rel dev {dv:.3e}")
        assert dv < ROUTE_TOL, dv
        h, l = split_bf16(of)
        assert torch.equal(oh, h) and torch.equal(ol, l)
    Tkv = max(1, T // 2 + 13)
    q, kv = rnd((B, 1, T, C), 600 + d, 1.2).to(DEV), rnd((B, 1, Tkv, 2 * C), 601 + d, 1.2).to(DEV)
    want = _cross_ref(q.view(B, T, C).double(), kv.view(B, Tkv, 2 * C).double(), heads, d)
    of = torch.full((B, 1, T, C), float("nan"), device=DEV)
    ex._attention_padded(pool, heads, d, (q, kv), 1, True, out_f32=of)
    torch.cuda.synchronize()
    dv = rel_dev(of.view(B, T, C), want)
    print(f" d {d} cross: rel dev {dv:.3e}")
    assert dv < ROUTE_TOL, dv


@pytest.mark.parametrize("B,T,heads", SHAPES)
@pytest.mark.parametrize("d", PAD_DIMS)
def test_training_functions_against_fp64(be, d, B, T, heads, monkeypatch):
    """AttentionCoreFn (both orders) and CrossAttentionCoreFn forward and backward against fp64 autograd."""
    from bbdm_b200 import train
    monkeypatch.setattr(train, "_BACKEND", be)
    C = heads * d
    H, W = 1, T
    for order in (0, 1):
        qkv = rnd((B, 3 * C, H, W), 700 + d + order, 1.2).to(DEV).requires_grad_(True)
        gy = rnd((B, C, H, W), 710 + d, 0.3).to(DEV)
        out = train.AttentionCoreFn.apply(qkv, heads, order)
        out.backward(gy)
        q64 = qkv.detach().double().requires_grad_(True)
        ref = _self_ref(q64.permute(0, 2, 3, 1).reshape(B, T, 3 * C), heads, order)
        ref.backward(gy.double().permute(0, 2, 3, 1).reshape(B, T, C))
        d_out = rel_dev(out.permute(0, 2, 3, 1).reshape(B, T, C), ref.detach())
        d_grad = rel_dev(qkv.grad, q64.grad)
        print(f" d {d} order {order}: out {d_out:.3e} dqkv {d_grad:.3e}")
        assert d_out < ROUTE_TOL and d_grad < ROUTE_TOL, (d_out, d_grad)
    Tkv = max(1, T // 2 + 13)
    q = rnd((B, C, H, W), 720 + d, 1.2).to(DEV).requires_grad_(True)
    kv = rnd((B, 2 * C, 1, Tkv), 721 + d, 1.2).to(DEV).requires_grad_(True)
    gy = rnd((B, C, H, W), 722 + d, 0.3).to(DEV)
    out = train.CrossAttentionCoreFn.apply(q, kv, heads)
    out.backward(gy)
    q64, kv64 = q.detach().double().requires_grad_(True), kv.detach().double().requires_grad_(True)
    ref = _cross_ref(q64.permute(0, 2, 3, 1).reshape(B, T, C), kv64.permute(0, 2, 3, 1).reshape(B, Tkv, 2 * C), heads, d)
    ref.backward(gy.double().permute(0, 2, 3, 1).reshape(B, T, C))
    devs = (rel_dev(out.permute(0, 2, 3, 1).reshape(B, T, C), ref.detach()), rel_dev(q.grad, q64.grad),
            rel_dev(kv.grad, kv64.grad))
    print(f" d {d} cross: out {devs[0]:.3e} dq {devs[1]:.3e} dkv {devs[2]:.3e}")
    assert max(devs) < ROUTE_TOL, devs


# ------------------------------------------------------------------------------------ drop-in models
@pytest.mark.parametrize("tag", list(PAD_HEAD_CONFIGS))
def test_pad_head_model_matches_reference_fixture(tag):
    g = load(tag)
    net = build(PAD_HEAD_CONFIGS[tag])
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
@pytest.mark.parametrize("tag", ["mid_hd20", "mid_hd60", "mid_st_hd36"])
def test_pad_head_training_step_matches_stock_graph(tag, monkeypatch):
    """Loss and every parameter gradient of one training step on the native path against the stock-PyTorch graph
    (TF32 off), with the repacks and the attention kernels run and no library-path warning.  Bounds as in
    test_gpu_attention_head_dims.py.  model_channels 64 (train_cfg): the conv bias gradients of 32-channel ResBlocks
    do not match the stock graph whatever the attention (input_blocks.2.0.in_layers.2.bias), which is not this
    route's to test."""
    import bbdm_b200.unet as U
    from bbdm_b200 import cabi, train
    net = build(train_cfg(tag), train=True)
    inputs = _fixture_inputs(tag)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    rec = _HeadsRecorder(cabi.CudaBackend())
    monkeypatch.setattr(train, "_BACKEND", rec)
    res = {}
    for native in (True, False):
        monkeypatch.setattr(U, "NATIVE_TRAIN_CONV", native)
        res[native] = _step(net, inputs)
    assert not res[True][2], res[True][2]
    want = {"prep heads pad", "prep heads unpad", "attention_bwd"}
    want |= {"attention_cross", "attention_cross_bwd"} if "_st_" in tag else set()
    assert want <= rec.calls, want - rec.calls
    loss_n, loss_s = float(res[True][0]), float(res[False][0])
    devs = {n: rel_dev(res[True][1][n], res[False][1][n]) for n in res[False][1]}
    worst = max(devs, key=devs.get)
    print(f"\n[{tag}] loss native {loss_n:.7f} stock {loss_s:.7f}; worst grad vs stock {worst} {devs[worst]:.3e}")
    assert abs(loss_n - loss_s) < 1e-4 * abs(loss_s)
    assert devs[worst] < 3e-4


def test_pad_head_graphed_and_checkpointed_steps_are_bit_identical():
    """mid_st_hd20: the use_checkpoint step and the graphed step reproduce the plain eager step bit for bit."""
    from bbdm_b200 import train_graph
    net = build(train_cfg("mid_st_hd20"), train=True)
    inputs = _fixture_inputs("mid_st_hd20")
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


def test_pad_head_training_step_allocates_no_attention_matrix():
    """AttentionCoreFn forward + backward at T = 4096 (64 x 64 map), 8 heads of 20, B = 2: the peak above the inputs is
    a few padded-qkv-sized buffers, below one [B * heads, T, T] fp32 matrix and far below the stock core's peak."""
    from bbdm_b200 import train
    from bbdm_b200.unet import AttentionBlock
    B, heads, d, H, W = 2, 8, 20, 64, 64
    C, T = heads * d, H * W
    qkv = rnd((B, 3 * C, H, W), 250, 1.0).to(DEV)
    gy = rnd((B, C, H, W), 251, 0.3).to(DEV)

    def peak(fn):
        x = qkv.clone().requires_grad_(True)
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = fn(x)
        out.backward(gy.view(out.shape))
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, x.grad

    matrix = B * heads * T * T * 4
    native, g_n = peak(lambda x: train.attention_core(x, heads, False))
    stock, g_s = peak(lambda x: AttentionBlock._attention_torch(SimpleNamespace(num_heads=heads, new_order=False),
                                                               x.view(B, 3 * C, T)))
    print(f"\npeak above inputs: native {native / 2**20:.1f} MiB, stock {stock / 2**20:.1f} MiB, "
          f"[B*heads, T, T] fp32 {matrix / 2**20:.1f} MiB")
    assert native < 6 * qkv.numel() * 4 and native < matrix / 10
    assert stock > matrix
    assert rel_dev(g_n, g_s.view(g_n.shape)) < 1e-4


# ------------------------------------------------------------------------------------ launch shadow over the guard
@contextlib.contextmanager
def _guarded(title, required):
    from bbdm_b200 import cabi
    g = Guard(cabi.CudaBackend())
    sh = PadHeadsShadow(g)
    yield sh
    torch.cuda.synchronize()
    print(f"\n{sh.table(title)}\n{g.summary(title)}")
    assert not sh.failures(), sh.failures()[:10]
    assert not g.findings, g.summary(title)
    checked = {c.what for c in sh.checks if c.method == "prep"}
    assert required <= checked, checked


def test_pad_head_sampling_forward_every_launch_against_fp64():
    from bbdm_b200.engine import UNetEngine
    from bbdm_b200.unet import UNetModel
    for tag in ("mid_hd60", "mid_st_hd20"):
        net = UNetModel(**PAD_HEAD_CONFIGS[tag]).eval()
        net.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1234))
        net = net.cuda()
        with _guarded(f"{tag} sampling forward, 32x32, B=2", {"heads pad planes", "heads unpad planes"}) as sh:
            eng = UNetEngine(net, backend=sh)
            eng.refresh_weights()
            sh.register_engine(eng)
            x, y = synth_images((2, 3, 32, 32), 11).cuda(), synth_images((2, 3, 32, 32), 12).cuda()
            out = eng.forward(x, torch.tensor([0, 999], dtype=torch.long).cuda(), y)
            assert torch.isfinite(out).all()


def test_pad_head_training_step_every_launch_against_fp64(monkeypatch):
    from bbdm_b200 import train
    from bbdm_b200.bridge import BridgeOps
    net = build(train_cfg("mid_st_hd20"), train=True)
    x, y, t, nz = _fixture_inputs("mid_st_hd20")
    # training pads into fp32 and planes and unpads into fp32
    with _guarded("mid_st_hd20 training step, 32x32, B=2", {"heads pad", "heads pad planes", "heads unpad"}) as sh:
        monkeypatch.setattr(BridgeOps, "backend_factory", staticmethod(lambda: sh))
        old = train._BACKEND
        train.set_backend(sh)
        try:
            loss, _ = net.p_losses(x, y, y, t, nz)
            loss.backward()
        finally:
            train.set_backend(old)
        assert torch.isfinite(loss)
