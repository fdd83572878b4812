"""-m gpu: attention heads wider than 128 (multiples of 8 up to 256) -- the wide mma.sync forwards (split planes, fp32
qkv, cross-attention) and both wide flash backwards against fp64 with canary tails behind every output, the drop-in
models against the reference-generated fixtures (tests/golden/mid_hd256.npz, mid_hd136*.npz, mid_st_hd160.npz),
training steps against the stock graph, the graphed and checkpointed steps against the eager one, every launch of a
sampling forward and a training step against its fp64 recomputation, and the memory of a T = 4096 training step."""
import gc

import pytest
import torch

from _launch_guard import canaried, tail_untouched
from _launch_shadow import Shadow
from _recipe import fill_state_dict, rel_dev, synth_images
from _wide_heads import WIDE_HEAD_CONFIGS
from oracle import bbdm_oracle as O
from test_gpu_attention_head_dims import (_Recorder, _cross_ref, _fixture_inputs, _same, _shadowed, _step, build,
                                          load, rnd, tol)

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL_PSAMPLE = 1e-4
WIDE_DIMS = [136, 160, 192, 200, 256]


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


def outputs(B, T, C):
    (out, ob), (oh, hb), (ol, lb) = canaried((B, T, C)), canaried((B, T, C), torch.bfloat16), \
        canaried((B, T, C), torch.bfloat16)
    return out, oh, ol, (ob, hb, lb)


def check_outputs(out, oh, ol, bufs, want, bound):
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()
    assert all(tail_untouched(b) for b in bufs)
    d = rel_dev(out, want)
    print(f" rel dev {d:.3e}")
    assert d < bound, d
    h, l = O.bf16_split(out.cpu())
    assert torch.equal(oh.float().cpu(), h) and torch.equal(ol.float().cpu(), l)


def planes(t):
    return tuple(z.to(torch.bfloat16).to(DEV) for z in O.bf16_split(t))


# ------------------------------------------------------------------------------------ forward kernels
SELF_SHAPES = [(2, 100, 2, 0), (1, 257, 1, 1), (1, 1024, 2, 1), (2, 64, 3, 0)]      # B, T, heads, order


@pytest.mark.parametrize("B,T,heads,order", SELF_SHAPES)
@pytest.mark.parametrize("D", WIDE_DIMS)
def test_attention_split_wide(be, D, B, T, heads, order):
    """The pre-split planes form against fp64 on the same planes."""
    C = heads * D
    qkv = rnd((B, T, 3 * C), 170 + D, 1.2)
    hi, lo = O.bf16_split(qkv)
    want = O.op_attention_nhwc((hi + lo).double(), heads, bool(order))
    out, oh, ol, bufs = outputs(B, T, C)
    be.attention_split(hi.to(torch.bfloat16).to(DEV), lo.to(torch.bfloat16).to(DEV), heads, order,
                       out_f32=out, out_hi=oh, out_lo=ol)
    check_outputs(out, oh, ol, bufs, want, tol(T))


@pytest.mark.parametrize("B,T,heads,order", SELF_SHAPES)
@pytest.mark.parametrize("D", WIDE_DIMS)
def test_attention_fp32_qkv_wide(be, D, B, T, heads, order):
    """The fp32-qkv form (q, k scaled by D^-1/4 and split in shared memory)."""
    C = heads * D
    qkv = rnd((B, T, 3 * C), 190 + D, 1.2)
    want = O.op_attention_nhwc(qkv.double(), heads, bool(order))
    out, oh, ol, bufs = outputs(B, T, C)
    be.attention(qkv.to(DEV), heads, order, out_f32=out, out_hi=oh, out_lo=ol)
    check_outputs(out, oh, ol, bufs, want, tol(T))


CROSS_SHAPES = [(2, 100, 77, 2), (1, 257, 1024, 1), (1, 64, 300, 2)]                # B, Tq, Tkv, heads


@pytest.mark.parametrize("B,Tq,Tkv,heads", CROSS_SHAPES)
@pytest.mark.parametrize("D", WIDE_DIMS)
def test_attention_cross_wide(be, D, B, Tq, Tkv, heads):
    C = heads * D
    q, kv = rnd((B, Tq, C), 220 + D, 1.2), rnd((B, Tkv, 2 * C), 221 + D, 1.2)
    qh, ql = O.bf16_split(q)
    kh, kl = O.bf16_split(kv)
    want = _cross_ref((qh + ql).double(), (kh + kl).double(), heads, D)
    out, oh, ol, bufs = outputs(B, Tq, C)
    be.attention_cross(*planes(q), *planes(kv), heads, out_f32=out, out_hi=oh, out_lo=ol)
    check_outputs(out, oh, ol, bufs, want, tol(Tkv))


def test_wide_entry_points_reject_heads_past_256(be):
    """head_dim 264 and 252 (not a multiple of 8) fail with the rule in the message; nothing is written."""
    for D, heads in ((264, 1), (252, 1)):
        C = heads * D
        qkv = torch.zeros((1, 64, 3 * C), device=DEV)
        out, buf = canaried((1, 64, C))
        with pytest.raises(RuntimeError, match="multiple of 8 up to 256"):
            be.attention(qkv, heads, 0, out_f32=out)
        with pytest.raises(RuntimeError, match="multiple of 8 up to 256"):
            be.attention_bwd(qkv, out, out, heads, 0, torch.empty_like(qkv), torch.empty(64, device=DEV),
                             torch.empty(64, device=DEV))
        torch.cuda.synchronize()
        assert torch.isnan(out).all() and tail_untouched(buf)


# ------------------------------------------------------------------------------------ backward kernels
@pytest.mark.parametrize("B,T,heads,order", [(2, 100, 2, 0), (1, 257, 1, 1), (1, 1024, 1, 0), (1, 64, 2, 1)])
@pytest.mark.parametrize("D", WIDE_DIMS)
def test_attention_bwd_wide(be, D, B, T, heads, order):
    Cc = heads * D
    qkv = rnd((B, T, 3 * Cc), 230 + D, 1.5)
    dout = rnd((B, T, Cc), 231 + D, 0.3)
    qd = qkv.double().requires_grad_(True)
    od = O.op_attention_nhwc(qd, heads, bool(order))
    od.backward(dout.double())
    dqkv, buf = canaried((B, T, 3 * Cc))
    (lse, lb), (delta, db) = canaried((B * heads * T,)), canaried((B * heads * T,))
    be.attention_bwd(qkv.to(DEV), od.detach().float().to(DEV), dout.to(DEV), heads, order, dqkv, lse, delta)
    torch.cuda.synchronize()
    assert not torch.isnan(dqkv).any() and not torch.isnan(lse).any() and not torch.isnan(delta).any()
    assert tail_untouched(buf) and tail_untouched(lb) and tail_untouched(db)
    d = rel_dev(dqkv, qd.grad)
    print(f" rel dev {d:.3e}")
    assert d < 2e-5, d


@pytest.mark.parametrize("B,Tq,Tkv,heads", [(2, 100, 77, 2), (1, 257, 130, 1), (1, 64, 1024, 1)])
@pytest.mark.parametrize("D", WIDE_DIMS)
def test_attention_cross_bwd_wide(be, D, B, Tq, Tkv, heads):
    C = heads * D
    q, kv = rnd((B, Tq, C), 240 + D, 1.2), rnd((B, Tkv, 2 * C), 241 + D, 1.2)
    dout = rnd((B, Tq, C), 242 + D, 0.3)
    qd, kvd = q.double().requires_grad_(True), kv.double().requires_grad_(True)
    od = _cross_ref(qd, kvd, heads, D)
    od.backward(dout.double())
    (dq, qb), (dkv, kb) = canaried((B, Tq, C)), canaried((B, Tkv, 2 * C))
    (lse, lb), (delta, db) = canaried((B * heads * Tq,)), canaried((B * heads * Tq,))
    be.attention_cross_bwd(q.to(DEV), kv.to(DEV), od.detach().float().to(DEV), dout.to(DEV), heads, dq, dkv, lse,
                           delta)
    torch.cuda.synchronize()
    assert not torch.isnan(dq).any() and not torch.isnan(dkv).any()
    assert all(tail_untouched(b) for b in (qb, kb, lb, db))
    dd = (rel_dev(dq, qd.grad), rel_dev(dkv, kvd.grad))
    print(f" rel dev dq {dd[0]:.3e} dkv {dd[1]:.3e}")
    assert max(dd) < 2e-5, dd


# ------------------------------------------------------------------------------------ drop-in models
@pytest.mark.parametrize("tag", list(WIDE_HEAD_CONFIGS))
def test_wide_head_model_matches_reference_fixture(tag):
    g = load(tag)
    net = build(WIDE_HEAD_CONFIGS[tag])
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
@pytest.mark.parametrize("tag", ["mid_hd256", "mid_st_hd160"])
def test_wide_head_training_step_matches_stock_graph(tag, monkeypatch):
    """Loss and every parameter gradient of one training step on the native path against the stock-PyTorch graph
    (TF32 off); the attention cores ran on the native Functions and no layer took the library path.  Bounds as in
    test_gpu_attention_head_dims.py."""
    import bbdm_b200.unet as U
    from bbdm_b200 import cabi, train
    net = build(WIDE_HEAD_CONFIGS[tag], train=True)
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
    assert "attention_tc" not in rec.calls
    loss_n, loss_s = float(res[True][0]), float(res[False][0])
    devs = {n: rel_dev(res[True][1][n], res[False][1][n]) for n in res[False][1]}
    worst = max(devs, key=devs.get)
    print(f"\n[{tag}] loss native {loss_n:.7f} stock {loss_s:.7f}; worst grad vs stock {worst} {devs[worst]:.3e}")
    assert abs(loss_n - loss_s) < 1e-4 * abs(loss_s)
    assert devs[worst] < 3e-4


def test_wide_head_graphed_and_checkpointed_steps_are_bit_identical():
    """mid_st_hd160: the use_checkpoint step and the graphed step reproduce the plain eager step bit for bit."""
    from bbdm_b200 import train_graph
    net = build(WIDE_HEAD_CONFIGS["mid_st_hd160"], train=True)
    inputs = _fixture_inputs("mid_st_hd160")
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


def test_wide_head_training_step_allocates_no_attention_matrix():
    """AttentionCoreFn forward + backward at T = 4096 (64 x 64 map), one head of 256, B = 2: the peak above the inputs
    is a few qkv-sized buffers (its NHWC copy, the gradient, the output), below one [B * heads, T, T] fp32 matrix and far
    below the stock core's peak, which keeps such matrices for its backward (measured on an H100: 64.1 against
    672.0 MiB)."""
    from bbdm_b200 import train
    from bbdm_b200.unet import AttentionBlock
    from types import SimpleNamespace
    B, C, H, W = 2, 256, 64, 64
    T = H * W
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
        p = torch.cuda.max_memory_allocated() - base
        return p, x.grad

    matrix = B * T * T * 4
    native, g_n = peak(lambda x: train.attention_core(x, 1, False))
    stock, g_s = peak(lambda x: AttentionBlock._attention_torch(SimpleNamespace(num_heads=1, new_order=False),
                                                               x.view(B, 3 * C, T)))
    print(f"\npeak above inputs: native {native / 2**20:.1f} MiB, stock {stock / 2**20:.1f} MiB, "
          f"[B*heads, T, T] fp32 {matrix / 2**20:.1f} MiB")
    assert native < 3 * qkv.numel() * 4 and native < matrix
    assert stock > matrix and native < stock / 5
    assert rel_dev(g_n, g_s.view(g_n.shape)) < 1e-4


# ------------------------------------------------------------------------------------ launch shadow
def test_wide_head_sampling_forward_every_launch_against_fp64():
    from bbdm_b200 import cabi
    from bbdm_b200.engine import UNetEngine
    from bbdm_b200.unet import UNetModel
    net = UNetModel(**WIDE_HEAD_CONFIGS["mid_st_hd160"]).eval()
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
    print(f"\n{sh.table('mid_st_hd160 sampling forward, 32x32, B=2')}")
    assert not fails, fails[:10]
    checked = {c.method for c in sh.checks}
    assert {"attention_split", "attention_cross"} <= checked, checked


def test_wide_head_training_step_every_launch_against_fp64(monkeypatch):
    net = build(WIDE_HEAD_CONFIGS["mid_hd256"], train=True)
    x, y, t, nz = _fixture_inputs("mid_hd256")
    with _shadowed(monkeypatch) as sh:
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
    torch.cuda.synchronize()
    fails = sh.failures()
    print(f"\n{sh.table('mid_hd256 training step, 32x32, B=2')}")
    assert torch.isfinite(loss)
    assert not fails, fails[:10]
    checked = {c.method for c in sh.checks}
    assert {"attention", "attention_bwd"} <= checked, checked
