"""-m gpu: attention heads wider than 256 on the GEMM-composed route -- softmax_rows_split's backward mode
(bbdm_softmax_rows_bwd) against fp64 with canary tails, both training Functions forward and backward
against fp64 autograd, the drop-in models against the reference-generated fixtures (tests/golden/mid_hd512.npz,
mid_hd1024.npz, mid_hd336_new.npz, mid_st_hd384.npz), a Template-LBBDM-f4-shaped UNet with single heads against its
fp64 module, training steps against the stock graph, the graphed and checkpointed steps against the eager one, every
launch of a sampling forward and a training step against its fp64 recomputation, and the memory of a T = 4096 core."""
import gc
from types import SimpleNamespace

import pytest
import torch

from _gemm_heads import GEMM_HEAD_CONFIGS
from _launch_guard import canaried, tail_untouched
from _launch_shadow import Shadow, pair_well_formed
from _launch_shadow_gemm_heads import GemmHeadsShadow
from _recipe import UNET_CONFIGS, fill_state_dict, rel_dev, synth_images
from oracle import bbdm_oracle as O
from test_gpu_attention_head_dims import _Recorder, _same, _step, build, load, rnd

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL_PSAMPLE = 1e-4


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


# ------------------------------------------------------------------------------------ softmax backward kernel
@pytest.mark.parametrize("rows,cols,valid", [(100, 128, 128), (100, 128, 100), (257, 1024, 1000), (64, 4096, 4096),
                                             (33, 64, 1), (16, 64, 61)])
def test_softmax_rows_split_grad(be, rows, cols, valid):
    """The backward mode (bbdm_softmax_rows_bwd): the planes of ds = scale p (dp - sum p dp) against fp64 over the block,
    a split pair, +0 past valid_cols, nothing written past the planes, the same bits on a second launch."""
    from _emu_backend_gemm_heads import softmax_rows_bwd64
    s = rnd((rows, cols), 1, 3.0).to(DEV)
    dp = rnd((rows, cols), 2, 1.0).to(DEV)
    scale = 0.05
    (hi, hb), (lo, lb) = canaried((rows, cols), torch.bfloat16), canaried((rows, cols), torch.bfloat16)
    be.softmax_rows_split(s, scale, hi, lo, valid_cols=valid, grad=dp)
    torch.cuda.synchronize()
    assert tail_untouched(hb) and tail_untouched(lb)
    _, ds64 = softmax_rows_bwd64(s, dp, scale, valid)
    got = hi.double() + lo.double()
    dev = rel_dev(got, ds64)
    print(f"\n ds rel dev {dev:.2e}")
    assert dev < 2e-5
    assert not pair_well_formed(hi, lo).any()
    assert not (hi[:, valid:].view(torch.int16).any() or lo[:, valid:].view(torch.int16).any())
    hi2, lo2 = torch.empty_like(hi), torch.empty_like(lo)
    be.softmax_rows_split(s, scale, hi2, lo2, valid_cols=valid, grad=dp)
    assert torch.equal(hi2, hi) and torch.equal(lo2, lo)


# ------------------------------------------------------------------------------------ the training Functions
def _attn64(q, k, v):
    """fp64 softmax(q k^T d^-1/2) v per head of [B, T, heads, d] tensors."""
    d = q.shape[-1]
    w = torch.einsum("bthd,bshd->bhts", q, k) * d ** -0.5
    return torch.einsum("bhts,bshd->bthd", w.softmax(-1), v)


@pytest.mark.parametrize("d,B,T,heads,order", [(264, 2, 100, 2, 0), (336, 2, 16, 2, 1), (512, 2, 1024, 1, 0),
                                               (1024, 1, 256, 1, 1), (512, 1, 4096, 1, 1), (336, 1, 100, 3, 1)])
def test_attention_core_fn_gemm_route(be, d, B, T, heads, order):
    from bbdm_b200 import train
    side = int(T ** 0.5)
    C = heads * d
    qkv = rnd((B, 3 * C, side, side), 11, 1.0).to(DEV).requires_grad_(True)
    gy = rnd((B, C, side, side), 12, 0.3).to(DEV)
    out = train.AttentionCoreFn.apply(qkv, heads, order)
    out.backward(gy)
    torch.cuda.synchronize()
    be.check_fault()
    q64 = qkv.detach().double().requires_grad_(True)
    t = q64.flatten(2).transpose(1, 2)                                    # [B, T, 3C]
    v = t.view(B, T, 3, heads, d) if order else t.view(B, T, heads, 3, d).transpose(2, 3)
    o64 = _attn64(v[:, :, 0], v[:, :, 1], v[:, :, 2]).reshape(B, T, C).transpose(1, 2).reshape(out.shape)
    o64.backward(gy.double())
    df, db = rel_dev(out, o64), rel_dev(qkv.grad, q64.grad)
    print(f"\n d {d} T {T}: out rel dev {df:.2e}, dqkv rel dev {db:.2e}")
    assert df < 3e-5 and db < 1e-4


@pytest.mark.parametrize("d,B,Tq,Tkv,heads", [(384, 2, 100, 25, 2), (512, 1, 1024, 64, 1), (264, 2, 16, 100, 1)])
def test_cross_attention_core_fn_gemm_route(be, d, B, Tq, Tkv, heads):
    from bbdm_b200 import train
    sq, skv = int(Tq ** 0.5), int(Tkv ** 0.5)
    C = heads * d
    q = rnd((B, C, sq, sq), 21, 1.0).to(DEV).requires_grad_(True)
    kv = rnd((B, 2 * C, skv, skv), 22, 1.0).to(DEV).requires_grad_(True)
    gy = rnd((B, C, sq, sq), 23, 0.3).to(DEV)
    out = train.CrossAttentionCoreFn.apply(q, kv, heads)
    out.backward(gy)
    torch.cuda.synchronize()
    q64, kv64 = (z.detach().double().requires_grad_(True) for z in (q, kv))
    qt = q64.flatten(2).transpose(1, 2).reshape(B, Tq, heads, d)
    kvt = kv64.flatten(2).transpose(1, 2).reshape(B, Tkv, 2, heads, d)
    o64 = _attn64(qt, kvt[:, :, 0], kvt[:, :, 1]).reshape(B, Tq, C).transpose(1, 2).reshape(out.shape)
    o64.backward(gy.double())
    devs = rel_dev(out, o64), rel_dev(q.grad, q64.grad), rel_dev(kv.grad, kv64.grad)
    print(f"\n d {d} Tq {Tq} Tkv {Tkv}: out / dq / dkv rel dev {devs}")
    assert devs[0] < 3e-5 and max(devs[1:]) < 1e-4


def test_gemm_route_core_memory_does_not_grow_with_batch():
    """AttentionCoreFn forward + backward at T = 4096 (64 x 64), one head of 512: the peak above the inputs is the qkv
    copy, its gradient, the output and dO copies (per batch) plus one image-head's scratch (independent of B).  The stock
    core keeps [B, T, T] fp32 matrices for its backward."""
    from bbdm_b200 import train
    from bbdm_b200.unet import AttentionBlock
    C, H, W, d = 512, 64, 64, 512
    T, tkvp = H * W, 4096

    def peak(fn, B):
        qkv = rnd((B, 3 * C, H, W), 250, 1.0).to(DEV).requires_grad_(True)
        gy = rnd((B, C, H, W), 251, 0.3).to(DEV)
        torch.cuda.synchronize()
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = fn(qkv)
        out.backward(gy.view(out.shape))
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    # per image: the qkv NHWC copy, the output, the dO copy, dqkv and the gradient autograd accumulates from it
    per_image = (3 * C + C + C + 3 * C + 3 * C) * T * 4
    scratch = (2 * T * tkvp * 4 + 4 * T * tkvp * 2                        # s, dp; the P and dS planes
               + 4 * tkvp * d * 4 + 12 * tkvp * d * 2 + 4 * T * d * 4 + 2 * tkvp * d * 4)   # padded operands, planes
    native = {B: peak(lambda x: train.attention_core(x, 1, False), B) for B in (1, 2, 4)}
    stock = peak(lambda x: AttentionBlock._attention_torch(SimpleNamespace(num_heads=1, new_order=False),
                                                            x.view(x.shape[0], 3 * C, T)), 2)
    print(f"\npeak above inputs (MiB): native {[round(v / 2**20, 1) for v in native.values()]}, stock (B=2) "
          f"{stock / 2**20:.1f}; bound per image {per_image / 2**20:.1f} + scratch {scratch / 2**20:.1f}")
    for B, v in native.items():
        assert v <= B * per_image + scratch, (B, v)
    assert native[4] - native[1] <= 3 * per_image
    assert stock > 2 * T * T * 4


# ------------------------------------------------------------------------------------ models
@pytest.mark.parametrize("tag", list(GEMM_HEAD_CONFIGS))
def test_gemm_head_model_matches_reference_fixture(tag):
    g = load(tag)
    net = build(GEMM_HEAD_CONFIGS[tag])
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


def test_lbbdm_f4_single_head_unet_samples_natively():
    """Template-LBBDM-f4's UNet with num_heads 1, num_head_channels -1: heads of 512 at 32x32 and 16x16 and of 1024 at
    8x8 and in the middle block.  The engine's forward against the fp64 module (oracle) with the same weights."""
    from bbdm_b200 import cabi
    from bbdm_b200.engine import UNetEngine
    from bbdm_b200.unet import UNetModel
    cfg = dict(UNET_CONFIGS["lbbdm_f4"], num_heads=1, num_head_channels=-1)
    net = UNetModel(**cfg).eval()
    net.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1234))
    net = net.cuda()
    rec = _Recorder(cabi.CudaBackend())
    eng = UNetEngine(net, backend=rec)
    x = synth_images((2, 3, 64, 64), 11).cuda()
    t = torch.tensor([5, 700], dtype=torch.long).cuda()
    out = eng.forward(x, t)
    torch.cuda.synchronize()
    sd = {k: v.cpu().double() for k, v in net.state_dict().items()}
    want = O.unet_forward(sd, O.unet_cfg(**cfg), x.cpu().double(), t.cpu())
    d = rel_dev(out, want)
    print(f"\nLBBDM-f4 single-head UNet vs fp64: {d:.3e}")
    assert {"softmax_rows_split", "split_grad"} <= rec.calls
    assert not rec.calls & {"attention", "attention_split", "attention_tc"}
    assert d < TOL_PSAMPLE


# ------------------------------------------------------------------------------------ training
def _synthetic_inputs(cfg, B=2):
    S = cfg["image_size"]
    x, y = synth_images((B, 3, S, S), 31).cuda(), synth_images((B, 3, S, S), 32).cuda()
    t = torch.tensor([(17 + 311 * i) % 1000 for i in range(B)], dtype=torch.long).cuda()
    nz = torch.randn(x.shape, generator=torch.Generator().manual_seed(77)).cuda()
    return x, y, t, nz


@pytest.mark.parametrize("tag", ["mid_hd512", "mid_st_hd384"])
def test_gemm_head_training_step_matches_stock_graph(tag, monkeypatch):
    """Loss and every parameter gradient of one training step on the native path against the stock-PyTorch graph
    (TF32 off): the attention cores ran the GEMM route, no flash kernel and no library path.  mid_hd336_new is not
    compared here: its 32-channel ResBlocks have one channel per GroupNorm group, so their conv1 bias gradients are zero
    up to rounding in both graphs; its masked key axis is checked launch by launch below."""
    import bbdm_b200.unet as U
    from bbdm_b200 import cabi, train
    net = build(GEMM_HEAD_CONFIGS[tag], train=True)
    inputs = _synthetic_inputs(GEMM_HEAD_CONFIGS[tag])
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    rec = _Recorder(cabi.CudaBackend())
    monkeypatch.setattr(train, "_BACKEND", rec)
    res = {}
    for native in (True, False):
        monkeypatch.setattr(U, "NATIVE_TRAIN_CONV", native)
        res[native] = _step(net, inputs)
    assert not res[True][2], res[True][2]
    assert {"softmax_rows_split", "conv_wgrad"} <= rec.calls
    assert not rec.calls & {"attention", "attention_bwd", "attention_cross", "attention_cross_bwd", "attention_tc"}
    loss_n, loss_s = float(res[True][0]), float(res[False][0])
    devs = {n: rel_dev(res[True][1][n], res[False][1][n]) for n in res[False][1]}
    worst = max(devs, key=devs.get)
    print(f"\n[{tag}] loss native {loss_n:.7f} stock {loss_s:.7f}; worst grad vs stock {worst} {devs[worst]:.3e}")
    assert abs(loss_n - loss_s) < 1e-4 * abs(loss_s)
    assert devs[worst] < 3e-4


def test_gemm_head_graphed_and_checkpointed_steps_are_bit_identical():
    """mid_st_hd384: the use_checkpoint step and the graphed step reproduce the plain eager step bit for bit."""
    from bbdm_b200 import train_graph
    net = build(GEMM_HEAD_CONFIGS["mid_st_hd384"], train=True)
    inputs = _synthetic_inputs(GEMM_HEAD_CONFIGS["mid_st_hd384"])
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
def test_gemm_head_sampling_forward_every_launch_against_fp64():
    from bbdm_b200 import cabi
    from bbdm_b200.engine import UNetEngine
    from bbdm_b200.unet import UNetModel
    net = UNetModel(**GEMM_HEAD_CONFIGS["mid_st_hd384"]).eval()
    net.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1234))
    net = net.cuda()
    sh = Shadow(cabi.CudaBackend())
    eng = UNetEngine(net, backend=sh)
    eng.refresh_weights()
    sh.register_engine(eng)
    x, y = synth_images((2, 3, 32, 32), 11).cuda(), synth_images((2, 3, 32, 32), 12).cuda()
    out = eng.forward(x, torch.tensor([0, 999], dtype=torch.long).cuda(), y)
    assert torch.isfinite(out).all()
    fails = sh.failures()
    print(f"\n{sh.table('mid_st_hd384 sampling forward, 32x32, B=2')}")
    assert not fails, fails[:10]
    assert "softmax_rows_split" in {c.method for c in sh.checks}


def test_gemm_head_training_step_every_launch_against_fp64(monkeypatch):
    """A 40x40 UNet with 2 heads of 352 in the new order: T = 100 tokens, the key axis padded to 128 and masked (the
    shadow's softmax references honour valid_cols and the backward mode).  Not mid_hd336_new: its 32-channel ResBlocks have one channel
    per GroupNorm group, so their conv1 bias gradients (split_grad's column sums) are zero up to rounding."""
    from bbdm_b200 import cabi, train
    cfg = dict(GEMM_HEAD_CONFIGS["mid_hd336_new"], model_channels=64, channel_mult=(1, 2, 11))
    net = build(cfg, train=True)
    x, y, t, nz = _synthetic_inputs(cfg)
    sh = GemmHeadsShadow(cabi.CudaBackend())
    monkeypatch.setattr(train, "_BACKEND", sh)
    loss, _ = net.p_losses(x, y, y, t, nz)
    loss.backward()
    torch.cuda.synchronize()
    fails = sh.failures()
    print(f"\n{sh.table('2 x 352 heads training step, 40x40, B=2')}")
    assert torch.isfinite(loss)
    assert not fails, fails[:10]
    assert "conv_wgrad" in {c.method for c in sh.checks}
    assert any(c.what == "score gradient hi + lo" for c in sh.checks)
