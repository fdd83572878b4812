"""-m gpu: channel counts that are multiples of 32 but not of 64 on the tensor-core kernels -- conv_umma in every form
and conv_wgrad against fp64 with canary tails behind every output, the training Functions against fp64 autograd, the
drop-in model against the reference-generated fixtures (tests/golden/mid_w*.npz), training steps against the stock
graph, the graphed and checkpointed steps against the eager one, and every launch of a sampling forward and a training
step against its fp64 recomputation."""
import contextlib
import gc
import os
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _launch_guard import CANARY, canaried as _canaried, tail_untouched
from _launch_shadow import Shadow
from _recipe import bb_namespace, fill_state_dict, rel_dev, synth_images
from _widths import WIDTH_CONFIGS
from oracle import bbdm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
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


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).float()


def split(x):
    h, l = O.bf16_split(x)
    return h.to(torch.bfloat16).to(DEV).contiguous(), l.to(torch.bfloat16).to(DEV).contiguous()


def canaried(shape, dtype=torch.float32):
    """(view of shape, whole buffer): the view and the tail of CANARY_N elements behind it hold CANARY."""
    return _canaried(shape, dtype, DEV, fill=CANARY)


# ------------------------------------------------------------------------------------------ conv_umma
# (B, H, W, Cin, Cout, form, Cin2, res_mode, out_split, stats).  form: t9 / t1 / t4o0 / t4o-1 (2x2 window at origin
# 0 / -1) / up2 (fused nearest-2x).  Maps of 64x64 at batch 4 take the 128-wide N tile where Cout % 128 is 0 or 96,
# 12x12 and smaller maps the 64-wide one (too few M tiles); Cout 160 / 288 always 64.
UMMA_CASES = [
    (4, 64, 64, 96, 96, "t9", 0, 0, False, True),
    (1, 12, 12, 96, 96, "t9", 0, 1, False, False),
    (2, 7, 9, 32, 32, "t9", 0, 0, False, False),
    (2, 12, 12, 64, 96, "t9", 0, 1, True, True),
    (2, 12, 12, 96, 64, "t9", 0, 0, False, True),
    (4, 32, 32, 160, 224, "t9", 0, 1, False, True),
    (4, 64, 64, 224, 224, "t9", 96, 0, False, True),
    (2, 12, 12, 224, 128, "t9", 288, 0, True, False),
    (2, 20, 20, 224, 160, "t1", 0, 0, True, False),
    (2, 16, 16, 288, 288, "t1", 0, 1, False, True),
    (4, 32, 32, 128, 224, "t1", 0, 3, False, False),
    (2, 16, 16, 96, 96, "t1", 0, 2, False, False),
    (2, 16, 16, 384, 96, "t4o-1", 0, 0, False, True),
    (2, 10, 14, 896, 224, "t4o-1", 0, 0, True, False),
    (2, 16, 16, 96, 160, "t4o0", 0, 0, False, False),
    (2, 10, 12, 96, 224, "up2", 0, 0, False, True),
    (2, 16, 16, 224, 96, "up2", 0, 2, False, False),
    (1, 8, 8, 160, 32, "up2", 0, 1, True, False),
]


def _umma_reference(x, w, bias, form, x2, w2, bias2, res, res_mode):
    """fp64 NHWC result; x [B,H,W,Cin], w OIHW."""
    xd = x.double().permute(0, 3, 1, 2)
    if form == "t9":
        o = F.conv2d(xd, w.double(), padding=1)
    elif form == "t1":
        o = F.conv2d(xd, w.double())
    elif form == "up2":
        o = F.conv2d(F.interpolate(xd, scale_factor=2, mode="nearest"), w.double(), padding=1)
    else:
        pad = (0, 1, 0, 1) if form == "t4o0" else (1, 0, 1, 0)
        o = F.conv2d(F.pad(xd, pad), w.double())
    o = o + bias.double()[None, :, None, None]
    if x2 is not None:
        o = o + F.conv2d(x2.double().permute(0, 3, 1, 2), w2.double()) + bias2.double()[None, :, None, None]
    o = o.permute(0, 2, 3, 1)
    if res_mode == 1:
        o = o + res.double()
    elif res_mode == 2:
        o = o + res.double().repeat_interleave(2, 1).repeat_interleave(2, 2)
    elif res_mode == 3:
        r = res.double()
        o = o + 0.25 * (r[:, 0::2, 0::2] + r[:, 0::2, 1::2] + r[:, 1::2, 0::2] + r[:, 1::2, 1::2])
    return o


@pytest.mark.parametrize("case", UMMA_CASES, ids=lambda c: "x".join(map(str, c[:5])) + f"-{c[5]}-k2{c[6]}-r{c[7]}"
                         + ("-split" if c[8] else "") + ("-stats" if c[9] else ""))
def test_conv_umma_widths(be, case):
    from bbdm_b200.weights import upsample_phase_weights
    B, H, W, Cin, Cout, form, Cin2, res_mode, out_split, stats = case
    taps, k = {"t9": (9, 3), "t1": (1, 1), "t4o0": (4, 2), "t4o-1": (4, 2), "up2": (4, 3)}[form]
    f = 2 if form == "up2" else 1
    OH, OW = f * H, f * W
    x = rnd((B, H, W, Cin), 1)
    w = rnd((Cout, Cin, k, k), 2, 1.0 / (Cin * k * k) ** 0.5)
    bias = rnd((Cout,), 3, 0.1)
    planes = upsample_phase_weights(w).permute(2, 0, 1) if form == "up2" else w.permute(2, 3, 0, 1).reshape(-1, Cout, Cin)
    a_hi, a_lo = split(x)
    w_hi, w_lo = split(planes.contiguous())
    kw = {}
    x2 = w2 = bias2 = None
    if Cin2:
        x2, w2, bias2 = rnd((B, H, W, Cin2), 4), rnd((Cout, Cin2, 1, 1), 5, 1.0 / Cin2 ** 0.5), rnd((Cout,), 6, 0.1)
        a2_hi, a2_lo = split(x2)
        w2_hi, w2_lo = split(w2.reshape(1, Cout, Cin2).contiguous())
        kw.update(Cin2=Cin2, a2_hi=a2_hi, a2_lo=a2_lo, w2_hi=w2_hi, w2_lo=w2_lo, bias2=bias2.to(DEV))
    res = None
    if res_mode:
        rs = {1: (OH, OW), 2: (OH // 2, OW // 2), 3: (2 * OH, 2 * OW)}[res_mode]
        res = rnd((B, rs[0], rs[1], Cout), 7)
        kw.update(residual=res.to(DEV), res_mode=res_mode)
    if form.startswith("t4"):
        kw.update(window_origin=0 if form == "t4o0" else -1)
    out, obuf = canaried((B, OH, OW, Cout))
    oh = ol = hbuf = lbuf = part = pbuf = None
    if out_split:
        oh, hbuf = canaried((B, OH, OW, Cout), torch.bfloat16)
        ol, lbuf = canaried((B, OH, OW, Cout), torch.bfloat16)
    rows = 0
    if stats:
        rows = be.conv_geometry(H, W)[3] * f * f
        assert rows > 0
        part, pbuf = canaried((B * rows, Cout, 2))
    be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=taps, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo,
                 bias=bias.to(DEV), out=out, out_hi=oh, out_lo=ol, passes=3, stats_partial=part,
                 upsample2x=form == "up2", **kw)
    torch.cuda.synchronize()
    be.check_fault()
    want = _umma_reference(x, w, bias, form, x2, w2, bias2, res, res_mode)
    d = rel_dev(out, want)
    print(f"\n[conv_umma widths] {case}: rel dev {d:.3e}")
    assert not torch.isnan(out).any() and d < 3e-5, d
    assert tail_untouched(obuf)
    if out_split:
        assert tail_untouched(hbuf) and tail_untouched(lbuf)
        assert rel_dev(oh.float() + ol.float(), out) < 1e-5
    if stats:
        assert tail_untouched(pbuf)
        s = part.view(B, rows, Cout, 2).double().sum(1)
        o = out.double().reshape(B, -1, Cout)
        assert rel_dev(s[..., 0], o.sum(1)) < 1e-5 and rel_dev(s[..., 1], (o * o).sum(1)) < 1e-5


@pytest.mark.parametrize("Cin", [96, 224, 160])
def test_conv_umma_padded_nchw_head(be, Cin):
    """The image head: 3x3 conv of Cin (a multiple of 32) to 3 channels on one zero-padded 64-wide N tile, stored NCHW."""
    B, H, W, C = 2, 16, 16, 3
    x = rnd((B, H, W, Cin), 11)
    w = rnd((C, Cin, 3, 3), 12, 1.0 / (9 * Cin) ** 0.5)
    bias = rnd((C,), 13, 0.1)
    wp = torch.zeros(9, 64, Cin)
    wp[:, :C] = w.permute(2, 3, 0, 1).reshape(9, C, Cin)
    bp = torch.zeros(64)
    bp[:C] = bias
    a_hi, a_lo = split(x)
    w_hi, w_lo = split(wp)
    out, obuf = canaried((B, C, H, W))
    be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=64, taps=9, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo,
                 bias=bp.to(DEV), out=out, passes=3, out_nchw_channels=C)
    torch.cuda.synchronize()
    be.check_fault()
    want = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), bias.double(), padding=1)
    assert rel_dev(out, want) < 3e-5 and tail_untouched(obuf)


# ------------------------------------------------------------------------------------------ conv_wgrad
def _wgrad64(a, g, taps, origin):
    B, H, W, Cin = a.shape
    Cout = g.shape[3]
    k = {1: 1, 4: 2, 9: 3}[taps]
    o = -1 if taps == 9 else origin
    ap = F.pad(a.double(), (0, 0, 1, 1, 1, 1))
    gr = g.double().reshape(-1, Cout).t()
    dw = torch.empty((Cout, Cin, k, k), dtype=torch.float64, device=a.device)
    for ky in range(k):
        for kx in range(k):
            dw[:, :, ky, kx] = gr @ ap[:, 1 + o + ky:1 + o + ky + H, 1 + o + kx:1 + o + kx + W].reshape(-1, Cin)
    return dw


# (B, H, W, Cin, Cout, taps, origin): ragged pixel counts P, N tiles of 128 (Cin 96 / 224) and 64 (32 / 160 / 288)
WGRAD_CASES = [
    (3, 12, 12, 96, 96, 9, 0), (2, 7, 9, 32, 32, 9, 0), (2, 24, 40, 160, 224, 9, 0), (3, 7, 7, 224, 96, 1, 0),
    (6, 4, 4, 288, 160, 1, 0), (2, 16, 16, 64, 96, 9, 0), (2, 16, 16, 96, 64, 9, 0), (2, 10, 14, 384, 96, 4, -1),
    (3, 9, 11, 96, 224, 4, 0), (2, 12, 12, 224, 384, 9, 0), (4, 32, 32, 96, 288, 1, 0),
]


@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: "x".join(map(str, c)))
def test_conv_wgrad_widths(be, case):
    from bbdm_b200.train import _transposed_planes
    B, H, W, Cin, Cout, taps, origin = case
    a = rnd((B, H, W, Cin), 21).to(DEV)
    g = rnd((B, H, W, Cout), 22, 0.1).to(DEV)
    P = B * H * W
    a_hi, a_lo = (t.to(torch.bfloat16) for t in O.bf16_split(a))
    ht, lt = _transposed_planes(Cout, P, a.device)
    be.split_grad(g.reshape(P, Cout).contiguous(), None, None, ht, lt)
    _, fl = be.wgrad_workspace(B, H, W, Cin, Cout, taps)
    ws = torch.empty(fl, device=DEV)
    k = {1: 1, 4: 2, 9: 3}[taps]
    dw, dbuf = canaried((Cout, Cin, k, k))
    be.conv_wgrad(ht, lt, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, ws, window_origin=origin)
    torch.cuda.synchronize()
    be.check_fault()
    want = _wgrad64(sum(O.bf16_split(a)), sum(O.bf16_split(g)), taps, origin)
    d = rel_dev(dw, want)
    print(f"\n[conv_wgrad widths] {case}: rel dev {d:.3e}")
    assert not torch.isnan(dw).any() and d < 2e-5, d
    assert tail_untouched(dbuf)


# ------------------------------------------------------------------------------------------ Functions
def fp64(*ts):
    return [None if t is None else t.detach().double().cpu().requires_grad_(True) for t in ts]


@pytest.mark.parametrize("B,H,W,Cin,Cout,k", [(3, 12, 12, 96, 96, 3), (2, 16, 16, 224, 160, 3), (3, 7, 7, 96, 288, 1),
                                              (2, 16, 16, 64, 96, 3)])
def test_conv2d_function_widths(B, H, W, Cin, Cout, k):
    from bbdm_b200.train import Conv2dFn, backend
    x = rnd((B, Cin, H, W), 6).to(DEV).requires_grad_(True)
    w = rnd((Cout, Cin, k, k), 7, 0.05).to(DEV).requires_grad_(True)
    b = rnd((Cout,), 8, 0.1).to(DEV).requires_grad_(True)
    gy = rnd((B, Cout, H, W), 9, 0.2).to(DEV)
    y = Conv2dFn.apply(x, w, b)
    y.backward(gy)
    backend().check_fault()
    xd, wd, bd = fp64(x, w, b)
    yd = F.conv2d(xd, wd, bd, padding=k // 2)
    yd.backward(gy.double().cpu())
    devs = [rel_dev(y, yd), rel_dev(x.grad, xd.grad), rel_dev(w.grad, wd.grad), rel_dev(b.grad, bd.grad)]
    print(f"\n[Conv2dFn {B}x{H}x{W} {Cin}->{Cout} k{k}] y / dx / dW / db rel dev {devs}")
    assert max(devs) < 3e-5


@pytest.mark.parametrize("B,Hs,Ws,C,Cout,film,resample", [
    (3, 12, 12, 96, 96, True, 0), (2, 6, 10, 224, 96, True, 1), (2, 24, 24, 96, 160, False, 2),
    (2, 16, 16, 288, 96, True, 0)])
def test_gn_act_conv_function_widths(B, Hs, Ws, C, Cout, film, resample):
    from bbdm_b200 import train
    from bbdm_b200.train import GNActConv2dFn
    H, W = (2 * Hs, 2 * Ws) if resample == 1 else ((Hs // 2, Ws // 2) if resample == 2 else (Hs, Ws))
    mk = lambda t: t.to(DEV).requires_grad_(True)
    x = mk(rnd((B, C, Hs, Ws), 10) + 0.2)
    gamma, beta = mk(1 + 0.1 * rnd((C,), 11)), mk(0.1 * rnd((C,), 12))
    scale = mk(0.3 * rnd((B, C), 13)) if film else None
    shift = mk(0.3 * rnd((B, C), 14)) if film else None
    w, b = mk(rnd((Cout, C, 3, 3), 15, 0.05)), mk(rnd((Cout,), 16, 0.1))
    gy = rnd((B, Cout, H, W), 17, 0.2).to(DEV)
    y = GNActConv2dFn.apply(x, gamma, beta, scale, shift, w, b, resample)
    y.backward(gy)
    train.backend().check_fault()
    xd, gd, bd, sd, hd, wd, bbd = fp64(x, gamma, beta, scale, shift, w, b)
    h = F.group_norm(xd, 32, gd, bd, 1e-5)
    if film:
        h = h * (1 + sd[:, :, None, None]) + hd[:, :, None, None]
    h = F.silu(h)
    if resample == 1:
        h = F.interpolate(h, scale_factor=2, mode="nearest")
    elif resample == 2:
        h = F.avg_pool2d(h, 2)
    yd = F.conv2d(h, wd, bbd, padding=1)
    yd.backward(gy.double().cpu())
    pairs = [(y, yd), (x.grad, xd.grad), (w.grad, wd.grad), (b.grad, bbd.grad), (gamma.grad, gd.grad),
             (beta.grad, bd.grad)] + ([(scale.grad, sd.grad), (shift.grad, hd.grad)] if film else [])
    devs = [rel_dev(a, e) for a, e in pairs]
    print(f"\n[GNActConv2dFn {B}x{Hs}x{Ws} {C}->{Cout} resample {resample}] rel devs {['%.2e' % d for d in devs]}")
    assert max(devs) < 1e-4


@pytest.mark.parametrize("B,H,W,Cin,Cout", [(3, 24, 24, 96, 96), (2, 14, 22, 224, 160), (2, 16, 16, 96, 192)])
def test_resampling_conv_functions_widths(B, H, W, Cin, Cout):
    from bbdm_b200.train import Stride2Conv2dFn, Up2Conv2dFn, backend
    for fn, (h, w_), ref in ((Stride2Conv2dFn, (H, W), lambda t, wt, bt: F.conv2d(t, wt, bt, stride=2, padding=1)),
                             (Up2Conv2dFn, (H // 2, W // 2),
                              lambda t, wt, bt: F.conv2d(F.interpolate(t, scale_factor=2, mode="nearest"), wt, bt,
                                                         padding=1))):
        x = rnd((B, Cin, h, w_), 20).to(DEV).requires_grad_(True)
        wt = rnd((Cout, Cin, 3, 3), 21, 0.05).to(DEV).requires_grad_(True)
        bt = rnd((Cout,), 22, 0.1).to(DEV).requires_grad_(True)
        y = fn.apply(x, wt, bt)
        gy = rnd(tuple(y.shape), 23, 0.2).to(DEV)
        y.backward(gy)
        backend().check_fault()
        xd, wd, bd = fp64(x, wt, bt)
        yd = ref(xd, wd, bd)
        yd.backward(gy.double().cpu())
        devs = [rel_dev(y, yd), rel_dev(x.grad, xd.grad), rel_dev(wt.grad, wd.grad), rel_dev(bt.grad, bd.grad)]
        print(f"\n[{fn.__name__} {B}x{h}x{w_} {Cin}->{Cout}] y / dx / dW / db rel dev {devs}")
        assert max(devs) < 3e-5


# ------------------------------------------------------------------------------------------ drop-in model
def build(u, train=False, **kw):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    net = BrownianBridgeModel(bb_namespace(u, **kw))
    net = net.train() if train else net.eval()
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(fill_state_dict(shapes, seed=1234))
    return net.to(DEV)


def load(tag):
    return {k: torch.from_numpy(v) if v.ndim else v for k, v in np.load(os.path.join(GOLD, tag + ".npz")).items()}


@pytest.mark.parametrize("tag", list(WIDTH_CONFIGS))
def test_width_model_matches_reference_fixture(tag):
    g = load(tag)
    net = build(WIDTH_CONFIGS[tag])
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
    net8 = build(WIDTH_CONFIGS[tag], sample_step=8)
    seq = iter(c(g["loop8_noise"]))
    net8._bridge.noise_source = lambda like: next(seq)
    d_loop = rel_dev(net8.sample(y, clip_denoised=True), g["loop8_out"])
    net._bridge.backend().check_fault()
    print(f"\n[{tag}] unet rel dev {d_unet:.3e}; p_sample rel dev {devs}; 8-step loop rel dev {d_loop:.3e}")
    assert d_unet < TOL_PSAMPLE
    assert max(devs.values()) < TOL_PSAMPLE
    assert d_loop < 2e-4


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


@pytest.mark.parametrize("tag", list(WIDTH_CONFIGS))
def test_width_training_step_matches_stock_graph(tag, monkeypatch):
    """Loss and every parameter gradient of one training step on the native path against the stock-PyTorch graph
    (TF32 off): no Conv2d module (cuDNN) call and no library-path warning on the native path, except for mid_w224_st's
    stem: 6 -> 224 channels is past the small-channel kernels' Cin*Cout <= 1024, whatever the channel multiple."""
    import bbdm_b200.unet as U
    net = build(WIDTH_CONFIGS[tag], train=True)
    inputs = _fixture_inputs(tag)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    convs_called = []
    fwd = torch.nn.Conv2d._conv_forward
    monkeypatch.setattr(torch.nn.Conv2d, "_conv_forward", lambda self, *a, **k: (convs_called.append(self),
                                                                                 fwd(self, *a, **k))[1])
    stem_in = WIDTH_CONFIGS[tag]["in_channels"]
    res = {}
    for native in (True, False):
        monkeypatch.setattr(U, "NATIVE_TRAIN_CONV", native)
        convs_called.clear()
        loss, grads, lib = _step(net, inputs)
        lib = {m for m in lib if f"Conv2d {stem_in}->" not in m}
        res[native] = (loss, grads, lib, sum(c.in_channels != stem_in for c in convs_called))
    assert not res[True][2], res[True][2]
    assert res[True][3] == 0 and res[False][3] > 0
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


@pytest.mark.parametrize("tag", ["mid_w96"])
def test_width_graphed_and_checkpointed_steps_are_bit_identical(tag):
    """mid_w96 (its 6 -> 96 stem on the small-channel kernels): the use_checkpoint step and the graphed step reproduce
    the plain eager step bit for bit."""
    from bbdm_b200 import train_graph
    net = build(WIDTH_CONFIGS[tag], train=True)
    inputs = _fixture_inputs(tag)
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


# ------------------------------------------------------------------------------------------ launch shadow
@pytest.mark.parametrize("tag", list(WIDTH_CONFIGS))
def test_width_sampling_forward_every_launch_against_fp64(tag):
    from bbdm_b200 import cabi
    from bbdm_b200.engine import UNetEngine
    from bbdm_b200.unet import UNetModel
    net = UNetModel(**WIDTH_CONFIGS[tag]).eval()
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
    print(f"\n{sh.table(f'{tag} sampling forward, 32x32, B=2')}")
    assert not fails, fails[:10]
    assert "conv_umma" in {c.method for c in sh.checks}


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


@pytest.mark.parametrize("tag", ["mid_w96_rs", "mid_w224_st"])
def test_width_training_step_every_launch_against_fp64(tag, monkeypatch):
    net = build(WIDTH_CONFIGS[tag], train=True)
    x, y, t, nz = _fixture_inputs(tag)
    with _shadowed(monkeypatch) as sh:
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
    torch.cuda.synchronize()
    fails = sh.failures()
    print(f"\n{sh.table(f'{tag} training step, 32x32, B=2')}")
    assert torch.isfinite(loss)
    assert not fails, fails[:10]
    assert {"conv_umma", "conv_wgrad"} <= {c.method for c in sh.checks}
