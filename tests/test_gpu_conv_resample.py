"""-m gpu: the UNet's standalone resampling convolutions (resblock_updown=False, conv_resample=True) on the tensor
cores -- the Downsample's 3x3 stride-2 conv as a 2x2-tap conv on the space-to-depth operand (conv_umma window_origin
-1) and the Upsample's nearest-2x + 3x3 conv -- in sampling and in training:

  * conv_umma with taps = 4 at both window origins, and conv_wgrad's taps = 4 mode, against fp64 torch;
  * Stride2Conv2dFn / Up2Conv2dFn: output, dx, dW and db against fp64 autograd of the reference ops;
  * an aligned resblock_updown=False UNet against the fixture the unmodified reference produced
    (tests/golden/make_golden_conv_resample.py): UNet output, p_sample and the gradients of one training step;
  * the paths: no stride-2 conv_direct while sampling, no cuDNN convolution and no library-path warning in training.
"""
import os
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _recipe import UNET_CONFIGS, bb_namespace, fill_state_dict, rel_dev
from oracle import bbdm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(__file__), "golden", "mid_resample.npz")

# mid_pixel with standalone Downsample / Upsample modules between the levels: 64 -> 128 -> 256 channels, 32x32
RS_CONFIGS = {"mid_resample": dict(UNET_CONFIGS["mid_pixel"], resblock_updown=False)}


def fixture_rows(t):
    """At most 16 evenly spread output rows of a parameter gradient (keeps the fixture small)."""
    step = max(1, t.shape[0] // 16)
    return t[::step][:16]


def picked_gradients(unet):
    """The gradients the fixture stores: every Downsample / Upsample conv, their neighbours and the ends."""
    keep = ("input_blocks.0.0", "input_blocks.2.0.op", "input_blocks.4.0.op", "input_blocks.3.0.in_layers.2",
            "output_blocks.1.2.conv", "output_blocks.3.1.conv", "output_blocks.2.0.in_layers.2", "out.2")
    return {n: p for n, p in unet.named_parameters() if n.startswith(keep)}


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
    return h.to(torch.bfloat16).to(DEV), l.to(torch.bfloat16).to(DEV)


# B, H, W of the conv's (space-to-depth) grid, Cin, Cout
TAP4_CASES = [(1, 8, 8, 64, 64), (2, 16, 16, 128, 64), (8, 8, 8, 512, 128), (2, 32, 32, 64, 128),
              (1, 64, 64, 128, 128), (2, 128, 128, 64, 64), (8, 16, 16, 512, 512)]


@pytest.mark.parametrize("origin", [0, -1])
@pytest.mark.parametrize("wscale", [0.02, 1.0])
@pytest.mark.parametrize("case", TAP4_CASES)
def test_conv_umma_taps4_window_origin(be, case, origin, wscale):
    B, H, W, Cin, Cout = case
    x = rnd((B, H, W, Cin), 1)
    w = rnd((Cout, Cin, 2, 2), 2, wscale)
    bias = rnd((Cout,), 3, 0.1)
    a_hi, a_lo = split(x)
    w_hi, w_lo = split(w.permute(2, 3, 0, 1).reshape(4, Cout, Cin).contiguous())
    out = torch.empty((B, H, W, Cout), device=DEV)
    be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=4, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo,
                 bias=bias.to(DEV), out=out, passes=3, window_origin=origin)
    torch.cuda.synchronize()
    be.check_fault()
    pad = (0, 1, 0, 1) if origin == 0 else (1, 0, 1, 0)
    want = F.conv2d(F.pad(x.double().permute(0, 3, 1, 2), pad), w.double(), bias.double()).permute(0, 2, 3, 1)
    d = rel_dev(out, want)
    print(f"\n[conv_umma taps 4 origin {origin}] {case} w*{wscale}: rel dev {d:.3e}")
    assert d < 3e-5, d


def test_conv_umma_window_origin_rejected_with_upsample2x(be):
    from bbdm_b200 import cabi
    t = torch.zeros((1, 8, 8, 64), dtype=torch.bfloat16, device=DEV)
    w = torch.zeros((16, 64, 64), dtype=torch.bfloat16, device=DEV)
    out = torch.empty((1, 16, 16, 64), device=DEV)
    with pytest.raises(cabi.BbdmError, match="window_origin"):
        be.conv_umma(B=1, H=8, W=8, Cin=64, Cout=64, taps=4, a_hi=t, a_lo=t, w_hi=w, w_lo=w, out=out,
                     upsample2x=True, window_origin=-1)


@pytest.mark.parametrize("origin", [0, -1])
@pytest.mark.parametrize("wscale", [0.02, 1.0])
@pytest.mark.parametrize("case", [(1, 8, 8, 64, 64), (2, 16, 16, 128, 512), (8, 8, 8, 512, 128),
                                  (2, 64, 64, 256, 128), (1, 128, 128, 64, 64)])
def test_conv_wgrad_taps4_window_origin(be, case, origin, wscale):
    """dW[co][ci][oy][ox] = sum_p dY[p][co] A[p + (oy, ox) + origin][ci]; wscale scales dY (the GEMM's A operand)."""
    B, H, W, Cin, Cout = case
    P = B * H * W
    x = rnd((B, H, W, Cin), 4)
    g = rnd((B, H, W, Cout), 5, wscale)
    a_hi, a_lo = split(x)
    ht = torch.empty((Cout, P), dtype=torch.bfloat16, device=DEV)
    lt = torch.empty_like(ht)
    be.split_grad(g.to(DEV).reshape(P, Cout), None, None, ht, lt)
    _, fl = be.wgrad_workspace(B, H, W, Cin, Cout, 4)
    ws = torch.empty(fl, device=DEV)
    dws = []
    for _ in range(2):
        dws.append(torch.full((Cout, Cin, 2, 2), float("nan"), device=DEV))
        be.conv_wgrad(ht, lt, a_hi, a_lo, B, H, W, Cin, Cout, 4, dws[-1], ws, window_origin=origin)
    torch.cuda.synchronize()
    be.check_fault()
    assert torch.equal(dws[0], dws[1])                         # fixed-order split-K reduction
    pad = (0, 1, 0, 1) if origin == 0 else (1, 0, 1, 0)
    xd = F.pad(x.double().permute(0, 3, 1, 2), pad)
    want = torch.nn.grad.conv2d_weight(xd, (Cout, Cin, 2, 2), g.double().permute(0, 3, 1, 2))
    d = rel_dev(dws[0], want)
    print(f"\n[conv_wgrad taps 4 origin {origin}] {case} dY*{wscale}: rel dev {d:.3e}")
    assert d < 3e-5, d


FN_CASES = [(2, 16, 16, 64, 128, True), (1, 32, 32, 128, 64, False), (8, 16, 16, 512, 512, True),
            (2, 64, 64, 64, 64, True)]


@pytest.mark.parametrize("wscale", [0.05, 1.0])
@pytest.mark.parametrize("B,H,W,Cin,Cout,bias", FN_CASES)
def test_stride2_conv_function_gradients(B, H, W, Cin, Cout, bias, wscale):
    from bbdm_b200.train import Stride2Conv2dFn
    x = rnd((B, Cin, H, W), 4).to(DEV).requires_grad_(True)
    w = rnd((Cout, Cin, 3, 3), 5, wscale).to(DEV).requires_grad_(True)
    b = rnd((Cout,), 6, 0.1).to(DEV).requires_grad_(True) if bias else None
    gy = rnd((B, Cout, H // 2, W // 2), 7, 0.2).to(DEV)
    y = Stride2Conv2dFn.apply(x, w, b)
    y.backward(gy)
    xd, wd = x.detach().double().cpu().requires_grad_(True), w.detach().double().cpu().requires_grad_(True)
    bd = None if b is None else b.detach().double().cpu().requires_grad_(True)
    yd = F.conv2d(xd, wd, bd, stride=2, padding=1)
    yd.backward(gy.double().cpu())
    devs = [rel_dev(y, yd), rel_dev(x.grad, xd.grad), rel_dev(w.grad, wd.grad)]
    print(f"\n[stride-2 Function] y / dx / dW rel dev {devs}")
    assert max(devs) < 3e-5
    if bias:
        assert rel_dev(b.grad, bd.grad) < 1e-5


@pytest.mark.parametrize("wscale", [0.05, 1.0])
@pytest.mark.parametrize("B,H,W,Cin,Cout,bias", FN_CASES)
def test_upsample_conv_function_gradients(B, H, W, Cin, Cout, bias, wscale):
    """H, W: the low-res input; the conv runs on the nearest-2x upsampling of it."""
    from bbdm_b200.train import Up2Conv2dFn
    H, W = H // 2, W // 2
    x = rnd((B, Cin, H, W), 8).to(DEV).requires_grad_(True)
    w = rnd((Cout, Cin, 3, 3), 9, wscale).to(DEV).requires_grad_(True)
    b = rnd((Cout,), 10, 0.1).to(DEV).requires_grad_(True) if bias else None
    gy = rnd((B, Cout, 2 * H, 2 * W), 11, 0.2).to(DEV)
    y = Up2Conv2dFn.apply(x, w, b)
    y.backward(gy)
    xd, wd = x.detach().double().cpu().requires_grad_(True), w.detach().double().cpu().requires_grad_(True)
    bd = None if b is None else b.detach().double().cpu().requires_grad_(True)
    yd = F.conv2d(F.interpolate(xd, scale_factor=2, mode="nearest"), wd, bd, padding=1)
    yd.backward(gy.double().cpu())
    devs = [rel_dev(y, yd), rel_dev(x.grad, xd.grad), rel_dev(w.grad, wd.grad)]
    print(f"\n[nearest-2x Function] y / dx / dW rel dev {devs}")
    assert max(devs) < 3e-5
    if bias:
        assert rel_dev(b.grad, bd.grad) < 1e-5


def build(**kw):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    net = BrownianBridgeModel(bb_namespace(RS_CONFIGS["mid_resample"], **kw))
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(fill_state_dict(shapes, seed=1234))
    return net.to(DEV)


def gold():
    return {k: torch.from_numpy(v) if v.ndim else v for k, v in np.load(GOLD).items()}


def test_sampling_matches_reference_fixture_without_stride2_direct_conv():
    from bbdm_b200 import engine as E
    g = gold()
    net = build().eval()
    c = lambda z: z.cuda()
    x, y, t = c(g["x"]), c(g["y"]), c(g["t"])
    be = net.denoise_fn.engine().be
    strides = []
    direct = be.conv_direct
    be.conv_direct = lambda *a, **k: (strides.append(a[7] if len(a) > 7 else k.get("stride", 1)), direct(*a, **k))[1]
    try:
        with torch.no_grad():
            out = net.denoise_fn(x, timesteps=t, context=y)
        devs = {}
        for i in g["ps_ids"].tolist():
            o, _ = net.p_sample(c(g[f"ps{i}_xt"]), y, y, i, clip_denoised=False, noise=c(g[f"ps{i}_noise"]))
            devs[i] = rel_dev(o, g[f"ps{i}_out"])
    finally:
        del be.conv_direct
    be.check_fault()
    d_unet = rel_dev(out, g["unet_out"])
    print(f"\n[mid_resample] unet rel dev {d_unet:.3e}; p_sample rel dev {devs}; conv_direct strides {strides}")
    assert all(s == 1 for s in strides), strides
    w = net.denoise_fn.engine()._w
    assert all("s2_hi" in w[n + ".op"] for n in ("input_blocks.2.0", "input_blocks.4.0"))
    assert isinstance(net.denoise_fn.input_blocks[2][0], E.Downsample)
    assert d_unet < 1e-4
    assert max(devs.values()) < 1e-4


def test_training_step_matches_reference_fixture_on_native_kernels():
    """One training step: no cuDNN convolution (every Conv2d module call is counted), no library-path warning, and
    the loss and parameter gradients against the reference's (fixture) to the bound of mid_pixel_grads."""
    g = gold()
    net = build().train()
    x, y, t, nz = (g[k].cuda() for k in ("x", "y", "t", "q_noise"))
    calls = []
    fwd = torch.nn.Conv2d._conv_forward
    torch.nn.Conv2d._conv_forward = lambda self, *a, **k: (calls.append(self), fwd(self, *a, **k))[1]
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter("always")
            net.zero_grad(set_to_none=True)
            loss, _ = net.p_losses(x, y, y, t, nz)
            loss.backward()
    finally:
        torch.nn.Conv2d._conv_forward = fwd
    torch.cuda.synchronize()
    from bbdm_b200 import train
    train.backend().check_fault()
    lib = [str(r.message) for r in rec if "stock PyTorch" in str(r.message)]
    assert not calls, f"{len(calls)} Conv2d calls on cuDNN"
    assert not lib, lib
    assert abs(float(loss) - float(g["loss"])) < 2e-4 * abs(float(g["loss"]))
    params = dict(net.denoise_fn.named_parameters())
    devs = {k[5:]: rel_dev(fixture_rows(params[k[5:]].grad), torch.from_numpy(np.asarray(g[k])))
            for k in g if k.startswith("grad:")}
    wname = max(devs, key=devs.get)
    print(f"\n[mid_resample train] loss {float(loss):.6f} vs {float(g['loss']):.6f}; {len(devs)} gradients, worst "
          f"{wname} {devs[wname]:.3e}")
    assert any(".op." in n for n in devs) and any(n.endswith(".conv.weight") for n in devs)
    assert devs[wname] < 3e-4
