"""The launch shadow of tests/_launch_shadow.py beyond the UNet sampling forward and the batch-32 training step, on the
CPU emulation (no GPU):

  * every launching method of cabi.CudaBackend has an OUTPUTS entry and an fp64 reference, so a new launch kind fails
    here rather than on its first shadowed GPU run;
  * the 2x2-window references at window origin -1 and 0 against torch's own stride-2 conv and its autograd;
  * the shadow accepts the VQGAN executor, a resblock_updown=False UNet forward and training step (capturable Adam),
    and the sampling loop with the SpatialRescaler condition on the emulation (tests/_emu_backend_origin.py), and flags
    exactly the launch whose output was perturbed;
  * inside a CUDA-graph capture the shadow runs each launch without copying, synchronising or checking it.
"""
import inspect
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from _emu_backend_origin import EmuBackendOrigin
from _launch_shadow import NOT_LAUNCHES, OUTPUTS, Shadow, missing_forms, space_to_depth, split_bf16
from _recipe import UNET_CONFIGS, VQGAN_CONFIGS, bb_namespace, fill_state_dict, synth_images, vqgan_namespace, \
    vqgan_state_dict
from bbdm_b200 import weights as Wt

GOLD = os.path.join(os.path.dirname(__file__), "golden")
RS_UNET = dict(UNET_CONFIGS["mid_pixel"], resblock_updown=False)
# the emulated F(6,3) chain on these activations (test_launch_shadow_host.py::EMU_BOUNDS)
EMU_BOUNDS = {"chain6": 2.5e-5}


# ------------------------------------------------------------------------------------------ completeness
def _cuda_launches():
    from bbdm_b200 import cabi
    return {n for n, f in inspect.getmembers(cabi.CudaBackend, inspect.isfunction)
            if not n.startswith("_")} - NOT_LAUNCHES - {"check_fault"}


def test_every_cuda_launch_has_outputs_and_a_reference():
    from bbdm_b200 import cabi
    launches = _cuda_launches()
    assert launches == set(OUTPUTS), (launches - set(OUTPUTS), set(OUTPUTS) - launches)
    for name in launches:
        assert callable(getattr(Shadow, "_ref_" + name, None)), name
        params = inspect.signature(getattr(cabi.CudaBackend, name)).parameters
        assert set(OUTPUTS[name]) <= set(params), (name, set(OUTPUTS[name]) - set(params))


# ------------------------------------------------------------------------------------------ reference self-checks
def _bf16_exact(shape, seed, scale=1.0):
    """Values that a bf16 hi plane holds exactly (lo = 0): the split products are then the exact conv."""
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).to(torch.bfloat16).float()


@pytest.mark.parametrize("B,C,Co,H,W", [(2, 8, 6, 8, 12), (1, 4, 4, 6, 4)])
def test_taps4_origin_references_equal_the_stride2_conv_and_its_weight_gradient(B, C, Co, H, W):
    x = _bf16_exact((B, C, H, W), 1)
    w = _bf16_exact((Co, C, 3, 3), 2, 0.1)
    xs = space_to_depth(x.permute(0, 2, 3, 1))                      # [B, H/2, W/2, 4C]
    s_hi, s_lo = split_bf16(xs)
    w2 = Wt.stride2_s2d_weights(w.double()).permute(2, 0, 1).contiguous()      # [4, Co, 4C]
    want = F.conv2d(x.double(), w.double(), stride=2, padding=1).permute(0, 2, 3, 1)
    c = dict(B=B, H=H // 2, W=W // 2, Cin=4 * C, Cout=Co, taps=4, a_hi=s_hi, a_lo=s_lo, w_hi=w2.to(torch.bfloat16),
             w_lo=torch.zeros_like(w2, dtype=torch.bfloat16), bias=None, Cin2=0, residual=None, res_mode=0, passes=3,
             upsample2x=False, weights_per_image=False, out_nchw_channels=0, window_origin=-1)
    a = dict(c, out=want, out_hi=None, out_lo=None, stats_partial=None)
    sh = Shadow(EmuBackendOrigin())
    sh._ref_conv_umma(0, "", [], c, a, {})
    assert sh.checks[-1].what == "out" and sh.checks[-1].dev < 1e-12
    sh._ref_conv_umma(1, "", [], dict(c, window_origin=0), a, {})      # the window at 0..1: a different conv
    assert sh.checks[-1].dev > 1e-2
    # weight gradient: the origin -1 2x2 reference over (x', dY), folded back to 3x3, is autograd's dW
    xd = x.double().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    y = F.conv2d(xd, wd, stride=2, padding=1)
    dy = _bf16_exact(tuple(y.shape), 3)
    y.backward(dy.double())
    dyt = dy.permute(1, 0, 2, 3).reshape(Co, -1)
    rows = lambda sl: dyt.reshape(Co, B, -1)[:, sl].reshape(Co, -1).to(torch.float64)
    g4 = Shadow._wgrad64(xs, rows, 2, -1)
    assert torch.allclose(Wt.stride2_fold_wgrad(g4), wd.grad, rtol=0, atol=1e-12)
    # origin 0, the VQGAN's (0, 1)-padded stride-2 conv: against torch's weight gradient of the same window
    g0 = Shadow._wgrad64(xs, rows, 2, 0)
    ref0 = torch.nn.grad.conv2d_weight(F.pad(xs.permute(0, 3, 1, 2).double(), (0, 1, 0, 1)), (Co, 4 * C, 2, 2),
                                       dy.double())
    assert torch.allclose(g0, ref0, rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------ emulated runs
def _vq_shadow(name, mutate=None):
    from bbdm_b200.vqgan import VQModel
    from bbdm_b200.vqgan_engine import VQGANEngine
    g = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}
    vq = VQModel(**vqgan_namespace(VQGAN_CONFIGS[name])).eval()
    vq.load_state_dict(vqgan_state_dict({k: tuple(v.shape) for k, v in vq.state_dict().items()}), strict=True)
    sh = Shadow(EmuBackendOrigin(), bounds=EMU_BOUNDS)
    sh.mutate = mutate or {}
    eng = VQGANEngine(vq, backend=sh)
    eng.wino_min_c, eng.wino_min_tiles = 64, 32          # the ResnetBlock convs on Winograd at the fixture's size
    eng.refresh_weights()
    sh.register_engine(eng)
    eng.encode(g["x"], quant_conv=False)
    eng.encode(g["x"], quant_conv=True)
    eng.decode(g["lat"], return_indices=True)
    eng.decode(g["lat_b"], quant_conv_first=True)
    return sh


VQ_FORMS = {"vq_tc": [("s2d_split", (), ()), ("conv_umma", ("taps 4",), ("origin", "upsample2x")),
                      ("softmax_rows_split", (), ()), ("vq_nearest", (), ()), ("wino_output", (), ())],
            "vq_small": [("conv_direct_pad", (), ()), ("attention", (), ()), ("vq_nearest", (), ())]}


@pytest.mark.parametrize("name", list(VQGAN_CONFIGS))
def test_shadow_accepts_the_emulated_vqgan_executor(name):
    sh = _vq_shadow(name)
    print("\n" + sh.table(f"VQGAN executor {name}, emulation"))
    assert not sh.failures(), sh.failures()[:5]
    assert not missing_forms(sh, VQ_FORMS[name]), missing_forms(sh, VQ_FORMS[name])
    chains = [c for c in sh.checks if c.what.startswith("chain")]
    assert len(chains) == sum(m == "wino_output" for m, _ in sh.launches)
    if name == "vq_tc":
        assert chains and any(c.what == "s2d taps vs module weight" for c in sh.checks)


def _unet_forward(mutate=None):
    from bbdm_b200.engine import UNetEngine
    from bbdm_b200.unet import UNetModel
    net = UNetModel(**RS_UNET).eval()
    net.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1234))
    sh = Shadow(EmuBackendOrigin(), bounds=EMU_BOUNDS)
    sh.mutate = mutate or {}
    eng = UNetEngine(net, backend=sh)
    eng.refresh_weights()
    sh.register_engine(eng)
    x, y = synth_images((2, 3, 32, 32), 1), synth_images((2, 3, 32, 32), 2)
    eng.forward(x, torch.tensor([3, 900]), y)
    return sh


def test_shadow_accepts_the_emulated_resblock_updown_false_forward():
    sh = _unet_forward()
    print("\n" + sh.table("mid_pixel with resblock_updown=False, 32x32, B=2, emulation"))
    assert not sh.failures(), sh.failures()[:5]
    assert not missing_forms(sh, [("s2d_split", (), ()), ("conv_umma", ("taps 4", "origin -1", "stats"), ())])
    assert any(c.what == "s2d taps vs module weight" for c in sh.checks)


def _train_step(monkeypatch, mutate=None):
    """q_sample, training forward and backward of mid_pixel with resblock_updown=False, two FusedAdam(capturable=True)
    steps."""
    from bbdm_b200 import train
    from bbdm_b200.bridge import BridgeOps
    from bbdm_b200.optim import FusedAdam
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    sh = Shadow(EmuBackendOrigin(), bounds=EMU_BOUNDS)
    sh.mutate = mutate or {}
    monkeypatch.setattr(BridgeOps, "backend_factory", staticmethod(lambda: sh))
    monkeypatch.setattr(FusedAdam, "backend_factory", staticmethod(lambda: sh))
    train.set_backend(sh)
    try:
        net = BrownianBridgeModel(bb_namespace(RS_UNET)).train()
        net.denoise_fn.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()},
                                                       seed=1234))
        x, y = synth_images((2, 3, 32, 32), 1), synth_images((2, 3, 32, 32), 2)
        nz = torch.randn((2, 3, 32, 32), generator=torch.Generator().manual_seed(3))
        opt = FusedAdam(net.get_parameters(), lr=1e-4, capturable=True)
        loss, _ = net.p_losses(x, y, y, torch.tensor([0, 999]), nz)
        loss.backward()
        opt.step()
        opt.step()
    finally:
        train.set_backend(None)
    return sh


RS_TRAIN_FORMS = [("s2d_split", (), ()), ("conv_umma", ("taps 4", "origin -1"), ()),
                  ("conv_umma", ("taps 4",), ("origin", "upsample2x")), ("conv_wgrad", ("taps 4", "origin -1"), ()),
                  ("adam_multi_dev", ("step 1",), ()), ("adam_multi_dev", ("step 2",), ())]


@pytest.fixture(scope="module")
def train_clean():
    with pytest.MonkeyPatch.context() as mp:
        sh = _train_step(mp)
    print("\n" + sh.table("mid_pixel resblock_updown=False training step, capturable FusedAdam, B=2, emulation"))
    return sh


def test_shadow_accepts_the_emulated_stride2_training_step(train_clean):
    assert not train_clean.failures(), train_clean.failures()[:5]
    assert not missing_forms(train_clean, RS_TRAIN_FORMS), missing_forms(train_clean, RS_TRAIN_FORMS)


def _sampling(monkeypatch, mutate=None):
    """The pixel bridge's eager loop over steps [999, 1, 0] with and without clip, one direct p_sample_dev launch (the
    graphed step's update) and denorm_to_uint8 of the result, and the SpatialRescaler condition stage."""
    from bbdm_b200 import cond
    from bbdm_b200.bridge import BridgeOps
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    sh = Shadow(EmuBackendOrigin(), bounds=EMU_BOUNDS)
    sh.mutate = mutate or {}
    monkeypatch.setattr(BridgeOps, "backend_factory", staticmethod(lambda: sh))
    monkeypatch.setattr(cond.SpatialRescaler, "backend_factory", staticmethod(lambda: sh))
    net = BrownianBridgeModel(bb_namespace(UNET_CONFIGS["mid_pixel"], sample_step=3)).eval()
    assert net.steps.tolist() == [999, 1, 0]
    net.denoise_fn.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()},
                                                   seed=1234))
    y = synth_images((2, 3, 32, 32), 2)
    net._bridge.backend()
    eng = net.denoise_fn.engine()
    eng.refresh_weights()
    sh.register_engine(eng)
    imgs = []
    for clip in (False, True):
        torch.manual_seed(5)
        imgs.append(net.sample(y, clip_denoised=clip))
    g = torch.Generator().manual_seed(7)
    x_t, eps, noise = (torch.randn((2, 3, 32, 32), generator=g) for _ in range(3))
    out, x0 = torch.empty_like(x_t), torch.empty_like(x_t)
    sh.p_sample_dev(x_t, y, eps, noise, net._bridge.coef_table()[0], net.objective, True, False, out, x0)
    sh.denorm_to_uint8(imgs[-1], True, torch.empty((2, 32, 32, 3), dtype=torch.uint8))
    with torch.no_grad():
        torch.manual_seed(6)
        cond.SpatialRescaler(n_stages=2, in_channels=3, out_channels=3, bias=True)(y)
        cond.SpatialRescaler(n_stages=1, in_channels=3)(y)
    return sh


SAMPLE_FORMS = [("p_sample", ("not last",), ("clip",)), ("p_sample", ("not last", "clip"), ()),
                ("p_sample", ("last",), ("not last",)), ("p_sample_dev", ("not last", "clip"), ()),
                ("denorm_to_uint8", ("to_normal",), ()), ("spatial_rescale", ("2 stages", "1x1 map"), ()),
                ("spatial_rescale", ("1 stages",), ("1x1 map",))]


def test_shadow_accepts_the_emulated_sampling_loop(monkeypatch):
    sh = _sampling(monkeypatch)
    print("\n" + sh.table("mid_pixel sampling loop, steps 999, 1, 0, B=2, emulation"))
    assert not sh.failures(), sh.failures()[:5]
    assert not missing_forms(sh, SAMPLE_FORMS), missing_forms(sh, SAMPLE_FORMS)


# ------------------------------------------------------------------------------------------ perturbations
def _first(launches, method, has=(), lacks=()):
    return next(i for i, (m, f) in enumerate(launches) if m == method and all(t in f for t in has)
                and not any(t in f for t in lacks))


def _flip_plane_bit(a):
    a["out_hi"][1].view(-1)[-1:].view(torch.int16).bitwise_xor_(1)          # one mantissa bit, last pixel, image 1


def _softmax_row(a):
    row = a["out_hi"].reshape(-1, a["out_hi"].shape[-1])[-1]
    row[0] = (row[0].float() + 0.01).to(torch.bfloat16)                      # one probability of the last row


def _farther_code(a):
    """The last pixel of image 1 gets the code farthest from it."""
    z = a["z"].reshape(a["z"].shape[0], -1, a["z"].shape[-1])[1, -1]
    a["indices"].reshape(a["indices"].shape[0], -1)[1, -1] = int(((a["codebook"] - z) ** 2).sum(1).argmax())


def _edge(key, image, rel=1e-4):
    def fn(a):
        o = a[key]
        o[image].view(-1)[-1] += rel * float(o[image].abs().max())
    return fn


def _one_ulp(a):
    o = a["x_out"][1].view(-1)
    o[-1] = torch.nextafter(o[-1], torch.tensor(math.inf))


def _step_scalar(a):
    a["step"] += 1


def _dw_row(a):
    a["dw"][-1].view(-1)[0] += 1e-4 * float(a["dw"].abs().max())


VQ_CASES = {
    "vq_tc": {"s2d_split plane bit": lambda L: (_first(L, "s2d_split"), _flip_plane_bit),
              "softmax row": lambda L: (_first(L, "softmax_rows_split"), _softmax_row),
              "vq index": lambda L: (_first(L, "vq_nearest"), _farther_code),
              "taps-4 conv": lambda L: (_first(L, "conv_umma", ("taps 4",), ("upsample2x",)), _edge("out", 1))},
    "vq_small": {"conv_direct_pad": lambda L: (_first(L, "conv_direct_pad"), _edge("out", 1))},
}


def _assert_flags_exactly(clean, run, cases):
    targets = {name: pick(clean.launches) for name, pick in cases.items()}
    sh = run(dict(targets.values()))
    assert sh.launches == clean.launches
    flagged = sh.flagged_launches()
    for name, (idx, _) in targets.items():
        assert idx in flagged, name
    assert flagged == sorted(idx for idx, _ in targets.values())


@pytest.mark.parametrize("name", list(VQ_CASES))
def test_shadow_flags_exactly_the_perturbed_vqgan_launches(name):
    _assert_flags_exactly(_vq_shadow(name), lambda m: _vq_shadow(name, m), VQ_CASES[name])


def test_shadow_flags_exactly_the_perturbed_origin_conv():
    cases = {"origin -1 conv": lambda L: (_first(L, "conv_umma", ("origin -1",)), _edge("out", 1))}
    _assert_flags_exactly(_unet_forward(), _unet_forward, cases)


def test_shadow_flags_exactly_the_perturbed_training_launches(train_clean, monkeypatch):
    cases = {"origin -1 wgrad": lambda L: (_first(L, "conv_wgrad", ("origin -1",)), _dw_row),
             "Adam step scalar": lambda L: (_first(L, "adam_multi_dev", ("step 2",)), _step_scalar)}
    _assert_flags_exactly(train_clean, lambda m: _train_step(monkeypatch, m), cases)


def test_shadow_flags_exactly_the_perturbed_sampling_launches(monkeypatch):
    cases = {"p_sample ulp": lambda L: (_first(L, "p_sample", ("not last",)), _one_ulp),
             "p_sample_dev ulp": lambda L: (_first(L, "p_sample_dev"), _one_ulp),
             "spatial_rescale": lambda L: (_first(L, "spatial_rescale"), _edge("out", 1)),
             "denorm byte": lambda L: (_first(L, "denorm_to_uint8"), lambda a: a["out"][1].view(-1)[-1:].add_(1))}
    _assert_flags_exactly(_sampling(monkeypatch), lambda m: _sampling(monkeypatch, m), cases)


# ------------------------------------------------------------------------------------------ capture
def test_launches_inside_a_capture_pass_through_unchecked(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    sh = Shadow(EmuBackendOrigin())
    sh.mutate = {0: _flip_plane_bit}                   # not applied: nothing is checked inside a capture
    src = torch.randn(2, 4, 6, 8)
    hi = torch.empty((2, 2, 3, 32), dtype=torch.bfloat16)
    lo = torch.empty_like(hi)
    sh.s2d_split(src, hi, lo)
    x = torch.randn(2, 3, 4, 4)
    out, x0 = torch.empty_like(x), torch.empty_like(x)
    coef = torch.tensor([0.5, 0.5, 0.7, 0.4, 0.6, 0.3, 0.2])
    sh.p_sample_dev(x, x, x, x, coef, "grad", False, False, out, x0)
    assert sh.captured == ["s2d_split", "p_sample_dev"]
    assert sh.launches == [] and sh.checks == []
    h, l = split_bf16(space_to_depth(src))
    assert torch.equal(hi, h) and torch.equal(lo, l)                 # the launch itself ran
    assert "captured, not checked: p_sample_dev 1, s2d_split 1" in sh.table("capture")
