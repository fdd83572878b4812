"""UNets whose channel counts are multiples of 32 but not all of 64 (tests/_widths.py), on CPU: the tensor-core gate at
the backend's channel multiple, the oracle against the reference-generated fixtures, and the sampling executor's and
the training Functions' routing on the emulation that declares CudaBackend's multiple of 32
(tests/_emu_backend_widths.py).  The kernels are checked by the -m gpu suite (tests/test_gpu_widths.py)."""
import os

import numpy as np
import pytest
import torch

from _emu_backend_ragged import EmuBackendRagged
from _emu_backend_widths import EmuBackendWidths
from _recipe import bb_namespace, fill_state_dict, rel_dev, synth_images
from _widths import WIDTH_CONFIGS
from bbdm_b200 import cabi, convs
from bbdm_b200.engine import UNetEngine
from bbdm_b200.unet import UNetModel
from oracle import bbdm_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")
TAGS = list(WIDTH_CONFIGS)


def build(cfg):
    net = UNetModel(**cfg).eval()
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    net.load_state_dict(fill_state_dict(shapes, seed=1234))
    return net


def load(tag):
    return {k: torch.from_numpy(v) if v.ndim else v for k, v in np.load(os.path.join(GOLD, tag + ".npz")).items()}


def _recording(base):
    """base with the input channel count of every conv_direct call recorded."""
    class Rec(base):
        def __init__(self):
            super().__init__()
            self.direct_cin = []

        def conv_direct(self, src, *a, **k):
            self.direct_cin.append(src.shape[3])
            return super().conv_direct(src, *a, **k)
    return Rec()


def test_channel_multiple_is_a_backend_capability():
    assert convs.channel_multiple(cabi.CudaBackend) == 32
    assert convs.channel_multiple(EmuBackendRagged()) == 64 and convs.channel_multiple(EmuBackendWidths()) == 32
    assert not convs.tensor_core_ok(96, 128, 32) and convs.tensor_core_ok(96, 128, 32, 32)
    assert convs.tensor_core_ok(224, 672, 4, 32) and not convs.tensor_core_ok(224, 672, 3, 32)
    assert not convs.tensor_core_ok(48, 64, 32, 32) and not convs.tensor_core_ok(64, 80, 32, 32)


def test_configs_have_the_widths():
    for tag in TAGS:
        net = UNetModel(**WIDTH_CONFIGS[tag])
        cins = {m.in_channels for m in net.modules() if isinstance(m, torch.nn.Conv2d)}
        assert any(c % 64 == 32 for c in cins) and all(c % 32 == 0 for c in cins if c > 8), (tag, sorted(cins))


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_matches_width_reference_fixture(tag):
    g = load(tag)
    cfg = O.unet_cfg(**WIDTH_CONFIGS[tag])
    sd = build(WIDTH_CONFIGS[tag]).state_dict()
    bufs, steps = O.make_schedule()
    x, y, t = g["x"], g["y"], g["t"]
    assert rel_dev(O.unet_forward(sd, cfg, x, t, y), g["unet_out"]) < 2e-6
    for i in g["ps_ids"].tolist():
        o, _ = O.p_sample(sd, cfg, bufs, steps, i, g[f"ps{i}_xt"], y, y, g[f"ps{i}_noise"], prefix="")
        assert rel_dev(o, g[f"ps{i}_out"]) < 2e-6


@pytest.mark.parametrize("tag", TAGS)
def test_sampling_runs_every_wide_layer_on_the_tensor_cores(tag):
    """Every ResBlock, attention, transformer and Downsample conv goes to conv_umma.  conv_direct is left with the stem
    where conv_stem does not take it (6 input channels), the SpatialTransformers' k|v projection of the 3-channel
    context, and the standalone Upsample convs, which the sampling executor runs on the upsampled fp32 map at every
    width (64-aligned ones included).  The emulated forward matches the reference fixture."""
    g = {k: v for k, v in load(tag).items() if isinstance(v, torch.Tensor)}
    be = _recording(EmuBackendWidths)
    net = build(WIDTH_CONFIGS[tag])
    out = UNetEngine(net, backend=be).forward(g["x"], g["t"], g["y"])
    assert not torch.isnan(out).any()
    assert rel_dev(out, g["unet_out"]) < 6e-5
    assert "conv_umma" in be.calls and "attention_tc" not in be.calls
    ups = [m.channels for m in net.modules() if type(m).__name__ == "Upsample" and m.use_conv]
    n_st = sum(type(m).__name__ == "SpatialTransformer" for m in net.modules())
    assert sorted(c for c in be.direct_cin if c > 6) == sorted(ups), be.direct_cin
    assert len(be.direct_cin) == ("conv_stem" not in be.calls) + n_st + len(ups)
    if tag == "mid_w96_rs":
        assert "s2d_split" in be.calls and ups


@pytest.mark.parametrize("tag", ["mid_w96", "mid_w96_rs"])
def test_sampling_on_a_backend_without_the_multiple_routes_as_before(tag):
    """The same model on a backend that declares no channel multiple: the 64 rule, so the 96-channel convs stay on the
    fp32 direct kernel (and the result is the same)."""
    g = {k: v for k, v in load(tag).items() if isinstance(v, torch.Tensor)}
    be = _recording(EmuBackendRagged)
    eng = UNetEngine(build(WIDTH_CONFIGS[tag]), backend=be)
    assert eng.conv_multiple == 64
    out = eng.forward(g["x"], g["t"], g["y"])
    assert rel_dev(out, g["unet_out"]) < 6e-5
    assert 96 in be.direct_cin and 288 in be.direct_cin      # 96-channel convs, the 192+96 concatenation


def test_spatial_transformer_width_224_needs_the_multiple():
    g = {k: v for k, v in load("mid_w224_st").items() if isinstance(v, torch.Tensor)}
    eng = UNetEngine(build(WIDTH_CONFIGS["mid_w224_st"]), backend=EmuBackendRagged())
    with pytest.raises(NotImplementedError, match="multiples of 64"):
        eng.forward(g["x"], g["t"], g["y"])


@pytest.mark.parametrize("tag", ["mid_w96", "mid_w96_rs"])
def test_training_step_runs_on_the_native_functions(tag, monkeypatch):
    """A training step (BrownianBridgeModel.p_losses + backward) on the emulation with the multiple of 32: no Conv2d
    module call and no library-path report, and the loss and gradients match the stock graph."""
    import bbdm_b200.unet as U
    from bbdm_b200 import train
    from bbdm_b200.bridge import BridgeOps
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    emu = EmuBackendWidths()
    train.set_backend(emu)
    monkeypatch.setattr(BridgeOps, "backend_factory", staticmethod(lambda: emu))
    library = []
    monkeypatch.setattr(train, "_library_path", lambda what, x: library.append((what, tuple(x.shape))))
    net = BrownianBridgeModel(bb_namespace(WIDTH_CONFIGS[tag])).train()
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(fill_state_dict(shapes, seed=1234))
    B, S = 2, 32
    x, y = synth_images((B, 3, S, S), seed=11), synth_images((B, 3, S, S), seed=12)
    t = torch.tensor([17, 328], dtype=torch.long)
    nz = torch.randn((B, 3, S, S), generator=torch.Generator().manual_seed(77))
    convs_called = []
    fwd = torch.nn.Conv2d._conv_forward
    monkeypatch.setattr(torch.nn.Conv2d, "_conv_forward", lambda self, *a, **k: (convs_called.append(self),
                                                                                 fwd(self, *a, **k))[1])
    res = {}
    try:
        for native in (True, False):
            U.NATIVE_TRAIN_CONV = native
            net.zero_grad(set_to_none=True)
            emu.calls.clear()
            convs_called.clear()
            library.clear()
            loss, _ = net.p_losses(x, y, y, t, nz)
            loss.backward()
            res[native] = (float(loss.detach()), {n: p.grad.detach().clone() for n, p in net.denoise_fn.named_parameters()},
                           set(emu.calls), len(convs_called), list(library))
    finally:
        U.NATIVE_TRAIN_CONV = True
        train.set_backend(None)
    assert res[True][3] == 0 and res[True][4] == [], res[True][4]
    assert res[False][3] > 0
    assert {"conv_umma", "conv_wgrad", "attention_bwd"} <= res[True][2]
    if tag == "mid_w96_rs":
        assert "s2d_split" in res[True][2]
    assert abs(res[True][0] - res[False][0]) < 1e-4 * abs(res[False][0])
    worst = max(rel_dev(res[True][1][n], res[False][1][n]) for n in res[False][1])
    assert worst < 3e-4, worst
