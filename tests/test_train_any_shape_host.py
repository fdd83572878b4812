"""Training at any map size and batch, host side (CPU): the one tensor-core gate (convs.tensor_core_ok) admits every
shape the forward takes, and a training step of the mid_pixel UNet at 48x48, batch 3 -- no level of which is a 64-pixel
box -- runs every conv on the native Functions (emulated kernels) and matches the stock graph."""
import pytest
import torch

from _emu_backend import EmuBackend
from _recipe import UNET_CONFIGS, bb_namespace, fill_state_dict, rel_dev, synth_images


class RaggedEmu(EmuBackend):
    """The emulation with bbdm_split_grad / bbdm_conv_wgrad's padded dY^T planes: [C, P] views whose rows are P rounded
    up to 8 apart (the pitch the kernel's TMA map needs), checked on every call."""

    def __init__(self):
        super().__init__()
        self.pitches = []

    def _check(self, t, rows, cols):
        assert tuple(t.shape) == (rows, cols) and t.stride(1) == 1 and t.stride(0) == -(-cols // 8) * 8, \
            (t.shape, t.stride())
        self.pitches.append((cols, t.stride(0)))

    def split_grad(self, src, hi, lo, hi_t, lo_t, colsum=None, workspace=None):
        self._check(hi_t, src.shape[-1], src.numel() // src.shape[-1])
        super().split_grad(src, hi, lo, hi_t, lo_t, colsum, workspace)

    def conv_wgrad(self, g_hi_t, g_lo_t, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, workspace):
        self._check(g_hi_t, Cout, B * H * W)
        super().conv_wgrad(g_hi_t, g_lo_t, a_hi, a_lo, B, H, W, Cin, Cout, taps, dw, workspace)


@pytest.fixture()
def emu():
    from bbdm_b200 import train
    be = RaggedEmu()
    train.set_backend(be)
    yield be
    train.set_backend(None)


# (UNet input, batch, channels per level): the levels of cfg2-style UNets at the sizes image-translation data and
# latent models use, and small per-rank batches -- the 64-pixel box rule took none, or only some, of them
GATE_TABLE = [
    (224, 8, (128, 512, 1024)), (320, 8, (128, 512, 1024)), (384, 8, (128, 512, 1024)), (96, 32, (128, 512, 1024)),
    (16, 6, (128, 512, 1024)), (256, 16, (128, 512, 1024)), (512, 2, (128, 256, 512)), (48, 3, (64, 128, 256)),
    (28, 3, (64, 128, 256)),
]


@pytest.mark.parametrize("size,batch,chans", GATE_TABLE)
def test_tensor_core_gate_admits_every_level(emu, size, batch, chans):
    from bbdm_b200 import convs, engine, train
    for lvl, c in enumerate(chans):
        s = size >> lvl
        x = torch.empty((batch, c, s, s))
        conv3 = torch.nn.Conv2d(c, c, 3, padding=1)
        conv1 = torch.nn.Conv2d(2 * c, c, 1)
        assert convs.tensor_core_ok(c, c, s)
        assert engine.KernelExecutor._umma_ok(None, c, c, s)                 # sampling: the same rule
        assert train.native_ok(conv3, x) and train.native_ok(conv1, torch.empty((batch, 2 * c, s, s)))


def test_tensor_core_gate_rejects_only_channels_and_narrow_maps():
    from bbdm_b200 import convs, train
    assert not hasattr(train, "_box64_ok") and not hasattr(train, "_tc_grid_ok")
    for B, H, W in [(1, 7, 7), (3, 7, 7), (2, 24, 40), (6, 4, 4), (5, 9, 13), (1, 1, 4)]:
        assert convs.tensor_core_ok(64, 128, W)
    assert not convs.tensor_core_ok(64, 128, 3)
    assert not convs.tensor_core_ok(96, 128, 32) and not convs.tensor_core_ok(64, 32, 32)


def test_training_step_48x48_batch3_matches_torch_graph(emu, monkeypatch):
    import bbdm_b200.unet as U
    from bbdm_b200.bridge import BridgeOps
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    monkeypatch.setattr(BridgeOps, "backend_factory", staticmethod(lambda: emu))          # q_sample
    net = BrownianBridgeModel(bb_namespace(dict(UNET_CONFIGS["mid_pixel"], image_size=48))).train()
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(fill_state_dict(shapes, seed=1234))
    B, S = 3, 48
    x, y = synth_images((B, 3, S, S), seed=11), synth_images((B, 3, S, S), seed=12)
    t = torch.tensor([(17 + 311 * i) % 1000 for i in range(B)], dtype=torch.long)
    nz = torch.randn((B, 3, S, S), generator=torch.Generator().manual_seed(77))
    res = {}
    convs_called = []
    fwd = torch.nn.Conv2d._conv_forward
    monkeypatch.setattr(torch.nn.Conv2d, "_conv_forward", lambda self, *a, **k: (convs_called.append(self),
                                                                                 fwd(self, *a, **k))[1])
    try:
        for native in (True, False):
            U.NATIVE_TRAIN_CONV = native
            net.zero_grad(set_to_none=True)
            emu.calls.clear()
            convs_called.clear()
            loss, _ = net.p_losses(x, y, y, t, nz)
            loss.backward()
            res[native] = (float(loss.detach()), {n: p.grad.detach().clone() for n, p in net.denoise_fn.named_parameters()},
                           set(emu.calls), len(convs_called))
    finally:
        U.NATIVE_TRAIN_CONV = True
    assert res[True][3] == 0, f"{res[True][3]} Conv2d module calls on the library path"
    assert res[False][3] > 0
    assert {"conv_umma", "conv_wgrad", "gn_bwd_reduce", "gn_bwd_apply", "attention_bwd"} <= res[True][2]
    # every level's weight gradient: 48x48, 24x24, 12x12 at batch 3
    assert {P for P, _ in emu.pitches} >= {3 * 48 * 48, 3 * 24 * 24, 3 * 12 * 12}
    assert abs(res[True][0] - res[False][0]) < 1e-4 * abs(res[False][0])
    worst = max(rel_dev(res[True][1][n], res[False][1][n]) for n in res[False][1])
    assert worst < 3e-4, worst
