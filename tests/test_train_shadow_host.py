"""The launch shadow of tests/_launch_shadow.py over a training micro-step on the CPU emulation (no GPU): its fp64
references accept every launch of q_sample, the training forward and backward of a SpatialTransformer UNet and two
FusedAdam steps, every form the batch-32 GPU runs must reach occurs, and a perturbation of one launch's output -- in
one image, one weight-gradient row, one edge tile or one parameter element -- is flagged on that launch alone."""
import pytest
import torch

from _launch_shadow import ST_TRAIN_FORMS, Shadow, missing_forms
from _recipe import UNET_CONFIGS, bb_namespace, fill_state_dict, synth_images
from test_transformer_training_host import EmuBackend

# LBBDM-f4's layout at a quarter of its size: 64 channels at 32x32, 256 at 16x16, the middle block's transformer (4
# heads of 64) attending over the 32x32 3-channel context.  With the Winograd thresholds lowered, the 32x32 level takes
# the F(4,3) training forward and data gradient at B = 2 (128 tiles) while the 16x16 level stays on the direct
# tensor-core conv, as the 16x16 and 64x64 levels of the batch-32 run do.
HOST_UNET = dict(UNET_CONFIGS["lbbdm_f4"], image_size=32, in_channels=6, model_channels=64, num_res_blocks=1,
                 channel_mult=(1, 4), use_spatial_transformer=True, context_dim=3, condition_key="SpatialRescaler")
LR = 1e-4


def _train_step(monkeypatch, mutate=None):
    """q_sample, training forward, L1 loss, backward and two FusedAdam steps (same gradients) under the shadow."""
    from bbdm_b200 import train
    from bbdm_b200.bridge import BridgeOps
    from bbdm_b200.optim import FusedAdam
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    sh = Shadow(EmuBackend())
    sh.mutate = mutate or {}
    monkeypatch.setattr(train, "WINO_MIN_C", 64)
    monkeypatch.setattr(train, "WINO_MIN_TILES", 128)
    monkeypatch.setattr(BridgeOps, "backend_factory", staticmethod(lambda: sh))
    monkeypatch.setattr(FusedAdam, "backend_factory", staticmethod(lambda: sh))
    train.set_backend(sh)
    try:
        net = BrownianBridgeModel(bb_namespace(HOST_UNET)).train()
        net.denoise_fn.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()},
                                                       seed=1234))
        B = 2
        x, y = synth_images((B, 3, 32, 32), 1), synth_images((B, 3, 32, 32), 2)
        nz = torch.randn((B, 3, 32, 32), generator=torch.Generator().manual_seed(3))
        t = torch.tensor([0, 999])
        opt = FusedAdam(net.get_parameters(), lr=LR)
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
        opt.step()
        opt.step()
    finally:
        train.set_backend(None)
    return sh


@pytest.fixture(scope="module")
def clean():
    with pytest.MonkeyPatch.context() as mp:
        sh = _train_step(mp)
    print("\n" + sh.table("training micro-step, quarter-size LBBDM-f4 + SpatialTransformer, B=2, emulation"))
    return sh


def test_shadow_accepts_the_emulated_training_step(clean):
    assert not clean.failures(), clean.failures()[:5]
    assert not missing_forms(clean, ST_TRAIN_FORMS), missing_forms(clean, ST_TRAIN_FORMS)
    # every Winograd chain, the data-gradient ones included, was paired with the weight its planes were packed from
    chains = [c for c in clean.checks if c.what.startswith("chain")]
    assert len(chains) == sum(m == "wino_output" for m, _ in clean.launches) > 0
    assert any(c.what == "chain F(4,3) dgrad vs fp64 conv" for c in chains)
    assert sum(m == "adam_multi" for m, _ in clean.launches) == 2


def _edge(key, image):
    """1e-4 of the image's max |value| added to the last element (bottom-right pixel, last row) of one image."""
    def fn(a):
        o = a[key]
        o[image].view(-1)[-1] += 1e-4 * float(o[image].abs().max())
    return fn


def _last_cout_row(a):
    dw = a["dw"]
    dw[-1, -1].view(-1)[0] += 1e-4 * float(dw.abs().max())


def _last_parameter(a):
    # Adam's first step moves every parameter by about lr
    a["tab"].tensors[-1].data.view(-1)[0] += 1e-4 * a["lr"]


def _after(launches, i, method):
    return next(j for j in range(i + 1, len(launches)) if launches[j][0] == method)


CASES = {
    "gn_bwd_apply dx": lambda L: (next(i for i, (m, _) in enumerate(L) if m == "gn_bwd_apply"), _edge("dx", 1)),
    "conv_wgrad dW": lambda L: (next(i for i, (m, f) in enumerate(L) if m == "conv_wgrad" and f == "taps 9"),
                                _last_cout_row),
    "dgrad wino_output": lambda L: (_after(L, next(i for i, (m, f) in enumerate(L) if m == "wino_input" and
                                                   "identity" in f), "wino_output"), _edge("out", 1)),
    "attention_bwd dqkv": lambda L: (next(i for i, (m, _) in enumerate(L) if m == "attention_bwd"), _edge("dqkv", 1)),
    "adam_multi update": lambda L: (next(i for i, (m, _) in enumerate(L) if m == "adam_multi"), _last_parameter),
}


def test_shadow_flags_exactly_the_perturbed_launches(clean, monkeypatch):
    """The five perturbations in one run (each launch's references read its own cloned inputs, so a perturbed value
    that later launches consume is not flagged again): the flagged launches are exactly the perturbed ones."""
    targets = {name: pick(clean.launches) for name, pick in CASES.items()}
    sh = _train_step(monkeypatch, mutate=dict(targets.values()))
    assert sh.launches == clean.launches
    flagged = sh.flagged_launches()
    for name, (idx, _) in targets.items():
        assert idx in flagged, name
    assert flagged == sorted(idx for idx, _ in targets.values())
