"""-m gpu: every kernel launch of one eager UNet forward of each benchmarked configuration, at the batch size bench.py
runs it, against an fp64 recomputation of that launch on the GPU (tests/_launch_shadow.py), and the cfg2 batch of 16
against its images run one at a time.

The fixture tests check the model end to end at B = 1 with a 1e-4 bound, about five times one F(6,3) chain's
deviation; here every launch is held to its own kernel's bound, per image, with the tile plans, argument layouts (FiLM
rows strided inside the projection buffer, reused pool buffers) and Winograd routes that the production batch sizes
take."""
import time

import pytest
import torch

from _launch_shadow import CFG2_FORMS, F43_FORMS, UPSAMPLE_FORMS, Shadow, missing_forms
from _recipe import UNET_CONFIGS, fill_state_dict, synth_images

pytestmark = pytest.mark.gpu

# bench.py's CONFIGS, restated: name -> (UNet of tests/_recipe.py, image side, batch)
CONFIGS = {"cfg2": ("cfg2", 256, 16), "cfg1": ("cfg1", 64, 4), "cfg3": ("lbbdm_f4", 64, 32),
           "cfg4": ("lbbdm_f8", 64, 64), "cfg5": ("lbbdm_f16", 64, 8)}
# forms each configuration must reach (a routing change that drops one from the check fails here); the 32x32 level of
# cfg3-cfg5 takes F(4,3) at their batch sizes, which cfg3 must show
REQUIRED = {"cfg2": CFG2_FORMS, "cfg1": UPSAMPLE_FORMS, "cfg3": F43_FORMS + UPSAMPLE_FORMS, "cfg4": UPSAMPLE_FORMS,
            "cfg5": UPSAMPLE_FORMS}


def _unet(name):
    from bbdm_b200.unet import UNetModel
    net = UNetModel(**UNET_CONFIGS[name]).eval()
    net.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1234))
    return net.cuda()


def _inputs(net, side, B, seed=11):
    """synth_images inputs; timesteps spread over 0..999, both ends included."""
    x = synth_images((B, net.out_channels, side, side), seed).cuda()
    y = None
    if net.condition_key != "nocond":
        y = synth_images((B, net.in_channels - net.out_channels, side, side), seed + 1).cuda()
    t = torch.linspace(0, 999, B).round().long().cuda()
    return x, t, y


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_every_launch_matches_its_fp64_recomputation(cfg):
    from bbdm_b200 import cabi
    from bbdm_b200.engine import UNetEngine
    name, side, B = CONFIGS[cfg]
    t0 = time.time()
    net = _unet(name)
    sh = Shadow(cabi.CudaBackend())
    eng = UNetEngine(net, backend=sh)
    eng.refresh_weights()
    sh.register_engine(eng)
    x, t, y = _inputs(net, side, B)
    out = eng.forward(x, t, y)
    assert torch.isfinite(out).all()
    fails = sh.failures()
    print(f"\n{sh.table(f'{cfg} ({name}, {side}x{side}, B={B})')}\n  wall time {time.time() - t0:.1f} s")
    for f in fails[:40]:
        print("  FAIL", f)
    assert not missing_forms(sh, REQUIRED[cfg])
    assert not fails, fails[:10]


def test_cfg2_production_batch_is_bit_identical_to_its_images_one_at_a_time():
    """Every image of the B = 16 cfg2 forward equals the B = 1 forward of that image bit for bit: GroupNorm statistics
    and every tile reduction are per image, in an order that does not depend on the batch, also where the conv plans of
    the two batch sizes differ (N tile, tiles per CTA)."""
    from bbdm_b200.engine import UNetEngine
    net = _unet("cfg2")
    eng = UNetEngine(net)
    x, t, y = _inputs(net, 256, 16)
    with torch.no_grad():
        full = eng.forward(x, t, y).clone()
        for i in range(16):
            one = eng.forward(x[i:i + 1], t[i:i + 1], y[i:i + 1])
            assert torch.equal(one[0], full[i]), i
    eng.be.check_fault()
