"""The launch shadow of tests/_launch_shadow.py over the CPU emulation (no GPU): its fp64 references accept every launch
of a cfg2-architecture forward, and a perturbation of one launch's output in one image is flagged on that launch alone.

The emulation's contract differs from the kernels' in where it puts the GroupNorm partial sums (all in row 0 of each
image) and in the tile count it pads the F(6,3) GEMMs to; the shadow compares only what the consumers read (the per-image
sums of the partial rows, the real tiles plus zero padding rows), so the same checks hold for both."""
import pytest
import torch

from _emu_backend_f63_pool import EmuBackendF63Pool
from _launch_shadow import CFG2_FORMS, Shadow, missing_forms
from _recipe import UNET_CONFIGS, fill_state_dict, synth_images
from bbdm_b200 import cabi, convs
from bbdm_b200.engine import KernelExecutor, UNetEngine
from bbdm_b200.unet import UNetModel

# The cfg2 UNet at half its channel widths, one ResBlock per level, image_size 192: levels at 192, 96 and 48 (64, 256,
# 512 channels).  Every F(6,3) form and every direct form that cfg2 routes to occurs here (the coverage assertion
# below), at about a seventh of the cfg2 architecture's CPU time.
SMALL_CFG2 = dict(UNET_CONFIGS["cfg2"], image_size=192, model_channels=64, num_res_blocks=1)
# The F(6,3) chain bound of the kernels is 2e-5 (the GPU launches of cfg1-cfg5 measure up to 1.84e-5).  The emulated
# chain reaches 2.06e-5 here (96x96, 256 -> 256 with residual) although its transforms are exact fp64 and its GEMM fp32:
# that is the deviation of F(6,3) with 22-bit fp16-pair planes on these activations, which the emulation shares with
# the kernels, not an error of the checker.
EMU_BOUNDS = {"chain6": 2.5e-5}


@pytest.fixture(scope="module")
def cfg2_shadow():
    net = UNetModel(**SMALL_CFG2).eval()
    net.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1234))
    sh = Shadow(EmuBackendF63Pool(), bounds=EMU_BOUNDS)
    eng = UNetEngine(net, backend=sh)
    eng.refresh_weights()
    sh.register_engine(eng)
    x, y = synth_images((1, 3, 192, 192), 1), synth_images((1, 3, 192, 192), 2)
    eng.forward(x, torch.tensor([500]), y)
    print("\n" + sh.table("cfg2 architecture, half width, 192x192, B=1, emulation"))
    return sh


def test_shadow_accepts_the_emulation_on_the_cfg2_architecture(cfg2_shadow):
    sh = cfg2_shadow
    assert not sh.failures(), sh.failures()[:5]
    assert not missing_forms(sh, CFG2_FORMS)
    # every Winograd chain was paired with its GEMM, its input transform and its module weight
    chains = [c for c in sh.checks if c.what.startswith("chain")]
    assert len(chains) == sum(m == "wino_output" for m, _ in sh.launches) > 0
    assert any(c.what == "phase taps vs module weight" for c in sh.checks)


def _resblock_flow(B, side, mutate=None):
    """A 128 -> 256 ResBlock on a side x side map with a 1x1 skip: conv1 on the direct tensor-core conv (128 inputs are
    below the F(6,3) channel rule), conv2 on F(6,3) with the skip GEMM's output as its residual.  side 44 leaves a
    ragged edge tile (8 tiles of 6 for 44 pixels)."""
    g = torch.Generator().manual_seed(side)
    cin, cout = 128, 256
    w1, w2, ws = (0.05 * torch.randn(s, generator=g) for s in ((cout, cin, 3, 3), (cout, cout, 3, 3), (cout, cin, 1, 1)))
    b1, b2, bs = (0.1 * torch.randn(cout, generator=g) for _ in range(3))
    norm1, norm2 = torch.nn.GroupNorm(32, cin), torch.nn.GroupNorm(32, cout)
    sh = Shadow(EmuBackendF63Pool())
    ex = KernelExecutor(backend=sh)
    packer = convs.WeightPacker(sh, torch.device("cpu"))
    e1, e2, es = packer.conv("c1", w1, b1), packer.conv("c2", w2, b2), packer.conv("skip", ws, bs)
    packer.winograd("c2", w2, tile=6)
    sh._weights[e2["u_hi"].data_ptr()] = (w2, False, "c2")
    sh.mutate = mutate or {}
    x = torch.randn(B, side, side, cin, generator=g)
    film = (0.1 * torch.randn(B, cout, generator=g), 0.1 * torch.randn(B, cout, generator=g))
    ex._resblock_flow(ex._pool(torch.device("cpu"), ("t", B)), x, None, norm1, norm2, e1, e2, es, cabi.RESAMPLE_NONE,
                      film=film)
    return sh


def test_resblock_flow_is_clean_and_routes_as_intended():
    sh = _resblock_flow(2, 44)
    assert not sh.failures(), sh.failures()[:5]
    forms = set(sh.launches)
    assert ("conv_umma", "taps 9 stats") in forms and ("wino_output", "F(6,3) res 1") in forms


def _perturb_last_pixel(key, image):
    """Adds 1e-4 of the image's max |value| to the last pixel (the bottom-right edge tile of an F(6,3) output) of one
    image of the launch's output `key`."""
    def fn(args):
        o = args[key]
        o[image, -1, -1, 0] += 1e-4 * float(o[image].abs().max())
    return fn


@pytest.mark.parametrize("target", ["wino_output", "conv_umma"])
def test_shadow_flags_exactly_the_perturbed_launch(target):
    clean = _resblock_flow(2, 44)
    idx = next(i for i, (m, form) in enumerate(clean.launches)
               if m == target and (target != "conv_umma" or form.startswith("taps 9")))
    sh = _resblock_flow(2, 44, mutate={idx: _perturb_last_pixel("out", 1)})
    assert sh.launches == clean.launches
    assert sh.flagged_launches() == [idx]
