"""-m gpu: the up-ResBlocks' nearest-2x + 3x3 conv as a phase-stacked F(6x6,3x3) conv on the low-res map
(WeightPacker.up_phase_winograd planes, convs.wino_conv(up2_phases=True): wino6 input -> 64 position GEMMs with 4*Cout
outputs -> the up-phase output transform) against the fp64 conv2d(nearest2x(GroupNorm-SiLU(x))), with the GroupNorm
partial sums, at both production shapes of the cfg2 UNet and on a ragged low-res map."""
import pytest
import torch
import torch.nn.functional as F

from _recipe import rel_dev

pytestmark = pytest.mark.gpu
DEV = "cuda"
# the F(6,3) chain bound of tests/test_gpu_winograd6.py
CHAIN_BOUND = 2e-5


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).float().to(DEV)


# (B, h, w, Cin, Cout): the two up-ResBlock conv1s of cfg2 (64x64 -> 128x128 at 1024 channels, 128x128 -> 256x256 at
# 512) and a low-res map that does not divide into 6-pixel tiles
CASES = [(2, 64, 64, 1024, 1024), (2, 128, 128, 512, 512), (3, 13, 10, 128, 192)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c)))
def test_up_phase_chain_matches_fp64_conv_of_upsampled_activation(be, case):
    from bbdm_b200 import convs
    B, h, w, Cin, Cout = case
    x = rnd((B, h, w, Cin), 1)
    wt, bias = rnd((Cout, Cin, 3, 3), 2, 0.02), rnd((Cout,), 3, 0.1)
    mean, rstd = rnd((B, 32), 5, 0.3), rnd((B, 32), 6, 0.2).abs() + 0.5
    gamma, beta = rnd((Cin,), 7, 0.2) + 1, rnd((Cin,), 8, 0.2)
    packer = convs.WeightPacker(be, torch.device(DEV))
    packer.conv("c", wt, bias)
    packer.up_phase_winograd("c", wt)
    u = packer.w["c"]["up6"]
    th = -(-h // 6)
    out = convs.wino_conv(be, convs.FreshBuffers(DEV), be.wino_geometry(B, h, w, tile=6), x, None, cout=Cout,
                          planes=(u["u_hi"], u["u_lo"], u["u_inv"]), bias=bias, stats=True, tile=6, up2_phases=True,
                          groups=32, mean=mean, rstd=rstd, gamma=gamma, beta=beta, silu=True)
    torch.cuda.synchronize()
    be.check_fault()
    xd = x.double().reshape(B, h, w, 32, Cin // 32)
    a = ((xd - mean.double()[:, None, None, :, None]) * rstd.double()[:, None, None, :, None]).reshape(B, h, w, Cin)
    a = F.silu(a * gamma.double() + beta.double()).permute(0, 3, 1, 2)
    ref = F.conv2d(F.interpolate(a, scale_factor=2, mode="nearest"), wt.double(), bias.double(), padding=1)
    ref = ref.permute(0, 2, 3, 1)
    assert out.shape == ref.shape and torch.isfinite(out).all()
    dev = rel_dev(out, ref)
    print(f"{case}: rel dev {dev:.2e}")
    assert dev < CHAIN_BOUND
    # GroupNorm partial sums: one row per (sample, tile row, phase), over the row's 6 low-res rows -- against fp64
    # sums of the stored output
    part, rows = out._gn
    assert rows == 4 * th and part.shape == (B * rows, Cout, 2)
    r = F.pad(out.double().reshape(B, h, 2, w, 2, Cout), (0, 0, 0, 0, 0, 0, 0, 0, 0, 6 * th - h))
    r = r.reshape(B, th, 6, 2, w, 2, Cout)
    want = torch.stack([r.sum(dim=(2, 4)), (r * r).sum(dim=(2, 4))], -1).reshape(B * rows, Cout, 2)
    scale = want.abs().amax(dim=0, keepdim=True)
    assert float(((part.double() - want).abs() / (scale + 1e-30)).max()) < 1e-5
