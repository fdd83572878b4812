"""-m gpu: the F(6x6,3x3) chains the UNet sampling executor gained for its wide-input conv1s and its down-ResBlock
conv1 against fp64, with the GroupNorm partial sums:
- the 2x2-pooled input form (down2): conv2d(avg_pool2(GroupNorm-SiLU(x))) at cfg2's 128x128 -> 64x64 block at 512
  channels and on a ragged pooled map from odd source sides;
- a two-source 640 -> 128 chain (cfg2's 256x256 conv1 after the skip concat) with the raw split-bf16 planes for the
  fused 1x1 skip, at production width and on a ragged map."""
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


def gn_silu(x, mean, rstd, gamma, beta):
    B, H, W, C = x.shape
    xd = x.double().reshape(B, H, W, 32, C // 32)
    a = ((xd - mean.double()[:, None, None, :, None]) * rstd.double()[:, None, None, :, None]).reshape(B, H, W, C)
    return F.silu(a * gamma.double() + beta.double()).permute(0, 3, 1, 2)


def check_partials(out, th):
    B, H, W, C = out.shape
    part, rows = out._gn
    assert rows == th and part.shape == (B * rows, C, 2)
    r = F.pad(out.double(), (0, 0, 0, 0, 0, 6 * th - H)).reshape(B, th, 6 * W, C)
    want = torch.stack([r.sum(2), (r * r).sum(2)], -1).reshape(B * rows, C, 2)
    scale = want.abs().amax(dim=0, keepdim=True)
    assert float(((part.double() - want).abs() / (scale + 1e-30)).max()) < 1e-5


def chain(be, src1, src2, wt, bias, gkw, *, h, w, down2=False, raw=None):
    from bbdm_b200 import convs
    B = src1.shape[0]
    Cout = wt.shape[0]
    packer = convs.WeightPacker(be, torch.device(DEV))
    packer.conv("c", wt, bias)
    packer.winograd("c", wt, tile=6)
    e = packer.w["c"]
    kw = dict(down2=True) if down2 else {}
    if raw is not None:
        kw.update(raw_hi=raw[0], raw_lo=raw[1])
    out = convs.wino_conv(be, convs.FreshBuffers(DEV), be.wino_geometry(B, h, w, tile=6), src1, src2, cout=Cout,
                          planes=(e["u_hi"], e["u_lo"], e["u_inv"]), bias=bias, stats=True, tile=6, **gkw, **kw)
    torch.cuda.synchronize()
    be.check_fault()
    return out


# (B, H, W, C, Cout) of the source map: cfg2's down-ResBlock (128x128 -> 64x64 at 512 channels) and odd source sides
POOLED = [(2, 128, 128, 512, 512), (3, 27, 31, 128, 192)]


@pytest.mark.parametrize("case", POOLED, ids=lambda c: "x".join(map(str, c)))
def test_pooled_chain_matches_fp64_conv_of_pooled_activation(be, case):
    B, H, W, C, Cout = case
    x = rnd((B, H, W, C), 1)
    wt, bias = rnd((Cout, C, 3, 3), 2, 0.02), rnd((Cout,), 3, 0.1)
    mean, rstd = rnd((B, 32), 5, 0.3), rnd((B, 32), 6, 0.2).abs() + 0.5
    gamma, beta = rnd((C,), 7, 0.2) + 1, rnd((C,), 8, 0.2)
    h, w = H // 2, W // 2
    out = chain(be, x, None, wt, bias, dict(groups=32, mean=mean, rstd=rstd, gamma=gamma, beta=beta, silu=True),
                h=h, w=w, down2=True)
    ref = F.conv2d(F.avg_pool2d(gn_silu(x, mean, rstd, gamma, beta), 2), wt.double(), bias.double(), padding=1)
    ref = ref.permute(0, 2, 3, 1)
    assert out.shape == ref.shape == (B, h, w, Cout) and torch.isfinite(out).all()
    dev = rel_dev(out, ref)
    print(f"{case}: rel dev {dev:.2e}")
    assert dev < CHAIN_BOUND
    check_partials(out, -(-h // 6))


# (B, H, W, c1, c2, Cout): cfg2's 640 -> 128 conv1 at 256x256, and a ragged map
TWO_SOURCE = [(1, 256, 256, 512, 128, 128), (2, 25, 19, 128, 128, 128)]


@pytest.mark.parametrize("case", TWO_SOURCE, ids=lambda c: "x".join(map(str, c)))
def test_two_source_chain_with_raw_planes_matches_fp64(be, case):
    B, H, W, c1, c2, Cout = case
    C = c1 + c2
    x1, x2 = rnd((B, H, W, c1), 11), rnd((B, H, W, c2), 12)
    wt, bias = rnd((Cout, C, 3, 3), 13, 0.02), rnd((Cout,), 14, 0.1)
    mean, rstd = rnd((B, 32), 15, 0.3), rnd((B, 32), 16, 0.2).abs() + 0.5
    gamma, beta = rnd((C,), 17, 0.2) + 1, rnd((C,), 18, 0.2)
    r_hi = torch.empty((B, H, W, C), dtype=torch.bfloat16, device=DEV)
    r_lo = torch.empty_like(r_hi)
    out = chain(be, x1, x2, wt, bias, dict(groups=32, mean=mean, rstd=rstd, gamma=gamma, beta=beta, silu=True),
                h=H, w=W, raw=(r_hi, r_lo))
    x = torch.cat([x1, x2], 3)
    ref = F.conv2d(gn_silu(x, mean, rstd, gamma, beta), wt.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    assert out.shape == ref.shape and torch.isfinite(out).all()
    dev = rel_dev(out, ref)
    print(f"{case}: rel dev {dev:.2e}")
    assert dev < CHAIN_BOUND
    check_partials(out, -(-H // 6))
    # the raw input's split-bf16 planes (A operand of the fused 1x1 skip): every pixel, hi + lo within bf16 pair rounding
    raw = r_hi.double() + r_lo.double()
    assert float((raw - x.double()).abs().max() / x.abs().max()) < 2e-5
