"""-m gpu: the Winograd F(6x6,3x3) path (bbdm_wino6_* + bbdm_conv_umma with 64 weights_per_image position GEMMs)
against the fp64 convolution of the same activated input: weight planes, input transform (incl. the zero GEMM padding
rows and the raw split side outputs), and the whole chain with every residual mode and the GroupNorm partial sums, at
the UNet sampling executor's production shapes and at maps that do not divide into 6-pixel tiles."""
import pytest
import torch
import torch.nn.functional as F

from _recipe import rel_dev

pytestmark = pytest.mark.gpu
DEV = "cuda"
# Lavin & Gray F(6x6,3x3), points 0, +-1, +-2, +-1/2
BT = torch.tensor([[1, 0, -21 / 4, 0, 21 / 4, 0, -1, 0], [0, 1, 1, -17 / 4, -17 / 4, 1, 1, 0],
                   [0, -1, 1, 17 / 4, -17 / 4, -1, 1, 0], [0, 1 / 2, 1 / 4, -5 / 2, -5 / 4, 2, 1, 0],
                   [0, -1 / 2, 1 / 4, 5 / 2, -5 / 4, -2, 1, 0], [0, 2, 4, -5 / 2, -5, 1 / 2, 1, 0],
                   [0, -2, 4, 5 / 2, -5, -1 / 2, 1, 0], [0, -1, 0, 21 / 4, 0, -21 / 4, 0, 1]], dtype=torch.float64)
G = torch.tensor([[1, 0, 0], [-2 / 9, -2 / 9, -2 / 9], [-2 / 9, 2 / 9, -2 / 9], [1 / 90, 1 / 45, 2 / 45],
                  [1 / 90, -1 / 45, 2 / 45], [32 / 45, 16 / 45, 8 / 45], [32 / 45, -16 / 45, 8 / 45], [0, 0, 1]],
                 dtype=torch.float64)


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


def rnd(shape, seed, scale=1.0, dev=DEV):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).float().to(dev)


def pack6(be, w):
    Cout, Cin = w.shape[:2]
    uh = torch.full((64, Cout, Cin), float("nan"), dtype=torch.float16, device=DEV)
    ul = torch.full_like(uh, float("nan"))
    inv = torch.full((1,), float("nan"), device=DEV)
    be.wino_pack_weight(w.contiguous(), uh, ul, inv_wscale=inv, tile=6)
    return uh, ul, inv


def activation(x, mean, rstd, gamma, beta, fs, fsh, groups=32):
    """fp64 GroupNorm affine -> FiLM -> SiLU of NHWC x with per-(sample, group) mean / rstd."""
    B, H, W, C = x.shape
    xd = x.double().reshape(B, H, W, groups, C // groups)
    a = ((xd - mean.double()[:, None, None, :, None]) * rstd.double()[:, None, None, :, None]).reshape(B, H, W, C)
    a = a * gamma.double() + beta.double()
    a = a * (1 + fs.double()[:, None, None, :]) + fsh.double()[:, None, None, :]
    return F.silu(a)


def chain(be, x1, x2, w, bias, *, residual=None, res_mode=0, gn_scale=1.0, raw=False):
    """The engine's launch sequence at tile 6; returns (out, partials, raw planes, reference pieces)."""
    B, H, W, c1 = x1.shape
    C = c1 + (0 if x2 is None else x2.shape[3])
    Cout = w.shape[0]
    th, tw, mt, ok = be.wino_geometry(B, H, W, tile=6)
    assert ok and th == -(-H // 6) and tw == -(-W // 6) and mt == max(128, -(-B * th * tw // 16) * 16)
    x = x1 if x2 is None else torch.cat([x1, x2], 3)
    mean, rstd = rnd((B, 32), 5, 0.3), rnd((B, 32), 6, 0.2).abs() * gn_scale + 0.5 * gn_scale
    gamma, beta = rnd((C,), 7, 0.2) + 1, rnd((C,), 8, 0.2)
    fs, fsh = rnd((B, 2 * C), 9, 0.1), rnd((B, 2 * C), 10, 0.1)
    vh = torch.full((64, mt, C), float("nan"), dtype=torch.float16, device=DEV)
    vl = torch.full_like(vh, float("nan"))
    rh = rl = None
    if raw:
        rh, rl = (torch.full(x.shape, float("nan"), dtype=torch.bfloat16, device=DEV) for _ in range(2))
    be.wino_input(x1, x2, groups=32, mean=mean, rstd=rstd, gamma=gamma, beta=beta, silu=True, v_hi=vh, v_lo=vl,
                  film_scale=fs[:, :C], film_shift=fsh[:, :C], film_stride=2 * C, raw_hi=rh, raw_lo=rl, tile=6)
    uh, ul, inv = pack6(be, w)
    m = torch.full((64, mt, Cout), float("nan"), device=DEV)
    be.conv_umma(B=64, H=mt // 16, W=16, Cin=C, Cout=Cout, taps=1, a_hi=vh, a_lo=vl, w_hi=uh, w_lo=ul, out=m,
                 passes=3, weights_per_image=True, operand_f16=True)
    out = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    part = torch.full((B * th, Cout, 2), float("nan"), device=DEV)
    be.wino_output(m, inv_wscale=inv, B=B, H=H, W=W, Cout=Cout, bias=bias, residual=residual, res_mode=res_mode,
                   out=out, stats_partial=part, tile=6)
    torch.cuda.synchronize()
    be.check_fault()
    act = activation(x, mean, rstd, gamma, beta, fs[:, :C], fsh[:, :C])
    return out, part, (rh, rl), (x, act, vh, vl, uh, ul, inv, m, th, tw, mt)


def conv_ref(act, w, bias, residual, res_mode):
    y = F.conv2d(act.permute(0, 3, 1, 2), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    if res_mode == 1:
        y = y + residual.double()
    elif res_mode == 2:
        y = y + residual.double().repeat_interleave(2, 1).repeat_interleave(2, 2)
    elif res_mode == 3:
        r = residual.double().permute(0, 3, 1, 2)
        y = y + F.avg_pool2d(r, 2).permute(0, 2, 3, 1)
    return y


def test_wino6_pack_weight(be):
    w = rnd((128, 64, 3, 3), 1, 0.02)
    uh, ul, inv = pack6(be, w)
    u = torch.einsum("ij,kcjl,ml->imkc", G, w.double().cpu(), G).reshape(64, 128, 64)
    got = (uh.double() + ul.double()).cpu() * float(inv.item())
    assert rel_dev(got, u) < 1e-6
    assert float((uh.double().abs().max() * inv.double()).item()) <= 1.56 * float(w.abs().max())


# Deviation from the fp64 conv measured on an H100 (these GroupNorm + FiLM + SiLU activations have a positive mean, like
# the F(4,3) tests' biased chains, bound 1.6e-5): 3.9e-6 (48x48x256) to 1.60e-5 (256x256x512, batch 16) and 1.59e-5
# (128x128x512); the range cases 9.8e-6 / 8.9e-6.  The CPU study (tools/studies/winograd_f63_accuracy.py) puts F(6,3)
# at about 1.5x F(4,3).
CHAIN_BOUND = 2e-5

# (B, H, W, c1, c2, Cout, res_mode): production maps of the UNet sampling executor and ragged edge tiles
CASES = [(1, 64, 64, 1024, 1024, 1024, 1), (1, 64, 64, 1024, 512, 1024, 1), (1, 128, 128, 512, 0, 512, 0),
         (1, 128, 128, 1024, 0, 512, 1), (16, 256, 256, 512, 0, 64, 0), (2, 48, 48, 256, 0, 256, 2),
         (1, 70, 64, 256, 256, 256, 1), (2, 64, 64, 256, 0, 128, 3), (3, 50, 46, 128, 0, 128, 0)]


@pytest.mark.parametrize("case", CASES)
def test_wino6_chain_vs_fp64_conv(be, case):
    B, H, W, c1, c2, Cout, res_mode = case
    x1 = rnd((B, H, W, c1), 11)
    x2 = rnd((B, H, W, c2), 12) if c2 else None
    C = c1 + c2
    w = rnd((Cout, C, 3, 3), 13, 0.02)
    bias = rnd((Cout,), 14, 0.1)
    rshape = {0: None, 1: (B, H, W, Cout), 2: (B, H // 2, W // 2, Cout), 3: (B, 2 * H, 2 * W, Cout)}[res_mode]
    residual = None if rshape is None else rnd(rshape, 15)
    out, part, (rh, rl), (x, act, vh, vl, uh, ul, inv, m, th, tw, mt) = chain(
        be, x1, x2, w, bias, residual=residual, res_mode=res_mode, raw=(res_mode == 1))
    assert not torch.isnan(out).any()
    # the GEMM's padding rows are exact zeros
    assert bool((vh[:, B * th * tw:] == 0).all()) and bool((vl[:, B * th * tw:] == 0).all())
    want = conv_ref(act, w, bias, residual, res_mode)
    dev = rel_dev(out, want)
    print(f"F(6,3) chain {case}: rel dev {dev:.2e}")
    assert dev < CHAIN_BOUND, dev
    # GroupNorm partial sums: one row per (sample, tile row), summed over the real pixels only
    o64 = out.double()
    rows = torch.stack([o64[:, 6 * r:6 * r + 6].sum((1, 2)) for r in range(th)], 1).reshape(B * th, Cout)
    sq = torch.stack([(o64[:, 6 * r:6 * r + 6] ** 2).sum((1, 2)) for r in range(th)], 1).reshape(B * th, Cout)
    assert rel_dev(part[..., 0], rows) < 1e-5 and rel_dev(part[..., 1], sq) < 1e-5
    if rh is not None:
        assert torch.equal((rh.float() + rl.float()).cpu(), (x.bfloat16().float() + (x - x.bfloat16().float()).bfloat16().float()).cpu())


def test_wino6_input_transform_exact_positions(be):
    """V planes against B^T d B of the fp64 activation, edge tiles included (70 x 64 map)."""
    B, H, W, C = 1, 70, 64, 128
    x1 = rnd((B, H, W, C), 21)
    w = rnd((64, C, 3, 3), 22, 0.02)
    _, _, _, (x, act, vh, vl, *_rest) = chain(be, x1, None, w, rnd((64,), 23))
    th, tw = -(-H // 6), -(-W // 6)
    a = F.pad(act.permute(0, 3, 1, 2), (1, 1 + 6 * tw - W, 1, 1 + 6 * th - H))
    t = a.unfold(2, 8, 6).unfold(3, 8, 6)                                          # [B, C, th, tw, 8, 8]
    V = torch.einsum("ij,bcxyjk,lk->ilbxyc", BT.to(DEV), t, BT.to(DEV)).reshape(64, B * th * tw, C)
    got = vh[:, :B * th * tw].double() + vl[:, :B * th * tw].double()
    assert rel_dev(got, V) < 1e-6


@pytest.mark.parametrize("amp", [4.0, 40.0])
def test_wino6_input_range(be, amp):
    """Activations far above GroupNorm scale stay finite and accurate: |act| up to ~200 (the fp16 V planes hold
    225 max|act| < 65504 up to max|act| = 291)."""
    B, H, W, C, Cout = 2, 48, 48, 256, 128
    x1 = rnd((B, H, W, C), 31)
    w = rnd((Cout, C, 3, 3), 32, 0.02)
    bias = rnd((Cout,), 33, 0.1)
    out, _, _, (x, act, *_rest) = chain(be, x1, None, w, bias, gn_scale=amp)
    assert float(act.abs().max()) > amp
    assert torch.isfinite(out).all()
    dev = rel_dev(out, conv_ref(act, w, bias, None, 0))
    print(f"F(6,3) range amp {amp}: max|act| {float(act.abs().max()):.1f}, rel dev {dev:.2e}")
    assert dev < CHAIN_BOUND, dev


def test_wino6_input_range_is_reported(be):
    """Activations past the fp16 range of the V planes (max|act| ~ 290) are not silent: the kernel completes, and the
    device status word that bbdm_check_device_fault reads names the launch.  In range, the word stays clear."""
    from bbdm_b200 import cabi
    B, H, W, C, Cout = 2, 48, 48, 256, 128
    x1 = rnd((B, H, W, C), 41)
    w = rnd((Cout, C, 3, 3), 42, 0.02)
    chain(be, x1, None, w, rnd((Cout,), 43), gn_scale=4.0)          # the chain itself checks the word is clear
    with pytest.raises(cabi.BbdmError, match="F\\(6x6,3x3\\) input transform of a 256-channel conv"):
        chain(be, x1, None, w, rnd((Cout,), 43), gn_scale=400.0)
    be.check_fault()                                                  # reading the word cleared it
