"""-m gpu: the Winograd F(4x4,3x3) path (csrc/winograd.cu + bbdm_conv_umma in weights_per_image / fp16 mode)
against the fp64 convolution of the same activated input (the oracle's op_gn_act + conv), kernel by kernel and as
the full chain the engine launches."""
import pytest
import torch
import torch.nn.functional as F

from _recipe import rel_dev
from oracle import bbdm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
BT = torch.tensor([[4, 0, -5, 0, 1, 0], [0, -4, -4, 1, 1, 0], [0, 4, -4, -1, 1, 0],
                   [0, -2, -1, 2, 1, 0], [0, 2, -1, -2, 1, 0], [0, 4, 0, -5, 0, 1]], dtype=torch.float64)
G = torch.tensor([[1 / 4, 0, 0], [-1 / 6, -1 / 6, -1 / 6], [-1 / 6, 1 / 6, -1 / 6],
                  [1 / 24, 1 / 12, 1 / 6], [1 / 24, -1 / 12, 1 / 6], [0, 0, 1]], dtype=torch.float64)


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).float()


def test_wino_pack_weight(be):
    Cout, Cin = 128, 192
    w = rnd((Cout, Cin, 3, 3), 1, 0.02)
    uh = torch.empty((36, Cout, Cin), dtype=torch.float16, device=DEV)
    ul = torch.empty_like(uh)
    be.wino_pack_weight(w.to(DEV), uh, ul)
    want = (torch.einsum("ij,kcjl,ml->imkc", G, w.double(), G) * 256.0).reshape(36, Cout, Cin)
    got = uh.double().cpu() + ul.double().cpu()
    assert rel_dev(got, want) < 2e-7                       # 22 mantissa bits
    assert float((uh.float().cpu() - want.float().to(torch.float16).float()).abs().max()) <= 2e-3 * float(want.abs().max())


@pytest.mark.parametrize("B,H,W,c1,c2,film", [(2, 32, 32, 128, 0, True), (1, 16, 64, 64, 64, False), (3, 8, 8, 256, 0, True)])
def test_wino_input_transform(be, B, H, W, c1, c2, film):
    C = c1 + c2
    x1, x2 = rnd((B, H, W, c1), 2, 1.5), (rnd((B, H, W, c2), 3, 1.5) if c2 else None)
    x = x1 if x2 is None else torch.cat([x1, x2], 3)
    mean, rstd = O.op_gn_stats(x, 32, 1e-5)
    gamma, beta = 1.0 + 0.1 * rnd((C,), 4), 0.1 * rnd((C,), 5)
    fs, fb = (0.1 * rnd((B, C), 6), 0.1 * rnd((B, C), 7)) if film else (None, None)
    act = O.op_gn_act(x, mean, rstd, gamma, beta, fs, fb, True, 0)
    t = F.pad(act.permute(0, 3, 1, 2).double(), (1, 1, 1, 1)).unfold(2, 6, 4).unfold(3, 6, 4)
    want = torch.einsum("ij,bcxyjk,lk->ilbxyc", BT, t, BT).reshape(36, -1, C)
    mt = B * (H // 4) * (W // 4)
    vh = torch.full((36, mt, C), float("nan"), dtype=torch.float16, device=DEV)
    vl = torch.full_like(vh, float("nan"))
    rh = torch.empty((B, H, W, C), dtype=torch.bfloat16, device=DEV)
    rl = torch.empty_like(rh)
    d = lambda z: None if z is None else z.to(DEV)
    kw = dict(film_scale=d(fs), film_shift=d(fb), film_stride=C) if film else {}
    be.wino_input(d(x1), d(x2), groups=32, mean=d(mean), rstd=d(rstd), gamma=d(gamma), beta=d(beta), silu=True,
                  v_hi=vh, v_lo=vl, raw_hi=rh, raw_lo=rl, **kw)
    got = vh.double().cpu() + vl.double().cpu()
    assert not torch.isnan(got).any()
    # fp32 SiLU (fast exp/div) + fp32 transform: a few 1e-7 of the largest transformed value
    assert rel_dev(got, want) < 2e-6, rel_dev(got, want)
    h, l = O.bf16_split(x)
    assert torch.equal(rh.float().cpu(), h) and torch.equal(rl.float().cpu(), l)


CHAIN = [  # B, H, W, c1, c2, Cout, res_mode
    (2, 32, 32, 256, 0, 256, 0),
    (2, 32, 32, 128, 128, 512, 1),
    (1, 16, 128, 64, 0, 192, 2),       # N tile 64, nearest-up residual
    (8, 16, 16, 320, 0, 128, 3),       # 2x2-avg residual, K = 5 blocks (odd chunk count)
    (1, 64, 64, 1024, 0, 256, 1),      # long K: 16 K-blocks, 8 promotion chunks
]


@pytest.mark.parametrize("case", CHAIN)
def test_wino_conv_chain_vs_fp64_conv(be, case):
    B, H, W, c1, c2, Cout, res_mode = case
    C = c1 + c2
    x1, x2 = rnd((B, H, W, c1), 10, 1.5), (rnd((B, H, W, c2), 11, 1.5) if c2 else None)
    x = x1 if x2 is None else torch.cat([x1, x2], 3)
    w, bias = rnd((Cout, C, 3, 3), 12, 0.02), rnd((Cout,), 13, 0.1)
    mean, rstd = O.op_gn_stats(x, 32, 1e-5)
    gamma, beta = 1.0 + 0.1 * rnd((C,), 14), 0.1 * rnd((C,), 15)
    act = O.op_gn_act(x, mean, rstd, gamma, beta, None, None, True, 0)
    want = O.op_conv_nhwc(act.double(), w.double(), bias.double())
    res = None
    if res_mode == 1:
        res = rnd((B, H, W, Cout), 16)
        want = want + res.double()
    elif res_mode == 2:
        res = rnd((B, H // 2, W // 2, Cout), 16)
        want = want + O.op_resample(res, 1).double()
    elif res_mode == 3:
        res = rnd((B, H * 2, W * 2, Cout), 16)
        want = want + O.op_resample(res.double(), 2)
    th, tw, mt, ok = be.wino_geometry(B, H, W)
    assert ok and mt == B * th * tw
    d = lambda z: None if z is None else z.to(DEV)
    vh = torch.empty((36, mt, C), dtype=torch.float16, device=DEV)
    vl = torch.empty_like(vh)
    be.wino_input(d(x1), d(x2), groups=32, mean=d(mean), rstd=d(rstd), gamma=d(gamma), beta=d(beta), silu=True,
                  v_hi=vh, v_lo=vl)
    uh = torch.empty((36, Cout, C), dtype=torch.float16, device=DEV)
    ul = torch.empty_like(uh)
    be.wino_pack_weight(d(w), uh, ul)
    m = torch.full((36, mt, Cout), float("nan"), device=DEV)
    be.conv_umma(B=36, H=mt // 16, W=16, Cin=C, Cout=Cout, taps=1, a_hi=vh, a_lo=vl, w_hi=uh, w_lo=ul, out=m,
                 passes=3, weights_per_image=True, operand_f16=True)
    torch.cuda.synchronize()
    be.check_fault()
    assert not torch.isnan(m).any()
    # the 36 position GEMMs themselves: fp64 evaluation of the same split products
    V, U = vh.double() + vl.double(), uh.double() + ul.double()
    m_want = torch.bmm(V, U.transpose(1, 2))
    assert rel_dev(m, m_want) < 3e-6, rel_dev(m, m_want)
    out = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    part = torch.full((B * th, Cout, 2), float("nan"), device=DEV)
    be.wino_output(m, B=B, H=H, W=W, Cout=Cout, bias=d(bias), residual=d(res), res_mode=res_mode, out=out,
                   stats_partial=part)
    dev = rel_dev(out, want)
    print(f"\n[wino chain {case}] rel dev vs fp64 conv {dev:.3e}")
    assert not torch.isnan(out).any()
    assert dev < 8e-6, dev
    # fused GroupNorm partial sums of the result (rows_per_image = tiles_h)
    s = part.view(B, th, Cout, 2).double().sum(1).cpu()
    o64 = out.double().cpu().reshape(B, -1, Cout)
    assert rel_dev(s[..., 0], o64.sum(1)) < 1e-5 and rel_dev(s[..., 1], (o64 ** 2).sum(1)) < 1e-5
    mean2, rstd2 = torch.empty((B, 32), device=DEV), torch.empty((B, 32), device=DEV)
    be.gn_finalize_partials(part, th, None, 0, B, H * W, 32, 1e-5, mean2, rstd2)
    mw, rw = O.op_gn_stats(out.cpu(), 32, 1e-5)
    assert rel_dev(mean2, mw) < 1e-5 and rel_dev(rstd2, rw) < 1e-5


FP16_CONV_CASES = [
    # B, H, W, Cin, Cout, passes
    (2, 16, 16, 128, 128, 3),                                # BN=64, one tile per CTA
    (2, 16, 16, 128, 128, 1),
    (4, 64, 64, 128, 256, 3), (4, 64, 64, 128, 256, 1),      # BN=128, several tiles per CTA
]


def test_conv_umma_fp16_operands_direct_conv(be):
    """operand_f16 on the ordinary 3x3 implicit GEMM: split-fp16 planes (22 mantissa bits) instead of split-bf16."""
    _check_fp16_direct_conv(be, *FP16_CONV_CASES[0])


@pytest.mark.parametrize("B,H,W,Cin,Cout,passes", FP16_CONV_CASES[1:])
def test_conv_umma_fp16_operands_direct_conv_plans(be, B, H, W, Cin, Cout, passes):
    """The same at passes 1 and with the BN=128 multi-tile plan."""
    _check_fp16_direct_conv(be, B, H, W, Cin, Cout, passes)


def _check_fp16_direct_conv(be, B, H, W, Cin, Cout, passes):
    """passes=3 is compared with the exact conv, passes=1 with the fp64 conv of the hi planes it multiplies."""
    a, w = rnd((B, H, W, Cin), 20).to(DEV), rnd((Cout, Cin, 3, 3), 21, 0.02).to(DEV)

    def split16(x):
        h = x.to(torch.float16)
        return h, (x - h.float()).to(torch.float16)
    a_hi, a_lo = split16(a)
    w_hi, w_lo = split16((w * 256.0).permute(2, 3, 0, 1).reshape(9, Cout, Cin).contiguous())
    out = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=9, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo, out=out,
                 passes=passes, operand_f16=True)
    if passes == 3:
        want = O.op_conv_nhwc(a.double(), w.double() * 256.0, None)
    else:
        want = O.op_conv_nhwc(a_hi.double(), (w * 256.0).to(torch.float16).double(), None)
    d = rel_dev(out, want)
    print(f"\n[direct conv, split-fp16 x{passes}] rel dev vs fp64 conv {d:.3e}")
    assert d < 2e-6, d
