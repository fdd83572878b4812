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


def pack(be, w, dgrad=False):
    """wino_pack_weight into fresh NaN-filled planes -> (u_hi, u_lo, inv_wscale [1] fp32 on the device)."""
    Cout, Cin = w.shape[:2]
    uh = torch.full((36, Cin, Cout) if dgrad else (36, Cout, Cin), float("nan"), dtype=torch.float16, device=DEV)
    ul = torch.full_like(uh, float("nan"))
    inv = torch.full((1,), float("nan"), device=DEV)
    be.wino_pack_weight(w.to(DEV).contiguous(), uh, ul, dgrad=dgrad, inv_wscale=inv)
    return uh, ul, inv


def wino_u_ref(w, dgrad=False):
    """fp64 G g G^T [36, Cout, Cin] (dgrad: of the flipped, channel-swapped kernel, [36, Cin, Cout])."""
    w = w.double()
    if dgrad:
        w = w.flip(2, 3).transpose(0, 1)
    return torch.einsum("ij,kcjl,ml->imkc", G.to(w.device), w, G.to(w.device)).reshape(36, w.shape[0], w.shape[1])


def wino_chain(be, x1, x2, w, *, mean=None, rstd=None, gamma=None, beta=None, film=None, silu=True, bias=None,
               residual=None, res_mode=0, stats=False):
    """wino_input -> conv_umma(weights_per_image, operand_f16) -> wino_output, as the engine launches them.
    film = (scale, shift, stride).  Returns (out, partial sums or None, (v_hi, v_lo, u_hi, u_lo, inv_wscale, m))."""
    B, H, W, c1 = x1.shape
    C = c1 + (0 if x2 is None else x2.shape[3])
    Cout = w.shape[0]
    th, tw, mt, ok = be.wino_geometry(B, H, W)
    assert ok and mt == B * th * tw
    fkw = {} if film is None else dict(film_scale=film[0], film_shift=film[1], film_stride=film[2])
    vh = torch.full((36, mt, C), float("nan"), dtype=torch.float16, device=DEV)
    vl = torch.full_like(vh, float("nan"))
    be.wino_input(x1, x2, groups=32, mean=mean, rstd=rstd, gamma=gamma, beta=beta, silu=silu, v_hi=vh, v_lo=vl, **fkw)
    uh, ul, inv = pack(be, w)
    m = torch.full((36, mt, Cout), float("nan"), device=DEV)
    be.conv_umma(B=36, H=mt // 16, W=16, Cin=C, Cout=Cout, taps=1, a_hi=vh, a_lo=vl, w_hi=uh, w_lo=ul, out=m,
                 passes=3, weights_per_image=True, operand_f16=True)
    out = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    part = torch.full((B * th, Cout, 2), float("nan"), device=DEV) if stats else None
    be.wino_output(m, inv_wscale=inv, B=B, H=H, W=W, Cout=Cout, bias=bias, residual=residual, res_mode=res_mode,
                   out=out, stats_partial=part)
    torch.cuda.synchronize()
    be.check_fault()
    return out, part, (vh, vl, uh, ul, inv, m)


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


@pytest.mark.parametrize("case", CHAIN)
def test_wino_conv_chain_tensor_scale(be, case):
    """The CHAIN cases with the weight planes at their per-tensor scale (inv_wscale passed to pack and output, as the
    engines run them), against the same fp64 reference as the fixed-2^8 calls above."""
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
    d = lambda z: None if z is None else z.to(DEV)
    out, _, (_, _, _, _, inv, _) = wino_chain(be, d(x1), d(x2), d(w), mean=d(mean), rstd=d(rstd), gamma=d(gamma),
                                              beta=d(beta), bias=d(bias), residual=d(res), res_mode=res_mode)
    dev = rel_dev(out, want)
    print(f"\n[wino chain, per-tensor scale 1/{1 / float(inv):g}, {case}] rel dev vs fp64 conv {dev:.3e}")
    assert float(inv) != 2.0 ** -8
    assert not torch.isnan(out).any()
    assert dev < 8e-6, dev


# Chains on layered_input: activations with a mean per channel, as a model's GroupNorm groups have.  The position
# GEMMs' accumulation error then dominates (measured on an H100 80GB HBM3 at 400 W: up to 1.1e-5 at weight std 2e-2,
# 8.5e-6 / 8.9e-6 for the cfg2 output-block convs); the unit-variance CHAIN cases stay within 8e-6.
CHAIN_BOUND_BIASED = 1.6e-5


def layered_input(B, H, W, c1, c2, seed):
    """cat(x1, x2) with a different mean and spread in every GroupNorm group (a mis-indexed group shows), as fp32 on
    the device: (x1, x2 or None, x)."""
    C = c1 + c2
    x = rnd((B, H, W, C), seed) * torch.linspace(0.5, 2.0, C) + torch.linspace(-2.0, 2.0, C)
    x = x.to(DEV)
    x1, x2 = x[..., :c1].contiguous(), (x[..., c1:].contiguous() if c2 else None)
    return x1, x2, x


def film_rows(B, C, seed, scale=0.1, off=4):
    """FiLM scale/shift rows inside a wider [B, 2C + 8] buffer at offset `off`, as the engine passes them."""
    buf = (scale * rnd((B, 2 * C + 8), seed)).to(DEV)
    return buf[:, off:off + C], buf[:, off + C:off + 2 * C], buf.shape[1]


def wino_v_ref(act):
    """fp64 B^T d B of every 6x6 tile of the (zero-padded) NHWC tensor act -> [36, tiles, C]."""
    t = F.pad(act.permute(0, 3, 1, 2).double(), (1, 1, 1, 1)).unfold(2, 6, 4).unfold(3, 6, 4)
    bt = BT.to(act.device)
    return torch.einsum("ij,bcxyjk,lk->ilbxyc", bt, t, bt).reshape(36, -1, act.shape[3])


# cfg2 output-block concat widths: (1024,512) and (512,128) put a 48- / 20-channel group across the src1/src2 boundary.
# W = 40: 10 tiles per row, two segments of the staged kernel, the second one partial.
LAYOUT_CASES = [(2, 8, 40, 1024, 1024), (2, 8, 40, 1024, 512), (2, 12, 40, 512, 128), (2, 8, 40, 512, 0)]


@pytest.mark.parametrize("B,H,W,c1,c2", LAYOUT_CASES)
def test_wino_input_production_layouts(be, B, H, W, c1, c2):
    """wino_input as the engine and the training path call it: FiLM rows at an offset inside the wide film buffer,
    concat inputs, raw and activated split-bf16 planes -- against fp64."""
    C = c1 + c2
    x1, x2, x = layered_input(B, H, W, c1, c2, 30)
    mean, rstd = O.op_gn_stats(x, 32, 1e-5)
    gamma, beta = (1.0 + 0.1 * rnd((C,), 31)).to(DEV), (0.1 * rnd((C,), 32)).to(DEV)
    fs, fb, fstride = film_rows(B, C, 33)
    assert fstride == 2 * C + 8 and fs.storage_offset() == 4
    act = O.op_gn_act(x.double(), mean.double(), rstd.double(), gamma.double(), beta.double(), fs.double(),
                      fb.double(), True, 0)
    mt = B * (H // 4) * (W // 4)
    vh = torch.full((36, mt, C), float("nan"), dtype=torch.float16, device=DEV)
    vl = torch.full_like(vh, float("nan"))
    rh, rl, ah, al = (torch.full((B, H, W, C), float("nan"), dtype=torch.bfloat16, device=DEV) for _ in range(4))
    be.wino_input(x1, x2, groups=32, mean=mean, rstd=rstd, gamma=gamma, beta=beta, film_scale=fs, film_shift=fb,
                  film_stride=fstride, silu=True, v_hi=vh, v_lo=vl, raw_hi=rh, raw_lo=rl, act_hi=ah, act_lo=al)
    torch.cuda.synchronize()
    be.check_fault()
    got = vh.double() + vl.double()
    assert not torch.isnan(got).any()
    d = rel_dev(got, wino_v_ref(act))
    # raw planes: exactly the split of the input; act planes: the split of the fp32 activation
    h, l = O.bf16_split(x)
    assert torch.equal(rh.float(), h) and torch.equal(rl.float(), l)
    a = ah.float() + al.float()
    assert not torch.isnan(a).any()
    da = rel_dev(a, act)
    r = a.to(torch.bfloat16).float()
    assert bool(((r == ah.float()) | ((r - ah.float()).abs() == 2 * al.float().abs())).all()), "act_hi is not bf16(act)"
    print(f"\n[wino_input {(B, H, W, c1, c2)}] V rel dev {d:.3e}, act planes rel dev {da:.3e}")
    assert d < 2e-6, d
    assert da < 8e-6, da                    # a split-bf16 pair carries 16 bits: 2^-17 = 7.6e-6 of the element


@pytest.mark.parametrize("B,H,W,c1,c2", [(2, 8, 40, 512, 0), (2, 8, 40, 1024, 512)])
def test_wino_input_identity_mode(be, B, H, W, c1, c2):
    """mean == NULL, no SiLU (the data-gradient conv transforms dY as it is): the plain transform of the input."""
    C = c1 + c2
    x1, x2, x = layered_input(B, H, W, c1, c2, 40)
    mt = B * (H // 4) * (W // 4)
    vh = torch.full((36, mt, C), float("nan"), dtype=torch.float16, device=DEV)
    vl = torch.full_like(vh, float("nan"))
    be.wino_input(x1, x2, groups=32, silu=False, v_hi=vh, v_lo=vl)
    torch.cuda.synchronize()
    be.check_fault()
    got = vh.double() + vl.double()
    assert not torch.isnan(got).any()
    d = rel_dev(got, wino_v_ref(x))
    print(f"\n[wino_input identity {(B, H, W, c1, c2)}] rel dev {d:.3e}")
    assert d < 1e-6, d


PROD_CHAIN = [  # B, H, W, c1, c2, Cout: conv1 of the cfg2 output blocks
    (1, 64, 64, 1024, 512, 1024),      # level 2
    (1, 128, 128, 512, 128, 512),      # level 1; 640 input channels: 10 K-blocks, chunk 4 with a tail of 2
]


@pytest.mark.parametrize("case", PROD_CHAIN)
def test_wino_chain_production_size(be, case):
    """The whole chain at the size and concat layout of the cfg2 output-block conv1, with fp64 references on the GPU."""
    B, H, W, c1, c2, Cout = case
    C = c1 + c2
    x1, x2, x = layered_input(B, H, W, c1, c2, 50)
    w, bias = rnd((Cout, C, 3, 3), 51, 0.02).to(DEV), rnd((Cout,), 52, 0.1).to(DEV)
    mean, rstd = O.op_gn_stats(x, 32, 1e-5)
    gamma, beta = (1.0 + 0.1 * rnd((C,), 53)).to(DEV), (0.1 * rnd((C,), 54)).to(DEV)
    out, _, (vh, vl, uh, ul, inv, m) = wino_chain(be, x1, x2, w, mean=mean, rstd=rstd, gamma=gamma, beta=beta,
                                                  bias=bias)
    assert not torch.isnan(m).any() and not torch.isnan(out).any()
    dm = rel_dev(m, torch.bmm(vh.double() + vl.double(), (uh.double() + ul.double()).transpose(1, 2)))
    act = O.op_gn_act(x.double(), mean.double(), rstd.double(), gamma.double(), beta.double(), None, None, True, 0)
    d = rel_dev(out, O.op_conv_nhwc(act, w.double(), bias.double()))
    print(f"\n[wino chain {case}] position GEMMs {dm:.3e}, rel dev vs fp64 conv {d:.3e}")
    assert dm < 3e-6, dm
    assert d < CHAIN_BOUND_BIASED, d


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
