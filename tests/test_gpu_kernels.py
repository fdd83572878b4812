"""-m gpu: every C-ABI kernel against its oracle restatement on the same seeded inputs."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from _recipe import rel_dev
from oracle import bbdm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).float()


# ------------------------------------------------------------------------------------ bridge
@pytest.mark.parametrize("objective", ["grad", "noise", "ysubx"])
def test_q_sample_bit_exact(be, objective):
    bufs, _ = O.make_schedule()
    B, shape = 5, (5, 3, 24, 24)
    x0, y, nz = rnd(shape, 1, 0.5), rnd(shape, 2, 0.5), rnd(shape, 3)
    t = torch.tensor([0, 1, 499, 998, 999])
    want_xt, want_obj = O.q_sample(bufs, x0, y, t, nz, objective)
    xt, obj = torch.empty(shape, device=DEV), torch.empty(shape, device=DEV)
    be.q_sample(x0.to(DEV), y.to(DEV), nz.to(DEV), t.to(DEV), bufs["m_t"].to(DEV), bufs["variance_t"].to(DEV),
                objective, xt, obj)
    assert torch.equal(xt.cpu(), want_xt) and torch.equal(obj.cpu(), want_obj)


@pytest.mark.parametrize("objective,eta", [("grad", 1.0), ("noise", 1.0), ("ysubx", 0.5)])
@pytest.mark.parametrize("clip", [False, True])
def test_p_sample_update_bit_exact(be, objective, eta, clip):
    from bbdm_b200.schedule import step_coefficients
    bufs, steps = O.make_schedule(sample_step=50)
    coef = step_coefficients(bufs["m_t"], bufs["variance_t"], steps, eta)
    shape = (3, 3, 20, 20)
    xt, y, eps, nz = rnd(shape, 4, 0.7), rnd(shape, 5, 0.5), rnd(shape, 6, 0.6), rnd(shape, 7)
    for i in (0, 1, 25, len(steps) - 2, len(steps) - 1):
        want, want_x0 = O.p_sample_update(bufs, steps, i, xt, y, eps, nz, objective, eta, clip)
        out, x0 = torch.empty(shape, device=DEV), torch.empty(shape, device=DEV)
        last = int(steps[i]) == 0
        be.p_sample(xt.to(DEV), y.to(DEV), eps.to(DEV), None if last else nz.to(DEV), coef[i].tolist(),
                    objective, clip, last, out, x0)
        assert torch.equal(x0.cpu(), want_x0), (objective, i)
        assert torch.equal(out.cpu(), want), (objective, i)


# ------------------------------------------------------------------------------------ layout / dense
def test_layout_roundtrip_and_cat(be):
    x, c = rnd((3, 3, 10, 12), 8), rnd((3, 5, 10, 12), 9)
    out = torch.empty((3, 10, 12, 8), device=DEV)
    be.nchw_to_nhwc_cat(x.to(DEV), c.to(DEV), out)
    assert torch.equal(out.cpu(), torch.cat([x, c], 1).permute(0, 2, 3, 1).contiguous())
    back = torch.empty((3, 8, 10, 12), device=DEV)
    be.nhwc_to_nchw(out, back)
    assert torch.equal(back.cpu(), torch.cat([x, c], 1))
    out1 = torch.empty((3, 10, 12, 3), device=DEV)
    be.nchw_to_nhwc_cat(x.to(DEV), None, out1)
    assert torch.equal(out1.cpu(), x.permute(0, 2, 3, 1).contiguous())


def test_gather_and_linear(be):
    tab = rnd((1000, 128), 10)
    idx = torch.tensor([999, 0, 17, 500, 3, 3, 998, 1, 2])
    out = torch.empty((9, 128), device=DEV)
    be.gather_rows(tab.to(DEV), idx.to(DEV), out)
    assert torch.equal(out.cpu(), tab[idx])
    x, w, b = rnd((9, 128), 11), rnd((515, 128), 12, 0.05), rnd((515,), 13, 0.02)
    for ai, ao in ((False, False), (True, False), (False, True)):
        o = torch.empty((9, 515), device=DEV)
        be.linear(x.to(DEV), w.to(DEV), b.to(DEV), o, act_in=ai, act_out=ao)
        z = torch.nn.functional.silu(x.double()) if ai else x.double()
        z = z @ w.double().T + b.double()
        z = torch.nn.functional.silu(z) if ao else z
        assert rel_dev(o, z) < 2e-6


# ------------------------------------------------------------------------------------ group norm / prep
@pytest.mark.parametrize("B,H,W,c1,c2", [(2, 16, 16, 128, 0), (3, 8, 8, 512, 128), (2, 4, 4, 32, 0),
                                         (2, 12, 10, 96, 32), (1, 64, 64, 1024, 512), (2, 8, 8, 35 * 32 // 32 * 32, 0)])
def test_gn_stats(be, B, H, W, c1, c2):
    from bbdm_b200 import cabi
    s1 = rnd((B, H, W, c1), 20) + 0.3
    s2 = (rnd((B, H, W, c2), 21, 2.0) - 0.5) if c2 else None
    x = s1 if s2 is None else torch.cat([s1, s2], 3)
    m_want, r_want = O.op_gn_stats(x)
    mean, rstd = torch.empty((B, 32), device=DEV), torch.empty((B, 32), device=DEV)
    ws = torch.empty(B * 32 * cabi.GN_MAX_SLICES * 2, dtype=torch.float64, device=DEV)
    be.gn_stats(s1.to(DEV), None if s2 is None else s2.to(DEV), 32, 1e-5, mean, rstd, ws)
    assert (mean.cpu() - m_want).abs().max() < 2e-6 and rel_dev(rstd, r_want) < 2e-6
    m2, r2 = torch.empty_like(mean), torch.empty_like(rstd)
    be.gn_stats(s1.to(DEV), None if s2 is None else s2.to(DEV), 32, 1e-5, m2, r2, ws)
    assert torch.equal(mean, m2) and torch.equal(rstd, r2)          # deterministic


@pytest.mark.parametrize("resample", [0, 1, 2])
@pytest.mark.parametrize("c1,c2,film,silu", [(128, 0, True, True), (512, 128, False, True), (32, 0, True, True),
                                              (64, 0, False, False), (1120, 0, False, True)])
def test_prep_operand(be, resample, c1, c2, film, silu):
    B, Hs, Ws = 2, 8, 12
    C = c1 + c2
    s1 = rnd((B, Hs, Ws, c1), 30)
    s2 = rnd((B, Hs, Ws, c2), 31, 1.5) if c2 else None
    x = s1 if s2 is None else torch.cat([s1, s2], 3)
    mean, rstd = O.op_gn_stats(x)
    gamma, beta = 1 + 0.1 * rnd((C,), 32), 0.1 * rnd((C,), 33)
    fbuf = 0.2 * rnd((B, 3 * C + 8), 34)
    fs, fh = (fbuf[:, 4:4 + C], fbuf[:, 4 + C:4 + 2 * C]) if film else (None, None)
    want_act = O.op_gn_act(x.double(), mean.double(), rstd.double(), gamma.double(), beta.double(),
                           None if fs is None else fs.double(), None if fh is None else fh.double(), silu, resample)
    want_raw = O.op_resample(x, resample)
    H, W = want_raw.shape[1:3]
    d = lambda t: None if t is None else t.to(DEV)
    act_f32, raw_f32 = torch.empty((B, H, W, C), device=DEV), torch.empty((B, H, W, C), device=DEV)
    bf = lambda: torch.empty((B, H, W, C), dtype=torch.bfloat16, device=DEV)
    act_hi, act_lo, raw_hi, raw_lo = bf(), bf(), bf(), bf()
    fdev = d(fbuf)
    be.prep(d(s1), d(s2), groups=32, mean=d(mean), rstd=d(rstd), gamma=d(gamma), beta=d(beta),
            film_scale=None if not film else fdev[:, 4:4 + C], film_shift=None if not film else fdev[:, 4 + C:4 + 2 * C],
            film_stride=fbuf.shape[1], silu=silu, resample=resample, act_f32=act_f32, act_hi=act_hi, act_lo=act_lo,
            raw_f32=raw_f32, raw_hi=raw_hi, raw_lo=raw_lo)
    assert rel_dev(act_f32, want_act) < 5e-6
    assert rel_dev(raw_f32, want_raw) < 1e-6
    # split planes: hi is exactly bf16(value), hi + lo reproduces the fp32 value to ~2^-17
    hi, lo = O.bf16_split(act_f32.cpu())
    assert torch.equal(act_hi.float().cpu(), hi) and torch.equal(act_lo.float().cpu(), lo)
    hi, lo = O.bf16_split(raw_f32.cpu())
    assert torch.equal(raw_hi.float().cpu(), hi) and torch.equal(raw_lo.float().cpu(), lo)
    assert rel_dev(act_hi.float() + act_lo.float(), act_f32) < 2 ** -16


# ------------------------------------------------------------------------------------ convolutions
def _pack_split(be, w):
    k = w.shape[-1]
    hi = torch.empty((k * k, w.shape[0], w.shape[1]), dtype=torch.bfloat16, device=DEV)
    lo = torch.empty_like(hi)
    be.pack_weight_split(w.to(DEV).contiguous(), hi, lo)
    return hi, lo


def test_pack_weights(be):
    w = rnd((128, 64, 3, 3), 40, 0.02)
    hi, lo = _pack_split(be, w)
    want = w.permute(2, 3, 0, 1).reshape(9, 128, 64)
    h, l = O.bf16_split(want)
    assert torch.equal(hi.float().cpu(), h) and torch.equal(lo.float().cpu(), l)
    f = torch.empty((9, 64, 128), device=DEV)
    be.pack_weight_f32(w.to(DEV), f)
    assert torch.equal(f.cpu(), w.permute(2, 3, 1, 0).reshape(9, 64, 128))


@pytest.mark.parametrize("B,H,W,Cin,Cout,k,stride", [(2, 16, 16, 6, 128, 3, 1), (2, 9, 11, 35, 3, 3, 1), (1, 16, 16, 128, 3, 3, 1),
                                                      (2, 8, 8, 32, 96, 1, 1), (2, 16, 16, 32, 32, 3, 2), (3, 4, 4, 64, 200, 3, 1)])
def test_conv_direct(be, B, H, W, Cin, Cout, k, stride):
    a = rnd((B, H, W, Cin), 41)
    w, b = rnd((Cout, Cin, k, k), 42, 0.05), rnd((Cout,), 43, 0.1)
    want = torch.nn.functional.conv2d(a.permute(0, 3, 1, 2).double(), w.double(), b.double(), stride=stride,
                                      padding=k // 2).permute(0, 2, 3, 1)
    res = rnd(tuple(want.shape), 44)
    wp = torch.empty((k * k, Cin, Cout), device=DEV)
    be.pack_weight_f32(w.to(DEV), wp)
    out = torch.empty(tuple(want.shape), device=DEV)
    be.conv_direct(a.to(DEV), wp, b.to(DEV), res.to(DEV), out, Cout, k, stride)
    assert rel_dev(out, want + res.double()) < 3e-6


CONV_CASES = [
    # B, H,  W,  Cin, Cout, taps, Cin2, res_mode
    # (tile plans: tests/_conv_plan.py; unless noted, a case runs BN=64 with one tile per CTA on 114 and 132 SMs)
    (2, 16, 16, 64, 64, 9, 0, 0),        # smallest aligned case
    (2, 16, 16, 128, 128, 9, 0, 1),      # same-res residual
    (1, 32, 32, 128, 256, 9, 64, 0),     # fused 1x1 skip operand
    (2, 8, 8, 256, 512, 9, 0, 2),        # TW=8 tile geometry, nearest-up residual
    (2, 16, 16, 64, 128, 9, 0, 3),       # 2x2-avg residual
    (3, 4, 4, 256, 256, 9, 0, 1),        # tile spans several images (TB=8 > B: OOB batch rows)
    (2, 12, 20, 64, 64, 9, 0, 1),        # ragged: H, W not multiples of the box
    (2, 16, 16, 128, 384, 1, 0, 1),      # 1x1 (qkv / proj_out shape)
    (1, 64, 64, 640, 128, 9, 640, 0),    # output-block shape: concat width + 1x1 skip
    (5, 16, 16, 1024, 1024, 9, 0, 1),    # K = 9216 (144 K-blocks); BN=64 with 160 tiles on 132 SMs, BN=128 on 114
    # the plans production runs: BN=128 with several tiles per CTA on 114 and 132 SMs
    (4, 64, 64, 128, 256, 9, 0, 1),      # KB 18: partial last promotion chunk
    (1, 256, 256, 128, 128, 9, 0, 1),    # level-0 geometry of the 256x256 model: 512 tiles
    (4, 64, 64, 256, 256, 9, 128, 0),    # fused 1x1 skip operand: KB 36 + 2
    (8, 32, 32, 512, 512, 9, 0, 2),      # nearest-up residual, KB 72
    (4, 64, 64, 128, 256, 9, 0, 3),      # 2x2-avg residual
    (4, 64, 64, 64, 256, 1, 0, 1),       # KB 1: the ring advances once per tile
    (4, 32, 32, 1024, 1024, 9, 0, 1),    # long K: KB 144
    (4, 64, 64, 128, 192, 9, 0, 1),      # BN=64 forced by Cout, several tiles per CTA
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("passes", [3, 1])
def test_conv_umma(be, case, passes):
    B, H, W, Cin, Cout, taps, Cin2, res_mode = case
    k = 3 if taps == 9 else 1
    a = rnd((B, H, W, Cin), 50).to(DEV)          # fp64 references on the GPU: the large cases take minutes on a CPU
    w, b = rnd((Cout, Cin, k, k), 51, 0.02).to(DEV), rnd((Cout,), 52, 0.1).to(DEV)
    a_hi, a_lo = (t.to(torch.bfloat16) for t in O.bf16_split(a))
    w_hi, w_lo = _pack_split(be, w)
    kw = {}
    d64 = torch.float64
    if passes == 3:
        want = O.op_conv_split3(a, w, b)
    else:
        want = O.op_conv_nhwc(O.bf16_split(a)[0].to(d64), O.bf16_split(w)[0].to(d64), b.to(d64))
    if Cin2:
        a2, w2, b2 = (t.to(DEV) for t in (rnd((B, H, W, Cin2), 53), rnd((Cout, Cin2, 1, 1), 54, 0.02), rnd((Cout,), 55, 0.1)))
        a2_hi, a2_lo = (t.to(torch.bfloat16) for t in O.bf16_split(a2))
        w2_hi, w2_lo = _pack_split(be, w2)
        kw = dict(Cin2=Cin2, a2_hi=a2_hi, a2_lo=a2_lo, w2_hi=w2_hi, w2_lo=w2_lo, bias2=b2)
        want = want + (O.op_conv_split3(a2, w2, b2) if passes == 3 else
                       O.op_conv_nhwc(O.bf16_split(a2)[0].to(d64), O.bf16_split(w2)[0].to(d64), b2.to(d64)))
    res = None
    if res_mode == 1:
        res = rnd((B, H, W, Cout), 56).to(DEV)
        want = want + res.double()
    elif res_mode == 2:
        res = rnd((B, H // 2, W // 2, Cout), 56).to(DEV)
        want = want + O.op_resample(res, 1).double()
    elif res_mode == 3:
        res = rnd((B, H * 2, W * 2, Cout), 56).to(DEV)
        want = want + O.op_resample(res.double(), 2)
    out = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    oh = torch.full((B, H, W, Cout), float("nan"), dtype=torch.bfloat16, device=DEV)
    ol = torch.full_like(oh, float("nan"))
    be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=taps, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo,
                 bias=b, residual=res, res_mode=res_mode, out=out, out_hi=oh, out_lo=ol, passes=passes, **kw)
    torch.cuda.synchronize()
    be.check_fault()
    assert not torch.isnan(out).any()
    # the kernel differs from the fp64 evaluation of the same split products only by fp32 accumulation
    assert rel_dev(out, want) < 6e-6, rel_dev(out, want)
    if passes == 3 and Cin2 == 0 and res_mode == 0:      # and the split scheme itself is fp32-class accurate
        assert rel_dev(out, O.op_conv_nhwc(a.double(), w.double(), b.double())) < 3e-5     # vs the exact conv
    h, l = O.bf16_split(out.cpu())
    assert torch.equal(oh.float().cpu(), h) and torch.equal(ol.float().cpu(), l)


def _uniform(shape, seed, lo, hi):
    g = torch.Generator().manual_seed(seed)
    return (lo + (hi - lo) * torch.rand(shape, generator=g)).float()


@pytest.mark.parametrize("case", [(4, 32, 32, 1024, 1024, 128), (2, 16, 16, 1024, 1024, 64)])
@pytest.mark.parametrize("passes", [3, 1])
def test_conv_umma_long_k_positive_operands(be, case, passes):
    """K = 9216 (144 K-blocks) with strictly positive operands, at both N tiles.  The tensor core's accumulator add
    truncates; with one sign, those errors add up instead of cancelling, so a chain that is not promoted to the fp32
    register accumulator every few K-blocks drifts.  Compared with the fp64 evaluation of the same split products;
    two launches must be bit-identical.  Measured on an H100 80GB HBM3 (132 SMs, 400 W power limit), both N tiles:
    1.1e-6 at passes 3 and 8.4e-7 at passes 1; with the whole chain left in the wgmma accumulator (no promotion)
    5.8e-5 and 3.7e-5."""
    from _conv_plan import conv_plan
    B, H, W, Cin, Cout, BN = case
    plan = conv_plan(B, H, W, Cin, Cout, 9, passes=passes)
    assert plan["BN"] == BN and plan["KB"] == 144
    a, w = _uniform((B, H, W, Cin), 57, 0.25, 1.25).to(DEV), _uniform((Cout, Cin, 3, 3), 58, 0.0, 0.02).to(DEV)
    a_hi, a_lo = (t.to(torch.bfloat16) for t in O.bf16_split(a))
    w_hi, w_lo = _pack_split(be, w)
    if passes == 3:
        want = O.op_conv_split3(a, w)
    else:
        want = O.op_conv_nhwc(O.bf16_split(a)[0].double(), O.bf16_split(w)[0].double())
    outs = []
    for _ in range(2):
        outs.append(torch.full((B, H, W, Cout), float("nan"), device=DEV))
        be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=9, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo,
                     out=outs[-1], passes=passes)
    torch.cuda.synchronize()
    be.check_fault()
    assert torch.equal(outs[0], outs[1])
    d = rel_dev(outs[0], want)
    print(f"\n[conv long K, positive operands, BN={BN} passes={passes}] rel dev {d:.3e}")
    assert d < 4e-6, d


def test_conv_umma_rejects_bad_shapes(be):
    from bbdm_b200.cabi import BbdmError
    z = torch.zeros(8, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(BbdmError, match="Cin"):
        be.conv_umma(B=1, H=8, W=8, Cin=48, Cout=64, taps=9, a_hi=z, a_lo=z, w_hi=z, w_lo=z, out=z)


# ------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("B,T,heads,D,order", [(2, 256, 4, 64, 0), (1, 1024, 2, 64, 0), (2, 16, 8, 32, 0),
                                                (2, 64, 4, 16, 1), (1, 100, 2, 64, 1), (2, 4096, 1, 64, 0)])
def test_attention(be, B, T, heads, D, order):
    C = heads * D
    qkv = rnd((B, T, 3 * C), 60, 1.2)
    want = O.op_attention_nhwc(qkv.double(), heads, bool(order))
    out = torch.empty((B, T, C), device=DEV)
    oh = torch.empty((B, T, C), dtype=torch.bfloat16, device=DEV)
    ol = torch.empty_like(oh)
    be.attention(qkv.to(DEV), heads, order, out_f32=out, out_hi=oh, out_lo=ol)
    assert rel_dev(out, want) < 2e-5, rel_dev(out, want)
    h, l = O.bf16_split(out.cpu())
    assert torch.equal(oh.float().cpu(), h) and torch.equal(ol.float().cpu(), l)


def test_conv_umma_head_mode_nchw_padded(be):
    """UNet head: 3 real couts zero-padded to one 64-wide N tile, result stored as NCHW."""
    B, H, W, Cin, Cout = 2, 32, 32, 128, 3
    a, w, b = rnd((B, H, W, Cin), 70), rnd((Cout, Cin, 3, 3), 71, 0.02), rnd((Cout,), 72, 0.1)
    a_hi, a_lo = (t.to(torch.bfloat16).to(DEV) for t in O.bf16_split(a))
    hi = torch.zeros((9, 64, Cin), dtype=torch.bfloat16, device=DEV)
    lo = torch.zeros_like(hi)
    be.pack_weight_split(w.to(DEV), hi, lo)
    assert float(hi[:, Cout:].float().abs().max()) == 0.0
    bias = torch.zeros(64, device=DEV)
    bias[:Cout] = b.to(DEV)
    out = torch.full((B, Cout, H, W), float("nan"), device=DEV)
    be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=64, taps=9, a_hi=a_hi, a_lo=a_lo, w_hi=hi, w_lo=lo, bias=bias,
                 out=out, passes=3, out_nchw_channels=Cout)
    want = O.op_conv_split3(a, w, b).permute(0, 3, 1, 2)
    assert rel_dev(out, want) < 6e-6


@pytest.mark.parametrize("B,T,heads,D,order", [(2, 256, 4, 64, 0), (1, 1024, 2, 64, 0), (2, 16, 8, 32, 0),
                                                (2, 64, 4, 16, 1), (1, 100, 2, 64, 1), (1, 4096, 2, 64, 0),
                                                (1, 200, 3, 32, 1)])
def test_attention_split(be, B, T, heads, D, order):
    """Attention core fed with the pre-split qkv planes the qkv conv epilogue writes."""
    C = heads * D
    qkv = rnd((B, T, 3 * C), 61, 1.2)
    hi, lo = O.bf16_split(qkv)
    want = O.op_attention_nhwc((hi + lo).double(), heads, bool(order))     # exact result for the planes' value
    out = torch.empty((B, T, C), device=DEV)
    oh = torch.empty((B, T, C), dtype=torch.bfloat16, device=DEV)
    ol = torch.empty_like(oh)
    be.attention_split(hi.to(torch.bfloat16).to(DEV), lo.to(torch.bfloat16).to(DEV), heads, order,
                       out_f32=out, out_hi=oh, out_lo=ol)
    assert rel_dev(out, want) < 2e-5, rel_dev(out, want)
    assert rel_dev(out, O.op_attention_nhwc(qkv.double(), heads, bool(order))) < 5e-5
    h, l = O.bf16_split(out.cpu())
    assert torch.equal(oh.float().cpu(), h) and torch.equal(ol.float().cpu(), l)


GN_STATS_CONV_CASES = [
    # B, H, W, Cin, Cout, c2
    (2, 16, 16, 64, 128, 0), (3, 32, 16, 128, 256, 64), (2, 12, 20, 64, 64, 0), (2, 16, 8, 64, 640, 128),
    (4, 64, 64, 128, 256, 0),      # BN=128, several tiles per CTA: the 128-wide statistics loop
    (4, 64, 64, 128, 256, 128),    # ... and a concat whose second conv also runs BN=128
]


@pytest.mark.parametrize("B,H,W,Cin,Cout,c2", GN_STATS_CONV_CASES)
def test_conv_umma_fused_groupnorm_statistics(be, B, H, W, Cin, Cout, c2):
    """GroupNorm partial sums written by the conv epilogue + finalize == statistics of the stored
    tensor (also for the concat of two conv outputs whose groups straddle the boundary)."""
    def conv_with_stats(cout, seed):
        a, w, b = rnd((B, H, W, Cin), seed), rnd((cout, Cin, 3, 3), seed + 1, 0.05), rnd((cout,), seed + 2, 0.3)
        a_hi, a_lo = (t.to(torch.bfloat16).to(DEV) for t in O.bf16_split(a))
        w_hi, w_lo = _pack_split(be, w)
        rows = be.conv_geometry(H, W)[3]
        assert rows > 0
        part = torch.full((B * rows, cout, 2), float("nan"), device=DEV)
        out = torch.empty((B, H, W, cout), device=DEV)
        be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=cout, taps=9, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo,
                     bias=b.to(DEV), out=out, passes=3, stats_partial=part)
        assert not torch.isnan(part).any()
        return out, part, rows

    o1, p1, r1 = conv_with_stats(Cout, 80)
    o2 = p2 = None
    r2 = 0
    if c2:
        o2, p2, r2 = conv_with_stats(c2, 90)
    x = o1.cpu() if o2 is None else torch.cat([o1.cpu(), o2.cpu()], 3)
    m_want, r_want = O.op_gn_stats(x)
    mean, rstd = torch.empty((B, 32), device=DEV), torch.empty((B, 32), device=DEV)
    be.gn_finalize_partials(p1, r1, p2, r2, B, H * W, 32, 1e-5, mean, rstd)
    assert (mean.cpu() - m_want).abs().max() < 3e-6 and rel_dev(rstd, r_want) < 3e-6
    assert be.conv_geometry(4, 4)[3] == 0        # tile spans images: caller must use bbdm_gn_stats


UPSAMPLE_CONV_CASES = [
    # B, H, W, Cin, Cout, res     (H, W: the low-res input)
    (2, 8, 8, 64, 64, False), (2, 16, 16, 128, 256, True), (1, 12, 20, 64, 128, False), (3, 4, 4, 256, 256, True),
    (4, 32, 32, 256, 256, True),   # BN=128, several tiles per CTA
]


@pytest.mark.parametrize("B,H,W,Cin,Cout,res", UPSAMPLE_CONV_CASES)
def test_conv_umma_fused_upsample(be, B, H, W, Cin, Cout, res):
    """nearest-2x + 3x3 conv as 4 phases x 2x2 taps on the low-res operand == conv on the upsampled tensor."""
    from bbdm_b200.weights import upsample_phase_weights
    a, w, b = rnd((B, H, W, Cin), 100).to(DEV), rnd((Cout, Cin, 3, 3), 101, 0.03), rnd((Cout,), 102, 0.1).to(DEV)
    a_hi, a_lo = (t.to(torch.bfloat16) for t in O.bf16_split(a))
    wp = upsample_phase_weights(w).to(DEV)
    w = w.to(DEV)
    hi = torch.empty((16, Cout, Cin), dtype=torch.bfloat16, device=DEV)
    lo = torch.empty_like(hi)
    be.pack_weight_split_taps(wp, hi, lo)
    a_val = sum(O.bf16_split(a)).double()                       # the value the planes carry
    want = O.op_conv_nhwc(O.op_resample(a_val, 1), w.double(), b.double())
    r = None
    if res:
        r = rnd((B, H, W, Cout), 103).to(DEV)
        want = want + O.op_resample(r.double(), 1)
    rows = 4 * be.conv_geometry(H, W)[3]
    part = torch.full((B * rows, Cout, 2), float("nan"), device=DEV) if rows else None
    out = torch.full((B, 2 * H, 2 * W, Cout), float("nan"), device=DEV)
    be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=4, a_hi=a_hi, a_lo=a_lo, w_hi=hi, w_lo=lo, bias=b,
                 residual=r, res_mode=2 if res else 0, out=out, passes=3, upsample2x=True, stats_partial=part)
    be.check_fault()
    assert not torch.isnan(out).any()
    assert rel_dev(out, want) < 3e-5           # weights are re-split after the tap sums: 2^-17-level difference
    if part is not None:
        mean, rstd = torch.empty((B, 32), device=DEV), torch.empty((B, 32), device=DEV)
        be.gn_finalize_partials(part, rows, None, 0, B, 4 * H * W, 32, 1e-5, mean, rstd)
        m_want, r_want = O.op_gn_stats(out.cpu())
        assert (mean.cpu() - m_want).abs().max() < 3e-6 and rel_dev(rstd, r_want) < 3e-6


def test_conv_cases_cover_dispatch_regimes(be):
    """The conv and weight-gradient cases of the suite, planned for this card, run every kernel instantiation and
    tile-plan regime the host can choose.  The N-tile and grid rules depend on the SM count; if they change, this
    fails until the cases are moved back into the regimes they claim."""
    from _conv_plan import conv_geometry, conv_plan, num_sms, wgrad_plan
    from test_gpu_training import WG_CASES
    from test_gpu_winograd import CHAIN, FP16_CONV_CASES, PROD_CHAIN
    from test_gpu_winograd_range import SWEEP_CASES
    sms = num_sms()
    conv = []

    def add(test, case, plan, passes=3, f16=False, res=0, cin2=False, out_hilo=False, stats=False, up2=False):
        conv.append(dict(test=test, case=case, passes=passes, f16=f16, res=res, cin2=cin2, out_hilo=out_hilo,
                         stats=stats, up2=up2, **plan))
        assert be.conv_geometry(case[1], case[2])[:3] == conv_geometry(case[1], case[2])

    for c in CONV_CASES:
        B, H, W, Cin, Cout, taps, Cin2, res = c
        for p in (3, 1):
            add("conv_umma", c, conv_plan(B, H, W, Cin, Cout, taps, Cin2, passes=p, sms=sms), passes=p, res=res,
                cin2=Cin2 > 0, out_hilo=True)
    for c in GN_STATS_CONV_CASES:
        B, H, W, Cin, Cout, c2 = c
        for co in (Cout, c2) if c2 else (Cout,):
            add("gn_stats", c, conv_plan(B, H, W, Cin, co, 9, sms=sms), stats=True)
    for c in UPSAMPLE_CONV_CASES:
        B, H, W, Cin, Cout, res = c
        add("upsample", c, conv_plan(B, H, W, Cin, Cout, 4, up2=True, sms=sms), res=2 if res else 0,
            stats=be.conv_geometry(H, W)[3] > 0, up2=True)
    for c in FP16_CONV_CASES:
        B, H, W, Cin, Cout, p = c
        add("fp16", c, conv_plan(B, H, W, Cin, Cout, 9, passes=p, sms=sms), passes=p, f16=True)
    # Winograd position GEMMs: 36 images (transform positions) of tiles/16 x 16 "pixels", one weight plane per position
    wino = []
    wino_cases = [(B, H, W, c1 + c2, Cout) for B, H, W, c1, c2, Cout, _ in CHAIN] + \
        [(B, H, W, c1 + c2, Cout) for B, H, W, c1, c2, Cout in PROD_CHAIN] + SWEEP_CASES
    for c in wino_cases:
        B, H, W, Cin, Cout = c
        mt = be.wino_geometry(B, H, W)[2]
        assert be.conv_geometry(mt // 16, 16)[:3] == conv_geometry(mt // 16, 16)
        plan = conv_plan(36, mt // 16, 16, Cin, Cout, 1, wpi=True, sms=sms)
        per_pos = plan["tiles"] // 36
        # a CTA walks tiles t, t + grid, ...: does any CTA move on to another position (another weight plane)?
        plan["pos_change"] = any(t // per_pos != (t + plan["grid"]) // per_pos for t in range(plan["tiles"] - plan["grid"]))
        wino.append(dict(case=c, **plan))

    wg = []
    for c in WG_CASES:
        B, H, W, Cin, Cout, k = c
        plan = wgrad_plan(B, H, W, Cin, Cout, k * k, sms=sms)
        assert be.wgrad_workspace(B, H, W, Cin, Cout, k * k) == (plan["splits_ws"], plan["workspace"])
        wg.append(dict(case=c, **plan))

    print(f"\n{sms} SMs\n{'test':10} {'case':36} {'p':>2} {'f16':>3} {'BN':>4} {'KB':>4} {'tail':>4} {'tiles':>6} {'/CTA':>4}")
    for r in conv:
        print(f"{r['test']:10} {str(r['case']):36} {r['passes']:2} {int(r['f16']):3} {r['BN']:4} {r['KB']:4} "
              f"{r['kb_tail']:4} {r['tiles']:6} {r['tiles_per_cta']:4}")
    print(f"{'wino':10} {'case':36} {'BN':>4} {'KB':>4} {'chunk':>5} {'tail':>4} {'tiles':>6} {'/CTA':>4} {'pos+':>4}")
    for r in wino:
        print(f"{'wino':10} {str(r['case']):36} {r['BN']:4} {r['KB']:4} {r['kb_per_chunk']:5} {r['kb_tail']:4} "
              f"{r['tiles']:6} {r['tiles_per_cta']:4} {int(r['pos_change']):4}")
    print(f"{'wgrad':10} {'case':36} {'BN':>4} {'splits':>6} {'kb/split':>8} {'last':>4} {'tail':>4} {'items':>6} {'/CTA':>4}")
    for r in wg:
        print(f"{'wgrad':10} {str(r['case']):36} {r['BN']:4} {r['splits']:6} {r['kb_per_split']:8} "
              f"{r['kb_last_split']:4} {r['kb_tail']:4} {r['items']:6} {r['items_per_cta']:4}")

    assert {(r["BN"], r["passes"], r["f16"]) for r in conv} == \
        {(bn, p, f) for bn in (64, 128) for p in (3, 1) for f in (False, True)}
    b128 = [r for r in conv if r["BN"] == 128]
    assert {1, 2, 3} <= {r["res"] for r in b128}
    for feature in ("cin2", "out_hilo", "stats", "up2"):
        assert any(r[feature] for r in b128), feature
    for bn in (64, 128):
        assert any(r["BN"] == bn and r["tiles_per_cta"] > 1 and r["kb_tail"] > 0 for r in conv), bn
        assert any(r["BN"] == bn and r["items_per_cta"] > 1 for r in wg), bn
    assert any(r["KB"] == 1 for r in conv)
    assert any(r["kb_tail"] > 0 for r in wg) and any(r["splits"] > 1 for r in wg)
    assert {r["BN"] for r in wino} == {64, 128}
    assert any(r["tiles_per_cta"] > 1 for r in wino)
    for chunk in (2, 4):
        assert any(r["kb_per_chunk"] == chunk and r["kb_tail"] > 0 for r in wino), chunk
    assert any(r["tiles_per_cta"] > 1 and r["pos_change"] for r in wino)


@pytest.mark.parametrize("B,T,heads,order", [(1, 128, 1, 0), (2, 256, 4, 0), (1, 1024, 2, 1), (1, 100, 2, 1), (1, 4096, 2, 0),
                                              (2, 200, 3, 0)])
def test_attention_tc(be, B, T, heads, order):
    """Warp-specialised wgmma attention (head_dim 64) against the exact result for the planes' value."""
    D = 64
    C = heads * D
    qkv = rnd((B, T, 3 * C), 62, 1.2)
    hi, lo = O.bf16_split(qkv)
    want = O.op_attention_nhwc((hi + lo).double(), heads, bool(order))
    out = torch.full((B, T, C), float("nan"), device=DEV)
    oh = torch.empty((B, T, C), dtype=torch.bfloat16, device=DEV)
    ol = torch.empty_like(oh)
    be.attention_tc(hi.to(torch.bfloat16).to(DEV), lo.to(torch.bfloat16).to(DEV), heads, order,
                    out_f32=out, out_hi=oh, out_lo=ol)
    torch.cuda.synchronize()
    be.check_fault()
    assert not torch.isnan(out).any()
    assert rel_dev(out, want) < 2e-5, rel_dev(out, want)
    h, l = O.bf16_split(out.cpu())
    assert torch.equal(oh.float().cpu(), h) and torch.equal(ol.float().cpu(), l)


# ------------------------------------------------------------------------------------ optimizer / EMA
def test_fused_adam_and_ema_match_torch_over_10_steps():
    """bbdm_adam_multi / bbdm_ema_multi (one launch over all tensors) against torch.optim.Adam and the reference EMA
    expression on the same gradients: 10 steps, odd tensor sizes, weight decay."""
    import torch.nn as nn
    from bbdm_b200.optim import FusedAdam, FusedEMA

    def make():
        torch.manual_seed(3)
        return nn.ParameterList([nn.Parameter(torch.randn(s, device=DEV) * 0.1) for s in
                                 [(128, 64, 3, 3), (513,), (7, 5), (1,), (1024, 333), (64,)]])
    pa, pb = make(), make()
    oa = torch.optim.Adam(pa, lr=2e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-3)
    ob = FusedAdam(pb, lr=2e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-3)
    ema = FusedEMA(0.995)
    holder = nn.Module()
    holder.p = pb
    ema.register(holder)
    shadow_ref = [p.data.clone() for p in pa]
    g = torch.Generator(device=DEV).manual_seed(5)
    for it in range(10):
        for i, (a, b) in enumerate(zip(pa, pb)):
            gr = torch.randn(a.shape, device=DEV, generator=g)
            a.grad, b.grad = gr.clone(), gr.clone()
        oa.step()
        if it % 2:
            ob.step(ema=ema, ema_update=True)                 # EMA fused into the Adam pass
        else:
            ob.step()
            ema.update(holder, with_decay=True)               # separate EMA launch
        shadow_ref = [(1.0 - 0.995) * p.data + 0.995 * s for p, s in zip(pa, shadow_ref)]
    for a, b in zip(pa, pb):
        assert rel_dev(b, a) < 2e-6, rel_dev(b, a)
    for (n, s), r in zip(ema.shadow.items(), shadow_ref):
        assert rel_dev(s, r) < 2e-6, rel_dev(s, r)
    pb[2].grad = None                      # a parameter without gradient: per-parameter step counts are not kept
    with pytest.raises(NotImplementedError):
        ob.step()
    sa, sb = oa.state_dict()["state"], ob.state_dict()["state"]
    for k in sa:      # (a one-element tensor can sit near zero: absolute floor at 1e-6 of the gradient scale)
        for f in ("exp_avg", "exp_avg_sq"):
            assert torch.allclose(sb[k][f], sa[k][f], rtol=1e-5, atol=1e-6), (k, f, rel_dev(sb[k][f], sa[k][f]))


def test_fused_adam_moments_match_torch_adam_per_tensor():
    """exp_avg and exp_avg_sq after the first and second step, per tensor, within fp32 rounding of torch.optim.Adam's
    at the benchmarks' settings (lr 1e-4, default betas, loss-gradient magnitudes).  The hyper-parameters reach the
    kernel as doubles: computed from an fp32-rounded beta2, 1 - 0.999 is 1.3e-5 off, and so was exp_avg_sq (found by
    the training launch shadow on an H100 80GB HBM3; the 10-step test above hides it under its atol)."""
    import torch.nn as nn
    from bbdm_b200.optim import FusedAdam

    def make():
        torch.manual_seed(4)
        return nn.ParameterList([nn.Parameter(0.02 * torch.randn(s, device=DEV)) for s in [(256, 128, 3, 3), (513,), (1,)]])
    pa, pb = make(), make()
    oa, ob = torch.optim.Adam(pa, lr=1e-4), FusedAdam(pb, lr=1e-4)
    g = torch.Generator(device=DEV).manual_seed(6)
    for it in range(2):
        for a, b in zip(pa, pb):
            gr = 1e-4 * torch.randn(a.shape, device=DEV, generator=g)
            a.grad, b.grad = gr.clone(), gr.clone()
        oa.step()
        ob.step()
        sa, sb = oa.state_dict()["state"], ob.state_dict()["state"]
        for k in sa:
            for f in ("exp_avg", "exp_avg_sq"):
                assert rel_dev(sb[k][f], sa[k][f]) < 1e-6, (it, k, f, rel_dev(sb[k][f], sa[k][f]))


def test_ema_update_bit_exact_vs_reference_expression():
    import torch.nn as nn
    from bbdm_b200.optim import FusedEMA
    net = nn.Sequential(nn.Conv2d(16, 32, 3), nn.Linear(77, 13)).to(DEV)
    ema = FusedEMA(0.999)
    ema.register(net)
    ref = {n: p.data.clone() for n, p in net.named_parameters()}
    with torch.no_grad():
        for p in net.parameters():
            p.add_(torch.randn_like(p) * 0.01)
    ema.update(net)
    for n, p in net.named_parameters():
        assert torch.equal(ema.shadow[n], (1.0 - 0.999) * p.data + 0.999 * ref[n])      # runners/base/EMA.py:26


# ------------------------------------------------------------------------------------ sample_to_eval output path
@pytest.mark.parametrize("to_normal", [True, False])
def test_denorm_to_uint8_byte_exact(be, to_normal):
    """bbdm_denorm_to_uint8 against the reference's per-image expression (runners/utils.py:67-74), including values
    outside [-1, 1] and exact rounding boundaries."""
    x = rnd((4, 3, 37, 29), 90, 0.8)
    x[0, 0, 0, :8] = torch.tensor([-1.0, 1.0, 0.0, -1.5, 1.5, 0.00392157, -0.00392157, 0.99607843])
    if not to_normal:
        x = x * 0.5 + 0.5
    out = torch.empty((4, 37, 29, 3), dtype=torch.uint8, device=DEV)
    be.denorm_to_uint8(x.to(DEV), to_normal, out)
    ref = x.clone()
    if to_normal:
        ref = ref.mul_(0.5).add_(0.5).clamp_(0, 1.)
    ref = ref.mul_(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 1).to(torch.uint8)
    assert torch.equal(out.cpu(), ref)


# ------------------------------------------------------------------------------------ cond stage
@pytest.mark.parametrize("n_stages,cout,bias,shape", [
    (2, 3, False, (4, 3, 256, 256)), (1, None, False, (2, 3, 37, 51)), (3, 8, True, (2, 5, 40, 72)),
    (0, 4, True, (1, 3, 9, 7)), (4, 16, False, (1, 16, 64, 96))])
def test_spatial_rescale(be, n_stages, cout, bias, shape):
    """bbdm_spatial_rescale against the reference's op chain (encoders/modules.py:124-131) on stock CUDA kernels
    (fp32, TF32 off): interpolation stages bit-for-bit class (both weights are exactly 0.5), 1x1 map to rounding."""
    x = rnd(shape, 95, 1.2).to(DEV)
    w = None if cout is None else rnd((cout, shape[1]), 96, 0.5).to(DEV)
    b = rnd((cout,), 97, 0.3).to(DEV) if bias else None
    want = x
    for _ in range(n_stages):
        want = F.interpolate(want, scale_factor=0.5, mode="bilinear")
    if w is not None:
        want = torch.einsum("oc,bchw->bohw", w.double(), want.double()) + (0 if b is None else b.double().view(1, -1, 1, 1))
    out = torch.empty((shape[0], shape[1] if w is None else cout, shape[2] >> n_stages, shape[3] >> n_stages), device=DEV)
    be.spatial_rescale(x, n_stages, w, b, out)
    assert out.shape == want.shape
    dev = float((out.double() - want.double()).abs().max() / want.double().abs().max())
    print(f"spatial_rescale n={n_stages} cout={cout}: rel dev {dev:.3e}")
    assert dev <= 1e-6
    if w is None:
        assert (out - want).abs().max() <= 2.4e-7 * float(want.abs().max())


def test_spatial_rescaler_module_native_path():
    """cond.SpatialRescaler under no_grad on CUDA == its own autograd (stock) path."""
    from bbdm_b200 import cabi
    from bbdm_b200.cond import SpatialRescaler
    torch.manual_seed(3)
    m = SpatialRescaler(n_stages=2, in_channels=3, out_channels=3).to(DEV).eval()
    x = rnd((4, 3, 128, 128), 98).to(DEV)
    n0 = cabi.LAUNCHES["n"]
    with torch.no_grad():
        got = m(x)
    assert cabi.LAUNCHES["n"] == n0 + 1
    want = x                                                 # the module's stock chain, channel map in fp64 (cuDNN
    for _ in range(2):                                       # would run the 1x1 conv in TF32 by default)
        want = F.interpolate(want, scale_factor=0.5, mode="bilinear")
    want = F.conv2d(want.double(), m.channel_mapper.weight.detach().double())
    assert got.shape == want.shape == (4, 3, 32, 32)
    assert (got.double() - want).abs().max() <= 1e-6 * float(want.abs().max())


# ------------------------------------------------------------------------------------ SpatialTransformer pieces
@pytest.mark.parametrize("rows,C", [(64, 128), (1000, 256), (257, 1024), (16, 2048)])
def test_layernorm_split(be, rows, C):
    x = rnd((rows, C), 100, 1.3) + 0.2
    g, b = 1 + 0.1 * rnd((C,), 101), 0.1 * rnd((C,), 102)
    want = F.layer_norm(x.double(), (C,), g.double(), b.double(), 1e-5)
    out = torch.empty((rows, C), device=DEV)
    oh = torch.empty((rows, C), dtype=torch.bfloat16, device=DEV)
    ol = torch.empty_like(oh)
    be.layernorm_split(x.to(DEV), g.to(DEV), b.to(DEV), 1e-5, out_f32=out, out_hi=oh, out_lo=ol)
    assert rel_dev(out, want) < 2e-6
    h, l = O.bf16_split(out.cpu())
    assert torch.equal(oh.float().cpu(), h) and torch.equal(ol.float().cpu(), l)


@pytest.mark.parametrize("rows,N", [(64, 512), (333, 1024), (5, 64)])
def test_geglu_split(be, rows, N):
    u = rnd((rows, 2 * N), 110, 1.5)
    a, gate = u.double().chunk(2, dim=-1)
    want = a * F.gelu(gate)
    out = torch.empty((rows, N), device=DEV)
    oh = torch.empty((rows, N), dtype=torch.bfloat16, device=DEV)
    ol = torch.empty_like(oh)
    be.geglu_split(u.to(DEV), out_f32=out, out_hi=oh, out_lo=ol)
    assert rel_dev(out, want) < 2e-6
    h, l = O.bf16_split(out.cpu())
    assert torch.equal(oh.float().cpu(), h) and torch.equal(ol.float().cpu(), l)


@pytest.mark.parametrize("B,Tq,Tkv,heads,D", [(2, 64, 256, 4, 32), (1, 16, 4096, 2, 64), (2, 100, 77, 8, 16), (1, 256, 256, 4, 64)])
def test_attention_cross(be, B, Tq, Tkv, heads, D):
    """Cross-attention core (queries and keys|values from different tensors of different lengths) against the
    reference CrossAttention expression (attention.py:178-191) in fp64."""
    C = heads * D
    q, kv = rnd((B, Tq, C), 120, 1.2), rnd((B, Tkv, 2 * C), 121, 1.2)
    sp = lambda t: t.double().reshape(B, t.shape[1], heads, D).permute(0, 2, 1, 3)
    w = torch.softmax(torch.einsum("bhid,bhjd->bhij", sp(q), sp(kv[..., :C])) * D ** -0.5, dim=-1)
    want = torch.einsum("bhij,bhjd->bhid", w, sp(kv[..., C:])).permute(0, 2, 1, 3).reshape(B, Tq, C)
    planes = lambda t: tuple(z.to(torch.bfloat16).to(DEV) for z in O.bf16_split(t))
    q_hi, q_lo = planes(q)
    kv_hi, kv_lo = planes(kv)
    out = torch.empty((B, Tq, C), device=DEV)
    oh = torch.empty((B, Tq, C), dtype=torch.bfloat16, device=DEV)
    ol = torch.empty_like(oh)
    be.attention_cross(q_hi, q_lo, kv_hi, kv_lo, heads, out_f32=out, out_hi=oh, out_lo=ol)
    assert rel_dev(out, want) < 2e-5, rel_dev(out, want)
    h, l = O.bf16_split(out.cpu())
    assert torch.equal(oh.float().cpu(), h) and torch.equal(ol.float().cpu(), l)


def test_attention_mma_bit_pinned(be):
    """The mma.sync attention entry points reproduce tests/golden/attention_mma.npz bit for bit: the fp32-qkv form
    keeps its own arithmetic (q, k scaled before the split, expf softmax), the split-plane forms theirs."""
    import json
    import numpy as np
    from golden import make_golden_attention_mma as G
    fx = np.load(os.path.join(os.path.dirname(__file__), "golden", "attention_mma.npz"))
    cases = json.loads(str(fx["cases"]))
    assert cases == G.CASES
    for i, case in enumerate(cases):
        got = G.run(be, case)
        assert sorted(got) == sorted(k.split("_", 1)[1] for k in fx.files if k.startswith(f"{i}_")), case
        for k, v in got.items():
            want = torch.from_numpy(fx[f"{i}_{k}"])
            assert torch.equal(v.view(torch.int16) if v.dtype == torch.bfloat16 else v, want), (case, k)


# ------------------------------------------------------------------------------------ stem
@pytest.mark.parametrize("B,H,W,Cin,Cout", [(2, 32, 64, 6, 128), (1, 16, 32, 3, 64), (3, 8, 32, 16, 128), (2, 40, 96, 4, 32)])
def test_conv_stem_equals_conv_direct_and_fuses_gn_partials(be, B, H, W, Cin, Cout):
    """The dedicated stem kernel: bit-identical to the general fp32 kernel (same FMA order), and its fused GroupNorm
    partial sums finalise to the statistics of the output."""
    x, w, b = rnd((B, H, W, Cin), 130), rnd((Cout, Cin, 3, 3), 131, 0.05), rnd((Cout,), 132, 0.1)
    wp = torch.empty((9, Cin, Cout), device=DEV)
    be.pack_weight_f32(w.to(DEV), wp)
    ref = torch.empty((B, H, W, Cout), device=DEV)
    be.conv_direct(x.to(DEV), wp, b.to(DEV), None, ref, Cout, 3, 1)
    out = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    part = torch.full((B * H, Cout, 2), float("nan"), device=DEV)
    be.conv_stem(x.to(DEV), wp, b.to(DEV), out, Cout, stats_partial=part)
    assert torch.equal(out, ref)
    assert rel_dev(out, O.op_conv_nhwc(x.double(), w.double(), b.double())) < 2e-6
    if Cout % 32 == 0 and Cout >= 32:
        mean, rstd = torch.empty((B, 32), device=DEV), torch.empty((B, 32), device=DEV)
        be.gn_finalize_partials(part, H, None, 0, B, H * W, 32, 1e-5, mean, rstd)
        mw, rw = O.op_gn_stats(out.cpu(), 32, 1e-5)
        assert rel_dev(mean, mw) < 1e-5 and rel_dev(rstd, rw) < 1e-5
