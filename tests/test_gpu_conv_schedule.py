"""-m gpu: a conv tile's results do not depend on how many tiles its CTA runs or where in the CTA's sequence it runs.

The tensor-core conv (bbdm_conv_umma) runs a tile's epilogue while the CTA's next tile is in its main loop, so
the epilogue of a CTA's last tile, of a tile followed by another, and of a CTA's only tile take different paths.
Each case runs one image at a shape where every CTA has at most one tile, then the same image as image 0 of a
batch of 4, where CTAs run several tiles, at the same N tile (tests/_conv_plan.py asserts both plans on this
card).  Image 0's fp32 output, split hi/lo planes and GroupNorm partial rows must be bit-identical, and so must
two launches of the same call.  Every <BN, passes, fp16 operands> instantiation is covered.
"""
import pytest
import torch

from _conv_plan import conv_plan
from bbdm_b200.cabi import RES_DOWN2, RES_NONE, RES_SAME, RES_UP2

pytestmark = pytest.mark.gpu
DEV = "cuda"
BATCH = 4


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


def _rnd(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return scale * torch.randn(shape, generator=g, device=DEV)


def _planes(x, f16):
    dt = torch.float16 if f16 else torch.bfloat16
    hi = x.to(dt)
    return hi, (x - hi.float()).to(dt)


# name: (H, W, Cin, Cout, taps, extras).  H, W: the conv input grid.  The N tile follows from Cout and the tile
# count: Cout 64 runs BN 64 on a 64x128 image (64 tiles; 256 in the batch), Cout 128 runs BN 128 on a 96x128
# image (96 tiles, at least 0.7 x SMs; 384 in the batch).
BN64 = dict(H=64, W=128, Cout=64)
BN128 = dict(H=96, W=128, Cout=128)
CASES = {
    # KB 18: a partial last promotion chunk at passes 3 (chunks of 4) and 1 (chunks of 8)
    "res_same_split_stats": dict(Cin=128, taps=9, res=RES_SAME, split=True, stats=True),
    "res_up2": dict(Cin=64, taps=9, res=RES_UP2),
    "res_down2_split": dict(Cin=64, taps=9, res=RES_DOWN2, split=True),
    "fused_1x1_stats": dict(Cin=64, taps=9, Cin2=128, split=True, stats=True),
    # fewer K blocks than epilogue slices
    "kb1_res_same": dict(Cin=64, taps=1, res=RES_SAME, split=True),
    "kb2_stats": dict(Cin=128, taps=1, stats=True),
    # fused nearest-2x upsample: 4 output phases
    "up2_res_stats": dict(Cin=64, taps=4, up2=True, res=RES_UP2, stats=True),
    # UNet head: 3 of 64 couts stored NCHW
    "nchw_head": dict(Cin=128, taps=9, nchw=3),
}
SHAPES = {
    64: dict(BN64, up2=dict(H=32, W=64)),
    128: dict(BN128, up2=dict(H=48, W=32, Cout=256)),
}


def _case_ids():
    for name, c in CASES.items():
        for bn in (64, 128):
            if c.get("nchw") and bn != 64:
                continue                       # the head's N tile is one 64-wide block
            yield name, bn


def _run(be, B, H, W, Cin, Cout, taps, passes, f16, *, Cin2=0, res=RES_NONE, split=False, stats=False, up2=False,
         nchw=0):
    """One launch at batch B on the first B images of seeded batch-4 tensors; returns image 0's results."""
    act = _planes(_rnd((BATCH, H, W, Cin), 1), f16)
    wtaps = 16 if up2 else taps
    wts = _planes(_rnd((wtaps, Cout, Cin), 2, 0.05), f16)
    bias = _rnd((Cout,), 3, 0.1)
    kw = {}
    if Cin2:
        a2 = _planes(_rnd((BATCH, H, W, Cin2), 4), f16)
        w2 = _planes(_rnd((1, Cout, Cin2), 5, 0.05), f16)
        kw.update(Cin2=Cin2, a2_hi=a2[0][:B], a2_lo=a2[1][:B], w2_hi=w2[0], w2_lo=w2[1], bias2=_rnd((Cout,), 6, 0.1))
    OH, OW = (2 * H, 2 * W) if up2 else (H, W)
    if res != RES_NONE:
        rshape = {RES_SAME: (OH, OW), RES_UP2: (OH // 2, OW // 2), RES_DOWN2: (2 * OH, 2 * OW)}[res]
        kw.update(residual=_rnd((BATCH, *rshape, Cout), 7)[:B], res_mode=res)
    if nchw:
        out = torch.full((B, nchw, OH, OW), float("nan"), device=DEV)
        kw.update(out_nchw_channels=nchw)
    else:
        out = torch.full((B, OH, OW, Cout), float("nan"), device=DEV)
    if split:
        kw.update(out_hi=torch.full((B, OH, OW, Cout), float("nan"), dtype=torch.bfloat16, device=DEV))
        kw.update(out_lo=torch.full_like(kw["out_hi"], float("nan")))
    rows = 0
    if stats:
        rows = be.conv_geometry(H, W)[3] * (4 if up2 else 1)
        assert rows > 0
        kw.update(stats_partial=torch.full((B * rows, Cout, 2), float("nan"), device=DEV))
    be.conv_umma(B=B, H=H, W=W, Cin=Cin, Cout=Cout, taps=taps, a_hi=act[0][:B], a_lo=act[1][:B], w_hi=wts[0],
                 w_lo=wts[1], bias=bias, out=out, passes=passes, upsample2x=up2, operand_f16=f16, **kw)
    torch.cuda.synchronize()
    be.check_fault()
    got = {"out": out[:1]}
    if split:
        got.update(hi=kw["out_hi"][:1], lo=kw["out_lo"][:1])
    if stats:
        got["stats"] = kw["stats_partial"][:rows]
    return {k: v.clone() for k, v in got.items()}


def _assert_bits_equal(a, b, what):
    assert a.keys() == b.keys()
    for k in a:
        assert not torch.isnan(a[k].float()).any(), (what, k)
        ai, bi = (t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16) for t in (a[k], b[k]))
        assert torch.equal(ai, bi), (what, k, int((ai != bi).sum()))


@pytest.mark.parametrize("f16", [False, True], ids=["bf16", "f16"])
@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("name,bn", list(_case_ids()))
def test_conv_tile_result_independent_of_cta_schedule(be, name, bn, passes, f16):
    c = dict(CASES[name])
    shape = dict(SHAPES[bn])
    up2_shape = shape.pop("up2")
    if c.get("up2"):
        shape.update(up2_shape)
    H, W, Cout = shape["H"], shape["W"], shape["Cout"]
    Cin, taps = c.pop("Cin"), c.pop("taps")
    plan_kw = dict(Cin2=c.get("Cin2", 0), up2=c.get("up2", False), passes=passes)
    one = conv_plan(1, H, W, Cin, Cout, taps, **plan_kw)
    many = conv_plan(BATCH, H, W, Cin, Cout, taps, **plan_kw)
    assert one["BN"] == many["BN"] == bn, (one, many)
    assert one["tiles_per_cta"] == 1 and many["tiles_per_cta"] > 1, (one, many)
    runs = [_run(be, B, H, W, Cin, Cout, taps, passes, f16, **c) for B in (1, 1, BATCH, BATCH)]
    _assert_bits_equal(runs[0], runs[1], "repeat, one tile per CTA")
    _assert_bits_equal(runs[2], runs[3], "repeat, several tiles per CTA")
    _assert_bits_equal(runs[0], runs[2], "one vs several tiles per CTA")


# Winograd position GEMMs (weights_per_image: the batch index is the transform position, each with its own
# weights).  The rows of a position are M tiles of 16 x H; a GEMM over fewer rows per position has the leading
# rows of a larger one, so its tiles are the larger one's first tiles of each position.
@pytest.mark.parametrize("f16", [False, True], ids=["bf16", "f16"])
@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("bn,h_one,h_many,Cin", [(64, 8, 32, 192), (128, 24, 64, 192), (128, 24, 64, 576)])
def test_winograd_position_gemm_independent_of_cta_schedule(be, bn, h_one, h_many, Cin, passes, f16):
    P, W, Cout = 36, 16, bn
    one = conv_plan(P, h_one, W, Cin, Cout, 1, passes=passes, wpi=True)
    many = conv_plan(P, h_many, W, Cin, Cout, 1, passes=passes, wpi=True)
    assert one["BN"] == many["BN"] == bn, (one, many)
    assert one["tiles_per_cta"] == 1 and many["tiles_per_cta"] > 1, (one, many)
    assert one["kb_tail"] > 0                    # KB 3 at chunks of 2, KB 9 at chunks of 4
    v = _planes(_rnd((P, h_many, W, Cin), 11), f16)
    u = _planes(_rnd((P, Cout, Cin), 12, 0.05), f16)
    bias = _rnd((Cout,), 13, 0.1)

    def run(h):
        vh, vl = (t[:, :h].contiguous() for t in v)
        m = torch.full((P, h, W, Cout), float("nan"), device=DEV)
        be.conv_umma(B=P, H=h, W=W, Cin=Cin, Cout=Cout, taps=1, a_hi=vh, a_lo=vl, w_hi=u[0], w_lo=u[1], bias=bias,
                     out=m, passes=passes, weights_per_image=True, operand_f16=f16)
        torch.cuda.synchronize()
        be.check_fault()
        return {"out": m[:, :h_one].contiguous()}

    runs = [run(h) for h in (h_one, h_one, h_many, h_many)]
    _assert_bits_equal(runs[0], runs[1], "repeat, one tile per CTA")
    _assert_bits_equal(runs[2], runs[3], "repeat, several tiles per CTA")
    _assert_bits_equal(runs[0], runs[2], "one vs several tiles per CTA")
