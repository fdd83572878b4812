"""-m gpu: attention at head_dim 128 -- every attention kernel against its fp64 result, the training Function and
AttentionBlock against fp64 / the stock graph, and the drop-in model against the reference-generated fixtures
(tests/golden/mid_hd128.npz, mid_st_hd128.npz) and the CPU oracle."""
import os

import numpy as np
import pytest
import torch

from _hd128 import HD128_CONFIGS
from _recipe import UNET_CONFIGS, bb_namespace, fill_state_dict, rel_dev, synth_images
from oracle import bbdm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 128
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL_PSAMPLE = 1e-4


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).float()


def out_buffers(B, T, C):
    out = torch.full((B, T, C), float("nan"), device=DEV)
    oh = torch.empty((B, T, C), dtype=torch.bfloat16, device=DEV)
    return out, oh, torch.empty_like(oh)


def check_split(out, oh, ol):
    h, l = O.bf16_split(out.cpu())
    assert torch.equal(oh.float().cpu(), h) and torch.equal(ol.float().cpu(), l)


# ------------------------------------------------------------------------------------ forward kernels
@pytest.mark.parametrize("B,T,heads,order", [(1, 128, 1, 0), (2, 128, 3, 1), (1, 100, 2, 1), (2, 200, 3, 0),
                                              (1, 1024, 2, 1), (1, 4096, 2, 0), (2, 4096, 1, 1)])
def test_attention_tc_hd128(be, B, T, heads, order):
    """Warp-specialised wgmma attention, two 64-column panels per tile, against the exact result for the planes'
    value; output planes are the split of the fp32 output."""
    C = heads * D
    qkv = rnd((B, T, 3 * C), 62, 1.2)
    hi, lo = O.bf16_split(qkv)
    want = O.op_attention_nhwc((hi + lo).double(), heads, bool(order))
    out, oh, ol = out_buffers(B, T, C)
    be.attention_tc(hi.to(torch.bfloat16).to(DEV), lo.to(torch.bfloat16).to(DEV), heads, order,
                    out_f32=out, out_hi=oh, out_lo=ol)
    torch.cuda.synchronize()
    be.check_fault()
    assert not torch.isnan(out).any()
    assert rel_dev(out, want) < 2e-5, rel_dev(out, want)
    check_split(out, oh, ol)


def test_attention_tc_still_rejects_other_head_dims(be):
    from bbdm_b200 import cabi
    z = torch.zeros((1, 64, 3 * 96), dtype=torch.bfloat16, device=DEV)
    o = torch.empty((1, 64, 96), device=DEV)
    with pytest.raises(cabi.BbdmError, match="head_dim 96"):
        be.attention_tc(z, z, 1, 0, out_f32=o)


@pytest.mark.parametrize("B,T,heads,order", [(2, 256, 2, 0), (1, 1024, 2, 0), (1, 100, 2, 1), (1, 4096, 2, 0),
                                              (1, 200, 3, 1)])
def test_attention_split_hd128(be, B, T, heads, order):
    """mma.sync attention on the pre-split planes (Q fragments staged in shared memory at head_dim 128)."""
    C = heads * D
    qkv = rnd((B, T, 3 * C), 61, 1.2)
    hi, lo = O.bf16_split(qkv)
    want = O.op_attention_nhwc((hi + lo).double(), heads, bool(order))
    out, oh, ol = out_buffers(B, T, C)
    be.attention_split(hi.to(torch.bfloat16).to(DEV), lo.to(torch.bfloat16).to(DEV), heads, order,
                       out_f32=out, out_hi=oh, out_lo=ol)
    assert rel_dev(out, want) < 2e-5, rel_dev(out, want)
    assert rel_dev(out, O.op_attention_nhwc(qkv.double(), heads, bool(order))) < 5e-5
    check_split(out, oh, ol)


@pytest.mark.parametrize("B,T,heads,order", [(2, 256, 2, 0), (1, 1024, 1, 0), (1, 100, 2, 1), (2, 4096, 1, 0)])
def test_attention_fp32_qkv_hd128(be, B, T, heads, order):
    """The fp32-qkv kernel (dynamic shared memory at head_dim 128)."""
    C = heads * D
    qkv = rnd((B, T, 3 * C), 60, 1.2)
    want = O.op_attention_nhwc(qkv.double(), heads, bool(order))
    out, oh, ol = out_buffers(B, T, C)
    be.attention(qkv.to(DEV), heads, order, out_f32=out, out_hi=oh, out_lo=ol)
    assert rel_dev(out, want) < 2e-5, rel_dev(out, want)
    check_split(out, oh, ol)


@pytest.mark.parametrize("B,Tq,Tkv,heads", [(2, 64, 256, 2), (1, 16, 4096, 2), (2, 100, 77, 2), (1, 256, 256, 1),
                                             (1, 4096, 77, 2)])
def test_attention_cross_hd128(be, B, Tq, Tkv, heads):
    C = heads * D
    q, kv = rnd((B, Tq, C), 120, 1.2), rnd((B, Tkv, 2 * C), 121, 1.2)
    sp = lambda t: t.double().reshape(B, t.shape[1], heads, D).permute(0, 2, 1, 3)
    w = torch.softmax(torch.einsum("bhid,bhjd->bhij", sp(q), sp(kv[..., :C])) * D ** -0.5, dim=-1)
    want = torch.einsum("bhij,bhjd->bhid", w, sp(kv[..., C:])).permute(0, 2, 1, 3).reshape(B, Tq, C)
    planes = lambda t: tuple(z.to(torch.bfloat16).to(DEV) for z in O.bf16_split(t))
    q_hi, q_lo = planes(q)
    kv_hi, kv_lo = planes(kv)
    out, oh, ol = out_buffers(B, Tq, C)
    be.attention_cross(q_hi, q_lo, kv_hi, kv_lo, heads, out_f32=out, out_hi=oh, out_lo=ol)
    assert rel_dev(out, want) < 2e-5, rel_dev(out, want)
    check_split(out, oh, ol)


# ------------------------------------------------------------------------------------ training
@pytest.mark.parametrize("B,T,heads,order", [(2, 64, 2, 0), (1, 64, 1, 1), (1, 100, 2, 1), (2, 100, 1, 0),
                                              (1, 1024, 2, 0), (1, 1024, 1, 1)])
def test_attention_bwd_hd128(be, B, T, heads, order):
    Cc = heads * D
    qkv = rnd((B, T, 3 * Cc), 30, 1.5)
    dout = rnd((B, T, Cc), 31, 0.3)
    qd = qkv.double().requires_grad_(True)
    od = O.op_attention_nhwc(qd, heads, bool(order))
    od.backward(dout.double())
    dqkv = torch.full((B, T, 3 * Cc), float("nan"), device=DEV)
    lse, delta = torch.empty(B * heads * T, device=DEV), torch.empty(B * heads * T, device=DEV)
    be.attention_bwd(qkv.to(DEV), od.detach().float().to(DEV), dout.to(DEV), heads, order, dqkv, lse, delta)
    torch.cuda.synchronize()
    assert not torch.isnan(dqkv).any()
    assert rel_dev(dqkv, qd.grad) < 2e-5, rel_dev(dqkv, qd.grad)


@pytest.mark.parametrize("B,H,W,heads,order", [(2, 8, 8, 2, 0), (1, 16, 16, 1, 1), (1, 10, 10, 2, 1)])
def test_attention_core_function_hd128(B, H, W, heads, order):
    """AttentionCoreFn at head_dim 128: wgmma forward, flash backward, against the fp64 graph."""
    from bbdm_b200.train import AttentionCoreFn
    C = heads * D
    qkv = (rnd((B, 3 * C, H, W), 32, 1.2).to(DEV).contiguous(memory_format=torch.channels_last)).requires_grad_(True)
    gy = rnd((B, C, H, W), 33, 0.3).to(DEV)
    y = AttentionCoreFn.apply(qkv, heads, order)
    y.backward(gy)
    qd = qkv.detach().double().cpu().requires_grad_(True)
    od = O.op_attention_nhwc(qd.permute(0, 2, 3, 1).reshape(B, H * W, 3 * C), heads, bool(order))
    od.backward(gy.double().cpu().permute(0, 2, 3, 1).reshape(B, H * W, C))
    assert rel_dev(y.permute(0, 2, 3, 1).reshape(B, H * W, C), od) < 3e-5
    assert rel_dev(qkv.grad, qd.grad) < 5e-5, rel_dev(qkv.grad, qd.grad)


def test_attention_block_hd128_training_matches_torch_graph():
    """AttentionBlock(256, num_heads=2) in training: native GN+qkv, attention core, proj vs the stock-PyTorch path.
    The stock arm runs in true fp32 (cuDNN's TF32 default off); both arms are also measured against the stock graph
    on the CPU (fp32, no TF32) for the log."""
    import copy
    import bbdm_b200.unet as U
    blk = U.AttentionBlock(256, num_heads=2).to(DEV)
    with torch.no_grad():
        for p_ in blk.parameters():
            p_.copy_(rnd(tuple(p_.shape), 40 + p_.numel() % 7, 0.05).to(DEV))
        blk.norm.weight.add_(1.0)
    x = rnd((2, 256, 16, 16), 41).to(DEV)
    gy = rnd((2, 256, 16, 16), 42, 0.2).to(DEV)

    def run(m, xx, g):
        m.zero_grad(set_to_none=True)
        xi = xx.clone().requires_grad_(True)
        y = m(xi)
        y.backward(g)
        return y.detach(), xi.grad, {n: p_.grad.clone() for n, p_ in m.named_parameters()}

    res = {}
    try:
        U.NATIVE_TRAIN_CONV = True
        res["native"] = run(blk, x, gy)
        U.NATIVE_TRAIN_CONV = False
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            res["stock"] = run(blk, x, gy)
    finally:
        U.NATIVE_TRAIN_CONV = True
    res["cpu"] = run(copy.deepcopy(blk).cpu(), x.cpu(), gy.cpu())
    for arm in ("native", "stock"):
        worst = max(rel_dev(res[arm][2][n], res["cpu"][2][n]) for n in res["cpu"][2])
        print(f"\n[AttentionBlock 256/2 heads] {arm} vs CPU stock: out {rel_dev(res[arm][0], res['cpu'][0]):.2e} "
              f"dx {rel_dev(res[arm][1], res['cpu'][1]):.2e} worst dparam {worst:.2e}")
    assert rel_dev(res["native"][0], res["stock"][0]) < 3e-5
    assert rel_dev(res["native"][1], res["stock"][1]) < 1e-4
    for n in res["stock"][2]:
        assert rel_dev(res["native"][2][n], res["stock"][2][n]) < 1e-4, n


# ------------------------------------------------------------------------------------ drop-in model
def build(u, **kw):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    net = BrownianBridgeModel(bb_namespace(u, **kw)).eval()
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    sd = fill_state_dict(shapes, seed=1234)
    net.denoise_fn.load_state_dict(sd)
    return net.to("cuda"), sd


@pytest.mark.parametrize("tag", ["mid_hd128", "mid_st_hd128"])
def test_hd128_model_matches_reference_fixture(tag):
    g = {k: torch.from_numpy(v) if v.ndim else v for k, v in np.load(os.path.join(GOLD, tag + ".npz")).items()}
    net, _ = build(HD128_CONFIGS[tag])
    c = lambda z: z.cuda()
    x, y, t = c(g["x"]), c(g["y"]), c(g["t"])
    with torch.no_grad():
        out = net.denoise_fn(x, timesteps=t, context=y)
    d_unet = rel_dev(out, g["unet_out"])
    xt, obj = net.q_sample(x, y, t, c(g["q_noise"]))
    assert torch.equal(xt.cpu(), g["q_xt"]) and torch.equal(obj.cpu(), g["q_obj"])      # bit-exact
    devs = {}
    for i in g["ps_ids"].tolist():
        for clip, key in ((False, f"ps{i}_out"), (True, f"ps{i}_out_clip")):
            o, _ = net.p_sample(c(g[f"ps{i}_xt"]), y, y, i, clip_denoised=clip, noise=c(g[f"ps{i}_noise"]))
            devs[(i, clip)] = rel_dev(o, g[key])
    net._bridge.backend().check_fault()
    print(f"\n[{tag}] unet rel dev {d_unet:.3e}; p_sample rel dev {devs}")
    assert d_unet < TOL_PSAMPLE
    assert max(devs.values()) < TOL_PSAMPLE
    if "loop8_out" in g:
        net8, _ = build(HD128_CONFIGS[tag], sample_step=8)
        seq = iter(c(g["loop8_noise"]))
        net8._bridge.noise_source = lambda like: next(seq)
        img = net8.sample(y, clip_denoised=True)
        d_loop = rel_dev(img, g["loop8_out"])
        print(f"[{tag}] 8-step loop rel dev {d_loop:.3e}")
        assert d_loop < 2e-4


def test_half_resolution_pixel_model_hd128_against_oracle():
    """128x128 pixel BBDM at full channel widths with heads sized by num_heads (8 heads, num_head_channels=-1): the
    middle block attends over T=1024 at 1024 channels = head_dim 128.  One p_sample against the CPU oracle."""
    u = dict(UNET_CONFIGS["cfg1"], image_size=128, num_heads=8, num_head_channels=-1)
    net, sd = build(u)
    xt, y = synth_images((1, 3, 128, 128), 31), synth_images((1, 3, 128, 128), 32)
    nz = torch.randn(1, 3, 128, 128, generator=torch.Generator().manual_seed(33))
    bufs, steps = O.make_schedule()
    threads = torch.get_num_threads()
    torch.set_num_threads(min(64, os.cpu_count() or 8))
    try:
        want, _ = O.p_sample(sd, O.unet_cfg(**u), bufs, steps, 150, xt, y, y, nz, prefix="")
    finally:
        torch.set_num_threads(threads)          # later CPU tests keep the process's thread count
    got, _ = net.p_sample(xt.cuda(), y.cuda(), y.cuda(), 150, noise=nz.cuda())
    net._bridge.backend().check_fault()
    d = rel_dev(got, want)
    print(f"\n[pixel 128x128, head_dim 128] p_sample rel dev vs oracle {d:.3e}")
    assert d < TOL_PSAMPLE
