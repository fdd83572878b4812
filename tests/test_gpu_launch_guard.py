"""-m gpu: every kernel launch of the shadowed routes run on guarded, NaN-poisoned copies of its operands
(tests/_launch_guard.py) under the fp64 launch shadow: Shadow(Guard(CudaBackend())).  Each case asserts no shadow
failure, no guard finding (no byte outside the output views changed, no output element left unwritten, no fault word
set) and the launch forms it must reach, and prints the shadow's table, the guard's summary, its wall time and its peak
device memory.

The cases are the shadow tests' routes at small batches (every launch is copied twice): sampling forwards of the cfg2
architecture, of LBBDM-f4 with resblock_updown=False and of the padded-, wide- and GEMM-head and 224-channel
SpatialTransformer UNets; the cfg1 sampling loop with the uint8 output path; the VQGAN executor, ragged T included;
training steps (q_sample, forward, L1 loss, backward, two FusedAdam steps) of the ragged 48x48 map, the quarter-size
LBBDM-f4 + SpatialTransformer, the 96-channel stride-2 UNet with the capturable Adam and the wide- and GEMM-head UNets;
the checkpointed step with the trimmed recompute, whose gradients must equal the plain step's bit for bit (under the NaN
fill that proves the recompute wrote everything the backward reads); and the ragged single-kernel shapes no model
reaches.

Not covered: a uint8 output byte the launch leaves unwritten where the right value is 255 (denorm_to_uint8 of a white
pixel) cannot be told from the fill.  CUDA-graph replays are not guarded; the eager runs of the same steps are."""
import contextlib
import os
import time

import numpy as np
import pytest
import torch

from _gemm_heads import GEMM_HEAD_CONFIGS
from _head_dims import HEAD_DIM_CONFIGS
from _launch_guard import Guard
from _launch_shadow import CFG2_FORMS, ST_TRAIN_FORMS, missing_forms
from _launch_shadow_gemm_heads import GemmHeadsShadow
from _recipe import UNET_CONFIGS, VQGAN_CONFIGS, bb_namespace, fill_state_dict, synth_images
from _vq_ragged import VQ_RAGGED_CONFIGS
from _wide_heads import WIDE_HEAD_CONFIGS
from _widths import WIDTH_CONFIGS
from test_gpu_launch_shadow_ends import RS_FORWARD_FORMS, RS_TRAIN_FORMS, SAMPLE_FORMS, VQ_FORMS, _vq_engine, _vq_run
from test_train_shadow_host import HOST_UNET

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
LR = 1e-4


def _guarded():
    """(shadow, guard): the GEMM-head shadow (the ragged and backward softmax references; the base shadow's elsewhere)
    over the guard over the CUDA backend."""
    from bbdm_b200 import cabi
    g = Guard(cabi.CudaBackend())
    return GemmHeadsShadow(g), g


@contextlib.contextmanager
def _run(title, required=()):
    """Times the case, then asserts no shadow failure, no guard finding and the required forms."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    sh, g = _guarded()
    yield sh, g
    torch.cuda.synchronize()
    fails = sh.failures()
    print(f"\n{sh.table(title)}\n{g.summary('  guard')}\n  wall time {time.time() - t0:.1f} s, peak allocated "
          f"{torch.cuda.max_memory_allocated() / 2**30:.2f} GiB on {torch.cuda.get_device_name()}")
    for f in fails[:40]:
        print("  FAIL", f)
    assert not g.findings, g.findings[:10]
    assert not fails, fails[:10]
    assert not missing_forms(sh, required), missing_forms(sh, required)
    assert len(g.launches) == len(sh.launches)
    chains = [c for c in sh.checks if c.what.startswith("chain")]
    assert len(chains) == sum(m == "wino_output" for m, _ in sh.launches)


@contextlib.contextmanager
def _hooks(sh, monkeypatch):
    """The shadow installed through the product's hooks: the training Functions' backend and the bridge's, FusedAdam's
    and the SpatialRescaler's backend factories."""
    from bbdm_b200 import cond, train
    from bbdm_b200.bridge import BridgeOps
    from bbdm_b200.optim import FusedAdam, FusedEMA
    for cls in (BridgeOps, FusedAdam, FusedEMA, cond.SpatialRescaler):
        monkeypatch.setattr(cls, "backend_factory", staticmethod(lambda: sh))
    old = train._BACKEND
    train.set_backend(sh)
    try:
        yield
    finally:
        train.set_backend(old)


def _unet(cfg):
    from bbdm_b200.unet import UNetModel
    net = UNetModel(**cfg).eval()
    net.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1234))
    return net.to(DEV)


def _bridge(cfg, train=True, **kw):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    net = BrownianBridgeModel(bb_namespace(cfg, **kw))
    net = net.train() if train else net.eval()
    net.denoise_fn.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()},
                                                   seed=1234))
    return net.to(DEV)


# ------------------------------------------------------------------------------------------ sampling forwards
ATTN_FORMS = {"gemm": [("softmax_rows_split", (), ("grad",))],
              "st": [("layernorm_split", (), ()), ("geglu_split", (), ()), ("attention_cross", (), ())]}
# name -> (UNet, side, batch, required forms)
FORWARDS = {
    # every F(6,3) form (plain, the wide-input conv1 with the raw planes of its fused skip, the pooled down conv1, the
    # phase-stacked up conv1), the direct tensor-core forms, the stem and attention (test_gpu_launch_shadow.py's cfg2)
    "cfg2 256x256 B=1": (UNET_CONFIGS["cfg2"], 256, 1, CFG2_FORMS + [(m, (), ()) for m in (
        "gather_rows", "linear", "nchw_to_nhwc_cat", "gn_finalize_partials", "prep", "pack_weight_split",
        "pack_weight_f32", "pack_weight_split_taps", "wino_pack_weight")]),
    # the space-to-depth split and the 2x2-tap conv at window origin -1 (test_gpu_launch_shadow_ends.py)
    "lbbdm_f4 resblock_updown=False 64x64 B=2": (dict(UNET_CONFIGS["lbbdm_f4"], resblock_updown=False), 64, 2,
                                                 RS_FORWARD_FORMS),
    # heads of 24 on the padded mma.sync kernel, 136 on the wide one, 336 on the GEMM route (T = 100 keys padded to
    # 128), Cout 96 column slices with LayerNorm, GEGLU and cross-attention
    "mid_hd24": (HEAD_DIM_CONFIGS["mid_hd24"], 32, 2, [("attention_split", (), ())]),
    "mid_hd136_new": (WIDE_HEAD_CONFIGS["mid_hd136_new"], 32, 2, [("attention_split", (), ())]),
    "mid_hd336_new": (GEMM_HEAD_CONFIGS["mid_hd336_new"], 40, 2, ATTN_FORMS["gemm"]),
    "mid_w224_st": (WIDTH_CONFIGS["mid_w224_st"], 32, 2, ATTN_FORMS["st"]),
}


@pytest.mark.parametrize("name", list(FORWARDS))
def test_sampling_forward_guarded(name):
    from bbdm_b200.engine import UNetEngine
    cfg, side, B, required = FORWARDS[name]
    net = _unet(cfg)
    with _run(f"{name} sampling forward", required) as (sh, g):
        eng = UNetEngine(net, backend=sh)
        eng.refresh_weights()
        sh.register_engine(eng)
        x = synth_images((B, net.out_channels, side, side), 11).to(DEV)
        y = None if net.condition_key == "nocond" else synth_images((B, net.in_channels - net.out_channels, side,
                                                                      side), 12).to(DEV)
        out = eng.forward(x, torch.linspace(0, 999, B).round().long().to(DEV), y)
        assert torch.isfinite(out).all()


# ------------------------------------------------------------------------------------------ sampling loop
SAMPLE_REQUIRED = SAMPLE_FORMS[1:] + [("denorm_to_uint8", ("to_normal",), ())]


def test_sampling_loop_guarded(monkeypatch):
    """cfg1's pixel BBDM at 64x64, B = 2, schedule [999, 1, 0] with clip, eagerly; denorm_to_uint8 of the result (the
    shadow holds it byte-exact); one p_sample_dev launch; the SpatialRescaler condition stage."""
    from bbdm_b200.cond import SpatialRescaler
    net = _bridge(UNET_CONFIGS["cfg1"], train=False, sample_step=3)
    assert net.steps.tolist() == [999, 1, 0]
    y = synth_images((2, 3, 64, 64), 2).to(DEV)
    with _run("cfg1 sampling loop (64x64, B=2, steps 999, 1, 0), eager", SAMPLE_REQUIRED) as (sh, g), _hooks(sh, monkeypatch):
        net._bridge.backend()
        eng = net.denoise_fn.engine()
        eng.refresh_weights()
        sh.register_engine(eng)
        net._bridge.use_cuda_graph = False
        torch.manual_seed(5)
        img = net.sample(y, clip_denoised=True)
        assert torch.isfinite(img).all()
        sh.denorm_to_uint8(img, True, torch.empty((2, 64, 64, 3), dtype=torch.uint8, device=DEV))
        # the graphed step's update, launched directly (graph replays are not guarded)
        x_t, eps, noise = (torch.randn((2, 3, 64, 64), generator=torch.Generator().manual_seed(7 + i)).to(DEV)
                           for i in range(3))
        sh.p_sample_dev(x_t, y, eps, noise, net._bridge.coef_table()[0].to(DEV), net.objective, True, False,
                        torch.empty_like(x_t), torch.empty_like(x_t))
        with torch.no_grad():
            torch.manual_seed(6)
            SpatialRescaler(n_stages=2, in_channels=3, out_channels=3, bias=True).to(DEV)(y)
            SpatialRescaler(n_stages=1, in_channels=3).to(DEV)(y)


# ------------------------------------------------------------------------------------------ VQGAN executor
VQ_CASES = {"vq_tc": VQGAN_CONFIGS["vq_tc"], "vq_small": VQGAN_CONFIGS["vq_small"],
            "vq_t196": VQ_RAGGED_CONFIGS["vq_t196"]}
VQ_REQUIRED = dict(VQ_FORMS, vq_t196=[("softmax_rows_split", ("256 columns", "196 valid"), ()),
                                      ("conv_umma", ("taps 1", "split out"), ())])


@pytest.mark.parametrize("name", list(VQ_CASES))
def test_vqgan_executor_guarded(name):
    """The fixture images and latents at the fixture batch: encode with and without quant_conv, decode in both orders."""
    gold = np.load(os.path.join(GOLD, name + ".npz"))
    with _run(f"VQGAN executor {name}", VQ_REQUIRED[name]) as (sh, g):
        _vq_run(_vq_engine(VQ_CASES[name], sh, 4321), torch.from_numpy(gold["x"]).to(DEV),
                torch.from_numpy(gold["lat"]).to(DEV))


# ------------------------------------------------------------------------------------------ training steps
def _train_step(sh, monkeypatch, cfg, side, B, capturable=False, ema=False):
    """q_sample, forward, L1 loss, backward, two FusedAdam steps; ema: the second step updates a FusedEMA shadow and
    FusedEMA.update runs once more on its own."""
    from bbdm_b200.optim import FusedAdam, FusedEMA
    net = _bridge(cfg)
    x, y = synth_images((B, 3, side, side), 1).to(DEV), synth_images((B, 3, side, side), 2).to(DEV)
    nz = torch.randn((B, 3, side, side), generator=torch.Generator().manual_seed(3)).to(DEV)
    t = torch.linspace(0, 999, B).round().long().to(DEV)
    with _hooks(sh, monkeypatch):
        opt = FusedAdam(net.get_parameters(), lr=LR, capturable=capturable)
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
        shadow = None
        if ema:
            shadow = FusedEMA(0.995)
            shadow.register(net)
        opt.step()
        opt.step(ema=shadow, ema_update=ema)
        if ema:
            shadow.update(net)
    assert torch.isfinite(loss)


ADAM2 = [("adam_multi", ("step 1",), ()), ("adam_multi", ("step 2",), ())]
# name -> (UNet, side, batch, capturable Adam, Winograd thresholds (WINO_MIN_C, WINO_MIN_TILES) or None, forms)
TRAININGS = {
    # levels 48 / 24 / 12: the weight gradients' 64-pixel K blocks straddle rows and images, the last one ragged; the
    # EMA shadow updated inside Adam's second step and by ema_multi
    "mid_pixel 48x48 B=3 EMA": (dict(UNET_CONFIGS["mid_pixel"], image_size=48), 48, 3, False, None,
                                [("conv_wgrad", ("taps 9",), ()), ("conv_wgrad", ("taps 1",), ()),
                                 ("pack_weight_split_both", (), ()), ("adam_multi", ("step 1",), ()),
                                 ("adam_multi", ("step 2",), ()), ("ema_multi", (), ())]),
    # test_train_shadow_host.py's UNet and thresholds: the F(4,3) forward and data gradient at 32x32, split_grad's
    # column sums, the GroupNorm, attention and cross-attention backwards
    "quarter lbbdm_f4 + SpatialTransformer 32x32 B=2": (HOST_UNET, 32, 2, False, (64, 128), ST_TRAIN_FORMS),
    "mid_w96_rs capturable Adam": (WIDTH_CONFIGS["mid_w96_rs"], 32, 2, True, None, RS_TRAIN_FORMS),
    # the wide flash backward (heads of 136), at 64 / 128 / 1088 channels (8 heads): mid_hd136's 32-channel ResBlocks
    # have one channel per GroupNorm group, so their bias gradients are zero up to rounding (as for mid_hd336_new below)
    "mid_hd136 (64 channels)": (dict(WIDE_HEAD_CONFIGS["mid_hd136"], model_channels=64, num_heads=8), 32, 2, False,
                                None, [("attention_bwd", (), ())] + ADAM2),
    # heads of 336 on the GEMM route: softmax_rows_split(grad=...) and conv_wgrad over the query pixels.  At 64 / 128 /
    # 704 channels as test_gpu_attention_gemm_heads.py's shadowed step: mid_hd336_new's 32-channel ResBlocks have one
    # channel per GroupNorm group, so their bias gradients are zero up to rounding and no relative bound holds them
    "mid_hd336_new (64 channels)": (dict(GEMM_HEAD_CONFIGS["mid_hd336_new"], model_channels=64,
                                         channel_mult=(1, 2, 11)), 40, 2, False, None,
                                    [("softmax_rows_split", ("grad",), ()), ("conv_wgrad", (), ())] + ADAM2),
}


@pytest.mark.parametrize("name", list(TRAININGS))
def test_training_step_guarded(name, monkeypatch):
    from bbdm_b200 import train
    cfg, side, B, capturable, wino, required = TRAININGS[name]
    if wino:
        monkeypatch.setattr(train, "WINO_MIN_C", wino[0])
        monkeypatch.setattr(train, "WINO_MIN_TILES", wino[1])
    with _run(f"{name} training step", required) as (sh, g):
        _train_step(sh, monkeypatch, cfg, side, B, capturable, ema="EMA" in name)


def test_checkpointed_step_guarded_is_bit_identical_to_the_plain_step(monkeypatch):
    """test_gpu_train_checkpoint.py's smallest case (mid_pixel, 32x32, B = 2) with use_checkpoint and the trimmed
    recompute, guarded and shadowed: every buffer the recompute writes starts as NaN, so gradients bit-identical to the
    unguarded plain step's mean the recompute wrote everything the backward reads."""
    from bbdm_b200 import train
    from test_gpu_train_checkpoint import _inputs, _model
    net = _model(UNET_CONFIGS["mid_pixel"])
    inputs = _inputs(2, 32)

    def step():
        x, y, t, nz = inputs
        net.zero_grad(set_to_none=True)
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
        torch.cuda.synchronize()
        return loss.detach().clone(), {n: p.grad.detach().clone() for n, p in net.denoise_fn.named_parameters()}

    plain = step()
    net.denoise_fn.use_checkpoint = True
    monkeypatch.setattr(train, "RECOMPUTE_TRIM", True)
    with _run("mid_pixel checkpointed step, trimmed recompute (32x32, B=2)") as (sh, g), _hooks(sh, monkeypatch):
        ck = step()
    assert torch.equal(plain[0], ck[0]), (float(plain[0]), float(ck[0]))
    bad = [n for n in plain[1] if not torch.equal(plain[1][n], ck[1][n])]
    assert not bad, bad[:5]


# ------------------------------------------------------------------------------------------ single-kernel edges
def _rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).float().to(DEV)


def _split(x):
    h = x.to(torch.bfloat16)
    return h, (x - h.float()).to(torch.bfloat16)


def _empty(*shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device=DEV)


def _attention_tc(be):          # test_gpu_kernels.py::test_attention_tc (1, 100, 2, 1): T = 100, new order
    hi, lo = _split(_rnd((1, 100, 3 * 128), 62, 1.2))
    o = _empty(1, 100, 128)
    be.attention_tc(hi, lo, 2, 1, out_f32=o, out_hi=torch.empty_like(o, dtype=torch.bfloat16),
                    out_lo=torch.empty_like(o, dtype=torch.bfloat16))


def _conv_direct(be):           # test_gpu_kernels.py::test_conv_direct (2, 9, 11, 35, 3, 3, 1)
    wp = _empty(9, 35, 3)
    be.pack_weight_f32(_rnd((3, 35, 3, 3), 42, 0.05), wp)
    be.conv_direct(_rnd((2, 9, 11, 35), 41), wp, _rnd((3,), 43, 0.1), _rnd((2, 9, 11, 3), 44), _empty(2, 9, 11, 3), 3,
                   3, 1)


def _conv_stem(be):             # test_gpu_kernels.py::test_conv_stem_equals_conv_direct_and_fuses_gn_partials (2, 40, 96, 4, 32)
    wp = _empty(9, 4, 32)
    be.pack_weight_f32(_rnd((32, 4, 3, 3), 131, 0.05), wp)
    be.conv_stem(_rnd((2, 40, 96, 4), 130), wp, _rnd((32,), 132, 0.1), _empty(2, 40, 96, 32), 32,
                 stats_partial=_empty(2 * 40, 32, 2))


def _gn_stats(B, H, W, c1, c2):  # test_gpu_kernels.py::test_gn_stats (2, 4, 4, 32, 0) and (3, 8, 8, 512, 128)
    def run(be):
        from bbdm_b200 import cabi
        be.gn_stats(_rnd((B, H, W, c1), 20) + 0.3, (_rnd((B, H, W, c2), 21, 2.0) - 0.5) if c2 else None, 32, 1e-5,
                    _empty(B, 32), _empty(B, 32), _empty(B * 32 * cabi.GN_MAX_SLICES * 2, dtype=torch.float64))
    return run


def _layernorm(be):             # test_gpu_kernels.py::test_layernorm_split (257, 1024)
    be.layernorm_split(_rnd((257, 1024), 100, 1.3) + 0.2, 1 + 0.1 * _rnd((1024,), 101), 0.1 * _rnd((1024,), 102), 1e-5,
                       out_f32=_empty(257, 1024), out_hi=_empty(257, 1024, dtype=torch.bfloat16),
                       out_lo=_empty(257, 1024, dtype=torch.bfloat16))


def _geglu(be):                 # test_gpu_kernels.py::test_geglu_split (5, 64)
    be.geglu_split(_rnd((5, 128), 110, 1.5), out_f32=_empty(5, 64), out_hi=_empty(5, 64, dtype=torch.bfloat16),
                   out_lo=_empty(5, 64, dtype=torch.bfloat16))


def _split_grad(P, C):          # test_gpu_training.py::test_split_grad (1000, 96) and (64, 200); hi_t / lo_t [C, P]
    def run(be):                # views of rows padded to a multiple of 8, as train._transposed_planes makes them
        ld = -(-P // 8) * 8
        ht, lt = (_empty(C, ld, dtype=torch.bfloat16)[:, :P] for _ in range(2))
        be.split_grad(_rnd((P, C), 1), _empty(P, C, dtype=torch.bfloat16), _empty(P, C, dtype=torch.bfloat16), ht, lt,
                      _empty(C), _empty(-(-P // 64) * C))
    return run


def _attention_cross(be):       # test_gpu_kernels.py::test_attention_cross (2, 100, 77, 8, 16)
    q_hi, q_lo = _split(_rnd((2, 100, 128), 120, 1.2))
    kv_hi, kv_lo = _split(_rnd((2, 77, 256), 121, 1.2))
    be.attention_cross(q_hi, q_lo, kv_hi, kv_lo, 8, out_f32=_empty(2, 100, 128),
                       out_hi=_empty(2, 100, 128, dtype=torch.bfloat16), out_lo=_empty(2, 100, 128, dtype=torch.bfloat16))


def _softmax_ragged(be):        # test_gpu_attention_gemm_heads.py::test_softmax_rows_split_grad (257, 1024, 1000)
    s, g = _rnd((257, 1024), 4, 30.0), _rnd((257, 1024), 7)
    for grad in (None, g):
        be.softmax_rows_split(s, 0.05, _empty(257, 1024, dtype=torch.bfloat16), _empty(257, 1024, dtype=torch.bfloat16),
                              valid_cols=1000, grad=grad)


def _nhwc_to_nchw(be):          # the ragged map of test_gpu_kernels.py::test_conv_direct (2, 9, 11, 35)
    be.nhwc_to_nchw(_rnd((2, 9, 11, 35), 45), _empty(2, 35, 9, 11))


def _pack_dgrad(be):            # a Cout of 96 and a Cin of 35: neither a multiple of 64
    be.pack_weight_split_dgrad(_rnd((96, 35, 3, 3), 46), _empty(9, 35, 96, dtype=torch.bfloat16),
                               _empty(9, 35, 96, dtype=torch.bfloat16))


def _vq_nearest(be):            # test_gpu_vqgan.py::test_vq_nearest (300, 1000, 8)
    be.vq_nearest(_rnd((300, 8), 5), _rnd((1000, 8), 6, 0.7), _empty(300, 8), _empty(300, dtype=torch.int64))


EDGES = {"attention_tc T=100": _attention_tc, "conv_direct 35->3 9x11": _conv_direct,
         "conv_stem 4->32 40x96": _conv_stem, "gn_stats 4x4": _gn_stats(2, 4, 4, 32, 0),
         "gn_stats 8x8 + 128": _gn_stats(3, 8, 8, 512, 128), "layernorm_split 257 rows": _layernorm,
         "geglu_split 5 rows": _geglu, "split_grad P=1000 C=96": _split_grad(1000, 96),
         "split_grad P=64 C=200": _split_grad(64, 200), "attention_cross 100x77 D=16": _attention_cross,
         "softmax_rows_split valid 1000 of 1024": _softmax_ragged, "vq_nearest": _vq_nearest,
         "nhwc_to_nchw 9x11x35": _nhwc_to_nchw, "pack_weight_split_dgrad 96x35": _pack_dgrad}


@pytest.mark.parametrize("name", list(EDGES))
def test_edge_launch_guarded(name):
    with _run(name, [(name.split()[0], (), ())]) as (sh, g):
        EDGES[name](sh)


def required_methods():
    """Every launch kind some case of this file must reach."""
    lists = [f[3] for f in FORWARDS.values()] + [t[5] for t in TRAININGS.values()] + list(VQ_REQUIRED.values()) + \
        [SAMPLE_REQUIRED, [(n.split()[0], (), ()) for n in EDGES]]
    return {r[0] for rs in lists for r in rs}
