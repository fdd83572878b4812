"""-m gpu: every kernel launch of the routes the UNet shadow tests do not take, against an fp64 recomputation of that
launch (tests/_launch_shadow.py):

  * the VQGAN executor, encode with and without quant_conv and decode in both orders: the fixture models vq_tc and
    vq_small, and Template-LBBDM-f4's autoencoder at 256x256 and f8's at 512x512 (one image each), whose AttnBlocks run
    S = Q K^T with Cout = T = 4096 and O = P V over K = T = 4096 softmax probabilities;
  * UNets with resblock_updown=False (the reference's default), whose Downsample runs the space-to-depth split and the
    2x2-tap conv at window origin -1: the LBBDM-f4 UNet at 64x64, B = 32 (bench cfg3's shape) and mid_resample, and a
    training step of mid_resample with FusedAdam(capturable=True);
  * a training step of mid_pixel at 48x48, B = 3, whose weight-gradient K blocks straddle rows and images;
  * the pixel sampling loop (cfg1 architecture, 64x64, B = 4, 3 steps ending at t = 0) eagerly with and without clip,
    and on the CUDA graph, whose warm-up step runs p_sample_dev; and the SpatialRescaler condition stage.
"""
import contextlib
import os
import time

import numpy as np
import pytest
import torch

from _launch_shadow import Shadow, missing_forms
from _recipe import (UNET_CONFIGS, VQGAN_CONFIGS, bb_namespace, fill_state_dict, synth_images, vqgan_namespace,
                     vqgan_state_dict)

pytestmark = pytest.mark.gpu
DEV = "cuda"
LR = 1e-4

# Template-LBBDM-f4 / f8 autoencoders (test_gpu_vqgan.py), at the image sizes the latent models feed them
VQ_FULL = {
    "f4 256x256": (256, dict(embed_dim=3, n_embed=8192,
                             ddconfig=dict(double_z=False, z_channels=3, resolution=256, in_channels=3, out_ch=3, ch=128,
                                           ch_mult=(1, 2, 4), num_res_blocks=2, attn_resolutions=[], dropout=0.0))),
    "f8 512x512": (512, dict(embed_dim=4, n_embed=16384,
                             ddconfig=dict(double_z=False, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128,
                                           ch_mult=(1, 2, 2, 4), num_res_blocks=2, attn_resolutions=[32],
                                           dropout=0.0))),
}
VQ_FORMS = {
    # fixture models at 32x32, batch 2: the tensor-core Downsample (origin 0: the VQGAN pads (0, 1)), the GEMM-composed
    # AttnBlock, the code search; and the CUDA-core stride-2 conv and the flash AttnBlock on fp32 qkv
    "vq_tc": [("s2d_split", (), ()), ("conv_umma", ("taps 4",), ("origin", "upsample2x")),
              ("softmax_rows_split", (), ()), ("vq_nearest", (), ()), ("split_grad", (), ("colsum",))],
    "vq_small": [("conv_direct_pad", (), ()), ("attention", (), ()), ("vq_nearest", (), ())],
    "f4 256x256": [("s2d_split", (), ()), ("softmax_rows_split", ("4096 columns",), ()),
                   ("conv_umma", ("taps 1", "long K"), ()), ("wino_output", (), ())],
    "f8 512x512": [("s2d_split", (), ()), ("softmax_rows_split", ("4096 columns",), ()),
                   ("conv_umma", ("taps 1", "long K"), ()), ("wino_output", (), ())],
}
RS_UNET = dict(UNET_CONFIGS["mid_pixel"], resblock_updown=False)          # test_gpu_conv_resample.py's mid_resample
RS_FORWARD_FORMS = [("s2d_split", (), ()), ("conv_umma", ("taps 4", "origin -1", "stats"), ())]
RS_TRAIN_FORMS = [("s2d_split", (), ()), ("conv_umma", ("taps 4", "origin -1"), ()),
                  ("conv_umma", ("taps 4",), ("origin", "upsample2x")),          # the stride-2 data gradient
                  ("conv_wgrad", ("taps 4", "origin -1"), ()), ("adam_multi_dev", ("step 1",), ()),
                  ("adam_multi_dev", ("step 2",), ())]
SAMPLE_FORMS = [("p_sample", ("not last",), ("clip",)), ("p_sample", ("not last", "clip"), ()),
                ("p_sample", ("last",), ("not last",)), ("p_sample_dev", ("not last",), ()),
                ("spatial_rescale", ("2 stages", "1x1 map"), ()), ("spatial_rescale", ("1 stages",), ("1x1 map",))]


def _report(sh, title, t0):
    fails = sh.failures()
    print(f"\n{sh.table(title)}\n  wall time {time.time() - t0:.1f} s")
    for f in fails[:40]:
        print("  FAIL", f)
    return fails


def _assert_clean(sh, required):
    fails = sh.failures()
    assert not missing_forms(sh, required), missing_forms(sh, required)
    assert not fails, fails[:10]
    chains = [c for c in sh.checks if c.what.startswith("chain")]
    assert len(chains) == sum(m == "wino_output" for m, _ in sh.launches)


@contextlib.contextmanager
def _shadowed(monkeypatch):
    """The shadow installed through the product's hooks: the training Functions' backend, the bridge's, FusedAdam's
    and the SpatialRescaler's backend factories."""
    from bbdm_b200 import cabi, cond, train
    from bbdm_b200.bridge import BridgeOps
    from bbdm_b200.optim import FusedAdam
    sh = Shadow(cabi.CudaBackend())
    for cls in (BridgeOps, FusedAdam, cond.SpatialRescaler):
        monkeypatch.setattr(cls, "backend_factory", staticmethod(lambda: sh))
    old = train._BACKEND
    train.set_backend(sh)
    try:
        yield sh
    finally:
        train.set_backend(old)


# ------------------------------------------------------------------------------------------ VQGAN executor
def _vq_engine(cfg, sh, seed):
    from bbdm_b200.vqgan import VQModel
    from bbdm_b200.vqgan_engine import VQGANEngine
    vq = VQModel(**vqgan_namespace(cfg)).eval()
    vq.load_state_dict(vqgan_state_dict({k: tuple(v.shape) for k, v in vq.state_dict().items()}, seed), strict=True)
    eng = VQGANEngine(vq.to(DEV), backend=sh)
    eng.refresh_weights()
    sh.register_engine(eng)
    return eng


def _vq_run(eng, x, lat=None):
    """encode without and with quant_conv, decode in both orders (lat: the encoding plus 0.2 N(0, 1) by default)."""
    eng.encode(x, quant_conv=False)
    z = eng.encode(x, quant_conv=True)
    if lat is None:
        lat = z + 0.2 * torch.randn(z.shape, generator=torch.Generator().manual_seed(32)).to(DEV)
    eng.decode(lat, return_indices=True)
    eng.decode(lat, quant_conv_first=True)


@pytest.mark.parametrize("name", ["vq_tc", "vq_small", "f4 256x256", "f8 512x512"])
def test_vqgan_executor_every_launch_against_fp64(name):
    from bbdm_b200 import cabi
    t0 = time.time()
    sh = Shadow(cabi.CudaBackend())
    if name in VQGAN_CONFIGS:        # the fixture's images and latents, at the fixture batch
        g = np.load(os.path.join(os.path.dirname(__file__), "golden", name + ".npz"))
        _vq_run(_vq_engine(VQGAN_CONFIGS[name], sh, 4321), torch.from_numpy(g["x"]).to(DEV),
                torch.from_numpy(g["lat"]).to(DEV))
    else:
        size, cfg = VQ_FULL[name]
        _vq_run(_vq_engine(cfg, sh, 99), synth_images((1, 3, size, size), 31).to(DEV))
    _report(sh, f"VQGAN executor {name}", t0)
    _assert_clean(sh, VQ_FORMS[name])
    if name in VQ_FULL:
        assert sum(m == "wino_output" for m, _ in sh.launches) > 0


# ------------------------------------------------------------------------------------------ resblock_updown=False
@pytest.mark.parametrize("name,unet,side,B", [("lbbdm_f4 resblock_updown=False", dict(UNET_CONFIGS["lbbdm_f4"],
                                                                                     resblock_updown=False), 64, 32),
                                              ("mid_resample", RS_UNET, 32, 2)])
def test_stride2_downsample_forward_every_launch_against_fp64(name, unet, side, B):
    from bbdm_b200 import cabi
    from bbdm_b200.engine import UNetEngine
    from bbdm_b200.unet import UNetModel
    t0 = time.time()
    net = UNetModel(**unet).eval()
    net.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1234))
    net = net.to(DEV)
    sh = Shadow(cabi.CudaBackend())
    eng = UNetEngine(net, backend=sh)
    eng.refresh_weights()
    sh.register_engine(eng)
    x = synth_images((B, net.out_channels, side, side), 11).to(DEV)
    y = None if net.condition_key == "nocond" else synth_images((B, net.in_channels - net.out_channels, side, side),
                                                               12).to(DEV)
    out = eng.forward(x, torch.linspace(0, 999, B).round().long().to(DEV), y)
    assert torch.isfinite(out).all()
    _report(sh, f"{name} ({side}x{side}, B={B})", t0)
    _assert_clean(sh, RS_FORWARD_FORMS)
    assert any(c.what == "s2d taps vs module weight" for c in sh.checks)


def _train_step(monkeypatch, unet, side, B, capturable):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    from bbdm_b200.optim import FusedAdam
    net = BrownianBridgeModel(bb_namespace(unet)).train()
    net.denoise_fn.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()},
                                                   seed=1234))
    net = net.to(DEV)
    x, y = synth_images((B, 3, side, side), 1).to(DEV), synth_images((B, 3, side, side), 2).to(DEV)
    nz = torch.randn((B, 3, side, side), generator=torch.Generator().manual_seed(3)).to(DEV)
    t = torch.linspace(0, 999, B).round().long().to(DEV)
    with _shadowed(monkeypatch) as sh:
        opt = FusedAdam(net.get_parameters(), lr=LR, capturable=capturable)
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
        opt.step()
        opt.step()
    assert torch.isfinite(loss)
    return sh


def test_stride2_downsample_training_step_with_capturable_adam(monkeypatch):
    t0 = time.time()
    sh = _train_step(monkeypatch, RS_UNET, 32, 2, capturable=True)
    _report(sh, "mid_resample training step, FusedAdam(capturable=True) (32x32, B=2)", t0)
    _assert_clean(sh, RS_TRAIN_FORMS)


def test_ragged_map_training_step(monkeypatch):
    """mid_pixel at 48x48, B = 3: levels 48 / 24 / 12, so the 64-pixel K blocks of the weight gradients wrap across
    rows and images and the last one is ragged."""
    t0 = time.time()
    sh = _train_step(monkeypatch, dict(UNET_CONFIGS["mid_pixel"], image_size=48), 48, 3, capturable=False)
    _report(sh, "mid_pixel_48 training step (48x48, B=3)", t0)
    _assert_clean(sh, [("conv_wgrad", ("taps 9",), ()), ("conv_wgrad", ("taps 1",), ()),
                       ("adam_multi", ("step 2",), ())])


# ------------------------------------------------------------------------------------------ sampling loop
def test_sampling_loop_eager_and_graphed(monkeypatch):
    """cfg1's pixel BBDM at 64x64, B = 4, schedule [999, 1, 0]: eager loops with and without clip (p_sample, the last
    step included), then the graphed loop, whose warm-up step runs p_sample_dev under the shadow while the capture
    passes through it; and the SpatialRescaler condition stage of the latent models on the same images."""
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    from bbdm_b200.cond import SpatialRescaler
    t0 = time.time()
    net = BrownianBridgeModel(bb_namespace(UNET_CONFIGS["cfg1"], sample_step=3)).eval()
    assert net.steps.tolist() == [999, 1, 0]
    net.denoise_fn.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()},
                                                   seed=1234))
    net = net.to(DEV)
    y = synth_images((4, 3, 64, 64), 2).to(DEV)
    with _shadowed(monkeypatch) as sh:
        net._bridge.backend()
        eng = net.denoise_fn.engine()
        eng.refresh_weights()
        sh.register_engine(eng)
        net._bridge.use_cuda_graph = False
        for clip in (False, True):
            torch.manual_seed(5)
            assert torch.isfinite(net.sample(y, clip_denoised=clip)).all()
        net._bridge.use_cuda_graph = True
        torch.manual_seed(5)
        img = net.sample(y, clip_denoised=True)
        assert torch.isfinite(img).all()
        with torch.no_grad():
            torch.manual_seed(6)
            SpatialRescaler(n_stages=2, in_channels=3, out_channels=3, bias=True).to(DEV)(y)
            SpatialRescaler(n_stages=1, in_channels=3).to(DEV)(y)
    _report(sh, "cfg1 sampling loop (64x64, B=4, steps 999, 1, 0), eager and graphed", t0)
    assert sh.captured and "p_sample_dev" in sh.captured
    _assert_clean(sh, SAMPLE_FORMS)
