"""-m gpu: the VQGAN AttnBlocks at token counts T = H*W that are not multiples of 64, on the sm_90a kernels:

  * bbdm_softmax_rows_split with valid_cols < cols against fp64 (exact +0 past valid_cols), and with all columns valid
    bit for bit what the unpadded row gives;
  * the executor against the fixtures of the unmodified reference VQModel at T = 196, 400, 784
    (tests/golden/make_golden_vqgan_ragged.py);
  * Template-LBBDM-f8's autoencoder at 224x224 and 480x480 and f16's at 224x224 and 320x320 against the fp64 module
    (the oracle's restatement of the reference, evaluated in float64 on the GPU), and the same runs under the launch
    shadow;
  * LatentBrownianBridgeModel with the f8 autoencoder at 224x224: sample(), encode / decode, sample_vqgan() and one
    training step stay on the kernels, without the module-path fallback or its warning.
"""
import os
import time
import warnings

import numpy as np
import pytest
import torch

from _launch_shadow import missing_forms
from _launch_shadow_ragged import RaggedShadow
from _recipe import UNET_CONFIGS, bb_namespace, fill_state_dict, rel_dev, synth_images, vqgan_namespace, \
    vqgan_state_dict
from _vq_ragged import LBBDM_F8, LBBDM_F16, VQ_RAGGED_CONFIGS
from oracle import bbdm_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(__file__), "golden")
# test_gpu_vqgan.py's bound for the aligned fixture models.  Measured up to 6.0e-5 (vq_t784's decoder) on an H100 80GB
# HBM3 (700 W); the split-bf16 emulation reaches 4.4e-5 there and 3.5e-5 against fp64 on the same model at an aligned
# T = 1024, so the deviation is that of the operand split, not of the padded key axis.
BOUND = 1e-4

# (tag, autoencoder, image size): the attention level at image/8 (f8) or image/16 (f16)
SIZES = [("f8 224x224 (T=784)", LBBDM_F8, 224), ("f8 480x480 (T=3600)", LBBDM_F8, 480),
         ("f16 224x224 (T=196)", LBBDM_F16, 224), ("f16 320x320 (T=400)", LBBDM_F16, 320)]


@pytest.fixture(scope="module")
def be():
    from bbdm_b200 import cabi
    b = cabi.CudaBackend()
    yield b
    b.check_fault()


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(shape, generator=g)).float()


def _planes(R, N):
    return (torch.full((R, N), float("nan"), dtype=torch.bfloat16, device=DEV),
            torch.full((R, N), float("nan"), dtype=torch.bfloat16, device=DEV))


@pytest.mark.parametrize("R,N,V", [(196, 256, 196), (400, 448, 400), (7, 832, 784), (5, 3648, 3600), (3, 1088, 1025),
                                   (9, 64, 1), (4, 64, 63), (2, 4096, 4093)])
def test_softmax_valid_cols_against_fp64(be, R, N, V):
    s = rnd((R, N), 4, 30.0)
    s[:, V:] = 1e4 * rnd((R, N - V), 5)            # padding scores far above the row: they must not count
    scale = float(int(512) ** (-0.5))
    hi, lo = _planes(R, N)
    be.softmax_rows_split(s.to(DEV), scale, hi, lo, valid_cols=V)
    got = (hi.double() + lo.double()).cpu()
    want = torch.softmax(s[:, :V].double() * scale, dim=-1)
    assert rel_dev(got[:, :V], want) < 2e-5
    assert not hi[:, V:].view(torch.int16).any() and not lo[:, V:].view(torch.int16).any()      # +0.0, both planes
    be.check_fault()


@pytest.mark.parametrize("R,N,Np", [(64, 64, 128), (100, 256, 320), (7, 1028, 1088), (256, 4096, 4160)])
def test_softmax_all_columns_valid_is_the_unpadded_kernel(be, R, N, Np):
    """valid_cols == cols gives the planes of valid_cols=None bit for bit, and so does a row of N columns padded to Np
    with valid_cols = N in its first N columns (the same per-thread chunks, the same reduction order)."""
    s = rnd((R, N), 6, 30.0)
    scale = float(int(128) ** (-0.5))
    ref = _planes(R, N)
    be.softmax_rows_split(s.to(DEV), scale, *ref)
    full = _planes(R, N)
    be.softmax_rows_split(s.to(DEV), scale, *full, valid_cols=N)
    assert torch.equal(ref[0].view(torch.int16), full[0].view(torch.int16))
    assert torch.equal(ref[1].view(torch.int16), full[1].view(torch.int16))
    sp = torch.cat([s, rnd((R, Np - N), 7, 30.0)], 1)
    pad = _planes(R, Np)
    be.softmax_rows_split(sp.to(DEV), scale, *pad, valid_cols=N)
    assert torch.equal(ref[0].view(torch.int16), pad[0][:, :N].contiguous().view(torch.int16))
    assert torch.equal(ref[1].view(torch.int16), pad[1][:, :N].contiguous().view(torch.int16))
    be.check_fault()


def _load(name):
    return {k: torch.from_numpy(v) for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}


def _container(cfg, seed=4321):
    from bbdm_b200.vqgan import VQModel
    vq = VQModel(**vqgan_namespace(cfg)).eval()
    sd = vqgan_state_dict({k: tuple(v.shape) for k, v in vq.state_dict().items()}, seed)
    vq.load_state_dict(sd, strict=True)
    return vq.to(DEV), sd


@pytest.mark.parametrize("name", list(VQ_RAGGED_CONFIGS))
def test_executor_matches_reference_fixture_at_ragged_t(name):
    g = _load(name)
    vq, _ = _container(VQ_RAGGED_CONFIGS[name])
    eng = vq.engine()
    d_enc = rel_dev(eng.encode(g["x"].to(DEV), quant_conv=False), g["enc"])
    d_qc = rel_dev(eng.encode(g["x"].to(DEV), quant_conv=True), g["enc_qc"])
    dec, idx = eng.decode(g["lat"].to(DEV), return_indices=True)
    assert torch.equal(idx.reshape(-1).cpu(), g["idx"])
    d_dec = rel_dev(dec, g["dec"])
    dec_b, idx_b = eng.decode(g["lat_b"].to(DEV), quant_conv_first=True, return_indices=True)
    same_b = torch.equal(idx_b.reshape(-1).cpu(), g["idx_b"])
    d_dec_b = rel_dev(dec_b, g["dec_b"]) if same_b else None
    rt, idx_rt = eng.decode(eng.encode(g["x"].to(DEV)), return_indices=True)
    clear = g["gap_rt"] > 1e-5
    assert torch.equal(idx_rt.reshape(-1).cpu()[clear], g["idx_rt"][clear])
    d_rt = rel_dev(rt, g["rt"]) if torch.equal(idx_rt.reshape(-1).cpu(), g["idx_rt"]) else None
    eng.be.check_fault()
    print(f"\n[{name}] encoder {d_enc:.2e}  +quant_conv {d_qc:.2e}  decode {d_dec:.2e}  decode(qc first) {d_dec_b}  "
          f"round trip {d_rt}")
    assert d_enc < BOUND and d_qc < BOUND and d_dec < BOUND
    assert (idx_b.reshape(-1).cpu() == g["idx_b"]).float().mean() > 0.99
    assert d_dec_b is None or d_dec_b < BOUND
    assert d_rt is None or d_rt < BOUND
    # replays on the pooled buffers (the zero-padded K and V^T planes included): identical results
    assert torch.equal(eng.decode(g["lat"].to(DEV)), dec)


@pytest.mark.parametrize("tag,cfg,size", SIZES, ids=[s[0] for s in SIZES])
def test_template_autoencoder_at_ragged_size_against_fp64_module(tag, cfg, size):
    vq, sd = _container(cfg, seed=77)
    sd64 = {k: v.to(DEV, torch.float64) for k, v in sd.items()}
    dd = cfg["ddconfig"]
    x = synth_images((1, 3, size, size), 41)
    eng = vq.engine()
    z = eng.encode(x.to(DEV))
    want_z = O.vqgan_encode(sd64, dd, x.to(DEV, torch.float64))
    d_enc = rel_dev(z, want_z)
    lat = want_z.float() + 0.2 * rnd(tuple(want_z.shape), 42).to(DEV)
    dec, idx = eng.decode(lat, return_indices=True)
    want_dec, want_idx = O.vqgan_decode(sd64, dd, lat.double())
    same = idx.reshape(-1) == want_idx
    eng.be.check_fault()
    d_dec = rel_dev(dec, want_dec) if bool(same.all()) else None
    print(f"\n[{tag}] encode rel dev {d_enc:.2e}; code agreement {float(same.float().mean()):.5f}; "
          f"decode rel dev {d_dec}")
    assert d_enc < 1e-4
    assert same.float().mean() > 0.999
    assert d_dec is None or d_dec < 1e-4


@pytest.mark.parametrize("tag,cfg,size", SIZES, ids=[s[0] for s in SIZES])
def test_template_autoencoder_at_ragged_size_every_launch_against_fp64(tag, cfg, size):
    from bbdm_b200 import cabi
    from bbdm_b200.vqgan_engine import VQGANEngine
    t0 = time.time()
    vq, _ = _container(cfg, seed=99)
    sh = RaggedShadow(cabi.CudaBackend())
    eng = VQGANEngine(vq, backend=sh)
    eng.refresh_weights()
    sh.register_engine(eng)
    x = synth_images((1, 3, size, size), 31).to(DEV)
    eng.encode(x, quant_conv=False)
    z = eng.encode(x, quant_conv=True)
    lat = z + 0.2 * torch.randn(z.shape, generator=torch.Generator().manual_seed(32)).to(DEV)
    eng.decode(lat, return_indices=True)
    eng.decode(lat, quant_conv_first=True)
    fails = sh.failures()
    print(f"\n{sh.table(tag)}\n  wall time {time.time() - t0:.1f} s")
    for f in fails[:40]:
        print("  FAIL", f)
    T = (size // (8 if cfg is LBBDM_F8 else 16)) ** 2
    Tp = -(-T // 64) * 64
    forms = [("softmax_rows_split", (f"{Tp} columns", f"{T} valid"), ()), ("s2d_split", (), ()),
             ("split_grad", (), ("colsum", "planes"))]
    assert not missing_forms(sh, forms), missing_forms(sh, forms)
    assert any(c.what == "padding columns +0" for c in sh.checks)
    assert not fails, fails[:10]
    chains = [c for c in sh.checks if c.what.startswith("chain")]
    assert len(chains) == sum(m == "wino_output" for m, _ in sh.launches)


def test_latent_model_at_224_stays_on_the_kernels():
    """LatentBrownianBridgeModel with Template-LBBDM-f8's autoencoder and UNet at 224x224 images (28x28 latents,
    AttnBlocks at T = 784): every end runs on the kernels, the model keeps native_vqgan and warns nothing."""
    import argparse
    from bbdm_b200 import cabi
    from model.BrownianBridge.LatentBrownianBridgeModel import LatentBrownianBridgeModel
    ns = bb_namespace(dict(UNET_CONFIGS["lbbdm_f8"], image_size=28), sample_step=3)
    ns.VQGAN = argparse.Namespace(params=argparse.Namespace(**vqgan_namespace(LBBDM_F8)))
    net = LatentBrownianBridgeModel(ns)
    net.denoise_fn.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()},
                                                   seed=11))
    sd = vqgan_state_dict({k: tuple(v.shape) for k, v in net.vqgan.state_dict().items()}, 77)
    net.vqgan.load_state_dict(sd)
    net = net.cuda().eval()
    x, xc = synth_images((2, 3, 224, 224), 41).cuda(), synth_images((2, 3, 224, 224), 42).cuda()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        n0 = cabi.LAUNCHES["n"]
        z = net.encode(xc, cond=True)
        assert cabi.LAUNCHES["n"] > n0 and z.shape == (2, 4, 28, 28)
        n0 = cabi.LAUNCHES["n"]
        img = net.decode(z, cond=False)
        assert cabi.LAUNCHES["n"] > n0 and img.shape == (2, 3, 224, 224)
        assert torch.isfinite(net.sample_vqgan(x)).all()
        torch.manual_seed(3)
        s = net.sample(xc)
        assert s.shape == (2, 3, 224, 224) and torch.isfinite(s).all()
        net.train()
        loss, _ = net(x, xc)
        loss.backward()
    assert torch.isfinite(loss) and all(p.grad is None for p in net.vqgan.parameters())
    assert net.native_vqgan
    assert not [w for w in caught if "module path" in str(w.message)], [str(w.message) for w in caught]
    net._bridge.backend().check_fault()
