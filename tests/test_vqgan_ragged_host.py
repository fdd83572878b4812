"""VQGAN AttnBlocks at token counts T = H*W that are not multiples of 64, on CPU: the oracle pinned to fixtures generated
by the unmodified reference VQModel (tests/golden/make_golden_vqgan_ragged.py), and the executor's padded-key attention
(K planes [Tp][C] and V^T planes [C][Tp] zero past T, the softmax over the first T of Tp columns) through the
emulation backend whose row softmax honours valid_cols (tests/_emu_backend_ragged.py) and under the launch shadow."""
import os

import numpy as np
import pytest
import torch

from _emu_backend_ragged import EmuBackendRagged
from _launch_shadow import missing_forms
from _launch_shadow_ragged import RaggedShadow
from _recipe import VQGAN_CONFIGS, rel_dev, synth_images, vqgan_namespace, vqgan_state_dict
from _vq_ragged import VQ_RAGGED_CONFIGS
from oracle import bbdm_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")
EMU_BOUNDS = {"chain6": 2.5e-5}          # test_launch_shadow_coverage_host.py


def load(name):
    return {k: torch.from_numpy(v) for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}


def container(cfg):
    from bbdm_b200.vqgan import VQModel
    vq = VQModel(**vqgan_namespace(cfg)).eval()
    sd = vqgan_state_dict({k: tuple(v.shape) for k, v in vq.state_dict().items()})
    vq.load_state_dict(sd, strict=True)
    return vq, sd


class SoftmaxSpy(EmuBackendRagged):
    """Records the keyword arguments of every row-softmax call as the executor passed them."""

    def __init__(self):
        super().__init__()
        self.softmax_kwargs = []

    def softmax_rows_split(self, *args, **kwargs):
        self.softmax_kwargs.append(dict(kwargs))
        return super().softmax_rows_split(*args, **kwargs)


@pytest.mark.parametrize("name", list(VQ_RAGGED_CONFIGS))
def test_oracle_pinned_to_reference_at_ragged_token_counts(name):
    g = load(name)
    _, sd = container(VQ_RAGGED_CONFIGS[name])
    dd = VQ_RAGGED_CONFIGS[name]["ddconfig"]
    assert rel_dev(O.vqgan_encode(sd, dd, g["x"], quant_conv=False), g["enc"]) < 1e-5
    assert rel_dev(O.vqgan_encode(sd, dd, g["x"], quant_conv=True), g["enc_qc"]) < 1e-5
    zq, idx = O.vqgan_quantize(sd, g["lat"])
    assert torch.equal(idx, g["idx"]) and torch.equal(zq, g["quant"])
    dec, _ = O.vqgan_decode(sd, dd, g["lat"])
    assert rel_dev(dec, g["dec"]) < 1e-5
    dec_b, idx_b = O.vqgan_decode(sd, dd, g["lat_b"], quant_conv_first=True)
    assert torch.equal(idx_b, g["idx_b"]) and rel_dev(dec_b, g["dec_b"]) < 1e-5
    rt, idx_rt = O.vqgan_decode(sd, dd, O.vqgan_encode(sd, dd, g["x"]))
    assert torch.equal(idx_rt, g["idx_rt"]) and rel_dev(rt, g["rt"]) < 1e-5


@pytest.mark.parametrize("name", list(VQ_RAGGED_CONFIGS))
def test_engine_host_logic_at_ragged_token_counts(name):
    from bbdm_b200.vqgan_engine import VQGANEngine
    g = load(name)
    vq, _ = container(VQ_RAGGED_CONFIGS[name])
    T = (VQ_RAGGED_CONFIGS[name]["ddconfig"]["resolution"] // 2) ** 2
    be = SoftmaxSpy()
    eng = VQGANEngine(vq, backend=be)
    assert rel_dev(eng.encode(g["x"], quant_conv=False), g["enc"]) < 1e-4
    assert rel_dev(eng.encode(g["x"], quant_conv=True), g["enc_qc"]) < 1e-4
    dec, idx = eng.decode(g["lat"], return_indices=True)
    assert torch.equal(idx.reshape(-1), g["idx"]) and rel_dev(dec, g["dec"]) < 1e-4
    dec_b, idx_b = eng.decode(g["lat_b"], quant_conv_first=True, return_indices=True)
    ok = g["idx_b"] == idx_b.reshape(-1)
    assert ok.float().mean() > 0.99            # quant_conv's rounding may flip a near-tie
    if bool(ok.all()):
        assert rel_dev(dec_b, g["dec_b"]) < 1e-4
    rt, idx_rt = eng.decode(eng.encode(g["x"]), return_indices=True)
    if torch.equal(idx_rt.reshape(-1), g["idx_rt"]):
        assert rel_dev(rt, g["rt"]) < 1e-4
    # every AttnBlock (C = 128) took the padded-key path: per image one softmax over the first T columns
    assert be.softmax_kwargs and all(k == {"valid_cols": T} for k in be.softmax_kwargs)
    # second call reuses every pooled buffer, the zero-padded operands included
    n = eng.pool_bytes()
    eng.encode(g["x"])
    eng.decode(g["lat"])
    assert eng.pool_bytes() == n
    # one image per pass: identical codes, results within the emulation's batch-size noise
    whole_e, (whole_d, whole_i) = eng.encode(g["x"]), eng.decode(g["lat"], return_indices=True)
    eng.max_pixels_per_pass = g["x"].shape[2] * g["x"].shape[3]
    part_e, (part_d, part_i) = eng.encode(g["x"]), eng.decode(g["lat"], return_indices=True)
    assert rel_dev(part_e, whole_e) < 5e-5 and rel_dev(part_d, whole_d) < 5e-5 and torch.equal(whole_i, part_i)


def test_padded_operands_are_zero_past_t_and_written_before_it():
    """After encode and decode the K planes are zero in rows T..Tp-1 and V^T in columns T..Tp-1, while the first T rows
    / columns hold the last image's K and V; the softmax planes hold exact zeros past T."""
    from bbdm_b200.vqgan_engine import VQGANEngine
    name = "vq_t196"
    g = load(name)
    vq, _ = container(VQ_RAGGED_CONFIGS[name])
    be = EmuBackendRagged()
    p_planes = []
    orig = be.softmax_rows_split

    def keep(src, scale, out_hi, out_lo, valid_cols=None):
        orig(src, scale, out_hi, out_lo, valid_cols=valid_cols)
        p_planes.append((out_hi.clone(), out_lo.clone(), valid_cols))

    be.softmax_rows_split = keep
    eng = VQGANEngine(vq, backend=be)
    eng.encode(g["x"])
    eng.decode(g["lat"])
    T, Tp, C = 196, 256, 128
    pads = [(k, t) for p in eng._pools.values() for k, t in p.padded.items()]
    assert sorted(k[0][0] for k, _ in pads) == ["attention K", "attention K", "attention V^T", "attention V^T"]
    for (tag, shape, dtype), t in pads:
        assert tag[1] == T and dtype == torch.bfloat16
        if tag[0] == "attention K":
            assert shape == (2, Tp, C)
            assert torch.equal(t[:, T:].float(), torch.zeros(2, Tp - T, C))
            assert bool((t[0, :T] != 0).any())
        else:
            assert shape == (2, C, Tp)
            assert torch.equal(t[:, :, T:].float(), torch.zeros(2, C, Tp - T))
            assert bool((t[0, :, :T] != 0).any())
    assert len(p_planes) == 2 * (2 + 3)          # batch 2 x (encoder: level + mid, decoder: mid + 2 in the level)
    for hi, lo, v in p_planes:
        assert v == T and hi.shape == (T, Tp)
        assert not bool(hi[:, T:].view(torch.int16).any()) and not bool(lo[:, T:].view(torch.int16).any())
        torch.testing.assert_close((hi.double() + lo.double())[:, :T].sum(1), torch.ones(T, dtype=torch.float64),
                                   rtol=0, atol=1e-5)


def test_aligned_token_count_passes_no_valid_cols():
    """vq_tc's AttnBlock (C = 128, T = 256) keeps the call it always made: no valid_cols argument."""
    from bbdm_b200.vqgan_engine import VQGANEngine
    g = load("vq_tc")
    vq, _ = container(VQGAN_CONFIGS["vq_tc"])
    be = SoftmaxSpy()
    eng = VQGANEngine(vq, backend=be)
    eng.encode(g["x"])
    eng.decode(g["lat"])
    assert be.softmax_kwargs and all(k == {} for k in be.softmax_kwargs)
    assert not any(p.padded for p in eng._pools.values())


@pytest.mark.parametrize("ch,mult,res", [(32, 3, 16), (64, 2, 6)])
def test_attention_still_out_of_scope_says_why(ch, mult, res):
    """C = 96 (not a multiple of 64, beyond the flash kernels' 64) and a 3x3 map (narrower than 4) keep the error."""
    from bbdm_b200.vqgan_engine import VQGANEngine
    cfg = dict(embed_dim=3, n_embed=32, ddconfig=dict(double_z=False, z_channels=3, resolution=res, in_channels=3,
                                                      out_ch=3, ch=ch, ch_mult=(1, mult), num_res_blocks=1,
                                                      attn_resolutions=[], dropout=0.0))
    vq, _ = container(cfg)
    eng = VQGANEngine(vq, backend=EmuBackendRagged())
    with pytest.raises(NotImplementedError, match="C % 64 == 0 and a map at least 4 wide"):
        eng.encode(synth_images((1, 3, res, res), 5))


def _shadowed_run(name, mutate=None):
    from bbdm_b200.vqgan_engine import VQGANEngine
    g = load(name)
    vq, _ = container(VQ_RAGGED_CONFIGS[name])
    sh = RaggedShadow(EmuBackendRagged(), bounds=EMU_BOUNDS)
    sh.mutate = mutate or {}
    eng = VQGANEngine(vq, backend=sh)
    eng.refresh_weights()
    sh.register_engine(eng)
    eng.encode(g["x"], quant_conv=False)
    eng.encode(g["x"], quant_conv=True)
    eng.decode(g["lat"], return_indices=True)
    eng.decode(g["lat_b"], quant_conv_first=True)
    return sh


def test_shadow_accepts_the_padded_attention_and_flags_a_nonzero_padding_column():
    sh = _shadowed_run("vq_t196")
    print("\n" + sh.table("VQGAN executor vq_t196, emulation"))
    assert not sh.failures(), sh.failures()[:5]
    forms = [("softmax_rows_split", ("256 columns", "196 valid"), ()), ("conv_umma", ("taps 1", "split out"), ()),
             ("split_grad", (), ("colsum", "planes"))]
    assert not missing_forms(sh, forms), missing_forms(sh, forms)
    assert any(c.what == "padding columns +0" for c in sh.checks)
    first = next(i for i, (m, f) in enumerate(sh.launches) if m == "softmax_rows_split")

    def poke(a):
        a["out_lo"].view(-1, 256)[0, 200] = 1e-6

    bad = _shadowed_run("vq_t196", mutate={first: poke})
    assert bad.flagged_launches() == [first]
