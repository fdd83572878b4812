"""The launch guard of tests/_launch_guard.py over the CPU emulation (no GPU): Shadow(Guard(emulation)) accepts an
emulated sampling forward and training micro-step with no finding, each seeded defect -- a store one element past or
before an output, a store into the pitch gap of a padded-row output, an output element left unwritten, a load one
element past an input -- is flagged on that launch alone with its kind and argument, an in-place residual launch gives
the same bits guarded and unguarded, launches inside a capture pass through, and every launch kind is guarded and
required by the GPU cases of tests/test_gpu_launch_guard.py."""
import collections
import inspect

import pytest
import torch

from _emu_backend_origin import EmuBackendOrigin
from _launch_guard import EXEMPT, GUARD_MIN, PASS_THROUGH, Guard
from _launch_shadow import OUTPUTS, Shadow, space_to_depth, split_bf16
from _recipe import UNET_CONFIGS, fill_state_dict, synth_images

# the emulated F(6,3) chain (test_launch_shadow_host.py::EMU_BOUNDS)
EMU_BOUNDS = {"chain6": 2.5e-5}
# The emulation's contract differs from the kernels' where the kernels keep backward scratch: the emulated attention
# backwards (tests/_emu_backend.py::EmuBackend.attention_bwd, test_transformer_training_host.py's attention_cross_bwd)
# differentiate the fp64 attention with autograd and write no softmax statistics, which only the kernels read.
_NO_STATS = "the emulated backward writes no softmax statistics"
EMU_EXEMPT = {(m, k): _NO_STATS for m in ("attention_bwd", "attention_cross_bwd") for k in ("lse", "delta")}


# ------------------------------------------------------------------------------------------ clean emulated runs
def test_guard_accepts_the_emulated_sampling_forward():
    from bbdm_b200.engine import UNetEngine
    from bbdm_b200.unet import UNetModel
    net = UNetModel(**UNET_CONFIGS["mid_pixel"]).eval()
    net.load_state_dict(fill_state_dict({k: tuple(v.shape) for k, v in net.state_dict().items()}, seed=1234))
    g = Guard(EmuBackendOrigin())
    sh = Shadow(g, bounds=EMU_BOUNDS)
    eng = UNetEngine(net, backend=sh)
    eng.refresh_weights()
    sh.register_engine(eng)
    x, y = synth_images((1, 3, 32, 32), 1), synth_images((1, 3, 32, 32), 2)
    eng.forward(x, torch.tensor([500]), y)
    print("\n" + sh.table("mid_pixel forward, 32x32, B=1, guarded emulation") + "\n" + g.summary())
    assert not g.findings, g.findings[:5]
    assert not sh.failures(), sh.failures()[:5]
    assert len(g.launches) == len(sh.launches) > 100


def test_guard_accepts_the_emulated_training_step(monkeypatch):
    import test_train_shadow_host as T
    g = Guard(T.EmuBackend(), exempt=EMU_EXEMPT)
    monkeypatch.setattr(T, "EmuBackend", lambda: g)          # Shadow(Guard(emulation)) in the host shadow test's step
    sh = T._train_step(monkeypatch)
    print("\n" + sh.table("training micro-step, quarter-size LBBDM-f4 + SpatialTransformer, B=2, guarded emulation")
          + "\n" + g.summary())
    assert not g.findings, g.findings[:5]
    assert not sh.failures(), sh.failures()[:5]
    assert {"adam_multi", "split_grad", "conv_wgrad", "attention_bwd"} <= set(g.launches)


# ------------------------------------------------------------------------------------------ seeded defects
def _elem(t, offset):
    """The one-element view of t's storage at element offset (relative to t's first element)."""
    return torch.as_strided(t, (1,), (1,), t.storage_offset() + offset)


class _Nth(EmuBackendOrigin):
    """The emulation whose DEFECTIVE method misbehaves on its second call only."""
    DEFECTIVE = None

    def __init__(self):
        super().__init__()
        self.n = collections.Counter()

    def _hit(self, name):
        self.n[name] += 1
        return self.n[name] == 2


class _WritesPastOut(_Nth):
    def nhwc_to_nchw(self, src, out):
        super().nhwc_to_nchw(src, out)
        if self._hit("nhwc_to_nchw"):
            _elem(out, out.numel()).fill_(0.0)


class _WritesBeforeOut(_Nth):
    def nhwc_to_nchw(self, src, out):
        super().nhwc_to_nchw(src, out)
        if self._hit("nhwc_to_nchw"):
            _elem(out, -1).fill_(0.0)


class _WritesPitchGap(_Nth):
    def split_grad(self, src, hi, lo, hi_t, lo_t, colsum=None, workspace=None):
        super().split_grad(src, hi, lo, hi_t, lo_t, colsum, workspace)
        if self._hit("split_grad"):
            _elem(hi_t, hi_t.shape[1]).fill_(0.0)          # behind row 0, before row 1


class _LeavesLastUnwritten(_Nth):
    def nhwc_to_nchw(self, src, out):
        if not self._hit("nhwc_to_nchw"):
            return super().nhwc_to_nchw(src, out)
        out.reshape(-1)[:-1].copy_(src.permute(0, 3, 1, 2).reshape(-1)[:-1])


class _ReadsPastInput(_Nth):
    def nhwc_to_nchw(self, src, out):
        super().nhwc_to_nchw(src, out)
        if self._hit("nhwc_to_nchw"):
            out.reshape(-1)[-1:] += 0.0 * _elem(src, src.numel())


def _drive(be):
    """Three layout copies and two gradient splits into padded-row transposed planes (train._transposed_planes: rows of
    P = 44 padded to 48) under Shadow(Guard(be)).  Launch indices: nhwc_to_nchw 0-2, split_grad 3-4."""
    g = Guard(be)
    sh = Shadow(g)
    gen = torch.Generator().manual_seed(5)
    for _ in range(3):
        src = torch.randn((2, 5, 7, 16), generator=gen)
        sh.nhwc_to_nchw(src, torch.empty((2, 16, 5, 7)))
    for _ in range(2):
        src = torch.randn((44, 32), generator=gen)
        hi_t, lo_t = (torch.empty((32, 48), dtype=torch.bfloat16)[:, :44] for _ in range(2))
        sh.split_grad(src, torch.empty((44, 32), dtype=torch.bfloat16), torch.empty((44, 32), dtype=torch.bfloat16),
                      hi_t, lo_t, torch.empty(32), torch.empty(32))
    return sh, g


def test_clean_drive_has_no_finding():
    sh, g = _drive(_Nth())
    assert g.launches == ["nhwc_to_nchw"] * 3 + ["split_grad"] * 2
    assert not g.findings and not sh.failures()


# defect -> (backend, launch, argument, kind, offset in bytes from the argument's first element / element index)
DEFECTS = {
    "write one element past out": (_WritesPastOut, 1, "out", "write after", 2 * 16 * 5 * 7 * 4),
    "write one element before out": (_WritesBeforeOut, 1, "out", "write before", -4),
    "write into the pitch gap": (_WritesPitchGap, 4, "hi_t", "write in gap", 44 * 2),
    "last output element unwritten": (_LeavesLastUnwritten, 1, "out", "unwritten", 2 * 16 * 5 * 7 - 1),
}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_seeded_defect_is_flagged_on_its_launch_alone(defect):
    cls, idx, arg, kind, offset = DEFECTS[defect]
    sh, g = _drive(cls())
    print("\n" + g.summary(defect))
    assert g.flagged() == [idx]
    assert [(f.argument, f.kind, f.count, f.offset) for f in g.findings] == [(arg, kind, 1 if kind == "unwritten" else
                                                                              4 if arg == "out" else 2, offset)]


def test_read_past_an_input_is_flagged_by_the_shadow_on_its_launch_alone():
    """The element behind src is NaN in the guarded buffer; the unguarded emulation reads whatever lies there."""
    sh, g = _drive(_ReadsPastInput())
    assert sh.flagged_launches() == [1]
    assert {f.launch for f in g.findings} <= {1}             # the NaN it computed is also a NaN output element


def test_guard_zone_holds_a_whole_stray_tile():
    """A store a full 128 x 256 fp32 tile (128 KiB) past the output still lands in the guard zone."""
    class FarPast(_Nth):
        def nhwc_to_nchw(self, src, out):
            super().nhwc_to_nchw(src, out)
            if self._hit("nhwc_to_nchw"):
                _elem(out, out.numel() + 128 * 256 - 1).fill_(0.0)
    assert GUARD_MIN > 128 * 256 * 4
    sh, g = _drive(FarPast())
    assert [(f.launch, f.kind) for f in g.findings] == [(1, "write after")]


# ------------------------------------------------------------------------------------------ aliasing and capture
def test_in_place_residual_is_bit_identical_guarded_and_unguarded():
    """conv_direct with residual aliasing out (out += conv(src)): the two arguments share one relocated buffer, so the
    launch reads the residual it overwrites exactly as it does unguarded."""
    gen = torch.Generator().manual_seed(9)
    src, w = torch.randn((2, 6, 7, 8), generator=gen), 0.1 * torch.randn((4, 8, 3, 3), generator=gen)
    res = torch.randn((2, 6, 7, 4), generator=gen)
    outs = []
    for wrap in (lambda be: be, Guard):
        be = wrap(EmuBackendOrigin())
        wp = torch.empty((9, 8, 4))
        be.pack_weight_f32(w, wp)
        out = res.clone()
        be.conv_direct(src, wp, None, out, out, 4, 3, 1)
        outs.append(out)
        if isinstance(be, Guard):
            assert not be.findings
    assert torch.equal(outs[0], outs[1])
    assert not torch.equal(outs[0], res)


def test_launches_inside_a_capture_pass_through(monkeypatch):
    """As test_launch_shadow_coverage_host.py::test_launches_inside_a_capture_pass_through_unchecked: inside a capture
    the guard neither relocates nor checks, and the launch runs on the caller's tensors."""
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    g = Guard(_WritesPastOut())
    sh = Shadow(g)
    src = torch.randn(2, 4, 6, 8)
    hi = torch.empty((2, 2, 3, 32), dtype=torch.bfloat16)
    lo = torch.empty_like(hi)
    sh.s2d_split(src, hi, lo)
    assert sh.captured == ["s2d_split"] and sh.launches == [] and g.launches == [] and g.findings == []
    h, l = split_bf16(space_to_depth(src))
    assert torch.equal(hi, h) and torch.equal(lo, l)


# ------------------------------------------------------------------------------------------ coverage
def test_every_launch_is_guarded_and_required_on_the_gpu():
    from bbdm_b200 import cabi
    from test_gpu_launch_guard import required_methods
    public = {n for n, f in inspect.getmembers(cabi.CudaBackend, inspect.isfunction) if not n.startswith("_")}
    assert public == set(OUTPUTS) | set(PASS_THROUGH), (public - set(OUTPUTS) - set(PASS_THROUGH))
    assert not set(OUTPUTS) & set(PASS_THROUGH)
    assert required_methods() == set(OUTPUTS), set(OUTPUTS) - required_methods()
    for (method, arg), reason in EXEMPT.items():
        assert arg in OUTPUTS[method] and reason, (method, arg)
