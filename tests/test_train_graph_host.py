"""Host logic of the graphed UNet training step (bbdm_b200/train_graph.py) with the capture stubbed out, and the
argument handling of FusedAdam(capturable=True) through the emulation backend.  No GPU."""
import copy

import pytest
import torch

from _emu_backend import EmuBackend
from _recipe import UNET_CONFIGS, bb_namespace
from bbdm_b200 import optim as O
from bbdm_b200 import train, train_graph
from bbdm_b200 import unet as U


def _unet(**kw):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    return BrownianBridgeModel(bb_namespace(dict(UNET_CONFIGS["tiny_variant"], **kw))).denoise_fn.train()


def _inputs(b=2, ctx=False, ctx_grad=False):
    x = torch.randn(b, 3, 16, 16)
    emb = U.timestep_embedding(torch.arange(b), 32)
    c = torch.randn(b, 3, 16, 16).requires_grad_(ctx_grad) if ctx else None
    return x, emb, c


def test_switch_defaults_off_and_follows_the_environment():
    assert U.UNetModel.train_graph is False
    import subprocess
    import sys
    code = "import bbdm_b200.unet as U; print(U.UNetModel.train_graph)"
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True,
                         env={**__import__("os").environ, "BBDM_TRAIN_GRAPH": "1"}, cwd=train.__file__.rsplit("/", 2)[0])
    assert out.stdout.strip() == "True", out.stderr


def test_cache_key_changes_with_everything_the_capture_depends_on(monkeypatch):
    net = _unet()
    x, emb, c = _inputs()
    k = train_graph.cache_key(net, x, emb, c)
    assert train_graph.cache_key(net, x.clone(), emb.clone(), c) == k           # values are not part of the key
    changed = {
        "batch": train_graph.cache_key(net, *_inputs(b=3)),
        "context": train_graph.cache_key(net, *_inputs(ctx=True)),
        "context grad": train_graph.cache_key(net, *_inputs(ctx=True, ctx_grad=True)),
        "dtype": train_graph.cache_key(net, x.double(), emb, c),
    }
    p = next(net.parameters())
    old = p.data
    p.data = p.data.clone()                         # an EMA apply_shadow: new addresses
    changed["address"] = train_graph.cache_key(net, x, emb, c)
    p.data = old                                    # restore: the old key again
    assert train_graph.cache_key(net, x, emb, c) == k
    p.requires_grad_(False)
    changed["requires_grad"] = train_graph.cache_key(net, x, emb, c)
    p.requires_grad_(True)
    net.eval()
    changed["eval"] = train_graph.cache_key(net, x, emb, c)
    net.train()
    for mod, name, val in ((U, "NATIVE_TRAIN_CONV", False), (train, "WINO_TRAIN", not train.WINO_TRAIN),
                           (train, "WINO_MIN_C", 1), (train, "WINO_MIN_TILES", 1)):
        with monkeypatch.context() as mp:
            mp.setattr(mod, name, val)
            changed[name] = train_graph.cache_key(net, x, emb, c)
    assert train_graph.cache_key(net, x, emb, c) == k
    assert all(v != k for v in changed.values()), [n for n, v in changed.items() if v == k]


def test_fallback_reasons(monkeypatch):
    net = _unet()
    x, emb, c = _inputs()
    assert train_graph.fallback_reason(net, x, emb, c) == "CPU input"
    with torch.autocast("cpu", dtype=torch.bfloat16):
        assert train_graph.fallback_reason(net, x, emb, c) == "autocast"
    assert train_graph.fallback_reason(_unet(dropout=0.1), x, emb, c) == "active dropout"
    assert train_graph.fallback_reason(_unet(dropout=0.1).eval(), x, emb, c) == "CPU input"   # eval: no dropout
    # inputs that claim to be on CUDA: the remaining checks (capture in progress, backend)
    fake = type("T", (), {"is_cuda": True})()
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: True)
    assert train_graph.fallback_reason(net, fake, fake, None) == "stream capture in progress"
    monkeypatch.setattr(torch.cuda, "is_current_stream_capturing", lambda: False)
    monkeypatch.setattr(train, "_BACKEND", EmuBackend())
    assert train_graph.fallback_reason(net, fake, fake, None) == "backend"


def test_one_capture_per_key_and_one_live_graph(monkeypatch):
    """forward() with the capture and the replay stubbed: a capture exactly when the key changes, the previous graph
    dropped first, and None (the eager graph) whenever fallback_reason says so."""
    net = _unet()
    log = []

    def capture(unet, x, emb, context, key):
        assert train_graph._STATES.get(unet) is None            # the old graph is released before the new capture
        log.append(key)
        train_graph.CAPTURES["n"] += 1
        st = train_graph._GraphState(key)
        return st

    monkeypatch.setattr(train_graph, "fallback_reason", lambda *a: None)
    monkeypatch.setattr(train_graph, "_capture", capture)
    monkeypatch.setattr(train_graph, "_apply", lambda st, x, emb, c: ("replayed", st))
    monkeypatch.setattr(torch.cuda, "device", lambda d: __import__("contextlib").nullcontext())
    x, emb, c = _inputs()
    n0 = train_graph.CAPTURES["n"]
    r1 = train_graph.forward(net, x, emb, c)
    r2 = train_graph.forward(net, x, emb, c)
    assert r1[0] == "replayed" and r1[1] is r2[1] and train_graph.CAPTURES["n"] - n0 == 1
    train_graph.forward(net, *_inputs(b=3))                      # batch size: one capture
    train_graph.forward(net, x, emb, c)                          # and back: one more (one live graph per model)
    assert train_graph.CAPTURES["n"] - n0 == 3 and len(log) == 3
    other = _unet()
    train_graph.forward(other, x, emb, c)                        # a second model keeps its own graph
    assert train_graph._STATES[net] is not train_graph._STATES[other]
    train_graph.release(net)
    assert net not in train_graph._STATES
    monkeypatch.setattr(train_graph, "fallback_reason", lambda *a: "autocast")
    assert train_graph.forward(net, x, emb, c) is None and train_graph.CAPTURES["n"] - n0 == 4


def test_unet_forward_switch_off_and_on_cpu_is_the_eager_graph(monkeypatch):
    """On CPU tensors the switch changes nothing: the same eager graph, bit for bit (train_graph never captures)."""
    monkeypatch.setattr(U, "NATIVE_TRAIN_CONV", False)
    net = _unet()
    x, _, _ = _inputs()
    t = torch.tensor([3, 700])
    n0 = train_graph.CAPTURES["n"]
    a = net(x, timesteps=t)
    net.train_graph = True
    b = net(x, timesteps=t)
    assert torch.equal(a, b) and train_graph.CAPTURES["n"] == n0


# ---- FusedAdam(capturable=True) -----------------------------------------------------------------------------------
class _EmuDev(EmuBackend):
    """The emulation with the device-step entry point: step incremented in place, lr read from its tensor."""

    def adam_multi_dev(self, tab, exp_avg, exp_avg_sq, *, step, lr, beta1, beta2, eps, weight_decay, ema_shadow=None,
                       ema_decay=0.0):
        step += 1
        self.adam_multi(tab, exp_avg, exp_avg_sq, lr=float(lr), beta1=beta1, beta2=beta2, eps=eps,
                        weight_decay=weight_decay, step=int(step), ema_shadow=ema_shadow, ema_decay=ema_decay)
        self.calls[-1] = "adam_multi_dev"


@pytest.fixture
def emu(monkeypatch):
    be = _EmuDev()
    monkeypatch.setattr(O.FusedAdam, "backend_factory", staticmethod(lambda: be))
    return be


def _net(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.SiLU(), torch.nn.Flatten(),
                               torch.nn.Linear(8 * 36, 5))


def test_capturable_argument_handling(emu):
    for flag in ("maximize", "differentiable", "decoupled_weight_decay"):
        with pytest.raises(NotImplementedError):
            O.FusedAdam(_net().parameters(), **{flag: True})
    with pytest.raises(NotImplementedError):
        O.FusedAdam(_net().parameters(), amsgrad=True)
    opt = O.FusedAdam(_net().parameters(), capturable=True)
    assert opt.param_groups[0]["capturable"] is True


def test_capturable_matches_host_form_and_state_dict_shape(emu):
    a, b = _net(), _net()
    oa = O.FusedAdam(a.parameters(), lr=1e-3, weight_decay=1e-4)
    ob = O.FusedAdam(b.parameters(), lr=1e-3, weight_decay=1e-4, capturable=True)
    x = torch.randn(4, 3, 6, 6)
    for it in range(4):
        for net, opt in ((a, oa), (b, ob)):
            opt.param_groups[0]["lr"] = 1e-3 / (it + 1)           # each eager step refreshes the device lr
            opt.zero_grad(set_to_none=True)
            net(x).square().mean().backward()
            opt.step()
    assert "adam_multi_dev" in emu.calls and "adam_multi" in emu.calls
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.equal(pa, pb)
    sa, sb = oa.state_dict(), ob.state_dict()
    assert sa["state"].keys() == sb["state"].keys()
    for k in sa["state"]:
        assert set(sa["state"][k]) == set(sb["state"][k]) == {"step", "exp_avg", "exp_avg_sq"}
        assert float(sb["state"][k]["step"]) == 4.0 and sb["state"][k]["step"].dtype == torch.float32
    # every parameter entry its own step tensor, like torch.optim.Adam's checkpoints
    assert len({id(s["step"]) for s in sb["state"].values()}) == len(sb["state"])
    assert sb["param_groups"][0]["capturable"] is True
    # checkpoints cross between the two forms and torch.optim.Adam
    t = torch.optim.Adam(_net().parameters(), lr=1e-3)
    t.load_state_dict(copy.deepcopy(sb))
    oa.load_state_dict(copy.deepcopy(sb))
    ob.load_state_dict(copy.deepcopy(sa))
    assert oa.param_groups[0]["capturable"] is False and ob.param_groups[0]["capturable"] is True
    for net, opt in ((a, oa), (b, ob)):
        opt.zero_grad(set_to_none=True)
        net(x).square().mean().backward()
        opt.step()
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.equal(pa, pb)
    assert float(ob.state_dict()["state"][0]["step"]) == 5.0


def test_capturable_state_must_exist_before_a_capture(emu, monkeypatch):
    net = _net()
    opt = O.FusedAdam(net.parameters(), capturable=True)
    net(torch.randn(2, 3, 6, 6)).sum().backward()
    monkeypatch.setattr(O, "_capturing", lambda: True)
    with pytest.raises(RuntimeError, match="eager step"):
        opt.step()
    monkeypatch.setattr(O, "_capturing", lambda: False)
    opt.step()
    for p in net.parameters():
        p.grad = p.grad.clone()                      # new gradient addresses
    monkeypatch.setattr(O, "_capturing", lambda: True)
    with pytest.raises(RuntimeError, match="changed address"):
        opt.step()


def test_header_declares_the_device_step_entry_point():
    """test_cabi_symbols checks every header symbol against the library and the binding; the new entry point is one."""
    from test_cabi_symbols import declared_symbols
    from bbdm_b200 import cabi
    assert "bbdm_adam_multi_dev" in declared_symbols()
    assert "bbdm_adam_multi_dev" in cabi.SYMBOLS
