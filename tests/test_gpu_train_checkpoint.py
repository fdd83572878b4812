"""-m gpu: UNetModel(use_checkpoint=True) on the sm_90a training kernels.  Every ResBlock, AttentionBlock and transformer
block recomputes its forward in the backward with the forward's own launches, so the loss and every parameter gradient
are bit-identical to the un-checkpointed step, eager and on CUDA-graph replays; toggling the flag costs one recapture;
and the memory one cfg2-architecture step allocates falls by more than half."""
import warnings

import pytest
import torch

from _hd128 import HD128_CONFIGS
from _recipe import UNET_CONFIGS, bb_namespace, fill_state_dict, synth_images

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (UNet config, batch): the aligned pixel UNet at 32x32 and at the ragged 48x48 / batch 3, a SpatialTransformer UNet
# (4 heads of 64, cross-attention over the 3-channel context) and the cfg2 architecture at 128x128
CASES = {
    "mid_pixel": (UNET_CONFIGS["mid_pixel"], 2),
    "mid_pixel_48_b3": (dict(UNET_CONFIGS["mid_pixel"], image_size=48), 3),
    "mid_st_hd64": (dict(HD128_CONFIGS["mid_st_hd128"], num_heads=4), 2),
    "cfg2_128_b2": (dict(UNET_CONFIGS["cfg2"], image_size=128), 2),
}


def _model(cfg):
    from model.BrownianBridge.BrownianBridgeModel import BrownianBridgeModel
    net = BrownianBridgeModel(bb_namespace(cfg)).train()
    shapes = {k: tuple(v.shape) for k, v in net.denoise_fn.state_dict().items()}
    net.denoise_fn.load_state_dict(fill_state_dict(shapes, seed=1234))
    return net.to(DEV)


def _inputs(B, S):
    x, y = synth_images((B, 3, S, S), seed=11, device=DEV), synth_images((B, 3, S, S), seed=12, device=DEV)
    t = torch.tensor([(17 + 311 * i) % 1000 for i in range(B)], dtype=torch.long, device=DEV)
    nz = torch.randn((B, 3, S, S), generator=torch.Generator().manual_seed(77)).to(DEV)
    return x, y, t, nz


def _step(net, inputs):
    """loss, {name: grad}, the library-path warnings of one training step."""
    from bbdm_b200 import train
    x, y, t, nz = inputs
    train._WARNED.clear()                       # every step reports its own library-path shapes
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        net.zero_grad(set_to_none=True)
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()
    torch.cuda.synchronize()
    train.backend().check_fault()
    lib = {str(r.message) for r in rec if "stock PyTorch" in str(r.message)}
    return loss.detach().clone(), {n: p.grad.detach().clone() for n, p in net.denoise_fn.named_parameters()}, lib


def _same(a, b, what):
    assert torch.equal(a[0], b[0]), (what, float(a[0]), float(b[0]))
    bad = [n for n in a[1] if not torch.equal(a[1][n], b[1][n])]
    assert not bad, (what, bad[:5])


def _captures():
    from bbdm_b200 import train_graph
    return train_graph.CAPTURES["n"]


@pytest.mark.parametrize("case", list(CASES))
def test_checkpointed_step_is_bit_identical_eager_and_graphed(case, monkeypatch):
    """The trimmed recompute (GroupNorm statistics reused, a ResBlock's tail convs skipped, Winograd-route planes from
    prep) and the whole-block recompute against the plain step, eager; the trimmed one on graph replays."""
    from bbdm_b200 import train, train_graph
    cfg, B = CASES[case]
    net = _model(cfg)
    inputs = _inputs(B, cfg["image_size"])
    plain = _step(net, inputs)
    net.denoise_fn.use_checkpoint = True
    monkeypatch.setattr(train, "RECOMPUTE_TRIM", False)
    _same(plain, _step(net, inputs), "eager, whole-block recompute")
    monkeypatch.setattr(train, "RECOMPUTE_TRIM", True)
    ck = _step(net, inputs)
    _same(plain, ck, "eager, trimmed recompute")
    assert ck[2] <= plain[2], ck[2] - plain[2]          # the recompute takes no library path the step does not take
    net.denoise_fn.train_graph = True
    n0 = _captures()
    for _ in range(2):
        _same(ck, _step(net, inputs), "graphed")
    assert _captures() - n0 == 1
    train_graph.release(net.denoise_fn)


def test_toggling_the_flag_costs_one_recapture():
    from bbdm_b200 import train_graph
    net = _model(UNET_CONFIGS["mid_pixel"])
    net.denoise_fn.train_graph = True
    inputs = _inputs(2, 32)
    plain = _step(net, inputs)
    n0 = _captures()
    net.denoise_fn.use_checkpoint = True
    ck = _step(net, inputs)
    _step(net, inputs)
    assert _captures() - n0 == 1
    net.denoise_fn.use_checkpoint = False
    again = _step(net, inputs)
    assert _captures() - n0 == 2
    _same(plain, ck, "toggled on")
    _same(plain, again, "toggled off")
    train_graph.release(net.denoise_fn)


def test_cfg2_step_memory_at_most_half():
    """Peak allocated memory of one cfg2-architecture training step (forward + backward) at 128x128, batch 4, above what
    is allocated before it: the weights and the gradient buffers of an earlier step, which both forms keep, are not part
    of what checkpointing can save."""
    cfg = dict(UNET_CONFIGS["cfg2"], image_size=128)
    net = _model(cfg)
    x, y, t, nz = _inputs(4, 128)

    def step():
        loss, _ = net.p_losses(x, y, y, t, nz)
        loss.backward()

    step()                                       # the gradient buffers exist from here on
    step_peak, total_peak = {}, {}
    for ck in (False, True):
        net.denoise_fn.use_checkpoint = ck
        net.zero_grad(set_to_none=False)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        step()
        torch.cuda.synchronize()
        total_peak[ck] = torch.cuda.max_memory_allocated()
        step_peak[ck] = total_peak[ck] - base
    print(f"\n[cfg2 128x128 b4] step peak above the resident state: plain {step_peak[False] / 2**30:.2f} GiB, checkpointed "
          f"{step_peak[True] / 2**30:.2f} GiB ({step_peak[True] / step_peak[False]:.3f}x); peak allocated in all: "
          f"{total_peak[False] / 2**30:.2f} / {total_peak[True] / 2**30:.2f} GiB ({total_peak[True] / total_peak[False]:.3f}x)")
    assert step_peak[True] <= 0.5 * step_peak[False], step_peak
