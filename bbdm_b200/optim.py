"""Multi-tensor Adam and EMA on flat state buffers.

``FusedAdam`` is a ``torch.optim.Adam`` whose ``step()`` is ONE kernel launch over every parameter tensor
(``bbdm_adam_multi``) instead of ~10 elementwise launches per tensor; same constructor, same hyper-parameters,
same ``state_dict`` layout (``step`` / ``exp_avg`` / ``exp_avg_sq`` per parameter -- the per-parameter tensors
are views into two flat buffers), so optimizer checkpoints written by the reference runner
(runners/BaseRunner.py:141-152) load and save unchanged.  ``capturable=True`` keeps the step counter and the learning
rate on the device (``bbdm_adam_multi_dev``), so ``step()`` can be captured into a CUDA graph like
``torch.optim.Adam(capturable=True)``; checkpoints of both forms and of torch.optim.Adam load into either.  The reference builds its optimizer in
runners/utils.py:48-57; the one-line switch is shown in INTEGRATION.md.

``FusedEMA`` has the interface of the reference ``EMA`` (runners/base/EMA.py:4-43: register / reset_device /
update / apply_shadow / restore, attributes ``shadow`` and ``backup``) with the shadow copy in one flat buffer
(``shadow[name]`` are views) and ``update`` as one launch (``bbdm_ema_multi``) -- the reference clones every
tensor per update.  ``runners/base/EMA.py`` of this repo overlays the reference module with it (namespace-package
overlay, like the two model files).

There is no CPU implementation: CPU parameters raise (tests inject an emulation backend).
"""
from __future__ import annotations

import torch

from . import cabi


class TensorTable:
    """Device-side description of a parameter list for the multi-tensor kernels: pointer arrays (refreshed when
    an address changes -- EMA ``.data`` swaps, fresh ``.grad`` tensors), element counts, offsets of each tensor's
    state inside the flat buffers (16-byte aligned) and the (tensor, chunk) work list, one entry per CTA."""

    def __init__(self, tensors, chunk_elems):
        self.tensors = list(tensors)
        assert self.tensors, "empty parameter list"
        dev = self.tensors[0].device
        for t in self.tensors:
            if t.device != dev or t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError("bbdm_b200.optim: parameters must be contiguous fp32 tensors on one device")
        self.device = dev
        numel = [t.numel() for t in self.tensors]
        offs, total = [], 0
        for n in numel:
            offs.append(total)
            total += (n + 3) // 4 * 4
        self.total = total
        self.numel_host, self.offsets_host = numel, offs
        ct, ci = [], []
        for i, n in enumerate(numel):
            for k in range((n + chunk_elems - 1) // chunk_elems):
                ct.append(i)
                ci.append(k)
        self.n_chunks = len(ct)
        self.numel = torch.tensor(numel, dtype=torch.int64, device=dev)
        self.offsets = torch.tensor(offs, dtype=torch.int64, device=dev)
        self.chunk_tensor = torch.tensor(ct, dtype=torch.int32, device=dev)
        self.chunk_index = torch.tensor(ci, dtype=torch.int32, device=dev)
        self.params = torch.zeros(len(numel), dtype=torch.int64, device=dev)
        self.grads = torch.zeros(len(numel), dtype=torch.int64, device=dev)
        self._pkey = self._gkey = None

    def views(self, flat):
        return [flat[o:o + n].view(t.shape) for o, n, t in zip(self.offsets_host, self.numel_host, self.tensors)]

    def key(self, with_grads=False):
        """(parameter addresses, gradient addresses or None) as the device tables should hold them."""
        pk = tuple(t.data_ptr() for t in self.tensors)
        if not with_grads:
            return pk, None
        gk = []
        for t in self.tensors:
            g = t.grad
            if g is None:
                gk.append(0)
                continue
            if g.dtype != torch.float32 or not g.is_contiguous() or g.is_sparse:
                raise ValueError("bbdm_b200.optim: gradients must be dense contiguous fp32")
            gk.append(g.data_ptr())
        return pk, tuple(gk)

    def refresh(self, with_grads=False):
        pk, gk = self.key(with_grads)
        if pk != self._pkey:
            self.params.copy_(torch.tensor(pk, dtype=torch.int64), non_blocking=False)
            self._pkey = pk
        if with_grads and gk != self._gkey:
            self.grads.copy_(torch.tensor(gk, dtype=torch.int64), non_blocking=False)
            self._gkey = gk


def _capturing():
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


def _backend_for(t, factory):
    be = factory()
    if not t.is_cuda and getattr(be, "requires_cuda", True):
        raise RuntimeError("bbdm_b200.optim runs only on a CUDA sm_90a device (kernels behind libbbdm_b200.so); "
                           "there is no CPU fallback.")
    return be


class FusedAdam(torch.optim.Adam):
    """torch.optim.Adam with a single-launch multi-tensor step.  ``ema`` (a FusedEMA registered on the same
    parameters, optional) lets ``step(ema_update=True)`` apply the EMA update in the same pass."""

    backend_factory = staticmethod(lambda: cabi.CudaBackend())

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, **kw):
        if amsgrad or any(kw.get(k) for k in ("maximize", "differentiable", "decoupled_weight_decay")):
            raise NotImplementedError("FusedAdam: amsgrad / maximize / differentiable / decoupled_weight_decay are not "
                                      "implemented")
        kw.pop("foreach", None)
        kw.pop("fused", None)
        self._capturable = bool(kw.get("capturable", False))
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, **kw)
        self._be = None
        self._flat = {}            # group index -> dict(table, exp_avg, exp_avg_sq, step[, lr])

    def _group_state(self, gi, group):
        st = self._flat.get(gi)
        plist = [p for p in group["params"] if p.requires_grad]
        if st is not None and len(st["table"].tensors) == len(plist) and all(a is b for a, b in zip(st["table"].tensors, plist)):
            return st
        if self._capturable and _capturing():
            raise RuntimeError("FusedAdam(capturable=True): the optimizer state is created by the first step(); run one "
                               "eager step (e.g. in the warm-up before the capture) first")
        if self._be is None:
            self._be = _backend_for(plist[0], self.backend_factory)
        tab = TensorTable(plist, self._be.optim_chunk_elems())
        m = torch.zeros(tab.total, dtype=torch.float32, device=tab.device)
        v = torch.zeros(tab.total, dtype=torch.float32, device=tab.device)
        count = 0.0
        # adopt state loaded through load_state_dict (or left by a previous table) into the flat buffers
        olds = []
        for p, mv, vv in zip(plist, tab.views(m), tab.views(v)):
            old = self.state.get(p)
            if old and "exp_avg" in old:
                mv.copy_(old["exp_avg"])
                vv.copy_(old["exp_avg_sq"])
                count = float(old["step"])
            olds.append((mv, vv))
        # one shared counter per group: a host scalar, or (capturable) an fp32 scalar on the parameters' device that
        # the update kernel increments, as torch.optim.Adam(capturable=True) keeps it
        step = torch.tensor(count, dtype=torch.float32, device=tab.device if self._capturable else "cpu")
        for p, (mv, vv) in zip(plist, olds):
            self.state[p] = {"step": step, "exp_avg": mv, "exp_avg_sq": vv}
        st = self._flat[gi] = {"table": tab, "exp_avg": m, "exp_avg_sq": v, "step": step}
        if self._capturable:
            st["lr"] = torch.zeros((), dtype=torch.float64, device=tab.device)
        return st

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        for group in self.param_groups:             # a checkpoint of either form loads into either form
            group["capturable"] = self._capturable
        self._flat = {}                             # re-adopt the loaded tensors on the next step

    def state_dict(self):
        # internally one step counter is shared by a group's parameters; a checkpoint gets one tensor per parameter
        # (stock torch.optim.Adam increments each entry separately after loading it)
        sd = super().state_dict()
        for st in sd["state"].values():
            if "step" in st:
                st["step"] = torch.as_tensor(st["step"]).clone()
        return sd

    @torch.no_grad()
    def step(self, closure=None, ema=None, ema_update=False):
        """capturable=True: the step counter and the learning rate are device scalars.  Outside a CUDA graph capture
        every call first writes group["lr"] into that scalar (so LR schedulers keep working); inside a capture the
        scalar is read as it stands when the graph replays.  A captured step needs the gradients at the addresses
        they had in the last eager step (e.g. ``zero_grad(set_to_none=False)``)."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        capturing = self._capturable and _capturing()
        for gi, group in enumerate(self.param_groups):
            have = [p.grad is not None for p in group["params"] if p.requires_grad]
            if not any(have):
                continue
            if not all(have):
                # torch.optim.Adam keeps a step count per parameter; the multi-tensor kernel keeps one per group
                raise NotImplementedError("FusedAdam: every trainable parameter of a group must receive a gradient in "
                                          "the same steps (true for the BBDM UNet); use torch.optim.Adam otherwise")
            st = self._group_state(gi, group)
            tab = st["table"]
            if capturing:
                # the pointer tables are refreshed by a blocking host-to-device copy, which a capture cannot hold
                if tab.key(with_grads=True) != (tab._pkey, tab._gkey):
                    raise RuntimeError("FusedAdam(capturable=True): a parameter or gradient changed address since the "
                                       "last eager step; a captured step needs them where the eager step saw them")
            else:
                tab.refresh(with_grads=True)
            beta1, beta2 = group["betas"]
            shadow, decay = None, 0.0
            if ema is not None and ema_update and ema.covers(tab):
                shadow, decay = ema.flat, ema.ema_decay
            hyper = dict(beta1=float(beta1), beta2=float(beta2), eps=float(group["eps"]),
                         weight_decay=float(group["weight_decay"]), ema_shadow=shadow, ema_decay=decay)
            if self._capturable:
                if not capturing:
                    st["lr"].fill_(float(group["lr"]))
                self._be.adam_multi_dev(tab, st["exp_avg"], st["exp_avg_sq"], step=st["step"], lr=st["lr"], **hyper)
            else:
                st["step"] += 1
                self._be.adam_multi(tab, st["exp_avg"], st["exp_avg_sq"], lr=float(group["lr"]), step=int(st["step"]),
                                    **hyper)
        return loss


class FusedEMA:
    """Interface of the reference EMA (runners/base/EMA.py); the shadow lives in one flat fp32 buffer."""

    backend_factory = staticmethod(lambda: cabi.CudaBackend())

    def __init__(self, ema_decay):
        self.ema_decay = ema_decay
        self.backup = {}
        self.shadow = {}
        self.flat = None
        self._table = None
        self._names = None
        self._be = None

    @staticmethod
    def _trainable(model):
        return [(n, p) for n, p in model.named_parameters() if p.requires_grad]

    def _build(self, model, source=None):
        """(Re)create the flat buffer for model's trainable parameters; contents from `source` (name -> tensor,
        e.g. a loaded checkpoint) or from the parameters themselves."""
        named = self._trainable(model)
        if self._be is None:
            self._be = _backend_for(named[0][1], self.backend_factory)
        tab = TensorTable([p.data for _, p in named], self._be.optim_chunk_elems())
        tab.tensors = [p for _, p in named]          # track the Parameters: .data swaps change data_ptr()
        flat = torch.empty(tab.total, dtype=torch.float32, device=tab.device)
        views = tab.views(flat)
        for (n, p), v in zip(named, views):
            v.copy_(p.data if source is None else source[n])
        self._table, self.flat, self._names = tab, flat, [n for n, _ in named]
        self.shadow = dict(zip(self._names, views))

    def _is_flat(self):
        if self._table is None or list(self.shadow) != self._names:
            return False
        return all(self.shadow[n].data_ptr() == self.flat.data_ptr() + 4 * o
                   for n, o in zip(self._names, self._table.offsets_host))

    def covers(self, table):
        return self._is_flat() and len(table.tensors) == len(self._table.tensors) and \
            all(a is b for a, b in zip(table.tensors, self._table.tensors))

    # ---- reference interface ------------------------------------------------------------------------------
    def register(self, current_model):
        self._build(current_model)

    def reset_device(self, current_model):
        # the runner assigns `ema.shadow = checkpoint['ema']` (BaseRunner.py:125) and then calls this
        self._build(current_model, source=self.shadow)

    def update(self, current_model, with_decay=True):
        if not self._is_flat():
            self._build(current_model, source=self.shadow if self.shadow else None)
        self._table.refresh()
        self._be.ema_multi(self._table, self.flat, self.ema_decay, with_decay)

    def apply_shadow(self, current_model):
        for name, param in self._trainable(current_model):
            assert name in self.shadow
            self.backup[name] = param.data
            param.data = self.shadow[name]

    def restore(self, current_model):
        for name, param in self._trainable(current_model):
            assert name in self.backup
            param.data = self.backup[name]
        self.backup = {}
