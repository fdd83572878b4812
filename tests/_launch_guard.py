"""TEST-ONLY: a backend wrapper that runs every kernel launch on guarded, NaN-poisoned copies of its operands.

The launch shadow (tests/_launch_shadow.py) judges the values in the tensors a launch was handed.  Three ways a kernel can
be wrong lie outside those values: a store before, after or between the output views (into a pool neighbour the launch
does not read), a load outside the operand views (in a test that memory is usually fresh and zero, which is also the
padding value most kernels mean to produce), and an output element the launch never writes (torch.empty hands back a
reused block, which may hold the right value from an earlier run of the same computation).  ``Guard`` closes them.  It
sits between the shadow and the real backend, ``Shadow(Guard(backend))``, so the shadow keeps seeing, cloning and
checking the executor's own tensors (its Winograd chains are paired by their addresses), and for each launch

- groups the tensor arguments by overlapping byte ranges of the same storage (an in-place residual aliasing ``out`` and
  views of one buffer stay aliased), and gives each group a fresh buffer: the group's span with a guard zone before and
  after it (GUARD_MIN bytes at least, and the span itself up to GUARD_CAP), its base congruent to the original's modulo
  4096 so that no alignment-dependent path changes;
- fills the buffer with 0xFF bytes (NaN in fp32, fp16, bf16 and fp64, -1 in int32 / int64, 255 in uint8) and copies in
  the elements of every input view and of every exempt output view (EXEMPT), honouring strides: every byte no view
  covers, and every element of a pure output, is then NaN;
- runs the real launch on the relocated views, synchronises and reads the fault word, and then checks that
  (a) every byte outside the output views is bit-identical to its pre-launch state (guard zones, gaps inside the span,
      inputs): otherwise 'write before', 'write after' or 'write in gap';
  (b) no prefilled float output holds a NaN, and no int64 index output a -1: otherwise 'unwritten';
  (c) the launch did not set the fault word (the F(6,3) input transform sets it when it reads NaN into V): 'fault';
- copies the output views back into the executor's tensors, so that the run carries on and the shadow compares the
  values.  A load outside the views shows there as NaN, an infinite deviation of that launch.

Inside a CUDA-graph capture each launch passes through unguarded, as it does through the shadow: nothing may be
allocated, copied or synchronised there.  The TensorTable pointer arrays of adam_multi(_dev) / ema_multi are not
relocated (the parameters and gradients they point to are the model's own); their tensor arguments are, as in-out
tensors.

The canary helpers of the single-kernel tests (a tail of CANARY_N canary elements behind an output view) live here too.
"""
import collections
import functools
import inspect

import torch

from _launch_shadow import OUTPUTS, _capturing
from test_launch_trace_host import NOT_LAUNCHES

GUARD_MIN = 1 << 20          # larger than any kernel's output tile (the wgmma conv's 128 x 256 fp32 tile is 128 KiB)
GUARD_CAP = 64 << 20
ALIGN = 4096

# names of the backend that are not launches: they pass through unguarded
PASS_THROUGH = dict({n: "not a launch: sizes, geometry or allocation (test_launch_trace_host.py::NOT_LAUNCHES)"
                     for n in NOT_LAUNCHES},
                    check_fault="reads the device fault word; the guard calls it after every launch itself")

# (method, argument) -> why the output is relocated with its contents instead of being prefilled with NaN.  Writes
# outside an exempt output are still checked.  An exemption is never the answer to a finding.
WORKSPACE = "scratch the launch writes before it reads: its contents are not a result"
IN_OUT = "in-out: the launch reads the previous value and updates it"
EXEMPT = {
    ("gn_stats", "workspace"): WORKSPACE + " (cabi.CudaBackend.gn_stats passes it as the partial-sum buffer)",
    ("split_grad", "workspace"): WORKSPACE + " (the column-sum partials of cabi.CudaBackend.split_grad)",
    ("conv_wgrad", "workspace"): WORKSPACE + " (split-K partials sized by cabi.CudaBackend.wgrad_workspace)",
    ("conv_wgrad_direct", "workspace"): WORKSPACE + " (per-block partials, its size passed as workspace.numel())",
    ("gn_bwd_reduce", "ws"): WORKSPACE + " (per-block partials of cabi.CudaBackend.gn_bwd_reduce)",
    ("layernorm_bwd", "workspace"): WORKSPACE + " (cabi.layernorm_bwd_workspace(rows, C) floats)",
    ("adam_multi", "exp_avg"): IN_OUT, ("adam_multi", "exp_avg_sq"): IN_OUT, ("adam_multi", "ema_shadow"): IN_OUT,
    ("adam_multi_dev", "exp_avg"): IN_OUT, ("adam_multi_dev", "exp_avg_sq"): IN_OUT,
    ("adam_multi_dev", "ema_shadow"): IN_OUT,
    ("adam_multi_dev", "step"): IN_OUT + " (cabi.CudaBackend.adam_multi_dev: 'incremented here on the device')",
    ("ema_multi", "shadow"): IN_OUT + " (with_decay: shadow = decay * shadow + (1 - decay) * param)",
    # bbdm_b200/convs.py, WeightPacker.conv: "freshly allocated: the padding rows must be zeroed" (hi.zero_(),
    # lo.zero_()), then the packer writes rows :Cout of the [k*k, Cout_pad, Cin] planes (cabi.CudaBackend.pack_weight_split:
    # "padding rows pre-zeroed"); the shadow holds the padding rows to their pre-launch contents
    ("pack_weight_split", "hi"): "written in part by design: the Cout padding rows are zeroed by the caller",
    ("pack_weight_split", "lo"): "written in part by design: the Cout padding rows are zeroed by the caller",
}

Finding = collections.namedtuple("Finding", "launch method argument kind count offset")


# ------------------------------------------------------------------------------------------------ views and bytes
def extent(t):
    """[lo, hi) byte addresses of the elements of view t."""
    es = t.element_size()
    lo = hi = 0
    for s, st in zip(t.shape, t.stride()):
        if st >= 0:
            hi += (s - 1) * st
        else:
            lo += (s - 1) * st
    return t.data_ptr() + lo * es, t.data_ptr() + (hi + 1) * es


def distinct(t):
    """t with its stride-0 dimensions narrowed to one element: a view every element of which is a distinct location, so
    that it can be written (the broadcast elements are the same memory)."""
    for d, (s, st) in enumerate(zip(t.shape, t.stride())):
        if st == 0 and s > 1:
            t = t.narrow(d, 0, 1)
    return t


def byte_view(m, t, base):
    """The bytes of view t, which lies in a byte buffer at address base, as a view of m (a byte-per-byte map of that
    buffer): shape t.shape + (element size,)."""
    es = t.element_size()
    return torch.as_strided(m, tuple(t.shape) + (es,), tuple(s * es for s in t.stride()) + (1,), t.data_ptr() - base)


def _group(tensors):
    """{name: tensor} -> lists of names whose views overlap in bytes of the same storage (transitively)."""
    by_storage = collections.defaultdict(list)
    for k, t in tensors.items():
        by_storage[t.untyped_storage().data_ptr()].append((extent(t), k))
    groups = []
    for items in by_storage.values():
        items.sort()
        cur, hi = [], None
        for (lo, h), k in items:
            if cur and lo < hi:
                cur.append(k)
                hi = max(hi, h)
            else:
                if cur:
                    groups.append(cur)
                cur, hi = [k], h
        groups.append(cur)
    return groups


class _Relocated:
    """One group of aliasing views moved into a guarded buffer."""

    def __init__(self, names, a):
        ext = {k: extent(a[k]) for k in names}
        self.names = names
        self.lo = min(e[0] for e in ext.values())
        self.span = max(e[1] for e in ext.values()) - self.lo
        zone = max(GUARD_MIN, min(self.span, GUARD_CAP))
        dev = a[names[0]].device
        total = -(-(2 * zone + ALIGN + self.span) // 16) * 16
        self.buf = torch.empty(total, dtype=torch.uint8, device=dev)
        self.start = zone + (self.lo - self.buf.data_ptr() - zone) % ALIGN
        self.buf.fill_(0xFF)
        self.views = {}
        for k in names:
            t = a[k]
            es = t.element_size()
            off = self.start + (t.data_ptr() - self.lo)
            assert off % es == 0, (k, off, es)
            self.views[k] = torch.as_strided(self.buf.view(t.dtype), t.shape, t.stride(), off // es)
        self.ext = {k: (e[0] - self.lo + self.start, e[1] - self.lo + self.start) for k, e in ext.items()}


# ------------------------------------------------------------------------------------------------ the guard
class Guard:
    def __init__(self, be, exempt=None):
        """exempt: entries to add to EXEMPT (the CPU emulation's contract, which differs from the kernels')."""
        self.be = be
        self.exempt = {**EXEMPT, **(exempt or {})}
        self.findings = []
        self.launches = []
        self.bytes_guarded = 0

    def summary(self, title="guard"):
        kinds = collections.Counter(f.kind for f in self.findings)
        lines = [f"{title}: {len(self.launches)} launches guarded, {self.bytes_guarded / 2**20:.1f} MiB relocated, "
                 f"{len(self.findings)} findings" + (" (" + ", ".join(f"{k} {n}" for k, n in sorted(kinds.items())) + ")"
                                                      if kinds else "")]
        for f in self.findings[:40]:
            lines.append(f"  FINDING launch {f.launch} {f.method}.{f.argument}: {f.kind}, {f.count} elements/bytes, "
                         f"first at offset {f.offset}")
        return "\n".join(lines)

    def flagged(self):
        return sorted({f.launch for f in self.findings})

    def __getattr__(self, name):
        attr = getattr(self.be, name)
        if name in PASS_THROUGH or not callable(attr):
            return attr
        if name not in OUTPUTS:
            raise NotImplementedError(f"no output list for launch {name}")
        sig = inspect.signature(attr)

        @functools.wraps(attr)
        def launch(*args, **kwargs):
            if _capturing():
                return attr(*args, **kwargs)
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            a = bound.arguments
            tensors = {k: v for k, v in a.items() if isinstance(v, torch.Tensor) and v.numel()}
            outs = {k for k in OUTPUTS[name] if k in tensors}
            groups = [_Relocated(g, tensors) for g in _group(tensors)]
            new = {}
            for g in groups:
                self.bytes_guarded += g.buf.numel()
                for k in g.names:
                    if k not in outs or (name, k) in self.exempt:
                        distinct(g.views[k]).copy_(distinct(tensors[k]))
                new.update(g.views)
            snaps = [g.buf.clone() for g in groups]
            call = dict(a, **new)
            r = attr(**call)
            idx = len(self.launches)
            self.launches.append(name)
            dev = next(iter(tensors.values())).device if tensors else None
            if dev is not None and dev.type == "cuda":
                torch.cuda.synchronize(dev)
            try:
                self.be.check_fault()
            except Exception as e:         # noqa: BLE001 -- the fault word is a finding of this launch
                self.findings.append(Finding(idx, name, "", "fault", 1, str(e)[:200]))
            for g, snap in zip(groups, snaps):
                self._check_writes(idx, name, g, snap, outs)
            for k in sorted(outs):
                if (name, k) not in self.exempt:
                    self._check_written(idx, name, k, new[k])
            for k in outs:
                distinct(tensors[k]).copy_(distinct(new[k]))
            return r
        return launch

    def _check_writes(self, idx, name, g, snap, outs):
        changed = g.buf != snap
        for k in g.names:
            if k in outs:
                byte_view(changed, g.views[k], g.buf.data_ptr()).zero_()
        pos = changed.nonzero().flatten()
        if not pos.numel():
            return
        end = g.start + g.span
        first_k = min(g.names, key=lambda k: g.ext[k][0])
        last_k = max(g.names, key=lambda k: g.ext[k][1])
        before, after = pos[pos < g.start], pos[pos >= end]
        gap = pos[(pos >= g.start) & (pos < end)]
        if before.numel():
            self.findings.append(Finding(idx, name, first_k, "write before", before.numel(),
                                         int(before[0]) - g.ext[first_k][0]))
        if after.numel():
            self.findings.append(Finding(idx, name, last_k, "write after", after.numel(),
                                         int(after[0]) - g.ext[last_k][0]))
        if gap.numel():
            p = int(gap[0])
            k = next((k for k in g.names if g.ext[k][0] <= p < g.ext[k][1]), "/".join(g.names))
            self.findings.append(Finding(idx, name, k, "write in gap", gap.numel(),
                                         p - g.ext[k][0] if k in g.ext else p - g.start))

    def _check_written(self, idx, name, k, v):
        if v.is_floating_point():
            bad = torch.isnan(v)
        elif v.dtype == torch.int64:
            bad = v == -1
        else:
            return                        # uint8 / int32: the fill is a value the launch may write
        bad = bad.reshape(-1)
        if bool(bad.any()):
            self.findings.append(Finding(idx, name, k, "unwritten", int(bad.sum()), int(bad.nonzero()[0])))


# ------------------------------------------------------------------------------------------------ canary tails
CANARY = 1234.5
CANARY_N = 4096


def canaried(shape, dtype=torch.float32, device="cuda", fill=float("nan")):
    """(view of shape pre-filled with fill, whole buffer): CANARY_N canary elements sit right behind the view."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + CANARY_N,), fill, dtype=dtype, device=device)
    buf[n:] = CANARY
    return buf[:n].view(shape), buf


def tail_untouched(buf):
    return bool((buf[-CANARY_N:] == torch.tensor(CANARY, dtype=buf.dtype)).all())
