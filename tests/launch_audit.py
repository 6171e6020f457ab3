"""TEST INFRASTRUCTURE ONLY -- the model-independent part of the launch audits (test_gpu_denoiser_launches.py,
test_gpu_vae_launches.py): a tracer that wraps named ops of ln3diff_b200.ops and hands every launch to an auditor, the
auditor's dispatch and assertions, and the report.  A model's auditor subclasses `Audit` and defines one `do_<kind>`
method per step kind of its written-down launch sequence."""
from __future__ import annotations

import collections
import contextlib

import numpy as np
import torch

import kernel_bounds as kb

Step = collections.namedtuple("Step", "op kind layer")
# The attention bound carries the bf16 rounding of P, 2^-8 of sum p |v| / l, which under diffuse attention over
# hundreds of keys is a few percent of |y|: a wrong K/V source or grouping moves the output by 20-90x that bound, not
# 100x.  The attention kinds' separations take this factor.
FMHA_FACTOR = 20.0


def _desc(v):
    if isinstance(v, torch.Tensor):
        return f"{tuple(v.shape)}/{tuple(v.stride())}+{v.storage_offset()} {str(v.dtype)[6:]}"
    return repr(v) if not isinstance(v, (tuple, list)) else "(" + ", ".join(_desc(a) for a in v) + ")"


def _clone(v):
    if isinstance(v, tuple):
        return tuple(_clone(a) for a in v)
    return v.clone() if isinstance(v, torch.Tensor) else v


class Audit:
    """The expected launch sequence `seq` (a list of Step), the counters, the largest error / bound per step kind and
    the separation factor per check kind."""

    def __init__(self, seq):
        self.seq = seq
        self.n_traced = self.n_checked = 0
        self.ratio = collections.defaultdict(float)     # step kind -> max error / bound
        self.sep = {}                                   # check kind -> median slip / bound
        self.step = None
        self.args_desc = ""

    def fail_msg(self, what, got, ref, bound, bad):
        score = torch.where(bad, ((got - ref).abs() / bound.clamp_min(1e-300)).nan_to_num(float("inf")),
                            torch.zeros_like(ref))
        i = tuple(int(v) for v in np.unravel_index(int(score.flatten().argmax()), tuple(ref.shape)))
        s = self.step
        return (f"step {s.kind} layer {s.layer} ({what}): {int(bad.sum())} of {ref.numel()} elements out of bound; "
                f"worst at index {i}: got {got[i].item()!r} expected {ref[i].item()!r} bound {bound[i].item():.3e}; "
                f"launch args {self.args_desc}")

    def within(self, what, got, ref, bound):
        got = got.to(torch.float64)
        bound = bound.to(torch.float64).expand_as(ref)
        assert got.shape == ref.shape, (self.step, what, got.shape, ref.shape)
        err = (got - ref).abs()
        bad = ~(err <= bound)                        # NaN counts as out of bound
        if bool(bad.any()):
            raise AssertionError(self.fail_msg(what, got, ref, bound, bad))
        r = float((err / bound.clamp_min(1e-300)).max())
        key = self.step.kind
        self.ratio[key] = max(self.ratio[key], r)

    def separated(self, kind, ref, wrong, bound, affected=None, factor=100.0):
        if kind not in self.sep:
            self.sep[kind] = kb.assert_sensitive(f"{self.step.kind} layer {self.step.layer}: {kind}", ref, wrong,
                                                 bound, affected, factor)

    def launch(self, i, op, args, kw, ret):
        self.n_traced += 1
        assert i < len(self.seq), f"launch {i} ({op}) beyond the {len(self.seq)} expected launches"
        self.step = st = self.seq[i]
        assert op == st.op, f"launch {i}: expected {st.op} ({st.kind} layer {st.layer}), traced {op}"
        self.args_desc = ", ".join([_desc(a) for a in args] + [f"{k}={_desc(v)}" for k, v in kw.items()
                                                              if v is not None])
        getattr(self, "do_" + st.kind)(st.layer, args, kw, _clone(ret))
        self.n_checked += 1


@contextlib.contextmanager
def traced(audit, monkeypatch, names, slip=None):
    """Wraps the ops `names` of ln3diff_b200.ops; `slip` = (kind, layer, fn(args, kw) -> (args, kw)) rewrites the
    arguments of that one launch before it runs (a seeded host-side mapping error)."""
    from ln3diff_b200 import ops
    counter = [0]

    def wrap(name, fn):
        def w(*args, **kw):
            i = counter[0]
            counter[0] += 1
            st = audit.seq[i] if i < len(audit.seq) else None
            if slip is not None and st is not None and (st.kind, st.layer) == slip[:2]:
                args, kw = slip[2](list(args), dict(kw))
            ret = fn(*args, **kw)
            audit.launch(i, name, args, kw, ret)
            return ret
        return w

    with monkeypatch.context() as mp:
        for name in names:
            mp.setattr(ops, name, wrap(name, getattr(ops, name)))
        yield
    assert counter[0] == len(audit.seq), f"traced {counter[0]} launches, expected {len(audit.seq)}"


def _report(audit, what):
    print(f"\n{what}: {len(audit.seq)} launches checked; max error / bound per step:")
    for k in sorted(audit.ratio):
        print(f"    {k:24s} {audit.ratio[k]:.3e}")
    print("  separation (median slip / bound): " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(audit.sep.items())))
