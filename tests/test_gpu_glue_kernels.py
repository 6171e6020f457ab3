"""GPU (-m gpu): the fp32 glue kernels of elementwise.cu (norm_modulate, final_layer, patch_embed,
timestep_embedding, sampler_affine_update) element by element against float64 references, on every dispatch path.

The references follow each kernel's order of operations, so every tolerance is derived from the arithmetic and
written beside its assert.  Every output view sits inside a buffer filled with a NaN bit pattern: bytes outside
the view must keep their bits, and an input read outside its view turns the result into NaN.  Each test also
recomputes its reference with one index mapping deliberately wrong (the neighbouring sample's gate or modulation
row, resid_rows shifted by one sample, p and q swapped, pos_embed off by one token, the neighbouring plane) and
asserts that the slip moves the affected elements by >= 100x the tolerance: the data can tell them apart."""
import zlib

import numpy as np
import pytest
import torch

from kernel_bounds import assert_sensitive, bf16_bound, nm_out_ref, nm_resid_ref, timestep_embedding_ref, ulp_bf16, \
    ulp_f32
from kernel_bounds import f32 as _f32
from kernel_bounds import final_layer_ref as _final_layer_ref
from kernel_bounds import patch_embed_ref as _patch_ref

pytestmark = pytest.mark.gpu

NAN_PAD = 64          # elements of NaN before and after every guarded view: 256 B of fp32 keeps 32-byte alignment


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


# ------------------------------------------------------------------ helpers
def assert_within(what: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> None:
    got = got.detach().cpu().to(torch.float64)
    ref, bound = ref.to(torch.float64), bound.to(torch.float64).expand_as(ref)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = (got - ref).abs()
    bad = ~(err <= bound)                         # NaN counts as out of bound
    if bool(bad.any()):
        score = torch.where(bad, (err / bound.clamp_min(1e-300)).nan_to_num(float("inf")), torch.zeros_like(err))
        idx = tuple(int(i) for i in np.unravel_index(int(score.flatten().argmax()), tuple(got.shape)))
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} elements out of bound; worst at index {idx}: "
                             f"got {got[idx].item()!r} expected {ref[idx].item()!r} bound {bound[idx].item():.3e}")


class Guarded:
    """A device view of `values` inside a larger buffer filled with a NaN bit pattern.  `ld` (2-D only) sets the
    row pitch, so the gaps between rows are NaN as well.  check() asserts that no element outside `region`
    (default: the whole view) changed its bits -- compared as integers, because NaN != NaN."""

    def __init__(self, values: torch.Tensor, dev, ld: int | None = None):
        shape = tuple(values.shape)
        if ld is not None:
            assert len(shape) == 2 and ld >= shape[1]
            strides, span = (ld, 1), shape[0] * ld
        else:
            strides, span = torch.empty(shape, device="meta").stride(), values.numel()
        flat = torch.full((2 * NAN_PAD + span,), float("nan"), dtype=values.dtype)
        flat.as_strided(shape, strides, NAN_PAD).copy_(values)
        self._bits = torch.int32 if values.dtype == torch.float32 else torch.int16
        self._before = flat.view(self._bits).clone()
        self.flat = flat.to(dev)
        self.view = self.flat.as_strided(shape, strides, NAN_PAD)

    def check(self, what: str, region: torch.Tensor | None = None) -> None:
        region = self.view if region is None else region
        inside = torch.zeros(self.flat.numel(), dtype=torch.bool)
        inside.as_strided(tuple(region.shape), region.stride(),
                          region.storage_offset() - self.flat.storage_offset()).fill_(True)
        now = self.flat.cpu().view(self._bits)
        changed = (now != self._before) & ~inside
        assert not bool(changed.any()), \
            f"{what}: {int(changed.sum())} elements outside the view were written (first at flat index " \
            f"{int(torch.nonzero(changed)[0])})"


def _dev64(t: torch.Tensor) -> torch.Tensor:
    return t.detach().cpu().to(torch.float64)


# ------------------------------------------------------------------ norm_modulate: reference (kernel_bounds.py)
def check_x(what, got, ref):
    """fp32 residual stream: at most 1 ulp (double-rounding ties only), and bit-exact almost everywhere."""
    assert_within(what, got, ref, ulp_f32(ref))
    exact = float((got.cpu().double() == ref).double().mean())
    assert exact >= 0.99, f"{what}: only {exact:.4f} of the elements are bit-exact"


# ------------------------------------------------------------------ norm_modulate: cases
# id: (D, rows, ldx, norm, eps, act, mod, mod_rows, tables, weight, resid, gate_rows, want_out)
#   mod   None | "table" (a column slice of a (G, 14 D) table: mod_ld > D) | "plain" ((G, D) tensors: mod_ld = D)
#         | "stride0" (mod_row.expand: mod_ld = 0)
#   resid None | "plain" (ungated) | "gated" (a column slice of a (G, 6 D) gate table) | "gate0" (stride-0 gate)
# Kernel: D % 256 == 0, D <= 1536, ldx % 8 == 0 -> norm_modulate_wide_kernel; otherwise norm_modulate_kernel.
L, R, N = 1, 2, 0
NM_CASES = {
    "dit-ln1-1024": (1024, 2 * 768 + 5, None, L, 1e-6, 0, "table", 768, False, False, "gated", 768, True),
    "dit-ln1-1024-ldx+4": (1024, 2 * 768 + 5, 1028, L, 1e-6, 0, "table", 768, False, False, "gated", 768, True),
    "dit-xb-768": (768, 2 * 768 + 5, None, N, 0, 0, None, 0, False, False, "gated", 768, True),
    "dit-xb-768-ldx+4": (768, 2 * 768 + 5, 772, N, 0, 0, None, 0, False, False, "gated", 768, True),
    "pixart-rms-1152-tables": (1152, 2 * 768 + 5, None, R, 1e-5, 0, "table", 768, True, True, "gated", 768, True),
    "pixart-rms-768-tables": (768, 300, None, R, 1e-5, 0, "table", 100, True, True, None, 0, True),
    "ln-1024-3groups": (1024, 300, None, L, 1e-6, 0, "table", 100, False, False, None, 0, True),
    "tower-ln-1024": (1024, 77, None, L, 1e-5, 0, "plain", 77, False, False, "gated", 77, True),
    "tower-ln-384": (384, 77, None, L, 1e-5, 0, "plain", 77, False, False, "gated", 77, True),
    "vit-rowmod-384": (384, 300, None, L, 1e-6, 0, "table", 1, False, False, "gated", 1, True),
    "vit-rowmod-768": (768, 300, None, L, 1e-6, 0, "table", 1, False, False, "gated", 1, True),
    "stride0-768": (768, 2 * 768 + 5, None, L, 1e-6, 0, "stride0", 768, False, False, "gate0", 768, True),
    "stride0-2048": (2048, 2 * 768 + 5, None, L, 1e-6, 0, "stride0", 768, False, False, "gate0", 768, True),
    "gate-rows-differ-1152": (1152, 300, None, L, 1e-6, 0, "table", 100, False, False, "gated", 77, True),
    "gate-rows-differ-1536": (1536, 300, None, L, 1e-6, 0, "table", 100, False, False, "gated", 77, True),
    "resid-only-1024-16x768": (1024, 16 * 768, None, N, 0, 0, None, 0, False, False, "gated", 768, False),
    "ln-ungated-1024-16x768": (1024, 16 * 768, None, L, 1e-6, 0, "table", 768, False, False, "plain", 0, True),
    "resid-only-1792": (1792, 300, None, N, 0, 0, None, 0, False, False, "gated", 100, False),
    "ungated-384": (384, 77, None, N, 0, 0, None, 0, False, False, "plain", 0, True),
    "silu-128": (128, 1, None, N, 0, 3, None, 0, False, False, None, 0, True),
    "silu-768": (768, 77, None, N, 0, 3, None, 0, False, False, None, 0, True),
    "gelu-erf-1792": (1792, 77, None, N, 0, 1, None, 0, False, False, None, 0, True),
    "gelu-tanh-1536": (1536, 300, None, N, 0, 2, None, 0, False, False, None, 0, True),
    "cast-768": (768, 77, None, N, 0, 0, None, 0, False, False, None, 0, True),
    "rms-768": (768, 77, None, R, 1e-5, 0, None, 0, False, True, None, 0, True),
    "rms-2048": (2048, 300, None, R, 1e-5, 0, None, 0, False, True, None, 0, True),
    "ln-1e-5-onegroup-1152": (1152, 5, None, L, 1e-5, 0, "plain", 5, False, False, None, 0, True),
    "ln-tables-1024-ldx+4": (1024, 2 * 768 + 5, 1028, L, 1e-6, 0, "table", 768, True, False, "gated", 768, True),
}


def _nm_inputs(g, D, rows, mod, mod_rows, tables, weight, resid, gate_rows):
    """Distinct values per sample: every gate / modulation row is its own random draw."""
    inp = dict(x=torch.randn(rows, D, generator=g) * 2 + 0.5)
    if mod is not None:
        G = -(-rows // mod_rows)
        if mod == "table":
            inp["mod"] = torch.randn(G, 14 * D, generator=g)
        elif mod == "plain":
            inp["shift"], inp["scale"] = torch.randn(G, D, generator=g), torch.randn(G, D, generator=g)
        else:
            inp["mod"] = torch.randn(1, 14 * D, generator=g)
    if tables:
        inp["shift_tab"], inp["scale_tab"] = torch.randn(D, generator=g) * 0.5, torch.randn(D, generator=g) * 0.5
    if weight:
        inp["weight"] = torch.randn(D, generator=g)
    if resid is not None:
        inp["resid"] = (torch.randn(rows, D, generator=g) * 3).bfloat16()
        if resid in ("gated", "gate0"):
            inp["gate"] = torch.randn(-(-rows // gate_rows) if resid == "gated" else 1, 6 * D, generator=g)
    return inp


@pytest.mark.parametrize("case", list(NM_CASES))
def test_norm_modulate(dev, case):
    from ln3diff_b200 import ops
    D, rows, ldx, norm, eps, act, mod, mod_rows, tables, weight, resid, gate_rows, want_out = NM_CASES[case]
    g = torch.Generator().manual_seed(zlib.crc32(case.encode()))
    inp = _nm_inputs(g, D, rows, mod, mod_rows, tables, weight, resid, gate_rows)
    x = Guarded(inp["x"], dev, ld=ldx)
    kw = dict(norm=norm, eps=eps, act=act)
    idx = torch.arange(rows)
    ref = {k: v.to(torch.float64) for k, v in inp.items()}
    guards = []
    if mod is not None:
        if "mod" in inp:
            m = Guarded(inp["mod"], dev)
            mv = m.view.expand(rows // mod_rows + 1, 14 * D) if mod == "stride0" else m.view
            kw.update(shift=mv[:, 3 * D:4 * D], scale=mv[:, 4 * D:5 * D])
            sh64, sc64 = ref["mod"][:, 3 * D:4 * D], ref["mod"][:, 4 * D:5 * D]
            mod_idx = idx // mod_rows if mod != "stride0" else torch.zeros(rows, dtype=torch.long)
        else:
            kw.update(shift=Guarded(inp["shift"], dev).view, scale=Guarded(inp["scale"], dev).view)
            sh64, sc64, mod_idx = ref["shift"], ref["scale"], idx // mod_rows
        kw["mod_rows"] = mod_rows
        if mod == "stride0":
            assert kw["shift"].stride(0) == 0
    if tables:
        kw.update(shift_tab=Guarded(inp["shift_tab"], dev).view, scale_tab=Guarded(inp["scale_tab"], dev).view)
    if weight:
        kw["weight"] = Guarded(inp["weight"], dev).view
    gate64 = gate_idx = None
    if resid is not None:
        kw["resid"] = Guarded(inp["resid"], dev).view
        if resid in ("gated", "gate0"):
            gt = Guarded(inp["gate"], dev)
            gv = gt.view if resid == "gated" else gt.view.expand(rows // gate_rows + 1, 6 * D)
            kw.update(resid_gate=gv[:, 5 * D:6 * D], resid_gate_rows=gate_rows)
            gate64 = ref["gate"][:, 5 * D:6 * D]
            gate_idx = idx // gate_rows if resid == "gated" else torch.zeros(rows, dtype=torch.long)
    out = None
    if want_out:
        out = Guarded(torch.zeros(rows, D, dtype=torch.bfloat16), dev)
        kw["out"] = out.view
    else:
        kw["want_out"] = False

    ops.norm_modulate(x.view, **kw)
    torch.cuda.synchronize()
    x.check(f"{case}: x")
    x_new = _dev64(x.view)

    # residual stream: the kernel's fmaf chain, <= 1 ulp
    x_ref = nm_resid_ref(ref["x"], ref.get("resid"), gate64, gate_idx)
    check_x(f"{case}: residual stream x", x_new, x_ref)
    if gate64 is not None and resid == "gated" and gate64.shape[0] > 1:
        wrong = nm_resid_ref(ref["x"], ref["resid"], gate64, (gate_idx + 1) % gate64.shape[0])
        assert_sensitive(f"{case}: neighbouring gate row", x_ref, wrong, ulp_f32(x_ref))

    if want_out:
        out.check(f"{case}: out")
        mk = dict(weight=ref.get("weight"), shift_tab=ref.get("shift_tab"), scale_tab=ref.get("scale_tab"))
        if mod is not None:
            mk.update(shift=sh64, scale=sc64, mod_idx=mod_idx)
        y, tau = nm_out_ref(x_new, norm, eps, act, **mk)       # from the kernel's own updated x
        bound = bf16_bound(y, tau)
        assert_within(f"{case}: bf16 out", out.view, y, bound)
        if mod is not None and sh64.shape[0] > 1 and mod != "stride0":
            mk["mod_idx"] = (mod_idx + 1) % sh64.shape[0]
            assert_sensitive(f"{case}: neighbouring modulation group", y, nm_out_ref(x_new, norm, eps, act, **mk)[0], bound)


# ------------------------------------------------------------------ norm_modulate: closed-form CFG rows
T_TOK, B_CF = 768, 4


@pytest.mark.parametrize("D,norm", [(1024, L), (1152, R)], ids=["dit-1024-wide", "pixart-1152-float4"])
@pytest.mark.parametrize("rr", [(2, 4), (0, 2), (0, 4), (0, 0)], ids=lambda r: f"rows{r[0]}T-{r[1]}T")
@pytest.mark.parametrize("out_gate", [False, True], ids=["bcast", "bcast+out_gate"])
def test_norm_modulate_closed_form_rows(dev, D, norm, rr, out_gate):
    """The pass after the cross-attention: rows in resid_rows add their own attention row, the others the per-sample
    broadcast row (identical context tokens) and, with resid_out_gate, first their own gate_msa * attn row."""
    from ln3diff_b200 import ops
    T, B = T_TOK, B_CF
    rows = B * T
    r0, r1 = rr[0] * T, rr[1] * T
    g = torch.Generator().manual_seed(1000 * D + 10 * rr[0] + rr[1] + out_gate)
    x0 = torch.randn(rows, D, generator=g) * 2 + 0.5
    mod = torch.randn(B, 14 * D, generator=g)
    val = (torch.randn(rows, D, generator=g) * 3).bfloat16()
    oc = (torch.randn(B, D, generator=g) * 3).bfloat16()
    w = torch.randn(D, generator=g) if norm == R else None
    x, m, vg, og = Guarded(x0, dev), Guarded(mod, dev), Guarded(val, dev), Guarded(oc, dev)
    out = Guarded(torch.zeros(rows, D, dtype=torch.bfloat16), dev)
    sl = lambda t, j: t[:, j * D:(j + 1) * D]
    kw = dict(norm=norm, eps=1e-6 if norm == L else 1e-5, shift=sl(m.view, 3), scale=sl(m.view, 4), mod_rows=T,
              out=out.view, resid=vg.view, resid_bcast=og.view, resid_bcast_rows=T, resid_rows=(r0, r1))
    if w is not None:
        kw["weight"] = Guarded(w, dev).view
    if out_gate:
        kw.update(resid_out_gate=sl(m.view, 2), resid_out_gate_rows=T)
    ops.norm_modulate(x.view, **kw)
    torch.cuda.synchronize()
    x.check("x")
    out.check("out")

    idx = torch.arange(rows)
    m64 = mod.double()
    rk = dict(resid=val.double(), gate=None, gate_idx=None, bcast=oc.double(), bcast_idx=idx // T,
              ogate=sl(m64, 2) if out_gate else None, ogate_idx=idx // T)
    inside = (idx >= r0) & (idx < r1)
    x_ref = nm_resid_ref(x0.double(), inside=inside, **rk)
    x_new = _dev64(x.view)
    check_x("residual stream x", x_new, x_ref)
    # resid_rows shifted by one sample (or, when that changes nothing, widened by one)
    wr = (min(r0 + T, rows), min(r1 + T, rows))
    if wr == (r0, r1) or (r1 == r0 and wr[0] == wr[1]):
        wr = (r0, min(r1 + T, rows)) if r1 < rows else (r0 + T, r1)
    inside_w = (idx >= wr[0]) & (idx < wr[1])
    assert_sensitive("resid_rows shifted by one sample", x_ref, nm_resid_ref(x0.double(), inside=inside_w, **rk),
                     ulp_f32(x_ref), (inside_w != inside)[:, None])
    if out_gate and r1 - r0 < rows:
        rk_w = dict(rk, ogate_idx=(idx // T + 1) % B)
        assert_sensitive("neighbouring resid_out_gate row", x_ref, nm_resid_ref(x0.double(), inside=inside, **rk_w),
                         ulp_f32(x_ref), (~inside)[:, None])
    rk_b = dict(rk, bcast_idx=(idx // T + 1) % B)
    if r1 - r0 < rows:
        assert_sensitive("neighbouring broadcast row", x_ref, nm_resid_ref(x0.double(), inside=inside, **rk_b),
                         ulp_f32(x_ref), (~inside)[:, None])

    y, tau = nm_out_ref(x_new, norm, kw["eps"], 0, weight=w.double() if w is not None else None,
                        shift=sl(m64, 3), scale=sl(m64, 4), mod_idx=idx // T)
    bound = bf16_bound(y, tau)
    assert_within("bf16 out", out.view, y, bound)


@pytest.mark.parametrize("D", [1024, 1152], ids=["wide", "float4"])
@pytest.mark.parametrize("g0,g1", [(2, 4), (0, 2), (1, 3)])
def test_norm_modulate_split_pass_row_slice(dev, D, g0, g1):
    """x2[r0:r1] += sl(2)[g0:g1] (per sample) * val[r0:r1], xb[r0:r1] = bf16(x): a row-slice view with a sliced gate;
    nothing outside the slice may change."""
    from ln3diff_b200 import ops
    T, B = T_TOK, B_CF
    rows, r0, r1 = B * T, g0 * T, g1 * T
    g = torch.Generator().manual_seed(7 * D + g0 + 10 * g1)
    x0 = torch.randn(rows, D, generator=g) * 2 + 0.5
    mod = torch.randn(B, 14 * D, generator=g)
    val = (torch.randn(rows, D, generator=g) * 3).bfloat16()
    x, m, vg = Guarded(x0, dev), Guarded(mod, dev), Guarded(val, dev)
    xb = Guarded(torch.zeros(rows, D, dtype=torch.bfloat16), dev)
    gate = m.view[:, 2 * D:3 * D][g0:g1]
    ops.norm_modulate(x.view[r0:r1], norm=N, out=xb.view[r0:r1], resid=vg.view[r0:r1], resid_gate=gate,
                      resid_gate_rows=T)
    torch.cuda.synchronize()
    x.check("x", x.view[r0:r1])
    xb.check("xb", xb.view[r0:r1])
    loc = torch.arange(r1 - r0)
    gate64 = mod.double()[g0:g1, 2 * D:3 * D]
    x_ref = nm_resid_ref(x0.double()[r0:r1], val.double()[r0:r1], gate64, loc // T)
    x_new = _dev64(x.view[r0:r1])
    check_x("residual stream x[r0:r1]", x_new, x_ref)
    wrong = nm_resid_ref(x0.double()[r0:r1], val.double()[r0:r1], mod.double()[:, 2 * D:3 * D], (g0 + loc // T + 1) % B)
    assert_sensitive("gate row of the neighbouring sample", x_ref, wrong, ulp_f32(x_ref))
    assert_within("bf16 xb[r0:r1]", xb.view[r0:r1], x_new, ulp_bf16(x_new) / 2)   # a plain rounding: tau = 0


# ------------------------------------------------------------------ final_layer
FL_CASES = {  # id: (D, Cout, S, B, tables, bias)
    "pair-768-S32-B2": (768, 4, 32, 2, False, True),
    "pair-768-S32-B1": (768, 4, 32, 1, False, True),
    "pair-768-S6-B3": (768, 4, 6, 3, True, True),
    "pair-768-S2-B16": (768, 4, 2, 16, False, False),
    "pair-1024-S6-B1": (1024, 4, 6, 1, False, True),
    "pair-1024-S6-B16": (1024, 4, 6, 16, True, False),
    "pair-1024-S2-B3": (1024, 4, 2, 3, False, True),
    "pair-1024-S32-B3": (1024, 4, 32, 3, True, True),
    "one-512-C1": (512, 1, 6, 3, False, True),
    "one-512-C8": (512, 8, 2, 16, True, True),
    "one-1152-C3": (1152, 3, 6, 3, True, True),
    "one-1152-C4": (1152, 4, 32, 2, True, True),
    "one-2048-C8": (2048, 8, 6, 3, False, False),
    "one-2048-C1": (2048, 1, 2, 16, True, True),
}


@pytest.mark.parametrize("case", list(FL_CASES))
def test_final_layer(dev, case):
    from ln3diff_b200 import ops
    D, Cout, S, B, tables, with_bias = FL_CASES[case]
    T = 3 * (S // 2) ** 2
    g = torch.Generator().manual_seed(zlib.crc32(case.encode()))
    x0 = torch.randn(B, T, D, generator=g) * 2 + 0.5
    W = torch.randn(4 * Cout, D, generator=g) * 0.05
    bias = torch.randn(4 * Cout, generator=g) if with_bias else None
    xg, wg = Guarded(x0, dev), Guarded(W, dev)
    out = Guarded(torch.zeros(B, 3 * Cout, S, S), dev)
    kw = dict(out=out.view)
    if tables:
        # the PixArt call: shift and scale are the same (B, D) tensor, the tables carry the difference
        t = torch.randn(B, D, generator=g)
        tabs = torch.randn(2, D, generator=g)
        tg = Guarded(t, dev)
        shift_d = scale_d = tg.view
        kw.update(shift_tab=Guarded(tabs[0], dev).view, scale_tab=Guarded(tabs[1], dev).view)
        sh64 = sc64 = t.double()
        tab64 = dict(shift_tab=tabs[0].double(), scale_tab=tabs[1].double())
    else:
        mod = torch.randn(B, 14 * D, generator=g)       # (B, (6L+2) D): the final layer's pair sits at 12 D
        mg = Guarded(mod, dev)
        shift_d, scale_d = mg.view[:, 12 * D:13 * D], mg.view[:, 13 * D:14 * D]
        sh64, sc64 = mod.double()[:, 12 * D:13 * D], mod.double()[:, 13 * D:14 * D]
        tab64 = {}
    ops.final_layer(xg.view, shift_d, scale_d, wg.view, Guarded(bias, dev).view if bias is not None else None, S, **kw)
    torch.cuda.synchronize()
    out.check(f"{case}: out")
    b64 = bias.double() if bias is not None else None
    ref, bound = _final_layer_ref(x0.double(), sh64, sc64, W.double(), b64, S, Cout, **tab64)
    assert_within(f"{case}: out", out.view, ref, bound)
    wrong, _ = _final_layer_ref(x0.double(), sh64, sc64, W.double(), b64, S, Cout, swap_pq=True, **tab64)
    pq = torch.zeros(1, 1, S, S, dtype=torch.bool)
    pq[..., 0::2, 1::2] = True
    pq[..., 1::2, 0::2] = True                                 # p != q: the elements the swap moves
    assert_sensitive(f"{case}: unpatchify p and q swapped", ref, wrong, bound, pq)
    if B > 1:
        wrong, _ = _final_layer_ref(x0.double(), sh64.roll(1, 0), sc64.roll(1, 0), W.double(), b64, S, Cout, **tab64)
        assert_sensitive(f"{case}: neighbouring sample's modulation", ref, wrong, bound)


def test_final_layer_rejects_unpaired_or_malformed_tables(dev):
    from ln3diff_b200 import ops
    x = torch.zeros(1, 3 * 16 ** 2, 768, device=dev)
    s, w = torch.zeros(1, 768, device=dev), torch.zeros(16, 768, device=dev)
    tab = torch.zeros(768, device=dev)
    with pytest.raises(ValueError, match="together"):
        ops.final_layer(x, s, s, w, None, 32, shift_tab=tab)
    with pytest.raises(ValueError, match="contiguous"):
        ops.final_layer(x, s, s, w, None, 32, shift_tab=torch.zeros(2, 768, device=dev)[:, 0], scale_tab=tab)
    with pytest.raises(ValueError, match="float32"):
        ops.final_layer(x, s, s, w, None, 32, shift_tab=tab.double(), scale_tab=tab)


# ------------------------------------------------------------------ patch_embed
PE_CASES = {  # id: (Cin, D, S, B, in_scale, bias, pos)     Cin = 4 and D % 4 == 0 -> patch_embed_k16_kernel
    "k16-S32-B2": (4, 768, 32, 2, False, True, True),
    "k16-S6-B5-scale": (4, 768, 6, 5, True, True, True),
    "k16-S10-B2-scale-nobias": (4, 768, 10, 2, True, False, True),
    "k16-S10-B1-scale-nopos": (4, 1152, 10, 1, True, True, False),
    "k16-S6-B2-1024": (4, 1024, 6, 2, True, True, True),
    "generic-Cin1": (1, 768, 6, 3, True, True, True),
    "generic-Cin3": (3, 768, 10, 2, True, True, False),
    "generic-Cin12": (12, 512, 6, 2, True, False, True),
    "generic-Cin16": (16, 1024, 6, 3, True, True, True),
    "generic-Cin4-D130": (4, 130, 10, 5, True, True, True),
}


@pytest.mark.parametrize("case", list(PE_CASES))
def test_patch_embed(dev, case):
    from ln3diff_b200 import ops
    Cin, D, S, B, with_scale, with_bias, with_pos = PE_CASES[case]
    T = 3 * (S // 2) ** 2
    g = torch.Generator().manual_seed(zlib.crc32(case.encode()))
    x = torch.randn(B, 3 * Cin, S, S, generator=g)
    W = torch.randn(D, Cin, 2, 2, generator=g)
    bias = torch.randn(D, generator=g) if with_bias else None
    pos = torch.randn(T, D, generator=g) if with_pos else None
    # distinct per sample, one of them 0
    in_scale = torch.tensor([0.0, 1.7, -0.3, 0.05, 2.5][:B]) if with_scale else None
    if in_scale is not None and B == 1:
        in_scale = torch.tensor([0.61])
    out = Guarded(torch.zeros(B, T, D), dev)
    dv = lambda t: Guarded(t, dev).view if t is not None else None
    ops.patch_embed(dv(x), dv(W), dv(bias), dv(pos), in_scale=dv(in_scale), out=out.view)
    torch.cuda.synchronize()
    out.check(f"{case}: tokens")
    a = dict(x=x.double(), in_scale=in_scale.double() if in_scale is not None else None, W=W.double(),
             bias=bias.double() if bias is not None else None, pos=pos.double() if pos is not None else None)
    ref, bound = _patch_ref(**a)
    assert_within(f"{case}: tokens", out.view, ref, bound)
    if pos is not None:
        assert_sensitive(f"{case}: pos_embed off by one token", ref, _patch_ref(**a, roll_pos=True)[0], bound)
    live = torch.ones(B, 1, 1, dtype=torch.bool) if in_scale is None else (in_scale != 0)[:, None, None]
    assert_sensitive(f"{case}: patch of the neighbouring plane", ref, _patch_ref(**a, roll_plane=True)[0], bound,
                     live.expand(B, T, 1))
    if in_scale is not None and B > 1:
        assert_sensitive(f"{case}: neighbouring sample's in_scale", ref, _patch_ref(**a, roll_scale=True)[0], bound)


# ------------------------------------------------------------------ timestep embedding
def _edm_c_noise(n=250, smin=0.002, smax=80.0, rho=7.0):
    """c_noise = ln(sigma) / 4 along a 250-step EDM (Karras) schedule: fractional and negative timesteps."""
    i = torch.arange(n, dtype=torch.float64)
    sig = (smax ** (1 / rho) + i / (n - 1) * (smin ** (1 / rho) - smax ** (1 / rho))) ** rho
    return (0.25 * sig.log()).float()


@pytest.mark.parametrize("B", [1, 5, 2048])
def test_timestep_embedding(dev, B):
    from ln3diff_b200 import ops
    special = torch.tensor([0.0, 1e-3, 0.37, 1.0, 17.0, 500.5, 999.0, 1000.0])
    if B == 1:
        t = torch.tensor([0.37])
    elif B == 5:
        t = torch.tensor([0.0, 1e-3, 17.0, 999.0, 1000.0])
    else:
        g = torch.Generator().manual_seed(B)
        t = torch.cat([special, _edm_c_noise(), torch.rand(B - 258, generator=g) * 1000])
    out = Guarded(torch.zeros(B, 256, dtype=torch.bfloat16), dev)
    ops.timestep_embedding(Guarded(t, dev).view, out=out.view)
    torch.cuda.synchronize()
    out.check("embedding")
    ref, bound = timestep_embedding_ref(t)
    assert_within(f"B={B}: [cos | sin]", out.view, ref, bound)
    if B > 1:
        wrong = timestep_embedding_ref(t.roll(1, 0))[0]
        assert_sensitive("neighbouring sample's t", ref, wrong, bound, (t != t.roll(1, 0))[:, None])
    assert_sensitive("cos and sin halves swapped", ref, ref.roll(128, 1), bound)


# ------------------------------------------------------------------ sampler update
def _sampler_ref(x, coef, m0, m1, noise):
    """x' = fmaf(s, noise, fmaf(w1, m1, fmaf(w0, m0, a * x))) in the kernel's order: each product is exact in
    float64, every step is rounded to fp32 (<= 1 ulp from a double-rounding tie)."""
    c = coef.reshape(coef.shape[0], *([1] * (x.dim() - 1)), 4)
    r = _f32(c[..., 0] * x)
    r = _f32(r + c[..., 1] * m0)
    if m1 is not None:
        r = _f32(r + c[..., 2] * m1)
    if noise is not None:
        r = _f32(r + c[..., 3] * noise)
    return r


@pytest.mark.parametrize("B,shape,m1,noise,alias", [
    (3, (12, 32, 32), True, True, False),
    (3, (12, 32, 32), False, False, False),
    (1, (12, 32, 32), True, False, True),
    (16, (12, 32, 32), True, True, True),
    (16, (12, 32, 32), False, True, False),
    (2, (2 ** 22 + 4,), True, True, False),      # grid-stride loop: 4 full passes and a partial fifth
    (2, (2 ** 22 + 4,), False, False, True),
], ids=["B3", "B3-m0only", "B1-m1-alias", "B16-alias", "B16-noise", "B2-4M", "B2-4M-m0only-alias"])
def test_sampler_affine_update(dev, B, shape, m1, noise, alias):
    from ln3diff_b200 import ops
    g = torch.Generator().manual_seed(B * 31 + len(shape) + 2 * m1 + noise)
    x0, a0, a1, nz = (torch.randn(B, *shape, generator=g) for _ in range(4))
    # per sample: zeros, negatives and the CFG pair (1 - 6.5, 6.5)
    pool = torch.tensor([[0.97, -5.5, 6.5, 0.013], [1.0, 0.0, -0.25, 0.0], [-0.5, 1.5, 0.0, -1.25],
                         [0.0, 2.0, -3.0, 0.5]])
    coef = pool[torch.arange(B) % 4] + 0.01 * torch.arange(B, dtype=torch.float32)[:, None] * (pool[torch.arange(B) % 4] != 0)
    x = Guarded(x0, dev)
    dv = lambda t: Guarded(t, dev).view
    out = x if alias else Guarded(torch.zeros_like(x0), dev)
    ops.sampler_affine_update(x.view, dv(coef), dv(a0), dv(a1) if m1 else None, dv(nz) if noise else None, out=out.view)
    torch.cuda.synchronize()
    out.check("x_out")
    if not alias:
        x.check("x")
        assert torch.equal(x.view.cpu(), x0), "x changed although out is a separate buffer"
    ref = _sampler_ref(x0.double(), coef.double(), a0.double(), a1.double() if m1 else None,
                       nz.double() if noise else None)
    check_x("x_out", _dev64(out.view), ref)
    if B > 1:
        wrong = _sampler_ref(x0.double(), coef.double().roll(1, 0), a0.double(), a1.double() if m1 else None,
                             nz.double() if noise else None)
        diff = (coef != coef.roll(1, 0)).any(1)
        assert_sensitive("neighbouring sample's coefficients", ref, wrong, ulp_f32(ref),
                         diff.reshape(B, *([1] * len(shape))))


# ------------------------------------------------------------------ dispatch coverage
def test_every_glue_kernel_path_runs(dev):
    """One call per intended dispatch path under torch.profiler: if the dispatch changes, this names the path
    that lost its element-wise coverage above.

    The calls run once in a warm-up cycle of the profiler's schedule and are recorded in the cycle after it.  Late in
    a long pytest process that has already run other profiling sessions, a single unscheduled window lost the activity
    records of its first kernel, or of all of them, although every kernel ran; the warm-up cycle starts CUPTI's
    activity recording before the recorded calls.  Every kind must still appear in the recorded cycle."""
    from torch.profiler import ProfilerActivity, profile, schedule

    from ln3diff_b200 import ops
    z = lambda *s: torch.randn(*s, device=dev)

    def calls():
        ops.norm_modulate(z(77, 1024), norm=L)                                     # wide
        ops.norm_modulate(z(77, 1028)[:, :1024], norm=L)                           # ldx = D + 4: float4
        ops.norm_modulate(z(77, 1152), norm=L)                                     # D % 256 != 0: float4
        ops.final_layer(z(2, 27, 768), z(2, 768), z(2, 768), z(16, 768), None, 6)  # Cout 4, D 768: two-token
        ops.final_layer(z(2, 27, 1152), z(2, 1152), z(2, 1152), z(12, 1152), None, 6)
        ops.patch_embed(z(2, 12, 6, 6), z(768, 4, 2, 2), z(768), None)             # Cin 4: k16
        ops.patch_embed(z(2, 9, 6, 6), z(768, 3, 2, 2), z(768), None)              # Cin 3: generic
        torch.cuda.synchronize()

    with profile(activities=[ProfilerActivity.CUDA], schedule=schedule(wait=0, warmup=1, active=1, repeat=1)) as prof:
        for _ in range(2):
            calls()
            prof.step()
    names = {e.key for e in prof.key_averages()}
    for k in ("norm_modulate_kernel", "norm_modulate_wide_kernel", "final_layer2_kernel", "final_layer_kernel",
              "patch_embed_k16_kernel", "patch_embed_kernel"):
        assert any(k in n for n in names), f"{k} never ran; kernels seen: {sorted(n for n in names if 'ln3' in n)}"
    print("glue kernels seen:", sorted(n for n in names if "ln3::" in n))
