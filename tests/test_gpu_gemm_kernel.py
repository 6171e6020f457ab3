"""GPU (-m gpu): the wgmma GEMM (ops.gemm -> gemm_wgmma.cu) element by element against float64 references, on
the DiT-L/2 hot shapes, the edges of the tile schedule and every epilogue.

Tolerances are derived from the arithmetic, beside each use:
  tau   fp32 accumulation of K exact bf16 products, then the bias add: <= (K + 1) 2^-23 (sum|a w| + |b|)
        (one fp32 ulp per add -- it allows for a tensor core that truncates instead of rounding -- over K + 1 adds)
  fp32  output: tau alone (plus the activation's own error and its slope times tau)
  bf16  output: the fp32 value rounded once: half a bf16 ulp at |y| + tau, plus tau
Every output view sits inside a NaN-filled buffer whose bytes outside the view must keep their bits, and every
case is launched three times with bit-identical results (the schedule is deterministic: no split-K, no atomics)."""
import json
import math
import os
import tempfile

import pytest
import torch

from kernel_bounds import SLOPE, act_ref, gemm_bf16_bound, gemm_tau, head_rmsnorm_ref, ulp

pytestmark = pytest.mark.gpu

PAD = 256           # NaN elements before and after every guarded view (512 B of bf16 keeps 16-byte alignment)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def guarded(shape, ld, dtype, dev, values=None):
    """(flat, view): a (rows, cols) view with row pitch `ld` inside a NaN-filled flat buffer."""
    rows, cols = shape
    flat = torch.full((2 * PAD + rows * ld,), float("nan"), dtype=dtype, device=dev)
    view = flat.as_strided((rows, cols), (ld, 1), PAD)
    if values is not None:
        view.copy_(values)
    return flat, view


def outside_unchanged(what, flat, view, before_bits):
    inside = torch.zeros(flat.numel(), dtype=torch.bool, device=flat.device)
    inside.as_strided(tuple(view.shape), view.stride(), view.storage_offset()).fill_(True)
    bits = torch.int16 if flat.dtype == torch.bfloat16 else torch.int32
    changed = (flat.view(bits) != before_bits) & ~inside
    assert not bool(changed.any()), f"{what}: {int(changed.sum())} elements outside the view were written"


def assert_within(what, got, ref, bound):
    err = (got.to(torch.float64) - ref).abs()
    bad = ~(err <= bound)                               # NaN counts as out of bound
    if bool(bad.any()):
        i = int(torch.where(bad, err / bound.clamp_min(1e-300), torch.zeros_like(err)).nan_to_num(float("inf"))
                .flatten().argmax())
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} out of bound; worst at flat {i}: got "
                             f"{got.flatten()[i].item()!r} expected {ref.flatten()[i].item()!r} "
                             f"bound {bound.flatten()[i].item():.3e}")


# ------------------------------------------------------------------ one case
def run_case(dev, M, N, K, *, bias=True, act=0, out_kind=0, ldo=None, gate_rows=0, out2=False, head_norm=False,
             seed=0):
    from ln3diff_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    a = torch.randn(M, K, device=dev, generator=g).bfloat16()
    w = (torch.randn(N, K, device=dev, generator=g) / math.sqrt(K)).bfloat16()
    b = torch.randn(N, device=dev, generator=g) if bias else None
    ldo = N if ldo is None else ldo
    a64, w64 = a.double(), w.double()
    y = a64 @ w64.T
    if b is not None:
        y = y + b.double()
    tau = gemm_tau(a64, w64, b.double() if b is not None else None)

    kw = {}
    if head_norm:
        # (nsec, sec_cols): every 64-column head its own section, or the production layouts -- sections of D columns
        # with heads of 64, and columns past the last section left without the norm
        nsec, sec_cols = (N // 64, 64) if head_norm is True else head_norm
        hw = 1 + 0.1 * torch.randn(nsec, 64, device=dev, generator=g)
        hn_eps = 1e-6 if head_norm is True else 1e-5
        kw.update(head_norm=hw, head_norm_sec_cols=sec_cols, head_norm_eps=hn_eps)
    if out_kind == ops.OUT_RESID_F32:
        x0 = torch.randn(M, N, device=dev, generator=g)
        flat, view = guarded((M, N), ldo, torch.float32, dev, x0)
        if gate_rows:
            gate = torch.randn((M + gate_rows - 1) // gate_rows, N, device=dev, generator=g)
            kw.update(gate=gate, gate_rows=gate_rows)
        if out2:
            flat2, view2 = guarded((M, N), ldo, torch.bfloat16, dev)
            kw.update(out2=view2)
    else:
        flat, view = guarded((M, N), ldo, torch.bfloat16 if out_kind == ops.OUT_BF16 else torch.float32, dev)
    bits = torch.int16 if flat.dtype == torch.bfloat16 else torch.int32
    before = flat.view(bits).clone()
    before2 = flat2.view(torch.int16).clone() if out2 else None

    results = []
    for _ in range(3):
        if out_kind == ops.OUT_RESID_F32:
            view.copy_(x0)
        ops.gemm(a, w, b, act=act, out_kind=out_kind, out=view, **kw)
        torch.cuda.synchronize()
        results.append((view.clone(), kw["out2"].clone() if out2 else None))
    what = f"M={M} N={N} K={K} act={act} out={out_kind} ldo={ldo}"
    for r in results[1:]:
        assert torch.equal(r[0].view(bits), results[0][0].view(bits)), f"{what}: launches differ"
        if out2:
            assert torch.equal(r[1].view(torch.int16), results[0][1].view(torch.int16)), f"{what}: out2 differs"
    outside_unchanged(what, flat, view, before)
    got = results[0][0]

    if head_norm:
        ref, tol = head_rmsnorm_ref(y, tau, hw, sec_cols, hn_eps)
        assert_within(what, got, ref, gemm_bf16_bound(ref, tol))
        return
    ref, act_err = act_ref(act, y)
    tol = SLOPE * tau + act_err if act else tau
    if out_kind == ops.OUT_BF16:
        assert_within(what, got, ref, ulp(ref.abs() + tol, 7) / 2 + tol)
    elif out_kind == ops.OUT_F32:
        assert_within(what, got, ref, tol)
    else:
        # x + g val by one fmaf: the gate times val's error, then one rounding of the sum
        gt = gate.double().repeat_interleave(gate_rows, 0)[:M] if gate_rows else torch.ones_like(ref)
        xn = x0.double() + gt * ref
        tol_x = gt.abs() * tol + ulp(xn.abs() + gt.abs() * tol, 23) / 2
        assert_within(what, got, xn, tol_x)
        if out2:
            outside_unchanged(what + " out2", flat2, kw["out2"], before2)
            assert_within(what + " out2", results[0][1], xn, ulp(xn.abs() + tol_x, 7) / 2 + tol_x)


# ------------------------------------------------------------------ cases
B, T, D = 16, 768, 1024        # bench.py's DiT-L/2 forward: 8 prompts with CFG, 768 tokens

HOT = {                        # name: (M, N, K, bias, act) of _denoiser.run_blocks
    "qkv": (B * T, 3 * D, D, True, 0),
    "proj": (B * T, D, D, True, 0),
    "cross_q": (B * T // 2, D, D, False, 0),
    "cross_out": (B * T // 2, D, D, True, 0),
    "fc1": (B * T, 4 * D, D, True, 1),
    "fc2": (B * T, D, 4 * D, True, 0),
}


@pytest.mark.parametrize("name", list(HOT))
def test_hot_shapes(dev, name):
    M, N, K, bias, act = HOT[name]
    run_case(dev, M, N, K, bias=bias, act=act)


@pytest.mark.parametrize("M,N,K", [
    (1, 256, 128),          # one row
    (77, 768, 768),         # a CLIP context
    (200, 384, 256),        # M % 128 != 0
    (256, 256, 512),        # 4 tiles: far fewer than the SMs, the second warpgroup has no tile
    (640, 128 * 53, 128),   # 265 tiles: one CTA more than two per SM, odd tile counts per CTA
    (384, 640, 64),         # K = 64: one k-block per tile, the ring wraps inside a tile sequence
    (512, 512, 4096),       # K = 4096
])
def test_tile_schedule_edges(dev, M, N, K):
    run_case(dev, M, N, K)


@pytest.mark.parametrize("act", [1, 2, 3, 4])
def test_bf16_activations(dev, act):
    run_case(dev, 333, 512, 256, act=act, seed=act)


@pytest.mark.parametrize("act", [0, 3])
def test_f32_output(dev, act):
    from ln3diff_b200 import ops
    run_case(dev, 333, 512, 256, act=act, out_kind=ops.OUT_F32)


@pytest.mark.parametrize("gate_rows,out2", [(0, False), (100, True), (0, True), (100, False)])
def test_residual_output(dev, gate_rows, out2):
    from ln3diff_b200 import ops
    run_case(dev, 333, 512, 256, out_kind=ops.OUT_RESID_F32, gate_rows=gate_rows, out2=out2)


def test_residual_output_with_activation(dev):
    from ln3diff_b200 import ops
    run_case(dev, 333, 512, 256, act=ops.ACT_GELU_TANH, out_kind=ops.OUT_RESID_F32, gate_rows=7)


def test_head_rmsnorm(dev):
    run_case(dev, 333, 1024, 512, bias=True, head_norm=True)


@pytest.mark.parametrize("N,nsec", [(3 * 768, 2), (2 * 768, 1)], ids=["qkv-nsec2-D768", "kv-nsec1-D768"])
def test_head_rmsnorm_sections(dev, N, nsec):
    """The denoisers' layouts: sections of D = 768 columns with heads of 64 -- qkv of the PixArt blocks (q and k
    normed, v untouched) and a cross-attention / second-source K|V (K normed, V untouched).  The columns past the
    last section take the epilogue's `sec >= nsec` skip and must come out as the plain GEMM."""
    run_case(dev, 333, N, 768, bias=True, head_norm=(nsec, 768))


@pytest.mark.parametrize("ldo", [1024 + 64, 512 + 2])
def test_output_pitch(dev, ldo):
    """ldo > N, and a pitch that is not a multiple of 8 elements (rows not 16-byte aligned)."""
    run_case(dev, 333, 512, 256, ldo=ldo)


def test_dit_forward_runs_the_pingpong_kernel(dev, monkeypatch):
    """The DiT-L/2 forward's GEMMs are the three-warpgroup (384-thread) ping-pong kernel."""
    from torch.profiler import ProfilerActivity, profile
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_t23d
    monkeypatch.setenv("LN3_CUDA_GRAPH", "0")
    model = build_t23d("DiT-L/2", seed=0, device=dev)
    model.prepare()
    tables = pipeline.edm_cfg_tables(250, 6.5, 1, dev)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 12, 32, 32, generator=g).to(dev)
    ctx = torch.cat([torch.zeros(1, 77, 768), torch.randn(1, 77, 768, generator=g)]).to(dev)
    model(x, tables["t_idx"][0], ctx, in_scale=tables["c_in"][0])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model(x, tables["t_idx"][1], ctx, in_scale=tables["c_in"][1])
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    gemms = [e for e in events if e.get("cat") == "kernel" and "gemm_bf16_kernel" in e.get("name", "")]
    assert len(gemms) >= 24 * 6, f"expected every block's GEMMs in the trace, found {len(gemms)}"
    blocks = {tuple(e["args"]["block"]) for e in gemms}
    assert blocks == {(384, 1, 1)}, blocks
