"""GPU (-m gpu): the FP8 wgmma GEMM (ops.gemm_fp8 -> gemm_fp8_wgmma.cu) element by element against float64.

Number format (include/ln3b200.h), restated: e4m3 codes (torch.float8_e4m3fn: 3 mantissa bits, +-448 saturation);
A carries fp32 block scales a_scale[m, kb] per 1 x 128 block, W per-output-channel scales w_scale[n];
    out = epilogue(fmaf(sum_kb a_scale[m, kb] * P(m, n, kb), w_scale[n], bias[n])),  P = sum_{k in block} q_a q_w
and an fp8 output block is s = fp32(absmax / 448), code = e4m3_rne_satfinite(fp32(v / s)) (s = 0: zero codes).

The operands here are e4m3 codes and arbitrary fp32 scales, so every product q_a q_w is exact (4 x 4 significant
bits) and the only arithmetic error is accumulation.  Bounds, with T = w_scale[n] sum_kb a_scale[m, kb] sum |q_a q_w|
(the same GEMM on absolute values):
  U_ACC   the tensor core's in-block fp8 accumulation.  NVIDIA does not document it; public measurements report about
          14 significant bits kept.  Assumed: each of the <= 128 additions of a block loses at most 2^-13 of the
          running magnitude, i.e. |P_kernel - P| <= 128 * 2^-13 * sum_block |q_a q_w|.
  fp32    the promotion fmaf per k-block and the epilogue fmaf: (K/128 + 2) 2^-23 (T + |bias|)
  E = 128 * 2^-13 * T + (K/128 + 2) 2^-23 (T + |bias|)
  bf16 output: E plus half a bf16 ulp at |y| + E
  fp8 output: the code must lie between the rounding of (v - d) / s and of (v + d) / s, d = slope * E + f_err
          (f_err: the GELU polynomial's own error, as in test_gpu_gemm_kernel.py), i.e. equal to the restated
          quantisation of the fp64 value except where that value is within d of a rounding boundary.
The largest error / bound ratio of each case is printed: if the hardware accumulates more coarsely than assumed,
that is what this file reports, and the bound stays where it is derived.
Outputs sit in NaN-filled buffers whose bytes outside the view must keep their bits, and three launches must give
identical bits (no split-K, no atomics)."""
import zlib

import pytest
import torch

from kernel_bounds import FP8, SLOPE, fp8_bf16_bound, fp8_out_check, gelu_ref
from kernel_bounds import fp8_acc_bound as acc_bound
from kernel_bounds import fp8_head_norm_ref as head_norm_ref
from kernel_bounds import fp8_reference as reference

pytestmark = pytest.mark.gpu

PAD = 512


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def guarded(rows, cols, ld, dtype, dev):
    """(flat, view): a (rows, cols) view with row pitch `ld` inside a NaN-filled flat buffer (0xFF bytes for fp8)."""
    if dtype == FP8:
        flat = torch.full((2 * PAD + rows * ld,), 255, dtype=torch.uint8, device=dev).view(FP8)
    else:
        flat = torch.full((2 * PAD + rows * ld,), float("nan"), dtype=dtype, device=dev)
    return flat, flat.as_strided((rows, cols), (ld, 1), PAD)


def raw(t):
    return t.view(torch.uint8) if t.dtype == FP8 else t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def outside_unchanged(what, flat, view, before):
    inside = torch.zeros(flat.numel(), dtype=torch.bool, device=flat.device)
    inside.as_strided(tuple(view.shape), view.stride(), view.storage_offset()).fill_(True)
    changed = (raw(flat) != before) & ~inside
    assert not bool(changed.any()), f"{what}: {int(changed.sum())} elements outside the view were written"


def random_codes(rows, cols, g, dev, zero_rows=()):
    """e4m3 codes spread over the whole range (normals, subnormals, zeros, +-448)."""
    v = torch.randn(rows, cols, generator=g) * torch.exp2(torch.randint(-8, 8, (rows, cols), generator=g).float())
    for r in zero_rows:
        v[r] = 0
    return v.clamp(-448, 448).to(FP8).to(dev)


def operands(M, N, K, dev, seed, bias=True):
    g = torch.Generator().manual_seed(seed)
    a_q = random_codes(M, K, g, dev, zero_rows=(0,) if M > 1 else ())
    w_q = random_codes(N, K, g, dev)
    a_s = (torch.rand(M, K // 128, generator=g) * 2 ** torch.randint(-10, 2, (M, K // 128), generator=g).float())
    a_s[0, 0] = 0.0
    w_s = torch.rand(N, generator=g) * 2.0 ** -6 + 2.0 ** -12
    b = torch.randn(N, generator=g) if bias else None
    return a_q, a_s.to(dev), w_q, w_s.to(dev), (b.to(dev) if bias else None)


def check_bf16(what, got, ref, E):
    bound = fp8_bf16_bound(ref, E)
    err = (got.to(torch.float64) - ref).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max())
    bad = ~(err <= bound)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {got.numel()} out of bound (max ratio {ratio:.3f})"
    return ratio


def check_fp8(what, q, s, v, d):
    """q / s the kernel's codes and block scales, v the fp64 epilogue value, d its error bound."""
    sratio, exact, ok, s_ok = fp8_out_check(q, s, v, d)
    assert bool(s_ok.all()), f"{what}: block scales off by up to {sratio:.3f} x bound"
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} of {q.numel()} codes off the restated quantisation"
    return sratio, exact


CASES = [
    # name, M, N, K, epilogue
    ("qkv_L2_B16", 12288, 3072, 1024, "bf16"),
    ("qkv_L2_B16_headnorm", 12288, 3072, 1024, "headnorm"),
    ("fc1_L2_B16_gelu_fp8", 12288, 4096, 1024, "gelu_fp8"),
    ("fc2_L2_B16", 12288, 1024, 4096, "bf16"),
    ("single_tile", 128, 128, 128, "bf16"),
    ("one_row", 1, 256, 256, "gelu_fp8"),
    ("m_tail_200", 200, 384, 384, "fp8"),
    ("m_tail_1000_headnorm", 1000, 768, 512, "headnorm"),
    ("more_tiles_than_sms_K128", 8193, 640, 128, "bf16"),
    ("fp8_out_no_act", 777, 1024, 640, "fp8"),
]


@pytest.mark.parametrize("name,M,N,K,epi", CASES, ids=[c[0] for c in CASES])
def test_gemm_fp8_elementwise(dev, name, M, N, K, epi):
    from ln3diff_b200 import ops
    a_q, a_s, w_q, w_s, b = operands(M, N, K, dev, seed=zlib.crc32(name.encode()) % 1000)
    ref, T = reference(a_q, a_s, w_q, w_s, b)
    E = acc_bound(T, K, b)
    kw, hn = {}, None
    if epi == "headnorm":
        g = torch.Generator().manual_seed(3)
        hn = (1 + 0.1 * torch.randn(2, 64, generator=g)).to(dev)
        kw = dict(head_norm=hn, head_norm_sec_cols=N // 3)
    fp8_out = epi in ("fp8", "gelu_fp8")
    ldo = N + 128
    flat, view = guarded(M, N, ldo, FP8 if fp8_out else torch.bfloat16, dev)
    sflat, sview = guarded(M, N // 128, N // 128 + 4, torch.float32, dev)
    before, sbefore = raw(flat).clone(), raw(sflat).clone()
    results = []
    for _ in range(3):
        if fp8_out:
            ops.gemm_fp8(a_q, a_s, w_q, w_s, b, act=ops.ACT_GELU_ERF if epi == "gelu_fp8" else ops.ACT_NONE,
                         out_kind=ops.OUT_FP8, out=view, out_scale=sview)
            results.append((raw(view).clone(), raw(sview).clone()))
        else:
            ops.gemm_fp8(a_q, a_s, w_q, w_s, b, out=view, **kw)
            results.append((raw(view).clone(),))
    torch.cuda.synchronize()
    for r in results[1:]:
        assert all(torch.equal(x, y) for x, y in zip(results[0], r)), f"{name}: launches differ"
    outside_unchanged(name, flat, view, before)
    if fp8_out:
        outside_unchanged(name + " scales", sflat, sview, sbefore)
        if epi == "gelu_fp8":
            v, ferr = gelu_ref(ref)
            d = SLOPE * E + ferr
        else:
            v, d = ref, E
        sratio, exact = check_fp8(name, view, sview, v, d)
        print(f"{name}: scale error / bound {sratio:.3e}, codes equal to the fp64 quantisation {exact:.5f}")
    else:
        if epi == "headnorm":
            ref, E = head_norm_ref(ref, E, hn, 2, N // 3)
        ratio = check_bf16(name, view, ref, E)
        # the assumed in-block accumulation alone: how much of it the hardware used
        print(f"{name}: max error / bound {ratio:.3e}")


def test_gemm_fp8_zero_and_saturated_operands(dev):
    """All-zero A blocks (scale 0) give exactly the bias; +-448 codes everywhere give the exact large sums."""
    from ln3diff_b200 import ops
    M, N, K = 256, 256, 256
    a_q = torch.full((M, K), 448.0, device=dev).to(FP8)
    a_q[:, :128] = 0
    w_q = torch.full((N, K), -448.0, device=dev).to(FP8)
    a_s = torch.ones(M, 2, device=dev)
    a_s[:, 0] = 0
    w_s = torch.full((N,), 2.0 ** -10, device=dev)
    b = torch.arange(N, device=dev, dtype=torch.float32)
    out = ops.gemm_fp8(a_q, a_s, w_q, w_s, b)
    ref = (-448.0 * 448.0 * 128 * 2.0 ** -10 + b.double())[None, :].expand(M, N)
    assert torch.equal(out.double(), ref.to(torch.bfloat16).double())
