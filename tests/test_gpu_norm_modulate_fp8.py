"""GPU (-m gpu): ln3_norm_modulate_fp8 and ln3_quantize_fp8_rows against the restated fp8 block format.

Format (include/ln3b200.h), restated: per 1 x 128 block of a row, s = fp32(absmax / 448) and
code = e4m3_rne_satfinite(fp32(y / s)); an all-zero block has s = 0 and zero codes.
  * NORM_NONE without modulation (y = x): codes and scales are bit-exact against torch evaluating the same formula
    (fp32 division, torch's float8_e4m3fn cast), for fp32 and bf16 inputs of ops.quantize_fp8 too.
  * LayerNorm / RMSNorm with modulation: the dequantised code * s is within half an e4m3 ulp of y / s (times s) of
    the float64 value, plus the fp32 normalisation error e = 64 u (|n| (1 + |scale|) + |shift|) (n the normalised
    value, u = 2^-24: a <= 40-deep summation and rsqrt moving n by far less than 64 u relative).
  * The residual stream x is updated bit-identically to ln3_norm_modulate on the same inputs."""
import pytest
import torch

from kernel_bounds import nm_fp8_error
from kernel_bounds import restated_fp8 as restated

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def inputs(rows, D, dev, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, D, generator=g) * 3 + 0.5
    if rows > 3:
        x[1, :128] = 0                               # one all-zero block
        x[2, 128:256] = 1e4                          # a block of large equal values
        x[3] *= 1e-8                                 # subnormal codes
    return x.to(dev)


def bits_equal(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.parametrize("rows,D", [(1, 256), (300, 1024), (12288, 1024), (97, 1536)])
def test_norm_none_and_quantize_are_bit_exact(dev, rows, D):
    from ln3diff_b200 import ops
    from ln3diff_b200._lib import NORM_NONE
    x = inputs(rows, D, dev, rows + D)
    q_ref, s_ref = restated(x)
    q, s = ops.norm_modulate_fp8(x.clone(), norm=NORM_NONE)
    assert bits_equal(q, q_ref) and torch.equal(s, s_ref)
    q2, s2 = ops.quantize_fp8(x)
    assert bits_equal(q2, q_ref) and torch.equal(s2, s_ref)
    xb = x.to(torch.bfloat16)
    q3, s3 = ops.quantize_fp8(xb)
    qb, sb = restated(xb.float())
    assert bits_equal(q3, qb) and torch.equal(s3, sb)


@pytest.mark.parametrize("norm_kind", ["layer", "rms"])
@pytest.mark.parametrize("rows,D,T", [(12288, 1024, 768), (257, 768, 64)])
def test_norm_modulate_fp8_within_half_ulp(dev, norm_kind, rows, D, T):
    from ln3diff_b200 import ops
    from ln3diff_b200._lib import NORM_LAYER, NORM_RMS
    g = torch.Generator().manual_seed(7)
    x = inputs(rows, D, dev, 11)
    groups = (rows + T - 1) // T
    mod = (torch.randn(groups, 2 * D, generator=g) * 0.5).to(dev)
    shift, scale = mod[:, :D], mod[:, D:]
    w = (1 + 0.2 * torch.randn(D, generator=g)).to(dev)
    if norm_kind == "layer":
        kw, eps = dict(norm=NORM_LAYER), 1e-6
    else:
        kw, eps = dict(norm=NORM_RMS, weight=w, eps=1e-5), 1e-5
    q, s = ops.norm_modulate_fp8(x, shift=shift, scale=scale, mod_rows=T, **kw)
    x64 = x.double()
    if norm_kind == "layer":
        n = (x64 - x64.mean(1, keepdim=True)) * torch.rsqrt(x64.var(1, unbiased=False, keepdim=True) + eps)
    else:
        n = x64 * torch.rsqrt((x64 * x64).mean(1, keepdim=True) + eps) * w.double()
    idx = torch.arange(rows, device=dev) // T
    sc, sh = scale.double()[idx], shift.double()[idx]
    y = n * (1 + sc) + sh
    e = 64 * 2.0 ** -24 * (n.abs() * (1 + sc.abs()) + sh.abs())
    err, bound = nm_fp8_error(q, s, y, e)
    assert bool((err <= bound).all()), f"{int((err > bound).sum())} values off; max ratio {float((err / bound).max()):.3f}"
    print(f"{norm_kind} {rows}x{D}: max error / bound {float((err / bound).max()):.3e}")


def test_residual_update_matches_bf16_kernel_bit_for_bit(dev):
    """The fused residual passes of run_blocks, including the closed-form broadcast rows with their second gate."""
    from ln3diff_b200 import ops
    from ln3diff_b200._lib import NORM_LAYER
    g = torch.Generator().manual_seed(5)
    B, T, D = 8, 256, 1024
    rows = B * T
    x = (torch.randn(rows, D, generator=g) * 2).to(dev)
    resid = torch.randn(rows, D, generator=g).to(dev, torch.bfloat16)
    gate = torch.randn(B, D, generator=g).to(dev)
    bcast = torch.randn(B, D, generator=g).to(dev, torch.bfloat16)
    ogate = torch.randn(B, D, generator=g).to(dev)
    mod = torch.randn(B, 2 * D, generator=g).to(dev)
    for extra in (dict(resid_gate=gate, resid_gate_rows=T),
                  dict(resid_bcast=bcast, resid_bcast_rows=T, resid_rows=(2 * T, 6 * T), resid_out_gate=ogate,
                       resid_out_gate_rows=T)):
        xa, xb = x.clone(), x.clone()
        ops.norm_modulate(xa, norm=NORM_LAYER, shift=mod[:, :D], scale=mod[:, D:], mod_rows=T, resid=resid, **extra)
        ops.norm_modulate_fp8(xb, norm=NORM_LAYER, shift=mod[:, :D], scale=mod[:, D:], mod_rows=T, resid=resid,
                              **extra)
        assert torch.equal(xa.view(torch.int32), xb.view(torch.int32))


def test_unsupported_width_is_refused(dev):
    from ln3diff_b200 import ops
    from ln3diff_b200._lib import NORM_LAYER
    x = torch.randn(4, 384, device=dev)
    with pytest.raises(RuntimeError, match="code -3"):
        ops.norm_modulate_fp8(x, norm=NORM_LAYER)
