"""CPU: the host side of the fp8 GEMM precision -- the new structs against the header, the exported symbols, the
C-level refusals of ln3_gemm_fp8 / ln3_norm_modulate_fp8 / ln3_quantize_fp8_rows, the ops-level dtype checks,
the weight quantiser and DenoiserMixin.set_gemm_precision.

Format restated (include/ln3b200.h): weights are e4m3 codes with one fp32 scale per output channel,
w_scale = fp32(absmax of the row / 448), codes = float8_e4m3fn(fp32(w / w_scale)); a zero row has scale 0.
The C-level calls use fabricated device addresses that are never dereferenced, as in test_abi_validation.py: a
refused call returns its code before any CUDA call, so these run only where there is no GPU."""
import ctypes as C
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, ECUDA, EUNSUPPORTED = -1, -2, -3
BASE = 1 << 36
no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="fabricated addresses must not reach a real device")


def _addr(i: int) -> int:
    return BASE + i * (1 << 24)


def _fields(cname: str) -> list:
    src = open(os.path.join(ROOT, "include", "ln3b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    body = re.search(r"typedef struct " + cname + r"\s*\{(.*?)\}\s*" + cname + ";", src, flags=re.S).group(1)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            decl = re.sub(r"^(const\s+)?(unsigned\s+)?[A-Za-z_0-9]+(\s+long)?\s*\**", "", decl, count=1)
            names += [n.strip().lstrip("*") for n in decl.split(",")]
    return names


def test_ctypes_structs_match_header():
    from ln3diff_b200 import _lib
    assert _fields("ln3_gemm_fp8_args") == [f[0] for f in _lib.GemmFp8Args._fields_]
    assert _fields("ln3_norm_modulate_fp8_args") == [f[0] for f in _lib.NormModulateFp8Args._fields_]
    assert _lib.NormModulateFp8Args._fields_[0][1] is _lib.NormModulateArgs


def test_new_symbols_are_exported(built_lib):
    lib = C.CDLL(str(built_lib))
    for s in ("ln3_gemm_fp8", "ln3_gemm_fp8_workspace_bytes", "ln3_norm_modulate_fp8", "ln3_quantize_fp8_rows"):
        assert hasattr(lib, s), s
    lib.ln3_gemm_fp8_workspace_bytes.restype = C.c_size_t
    assert lib.ln3_gemm_fp8_workspace_bytes() == 0


# ------------------------------------------------------------------ C-level refusals
@pytest.fixture(scope="module")
def lib(built_lib):
    from ln3diff_b200 import _lib
    return _lib.lib()


def _gemm_args(**kw):
    from ln3diff_b200 import _lib
    a = _lib.GemmFp8Args()
    a.A, a.a_scale, a.W, a.w_scale, a.bias, a.out, a.out_scale = (_addr(i) for i in range(7))
    a.M, a.N, a.K = 300, 1024, 1024
    a.lda, a.ldw, a.ldo, a.a_scale_ld, a.out_scale_ld = 1024, 1024, 1024, 8, 8
    a.act, a.out_kind = 0, 0
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _rc(lib, fn, args):
    rc = getattr(lib, fn)(C.byref(args), C.c_void_p(0))
    return rc, lib.ln3_last_error().decode(errors="replace")


@no_gpu
@pytest.mark.parametrize("kw,code,msg", [
    (dict(K=1000, lda=1024, ldw=1024), EINVAL, "multiple of 128"),
    (dict(N=1000), EINVAL, "multiple of 128"),
    (dict(M=0), EINVAL, "empty"),
    (dict(a_scale=None), EINVAL, "a_scale"),
    (dict(w_scale=None), EINVAL, "w_scale"),
    (dict(lda=1000), EINVAL, "lda"),
    (dict(A=_addr(0) + 8), EINVAL, "16-byte aligned"),
    (dict(bias=_addr(4) + 4), EINVAL, "16-byte aligned"),
    (dict(a_scale_ld=4), EINVAL, "a_scale_ld"),
    (dict(ldo=1028), EINVAL, "ldo"),
    (dict(out_kind=3, out_scale=None), EINVAL, "out_scale"),
    (dict(out_kind=3, out_scale_ld=4), EINVAL, "out_scale"),
    (dict(act=1), EUNSUPPORTED, "not implemented"),
    (dict(out_kind=1), EUNSUPPORTED, "not implemented"),
    (dict(out_kind=3, act=3), EUNSUPPORTED, "not implemented"),
    (dict(out_kind=3, head_norm_w=_addr(8), head_norm_nsec=2, head_norm_sec_cols=1024), EUNSUPPORTED, "head_norm"),
    (dict(head_norm_w=_addr(8), head_norm_nsec=2, head_norm_sec_cols=100), EINVAL, "head_norm"),
])
def test_gemm_fp8_refusals(lib, kw, code, msg):
    rc, err = _rc(lib, "ln3_gemm_fp8", _gemm_args(**kw))
    assert rc == code and msg in err, (rc, err)


@no_gpu
@pytest.mark.parametrize("kw", [dict(), dict(out_kind=3, act=1), dict(ldo=2048, out_kind=3)])
def test_gemm_fp8_valid_arguments_reach_the_device(lib, kw):
    rc, _ = _rc(lib, "ln3_gemm_fp8", _gemm_args(**kw))
    assert rc == ECUDA


def _nm_args(D=1024, **kw):
    from ln3diff_b200 import _lib
    f = _lib.NormModulateFp8Args()
    f.base.x, f.base.rows, f.base.D, f.base.ldx, f.base.norm = _addr(0), 64, D, D, 1
    f.out, f.out_scale, f.ldo, f.out_scale_ld = _addr(1), _addr(2), D, D // 128
    for k, v in kw.items():
        if k.startswith("base_"):
            setattr(f.base, k[5:], v)
        else:
            setattr(f, k, v)
    return f


@no_gpu
@pytest.mark.parametrize("kw,code,msg", [
    (dict(base_out=_addr(3)), EINVAL, "base.out must be NULL"),
    (dict(out=None), EINVAL, "out and out_scale"),
    (dict(out_scale=None), EINVAL, "out and out_scale"),
    (dict(ldo=1032), EINVAL, "multiple of 16"),
    (dict(out_scale_ld=4), EINVAL, "out_scale_ld"),
    (dict(out=_addr(1) + 8), EINVAL, "16-byte aligned"),
    (dict(D=384, ldo=384, out_scale_ld=3, base_ldx=384), EUNSUPPORTED, "D % 256"),
    (dict(D=1792, ldo=1792, out_scale_ld=14, base_ldx=1792), EUNSUPPORTED, "D <= 1536"),
    (dict(base_x=_addr(0) + 16), EUNSUPPORTED, "32-byte aligned"),
    (dict(base_shift=_addr(4)), EINVAL, "shift and scale"),
])
def test_norm_modulate_fp8_refusals(lib, kw, code, msg):
    D = kw.pop("D", 1024)
    rc, err = _rc(lib, "ln3_norm_modulate_fp8", _nm_args(D, **kw))
    assert rc == code and msg in err, (rc, err)


@no_gpu
def test_norm_modulate_fp8_valid_arguments_reach_the_device(lib):
    assert _rc(lib, "ln3_norm_modulate_fp8", _nm_args())[0] == ECUDA


@no_gpu
@pytest.mark.parametrize("args,msg", [
    ((_addr(0), 0, 1024, 4, 1000, _addr(1), 1024, _addr(2), 8), "multiple of 128"),
    ((_addr(0), 0, 1024, 4, 1024, _addr(1), 1024, None, 8), "null"),
    ((_addr(0), 0, 1024, 4, 1024, _addr(1), 1024, _addr(2), 4), "out_scale_ld"),
    ((_addr(0), 1, 1028, 4, 1024, _addr(1), 1024, _addr(2), 8), "16-byte"),
    ((_addr(0) + 4, 0, 1024, 4, 1024, _addr(1), 1024, _addr(2), 8), "16-byte"),
    ((_addr(0), 0, 1024, 4, 1024, _addr(1), 1032, _addr(2), 8), "16-byte"),
])
def test_quantize_fp8_rows_refusals(lib, args, msg):
    rc = lib.ln3_quantize_fp8_rows(*args, None)
    assert rc == EINVAL and msg in lib.ln3_last_error().decode(), lib.ln3_last_error()
    assert lib.ln3_quantize_fp8_rows(_addr(0), 0, 1024, 0, 1024, _addr(1), 1024, _addr(2), 8, None) == 0  # no rows


# ------------------------------------------------------------------ ops-level checks (before any device call)
def test_ops_refuse_host_tensors_and_wrong_dtypes():
    from ln3diff_b200 import ops
    q = torch.zeros(128, 128, dtype=ops.FP8)
    s = torch.zeros(128, 1)
    with pytest.raises(ValueError, match="CUDA"):
        ops.gemm_fp8(q, s, q, torch.zeros(128))
    with pytest.raises(ValueError, match="CUDA"):
        ops.quantize_fp8(torch.zeros(4, 128))
    with pytest.raises(ValueError, match="CUDA"):
        ops.norm_modulate_fp8(torch.zeros(4, 256), norm=1)


# ------------------------------------------------------------------ weight quantiser
def test_weight_quantiser_scales_zero_rows_saturation_and_round_trip():
    from ln3diff_b200 import ops
    g = torch.Generator().manual_seed(0)
    w = torch.randn(64, 256, generator=g) * torch.exp2(torch.randint(-6, 6, (64, 1), generator=g).float())
    w[3] = 0
    w[5, 7] = 1e30                                   # one huge entry: its row's codes saturate at exactly +-448
    q, s = ops.quantize_weight_fp8(w)
    assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32 and q.shape == w.shape and s.shape == (64,)
    amax = w.abs().amax(1)
    assert torch.equal(s, amax / torch.full_like(amax, 448.0))
    assert float(s[3]) == 0 and bool((q[3].float() == 0).all())
    assert float(q[5, 7].float()) == 448.0
    assert bool(torch.isfinite(q.float()).all()) and float(q.float().abs().max()) <= 448
    # round trip: |q s - w| <= half an e4m3 ulp of w / s, times s (subnormal spacing 2^-9 below 2^-6)
    t = w / torch.where(s > 0, s, torch.ones_like(s))[:, None]
    _, e = torch.frexp(t.abs().double().clamp_min(2.0 ** -6))
    half = torch.ldexp(torch.full_like(t, 0.5, dtype=torch.float64), (e - 4).to(torch.int32))
    err = (q.double() * s.double()[:, None] - w.double()).abs()
    assert bool((err <= half * s.double()[:, None] * (1 + 2 ** -20)).all())


# ------------------------------------------------------------------ set_gemm_precision
def test_set_gemm_precision_invalidates_derived_state_only():
    from ln3diff_b200.utils import build_t23d
    m = build_t23d("DiT-B/2")
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    assert m.gemm_precision == "bf16"
    m._prep, m._ws, m._graphs = {"sentinel": 1}, {2: {}}, {("k",): object()}
    m._ctx_static = {"x": 1}
    cache = m._ctx_cache
    assert m.set_gemm_precision("fp8") is m and m.gemm_precision == "fp8"
    assert m._prep is None and m._ws == {} and m._graphs == {} and m._ctx_static == {} and m._ctx_cache is not cache
    m._prep = {"sentinel": 2}
    m.set_gemm_precision("fp8")                       # no change: derived state kept
    assert m._prep == {"sentinel": 2}
    with pytest.raises(ValueError, match="bf16' or 'fp8"):
        m.set_gemm_precision("fp16")
    m.set_gemm_precision("bf16")
    assert m._prep is None
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
