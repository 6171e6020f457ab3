"""Thin, checked Python entry points over the C ABI (one function per exported op).

Shape / dtype / contiguity violations raise here (mirroring the TORCH_CHECKs of the reference's
own native ops, utils/torch_utils/ops/bias_act.cpp:39-60); everything else is the C call.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import (ACT_GELU_ERF, ACT_GELU_TANH, ACT_NONE, ACT_QUICK_GELU, ACT_SILU, OUT_BF16, OUT_F32, OUT_FP8,
                   OUT_RESID_F32)

__all__ = ["gemm", "gemm_fp8", "norm_modulate_fp8", "quantize_fp8", "quantize_weight_fp8", "ACT_NONE", "ACT_GELU_ERF",
           "ACT_GELU_TANH", "ACT_SILU", "ACT_QUICK_GELU", "OUT_BF16", "OUT_F32", "OUT_RESID_F32", "OUT_FP8"]

FP8 = torch.float8_e4m3fn
FP8_MAX = 448.0


def _req(cond: bool, msg: str) -> None:
    if not cond:
        raise ValueError(msg)


def _cuda(t: torch.Tensor, name: str, dtype=None) -> None:
    _req(t.is_cuda, f"{name} must be a CUDA tensor (no CPU fallback)")
    if dtype is not None:
        _req(t.dtype == dtype, f"{name} must be {dtype}, got {t.dtype}")


def gemm(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, *,
         act: int = ACT_NONE, out_kind: int = OUT_BF16, out: torch.Tensor | None = None,
         out2: torch.Tensor | None = None, gate: torch.Tensor | None = None,
         gate_rows: int = 1, head_norm: torch.Tensor | None = None, head_norm_sec_cols: int = 0,
         head_norm_eps: float = 1e-5) -> torch.Tensor:
    """out = epilogue(a @ w.T); a (M,K) bf16, w (N,K) bf16 (nn.Linear weight layout).

    OUT_RESID_F32: `out` is the fp32 residual stream (M,N), updated in place with
    out += gate[(m // gate_rows)] * val; `gate` is a 2-D fp32 view (G,N) with unit inner stride.
    """
    _cuda(a, "a", torch.bfloat16)
    _cuda(w, "w", torch.bfloat16)
    _req(a.dim() == 2 and w.dim() == 2, "a and w must be 2-D")
    _req(a.stride(1) == 1 and w.stride(1) == 1, "a and w must have unit inner stride")
    M, K = a.shape
    N, K2 = w.shape
    _req(K == K2, f"inner dims differ: {K} vs {K2}")
    if out is None:
        _req(out_kind != OUT_RESID_F32, "OUT_RESID_F32 needs the residual tensor as `out`")
        out = torch.empty((M, N), device=a.device,
                          dtype=torch.bfloat16 if out_kind == OUT_BF16 else torch.float32)
    _cuda(out, "out", torch.bfloat16 if out_kind == OUT_BF16 else torch.float32)
    _req(out.shape == (M, N) and out.stride(1) == 1, "out must be (M,N) with unit inner stride")
    args = _lib.GemmArgs()
    args.A, args.W, args.out = a.data_ptr(), w.data_ptr(), out.data_ptr()
    args.M, args.N, args.K = M, N, K
    args.lda, args.ldw, args.ldo = a.stride(0), w.stride(0), out.stride(0)
    if bias is not None:
        _cuda(bias, "bias", torch.float32)
        _req(bias.shape == (N,) and bias.is_contiguous(), "bias must be contiguous (N,)")
        args.bias = bias.data_ptr()
    if out2 is not None:
        _cuda(out2, "out2", torch.bfloat16)
        _req(out2.shape == (M, N) and out2.stride(1) == 1, "out2 must be (M,N)")
        args.out2, args.ldo2 = out2.data_ptr(), out2.stride(0)
    if gate is not None:
        _cuda(gate, "gate", torch.float32)
        _req(gate.dim() == 2 and gate.shape[1] == N and gate.stride(1) == 1, "gate must be (G,N)")
        _req(gate.shape[0] * gate_rows >= M, "gate has too few rows")
        args.gate, args.gate_ld, args.gate_rows = gate.data_ptr(), gate.stride(0), gate_rows
    if head_norm is not None:
        _cuda(head_norm, "head_norm", torch.float32)
        _req(head_norm.dim() == 2 and head_norm.shape[1] == 64 and head_norm.is_contiguous(),
             "head_norm must be contiguous (nsec, 64): the head-RMSNorm epilogue normalises 64-wide heads only")
        args.head_norm_w, args.head_norm_nsec = head_norm.data_ptr(), head_norm.shape[0]
        args.head_norm_sec_cols, args.head_norm_eps = head_norm_sec_cols, head_norm_eps
    args.act, args.out_kind = act, out_kind
    _lib.check(_lib.lib().ln3_gemm_bf16(C.byref(args), _lib.current_stream()), "ln3_gemm_bf16")
    return out


def fmha(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, *,
         out: torch.Tensor | None = None, scale: float | None = None,
         k2: torch.Tensor | None = None, v2: torch.Tensor | None = None, causal: bool = False) -> torch.Tensor:
    """softmax(q k^T * scale) v per head.  q (B,Lq,H*hd), k/v (B,Lkv,H*hd) bf16 views with unit
    inner stride (slices of a packed qkv buffer are fine), head width hd 64 or 72 (k2/v2 need 64);
    returns (B,Lq,H*hd) bf16.  scale defaults to hd ** -0.5.
    causal=True: key j is visible to query i only when j <= i (CLIP text tower)."""
    for name, t in (("q", q), ("k", k), ("v", v)):
        _cuda(t, name, torch.bfloat16)
        _req(t.dim() == 3 and t.stride(2) == 1, f"{name} must be (B,L,H*head_dim) with unit inner stride")
    B, Lq, C_ = q.shape
    _req(heads > 0 and C_ % heads == 0, "q's width must be heads * head_dim")
    hd = C_ // heads
    _req(hd in (64, 72), f"head_dim must be 64 or 72, got {hd}")
    _req(k.shape == v.shape and k.shape[0] == B and k.shape[2] == C_, "k/v shape mismatch")
    Lkv = k.shape[1]
    if out is None:
        out = torch.empty((B, Lq, C_), device=q.device, dtype=torch.bfloat16)
    _cuda(out, "out", torch.bfloat16)
    _req(out.shape == (B, Lq, C_) and out.stride(2) == 1, "out must be (B,Lq,H*head_dim)")
    a = _lib.FmhaArgs()
    a.q, a.k, a.v, a.out = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    a.B, a.H, a.Lq, a.Lkv, a.head_dim = B, heads, Lq, Lkv, hd
    a.q_ld, a.q_bs = q.stride(1), q.stride(0)
    a.k_ld, a.k_bs = k.stride(1), k.stride(0)
    a.v_ld, a.v_bs = v.stride(1), v.stride(0)
    a.o_ld, a.o_bs = out.stride(1), out.stride(0)
    a.scale = float(scale if scale is not None else hd ** -0.5)
    a.causal = 1 if causal else 0
    _req(not (causal and k2 is not None), "causal attention takes a single K/V source")
    if k2 is not None:
        for name, t in (("k2", k2), ("v2", v2)):
            _cuda(t, name, torch.bfloat16)
            _req(t.dim() == 3 and t.stride(2) == 1 and t.shape[0] == B and t.shape[2] == C_,
                 f"{name} must be (B,L2,H*head_dim)")
        _req(k2.shape == v2.shape, "k2/v2 shape mismatch")
        a.k2, a.v2, a.Lkv2 = k2.data_ptr(), v2.data_ptr(), k2.shape[1]
        a.k2_ld, a.k2_bs, a.v2_ld, a.v2_bs = k2.stride(1), k2.stride(0), v2.stride(1), v2.stride(0)
    _lib.check(_lib.lib().ln3_fmha_fwd(C.byref(a), _lib.current_stream()), "ln3_fmha_fwd")
    return out


def norm_modulate(x: torch.Tensor, *, norm: int, shift: torch.Tensor | None = None,
                  scale: torch.Tensor | None = None, mod_rows: int = 1,
                  shift_tab: torch.Tensor | None = None, scale_tab: torch.Tensor | None = None,
                  weight: torch.Tensor | None = None, eps: float = 1e-6, act: int = ACT_NONE,
                  out: torch.Tensor | None = None, resid: torch.Tensor | None = None,
                  resid_gate: torch.Tensor | None = None, resid_gate_rows: int = 1,
                  want_out: bool = True, resid_bcast: torch.Tensor | None = None, resid_bcast_rows: int = 1,
                  resid_rows: tuple | None = None, resid_out_gate: torch.Tensor | None = None,
                  resid_out_gate_rows: int = 1) -> torch.Tensor | None:
    """bf16( norm(x) * (1 + scale[g]) + shift[g] ), x fp32 (rows, D); shift/scale 2-D fp32 views
    (groups, D) with unit inner stride and equal row stride; row r uses group r // mod_rows.
    With `resid` (bf16 (rows, D)) the residual update x += resid_gate[r // resid_gate_rows] * resid is
    applied first, IN PLACE on x; want_out=False then skips the normalised output.  With `resid_bcast`
    ((groups, D) bf16) rows outside resid_rows=(begin, end) use resid_bcast[r // resid_bcast_rows] as
    their residual row instead of resid[r]; with `resid_out_gate` ((groups, D) fp32) those outside rows first add
    resid_out_gate[r // resid_out_gate_rows] * resid[r] (their own, not yet applied, gated residual) as well."""
    _cuda(x, "x", torch.float32)
    _req(x.dim() == 2 and x.stride(1) == 1, "x must be (rows, D) with unit inner stride")
    rows, D = x.shape
    a = _lib.NormModulateArgs()
    if want_out:
        if out is None:
            out = torch.empty((rows, D), device=x.device, dtype=torch.bfloat16)
        _cuda(out, "out", torch.bfloat16)
        _req(out.shape == (rows, D) and out.stride(1) == 1, "out must be (rows, D)")
        a.out, a.ldo = out.data_ptr(), out.stride(0)
    else:
        _req(resid is not None, "want_out=False needs a residual update")
        out = None
    _norm_modulate_inputs(a, x, norm=norm, shift=shift, scale=scale, mod_rows=mod_rows, shift_tab=shift_tab,
                          scale_tab=scale_tab, weight=weight, eps=eps, act=act, resid=resid, resid_gate=resid_gate,
                          resid_gate_rows=resid_gate_rows, resid_bcast=resid_bcast, resid_bcast_rows=resid_bcast_rows,
                          resid_rows=resid_rows, resid_out_gate=resid_out_gate, resid_out_gate_rows=resid_out_gate_rows)
    _lib.check(_lib.lib().ln3_norm_modulate(C.byref(a), _lib.current_stream()), "ln3_norm_modulate")
    return out


def _norm_modulate_inputs(a, x, *, norm, shift, scale, mod_rows, shift_tab, scale_tab, weight, eps, act, resid,
                          resid_gate, resid_gate_rows, resid_bcast, resid_bcast_rows, resid_rows, resid_out_gate,
                          resid_out_gate_rows) -> None:
    """Checks every input of norm_modulate except the output and fills them into the NormModulateArgs `a`."""
    rows, D = x.shape
    if resid is not None:
        _cuda(resid, "resid", torch.bfloat16)
        _req(resid.shape == (rows, D) and resid.stride(1) == 1, "resid must be (rows, D) bf16")
        a.resid, a.resid_ld = resid.data_ptr(), resid.stride(0)
        if resid_gate is not None:
            _cuda(resid_gate, "resid_gate", torch.float32)
            _req(resid_gate.dim() == 2 and resid_gate.shape[1] == D and resid_gate.stride(1) == 1
                 and resid_gate.shape[0] * resid_gate_rows >= rows, "resid_gate must be a (groups, D) view")
            a.resid_gate, a.resid_gate_ld, a.resid_gate_rows = resid_gate.data_ptr(), resid_gate.stride(0), resid_gate_rows
    if resid_bcast is not None:
        _req(resid is not None and resid_rows is not None, "resid_bcast needs resid and resid_rows=(begin, end)")
        _cuda(resid_bcast, "resid_bcast", torch.bfloat16)
        _req(resid_bcast.dim() == 2 and resid_bcast.shape[1] == D and resid_bcast.stride(1) == 1
             and resid_bcast.shape[0] * resid_bcast_rows >= rows, "resid_bcast must be a (groups, D) bf16 view")
        _req(0 <= resid_rows[0] <= resid_rows[1] <= rows, "resid_rows out of range")
        a.resid_bcast, a.resid_bcast_ld, a.resid_bcast_rows = resid_bcast.data_ptr(), resid_bcast.stride(0), resid_bcast_rows
        a.resid_row_begin, a.resid_row_end = resid_rows
        if resid_out_gate is not None:
            _cuda(resid_out_gate, "resid_out_gate", torch.float32)
            _req(resid_out_gate.dim() == 2 and resid_out_gate.shape[1] == D and resid_out_gate.stride(1) == 1
                 and resid_out_gate.shape[0] * resid_out_gate_rows >= rows, "resid_out_gate must be a (groups, D) view")
            a.resid_out_gate, a.resid_out_gate_ld = resid_out_gate.data_ptr(), resid_out_gate.stride(0)
            a.resid_out_gate_rows = resid_out_gate_rows
    else:
        _req(resid_out_gate is None, "resid_out_gate needs resid_bcast")
    a.x, a.rows, a.D = x.data_ptr(), rows, D
    a.ldx = x.stride(0)
    if shift is not None:
        _cuda(shift, "shift", torch.float32)
        _cuda(scale, "scale", torch.float32)
        _req(shift.dim() == 2 and scale.dim() == 2 and shift.shape == scale.shape
             and shift.shape[1] == D and shift.stride(1) == 1 and scale.stride(1) == 1
             and shift.stride(0) == scale.stride(0), "shift/scale must be matching (groups, D) views")
        _req(shift.shape[0] * mod_rows >= rows, "too few modulation rows")
        a.shift, a.scale, a.mod_ld, a.mod_rows = shift.data_ptr(), scale.data_ptr(), shift.stride(0), mod_rows
    if shift_tab is not None:
        _cuda(shift_tab, "shift_tab", torch.float32)
        _cuda(scale_tab, "scale_tab", torch.float32)
        _req(shift_tab.shape == (D,) and scale_tab.shape == (D,) and shift_tab.is_contiguous()
             and scale_tab.is_contiguous(), "tables must be contiguous (D,)")
        a.shift_tab, a.scale_tab = shift_tab.data_ptr(), scale_tab.data_ptr()
    if weight is not None:
        _cuda(weight, "weight", torch.float32)
        _req(weight.shape == (D,) and weight.is_contiguous(), "weight must be contiguous (D,)")
        a.weight = weight.data_ptr()
    a.norm, a.act, a.eps = norm, act, eps


def _fp8_pair(rows: int, cols: int, device, out, out_scale, what: str):
    """Checked (or new) e4m3 codes (rows, cols) and fp32 block scales (rows, cols/128) with unit inner strides."""
    if out is None:
        out = torch.empty((rows, cols), device=device, dtype=FP8)
    if out_scale is None:
        out_scale = torch.empty((rows, cols // 128), device=device, dtype=torch.float32)
    _cuda(out, f"{what} out", FP8)
    _cuda(out_scale, f"{what} out_scale", torch.float32)
    _req(out.shape == (rows, cols) and out.stride(1) == 1, f"{what}: out must be ({rows}, {cols}) with unit inner stride")
    _req(out_scale.shape == (rows, cols // 128) and out_scale.stride(1) == 1,
         f"{what}: out_scale must be ({rows}, {cols // 128}) with unit inner stride")
    return out, out_scale


def norm_modulate_fp8(x: torch.Tensor, *, norm: int, out: torch.Tensor | None = None,
                      out_scale: torch.Tensor | None = None, shift: torch.Tensor | None = None,
                      scale: torch.Tensor | None = None, mod_rows: int = 1,
                      shift_tab: torch.Tensor | None = None, scale_tab: torch.Tensor | None = None,
                      weight: torch.Tensor | None = None, eps: float = 1e-6, act: int = ACT_NONE,
                      resid: torch.Tensor | None = None, resid_gate: torch.Tensor | None = None,
                      resid_gate_rows: int = 1, resid_bcast: torch.Tensor | None = None, resid_bcast_rows: int = 1,
                      resid_rows: tuple | None = None, resid_out_gate: torch.Tensor | None = None,
                      resid_out_gate_rows: int = 1):
    """norm_modulate with an fp8 output: returns (codes e4m3 (rows, D), block scales fp32 (rows, D/128)) in the
    1 x 128 block format of include/ln3b200.h.  The residual update of x is the bf16 op's, bit for bit."""
    _cuda(x, "x", torch.float32)
    _req(x.dim() == 2 and x.stride(1) == 1, "x must be (rows, D) with unit inner stride")
    rows, D = x.shape
    _req(D % 128 == 0, f"D={D} must be a multiple of 128")
    out, out_scale = _fp8_pair(rows, D, x.device, out, out_scale, "norm_modulate_fp8")
    f = _lib.NormModulateFp8Args()
    _norm_modulate_inputs(f.base, x, norm=norm, shift=shift, scale=scale, mod_rows=mod_rows, shift_tab=shift_tab,
                          scale_tab=scale_tab, weight=weight, eps=eps, act=act, resid=resid, resid_gate=resid_gate,
                          resid_gate_rows=resid_gate_rows, resid_bcast=resid_bcast, resid_bcast_rows=resid_bcast_rows,
                          resid_rows=resid_rows, resid_out_gate=resid_out_gate, resid_out_gate_rows=resid_out_gate_rows)
    f.out, f.ldo = out.data_ptr(), out.stride(0)
    f.out_scale, f.out_scale_ld = out_scale.data_ptr(), out_scale.stride(0)
    _lib.check(_lib.lib().ln3_norm_modulate_fp8(C.byref(f), _lib.current_stream()), "ln3_norm_modulate_fp8")
    return out, out_scale


def quantize_fp8(x: torch.Tensor, out: torch.Tensor | None = None, out_scale: torch.Tensor | None = None):
    """x fp32 or bf16 (rows, D), D % 128 == 0 -> (e4m3 codes (rows, D), fp32 block scales (rows, D/128)):
    s = fp32(absmax of the 128-column block / 448), code = e4m3 rn-satfinite of fp32(x / s); s = 0 -> zero codes."""
    _cuda(x, "x")
    _req(x.dtype in (torch.float32, torch.bfloat16), f"x must be float32 or bfloat16, got {x.dtype}")
    _req(x.dim() == 2 and x.stride(1) == 1, "x must be (rows, D) with unit inner stride")
    rows, D = x.shape
    _req(D > 0 and D % 128 == 0, f"D={D} must be a positive multiple of 128")
    out, out_scale = _fp8_pair(rows, D, x.device, out, out_scale, "quantize_fp8")
    _lib.check(_lib.lib().ln3_quantize_fp8_rows(
        x.data_ptr(), int(x.dtype == torch.bfloat16), x.stride(0), rows, D, out.data_ptr(), out.stride(0),
        out_scale.data_ptr(), out_scale.stride(0), _lib.current_stream()), "ln3_quantize_fp8_rows")
    return out, out_scale


@torch.no_grad()
def quantize_weight_fp8(w: torch.Tensor):
    """nn.Linear weight (N, K) -> (e4m3 codes (N, K), fp32 per-output-channel scales (N,)), on w's device:
    w_scale = fp32(absmax of the row / 448), codes = torch's float8_e4m3fn cast of fp32(w / w_scale); a zero row has
    scale 0 and zero codes.  Runs once per model (prepare()), not on the hot path."""
    w = w.detach().float()
    amax = w.abs().amax(dim=1)
    s = amax / torch.full_like(amax, FP8_MAX)     # elementwise division (a Python scalar divisor becomes * (1/448))
    q = torch.where(s[:, None] > 0, w / torch.where(s > 0, s, torch.ones_like(s))[:, None], torch.zeros_like(w))
    return q.clamp(-FP8_MAX, FP8_MAX).to(FP8).contiguous(), s.contiguous()


def gemm_fp8(a_q: torch.Tensor, a_scale: torch.Tensor, w_q: torch.Tensor, w_scale: torch.Tensor,
             bias: torch.Tensor | None = None, *, act: int = ACT_NONE, out_kind: int = OUT_BF16,
             out: torch.Tensor | None = None, out_scale: torch.Tensor | None = None,
             head_norm: torch.Tensor | None = None, head_norm_sec_cols: int = 0, head_norm_eps: float = 1e-5):
    """out = epilogue(w_scale[n] * sum_kb a_scale[m, kb] * (a_q[m, kb] . w_q[n, kb])) on the fp8 tensor cores.
    a_q (M, K) and w_q (N, K) e4m3 codes, a_scale (M, K/128) and w_scale (N,) fp32 (format: include/ln3b200.h).
    OUT_BF16 (act NONE, optional head_norm as in `gemm`) returns the bf16 (M, N) output; OUT_FP8 (act NONE or
    GELU_ERF) returns (codes (M, N), block scales (M, N/128)), the A operand of a following gemm_fp8."""
    _cuda(a_q, "a_q", FP8)
    _cuda(w_q, "w_q", FP8)
    _cuda(a_scale, "a_scale", torch.float32)
    _cuda(w_scale, "w_scale", torch.float32)
    _req(a_q.dim() == 2 and w_q.dim() == 2, "a_q and w_q must be 2-D")
    _req(a_q.stride(1) == 1 and w_q.stride(1) == 1, "a_q and w_q must have unit inner stride")
    M, K = a_q.shape
    N, K2 = w_q.shape
    _req(K == K2, f"inner dims differ: {K} vs {K2}")
    _req(K % 128 == 0 and N % 128 == 0, f"K={K} and N={N} must be multiples of 128")
    _req(a_scale.dim() == 2 and a_scale.shape == (M, K // 128) and a_scale.stride(1) == 1,
         f"a_scale must be ({M}, {K // 128}) with unit inner stride")
    _req(w_scale.shape == (N,) and w_scale.is_contiguous(), f"w_scale must be contiguous ({N},)")
    args = _lib.GemmFp8Args()
    if out_kind == OUT_FP8:
        out, out_scale = _fp8_pair(M, N, a_q.device, out, out_scale, "gemm_fp8")
        args.out_scale, args.out_scale_ld = out_scale.data_ptr(), out_scale.stride(0)
    else:
        _req(out_kind == OUT_BF16, "gemm_fp8 writes OUT_BF16 or OUT_FP8")
        if out is None:
            out = torch.empty((M, N), device=a_q.device, dtype=torch.bfloat16)
        _cuda(out, "out", torch.bfloat16)
        _req(out.shape == (M, N) and out.stride(1) == 1, "out must be (M,N) with unit inner stride")
    args.A, args.a_scale, args.W, args.w_scale = a_q.data_ptr(), a_scale.data_ptr(), w_q.data_ptr(), w_scale.data_ptr()
    args.out = out.data_ptr()
    args.M, args.N, args.K = M, N, K
    args.lda, args.ldw, args.ldo, args.a_scale_ld = a_q.stride(0), w_q.stride(0), out.stride(0), a_scale.stride(0)
    if bias is not None:
        _cuda(bias, "bias", torch.float32)
        _req(bias.shape == (N,) and bias.is_contiguous(), "bias must be contiguous (N,)")
        args.bias = bias.data_ptr()
    if head_norm is not None:
        _cuda(head_norm, "head_norm", torch.float32)
        _req(head_norm.dim() == 2 and head_norm.shape[1] == 64 and head_norm.is_contiguous(),
             "head_norm must be contiguous (nsec, 64): the head-RMSNorm epilogue normalises 64-wide heads only")
        args.head_norm_w, args.head_norm_nsec = head_norm.data_ptr(), head_norm.shape[0]
        args.head_norm_sec_cols, args.head_norm_eps = head_norm_sec_cols, head_norm_eps
    args.act, args.out_kind = act, out_kind
    _lib.check(_lib.lib().ln3_gemm_fp8(C.byref(args), _lib.current_stream()), "ln3_gemm_fp8")
    return (out, out_scale) if out_kind == OUT_FP8 else out


def timestep_embedding(t: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """(B,) fp32 timesteps -> (B,256) bf16 [cos | sin] features."""
    _cuda(t, "t", torch.float32)
    _req(t.dim() == 1 and t.is_contiguous(), "t must be contiguous (B,)")
    if out is None:
        out = torch.empty((t.shape[0], 256), device=t.device, dtype=torch.bfloat16)
    _cuda(out, "out", torch.bfloat16)
    _req(out.shape == (t.shape[0], 256) and out.is_contiguous(), "out must be contiguous (B,256)")
    _lib.check(_lib.lib().ln3_timestep_embedding(_lib.ptr(t), t.shape[0], _lib.ptr(out),
                                                 _lib.current_stream()), "ln3_timestep_embedding")
    return out


def patch_embed(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None,
                pos_embed: torch.Tensor | None, in_scale: torch.Tensor | None = None,
                out: torch.Tensor | None = None) -> torch.Tensor:
    """x fp32 (B,3*Cin,S,S) -> fp32 tokens (B, 3*(S/2)^2, D) (roll-out patch embed + pos_embed)."""
    _cuda(x, "x", torch.float32)
    _cuda(weight, "weight", torch.float32)
    _req(x.dim() == 4 and x.is_contiguous() and weight.is_contiguous(), "x/weight must be contiguous")
    B, C3, S, _ = x.shape
    D, Cin = weight.shape[0], weight.shape[1]
    _req(C3 == 3 * Cin and weight.shape[2:] == (2, 2), "patch_embed expects 3 planes and 2x2 patches")
    T = 3 * (S // 2) ** 2
    if out is None:
        out = torch.empty((B, T, D), device=x.device, dtype=torch.float32)
    _req(out.shape == (B, T, D) and out.is_contiguous() and out.dtype == torch.float32, "bad out")
    a = _lib.PatchEmbedArgs()
    a.x, a.weight, a.tokens = x.data_ptr(), weight.data_ptr(), out.data_ptr()
    if bias is not None:
        _cuda(bias, "bias", torch.float32)
        a.bias = bias.data_ptr()
    if pos_embed is not None:
        _cuda(pos_embed, "pos_embed", torch.float32)
        _req(pos_embed.numel() == T * D and pos_embed.is_contiguous(), "pos_embed must be (1,T,D)")
        a.pos_embed = pos_embed.data_ptr()
    if in_scale is not None:
        _cuda(in_scale, "in_scale", torch.float32)
        _req(in_scale.shape == (B,) and in_scale.is_contiguous(), "in_scale must be (B,)")
        a.in_scale = in_scale.data_ptr()
    a.B, a.Cin, a.S, a.D = B, Cin, S, D
    _lib.check(_lib.lib().ln3_patch_embed(C.byref(a), _lib.current_stream()), "ln3_patch_embed")
    return out


PLUCKER_COLS = 9 * 14 * 14          # RGB + 6 Plücker channels of a 14x14 patch


def plucker_patchify(image: torch.Tensor, cams: torch.Tensor, out: torch.Tensor | None = None,
                     ldo: int = 1792) -> torch.Tensor:
    """image fp32 (N,3,224,224) pre-processed views, cams fp32 (N,25) -> the bf16 patch operand (N*256, ldo) of the
    9-channel 14x14 patch embedding: RGB | o x d | d per pixel in Conv2d.weight.reshape(D, -1) column order,
    columns [1764, ldo) zero (FrozenDinov2ImageEmbedderMVPlucker's gen_rays / get_plucker_ray / cat / cast)."""
    _cuda(image, "image", torch.float32)
    _cuda(cams, "cams", torch.float32)
    _req(image.dim() == 4 and image.shape[1:] == (3, 224, 224) and image.is_contiguous(),
         "image must be contiguous (N,3,224,224)")
    N = image.shape[0]
    _req(cams.shape == (N, 25) and cams.is_contiguous(), "cams must be contiguous (N,25)")
    if out is None:
        out = torch.empty((N * 256, ldo), device=image.device, dtype=torch.bfloat16)
    _cuda(out, "out", torch.bfloat16)
    _req(out.dim() == 2 and out.shape[0] == N * 256 and out.shape[1] >= PLUCKER_COLS and out.stride(1) == 1,
         "out must be (N*256, >= 1764) with unit inner stride")
    # the kernel writes whole rows of `ldo` elements (zero padding up to the pitch)
    _req(out.shape[1] % 8 == 0 and (N == 0 or out.stride(0) == out.shape[1]),
         "out rows must be a multiple of 8 elements wide, with the row pitch equal to the width")
    for nm, t_ in (("image", image), ("cams", cams), ("out", out)):
        _req(t_.data_ptr() % 16 == 0, f"{nm} must be 16-byte aligned")
    a = _lib.PluckerPatchifyArgs()
    a.image, a.cams, a.out, a.N, a.ldo = image.data_ptr(), cams.data_ptr(), out.data_ptr(), N, out.shape[1]
    _lib.check(_lib.lib().ln3_plucker_patchify(C.byref(a), _lib.current_stream()), "ln3_plucker_patchify")
    return out


def final_layer(x: torch.Tensor, shift: torch.Tensor, scale: torch.Tensor, weight: torch.Tensor,
                bias: torch.Tensor | None, S: int, *, shift_tab: torch.Tensor | None = None,
                scale_tab: torch.Tensor | None = None, out: torch.Tensor | None = None) -> torch.Tensor:
    """tokens fp32 (B,T,D) -> fp32 (B, 3*Cout, S, S): LN + modulate + Linear + unpatchify."""
    _cuda(x, "x", torch.float32)
    _req(x.dim() == 3 and x.is_contiguous(), "x must be contiguous (B,T,D)")
    B, T, D = x.shape
    _req(T == 3 * (S // 2) ** 2, "token count does not match S")
    _cuda(weight, "weight", torch.float32)
    _req(weight.dim() == 2 and weight.shape[1] == D and weight.is_contiguous(), "weight must be (4*Cout, D)")
    Cout = weight.shape[0] // 4
    for n_, t_ in (("shift", shift), ("scale", scale)):
        _cuda(t_, n_, torch.float32)
        _req(t_.dim() == 2 and t_.shape == (B, D) and t_.stride(1) == 1, f"{n_} must be a (B,D) view")
    _req(shift.stride(0) == scale.stride(0), "shift/scale row strides differ")
    if out is None:
        out = torch.empty((B, 3 * Cout, S, S), device=x.device, dtype=torch.float32)
    _req(out.shape == (B, 3 * Cout, S, S) and out.is_contiguous() and out.dtype == torch.float32, "bad out")
    a = _lib.FinalLayerArgs()
    a.x, a.shift, a.scale, a.weight, a.out = (x.data_ptr(), shift.data_ptr(), scale.data_ptr(),
                                              weight.data_ptr(), out.data_ptr())
    if bias is not None:
        _cuda(bias, "bias", torch.float32)
        a.bias = bias.data_ptr()
    _req((shift_tab is None) == (scale_tab is None), "shift_tab and scale_tab must be given together")
    if shift_tab is not None:
        _cuda(shift_tab, "shift_tab", torch.float32)
        _cuda(scale_tab, "scale_tab", torch.float32)
        _req(shift_tab.shape == (D,) and scale_tab.shape == (D,) and shift_tab.is_contiguous()
             and scale_tab.is_contiguous(), "tables must be contiguous (D,)")
        a.shift_tab, a.scale_tab = shift_tab.data_ptr(), scale_tab.data_ptr()
    a.B, a.S, a.D, a.Cout, a.mod_ld = B, S, D, Cout, shift.stride(0)
    _lib.check(_lib.lib().ln3_final_layer(C.byref(a), _lib.current_stream()), "ln3_final_layer")
    return out


def sampler_affine_update(x: torch.Tensor, coef: torch.Tensor, m0: torch.Tensor,
                          m1: torch.Tensor | None = None, noise: torch.Tensor | None = None,
                          out: torch.Tensor | None = None) -> torch.Tensor:
    """x_out[b] = a_b x[b] + w0_b m0[b] + w1_b m1[b] + s_b noise[b]; coef (B,4) fp32."""
    _cuda(x, "x", torch.float32)
    _cuda(coef, "coef", torch.float32)
    B = x.shape[0]
    _req(coef.shape == (B, 4) and coef.is_contiguous(), "coef must be contiguous (B,4)")
    n = x[0].numel()
    for nm, t_ in (("x", x), ("m0", m0), ("m1", m1), ("noise", noise)):
        if t_ is None:
            continue
        _cuda(t_, nm, torch.float32)
        _req(t_.is_contiguous() and t_.shape[0] == B and t_[0].numel() == n, f"{nm} must be contiguous, same shape as x")
        _req(t_.data_ptr() % 16 == 0, f"{nm} must be 16-byte aligned (the kernel uses 128-bit accesses)")
    _req(n % 4 == 0, "elements per sample must be a multiple of 4")
    if out is None:
        out = torch.empty_like(x)
    _req(out.is_contiguous() and out.shape == x.shape and out.dtype == torch.float32 and out.data_ptr() % 16 == 0, "bad out")
    a = _lib.SamplerUpdateArgs()
    a.x, a.m0, a.coef, a.x_out = x.data_ptr(), m0.data_ptr(), coef.data_ptr(), out.data_ptr()
    a.m1 = m1.data_ptr() if m1 is not None else None
    a.noise = noise.data_ptr() if noise is not None else None
    a.B, a.n_per_sample = B, n
    _lib.check(_lib.lib().ln3_sampler_affine_update(C.byref(a), _lib.current_stream()),
               "ln3_sampler_affine_update")
    return out


SAMPLER_STEP_COEFS = 12   # (k0, k1, k2, a, b, c, h0, h1, h2, s, 0, 0)


def sampler_step(x: torch.Tensor, x_eval: torch.Tensor, coef: torch.Tensor, net_u: torch.Tensor,
                 net_c: torch.Tensor | None = None, hist=(), noise: torch.Tensor | None = None, *,
                 x_out: torch.Tensor | None = None, eval_out: torch.Tensor | None = None,
                 hist_out: torch.Tensor | None = None) -> None:
    """One sampler evaluation's elementwise tail (include/ln3b200.h, ln3_sampler_step_args), per sample b:
        e = k0 x_eval + k1 net_u + k2 net_c
        v = a x + b x_eval + c e + h0 hist[0] + h1 hist[1] + h2 hist[2] + s noise
        x_out[b] = v;  eval_out[b] = eval_out[B+b] = v;  hist_out[b] = e
    coef (B, 12) fp32.  Every tensor is CUDA fp32, contiguous and 16-byte aligned, with B rows of n elements
    (n % 4 == 0) except eval_out's 2B.  Outputs are written in place; at least one is required.  No output may
    overlap another output or an input, except x_out is x and eval_out starting at x_eval."""
    _cuda(x, "x", torch.float32)
    B = x.shape[0]
    n = x[0].numel() if B else 0
    _cuda(coef, "coef", torch.float32)
    _req(coef.shape == (B, SAMPLER_STEP_COEFS) and coef.is_contiguous(), "coef must be contiguous (B, 12)")
    hist = tuple(hist)
    _req(len(hist) <= 3, "at most 3 history operands")
    hist = hist + (None,) * (3 - len(hist))
    ins = [("x", x), ("x_eval", x_eval), ("net_u", net_u), ("net_c", net_c), ("hist[0]", hist[0]),
           ("hist[1]", hist[1]), ("hist[2]", hist[2]), ("noise", noise)]
    outs = [("x_out", x_out, B), ("eval_out", eval_out, 2 * B), ("hist_out", hist_out, B)]
    _req(x_eval is not None and net_u is not None, "x_eval and net_u are required")
    _req(any(t_ is not None for _, t_, _ in outs), "at least one of x_out, eval_out, hist_out is required")
    _req(n % 4 == 0, "elements per sample must be a multiple of 4")
    for nm, t_, rows in [(nm, t_, B) for nm, t_ in ins] + outs:
        if t_ is None:
            continue
        _cuda(t_, nm, torch.float32)
        _req(t_.is_contiguous() and t_.shape[0] == rows and t_.numel() == rows * n,
             f"{nm} must be contiguous with {rows} rows of {n} elements")
        _req(t_.data_ptr() % 16 == 0, f"{nm} must be 16-byte aligned (the kernel uses 128-bit accesses)")
    _req(coef.data_ptr() % 16 == 0, "coef must be 16-byte aligned")

    def span(t_):
        return t_.data_ptr(), t_.data_ptr() + t_.numel() * 4

    in_spans = [(nm, t_) for nm, t_ in ins if t_ is not None] + [("coef", coef)]
    out_spans = [(nm, t_) for nm, t_, _ in outs if t_ is not None]
    for i, (on, ot) in enumerate(out_spans):
        o0, o1 = span(ot)
        for nm, t_ in out_spans[i + 1:] + in_spans:
            a0, a1 = span(t_)
            alias = ot.data_ptr() == t_.data_ptr() and (on, nm) in (("x_out", "x"), ("eval_out", "x_eval"))
            _req(alias or o1 <= a0 or a1 <= o0, f"{on} overlaps {nm}")
    a = _lib.SamplerStepArgs()
    a.x, a.x_eval, a.net_u, a.coef = x.data_ptr(), x_eval.data_ptr(), net_u.data_ptr(), coef.data_ptr()
    ptr = lambda t_: t_.data_ptr() if t_ is not None else None
    a.net_c, a.noise = ptr(net_c), ptr(noise)
    for j in range(3):
        a.hist[j] = ptr(hist[j])
    a.x_out, a.eval_out, a.hist_out = ptr(x_out), ptr(eval_out), ptr(hist_out)
    a.B, a.n_per_sample = B, n
    _lib.check(_lib.lib().ln3_sampler_step(C.byref(a), _lib.current_stream()), "ln3_sampler_step")


SDE_DRIFT, SDE_VELOCITY, SDE_SCORE = 0, 1, 2   # LN3_SDE_*: d = v + D sc | v | sc


def flow_sde_step(y: torch.Tensor, f: torch.Tensor, *, cfg_scale: float, t: float, var: float,
                  diffusion: float = 0.0, mode: int = SDE_DRIFT, x: torch.Tensor | None = None,
                  hist: torch.Tensor | None = None, noise: torch.Tensor | None = None,
                  x_out: torch.Tensor | None = None, cx=(0.0,) * 5, y_out: torch.Tensor | None = None,
                  cy=(0.0,) * 5, hist_out: torch.Tensor | None = None) -> None:
    """One drift evaluation's elementwise tail of the flow SDE samplers (include/ln3b200.h, ln3_flow_sde_step_args)
    over the 2R-row CFG state (conditional rows first), per row r and j = r mod R:
        v = f[R+j] + s (f[j] - f[R+j]);  sc = (t v - y[r]) / var;  d = v + D sc | v | sc  (mode)
        o(k) = k0 x[r] + k1 y[r] + k2 d + k3 hist[r] + k4 noise[noise_row(r)]
        x_out[r] = o(cx);  y_out[r] = o(cy);  hist_out[r] = d
    `noise` is one (2N, ...) draw: rows [0, N) serve the conditional half and [N, 2N) the unconditional half of
    every one of the R / N conditions.  Every tensor is CUDA fp32, contiguous and 16-byte aligned, with 2R rows of n
    elements (n % 4 == 0).  Outputs are written in place; at least one is required.  No output may overlap another
    output or an input, except x_out is x and y_out is y (checked by the library)."""
    _cuda(y, "y", torch.float32)
    _req(y.dim() >= 1 and y.shape[0] % 2 == 0, "y must hold 2R rows")
    R2 = y.shape[0]
    n = y[0].numel() if R2 else 0
    _req(n % 4 == 0, "elements per row must be a multiple of 4")
    _req(mode in (SDE_DRIFT, SDE_VELOCITY, SDE_SCORE), f"unknown mode {mode}")
    _req(any(o is not None for o in (x_out, y_out, hist_out)), "at least one of x_out, y_out, hist_out is required")
    N = 0
    if noise is not None:
        _req(noise.dim() >= 1 and noise.shape[0] % 2 == 0, "noise must hold 2N rows")
        N = noise.shape[0] // 2
    for nm, t_, rows in (("y", y, R2), ("f", f, R2), ("x", x, R2), ("hist", hist, R2), ("noise", noise, 2 * N),
                         ("x_out", x_out, R2), ("y_out", y_out, R2), ("hist_out", hist_out, R2)):
        if t_ is None:
            continue
        _cuda(t_, nm, torch.float32)
        _req(t_.is_contiguous() and t_.shape[0] == rows and t_.numel() == rows * n,
             f"{nm} must be contiguous with {rows} rows of {n} elements")
        _req(t_.data_ptr() % 16 == 0, f"{nm} must be 16-byte aligned (the kernel uses 128-bit accesses)")
    _req(len(cx) == 5 and len(cy) == 5, "cx and cy hold (a, b, c, h, sigma)")
    a = _lib.FlowSdeStepArgs()
    ptr = lambda t_: t_.data_ptr() if t_ is not None else None
    a.x, a.y, a.f, a.hist, a.noise = ptr(x), y.data_ptr(), f.data_ptr(), ptr(hist), ptr(noise)
    a.x_out, a.y_out, a.hist_out = ptr(x_out), ptr(y_out), ptr(hist_out)
    for k in range(5):
        a.cx[k], a.cy[k] = float(cx[k]), float(cy[k])
    a.cfg_scale, a.t, a.var, a.diffusion = float(cfg_scale), float(t), float(var), float(diffusion)
    a.mode, a.R, a.N, a.n = int(mode), R2 // 2, N, n
    _lib.check(_lib.lib().ln3_flow_sde_step(C.byref(a), _lib.current_stream()), "ln3_flow_sde_step")


# ---------------------------------------------------------------------------------------------- grouped dopri5
ODE_GROUP_BYTES = C.sizeof(_lib.OdeGroup)
_ODE_F64 = ("t", "dt", "t_prev", "dt_step", "ratio", "aux")
_ODE_I32 = ("nfe", "accepted", "rejected", "status", "event")


def ode_state(n_groups: int, t0: float, device) -> torch.Tensor:
    """A fresh per-group state block (uint8 (G, sizeof(ln3_ode_group))) on `device`: t = t_prev = t0, running."""
    _req(n_groups > 0, "n_groups must be positive")
    st = torch.zeros(n_groups, ODE_GROUP_BYTES, dtype=torch.uint8)
    f = st.view(torch.float64)
    f[:, 0] = t0
    f[:, 2] = t0
    return st.to(device)


def ode_state_fields(state: torch.Tensor) -> dict:
    """The fields of a state block (device or host copy) as CPU tensors: float64 t ... aux, int32 nfe ... event."""
    st = state.detach().cpu().contiguous()
    f, i = st.view(torch.float64), st.view(torch.int32)
    out = {k: f[:, j].clone() for j, k in enumerate(_ODE_F64)}
    out.update({k: i[:, 12 + j].clone() for j, k in enumerate(_ODE_I32)})
    return out


def _ode_buf(t_: torch.Tensor, nm: str, B: int, n: int) -> None:
    _cuda(t_, nm, torch.float32)
    _req(t_.is_contiguous() and t_.dim() >= 1 and t_.shape[0] == B and t_.numel() == B * n,
         f"{nm} must be contiguous with the state's shape")
    _req(t_.data_ptr() % 16 == 0, f"{nm} must be 16-byte aligned (the kernels use 128-bit accesses)")


def ode_args(y: torch.Tensor, f0: torch.Tensor, y_stage: torch.Tensor, t_rows: torch.Tensor, out: torch.Tensor,
             row_group: torch.Tensor, state: torch.Tensor, *, t_end: float, rtol: float, atol: float,
             safety: float = 0.9, ifactor: float = 10.0, dfactor: float = 0.2,
             max_num_steps: int = 2 ** 31 - 1) -> _lib.OdeArgs:
    """The argument block of the ln3_ode_* entry points.  y, f0, y_stage, out: contiguous fp32 (B, ...) CUDA tensors;
    t_rows fp32 (B,); row_group int32 (B,) group of each row (any device: a host and a device copy are kept);
    state from `ode_state`.  The returned struct holds references to every tensor it points to."""
    _cuda(y, "y", torch.float32)
    B = y.shape[0]
    n = y.numel() // max(B, 1)
    _req(B > 0 and n > 0 and n % 4 == 0, "elements per row must be a positive multiple of 4")
    for nm, t_ in (("y", y), ("f0", f0), ("y_stage", y_stage), ("out", out)):
        _ode_buf(t_, nm, B, n)
    _cuda(t_rows, "t_rows", torch.float32)
    _req(t_rows.shape == (B,) and t_rows.is_contiguous(), "t_rows must be contiguous (B,)")
    _req(row_group.dim() == 1 and row_group.shape[0] == B, "row_group must be (B,)")
    rg_host = row_group.detach().to("cpu", torch.int32).contiguous()
    G = state.shape[0] if state.dim() == 2 else 0
    _cuda(state, "state", torch.uint8)
    _req(state.shape == (G, ODE_GROUP_BYTES) and state.is_contiguous() and state.data_ptr() % 8 == 0,
         "state must be an ode_state block")
    rg_dev = rg_host.to(y.device)
    ws = torch.empty(int(_lib.lib().ln3_ode_workspace_bytes(B, n)), dtype=torch.uint8, device=y.device)
    a = _lib.OdeArgs()
    a.y, a.f0, a.y_stage, a.t_rows, a.out = (t_.data_ptr() for t_ in (y, f0, y_stage, t_rows, out))
    a.row_group, a.row_group_host, a.state = rg_dev.data_ptr(), rg_host.data_ptr(), state.data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    a.B, a.G, a.n_per_sample = B, G, n
    a.t_end, a.rtol, a.atol, a.safety, a.ifactor, a.dfactor = t_end, rtol, atol, safety, ifactor, dfactor
    a.max_num_steps = max_num_steps
    a.tensors = (y, f0, y_stage, t_rows, out, rg_dev, rg_host, state, ws)
    return a


def _ode_k(a: _lib.OdeArgs, ks) -> None:
    _req(len(ks) <= 6, "at most six stage derivatives")
    for i in range(6):
        if i < len(ks):
            _ode_buf(ks[i], f"k[{i}]", a.B, a.n_per_sample)
            _req(ks[i].device == a.tensors[0].device, f"k[{i}] must be on the state's device")
            a.k[i] = ks[i].data_ptr()
        else:
            a.k[i] = None
    a.ks = tuple(ks)                                  # keeps the stage tensors alive with the argument block


def ode_stages(method: int = _lib.ODE_METHODS["dopri5"]) -> int:
    """ln3_ode_stages: the stage forwards per attempt of an ln3_ode_rk_* method (_lib.ODE_METHODS)."""
    n = int(_lib.lib().ln3_ode_stages(int(method)))
    if n < 0:
        _lib.check(n, "ln3_ode_stages")
    return n


def ode_stage(a: _lib.OdeArgs, stage: int, ks=(), method: int = _lib.ODE_METHODS["dopri5"]) -> None:
    """ln3_ode_rk_stage: y_stage and t_rows of stage `stage` (1..S of `method`, reading f0 and ks[:stage-1]) or of
    the initial-step probe (stage 0)."""
    _req(0 <= stage <= 6 and len(ks) >= max(stage - 1, 0), "stage i needs the i-1 previous stage derivatives")
    _ode_k(a, ks)
    _lib.check(_lib.lib().ln3_ode_rk_stage(C.byref(a), int(method), stage, _lib.current_stream()), "ln3_ode_stage")


def ode_initial_step(a: _lib.OdeArgs, phase: int, k0: torch.Tensor | None = None,
                     method: int = _lib.ODE_METHODS["dopri5"]) -> None:
    """ln3_ode_rk_initial_step: phase 0 -> h0 per group; phase 1 (k0 = forward at the stage-0 probe) -> first dt."""
    _req(phase in (0, 1) and (phase == 0 or k0 is not None), "phase 1 needs k0")
    _ode_k(a, () if k0 is None else (k0,))
    _lib.check(_lib.lib().ln3_ode_rk_initial_step(C.byref(a), int(method), phase, _lib.current_stream()),
               "ln3_ode_initial_step")


def ode_step(a: _lib.OdeArgs, ks, method: int = _lib.ODE_METHODS["dopri5"]) -> None:
    """ln3_ode_rk_step: error ratio, accept / reject, next dt, commit and dense output, from the S stage
    derivatives of `method` (six for dopri5)."""
    _req(len(ks) == ode_stages(method), "ode_step needs one stage derivative per stage of the method")
    _ode_k(a, ks)
    _lib.check(_lib.lib().ln3_ode_rk_step(C.byref(a), int(method), _lib.current_stream()), "ln3_ode_step")


def generate_rays(cams: torch.Tensor, res: int):
    """cams fp32 (V,25) -> ray_o, ray_d fp32 (V, res*res, 3) (RaySampler.forward)."""
    _cuda(cams, "cams", torch.float32)
    _req(cams.dim() == 2 and cams.shape[1] == 25 and cams.is_contiguous(), "cams must be contiguous (V,25)")
    V = cams.shape[0]
    o = torch.empty((V, res * res, 3), device=cams.device, dtype=torch.float32)
    d = torch.empty_like(o)
    _lib.check(_lib.lib().ln3_generate_rays(_lib.ptr(cams), V, res, _lib.ptr(o), _lib.ptr(d),
                                            _lib.current_stream()), "ln3_generate_rays")
    return o, d


def planes_to_channels_last(planes: torch.Tensor) -> torch.Tensor:
    """(N, 96, H, W) or (N, 3, 32, H, W) fp32 -> (N, 3, H, W, 32) fp32."""
    _cuda(planes, "planes", torch.float32)
    _req(planes.is_contiguous(), "planes must be contiguous")
    if planes.dim() == 4:
        N, C3, H, W = planes.shape
        _req(C3 == 96, "planes must have 3*32 channels")
    else:
        N, three, C, H, W = planes.shape
        _req(three == 3 and C == 32, "planes must be (N,3,32,H,W)")
    out = torch.empty((N, 3, H, W, 32), device=planes.device, dtype=torch.float32)
    _lib.check(_lib.lib().ln3_planes_to_channels_last(_lib.ptr(planes), N, 32, H, W, _lib.ptr(out),
                                                      _lib.current_stream()),
               "ln3_planes_to_channels_last")
    return out


def pack_frames(image: torch.Tensor, depth: torch.Tensor | None = None, lut_u8: torch.Tensor | None = None,
                out: torch.Tensor | None = None) -> torch.Tensor:
    """image (N,3,H,W) fp32 in [-1,1] [+ depth (N,1,H,W) fp32, lut_u8 (256,3) uint8 colormap bytes] ->
    uint8 HWC video frames (N, H, W, 3), or (N, H, 2W, 3) = [image | colour-mapped, per-view normalised
    depth] (the frame TrainLoopDiffusionWithRec.render_video_given_triplane appends,
    nsr/train_util_diffusion.py:292-376)."""
    _cuda(image, "image", torch.float32)
    _req(image.dim() == 4 and image.shape[1] == 3 and image.is_contiguous(), "image must be contiguous (N,3,H,W)")
    N, _, H, W = image.shape
    _req(W % 4 == 0, "W must be a multiple of 4")
    a = _lib.PackFramesArgs()
    Wout = W
    ws = None
    if depth is not None:
        _cuda(depth, "depth", torch.float32)
        _req(depth.shape == (N, 1, H, W) and depth.is_contiguous(), "depth must be contiguous (N,1,H,W)")
        _req(lut_u8 is not None, "depth needs the colormap byte table")
        _cuda(lut_u8, "lut_u8", torch.uint8)
        _req(lut_u8.shape == (256, 3) and lut_u8.is_contiguous(), "lut_u8 must be contiguous (256,3) uint8")
        ws = torch.empty(2 * N, device=image.device, dtype=torch.float32)
        a.depth, a.lut, a.workspace = depth.data_ptr(), lut_u8.data_ptr(), ws.data_ptr()
        Wout = 2 * W
    if out is None:
        out = torch.empty((N, H, Wout, 3), device=image.device, dtype=torch.uint8)
    _cuda(out, "out", torch.uint8)
    _req(out.shape == (N, H, Wout, 3) and out.is_contiguous(), "out must be contiguous (N,H,Wout,3) uint8")
    a.image, a.out, a.N, a.H, a.W = image.data_ptr(), out.data_ptr(), N, H, W
    _lib.check(_lib.lib().ln3_pack_frames(C.byref(a), _lib.current_stream()), "ln3_pack_frames")
    return out


def render_views(planes_cl: torch.Tensor, ray_o: torch.Tensor, ray_d: torch.Tensor,
                 noise_coarse: torch.Tensor, noise_fine: torch.Tensor, osg: tuple, *,
                 view_obj: torch.Tensor | None = None, views_per_obj: int = 0, group_size: int = 1,
                 box_warp: float = 0.9, bbox_min: float = -0.45, bbox_max: float = 0.45,
                 white_back: bool = True, debug: bool = False, mlp_tf32: bool = False,
                 image_width: int | None = None, samples_per_ray: int = 64):
    """Fused ImportanceRenderer.forward for V views.  Returns dict(rgb (V,3,M), depth (V,1,M),
    weights (V,1,M)) (+ debug index tensors).  mlp_tf32: evaluate the OSG MLP on the tensor cores (TF32
    operands, fp32 accumulate; pixel error ~1e-4 rel-L2) instead of exact fp32.  samples_per_ray S: the coarse and
    the importance sample count (64 or 96); the noise tensors hold V*M*S values."""
    for nm, t_ in (("planes_cl", planes_cl), ("ray_o", ray_o), ("ray_d", ray_d),
                   ("noise_coarse", noise_coarse), ("noise_fine", noise_fine)):
        _cuda(t_, nm, torch.float32)
        _req(t_.is_contiguous(), f"{nm} must be contiguous")
    _req(planes_cl.dim() == 5 and planes_cl.shape[1] == 3 and planes_cl.shape[4] == 32,
         "planes_cl must be (N,3,H,W,32)")
    V, M, _ = ray_o.shape
    _req(ray_d.shape == (V, M, 3), "ray_d shape")
    S = int(samples_per_ray)
    _req(S in (64, 96), f"samples_per_ray must be 64 or 96, got {samples_per_ray}")
    _req(noise_coarse.numel() == V * M * S and noise_fine.numel() == V * M * S,
         f"noise tensors must hold V*M*{S} values")
    w1, b1, w2, b2 = osg
    for nm, t_, shp in (("w1", w1, (64, 32)), ("b1", b1, (64,)), ("w2", w2, (4, 64)), ("b2", b2, (4,))):
        _cuda(t_, nm, torch.float32)
        _req(tuple(t_.shape) == shp and t_.is_contiguous(), f"{nm} must be contiguous {shp}")
    dev = ray_o.device
    a = _lib.RenderArgs()
    if view_obj is not None:
        _req(view_obj.is_cuda and view_obj.dtype == torch.int32 and view_obj.shape == (V,), "view_obj int32 (V,)")
        a.view_obj = view_obj.data_ptr()
    else:
        _req(views_per_obj > 0, "need view_obj or views_per_obj")
    rgb = torch.empty((V, 3, M), device=dev, dtype=torch.float32)
    depth = torch.empty((V, 1, M), device=dev, dtype=torch.float32)
    wts = torch.empty((V, 1, M), device=dev, dtype=torch.float32)
    nbytes = _lib.lib().ln3_render_workspace_bytes(V, M, group_size)
    ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
    a.planes_cl, a.ray_o, a.ray_d = planes_cl.data_ptr(), ray_o.data_ptr(), ray_d.data_ptr()
    a.noise_coarse, a.noise_fine = noise_coarse.data_ptr(), noise_fine.data_ptr()
    a.w1, a.b1, a.w2, a.b2 = w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr()
    a.rgb, a.depth, a.weights = rgb.data_ptr(), depth.data_ptr(), wts.data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), nbytes
    out = dict(rgb=rgb, depth=depth, weights=wts)
    if debug:
        out["inbox"] = torch.empty((V * M, 2 * S), device=dev, dtype=torch.uint8)
        out["inds"] = torch.empty((V * M, S), device=dev, dtype=torch.int32)
        out["order"] = torch.empty((V * M, 2 * S), device=dev, dtype=torch.int32)
        out["z_fine"] = torch.empty((V * M, S), device=dev, dtype=torch.float32)
        a.dbg_inbox, a.dbg_inds = out["inbox"].data_ptr(), out["inds"].data_ptr()
        a.dbg_order, a.dbg_zfine = out["order"].data_ptr(), out["z_fine"].data_ptr()
    a.V, a.M, a.H, a.W, a.C = V, M, planes_cl.shape[2], planes_cl.shape[3], 32
    a.S, a.S_importance, a.hidden_dim, a.decoder_output_dim = S, S, 64, 3
    a.group_size, a.views_per_obj, a.white_back = group_size, views_per_obj, int(white_back)
    a.box_warp, a.bbox_min, a.bbox_max = box_warp, bbox_min, bbox_max
    a.mlp_precision = _lib.MLP_TF32 if mlp_tf32 else _lib.MLP_FP32
    a.image_w = _render_image_width(M, image_width)
    _lib.check(_lib.lib().ln3_render_views(C.byref(a), _lib.current_stream()), "ln3_render_views")
    return out


def _render_image_width(M: int, image_width: int | None) -> int:
    # rays in RaySampler order (m = y*W + x): square views get the 4x4 pixel-tile schedule; image_width=0 forces
    # the plain ray order (rays that are not an image, e.g. PatchRaySampler training patches)
    if image_width is None:
        r = int(round(M ** 0.5))
        image_width = r if r * r == M else 0
    return int(image_width)


def render_tile_width(M: int, image_width: int | None = None) -> int:
    """The schedule render_views(..., image_width=image_width) takes for M rays per view: the width of the image
    whose 4x4 pixel tiles the kernel walks, or 0 for the plain ray order (16 consecutive rays per work item)."""
    return int(_lib.lib().ln3_render_tile_width(M, _render_image_width(M, image_width)))


def query_points(planes_cl: torch.Tensor, osg: tuple, *, points: torch.Tensor | None = None,
                 grid_size: int = 0, aabb_min=(-0.45,) * 3, aabb_max=(0.45,) * 3, box_warp: float = 0.9,
                 mlp_tf32: bool = False):
    """ImportanceRenderer._run_model at arbitrary points: planes_cl (N,3,H,W,32) channels-last,
    points (N,P,3) fp32 or None for the reference's linspace grid of grid_size^3 points over the aabb.
    Returns sigma (N,P,1) (raw density logit) and rgb (N,P,3)."""
    _cuda(planes_cl, "planes_cl", torch.float32)
    _req(planes_cl.dim() == 5 and planes_cl.shape[1] == 3 and planes_cl.shape[4] == 32 and planes_cl.is_contiguous(),
         "planes_cl must be contiguous (N,3,H,W,32)")
    N = planes_cl.shape[0]
    a = _lib.QueryPointsArgs()
    if points is not None:
        _cuda(points, "points", torch.float32)
        _req(points.dim() == 3 and points.shape[0] == N and points.shape[2] == 3 and points.is_contiguous(),
             "points must be contiguous (N,P,3)")
        P = points.shape[1]
        a.points = points.data_ptr()
    else:
        _req(grid_size >= 2, "need points or grid_size >= 2")
        P = grid_size ** 3
        a.grid_size = grid_size
        a.aabb_min_x, a.aabb_min_y, a.aabb_min_z = (float(v) for v in aabb_min)
        a.aabb_max_x, a.aabb_max_y, a.aabb_max_z = (float(v) for v in aabb_max)
    w1, b1, w2, b2 = osg
    for nm, t_, shp in (("w1", w1, (64, 32)), ("b1", b1, (64,)), ("w2", w2, (4, 64)), ("b2", b2, (4,))):
        _cuda(t_, nm, torch.float32)
        _req(tuple(t_.shape) == shp and t_.is_contiguous(), f"{nm} must be contiguous {shp}")
    sigma = torch.empty((N, P, 1), device=planes_cl.device, dtype=torch.float32)
    rgb = torch.empty((N, P, 3), device=planes_cl.device, dtype=torch.float32)
    a.planes_cl, a.sigma, a.rgb, a.P = planes_cl.data_ptr(), sigma.data_ptr(), rgb.data_ptr(), P
    a.w1, a.b1, a.w2, a.b2 = w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr()
    a.n_obj, a.C, a.H, a.W = N, 32, planes_cl.shape[2], planes_cl.shape[3]
    a.hidden_dim, a.decoder_output_dim, a.box_warp = 64, 3, box_warp
    a.mlp_precision = _lib.MLP_TF32 if mlp_tf32 else _lib.MLP_FP32
    _lib.check(_lib.lib().ln3_query_points(C.byref(a), _lib.current_stream()), "ln3_query_points")
    return sigma, rgb


def conv_nhwc(x: torch.Tensor, w_packed: torch.Tensor, bias: torch.Tensor | None, *, ksize: int,
              upsample: bool = False, gn: tuple | None = None, swish: bool = False,
              residual: torch.Tensor | None = None, out: torch.Tensor | None = None,
              tf32: bool = False) -> torch.Tensor:
    """NHWC fp32 conv (stride 1, pad ksize//2); tf32=True runs 3x3 convs on the tensor cores (TF32 operands,
    fp32 accumulate).  x (N,Hin,Win,Cin); w_packed (ksize*ksize, Cin, Cout);
    gn = (scale, shift) (N,Cin) fuses GroupNorm-apply (+ swish) into the input load; upsample = fused
    nearest 2x of the input; residual (N,H,W,Cout) is added to the result."""
    _cuda(x, "x", torch.float32)
    _cuda(w_packed, "w_packed", torch.float32)
    _req(x.dim() == 4 and x.is_contiguous() and w_packed.dim() == 3 and w_packed.is_contiguous(), "bad conv operands")
    N, Hin, Win, Cin = x.shape
    _req(w_packed.shape[0] == ksize * ksize and w_packed.shape[1] == Cin, "weight/ksize mismatch")
    Cout = w_packed.shape[2]
    H, W = (2 * Hin, 2 * Win) if upsample else (Hin, Win)
    if out is None:
        out = torch.empty((N, H, W, Cout), device=x.device, dtype=torch.float32)
    _req(out.shape == (N, H, W, Cout) and out.is_contiguous() and out.dtype == torch.float32, "bad out")
    a = _lib.ConvArgs()
    a.x, a.w, a.out = x.data_ptr(), w_packed.data_ptr(), out.data_ptr()
    if bias is not None:
        _cuda(bias, "bias", torch.float32)
        a.bias = bias.data_ptr()
    if gn is not None:
        sc, sh = gn
        _req(sc.shape == (N, Cin) and sh.shape == (N, Cin) and sc.is_contiguous() and sh.is_contiguous(), "bad gn")
        a.in_scale, a.in_shift = sc.data_ptr(), sh.data_ptr()
    if residual is not None:
        _cuda(residual, "residual", torch.float32)
        _req(residual.shape == out.shape and residual.is_contiguous(), "bad residual")
        a.residual = residual.data_ptr()
    a.N, a.H, a.W, a.Cin, a.Cout = N, H, W, Cin, Cout
    a.ksize, a.upsample, a.in_swish = ksize, int(upsample), int(swish)
    a.precision = _lib.MLP_TF32 if (tf32 and ksize == 3) else _lib.MLP_FP32
    _lib.check(_lib.lib().ln3_conv_nhwc(C.byref(a), _lib.current_stream()), "ln3_conv_nhwc")
    return out


def conv_cout_tile(N: int, H: int, W: int, Cout: int) -> int:
    """The output channels per CTA (32 or 64) conv_nhwc takes for an (N, H, W, Cout) output on the current device."""
    return int(_lib.lib().ln3_conv_cout_tile(N, H, W, Cout))


def downsample_nhwc(x: torch.Tensor, w_packed: torch.Tensor, bias: torch.Tensor | None, *,
                    out: torch.Tensor | None = None, tf32: bool = False) -> torch.Tensor:
    """The encoder's Downsample: 3x3 conv, stride 2, on F.pad(x, (0,1,0,1)).  x (N,H,W,Cin) NHWC fp32 with H, W
    even; w_packed (9, Cin, Cout); returns (N, H/2, W/2, Cout).  tf32=True: TF32 operands, fp32 accumulate."""
    _cuda(x, "x", torch.float32)
    _cuda(w_packed, "w_packed", torch.float32)
    _req(x.dim() == 4 and x.is_contiguous() and w_packed.dim() == 3 and w_packed.is_contiguous(), "bad conv operands")
    N, H, W, Cin = x.shape
    _req(H % 2 == 0 and W % 2 == 0, "downsample needs even H, W")
    _req(w_packed.shape[0] == 9 and w_packed.shape[1] == Cin, "weight must be (9, Cin, Cout)")
    Cout = w_packed.shape[2]
    if out is None:
        out = torch.empty((N, H // 2, W // 2, Cout), device=x.device, dtype=torch.float32)
    _cuda(out, "out", torch.float32)
    _req(out.shape == (N, H // 2, W // 2, Cout) and out.is_contiguous(), "bad out")
    a = _lib.ConvArgs()
    a.x, a.w, a.out = x.data_ptr(), w_packed.data_ptr(), out.data_ptr()
    if bias is not None:
        _cuda(bias, "bias", torch.float32)
        _req(bias.shape == (Cout,) and bias.is_contiguous(), "bias must be contiguous (Cout,)")
        a.bias = bias.data_ptr()
    a.N, a.H, a.W, a.Cin, a.Cout, a.ksize = N, H, W, Cin, Cout, 3
    a.precision = _lib.MLP_TF32 if tf32 else _lib.MLP_FP32
    _lib.check(_lib.lib().ln3_downsample_nhwc(C.byref(a), _lib.current_stream()), "ln3_downsample_nhwc")
    return out


def vae_posterior(moments: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, noise: torch.Tensor | None = None):
    """moments (B,S,S,24) NHWC fp32 -> (mean, logvar, z), each (B,12,S,S) fp32: quant_conv (w (24,8), bias (24,)),
    the soft-clamped logvar and z = mean + exp(0.5 logvar) * noise (noise (B,12,S,S), or None for z = mean)."""
    _cuda(moments, "moments", torch.float32)
    _req(moments.dim() == 4 and moments.shape[3] == 24 and moments.shape[1] == moments.shape[2]
         and moments.is_contiguous(), "moments must be contiguous (B,S,S,24)")
    B, S = moments.shape[0], moments.shape[1]
    for nm, t_, shp in (("w", w, (24, 8)), ("bias", bias, (24,))):
        _cuda(t_, nm, torch.float32)
        _req(tuple(t_.shape) == shp and t_.is_contiguous(), f"{nm} must be contiguous {shp}")
    mean, logvar, z = (torch.empty((B, 12, S, S), device=moments.device, dtype=torch.float32) for _ in range(3))
    a = _lib.VaePosteriorArgs()
    if noise is not None:
        _cuda(noise, "noise", torch.float32)
        _req(noise.shape == (B, 12, S, S) and noise.is_contiguous(), "noise must be contiguous (B,12,S,S)")
        a.noise = noise.data_ptr()
    a.moments, a.w, a.bias = moments.data_ptr(), w.data_ptr(), bias.data_ptr()
    a.mean, a.logvar, a.z, a.B, a.S = mean.data_ptr(), logvar.data_ptr(), z.data_ptr(), B, S
    _lib.check(_lib.lib().ln3_vae_posterior(C.byref(a), _lib.current_stream()), "ln3_vae_posterior")
    return mean, logvar, z


def view_mean_nhwc(x: torch.Tensor, num_frames: int) -> torch.Tensor:
    """x (B*F, S, S, C) NHWC fp32 -> (B, S, S, C): the mean over each object's F = num_frames consecutive views."""
    _cuda(x, "x", torch.float32)
    _req(x.dim() == 4 and x.shape[1] == x.shape[2] and x.is_contiguous(), "x must be contiguous (N,S,S,C)")
    F_ = int(num_frames)
    _req(F_ > 0 and x.shape[0] % F_ == 0, f"x holds {x.shape[0]} views, not a multiple of num_frames={num_frames}")
    N, S, _, Cc = x.shape
    out = torch.empty((N // F_, S, S, Cc), device=x.device, dtype=torch.float32)
    _lib.check(_lib.lib().ln3_view_mean_nhwc(_lib.ptr(x), _lib.ptr(out), N // F_, F_, S, Cc, _lib.current_stream()),
               "ln3_view_mean_nhwc")
    return out


def groupnorm_stats(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int = 32,
                    eps: float = 1e-6):
    """x (N,H,W,C) fp32 NHWC -> per-(image, channel) (scale, shift) of GroupNorm(groups, C, eps)."""
    _cuda(x, "x", torch.float32)
    _req(x.dim() == 4 and x.is_contiguous(), "x must be contiguous NHWC")
    N, H, W, Cc = x.shape
    sc = torch.empty((N, Cc), device=x.device, dtype=torch.float32)
    sh = torch.empty_like(sc)
    _lib.check(_lib.lib().ln3_groupnorm_stats(_lib.ptr(x), _lib.ptr(gamma), _lib.ptr(beta), N, H * W, Cc, groups,
                                              C.c_float(eps), _lib.ptr(sc), _lib.ptr(sh), _lib.current_stream()),
               "ln3_groupnorm_stats")
    return sc, sh


def attn_single_head(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """q/k/v (N, L, C) fp32 -> softmax(q k^T / sqrt(C)) v (the ldm mid-block attention core)."""
    for t_ in (q, k, v):
        _cuda(t_, "qkv", torch.float32)
        _req(t_.is_contiguous() and t_.shape == q.shape, "q/k/v must be contiguous and equal-shaped")
    N = q.shape[0]
    Cc = q.shape[-1]
    L = q.numel() // (N * Cc)
    out = torch.empty_like(q)
    _lib.check(_lib.lib().ln3_attn_single_head(_lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(out), N, L, Cc,
                                               _lib.current_stream()), "ln3_attn_single_head")
    return out


def patch_embed_triplane(latent: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None,
                         in_mul: float = 1.0, want_silu_bf16: bool = True):
    """latent fp32 (B, 3*Cz, S, S) -> tokens fp32 (B, 3*(S/2)^2, E) [+ bf16 SiLU(tokens)]."""
    _cuda(latent, "latent", torch.float32)
    _cuda(weight, "weight", torch.float32)
    _req(latent.is_contiguous() and weight.is_contiguous(), "latent/weight must be contiguous")
    B, C3, S, _ = latent.shape
    E3, Cz = weight.shape[0], weight.shape[1]
    _req(C3 == 3 * Cz and E3 % 3 == 0 and weight.shape[2:] == (2, 2), "PatchEmbedTriplane shapes")
    E = E3 // 3
    T = 3 * (S // 2) ** 2
    tok = torch.empty((B, T, E), device=latent.device, dtype=torch.float32)
    sb = torch.empty((B, T, E), device=latent.device, dtype=torch.bfloat16) if want_silu_bf16 else None
    _lib.check(_lib.lib().ln3_patch_embed_triplane(_lib.ptr(latent), _lib.ptr(weight), _lib.ptr(bias), B, Cz, S, E,
                                                   C.c_float(in_mul), _lib.ptr(tok), _lib.ptr(sb),
                                                   _lib.current_stream()), "ln3_patch_embed_triplane")
    return tok, sb


def marching_cubes(volume: torch.Tensor, isovalue: float, *, scale=(1.0, 1.0, 1.0), offset=(0.0, 0.0, 0.0)):
    """Device marching cubes (`mcubes.marching_cubes(volume, isovalue)`, nsr/train_util_diffusion.py:221-223).
    volume (nx, ny, nz) fp32 CUDA, z fastest.  Returns (vertices fp32 (V, 3), faces int32 (F, 3)) on the device;
    vertices are index coordinates times `scale` plus `offset` per axis.  One host sync (the mesh size is data
    dependent: the counts are read back between the count and the emit pass)."""
    _cuda(volume, "volume", torch.float32)
    _req(volume.dim() == 3 and volume.is_contiguous(), "volume must be contiguous (nx, ny, nz)")
    nx, ny, nz = (int(v) for v in volume.shape)
    _req(min(nx, ny, nz) >= 2, "every volume dimension must be >= 2")
    dev = volume.device
    wbytes = int(_lib.lib().ln3_marching_cubes_workspace_bytes(nx, ny, nz))
    ws = torch.empty(wbytes, dtype=torch.uint8, device=dev)
    totals = torch.zeros(2, dtype=torch.int32, device=dev)
    a = _lib.MarchingCubesArgs()
    a.grid, a.workspace, a.workspace_bytes, a.totals = volume.data_ptr(), ws.data_ptr(), wbytes, totals.data_ptr()
    a.nx, a.ny, a.nz, a.iso = nx, ny, nz, float(isovalue)
    for q in range(3):
        a.scale[q], a.offset[q] = float(scale[q]), float(offset[q])
    _lib.check(_lib.lib().ln3_marching_cubes_count(C.byref(a), _lib.current_stream()), "ln3_marching_cubes_count")
    nv, nf = (int(v) for v in totals.tolist())
    vertices = torch.empty((nv, 3), dtype=torch.float32, device=dev)
    faces = torch.empty((nf, 3), dtype=torch.int32, device=dev)
    if nv == 0 and nf == 0:
        return vertices, faces
    # ctypes rejects NULL-size tensors' data_ptr() == 0 only when both are empty (handled above)
    a.vertices = vertices.data_ptr() if nv else ws.data_ptr()
    a.faces = faces.data_ptr() if nf else ws.data_ptr()
    a.max_vertices, a.max_faces = nv, nf
    _lib.check(_lib.lib().ln3_marching_cubes_emit(C.byref(a), _lib.current_stream()), "ln3_marching_cubes_emit")
    return vertices, faces
