"""Thin, checked Python entry points over the C ABI (one function per exported op).

Shape / dtype / contiguity violations raise here (mirroring the TORCH_CHECKs of the reference's
own native ops, utils/torch_utils/ops/bias_act.cpp:39-60); everything else is the C call.
"""
from __future__ import annotations

import os

import ctypes as C

import torch

from . import _lib
from ._lib import (ACT_GELU_ERF, ACT_GELU_TANH, ACT_NONE, ACT_QUICK_GELU, ACT_SILU, OUT_BF16, OUT_F32,
                   OUT_RESID_F32)

__all__ = ["gemm", "ACT_NONE", "ACT_GELU_ERF", "ACT_GELU_TANH", "ACT_SILU", "ACT_QUICK_GELU", "OUT_BF16", "OUT_F32",
           "OUT_RESID_F32"]


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
             "head_norm must be contiguous (nsec, 64)")
        args.head_norm_w, args.head_norm_nsec = head_norm.data_ptr(), head_norm.shape[0]
        args.head_norm_sec_cols, args.head_norm_eps = head_norm_sec_cols, head_norm_eps
    args.act, args.out_kind = act, out_kind
    _lib.check(_lib.lib().ln3_gemm_bf16(C.byref(args), _lib.current_stream()), "ln3_gemm_bf16")
    return out


def fmha(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, *,
         out: torch.Tensor | None = None, scale: float | None = None,
         k2: torch.Tensor | None = None, v2: torch.Tensor | None = None, causal: bool = False) -> torch.Tensor:
    """softmax(q k^T * scale) v per head.  q (B,Lq,H*64), k/v (B,Lkv,H*64) bf16 views with unit
    inner stride (slices of a packed qkv buffer are fine); returns (B,Lq,H*64) bf16.
    causal=True: key j is visible to query i only when j <= i (CLIP text tower)."""
    for name, t in (("q", q), ("k", k), ("v", v)):
        _cuda(t, name, torch.bfloat16)
        _req(t.dim() == 3 and t.stride(2) == 1, f"{name} must be (B,L,H*64) with unit inner stride")
    B, Lq, C_ = q.shape
    _req(C_ == heads * 64, "head_dim must be 64")
    _req(k.shape == v.shape and k.shape[0] == B and k.shape[2] == C_, "k/v shape mismatch")
    Lkv = k.shape[1]
    if out is None:
        out = torch.empty((B, Lq, C_), device=q.device, dtype=torch.bfloat16)
    _cuda(out, "out", torch.bfloat16)
    _req(out.shape == (B, Lq, C_) and out.stride(2) == 1, "out must be (B,Lq,H*64)")
    a = _lib.FmhaArgs()
    a.q, a.k, a.v, a.out = q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr()
    a.B, a.H, a.Lq, a.Lkv, a.head_dim = B, heads, Lq, Lkv, 64
    a.q_ld, a.q_bs = q.stride(1), q.stride(0)
    a.k_ld, a.k_bs = k.stride(1), k.stride(0)
    a.v_ld, a.v_bs = v.stride(1), v.stride(0)
    a.o_ld, a.o_bs = out.stride(1), out.stride(0)
    a.scale = float(scale if scale is not None else 64 ** -0.5)
    a.causal = 1 if causal else 0
    _req(not (causal and k2 is not None), "causal attention takes a single K/V source")
    if k2 is not None:
        for name, t in (("k2", k2), ("v2", v2)):
            _cuda(t, name, torch.bfloat16)
            _req(t.dim() == 3 and t.stride(2) == 1 and t.shape[0] == B and t.shape[2] == C_, f"{name} must be (B,L2,H*64)")
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
    _lib.check(_lib.lib().ln3_norm_modulate(C.byref(a), _lib.current_stream()), "ln3_norm_modulate")
    return out


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
                 image_width: int | None = None):
    """Fused ImportanceRenderer.forward for V views.  Returns dict(rgb (V,3,M), depth (V,1,M),
    weights (V,1,M)) (+ debug index tensors).  mlp_tf32: evaluate the OSG MLP on the tensor cores (TF32
    operands, fp32 accumulate; pixel error ~1e-4 rel-L2) instead of exact fp32."""
    for nm, t_ in (("planes_cl", planes_cl), ("ray_o", ray_o), ("ray_d", ray_d),
                   ("noise_coarse", noise_coarse), ("noise_fine", noise_fine)):
        _cuda(t_, nm, torch.float32)
        _req(t_.is_contiguous(), f"{nm} must be contiguous")
    _req(planes_cl.dim() == 5 and planes_cl.shape[1] == 3 and planes_cl.shape[4] == 32,
         "planes_cl must be (N,3,H,W,32)")
    V, M, _ = ray_o.shape
    _req(ray_d.shape == (V, M, 3), "ray_d shape")
    _req(noise_coarse.numel() == V * M * 64 and noise_fine.numel() == V * M * 64,
         "noise tensors must hold V*M*64 values")
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
        out["inbox"] = torch.empty((V * M, 128), device=dev, dtype=torch.uint8)
        out["inds"] = torch.empty((V * M, 64), device=dev, dtype=torch.int32)
        out["order"] = torch.empty((V * M, 128), device=dev, dtype=torch.int32)
        out["z_fine"] = torch.empty((V * M, 64), device=dev, dtype=torch.float32)
        a.dbg_inbox, a.dbg_inds = out["inbox"].data_ptr(), out["inds"].data_ptr()
        a.dbg_order, a.dbg_zfine = out["order"].data_ptr(), out["z_fine"].data_ptr()
    a.V, a.M, a.H, a.W, a.C = V, M, planes_cl.shape[2], planes_cl.shape[3], 32
    a.S, a.S_importance, a.hidden_dim, a.decoder_output_dim = 64, 64, 64, 3
    a.group_size, a.views_per_obj, a.white_back = group_size, views_per_obj, int(white_back)
    a.box_warp, a.bbox_min, a.bbox_max = box_warp, bbox_min, bbox_max
    a.mlp_precision = _lib.MLP_TF32 if mlp_tf32 else _lib.MLP_FP32
    # rays in RaySampler order (m = y*W + x): square views get the 4x4 pixel-tile schedule; image_width=0 forces
    # the plain ray order (rays that are not an image, e.g. PatchRaySampler training patches)
    if image_width is None:
        r = int(round(M ** 0.5))
        image_width = r if r * r == M else 0
    a.image_w = int(image_width) if os.environ.get("LN3_RENDER_TILES", "1") != "0" else 0
    _lib.check(_lib.lib().ln3_render_views(C.byref(a), _lib.current_stream()), "ln3_render_views")
    return out


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
