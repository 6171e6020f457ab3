"""TEST INFRASTRUCTURE ONLY -- the float64 references and error bounds of the CUDA kernels, shared by the per-kernel
tests (test_gpu_gemm_kernel.py, test_gpu_fmha_kernel.py, test_gpu_glue_kernels.py, test_gpu_gemm_fp8.py,
test_gpu_norm_modulate_fp8.py, test_gpu_decoder_conv_conformance.py, test_gpu_vae_encoder.py, test_gpu_vae_xl.py)
and the launch audits of the DiT denoisers and the VAE (test_gpu_denoiser_launches.py, test_gpu_vae_launches.py).  Each
bound is derived from its kernel's arithmetic in the docstring or comment beside it; the product package never
imports this module."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import dit as odit

U32 = 2.0 ** -24      # unit roundoff of fp32
SLOPE = 1.13          # max |f'| of every activation (GELU 1.129, SiLU / QuickGELU 1.0998 in their scaled argument)
FP8 = torch.float8_e4m3fn


# ------------------------------------------------------------------ rounding grids
def ulp(v: torch.Tensor, mant_bits: int) -> torch.Tensor:
    """Spacing of the floating-point grid with `mant_bits` stored mantissa bits at |v| (0 at v == 0)."""
    m, e = torch.frexp(v.abs().to(torch.float64))
    return torch.where(v == 0, torch.zeros_like(v, dtype=torch.float64),
                       torch.ldexp(torch.ones_like(m), (e - 1 - mant_bits).to(torch.int32)))


def ulp_f32(v):
    return ulp(v, 23)


def ulp_bf16(v):
    return ulp(v, 7)


def f32(t: torch.Tensor) -> torch.Tensor:
    """Round a float64 tensor to fp32 (one IEEE round-to-nearest) and keep it in float64."""
    return t.to(torch.float32).to(torch.float64)


def bf16_bound(y, tau):
    """bf16 output = the fp32 value rounded once: half a bf16 ulp of the exact value plus the fp32 error tau."""
    return ulp_bf16(y) / 2 + tau


def assert_sensitive(what: str, ref: torch.Tensor, wrong: torch.Tensor, tol: torch.Tensor,
                     affected: torch.Tensor | None = None, factor: float = 100.0) -> float:
    """The reference with one index mapping wrong must differ from the true one by >= `factor` (100) x the tolerance
    on the affected elements (median, so that elements whose operands happen to coincide do not decide it).  Returns
    the median ratio."""
    tol = tol.to(torch.float64).expand_as(ref)
    ratio = (wrong - ref).abs() / tol.clamp_min(1e-300)
    if affected is not None:
        ratio = ratio[affected.to(ratio.device).expand_as(ref)]
    assert ratio.numel() > 0, f"{what}: the slip affects no element"
    med = float(ratio.median())
    assert med >= factor, f"{what}: a slip moves the affected elements by only {med:.1f}x the tolerance (median)"
    return med


# ------------------------------------------------------------------ wgmma GEMM (gemm_wgmma.cu)
def act_ref(act, x):
    """(f(x) in float64, the bound on the kernel's own fp32 evaluation error at x)."""
    from ln3diff_b200 import ops
    u = 2.0 ** -24
    ax = x.abs()
    if act == ops.ACT_NONE:
        return x, torch.zeros_like(x)
    if act == ops.ACT_GELU_ERF:
        # the default packed polynomial: |abs error| <= 1.1e-5 for |x| < 4 (fp32 evaluation included); beyond,
        # Phi saturates where the true Phi(4) = 1 - 3.2e-5, so the error is <= 3.2e-5 |x| (and the flushed
        # negative tail is smaller than |x| Phi(-4) <= 3.2e-5 |x|)
        return 0.5 * x * (1 + torch.special.erf(x / math.sqrt(2))), 1.1e-5 + 3.2e-5 * ax
    if act == ops.ACT_GELU_TANH:
        # 0.5 x (1 + tanhf(arg)): tanhf 2 ulp of |t| <= 1 (2^-22); ~5 roundings in arg move t by
        # <= 5 u |arg| sech^2(arg) <= 5 u 0.45; the last two products round once each: <= 0.5|x| 2^-21 + 2u|x|
        k0, k1 = math.sqrt(2 / math.pi), 0.044715
        return 0.5 * x * (1 + torch.tanh(k0 * (x + k1 * x ** 3))), ax * 2.0 ** -20
    # x / (1 + __expf(-k x)): __expf is within (2 + 1.173 k|x|) ulp, the rounded argument adds k|x| u relative;
    # x e / (1 + e)^2 <= |x| / 4 turns e's relative error into the result's; the add and IEEE divide: 2u |x|
    k = 1.0 if act == ops.ACT_SILU else 1.702
    rel_e = 2 * u * (2 + 1.173 * k * ax) + k * ax * u
    return x * torch.sigmoid(k * x), 0.25 * ax * rel_e + 2 * u * ax


def gemm_tau(a64: torch.Tensor, w64: torch.Tensor, b64: torch.Tensor | None) -> torch.Tensor:
    """fp32 accumulation of K exact bf16 products, then the bias add: (K + 1) 2^-23 (sum|a w| + |b|) -- one fp32
    ulp per add (it allows for a tensor core that truncates instead of rounding) over K + 1 adds."""
    tau = a64.abs() @ w64.abs().T
    if b64 is not None:
        tau = tau + b64.abs()
    return (a64.shape[1] + 1) * 2.0 ** -23 * tau


def head_rmsnorm_ref(y: torch.Tensor, tau: torch.Tensor, hw: torch.Tensor, sec_cols: int, eps: float):
    """The GEMM epilogue's per-head RMSNorm in float64: the 64-column heads of section s (columns
    [s sec_cols, (s + 1) sec_cols)) scaled by hw[s], for s < nsec = hw.shape[0]; columns past the last section keep
    the plain output.  Returns (ref, tol) before the bf16 rounding.
    y_n = y rstd w: rstd from the fp32 sum of 64 squares (2 tau / |y| relative per term, 64 u for the sum),
    rsqrtf 2 ulp, then two rounded products per element."""
    M, N = y.shape
    ref, tol = y.clone(), tau.clone()
    hw64 = hw.to(torch.float64)
    for s in range(hw.shape[0]):
        c0, c1 = s * sec_cols, min((s + 1) * sec_cols, N)
        if c0 >= N:
            break
        yh = y[:, c0:c1].reshape(M, -1, 64)
        th = tau[:, c0:c1].reshape(M, -1, 64)
        ms = (yh * yh).mean(-1, keepdim=True)
        r = torch.rsqrt(ms + eps)
        rel_r = 0.5 * ((2 * yh.abs() * th + th * th).sum(-1, keepdim=True) / (64 * ms + 64 * eps) + 66 * 2.0 ** -24) \
            + 2.0 ** -22
        w = hw64[s].view(1, 1, 64)
        rh = yh * r * w
        ref[:, c0:c1] = rh.reshape(M, -1)
        tol[:, c0:c1] = ((th * r + yh.abs() * r * rel_r) * w.abs() + 4 * 2.0 ** -24 * rh.abs()).reshape(M, -1)
    return ref, tol


def gemm_bf16_bound(ref: torch.Tensor, tol: torch.Tensor) -> torch.Tensor:
    """bf16 output: the fp32 value rounded once: half a bf16 ulp at |y| + tol, plus tol."""
    return ulp(ref.abs() + tol, 7) / 2 + tol


# ------------------------------------------------------------------ flash attention (attention_wgmma.cu)
KT = 128             # keys per block of the kernel (for the count of rescales)
LOG2E = 1.4426950408889634


def heads(t: torch.Tensor, H: int) -> torch.Tensor:
    """(B, L, H 64) -> (B, H, L, 64) float64."""
    return t.to(torch.float64).unflatten(2, (H, 64)).transpose(1, 2)


def fmha_reference(q, k, v, H, scale, causal):
    """(y, tol) in float64, both (B, Lq, H 64); k / v already hold both K/V sources.  Per output element
    y = sum_j p_j v_j / sum_j p_j with p_j = 2^(s_j c - m) (c = scale log2 e):
      e_j   relative error of the kernel's unrounded p_j: an absolute error d_j of the exponent gives ln2 d_j, where
            d_j = c 64 2^-23 sum_d |q_d k_jd| (fp32 accumulation of the 64 exact bf16 products of S)
                + 2^-22 (|s_j c| + |m|)    (the fp32 constant c, the rounded product s c and the subtraction of m:
                                            2^-24 (3 |s_j c| + 2 |m|))
            plus the ex2.approx error, taken as 2^-21 relative.  The running-max rescale multiplies numerator and
            denominator by the same factor alpha, so alpha's own error cancels in the ratio.
      num   P is rounded to bf16 before P V while the row sum l adds the unrounded values.  bf16 keeps 8 significant
            bits, so round-to-nearest is off by up to 2^-8 relative (half an ulp just above a power of two):
            |d num| <= sum_j p_j |v_j| (e_j + 2^-8 (1 + e_j)) + n_acc 2^-23 sum_j p_j |v_j| (1 + e_j + 2^-8)
      den   |d l| <= sum_j p_j e_j + n_acc 2^-23 sum_j p_j (1 + e_j)
            n_acc = Lkv_total + 2 nblocks: one fp32 add per key (one ulp: allows a tensor core that truncates) and
            one rescale product per 128-key block in each of the accumulators.
      y     (|d num| + |y| |d l|) / (l - |d l|), plus two roundings (1/l and the product: 2^-23 |y|); the final bf16
            rounding is gemm_bf16_bound's: half a bf16 ulp at |y| + tol."""
    B, Lq, D = q.shape
    Lkv = k.shape[1]
    c = scale * LOG2E
    n_acc = Lkv + 2 * math.ceil(Lkv / KT)
    ys, tols = [], []
    step = max(1, (1 << 24) // (H * Lq * Lkv))
    for b0 in range(0, B, step):
        qh, kh, vh = (heads(t[b0:b0 + step], H) for t in (q, k, v))
        s = (qh @ kh.transpose(-1, -2)) * c                        # log2 units
        a = qh.abs() @ kh.abs().transpose(-1, -2)
        if causal:
            mask = torch.ones(Lq, Lkv, dtype=torch.bool, device=q.device).tril()
            s = s.masked_fill(~mask, -math.inf)
        m = s.amax(-1, keepdim=True)
        p = torch.exp2(s - m)                                     # 0 where masked
        d = c * 64 * 2.0 ** -23 * a + 2.0 ** -22 * (s.abs() + m.abs())
        e = math.log(2) * d + 2.0 ** -21
        e = torch.where(p > 0, e, torch.zeros_like(e))
        l = p.sum(-1, keepdim=True)
        y = (p @ vh) / l
        pv = p @ vh.abs()
        d_num = (p * (e + 2.0 ** -8 * (1 + e))) @ vh.abs() + n_acc * 2.0 ** -23 * (1 + 2.0 ** -7) * pv
        d_den = (p * e).sum(-1, keepdim=True) + n_acc * 2.0 ** -23 * (p * (1 + e)).sum(-1, keepdim=True)
        tol = (d_num + y.abs() * d_den) / (l - d_den) + 2.0 ** -23 * y.abs()
        ys.append(y.transpose(1, 2).flatten(2))
        tols.append(tol.transpose(1, 2).flatten(2))
    return torch.cat(ys), torch.cat(tols)


# ------------------------------------------------------------------ glue kernels (elementwise.cu)
def nm_tau(x: torch.Tensor, norm: int, nhat: torch.Tensor, w, one_p_s1, s0, y: torch.Tensor) -> torch.Tensor:
    """Error of the fp32 statistics and the modulation roundings of one norm_modulate / final_layer row, before
    the bf16 rounding.  A lane sums D/32 values, then 5 shuffle levels, then the division: every fp32 sum here has
    at most k = D/32 + 8 rounded additions, so its relative error is <= gamma = k * 2^-24 (Higham 3.1):
      LAYER  |mean error| <= gamma * mean|x|; rstd's relative error <= gamma/2 (variance) + 2^-22 (rsqrtf, 2 ulp)
             + 2^-24 (the eps add);
      RMS    no mean, the same rstd term;
      n^ = (x - mean) * rstd: two more roundings; * weight and the fma with (1 + scale): one each (2^-23 * |y|),
    so tau = |w (1 + s1)| * (rstd * |mean error| + |n^| * (gamma + 2^-21)) + 2^-23 * (|y| + |s0|)."""
    if norm == 0:
        return torch.zeros_like(y)
    D = x.shape[-1]
    gamma = (D / 32 + 8) * U32
    if norm == 1:
        mean_err = gamma * x.abs().mean(-1, keepdim=True)
        rstd = torch.rsqrt(((x - x.mean(-1, keepdim=True)) ** 2).mean(-1, keepdim=True) + 1e-6)
    else:
        mean_err = torch.zeros_like(x[..., :1])
        rstd = torch.rsqrt((x * x).mean(-1, keepdim=True) + 1e-6)
    amp = torch.ones_like(y)
    if w is not None:
        amp = amp * w.abs()
    if one_p_s1 is not None:
        amp = amp * one_p_s1.abs()
    t = amp * (rstd * mean_err + nhat.abs() * (gamma + 2.0 ** -21)) + 2.0 ** -23 * y.abs()
    if s0 is not None:
        t = t + 2.0 ** -23 * s0.abs()
    return t


ACT_REF = {  # act -> (float64 function, tau(x, y)): kernel error before the bf16 rounding
    # x / (1 + __expf(-x)): __expf is within (2 + 1.173|x|) ulp, the add and the IEEE divide round once each
    3: (lambda v: v * torch.sigmoid(v), lambda v, y: y.abs() * (3 + 1.2 * v.abs()) * 2.0 ** -23),
    # 0.5 x (1 + erff(x / sqrt2)): erff 2 ulp of |erf| <= 1, the scaled argument moves erf by <= 2^-24,
    # three more roundings on the product: 0.5 |x| * 2^-21 + 2^-22 |y|
    1: (lambda v: 0.5 * v * (1 + torch.erf(v / math.sqrt(2))), lambda v, y: 2.0 ** -22 * (v.abs() + y.abs())),
    # 0.5 x (1 + tanhf(k0 (x + k1 x^3))): the argument carries 5 roundings (relative 5 * 2^-24, tanh' <= 1),
    # tanhf 2 ulp; then 1 +, 0.5 x *: 0.5 |x| (5 * 2^-24 |arg| + 2^-22) + 2^-22 |y|
    2: (lambda v: 0.5 * v * (1 + torch.tanh(math.sqrt(2 / math.pi) * (v + 0.044715 * v ** 3))),
        lambda v, y: 0.5 * v.abs() * (5 * U32 * (0.8 * v.abs() + 0.036 * v.abs() ** 3) + 2.0 ** -22)
        + 2.0 ** -22 * y.abs()),
}


def nm_resid_ref(x, resid, gate, gate_idx, bcast=None, bcast_idx=None, inside=None, ogate=None, ogate_idx=None):
    """The kernel's residual update, one fp32 fmaf(g, r, x) per term: g * r (fp32 x bf16) is exact in float64, so
    rounding the float64 sum to fp32 matches fmaf except where a tie of the double rounding lands (<= 1 ulp).
    Outside rows with resid_out_gate add their own gated row first, then the ungated broadcast row."""
    if resid is None:
        return x.clone()
    rows = x.shape[0]
    g = gate[gate_idx] if gate is not None else torch.ones_like(x)
    if bcast is None:
        return f32(x + g * resid)
    out = torch.empty_like(x)
    ins = inside if inside is not None else torch.ones(rows, dtype=torch.bool, device=x.device)
    out[ins] = f32(x[ins] + g[ins] * resid[ins])
    o = ~ins
    if ogate is not None:
        t = f32(x[o] + ogate[ogate_idx[o]] * resid[o])
        out[o] = f32(t + bcast[bcast_idx[o]])
    else:
        out[o] = f32(x[o] + g[o] * bcast[bcast_idx[o]])
    return out


def nm_out_ref(xn, norm, eps, act, weight=None, shift=None, scale=None, mod_idx=None, shift_tab=None, scale_tab=None):
    """bf16 output before its rounding, from the (updated) fp32 row xn; returns (y, tau)."""
    if norm == 1:
        nhat = odit.layer_norm(xn, eps)
    elif norm == 2:
        nhat = odit.rms_norm(xn, None, eps)
    else:
        nhat = xn
    y = nhat * weight if weight is not None else nhat
    one_p, s0 = None, None
    if shift is not None:
        s1, s0 = scale[mod_idx], shift[mod_idx]
        if scale_tab is not None:
            s1, s0 = f32(s1 + scale_tab), f32(s0 + shift_tab)    # the kernel adds the tables in fp32
        one_p = f32(1 + s1)                                     # and rounds 1 + scale before the fma
        y = y * one_p + s0
    tau = nm_tau(xn, norm, nhat, weight, one_p, s0, y)
    if act:
        f, tau_act = ACT_REF[act]
        y, tau = f(xn), tau_act(xn, f(xn))                      # activations run with LN3_NORM_NONE only
    return y, tau


def final_layer_ref(x, shift, scale, W, bias, S, Cout, shift_tab=None, scale_tab=None, swap_pq=False):
    """(out, bound) in float64: LN (eps 1e-6) -> modulate with the kernel's fp32 roundings -> Linear -> unpatchify."""
    B = x.shape[0]
    s1, s0 = scale[:, None, :], shift[:, None, :]
    if scale_tab is not None:
        s1, s0 = f32(s1 + scale_tab), f32(s0 + shift_tab)
    one_p = f32(1 + s1)
    nhat = odit.layer_norm(x, 1e-6)
    y = nhat * one_p + s0
    tau = nm_tau(x, 1, nhat, None, one_p, s0, y)
    feat = y @ W.t() + (bias if bias is not None else 0)
    # fp32 dot product of D terms plus the bias: (n_terms + 4) * 2^-24 * sum|terms|, plus the LN error carried
    # through the weights, sum_d |W_od| * tau_d
    terms = y.abs() @ W.abs().t() + (bias.abs() if bias is not None else 0)
    fb = (x.shape[-1] + 1 + 4) * U32 * terms + tau @ W.abs().t()
    if swap_pq:      # feature index (p * 2 + q) * Cout + c read with p and q exchanged
        feat = feat.reshape(B, -1, 2, 2, Cout).transpose(2, 3).reshape(feat.shape)
    return odit.unpatchify_rollout(feat, Cout), odit.unpatchify_rollout(fb, Cout)


def patch_embed_ref(x, in_scale, W, bias, pos, roll_pos=False, roll_plane=False, roll_scale=False):
    """(tokens, bound) in float64.  The kernel scales x in fp32 (one rounding), then acc = bias, one fmaf per
    input, + pos_embed: (n_terms + 4) * 2^-24 * sum|terms| with n_terms = 4 Cin + 2."""
    B, C3, S, _ = x.shape
    if in_scale is not None:
        s = in_scale.roll(1, 0) if roll_scale else in_scale
        x = f32(s[:, None, None, None] * x)
    if roll_plane:   # the patch of the neighbouring plane n
        x = x.reshape(B, C3 // 3, 3, S, S).roll(1, 2).reshape(x.shape)
    tok = odit.patch_embed_rollout({"x_embedder.proj.weight": W, "x_embedder.proj.bias": bias}, x)
    terms = odit.patch_embed_rollout({"x_embedder.proj.weight": W.abs(),
                                      "x_embedder.proj.bias": bias.abs() if bias is not None else None}, x.abs())
    if pos is not None:
        p = pos.roll(1, 0) if roll_pos else pos
        tok, terms = tok + p, terms + pos.abs()
    return tok, (4 * C3 // 3 + 2 + 4) * U32 * terms


def timestep_embedding_ref(t: torch.Tensor):
    """([cos | sin] in float64, bound) for fp32 timesteps t: the oracle's fp32 frequencies (torch.exp of the fp32
    exponent), the argument t * f exactly.  The kernel's fp32 argument: expf vs torch.exp (1 ulp each way) and the
    rounded product t * f, both relative <= 2^-23 * t f <= 2^-23 |t| (f <= 1); cosf / sinf add 2 ulp of a value
    <= 1: tau = 2^-22 (|t| + 1), then the bf16 rounding."""
    freqs = torch.exp(-math.log(10000.0) * torch.arange(128, dtype=torch.float32) / 128).double().to(t.device)
    arg = t.double()[:, None] * freqs[None]
    ref = torch.cat([arg.cos(), arg.sin()], -1)
    tau = 2.0 ** -22 * (t.double().abs()[:, None] + 1)
    return ref, ulp_bf16(ref) / 2 + tau


# ------------------------------------------------------------------ fp8 (gemm_fp8_wgmma.cu, norm_modulate_fp8)
U_ACC = 2.0 ** -13    # assumed in-block fp8 accumulation of the tensor core: see test_gpu_gemm_fp8.py


def fp8_reference(a_q, a_s, w_q, w_s, b):
    """(y, T) in float64: y the exact scaled GEMM + bias, T the same GEMM on absolute values."""
    M, K = a_q.shape
    A = a_q.to(torch.float64).view(M, K // 128, 128) * a_s.to(torch.float64)[:, :, None]
    A = A.view(M, K)
    W = w_q.to(torch.float64)
    y = (A @ W.T) * w_s.to(torch.float64)
    T = (A.abs() @ W.abs().T) * w_s.to(torch.float64)
    if b is not None:
        y = y + b.to(torch.float64)
    return y, T


def fp8_acc_bound(T, K, b):
    """E = 128 U_ACC T + (K/128 + 2) 2^-23 (T + |bias|): the in-block accumulation, the promotion fmaf per k-block
    and the epilogue fmaf."""
    bb = b.to(torch.float64).abs() if b is not None else 0.0
    return 128 * U_ACC * T + (K // 128 + 2) * 2.0 ** -23 * (T + bb)


def gelu_ref(x):
    return 0.5 * x * (1 + torch.special.erf(x / math.sqrt(2))), 1.1e-5 + 3.2e-5 * x.abs()


def fp8_head_norm_ref(y, E, w, nsec, sec_cols, eps=1e-5):
    """Per-head RMSNorm of the first nsec sections in float64 and the propagated bound: a perturbation |d_i| <= E_i
    of the head moves rms by at most max E, so y_i r w_i moves by |w_i| r (E_i + |y_i| r max E) (first order, with
    a 1 % margin), plus the kernel's own fp32 evaluation (64 products summed, rsqrt, two products: 80 u |out|)."""
    out, bound = y.clone(), E.clone()
    M, N = y.shape
    w = w.to(torch.float64)
    for sec in range(nsec):
        for h0 in range(sec * sec_cols, (sec + 1) * sec_cols, 64):
            if h0 >= N:
                break
            yh, Eh = y[:, h0:h0 + 64], E[:, h0:h0 + 64]
            r = torch.rsqrt((yh * yh).mean(dim=1, keepdim=True) + eps)
            wh = w[sec][None, :]
            out[:, h0:h0 + 64] = yh * r * wh
            bound[:, h0:h0 + 64] = (1.01 * wh.abs() * r * (Eh + yh.abs() * r * Eh.amax(dim=1, keepdim=True))
                                    + 80 * 2.0 ** -24 * (yh * r * wh).abs())
    return out, bound


def fp8_bf16_bound(ref, E):
    """bf16 output of the fp8 GEMM: E plus half a bf16 ulp at |y| + E."""
    return E + 0.5 * ulp(ref.abs() + E, 7)


def fp8_out_check(q, s, v, d):
    """q / s the kernel's codes and block scales, v the fp64 epilogue value, d its error bound: the block scale within
    d + 2^-22 amax of amax / 448, and every code between the roundings of (v - d) / s and (v + d) / s.  Returns
    (scale error / bound, fraction of codes equal to the fp64 quantisation, ok mask of the codes, scale ok mask)."""
    M, N = v.shape
    vb = v.view(M, N // 128, 128)
    db = d.view(M, N // 128, 128)
    amax = vb.abs().amax(dim=2)
    dmax = db.amax(dim=2)
    s64 = s.to(torch.float64)
    serr = (s64 * 448 - amax).abs()
    sbound = dmax + 2.0 ** -22 * amax
    sk = s64[:, :, None]
    safe = torch.where(sk > 0, sk, torch.ones_like(sk))
    t = vb / safe
    dt = db / safe + 2.0 ** -22 * t.abs()
    rnd = lambda z: z.clamp(-448, 448).to(torch.float32).to(FP8).to(torch.float64)
    lo, hi = rnd(t - dt), rnd(t + dt)
    got = q.reshape(M, N // 128, 128).to(torch.float64)
    zero_blocks = (sk == 0).expand_as(got)
    ok = torch.where(zero_blocks, got == 0, (got >= lo) & (got <= hi))
    exact = float((got == rnd(t)).to(torch.float64).mean())
    return float((serr / sbound.clamp_min(1e-300)).max()), exact, ok.view(M, N), serr <= sbound


def restated_fp8(y32: torch.Tensor):
    """The activation block format evaluated by torch on fp32 values: (codes, scales)."""
    rows, D = y32.shape
    b = y32.view(rows, D // 128, 128)
    amax = b.abs().amax(dim=2)
    s = amax / torch.full_like(amax, 448.0)         # a true division: torch turns `/ 448.0` into `* (1/448)`
    safe = torch.where(s > 0, s, torch.ones_like(s))
    t = torch.where(s[:, :, None] > 0, b / safe[:, :, None], torch.zeros_like(b))
    return t.clamp(-448, 448).to(FP8).view(rows, D), s


def restated_weight_fp8(w: torch.Tensor):
    """ops.quantize_weight_fp8's documented rule on an nn.Linear weight (N, K): w_scale = fp32(absmax of the row /
    448), codes = the float8_e4m3fn cast of fp32(w / w_scale); a zero row has scale 0 and zero codes."""
    w = w.detach().float()
    amax = w.abs().amax(dim=1)
    s = amax / torch.full_like(amax, 448.0)
    safe = torch.where(s > 0, s, torch.ones_like(s))
    q = torch.where(s[:, None] > 0, w / safe[:, None], torch.zeros_like(w))
    return q.clamp(-448, 448).to(FP8), s


def half_ulp_e4m3(t: torch.Tensor) -> torch.Tensor:
    """Half the e4m3 spacing at |t| (subnormal spacing 2^-9 below 2^-6)."""
    _, e = torch.frexp(t.abs().to(torch.float64).clamp_min(2.0 ** -6))
    return torch.ldexp(torch.full_like(t, 0.5, dtype=torch.float64), (e - 1 - 3).to(torch.int32))


def nm_fp8_error(q, s, y, e):
    """(|dequantised - y|, bound) of norm_modulate_fp8: the dequantised code * s within half an e4m3 ulp of y / s
    (times s) of the float64 value y, plus the fp32 normalisation error e = 64 u (|n| (1 + |scale|) + |shift|)
    (n the normalised value, u = 2^-24: a <= 40-deep summation and rsqrt moving n by far less than 64 u relative)."""
    s64 = s.double().repeat_interleave(128, dim=1)
    deq = q.double() * s64
    safe = torch.where(s64 > 0, s64, torch.ones_like(s64))
    bound = half_ulp_e4m3((y.abs() + e) / safe) * s64 + e + 2.0 ** -22 * y.abs()
    return (deq - y).abs(), bound


# ------------------------------------------------------------------ NHWC conv / GroupNorm / single-head attention /
# tri-plane patch embed (decoder_conv.cu)
SWISH_SLOPE = 1.1         # max |d/dz z sigmoid(z)| = 1.0998
KB = 32                   # keys per block of ln3_attn_single_head


def _expf_rel(z):
    """__expf(x) error relative to exp(x): at most 2 + floor(|1.173 x|) ulp (CUDA programming guide), an ulp <= 2u."""
    return (2 + torch.floor(1.173 * z.abs())) * 2 * U32


def _swish_tol(z, dz):
    """Error of the kernel's v / (1 + __expf(-v)) with v = z + dz (|dz| the error of the fp32 pre-activation):
    the input error passes with slope <= 1.1; __expf(-v) is off by _expf_rel relative, which moves 1 + e and so the
    quotient by at most that much relative; the add and the division round once each (2u).  Below z = -88.7
    __expf(-v) overflows to inf and the kernel returns -0: the whole value |s| is lost there (and is < 3e-37), and the
    2^-126 floor covers quotients that fall into the subnormal range."""
    s = z * torch.sigmoid(z)
    rel = torch.where(z < -80, torch.ones_like(z), _expf_rel(z) + 3 * U32)
    return s, SWISH_SLOPE * dz + s.abs() * rel + 2.0 ** -126


def conv_reference(x, w, b, *, ksize, up, sc=None, sh=None, swish=False, res=None, tf32=False, dz=None):
    """(ref, tol) in float64, NCHW.  x fp32 NHWC (N, Hin, Win, Cin) on the device; sc, sh fp32 (N, Cin) are the very
    values the kernel gets, so the reference input is x_hat = swish(x sc + sh) evaluated in float64 and this isolates
    the conv.  Per output element, with T = conv(|x_hat|, |w|) + |b| and K = ksize^2 Cin:
      fp32: a chain of K fmaf plus the bias add: (K + 4) u T;
      TF32: both operands rounded to nearest 10-bit mantissas (2^-11 relative each) before the fp32-accumulated
            mma: 2^-10 T more;
      input: the kernel's x_hat is off by d = u |z| (the fmaf z = x sc + sh rounds once), passed through swish by
            _swish_tol, and the conv carries d through |w|: conv(d, |w|) (times 1 + 2^-9 for the TF32 rounding of
            the perturbed value);
      residual: the final add rounds once more, u |out|.
    dz (N, Hin, Win, Cin) adds an upstream error of z (the composed GroupNorm test)."""
    x64 = x.double()
    d = torch.zeros_like(x64)
    if sc is not None:
        z = x64 * sc.double()[:, None, None, :] + sh.double()[:, None, None, :]
        d = U32 * z.abs() + (dz if dz is not None else 0.0)
        if swish:
            xh, d = _swish_tol(z, d)
        else:
            xh = z
    else:
        xh = x64
    xh, d = xh.permute(0, 3, 1, 2), d.permute(0, 3, 1, 2)
    if up:
        xh, d = F.interpolate(xh, scale_factor=2.0, mode="nearest"), F.interpolate(d, scale_factor=2.0, mode="nearest")
    w64 = w.double()
    pad = ksize // 2
    ref = F.conv2d(xh, w64, None if b is None else b.double(), padding=pad)
    T = F.conv2d(xh.abs(), w64.abs(), None if b is None else b.double().abs(), padding=pad)
    K = ksize * ksize * x.shape[3]
    tol = ((2.0 ** -10 if tf32 else 0.0) + (K + 4) * U32) * T + (1 + 2.0 ** -9) * F.conv2d(d, w64.abs(), padding=pad)
    if res is not None:
        ref = ref + res.double().permute(0, 3, 1, 2)
        tol = tol + U32 * ref.abs()
    return ref, tol


def gn_reference(x, gamma, beta, G, eps=1e-6):
    """(sc, sh, tol_sc, tol_sh, e_mu, mu) in float64, each (N, C).  The kernel, per (image, group) of cnt = HW C/G
    elements: each of 256 threads adds m = ceil(cnt / 256) terms in sequence, then a 5-level shuffle tree in each warp
    and a 5-level tree over the 8 warp sums, so every term meets at most m + 10 roundings; the mean divides once more:
      e_mu  <= (m + 11) u A,   A = sum |x| / cnt.
    The second pass adds fmaf(d, d, q) of d = fl(x - mu_hat) (2u relative on d^2) over the same m + 10 levels, and
    sum (x - mu_hat)^2 = sum (x - mu)^2 + cnt e_mu^2, so with var = biased variance
      |var_hat - var| <= (m + 13) u var + e_mu^2        (the division by cnt included).
    var + eps rounds (u) and rsqrtf is within 2 ulp (4u), so rstd is off by rel_r = 1/2 rel(var + eps) + 4u; then
      sc = fl(gamma rstd):               |d sc| <= |sc| (rel_r + u)
      sh = fl(beta - fl(mu_hat sc_hat)): |d sh| <= |sc| e_mu + |mu| |d sc| + u |mu sc| + u |sh|
    every term taken 1 % larger for the second-order products."""
    N, H, W, Cc = x.shape
    cpg, cnt = Cc // G, H * W * Cc // G
    m = -(-cnt // 256)
    xg = x.double().reshape(N, H * W, G, cpg)
    mu = xg.mean(dim=(1, 3))                                             # (N, G)
    var = ((xg - mu[:, None, :, None]) ** 2).mean(dim=(1, 3))
    A = xg.abs().mean(dim=(1, 3))
    e_mu = 1.01 * (m + 11) * U32 * A
    e_var = 1.01 * ((m + 13) * U32 * var + e_mu ** 2)
    rstd = 1 / torch.sqrt(var + eps)
    rel_r = 1.01 * (0.5 * (e_var / (var + eps) + U32) + 4 * U32)
    rep = lambda t: t.repeat_interleave(cpg, dim=1)                      # (N, G) -> (N, C)
    g64, b64 = gamma.double()[None], beta.double()[None]
    sc = g64 * rep(rstd)
    sh = b64 - rep(mu) * sc
    tol_sc = 1.01 * sc.abs() * (rep(rel_r) + U32)
    tol_sh = 1.01 * (sc.abs() * rep(e_mu) + rep(mu).abs() * tol_sc + U32 * (rep(mu) * sc).abs() + U32 * sh.abs())
    return sc, sh, tol_sc, tol_sh, rep(e_mu), rep(mu)


def attn_reference(q, k, v):
    """(y, tol) in float64, (N, L, C).  The kernel pre-multiplies q by scale = fl(1 / sqrtf(C)) (scale 2u off the exact
    C^-1/2, the product one more rounding), scores s_j with a C-term fmaf chain, so with a_j = C^-1/2 sum |q k_j|
      |d s_j| <= (C + 4) u a_j;
    p_j = __expf(fl(s_j - m)) with m the running max of the scores: the subtraction rounds (u |s_j - m|) and __expf adds
    _expf_rel(s_j - m).  Shifting every score by the same m does not change the ratio, so m's own error drops out, and
    |s_j - m| is largest with the final m, which the reference uses.  When a block raises the running max from m_old to
    m_new, the kernel multiplies the numerator and the denominator accumulated so far by alpha = __expf(fl(m_old - m_new)).
    That scales the keys already seen against the later ones, so alpha's own error is charged to each earlier key: key j
    sees at most nb - 1 such rescales (nb = ceil(L / 32)), each with |m_old - m_new| <= m - s_j + 2 d_max (m_old >= s_j
    since key j is already in, m_new <= m; d_max = the largest |d s|), so each is off by at most
      eps_j = expm1(u r_j) + _expf_rel(r_j),  r_j = |s_j - m| + 2 d_max.
    P stays fp32, so the relative error of the kernel's weight of key j is
      e_j   = (1 + expm1((C + 4) u a_j + u |s_j - m|) + _expf_rel(s_j - m)) (1 + eps_j)^(nb - 1) - 1
            (1 below -80, where ex2.approx flushes to 0)
      num   |d num| <= sum_j p_j |v_j| e_j + n_acc 2u sum_j p_j |v_j| (1 + e_j)
      den   |d l|   <= sum_j p_j e_j + n_acc 2u sum_j p_j (1 + e_j)
      n_acc = L + 2 ceil(L / 32): one add per key (the 5-level block sum adds only the block's keys), one rescale
              product per 32-key block in each accumulator
      y     (|d num| + |y| |d l|) / (l - |d l|) + 2u |y| (1 / l and the product)."""
    N, L, Cc = q.shape
    q64, k64, v64 = q.double(), k.double(), v.double()
    sc = Cc ** -0.5
    s = (q64 @ k64.transpose(1, 2)) * sc
    a = (q64.abs() @ k64.abs().transpose(1, 2)) * sc
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    arg = (s - m).abs()
    nb = math.ceil(L / KB)
    r = arg + 2 * (Cc + 4) * U32 * a.amax(-1, keepdim=True)
    eps = torch.expm1(U32 * r) + _expf_rel(r)
    e = (1 + torch.expm1((Cc + 4) * U32 * a + U32 * arg) + _expf_rel(arg)) * (1 + eps) ** (nb - 1) - 1
    e = torch.where(arg > 80, torch.ones_like(e), e)
    n_acc = L + 2 * nb
    l = p.sum(-1, keepdim=True)
    y = (p @ v64) / l
    d_num = (p * e) @ v64.abs() + n_acc * 2 * U32 * ((p * (1 + e)) @ v64.abs())
    d_den = (p * e).sum(-1, keepdim=True) + n_acc * 2 * U32 * (p * (1 + e)).sum(-1, keepdim=True)
    tol = (d_num + y.abs() * d_den) / (l - d_den) + 2 * U32 * y.abs()
    return y, tol


def pet_reference(lat, w, b, in_mul):
    """(tokens, tol_tok, silu, tol_silu) in float64.  The kernel input is fl(lat in_mul), the same rounding torch does
    for `lat * in_mul`, so the reference starts from that fp32 product.  Each token is a chain of K = 4 Cz fmaf
    started from the bias: |d tok| <= (4 Cz + 2) u T, T = sum |w x| + |b|.  The bf16 copy is
    fl_bf16(silu_k(tok_hat)): swish of a value off by d tok (_swish_tol), then round to nearest bf16: half an ulp of
    8 significant bits, up to 2^-8 |silu| just above a power of two (+ 2^-8 of its error, and half the 2^-133 spacing
    below bf16's normal range)."""
    B, C3, S, _ = lat.shape
    Cz, E = C3 // 3, w.shape[0] // 3
    x = (lat * in_mul).double()                                       # fp32 product, as torch rounds it
    w64 = w.double()
    y = F.conv2d(x, w64, None if b is None else b.double(), stride=2, groups=3)
    T = F.conv2d(x.abs(), w64.abs(), None if b is None else b.double().abs(), stride=2, groups=3)
    tok = lambda t: t.reshape(B, E, 3, S // 2, S // 2).flatten(2).transpose(1, 2)     # B (3 h w) E
    y, T = tok(y), tok(T)
    tol = (4 * Cz + 2) * U32 * T
    silu, tol_s = _swish_tol(y, tol)
    tol_s = tol_s * (1 + 2.0 ** -8) + 2.0 ** -8 * silu.abs() + 2.0 ** -134
    return y, tol, silu, tol_s


# ------------------------------------------------------------------ encoder Downsample, VAE posterior, view mean
def downsample_reference(x, w, b, tf32):
    """(ref, tol) in float64, NCHW, of F.conv2d(F.pad(x, (0,1,0,1)), w, b, stride=2); x NHWC fp32, w (Cout, Cin, 3, 3).
    Per element, with T = sum |w x| + |b| over the K = 9 Cin terms:
      fp32: a chain of K fused multiply-adds plus the bias add, |err| <= (K + 4) 2^-24 T;
      TF32: both operands rounded to 10-bit mantissas (relative 2^-11 each, so 2^-10 per product) on top of the
            fp32 accumulation: |err| <= (2^-10 + (K + 4) 2^-24) T."""
    xc = x.double().permute(0, 3, 1, 2)
    w64, b64 = w.double(), b.double()
    ref = F.conv2d(F.pad(xc, (0, 1, 0, 1)), w64, b64, stride=2)
    T = F.conv2d(F.pad(xc.abs(), (0, 1, 0, 1)), w64.abs(), stride=2) + b64.abs()[:, None, None]
    K = 9 * x.shape[3]
    return ref, ((2.0 ** -10 if tf32 else 0.0) + (K + 4) * U32) * T


def _posterior_tol(qw, qb, mom, mean, lv, z, noise):
    """Float64 vs kernel (an ulp is at most 2^-23 = 2u of the value).  Moments: an 8-term fmaf chain plus the bias add,
    <= 9u T (T = sum |w h| + |b|, mom NCHW).  logvar: the input error passes tanh with slope <= 1; div (1/2 ulp), tanhf (2 ulp)
    and mul (1/2 ulp) add 3 ulp <= 6u |lv|, bounded by 8u.  std = exp(0.5 lv): 0.5 lv is exact, so a relative error of
    0.5 err(lv) + 2 ulp (expf) = 0.5 err(lv) + 4u; the product std * noise adds u, the final sum u |z| (bounded by 2u)."""
    T = F.conv2d(mom.abs(), qw.abs(), groups=3) + qb.abs()[None, :, None, None]
    tol_m = 9 * U32 * T[:, :12] + U32 * mean.abs()
    tol_lv = 9 * U32 * T[:, 12:] + 8 * U32 * lv.abs()
    std = torch.exp(0.5 * lv)
    tol_z = tol_m + std * noise.abs() * (0.5 * tol_lv + 6 * U32) + 2 * U32 * z.abs()
    return tol_m, tol_lv, tol_z


def view_mean_tol(xv):
    """ln3_view_mean_nhwc of xv (B, F, ...): an fp32 sum over the F views in order, then one division by F, within
    (F + 1) u sum|x| / F of the float64 mean."""
    F_ = xv.shape[1]
    return (F_ + 1) * U32 * xv.double().abs().sum(1) / F_


def _chunk_mean(h, num_frames):
    """torch.chunk(N // num_frames) + mean(dim=0) per chunk, as the reference pools, in the kernel's summation order.  The
    division is by a tensor: torch's CUDA division by a Python scalar multiplies by its reciprocal instead."""
    outs = []
    for f in h.chunk(h.shape[0] // num_frames):
        s = f[0].clone()
        for v in range(1, f.shape[0]):
            s = s + f[v]
        outs.append((s / torch.full_like(s, f.shape[0]))[None])
    return torch.cat(outs)
