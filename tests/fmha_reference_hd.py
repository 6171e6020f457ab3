"""TEST INFRASTRUCTURE ONLY -- the float64 flash-attention reference and bound of kernel_bounds.fmha_reference for any
head width: the fp32 accumulation of S carries hd exact bf16 products per entry (at head_dim 72 the kernel pads the
contraction to 80 with exact zeros, which add exactly 0).  See kernel_bounds.fmha_reference for the derivation."""
import math

import torch

from kernel_bounds import KT, LOG2E


def fmha_reference_hd(q, k, v, H, hd, scale, causal=False):
    """(y, tol) in float64, both (B, Lq, H hd); k / v (B, Lkv, H hd)."""
    B, Lq, _ = q.shape
    Lkv = k.shape[1]
    c = scale * LOG2E
    n_acc = Lkv + 2 * math.ceil(Lkv / KT)
    heads = lambda t: t.to(torch.float64).unflatten(2, (H, hd)).transpose(1, 2)
    ys, tols = [], []
    step = max(1, (1 << 24) // (H * Lq * Lkv))
    for b0 in range(0, B, step):
        qh, kh, vh = (heads(t[b0:b0 + step]) for t in (q, k, v))
        s = (qh @ kh.transpose(-1, -2)) * c
        a = qh.abs() @ kh.abs().transpose(-1, -2)
        if causal:
            mask = torch.ones(Lq, Lkv, dtype=torch.bool, device=q.device).tril()
            s = s.masked_fill(~mask, -math.inf)
        m = s.amax(-1, keepdim=True)
        p = torch.exp2(s - m)
        d = c * hd * 2.0 ** -23 * a + 2.0 ** -22 * (s.abs() + m.abs())
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
