"""Mirror of reference dit/dit_models_xformers.py (hot-path classes only).

The classes below are *parameter containers with the reference's names and state_dict keys*
(`blocks.{i}.attn.qkv.weight`, `blocks.{i}.mlp.mlp.0.weight`, `blocks.{i}.cross_attn.to_q.weight`,
`final_layer.adaLN_modulation.1.weight`, ... -- SURVEY.md appendix B) so checkpoints of the
reference load unchanged.  Their arithmetic runs in `ln3diff_b200.dit._denoiser` on hand-written
sm_90a kernels; there is no PyTorch-eager fallback.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn


def modulate(x, shift, scale):
    """reference dit_models_xformers.py:47-48 (kept for API parity; the fused kernel is
    ln3_norm_modulate)."""
    return x * (1 + scale.unsqueeze(1)) + shift.unsqueeze(1)


def t2i_modulate(x, shift, scale):
    return x * (1 + scale) + shift


def approx_gelu():
    return nn.GELU(approximate="tanh")


class TimestepEmbedder(nn.Module):
    """reference dit_models_xformers.py:87-127: sinusoid(256) -> Linear -> SiLU -> Linear."""

    def __init__(self, hidden_size, frequency_embedding_size=256):
        super().__init__()
        self.mlp = nn.Sequential(
            nn.Linear(frequency_embedding_size, hidden_size, bias=True),
            nn.SiLU(),
            nn.Linear(hidden_size, hidden_size, bias=True),
        )
        self.frequency_embedding_size = frequency_embedding_size

    @staticmethod
    def timestep_embedding(t, dim, max_period=10000):
        half = dim // 2
        freqs = torch.exp(-math.log(max_period) * torch.arange(0, half, dtype=torch.float32) / half
                          ).to(device=t.device)
        args = t[:, None].float() * freqs[None]
        return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


class _Mlp(nn.Module):
    """timm.models.vision_transformer.Mlp parameter layout (fc1 / fc2)."""

    def __init__(self, in_features, hidden_features, out_features):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden_features)
        self.fc2 = nn.Linear(hidden_features, out_features)


class CaptionEmbedder(nn.Module):
    """reference dit_models_xformers.py:183-223: y_proj = Mlp(in -> hidden -> hidden, tanh-GELU)."""

    def __init__(self, in_channels, hidden_size, act_layer=None, token_num=120):
        super().__init__()
        self.y_proj = _Mlp(in_channels, hidden_size, hidden_size)


class _BiasOnly(nn.Module):
    def __init__(self, n):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(n))


class _FusedMLP(nn.Module):
    """xformers FusedMLP parameter layout: mlp.0.weight, mlp.1.bias, mlp.2.weight, mlp.3.bias."""

    def __init__(self, dim_model, hidden_layer_multiplier=4):
        super().__init__()
        hid = hidden_layer_multiplier * dim_model
        self.mlp = nn.Sequential(nn.Linear(dim_model, hid, bias=False), _BiasOnly(hid),
                                 nn.Linear(hid, dim_model, bias=False), _BiasOnly(dim_model))


class _RMSNormParam(nn.Module):
    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(dim))


class Attention(nn.Module):
    """vit/vision_transformer.py:60-87 MemEffAttention parameters (qkv, proj, optional q/k norm)."""

    def __init__(self, dim, num_heads=8, qkv_bias=False, qk_norm=False, **_):
        super().__init__()
        self.num_heads = num_heads
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)
        self.qk_norm = qk_norm
        if qk_norm:
            self.q_norm = _RMSNormParam(dim // num_heads)
            self.k_norm = _RMSNormParam(dim // num_heads)


class MemoryEfficientCrossAttention(nn.Module):
    """ldm/modules/attention.py:245-277 parameters (to_q/to_k/to_v without bias, to_out.0)."""

    def __init__(self, query_dim, context_dim=None, heads=8, dim_head=64, dropout=0.0,
                 enable_rmsnorm=False, qk_norm=False):
        super().__init__()
        inner = dim_head * heads
        context_dim = context_dim if context_dim is not None else query_dim
        self.heads, self.dim_head = heads, dim_head
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(context_dim, inner, bias=False)
        self.to_v = nn.Linear(context_dim, inner, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, query_dim), nn.Dropout(dropout))
        self.qk_norm = qk_norm
        if qk_norm:
            self.q_norm = _RMSNormParam(dim_head)
            self.k_norm = _RMSNormParam(dim_head)


class DiTBlock(nn.Module):
    """reference dit_models_xformers.py:231-295 (adaLN-Zero block) -- parameters only."""

    def __init__(self, hidden_size, num_heads, mlp_ratio=4.0, context_dim=None,
                 enable_rmsnorm=False, norm_type="layernorm", qk_norm=False, **block_kwargs):
        super().__init__()
        assert norm_type == "layernorm", "rmsnorm blocks: see dit_i23d (not built yet)"
        self.hidden_size, self.num_heads = hidden_size, num_heads
        self.attn = Attention(hidden_size, num_heads=num_heads, qkv_bias=True, qk_norm=qk_norm)
        self.mlp = _FusedMLP(hidden_size, int(mlp_ratio))
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 6 * hidden_size,
                                                                   bias=True))


class TextCondDiTBlock(DiTBlock):
    """reference dit_models_xformers.py:298-323: DiTBlock + un-gated, un-normed cross-attention."""

    def __init__(self, hidden_size, num_heads, mlp_ratio=4, **block_kwargs):
        super().__init__(hidden_size, num_heads, mlp_ratio, **block_kwargs)
        self.cross_attn = MemoryEfficientCrossAttention(query_dim=hidden_size, heads=num_heads)


class PixelArtTextCondDiTBlock(nn.Module):
    """reference dit_models_xformers.py:326-369 -- parameters only: RMSNorm pre-norms (eps 1e-5), plain
    attention, un-gated cross-attention on the block's own RMS-normed text tokens (attention_y_norm over
    context_dim), shared adaLN + per-block scale_shift_table (adaLN_modulation is None)."""

    def __init__(self, hidden_size, num_heads, mlp_ratio=4, context_dim=None, **block_kwargs):
        super().__init__()
        self.hidden_size, self.num_heads = hidden_size, num_heads
        self.norm1 = _RMSNormParam(hidden_size, eps=1e-5)
        self.norm2 = _RMSNormParam(hidden_size, eps=1e-5)
        self.attn = Attention(hidden_size, num_heads=num_heads, qkv_bias=True)
        self.mlp = _FusedMLP(hidden_size, int(mlp_ratio))
        self.cross_attn = MemoryEfficientCrossAttention(query_dim=hidden_size, context_dim=context_dim, heads=num_heads)
        self.scale_shift_table = nn.Parameter(torch.randn(6, hidden_size) / hidden_size ** 0.5)
        self.adaLN_modulation = None
        self.attention_y_norm = _RMSNormParam(context_dim, eps=1e-5)


class FinalLayer(nn.Module):
    """reference dit_models_xformers.py:655-678."""

    def __init__(self, hidden_size, patch_size, out_channels):
        super().__init__()
        self.linear = nn.Linear(hidden_size, patch_size * patch_size * out_channels, bias=True)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 2 * hidden_size,
                                                                   bias=True))


class T2IFinalLayer(nn.Module):
    """reference dit_models_xformers.py:61-84 (PixArt final layer with scale_shift_table)."""

    def __init__(self, hidden_size, patch_size, out_channels):
        super().__init__()
        self.linear = nn.Linear(hidden_size, patch_size * patch_size * out_channels, bias=True)
        self.scale_shift_table = nn.Parameter(torch.randn(2, hidden_size) / hidden_size ** 0.5)
        self.adaLN_modulation = None
        self.out_channels = out_channels


class _PatchEmbed(nn.Module):
    """timm PatchEmbed parameter layout (`proj` Conv2d k = s = patch)."""

    def __init__(self, img_size, patch_size, in_chans, embed_dim, bias=True):
        super().__init__()
        self.patch_size = (patch_size, patch_size)
        self.num_patches = (img_size // patch_size) ** 2
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size, bias=bias)


# ------------------------------------------------------------------ sin-cos positional tables
def get_1d_sincos_pos_embed_from_grid(embed_dim, pos):
    omega = np.arange(embed_dim // 2, dtype=np.float64)
    omega /= embed_dim / 2.0
    omega = 1.0 / 10000 ** omega
    out = np.einsum("m,d->md", pos.reshape(-1), omega)
    return np.concatenate([np.sin(out), np.cos(out)], axis=1)


def get_2d_sincos_pos_embed_from_grid(embed_dim, grid):
    emb_h = get_1d_sincos_pos_embed_from_grid(embed_dim // 2, grid[0])
    emb_w = get_1d_sincos_pos_embed_from_grid(embed_dim // 2, grid[1])
    return np.concatenate([emb_h, emb_w], axis=1)


def get_2d_sincos_pos_embed(embed_dim, grid_size, cls_token=False, extra_tokens=0):
    """reference dit_models_xformers.py:965-990 (tuple grid = (planes, tokens-per-plane))."""
    if isinstance(grid_size, tuple):
        gh, gw = grid_size
    else:
        gh = gw = grid_size
    grid_h = np.arange(gh, dtype=np.float32)
    grid_w = np.arange(gw, dtype=np.float32)
    grid = np.stack(np.meshgrid(grid_w, grid_h), axis=0).reshape([2, 1, gh, gw])
    return get_2d_sincos_pos_embed_from_grid(embed_dim, grid)
