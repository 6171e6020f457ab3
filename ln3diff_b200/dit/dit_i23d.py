"""Mirror of reference dit/dit_i23d.py: the image-conditioned flow-matching denoiser
`DiT_I23D_PixelArt` (:173-290) with `ImageCondDiTBlockPixelArtRMSNorm` blocks
(dit/dit_models_xformers.py:481-539,604-618) and `T2IFinalLayer` (:61-84), + the DiT_models registry
(:685-697).  Release I23D = `DiT_models['DiT-PixArt-L/2'](input_size=32, num_classes=0,
learn_sigma=False, in_channels=4, context_dim=1024, pooling_ctx_dim=768, roll_out=True)`.

What the reference recomputes every step although it is step-invariant is computed once per
prompt batch here and cached: the pooled-CLIP embedding (cap_embedder), the RMS-normalised CLIP
tokens and every layer's cross-attention K/V of them, the DINO projection and every layer's
self-attention K/V of the 256 DINO tokens (the reference concatenates them to the 768 latent tokens,
runs qkv/attention/proj on all 1024 rows and throws the DINO rows away, :522-530 -- here only the 768
latent query rows exist and the DINO K/V enter the attention kernel as a second K/V source).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import _lib, ops
from .._lib import NORM_LAYER, NORM_NONE, NORM_RMS
from ._pixart import PixArtGraphMixin
from .dit_trilatent import _attention_rows
from .dit_models_xformers import (Attention, CaptionEmbedder, MemoryEfficientCrossAttention, T2IFinalLayer,
                                  TimestepEmbedder, _FusedMLP, _PatchEmbed, _RMSNormParam,
                                  get_2d_sincos_pos_embed)


class ImageCondDiTBlockPixelArtRMSNorm(nn.Module):
    """Parameter container with the reference's keys: scale_shift_table (6, D), norm1/norm2 RMSNorm,
    attn (qkv, proj, q_norm, k_norm), cross_attn (to_q/k/v/out, q_norm, k_norm), mlp,
    attention_y_norm (unused in forward, kept for checkpoint compatibility)."""

    def __init__(self, hidden_size, num_heads, context_dim, mlp_ratio=4, **block_kwargs):
        super().__init__()
        self.norm1 = _RMSNormParam(hidden_size, eps=1e-5)
        self.norm2 = _RMSNormParam(hidden_size, eps=1e-5)
        self.attn = Attention(hidden_size, num_heads=num_heads, qkv_bias=True, qk_norm=True)
        self.mlp = _FusedMLP(hidden_size, int(mlp_ratio))
        self.cross_attn = MemoryEfficientCrossAttention(query_dim=hidden_size, context_dim=context_dim,
                                                        heads=num_heads, qk_norm=True)
        self.attention_y_norm = _RMSNormParam(1024, eps=1e-5)
        self.scale_shift_table = nn.Parameter(torch.randn(6, hidden_size) / hidden_size ** 0.5)
        self.adaLN_modulation = None


class ImageCondDiTBlockPixelArtRMSNormNoClip(ImageCondDiTBlockPixelArtRMSNorm):
    """reference dit/dit_models_xformers.py:541-601,621-635: the same parameters (attention_y_norm included, unused);
    its forward runs self-attention over the latent tokens only and cross-attends the multi-view DINO tokens."""


class DiT_I23D_PixelArt(PixArtGraphMixin, nn.Module):
    _ln3_fused_in_scale = False
    _vit_blk = ImageCondDiTBlockPixelArtRMSNorm

    def __init__(self, input_size=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4, class_dropout_prob=0.1, num_classes=1000, learn_sigma=True, mixing_logit_init=-3,
                 mixed_prediction=True, context_dim=False, pooling_ctx_dim=768, roll_out=False,
                 vit_blk=ImageCondDiTBlockPixelArtRMSNorm, final_layer_blk=None):
        super().__init__()
        assert roll_out
        if patch_size != 2 or hidden_size // num_heads != 64:
            raise NotImplementedError("libln3b200 implements patch_size=2, head_dim=64")
        if vit_blk is not self._vit_blk:
            raise NotImplementedError(f"{type(self).__name__} uses {self._vit_blk.__name__}")
        assert num_classes == 0
        self.plane_n, self.depth, self.mlp_ratio = 3, depth, mlp_ratio
        self.learn_sigma, self.in_channels = learn_sigma, in_channels
        self.out_channels = in_channels * 2 if learn_sigma else in_channels
        self.patch_size, self.num_heads, self.embed_dim = patch_size, num_heads, hidden_size
        self.input_size, self.roll_out = input_size, roll_out
        self.clip_ctx_dim = 1024
        self.x_embedder = _PatchEmbed(input_size, patch_size, in_channels, hidden_size, bias=True)
        self.t_embedder = TimestepEmbedder(hidden_size)
        self.y_embedder = None
        self.pos_embed = nn.Parameter(torch.zeros(1, 3 * self.x_embedder.num_patches, hidden_size), requires_grad=False)
        self.blocks = nn.ModuleList([vit_blk(hidden_size=hidden_size, num_heads=num_heads, mlp_ratio=mlp_ratio,
                                             context_dim=context_dim) for _ in range(depth)])
        self.final_layer = T2IFinalLayer(hidden_size, patch_size, self.out_channels)  # dit_i23d.py:48-52 ignores final_layer_blk
        self.dino_proj = CaptionEmbedder(context_dim, hidden_size)
        self.clip_spatial_proj = CaptionEmbedder(1024, hidden_size)   # unused in forward (kept for checkpoints)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 6 * hidden_size, bias=True))
        self.cap_embedder = nn.Sequential(nn.LayerNorm(pooling_ctx_dim), nn.Linear(pooling_ctx_dim, hidden_size))
        self.attention_y_norm = _RMSNormParam(1024, eps=1e-5)
        self.initialize_weights()
        self._invalidate()

    def initialize_weights(self):
        def _basic_init(m):
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
        self.apply(_basic_init)
        w = self.x_embedder.proj.weight.data
        nn.init.xavier_uniform_(w.view([w.shape[0], -1]))
        nn.init.constant_(self.x_embedder.proj.bias, 0)
        nn.init.normal_(self.t_embedder.mlp[0].weight, std=0.02)
        nn.init.normal_(self.t_embedder.mlp[2].weight, std=0.02)
        nn.init.constant_(self.final_layer.linear.weight, 0)
        nn.init.constant_(self.final_layer.linear.bias, 0)
        nn.init.constant_(self.adaLN_modulation[-1].weight, 0)
        nn.init.constant_(self.adaLN_modulation[-1].bias, 0)
        nn.init.constant_(self.cap_embedder[-1].weight, 0)
        nn.init.constant_(self.cap_embedder[-1].bias, 0)
        p = int(self.x_embedder.num_patches ** 0.5)
        D = self.pos_embed.shape[-1]
        pe = get_2d_sincos_pos_embed(D, (3, p * p)).reshape(3 * p * p, D)
        self.pos_embed.data.copy_(torch.from_numpy(pe).float().unsqueeze(0))

    @torch.no_grad()
    def prepare(self):
        dev = self.pos_embed.device
        if dev.type != "cuda":
            raise RuntimeError("ln3diff_b200 DiT runs on CUDA only (no CPU fallback)")
        bf = lambda w: w.detach().to(dev, torch.bfloat16).contiguous()
        f32 = lambda w: w.detach().to(dev, torch.float32).contiguous()
        D = self.embed_dim
        P = dict(t0_w=bf(self.t_embedder.mlp[0].weight), t0_b=f32(self.t_embedder.mlp[0].bias),
                 t2_w=bf(self.t_embedder.mlp[2].weight), t2_b=f32(self.t_embedder.mlp[2].bias),
                 ada_w=bf(self.adaLN_modulation[1].weight), ada_b=f32(self.adaLN_modulation[1].bias),
                 pe_w=f32(self.x_embedder.proj.weight), pe_b=f32(self.x_embedder.proj.bias), pos=f32(self.pos_embed),
                 fin_w=f32(self.final_layer.linear.weight), fin_b=f32(self.final_layer.linear.bias),
                 fin_tab=f32(self.final_layer.scale_shift_table),
                 tables=f32(torch.stack([b.scale_shift_table.detach().reshape(-1) for b in self.blocks], 0)),
                 **self._prepare_context_weights(bf, f32))
        blocks = []
        for b in self.blocks:
            qkv_w, qkv_b = b.attn.qkv.weight.detach(), b.attn.qkv.bias.detach()
            blocks.append(dict(
                n1_w=f32(b.norm1.weight), n2_w=f32(b.norm2.weight),
                qkv_w=bf(qkv_w), qkv_b=f32(qkv_b),
                qk_norm=f32(torch.stack([b.attn.q_norm.weight.detach(), b.attn.k_norm.weight.detach()], 0)),
                **self._prepare_block_context_weights(b, bf, f32),
                proj_w=bf(b.attn.proj.weight), proj_b=f32(b.attn.proj.bias),
                cq_w=bf(b.cross_attn.to_q.weight), cq_norm=f32(b.cross_attn.q_norm.weight.detach()[None]),
                ckv_w=bf(torch.cat([b.cross_attn.to_k.weight.detach(), b.cross_attn.to_v.weight.detach()], 0)),
                ck_norm=f32(b.cross_attn.k_norm.weight.detach()[None]),
                co_w=bf(b.cross_attn.to_out[0].weight), co_b=f32(b.cross_attn.to_out[0].bias),
                fc1_w=bf(b.mlp.mlp[0].weight), fc1_b=f32(b.mlp.mlp[1].bias),
                fc2_w=bf(b.mlp.mlp[2].weight), fc2_b=f32(b.mlp.mlp[3].bias)))
        P["blocks"] = blocks
        self._invalidate()
        self._prep = P
        return P

    def _prepare_context_weights(self, bf, f32) -> dict:
        """Model-level weights of the conditioning: cap_embedder, attention_y_norm, dino_proj."""
        return dict(cap_ln_w=f32(self.cap_embedder[0].weight), cap_ln_b=f32(self.cap_embedder[0].bias),
                    cap_w=bf(self.cap_embedder[1].weight), cap_b=f32(self.cap_embedder[1].bias),
                    ynorm_w=f32(self.attention_y_norm.weight),
                    d1_w=bf(self.dino_proj.y_proj.fc1.weight), d1_b=f32(self.dino_proj.y_proj.fc1.bias),
                    d2_w=bf(self.dino_proj.y_proj.fc2.weight), d2_b=f32(self.dino_proj.y_proj.fc2.bias))

    def _prepare_block_context_weights(self, b, bf, f32) -> dict:
        """Per-block K|V rows of the qkv projection (and the k_norm) for the DINO tokens of self-attention."""
        D = self.embed_dim
        return dict(kv_w=bf(b.attn.qkv.weight[D:]), kv_b=f32(b.attn.qkv.bias[D:]),
                    k_norm=f32(b.attn.k_norm.weight.detach()[None]))

    @torch.no_grad()
    def _context(self, context):
        """Step-invariant conditioning, once per prompt batch: pooled-CLIP embedding, per-layer
        cross-attention K/V of the RMS-normed CLIP tokens, per-layer self-attention K/V of the
        projected DINO tokens."""
        vec0, ca0 = vec, ca = context["vector"], context["crossattn"]
        hit = self._ctx_cache.get(vec0, ca0)
        if hit is not None:
            return hit
        P, D = self._prep, self.embed_dim
        B, Lc, _ = ca.shape
        dev = ca.device
        # model-owned static outputs (captured graphs read them through raw pointers; see dit/_graph.py)
        st = self._static((B, Lc), lambda: dict(
            cls=torch.empty(B, D, device=dev, dtype=torch.float32),
            ckv=torch.empty(self.depth, B, Lc, 2 * D, device=dev, dtype=torch.bfloat16),
            dkv=torch.empty(self.depth, B, Lc, 2 * D, device=dev, dtype=torch.bfloat16),
            oc=torch.empty(self.depth, B, D, device=dev, dtype=torch.bfloat16)))
        vec = vec.float().contiguous()
        ones = torch.ones(1, device=dev)
        # cap_embedder: LayerNorm(affine, eps 1e-5) -> Linear.  LN(x)*w + b == LN(x)*(1 + (w-1)) + b
        vn = ops.norm_modulate(vec, norm=NORM_LAYER, eps=1e-5, shift=P["cap_ln_b"][None], scale=(P["cap_ln_w"] - 1)[None],
                               mod_rows=B)
        cls = ops.gemm(vn, P["cap_w"], P["cap_b"], out_kind=ops.OUT_F32, out=st["cls"])   # (B, D) fp32
        ca = ca.float()
        clip = ops.norm_modulate(ca[..., :1024].reshape(B * Lc, 1024).contiguous(), norm=NORM_RMS, weight=P["ynorm_w"], eps=1e-5)
        dino_in = ops.norm_modulate(ca[..., 1024:].reshape(B * Lc, -1).contiguous(), norm=NORM_NONE)
        dino = ops.gemm(ops.gemm(dino_in, P["d1_w"], P["d1_b"], act=ops.ACT_GELU_TANH), P["d2_w"], P["d2_b"])
        ckv, dkv = st["ckv"], st["dkv"]
        for l, W in enumerate(P["blocks"]):
            ops.gemm(clip, W["ckv_w"], out=ckv[l].view(B * Lc, 2 * D), head_norm=W["ck_norm"], head_norm_sec_cols=D)
            ops.gemm(dino, W["kv_w"], W["kv_b"], out=dkv[l].view(B * Lc, 2 * D), head_norm=W["k_norm"], head_norm_sec_cols=D)
        out = dict(cls=cls, ckv=ckv, dkv=dkv, rows=(0, B), oconst=None)
        # identical CLIP tokens (the all-zero unconditional half of forward_with_cfg): softmax over identical
        # keys is uniform -> cross-attention output = to_out(v_row); see DiT_TriLatent._context_kv
        rows = _attention_rows(ca[..., :1024])
        if rows is not None:
            oc = st["oc"]
            for l, W in enumerate(P["blocks"]):
                ops.gemm(ckv[l][:, 0, D:].contiguous(), W["co_w"], W["co_b"], out=oc[l])
            out.update(rows=rows, oconst=oc)
        return self._ctx_cache.put((vec0, ca0), out)

    @torch.no_grad()
    def forward(self, x, timesteps=None, context=None, y=None, get_attr="", **kwargs):
        """x (B, 12, 32, 32); timesteps (B,) float in [0,1]; context {'vector','crossattn'}."""
        if get_attr != "":
            return getattr(self, get_attr)
        assert isinstance(context, dict)
        if not x.is_cuda:
            raise RuntimeError("ln3diff_b200 DiT runs on CUDA only (no CPU fallback)")
        if self._prep is None:
            self.prepare()
        t = timesteps.to(device=x.device, dtype=torch.float32).contiguous()
        return self._run(x, t, self._context(context))

    @torch.no_grad()
    def forward_with_cfg(self, x, t, context, cfg_scale):
        """reference dit_i23d.py:155-168 (cond first, uncond second; returns cat([half, half]))."""
        eps = self.forward(x, t, context)
        cond_eps, uncond_eps = torch.split(eps, len(eps) // 2, dim=0)
        half = uncond_eps + cfg_scale * (cond_eps - uncond_eps)
        return torch.cat([half, half], dim=0)


class DiT_I23D_PixelArt_MVCond_noClip(DiT_I23D_PixelArt):
    """Mirror of reference dit/dit_i23d.py:392-492, the multi-view denoiser of the MV23D release
    (`DiT-PixArt-MV-L/2`, shell_scripts/final_release/inference/sample_obajverse_mv23d_dit.sh): the I23D PixArt
    model without dino_proj / clip_spatial_proj / cap_embedder, so t = t_embedder(timesteps) alone, and
    `ImageCondDiTBlockPixelArtRMSNormNoClip` blocks: self-attention over the 768 latent tokens only and
    cross-attention to the flattened multi-view DINO tokens context['concat'] (B, V, 256, C) -> (B, V*256, C), with
    no attention_y_norm.  Same launch sequence as DiT_I23D_PixelArt (`pixart_forward`): the pooled embedding is a
    zero row, there is no second self-attention K/V source, and every layer's cross-attention K|V of the DINO tokens
    is computed once per condition batch."""
    _vit_blk = ImageCondDiTBlockPixelArtRMSNormNoClip

    def __init__(self, input_size=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4, class_dropout_prob=0.1, num_classes=1000, learn_sigma=True, mixing_logit_init=-3,
                 mixed_prediction=True, context_dim=False, pooling_ctx_dim=768, roll_out=False, vit_blk=None,
                 final_layer_blk=None):
        # the reference passes ImageCondDiTBlockPixelArtRMSNormNoClip whatever vit_blk says (:413-420)
        super().__init__(input_size, patch_size, in_channels, hidden_size, depth, num_heads, mlp_ratio,
                         class_dropout_prob, num_classes, learn_sigma, mixing_logit_init, mixed_prediction, context_dim,
                         pooling_ctx_dim, roll_out, ImageCondDiTBlockPixelArtRMSNormNoClip, final_layer_blk)
        del self.dino_proj
        del self.clip_spatial_proj, self.cap_embedder

    def _prepare_context_weights(self, bf, f32) -> dict:
        return {}

    def _prepare_block_context_weights(self, b, bf, f32) -> dict:
        return {}

    @torch.no_grad()
    def _context(self, context):
        """Step-invariant conditioning, once per condition batch: every layer's cross-attention K|V of the
        flattened DINO tokens (one GEMM per layer with the k_norm head epilogue)."""
        ca0 = context["concat"]
        hit = self._ctx_cache.get(ca0)
        if hit is not None:
            return hit
        P, D = self._prep, self.embed_dim
        B = ca0.shape[0]
        tok = ca0.reshape(B, -1, ca0.shape[-1]).float()               # 'b v l c -> b (v l) c'
        Lc = tok.shape[1]
        dev = tok.device
        st = self._static((B, Lc), lambda: dict(
            cls=torch.zeros(B, D, device=dev, dtype=torch.float32),  # no pooled embedding: t + 0 == t
            ckv=torch.empty(self.depth, B, Lc, 2 * D, device=dev, dtype=torch.bfloat16),
            oc=torch.empty(self.depth, B, D, device=dev, dtype=torch.bfloat16)))
        ctx = ops.norm_modulate(tok.reshape(B * Lc, -1).contiguous(), norm=NORM_NONE)   # bf16 GEMM operand
        ckv = st["ckv"]
        for l, W in enumerate(P["blocks"]):
            ops.gemm(ctx, W["ckv_w"], out=ckv[l].view(B * Lc, 2 * D), head_norm=W["ck_norm"], head_norm_sec_cols=D)
        out = dict(cls=st["cls"], ckv=ckv, rows=(0, B), oconst=None)
        # the all-zero unconditional half: closed-form cross-attention (see DiT_I23D_PixelArt._context)
        rows = _attention_rows(tok)
        if rows is not None:
            oc = st["oc"]
            for l, W in enumerate(P["blocks"]):
                ops.gemm(ckv[l][:, 0, D:].contiguous(), W["co_w"], W["co_b"], out=oc[l])
            out.update(rows=rows, oconst=oc)
        return self._ctx_cache.put((ca0,), out)


def _mk(depth, hidden, heads, cls=DiT_I23D_PixelArt):
    def f(**kwargs):
        return cls(depth=depth, hidden_size=hidden, patch_size=2, num_heads=heads, **kwargs)
    return f


def _unbuilt(name):
    def f(**kwargs):
        raise NotImplementedError(f"{name}: not implemented in ln3diff_b200 (release I23D = DiT-PixArt-L/2, "
                                  f"release MV23D = DiT-PixArt-MV-L/2)")
    return f


# reference dit/dit_i23d.py:685-697 ('DiT-PixArt-MV-L/2' -> DiT_L_Pixelart_MV_2_noclip, :651-656,693)
DiT_models = {"DiT-PixArt-L/2": _mk(24, 1024, 16), "DiT-PixArt-B/2": _mk(12, 768, 12),
              "DiT-PixArt-MV-L/2": _mk(24, 1024, 16, DiT_I23D_PixelArt_MVCond_noClip),
              **{k: _unbuilt(k) for k in ("DiT-XL/2", "DiT-L/2", "DiT-B/2", "DiT-B/1", "DiT-PixArt-MV-XL/2",
                                         "DiT-PixArt-MV-PCD-L", "DiT-PixArt-MV-B/2")}}
