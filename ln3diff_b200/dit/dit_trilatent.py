"""Mirror of reference dit/dit_trilatent.py: DiT_TriLatent (T23D denoiser) + DiT_models registry.

`DiT_models[arch](input_size=32, num_classes=0, learn_sigma=False, in_channels=4,
context_dim=768, roll_out=True, vit_blk=TextCondDiTBlock)` is how the reference builds the
denoiser (guided_diffusion/script_util.py:407-415); `.forward(x, timesteps, context)` returns the
fp32 contiguous (B, 3*C, 32, 32) prediction (dit_trilatent.py:74-143).  The forward is a fixed
sequence of libln3b200 launches (dit/_denoiser.py) -- wgmma GEMMs with fused bias/GELU/gate-residual
epilogues, the wgmma attention kernel, and three small SIMT kernels -- with fp32 residual
stream and bf16 GEMM operands (the reference's bf16-autocast GPU path keeps the same split).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import ops
from .._lib import NORM_LAYER, NORM_NONE, NORM_RMS
from ._denoiser import DenoiserMixin, PixArtMixin, cross_attention_context, run_blocks, split_kv
from ._denoiser import _attention_rows  # noqa: F401  (re-exported: callers import it from this module)
from ._graph import ForwardGraph
from .dit_models_xformers import (CaptionEmbedder, DiTBlock, FinalLayer, PixelArtTextCondDiTBlock, T2IFinalLayer,
                                  TextCondDiTBlock, TimestepEmbedder, _PatchEmbed)


class DiT_TriLatent(DenoiserMixin, nn.Module):
    """reference dit/dit_trilatent.py:22-143 (+ base dit_models_xformers.py:681-819)."""

    _ln3_fused_in_scale = True

    def __init__(self, input_size=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28,
                 num_heads=16, mlp_ratio=4, class_dropout_prob=0.1, num_classes=1000,
                 learn_sigma=True, mixing_logit_init=-3, mixed_prediction=True, context_dim=False,
                 roll_out=False, vit_blk=DiTBlock, final_layer_blk=FinalLayer):
        super().__init__()
        assert roll_out, "DiT_TriLatent requires roll_out=True (dit_trilatent.py:49)"
        if patch_size != 2:
            raise NotImplementedError("libln3b200 implements patch_size=2 (every release config)")
        if hidden_size % num_heads or hidden_size // num_heads not in (64, 72):
            raise NotImplementedError("libln3b200 attention implements head_dim 64 (DiT-S/B/L) and 72 (DiT-XL)")
        if vit_blk is not TextCondDiTBlock:
            raise NotImplementedError("T23D path is built with vit_blk=TextCondDiTBlock "
                                      "(guided_diffusion/script_util.py:407-415)")
        self.plane_n = 3
        self.depth, self.mlp_ratio = depth, mlp_ratio
        self.learn_sigma, self.in_channels = learn_sigma, in_channels
        self.out_channels = in_channels * 2 if learn_sigma else in_channels
        self.patch_size, self.num_heads, self.embed_dim = patch_size, num_heads, hidden_size
        self.input_size = input_size
        self.roll_out = roll_out

        self.x_embedder = _PatchEmbed(input_size, patch_size, in_channels, hidden_size, bias=True)
        self.t_embedder = TimestepEmbedder(hidden_size)
        self.y_embedder = None
        assert num_classes == 0, "class-conditional label embedding is not on the hot path"
        self.clip_text_proj = CaptionEmbedder(context_dim, hidden_size) if context_dim else None
        self.pos_embed = nn.Parameter(
            torch.zeros(1, self.plane_n * self.x_embedder.num_patches, hidden_size),
            requires_grad=False)
        self.blocks = nn.ModuleList([
            vit_blk(hidden_size=hidden_size, num_heads=num_heads, mlp_ratio=mlp_ratio,
                    context_dim=context_dim) for _ in range(depth)])
        self.final_layer = final_layer_blk(hidden_size, patch_size, self.out_channels)
        self.initialize_weights()
        self._invalidate()

    def initialize_weights(self):
        """reference :786-819: adaLN-Zero (every block's and the final layer's adaLN_modulation)."""
        zeroed = [b.adaLN_modulation[-1] for b in self.blocks]
        if getattr(self.final_layer, "adaLN_modulation", None) is not None:
            zeroed.append(self.final_layer.adaLN_modulation[-1])
        super().initialize_weights(zeroed)

    def _pack(self, bf, f32) -> dict:
        """adaLN projections of all blocks + final layer are concatenated so one GEMM per step produces every
        shift/scale/gate; the K/V projections of the (step-invariant) context for all layers likewise."""
        ada_w = [b.adaLN_modulation[1].weight for b in self.blocks]
        ada_b = [b.adaLN_modulation[1].bias for b in self.blocks]
        if getattr(self.final_layer, "adaLN_modulation", None) is not None:
            ada_w.append(self.final_layer.adaLN_modulation[1].weight)
            ada_b.append(self.final_layer.adaLN_modulation[1].bias)
        P = dict(ada_w=bf(torch.cat([w.detach() for w in ada_w], 0)),
                 ada_b=f32(torch.cat([b.detach() for b in ada_b], 0)),
                 kv_w=bf(torch.cat([torch.cat([b.cross_attn.to_k.weight.detach(),
                                               b.cross_attn.to_v.weight.detach()], 0) for b in self.blocks], 0)))
        if self.clip_text_proj is not None:
            P["c1_w"], P["c1_b"] = bf(self.clip_text_proj.y_proj.fc1.weight), f32(self.clip_text_proj.y_proj.fc1.bias)
            P["c2_w"], P["c2_b"] = bf(self.clip_text_proj.y_proj.fc2.weight), f32(self.clip_text_proj.y_proj.fc2.bias)
        return P

    def _mod_workspace(self, B, e) -> dict:
        return dict(mod=e(B, self._prep["ada_w"].shape[0], dt=torch.float32))

    @torch.no_grad()
    def _context(self, context):
        """context (B, L, ctx_dim) or {'crossattn': ...}: clip_text_proj + every layer's to_k/to_v, and the
        closed-form rows of identical-token samples (`cross_attention_context`).  The reference recomputes these
        every step (dit_trilatent.py:107, ldm/modules/attention.py:281-283) although the context is
        step-invariant; cached here keyed on the tensor identity/version."""
        assert context is not None
        if isinstance(context, dict):
            context = context["crossattn"]
        hit = self._ctx_cache.get(context)
        if hit is not None:
            return hit
        P = self._prep
        B, Lc, Cc = context.shape
        D = self.embed_dim
        E = self.blocks[0].cross_attn.to_k.out_features   # 64 x heads: D, or 1024 for DiT-XL/2
        # Static, model-owned output buffers per (B, Lc): captured graphs read K/V and the closed-form rows
        # through raw pointers, so a new prompt batch rewrites them in place and replays the same graph.
        st = self._static((B, Lc), lambda: dict(
            kv=torch.empty(B * Lc, self.depth * 2 * E, device=context.device, dtype=torch.bfloat16),
            oc=torch.empty(self.depth, B, D, device=context.device, dtype=torch.bfloat16)))
        c = context.reshape(B * Lc, Cc).float().contiguous()
        cb = ops.norm_modulate(c, norm=NORM_NONE)
        c1 = ops.gemm(cb, P["c1_w"], P["c1_b"], act=ops.ACT_GELU_TANH)
        c2 = ops.gemm(c1, P["c2_w"], P["c2_b"])
        ops.gemm(c2, P["kv_w"], out=st["kv"])  # every layer's K|V in one GEMM: (B*Lc, depth*2*E)
        kv = st["kv"].view(B, Lc, self.depth, 2, E)
        kv = [(kv[:, :, l, 0], kv[:, :, l, 1]) for l in range(self.depth)]
        return self._ctx_cache.put((context,), cross_attention_context(kv, c2.view(B, Lc, -1), P["blocks"], st["oc"]))

    @torch.no_grad()
    def modulation_table(self, t_values: torch.Tensor) -> torch.Tensor:
        """adaLN modulations of every block + final layer for S timestep values at once: (S, (6L+2)·D) fp32.
        In a sampling loop all samples of a step share one timestep, so the reference's per-step
        `t_embedder` + 25 `adaLN_modulation` evaluations (identical rows for the whole batch,
        dit_trilatent.py:91, dit_models_xformers.py:285-294) collapse into one row per step; computing all
        steps' rows in one pass reads the 302 MB of adaLN weights once per sampling run instead of once per
        step.  Same kernels, same per-row arithmetic as the in-forward path."""
        if self._prep is None:
            self.prepare()
        P = self._prep
        t = t_values.to(device=self.pos_embed.device, dtype=torch.float32).contiguous()
        tf = ops.timestep_embedding(t)
        th = ops.gemm(tf, P["t0_w"], P["t0_b"], act=ops.ACT_SILU)
        st = ops.gemm(th, P["t2_w"], P["t2_b"], act=ops.ACT_SILU)
        return ops.gemm(st, P["ada_w"], P["ada_b"], out_kind=ops.OUT_F32)

    def _forward_impl(self, x, t, cx, in_scale, mod_row):
        """The fixed launch sequence of one forward.  `in_scale` (B,) or None: the denoiser's c_in, folded into
        the patch embed.  `mod_row` (1, (6L+2)·D): a row of modulation_table() shared by every sample of the
        batch (replaces the timestep embedder + adaLN GEMM)."""
        P = self._prep
        B = x.shape[0]
        D, T = self.embed_dim, self.pos_embed.shape[1]
        ws = self._workspace(B)
        if mod_row is not None:
            mod = mod_row.expand(B, mod_row.shape[1])       # stride-0 rows: every sample reads the same row
        else:
            ops.timestep_embedding(t, out=ws["tfeat"])
            ops.gemm(ws["tfeat"], P["t0_w"], P["t0_b"], act=ops.ACT_SILU, out=ws["th"])
            ops.gemm(ws["th"], P["t2_w"], P["t2_b"], act=ops.ACT_SILU, out=ws["st"])  # silu(t_emb)
            mod = ops.gemm(ws["st"], P["ada_w"], P["ada_b"], out_kind=ops.OUT_F32, out=ws["mod"])
        xs = ops.patch_embed(x, P["pe_w"], P["pe_b"], P["pos"], in_scale=in_scale, out=ws["x"])
        mods = [mod[:, l * 6 * D:(l + 1) * 6 * D] for l in range(self.depth)]
        run_blocks(P["blocks"], cx, ws, xs.view(B * T, D), mods, self.num_heads, T)
        f0 = self.depth * 6 * D
        return ops.final_layer(xs, mod[:, f0:f0 + D], mod[:, f0 + D:f0 + 2 * D], P["fin_w"],
                               P["fin_b"], self.input_size)

    @torch.no_grad()
    def capture_graph(self, B, context, shared_mod: bool = False) -> ForwardGraph:
        """CUDA graph of one forward for batch B conditioned on `context`: the ~270 launches of a forward
        replay as one graph launch.  Computes the step-invariant conditioning of `context` (into the model's
        static buffers) and returns the graph cached for this launch-sequence shape -- a later call with a
        new prompt batch of the same shape refreshes the buffers and returns the SAME graph object, it does
        not capture again.  Static inputs .x (B,3C,S,S), .t (B,), .in_scale (B,), [.mod]; static output .out;
        .replay().  The graph always reflects the context of the most recent `capture_graph`/`forward` call."""
        if self._prep is None:
            self.prepare()
        return self._graph(B, self._context(context), shared_mod)


class DiT_TriLatent_PixelArt(PixArtMixin, nn.Module):
    """reference dit/dit_trilatent.py:146-246: the PixArt-style T23D denoiser -- one shared adaLN
    (`adaLN_modulation` on t_emb + cap_embedder(pooled CLIP)) plus per-block `scale_shift_table`,
    `PixelArtTextCondDiTBlock` blocks, `T2IFinalLayer`.  context = {'vector': (B, context_dim) pooled
    CLIP, 'crossattn': (B, 77, context_dim) CLIP tokens}.

    Step-invariant work is cached per prompt batch: the pooled-CLIP embedding and every block's
    cross-attention K/V (each block RMS-normalises the tokens with its own `attention_y_norm` first; the
    reference redoes both in every block of every step, dit_models_xformers.py:364)."""

    def __init__(self, input_size=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28, num_heads=16,
                 mlp_ratio=4, class_dropout_prob=0.1, num_classes=1000, learn_sigma=True, mixing_logit_init=-3,
                 mixed_prediction=True, context_dim=False, roll_out=False, vit_blk=None, final_layer_blk=T2IFinalLayer):
        super().__init__()
        assert roll_out, "DiT_TriLatent requires roll_out=True (dit_trilatent.py:49)"
        if patch_size != 2 or hidden_size // num_heads != 64:
            raise NotImplementedError("libln3b200 implements patch_size=2, head_dim=64")
        if final_layer_blk is not T2IFinalLayer:
            raise NotImplementedError("the PixelArt T23D registry entries use T2IFinalLayer (dit_trilatent.py:301-316)")
        assert num_classes == 0 and context_dim
        self.plane_n, self.depth, self.mlp_ratio = 3, depth, mlp_ratio
        self.learn_sigma, self.in_channels = learn_sigma, in_channels
        self.out_channels = in_channels * 2 if learn_sigma else in_channels
        self.patch_size, self.num_heads, self.embed_dim = patch_size, num_heads, hidden_size
        self.input_size, self.roll_out, self.context_dim = input_size, roll_out, context_dim
        self.x_embedder = _PatchEmbed(input_size, patch_size, in_channels, hidden_size, bias=True)
        self.t_embedder = TimestepEmbedder(hidden_size)
        self.y_embedder = None
        self.pos_embed = nn.Parameter(torch.zeros(1, 3 * self.x_embedder.num_patches, hidden_size), requires_grad=False)
        # the reference ignores the caller's vit_blk here (dit_trilatent.py:167-171)
        self.blocks = nn.ModuleList([PixelArtTextCondDiTBlock(hidden_size=hidden_size, num_heads=num_heads,
                                                              mlp_ratio=mlp_ratio, context_dim=context_dim)
                                     for _ in range(depth)])
        self.final_layer = T2IFinalLayer(hidden_size, patch_size, self.out_channels)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 6 * hidden_size, bias=True))
        self.cap_embedder = nn.Sequential(nn.LayerNorm(context_dim), nn.Linear(context_dim, hidden_size))
        self.initialize_weights()
        self._invalidate()

    def initialize_weights(self):
        super().initialize_weights([self.cap_embedder[-1]])

    def _pack_context(self, bf, f32) -> dict:
        return dict(cap_ln_w=f32(self.cap_embedder[0].weight), cap_ln_b=f32(self.cap_embedder[0].bias),
                    cap_w=bf(self.cap_embedder[1].weight), cap_b=f32(self.cap_embedder[1].bias))

    def _pack_block(self, b, bf, f32) -> dict:
        return dict(n1_w=f32(b.norm1.weight), n2_w=f32(b.norm2.weight), yn_w=f32(b.attention_y_norm.weight),
                    ckv_w=bf(torch.cat([b.cross_attn.to_k.weight.detach(), b.cross_attn.to_v.weight.detach()], 0)))

    @torch.no_grad()
    def _context(self, context):
        assert context is not None and isinstance(context, dict), "PixelArt T23D needs {'vector','crossattn'}"
        vec0, ca0 = vec, ca = context["vector"], context["crossattn"]
        hit = self._ctx_cache.get(vec0, ca0)
        if hit is not None:
            return hit
        P, D = self._prep, self.embed_dim
        B, Lc, Cc = ca.shape
        st = self._static((B, Lc), lambda: dict(
            cls=torch.empty(B, D, device=ca.device, dtype=torch.float32),
            ckv=torch.empty(self.depth, B, Lc, 2 * D, device=ca.device, dtype=torch.bfloat16),
            oc=torch.empty(self.depth, B, D, device=ca.device, dtype=torch.bfloat16)))
        vec = vec.float().contiguous()
        # cap_embedder: LayerNorm(affine, eps 1e-5) -> Linear.  LN(x)*w + b == LN(x)*(1 + (w-1)) + b
        vn = ops.norm_modulate(vec, norm=NORM_LAYER, eps=1e-5, shift=P["cap_ln_b"][None], scale=(P["cap_ln_w"] - 1)[None],
                               mod_rows=B)
        cls = ops.gemm(vn, P["cap_w"], P["cap_b"], out_kind=ops.OUT_F32, out=st["cls"])   # (B, D) fp32
        ca2 = ca.float().reshape(B * Lc, Cc).contiguous()
        ckv = st["ckv"]
        for l, W in enumerate(P["blocks"]):
            y = ops.norm_modulate(ca2, norm=NORM_RMS, weight=W["yn_w"], eps=1e-5)
            ops.gemm(y, W["ckv_w"], out=ckv[l].view(B * Lc, 2 * D))
        return self._ctx_cache.put((vec0, ca0), cross_attention_context(split_kv(ckv), ca.float(), P["blocks"],
                                                                         st["oc"], cls=cls))


def DiT_XL_2(**kwargs):
    return DiT_TriLatent(depth=28, hidden_size=1152, patch_size=2, num_heads=16, **kwargs)


def DiT_L_2(**kwargs):
    return DiT_TriLatent(depth=24, hidden_size=1024, patch_size=2, num_heads=16, **kwargs)


def DiT_B_2(**kwargs):
    return DiT_TriLatent(depth=12, hidden_size=768, patch_size=2, num_heads=12, **kwargs)


def DiT_B_1(**kwargs):
    return DiT_TriLatent(depth=12, hidden_size=768, patch_size=1, num_heads=12, **kwargs)


def DiT_B_Pixelart_2(**kwargs):
    return DiT_TriLatent_PixelArt(depth=12, hidden_size=768, patch_size=2, num_heads=12,
                                  final_layer_blk=T2IFinalLayer, **kwargs)


def DiT_L_Pixelart_2(**kwargs):
    return DiT_TriLatent_PixelArt(depth=24, hidden_size=1024, patch_size=2, num_heads=16,
                                  final_layer_blk=T2IFinalLayer, **kwargs)


# reference dit/dit_trilatent.py:320-327
DiT_models = {
    "DiT-XL/2": DiT_XL_2,
    "DiT-L/2": DiT_L_2,
    "DiT-PixelArt-L/2": DiT_L_Pixelart_2,
    "DiT-PixelArt-B/2": DiT_B_Pixelart_2,
    "DiT-B/2": DiT_B_2,
    "DiT-B/1": DiT_B_1,
}
