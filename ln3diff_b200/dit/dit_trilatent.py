"""Mirror of reference dit/dit_trilatent.py: DiT_TriLatent (T23D denoiser) + DiT_models registry.

`DiT_models[arch](input_size=32, num_classes=0, learn_sigma=False, in_channels=4,
context_dim=768, roll_out=True, vit_blk=TextCondDiTBlock)` is how the reference builds the
denoiser (guided_diffusion/script_util.py:407-415); `.forward(x, timesteps, context)` returns the
fp32 contiguous (B, 3*C, 32, 32) prediction (dit_trilatent.py:74-143).  The forward below is a
fixed sequence of libln3b200 launches -- wgmma GEMMs with fused bias/GELU/gate-residual
epilogues, the wgmma attention kernel, and three small SIMT kernels -- with fp32 residual
stream and bf16 GEMM operands (the reference's bf16-autocast GPU path keeps the same split).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .. import _lib, ops
from .._lib import NORM_LAYER, NORM_NONE, NORM_RMS
from ._graph import ContextCache, ForwardGraph, capture_forward, graphs_enabled
from ._pixart import PixArtGraphMixin
from .dit_models_xformers import (CaptionEmbedder, DiTBlock, FinalLayer, PixelArtTextCondDiTBlock, T2IFinalLayer,
                                  TextCondDiTBlock, TimestepEmbedder, _PatchEmbed,
                                  get_2d_sincos_pos_embed)


def _closed_form_uncond() -> bool:
    """LN3_UNCOND_CLOSED_FORM=0 forces full cross-attention for identical-token samples (A/B, tests)."""
    import os
    return os.environ.get("LN3_UNCOND_CLOSED_FORM", "1") != "0"


def _split_residual_pass() -> bool:
    """LN3_SPLIT_RESID_PASS=0: the post-self-attention residual pass covers every row (A/B, tests)."""
    import os
    return os.environ.get("LN3_SPLIT_RESID_PASS", "1") != "0"


def _attention_rows(tokens: torch.Tensor):
    """tokens (B, L, C) as the cross-attention sees them.  Returns (g0, g1): the contiguous block of samples
    that needs real attention when the samples whose L tokens are all identical form a prefix and/or suffix
    of the batch (both CFG layouts of the reference), else None.  One host sync; callers cache per context."""
    B, L, _ = tokens.shape
    if not _closed_form_uncond() or L < 2:
        return None
    same = (tokens == tokens[:, :1]).all(dim=2).all(dim=1).tolist()
    g0 = 0
    while g0 < B and same[g0]:
        g0 += 1
    g1 = B
    while g1 > g0 and same[g1 - 1]:
        g1 -= 1
    if (g0 > 0 or g1 < B) and not any(same[g0:g1]):
        return g0, g1
    return None


class DiT_TriLatent(nn.Module):
    """reference dit/dit_trilatent.py:22-143 (+ base dit_models_xformers.py:681-819)."""

    _ln3_fused_in_scale = True  # forward(..., in_scale=) folds the denoiser's c_in into patch embed

    def __init__(self, input_size=32, patch_size=2, in_channels=4, hidden_size=1152, depth=28,
                 num_heads=16, mlp_ratio=4, class_dropout_prob=0.1, num_classes=1000,
                 learn_sigma=True, mixing_logit_init=-3, mixed_prediction=True, context_dim=False,
                 roll_out=False, vit_blk=DiTBlock, final_layer_blk=FinalLayer):
        super().__init__()
        assert roll_out, "DiT_TriLatent requires roll_out=True (dit_trilatent.py:49)"
        if patch_size != 2:
            raise NotImplementedError("libln3b200 implements patch_size=2 (every release config)")
        if hidden_size // num_heads != 64:
            raise NotImplementedError("libln3b200 attention implements head_dim=64 (DiT-S/B/L)")
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

    def _invalidate(self):
        """Drop everything derived from the parameters: bf16 repacks, workspaces, the cached conditioning
        and its static buffers, and the captured graphs (they hold raw pointers into all of those)."""
        self._prep = None
        self._ws = {}
        self._ctx_cache = ContextCache()
        self._ctx_static = {}
        self._graphs = {}

    # ------------------------------------------------------------------ init (reference :786-819)
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
        for block in self.blocks:
            nn.init.constant_(block.adaLN_modulation[-1].weight, 0)
            nn.init.constant_(block.adaLN_modulation[-1].bias, 0)
        if getattr(self.final_layer, "adaLN_modulation", None) is not None:
            nn.init.constant_(self.final_layer.adaLN_modulation[-1].weight, 0)
            nn.init.constant_(self.final_layer.adaLN_modulation[-1].bias, 0)
        nn.init.constant_(self.final_layer.linear.weight, 0)
        nn.init.constant_(self.final_layer.linear.bias, 0)
        self.init_PE_3D_aware()

    def init_PE_3D_aware(self):
        p = int(self.x_embedder.num_patches ** 0.5)
        D = self.pos_embed.shape[-1]
        pe = get_2d_sincos_pos_embed(D, (self.plane_n, p * p)).reshape(self.plane_n * p * p, D)
        self.pos_embed.data.copy_(torch.from_numpy(pe).float().unsqueeze(0))

    # ------------------------------------------------------------------ weight repack
    def _apply(self, fn, *a, **kw):
        self._invalidate()
        return super()._apply(fn, *a, **kw)

    def load_state_dict(self, *a, **kw):
        self._invalidate()
        return super().load_state_dict(*a, **kw)

    @torch.no_grad()
    def prepare(self):
        """One-time bf16 repack of the GEMM weights (owned by the module, rebuilt after
        load_state_dict / .to()); adaLN projections of all blocks + final layer are concatenated
        so one GEMM per step produces every shift/scale/gate."""
        dev = self.pos_embed.device
        if dev.type != "cuda":
            raise RuntimeError("ln3diff_b200 DiT runs on CUDA only (no CPU fallback)")
        bf = lambda w: w.detach().to(dev, torch.bfloat16).contiguous()
        f32 = lambda w: w.detach().to(dev, torch.float32).contiguous()
        P = {}
        P["t0_w"], P["t0_b"] = bf(self.t_embedder.mlp[0].weight), f32(self.t_embedder.mlp[0].bias)
        P["t2_w"], P["t2_b"] = bf(self.t_embedder.mlp[2].weight), f32(self.t_embedder.mlp[2].bias)
        ada_w = [b.adaLN_modulation[1].weight for b in self.blocks]
        ada_b = [b.adaLN_modulation[1].bias for b in self.blocks]
        if getattr(self.final_layer, "adaLN_modulation", None) is not None:
            ada_w.append(self.final_layer.adaLN_modulation[1].weight)
            ada_b.append(self.final_layer.adaLN_modulation[1].bias)
        P["ada_w"] = bf(torch.cat([w.detach() for w in ada_w], 0))
        P["ada_b"] = f32(torch.cat([b.detach() for b in ada_b], 0))
        if self.clip_text_proj is not None:
            P["c1_w"], P["c1_b"] = bf(self.clip_text_proj.y_proj.fc1.weight), f32(self.clip_text_proj.y_proj.fc1.bias)
            P["c2_w"], P["c2_b"] = bf(self.clip_text_proj.y_proj.fc2.weight), f32(self.clip_text_proj.y_proj.fc2.bias)
        # K/V projections of the (step-invariant) context for all layers in one weight matrix
        P["kv_w"] = bf(torch.cat([torch.cat([b.cross_attn.to_k.weight.detach(),
                                              b.cross_attn.to_v.weight.detach()], 0)
                                  for b in self.blocks], 0))
        blocks = []
        for b in self.blocks:
            blocks.append(dict(
                qkv_w=bf(b.attn.qkv.weight), qkv_b=f32(b.attn.qkv.bias),
                proj_w=bf(b.attn.proj.weight), proj_b=f32(b.attn.proj.bias),
                q_w=bf(b.cross_attn.to_q.weight),
                o_w=bf(b.cross_attn.to_out[0].weight), o_b=f32(b.cross_attn.to_out[0].bias),
                fc1_w=bf(b.mlp.mlp[0].weight), fc1_b=f32(b.mlp.mlp[1].bias),
                fc2_w=bf(b.mlp.mlp[2].weight), fc2_b=f32(b.mlp.mlp[3].bias)))
        P["blocks"] = blocks
        P["pe_w"], P["pe_b"] = f32(self.x_embedder.proj.weight), f32(self.x_embedder.proj.bias)
        P["pos"] = f32(self.pos_embed)
        P["fin_w"], P["fin_b"] = f32(self.final_layer.linear.weight), f32(self.final_layer.linear.bias)
        self._invalidate()
        self._prep = P
        return P

    def _workspace(self, B):
        ws = self._ws.get(B)
        if ws is None:
            dev = self.pos_embed.device
            D, T = self.embed_dim, self.pos_embed.shape[1]
            M = B * T
            e = lambda *s, dt=torch.bfloat16: torch.empty(*s, device=dev, dtype=dt)
            ws = dict(tfeat=e(B, 256), th=e(B, D), st=e(B, D),
                      mod=e(B, self._prep["ada_w"].shape[0], dt=torch.float32),
                      x=e(B, T, D, dt=torch.float32), xb=e(M, D), a=e(M, D), v=e(M, D), qkv=e(M, 3 * D),
                      att=e(M, D), q=e(M, D), h=e(M, int(self.mlp_ratio) * D))
            self._ws[B] = ws
        return ws

    @torch.no_grad()
    def _context_kv(self, context):
        """clip_text_proj + every layer's to_k/to_v on the context.  The reference recomputes
        these every step (dit_trilatent.py:107, ldm/modules/attention.py:281-283) although the
        context is step-invariant; cached here keyed on the tensor identity/version.

        Also detects samples whose context tokens are all identical -- the zero-embedding unconditional
        half of classifier-free guidance (force_uc_zero_embeddings; every token becomes the same
        clip_text_proj(0) row).  For those, softmax(q k^T) is uniform whatever q is, so the cross-attention
        output of every query is `to_out(v_row)`: one (D,) row per layer and sample, computed here once.
        `rows` is the contiguous block of samples that still needs real attention (the identical-token
        samples must form a prefix and/or suffix of the batch, as both CFG layouts of the reference do)."""
        hit = self._ctx_cache.get(context)
        if hit is not None:
            return hit
        P = self._prep
        B, Lc, Cc = context.shape
        D = self.embed_dim
        # Static, model-owned output buffers per (B, Lc): captured graphs read K/V and the closed-form rows
        # through raw pointers, so a new prompt batch rewrites them in place and replays the same graph.
        st = self._ctx_static.get((B, Lc))
        if st is None:
            st = dict(kv=torch.empty(B * Lc, self.depth * 2 * D, device=context.device, dtype=torch.bfloat16),
                      oc=torch.empty(self.depth, B, D, device=context.device, dtype=torch.bfloat16))
            self._ctx_static[(B, Lc)] = st
        c = context.reshape(B * Lc, Cc).float().contiguous()
        cb = ops.norm_modulate(c, norm=NORM_NONE)
        c1 = ops.gemm(cb, P["c1_w"], P["c1_b"], act=ops.ACT_GELU_TANH)
        c2 = ops.gemm(c1, P["c2_w"], P["c2_b"])
        ops.gemm(c2, P["kv_w"], out=st["kv"])  # (B*Lc, depth*2*D)
        kv = st["kv"].view(B, Lc, self.depth, 2, D)
        out = dict(kv=kv, rows=(0, B), oconst=None)
        rows = _attention_rows(c2.view(B, Lc, -1))                        # one host sync per prompt batch
        if rows is not None:
            oc = st["oc"]
            for l, W in enumerate(P["blocks"]):
                ops.gemm(kv[:, 0, l, 1].contiguous(), W["o_w"], W["o_b"], out=oc[l])
            out = dict(kv=kv, rows=rows, oconst=oc)
        return self._ctx_cache.put((context,), out)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, x, timesteps=None, context=None, y=None, get_attr="", in_scale=None, **kwargs):
        """x (B, 3*C, S, S) fp32; timesteps (B,) int64 index / float; context (B, L, ctx_dim) or
        {'crossattn': ...} -> (B, 3*C_out, S, S) fp32 contiguous.  `in_scale` (B,) optionally
        folds the denoiser's c_in into the patch embed."""
        if get_attr != "":
            return getattr(self, get_attr)
        assert context is not None
        if isinstance(context, dict):
            context = context["crossattn"]
        if not x.is_cuda:
            raise RuntimeError("ln3diff_b200 DiT runs on CUDA only (no CPU fallback)")
        if self._prep is None:
            self.prepare()
        cx = self._context_kv(context)
        t = timesteps.to(device=x.device, dtype=torch.float32).contiguous()
        if graphs_enabled() and not torch.cuda.is_current_stream_capturing():
            # one graph launch instead of ~270 kernel launches; the result leaves the static buffer
            g = self._graph(x.shape[0], cx, shared_mod=False)
            g.x.copy_(x)
            g.t.copy_(t)
            if in_scale is None:
                g.in_scale.fill_(1.0)
            else:
                g.in_scale.copy_(in_scale)
            g.replay()
            return g.out.clone()
        return self._forward_impl(x.float().contiguous(), t, cx, in_scale)

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

    def _forward_impl(self, x, t, cx, in_scale, mod_row=None):
        """The fixed launch sequence of one forward (capturable in a CUDA graph: no host syncs, all
        intermediates in the per-batch workspace).  `mod_row` (1, (6L+2)·D): a row of modulation_table()
        shared by every sample of the batch (replaces the timestep embedder + adaLN GEMM)."""
        P = self._prep
        B = x.shape[0]
        D, H, T = self.embed_dim, self.num_heads, self.pos_embed.shape[1]
        M = B * T
        kv, (g0, g1), oconst = cx["kv"], cx["rows"], cx["oconst"]
        r0, r1 = g0 * T, g1 * T        # token rows that need real cross-attention
        ws = self._workspace(B)
        if mod_row is not None:
            mod = mod_row.expand(B, mod_row.shape[1])       # stride-0 rows: every sample reads the same row
        else:
            ops.timestep_embedding(t, out=ws["tfeat"])
            ops.gemm(ws["tfeat"], P["t0_w"], P["t0_b"], act=ops.ACT_SILU, out=ws["th"])
            ops.gemm(ws["th"], P["t2_w"], P["t2_b"], act=ops.ACT_SILU, out=ws["st"])  # silu(t_emb)
            mod = ops.gemm(ws["st"], P["ada_w"], P["ada_b"], out_kind=ops.OUT_F32, out=ws["mod"])

        xs = ops.patch_embed(x, P["pe_w"], P["pe_b"], P["pos"], in_scale=in_scale, out=ws["x"])
        x2 = xs.view(M, D)
        qkv3 = ws["qkv"].view(B, T, 3 * D)
        att3 = ws["att"].view(B, T, D)
        q3 = ws["q"].view(B, T, D)
        # Residual adds are deferred: every projection GEMM writes its bf16 output `val`; the next
        # norm kernel applies x += gate * val while it reads x anyway (one coalesced pass instead of a
        # thread-per-row read-modify-write in the GEMM epilogue).
        val, pend_gate = ws["v"], None
        for l, W in enumerate(P["blocks"]):
            m0 = l * 6 * D
            sl = lambda j: mod[:, m0 + j * D: m0 + (j + 1) * D]
            ops.norm_modulate(x2, norm=NORM_LAYER, shift=sl(0), scale=sl(1), mod_rows=T, out=ws["a"],
                              resid=val if l > 0 else None, resid_gate=pend_gate, resid_gate_rows=T)
            ops.gemm(ws["a"], W["qkv_w"], W["qkv_b"], out=ws["qkv"])
            ops.fmha(qkv3[:, :, 0:D], qkv3[:, :, D:2 * D], qkv3[:, :, 2 * D:3 * D], H, out=att3)
            ops.gemm(ws["att"], W["proj_w"], W["proj_b"], out=val)
            # x += gate_msa * attn ; xb = bf16(x): the un-normalised query input of the cross-attention.  Only the
            # attended rows need xb: with closed-form samples present the pass covers rows [r0, r1) only and the
            # next pass applies the other rows' gate_msa * attn together with their closed-form cross-attention row.
            split = oconst is not None and _split_residual_pass()
            if split:
                if r1 > r0:
                    ops.norm_modulate(x2[r0:r1], norm=NORM_NONE, out=ws["xb"][r0:r1], resid=val[r0:r1],
                                      resid_gate=sl(2)[g0:g1], resid_gate_rows=T)
            else:
                ops.norm_modulate(x2, norm=NORM_NONE, out=ws["xb"], resid=val, resid_gate=sl(2), resid_gate_rows=T)
            if r1 > r0:
                ops.gemm(ws["xb"][r0:r1], W["q_w"], out=ws["q"][r0:r1])
                ops.fmha(q3[g0:g1], kv[g0:g1, :, l, 0], kv[g0:g1, :, l, 1], H, out=att3[g0:g1])
                ops.gemm(ws["att"][r0:r1], W["o_w"], W["o_b"], out=val[r0:r1])
            # x += cross_attn (no gate) ; a = modulate(LN(x)).  Identical-token samples take the closed form.
            ops.norm_modulate(x2, norm=NORM_LAYER, shift=sl(3), scale=sl(4), mod_rows=T, out=ws["a"], resid=val,
                              resid_bcast=oconst[l] if oconst is not None else None, resid_bcast_rows=T,
                              resid_rows=(r0, r1) if oconst is not None else None,
                              resid_out_gate=sl(2) if split else None, resid_out_gate_rows=T)
            ops.gemm(ws["a"], W["fc1_w"], W["fc1_b"], act=ops.ACT_GELU_ERF, out=ws["h"])
            ops.gemm(ws["h"], W["fc2_w"], W["fc2_b"], out=val)
            pend_gate = sl(5)
        ops.norm_modulate(x2, norm=NORM_NONE, resid=val, resid_gate=pend_gate, resid_gate_rows=T, want_out=False)
        f0 = self.depth * 6 * D
        return ops.final_layer(xs, mod[:, f0:f0 + D], mod[:, f0 + D:f0 + 2 * D], P["fin_w"],
                               P["fin_b"], self.input_size)

    def _graph(self, B, cx, shared_mod: bool) -> ForwardGraph:
        """The captured forward for batch B and the launch sequence `cx` implies (context length,
        closed-form row split); captured on first use, then cached on the model."""
        key = (B, cx["kv"].shape[1], cx["rows"], cx["oconst"] is not None, bool(shared_mod))
        g = self._graphs.get(key)
        if g is None:
            dev = self.pos_embed.device
            g = ForwardGraph()
            g.key, g.cross_attention_rows = key, cx["rows"]
            g.x = torch.zeros(B, 3 * self.in_channels, self.input_size, self.input_size, device=dev)
            g.t = torch.zeros(B, device=dev)
            g.in_scale = torch.ones(B, device=dev)
            # shared_mod: the caller writes one modulation_table() row per step into g.mod (g.t is then unused)
            g.mod = torch.zeros(1, self._prep["ada_w"].shape[0], device=dev) if shared_mod else None
            capture_forward(g, lambda: self._forward_impl(g.x, g.t, cx, g.in_scale, g.mod), dev)
            self._graphs[key] = g
        return g

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
        if isinstance(context, dict):
            context = context["crossattn"]
        return self._graph(B, self._context_kv(context), shared_mod)

    @torch.no_grad()
    def forward_with_cfg(self, x, t, context, cfg_scale):
        """reference dit_trilatent.py:249-262 (cond first, uncond second; returns cat([half, half]))."""
        eps = self.forward(x, t, context)
        cond_eps, uncond_eps = torch.split(eps, len(eps) // 2, dim=0)
        half = uncond_eps + cfg_scale * (cond_eps - uncond_eps)
        return torch.cat([half, half], dim=0)


class DiT_TriLatent_PixelArt(PixArtGraphMixin, nn.Module):
    """reference dit/dit_trilatent.py:146-246: the PixArt-style T23D denoiser -- one shared adaLN
    (`adaLN_modulation` on t_emb + cap_embedder(pooled CLIP)) plus per-block `scale_shift_table`,
    `PixelArtTextCondDiTBlock` blocks, `T2IFinalLayer`.  context = {'vector': (B, context_dim) pooled
    CLIP, 'crossattn': (B, 77, context_dim) CLIP tokens}.

    Step-invariant work is cached per prompt batch: the pooled-CLIP embedding and every block's
    cross-attention K/V (each block RMS-normalises the tokens with its own `attention_y_norm` first; the
    reference redoes both in every block of every step, dit_models_xformers.py:364)."""

    _ln3_fused_in_scale = False

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
        P = dict(t0_w=bf(self.t_embedder.mlp[0].weight), t0_b=f32(self.t_embedder.mlp[0].bias),
                 t2_w=bf(self.t_embedder.mlp[2].weight), t2_b=f32(self.t_embedder.mlp[2].bias),
                 ada_w=bf(self.adaLN_modulation[1].weight), ada_b=f32(self.adaLN_modulation[1].bias),
                 cap_ln_w=f32(self.cap_embedder[0].weight), cap_ln_b=f32(self.cap_embedder[0].bias),
                 cap_w=bf(self.cap_embedder[1].weight), cap_b=f32(self.cap_embedder[1].bias),
                 pe_w=f32(self.x_embedder.proj.weight), pe_b=f32(self.x_embedder.proj.bias), pos=f32(self.pos_embed),
                 fin_w=f32(self.final_layer.linear.weight), fin_b=f32(self.final_layer.linear.bias),
                 fin_tab=f32(self.final_layer.scale_shift_table),
                 tables=f32(torch.stack([b.scale_shift_table.detach().reshape(-1) for b in self.blocks], 0)))
        P["blocks"] = [dict(
            n1_w=f32(b.norm1.weight), n2_w=f32(b.norm2.weight), yn_w=f32(b.attention_y_norm.weight),
            qkv_w=bf(b.attn.qkv.weight), qkv_b=f32(b.attn.qkv.bias),
            proj_w=bf(b.attn.proj.weight), proj_b=f32(b.attn.proj.bias),
            cq_w=bf(b.cross_attn.to_q.weight),
            ckv_w=bf(torch.cat([b.cross_attn.to_k.weight.detach(), b.cross_attn.to_v.weight.detach()], 0)),
            co_w=bf(b.cross_attn.to_out[0].weight), co_b=f32(b.cross_attn.to_out[0].bias),
            fc1_w=bf(b.mlp.mlp[0].weight), fc1_b=f32(b.mlp.mlp[1].bias),
            fc2_w=bf(b.mlp.mlp[2].weight), fc2_b=f32(b.mlp.mlp[3].bias)) for b in self.blocks]
        self._invalidate()
        self._prep = P
        return P

    @torch.no_grad()
    def _context(self, context):
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
        out = dict(cls=cls, ckv=ckv, rows=(0, B), oconst=None)
        # identical text tokens (the zero-embedding CFG half): closed-form cross-attention, see DiT_TriLatent
        rows = _attention_rows(ca.float())
        if rows is not None:
            oc = st["oc"]
            for l, W in enumerate(P["blocks"]):
                ops.gemm(ckv[l][:, 0, D:].contiguous(), W["co_w"], W["co_b"], out=oc[l])
            out.update(rows=rows, oconst=oc)
        return self._ctx_cache.put((vec0, ca0), out)

    @torch.no_grad()
    def forward(self, x, timesteps=None, context=None, y=None, get_attr="", **kwargs):
        if get_attr != "":
            return getattr(self, get_attr)
        assert context is not None and isinstance(context, dict), "PixelArt T23D needs {'vector','crossattn'}"
        if not x.is_cuda:
            raise RuntimeError("ln3diff_b200 DiT runs on CUDA only (no CPU fallback)")
        if self._prep is None:
            self.prepare()
        t = timesteps.to(device=x.device, dtype=torch.float32).contiguous()
        return self._run(x, t, self._context(context))

    @torch.no_grad()
    def forward_with_cfg(self, x, t, context, cfg_scale):
        """reference dit_trilatent.py:249-262 (cond first, uncond second; returns cat([half, half]))."""
        eps = self.forward(x, t, context)
        cond_eps, uncond_eps = torch.split(eps, len(eps) // 2, dim=0)
        half = uncond_eps + cfg_scale * (cond_eps - uncond_eps)
        return torch.cat([half, half], dim=0)


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
