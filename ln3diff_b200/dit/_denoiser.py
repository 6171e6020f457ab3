"""What the DiT denoisers share: the launch sequence of their blocks, the closed-form cross-attention of
identical-token samples, weight init and repack, and the derived state around a forward (repacked weights,
workspaces, the conditioning cache and the CUDA graphs).  The families are `DiT_TriLatent` (T23D, LayerNorm
blocks with per-block adaLN) and the PixArt-style `DiT_TriLatent_PixelArt` (dit/dit_trilatent.py),
`DiT_I23D_PixelArt` and `DiT_I23D_PixelArt_MVCond_noClip` (dit/dit_i23d.py).

Their blocks differ only in data, carried by the prepared block weights and the cached conditioning: RMSNorm
pre-norm weights (`n1_w` / `n2_w`; LayerNorm without them), q/k head-norm weights (`qk_norm` / `cq_norm`), a
second self-attention K/V source (`dkv`, I23D) and where each layer's cross-attention K/V live.  Each family
keeps its own prologue (timestep embedding -> per-layer modulation rows) and final layer."""
from __future__ import annotations

import os

import torch
import torch.nn as nn

from .. import ops
from .._lib import NORM_LAYER, NORM_NONE, NORM_RMS
from ._graph import ContextCache, ForwardGraph, capture_forward, graphs_enabled
from .dit_models_xformers import get_2d_sincos_pos_embed


def _attention_rows(tokens: torch.Tensor):
    """tokens (B, L, C) as the cross-attention sees them.  Returns (g0, g1): the contiguous block of samples
    that needs real attention when the samples whose L tokens are all identical form a prefix and/or suffix
    of the batch (both CFG layouts of the reference), else None.  One host sync; callers cache per context.
    LN3_UNCOND_CLOSED_FORM=0 forces full cross-attention for identical-token samples (A/B, tests)."""
    B, L, _ = tokens.shape
    if os.environ.get("LN3_UNCOND_CLOSED_FORM", "1") == "0" or L < 2:
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


def split_kv(buf: torch.Tensor) -> list:
    """(depth, B, L, 2D) per-layer K|V buffer -> [(k, v)] per layer, (B, L, D) views."""
    D = buf.shape[-1] // 2
    return [(b[:, :, :D], b[:, :, D:]) for b in buf]


def cross_attention_context(kv: list, tokens: torch.Tensor, blocks: list, oc: torch.Tensor, **extra) -> dict:
    """The cached conditioning a forward reads: every layer's cross-attention (k, v) views `kv`, `extra`, and the
    closed form of samples whose context tokens are all identical -- the zero-embedding unconditional half of
    classifier-free guidance (force_uc_zero_embeddings).  For those samples softmax(q k^T) is uniform whatever q
    is, so the cross-attention output of every query is to_out(v_row): one (D,) row per layer and sample,
    computed here into the model-owned `oc` (depth, B, D).  'rows' is the contiguous block of samples that still
    needs real attention, 'oconst' is `oc` or None when no sample takes the closed form."""
    cx = dict(extra, kv=kv, rows=(0, tokens.shape[0]), oconst=None)
    rows = _attention_rows(tokens)                                      # one host sync per prompt batch
    if rows is not None:
        for l, ((_, v), W) in enumerate(zip(kv, blocks)):
            ops.gemm(v[:, 0].contiguous(), W["co_w"], W["co_b"], out=oc[l])
        cx.update(rows=rows, oconst=oc)
    return cx


def _pre_norm(W: dict, key: str) -> dict:
    """RMSNorm with the block's weight when it has one (PixArt blocks), else LayerNorm without affine."""
    w = W.get(key)
    return dict(norm=NORM_LAYER) if w is None else dict(norm=NORM_RMS, weight=w, eps=1e-5)


def run_blocks(blocks: list, cx: dict, ws: dict, x2: torch.Tensor, mods, heads: int, T: int) -> None:
    """Every block of one forward as a fixed launch sequence over the workspace `ws` (no host syncs, so it
    can be captured in a CUDA graph).  x2 (B·T, D) fp32 residual stream, updated in place; mods[l] (B, 6D) fp32:
    layer l's shift / scale / gate rows of the attention (0-2) and of the MLP (3-5).  cx: 'kv' [(k, v)] per layer,
    (B, Lc, E) views; 'rows' / 'oconst' from `cross_attention_context`; optional 'dkv' [(k, v)] per layer, a
    second self-attention K/V source.  E, the cross-attention's inner width (heads x its head width), is D except
    in DiT-XL/2, whose cross-attention keeps 64-wide heads (E = 1024) beside 72-wide self-attention heads; its
    output then takes the first M·E elements of ws['att']."""
    M, D = x2.shape
    B = M // T
    E = blocks[0]["cq_w"].shape[0]
    qkv3, att3, q3 = ws["qkv"].view(B, T, 3 * D), ws["att"].view(B, T, D), ws["q"].view(B, T, E)
    attc = ws["att"].view(-1)[:M * E].view(M, E)
    attc3 = attc.view(B, T, E)
    (g0, g1), oconst = cx["rows"], cx["oconst"]
    r0, r1 = g0 * T, g1 * T        # token rows that need real cross-attention
    # x += gate_msa * attn ; xb = bf16(x): the un-normalised query input of the cross-attention.  Only the
    # attended rows need xb: with closed-form samples present the pass covers rows [r0, r1) only and the
    # next pass applies the other rows' gate_msa * attn together with their closed-form cross-attention row.
    # LN3_SPLIT_RESID_PASS=0: the pass covers every row (A/B, tests).
    split = oconst is not None and os.environ.get("LN3_SPLIT_RESID_PASS", "1") != "0"
    dkv = cx.get("dkv", [(None, None)] * len(blocks))
    # Residual adds are deferred: every projection GEMM writes its bf16 output `val`; the next
    # norm kernel applies x += gate * val while it reads x anyway (one coalesced pass instead of a
    # thread-per-row read-modify-write in the GEMM epilogue).
    val, pend_gate = ws["v"], None
    # fp8 precision (set_gemm_precision): qkv / fc1 / fc2 read e4m3 operands with block scales, written by the norm
    # passes that precede qkv and fc1 and by fc1's epilogue; every other launch is the same as in bf16
    fp8 = "a8" in ws
    if fp8:
        a8 = dict(out=ws["a8"], out_scale=ws["a8s"])
        norm_a = lambda **kw: ops.norm_modulate_fp8(x2, **a8, **kw)
    else:
        norm_a = lambda **kw: ops.norm_modulate(x2, out=ws["a"], **kw)
    for l, (W, mod, (k, v), (k2, v2)) in enumerate(zip(blocks, mods, cx["kv"], dkv)):
        sl = lambda j: mod[:, j * D:(j + 1) * D]
        norm_a(**_pre_norm(W, "n1_w"), shift=sl(0), scale=sl(1), mod_rows=T,
               resid=val if l > 0 else None, resid_gate=pend_gate, resid_gate_rows=T)
        if fp8:
            ops.gemm_fp8(ws["a8"], ws["a8s"], W["qkv_q"], W["qkv_s"], W["qkv_b"], out=ws["qkv"],
                         head_norm=W.get("qk_norm"), head_norm_sec_cols=D)
        else:
            ops.gemm(ws["a"], W["qkv_w"], W["qkv_b"], out=ws["qkv"], head_norm=W.get("qk_norm"), head_norm_sec_cols=D)
        ops.fmha(qkv3[:, :, :D], qkv3[:, :, D:2 * D], qkv3[:, :, 2 * D:], heads, out=att3, k2=k2, v2=v2)
        ops.gemm(ws["att"], W["proj_w"], W["proj_b"], out=val)
        if split:
            if r1 > r0:
                ops.norm_modulate(x2[r0:r1], norm=NORM_NONE, out=ws["xb"][r0:r1], resid=val[r0:r1],
                                  resid_gate=sl(2)[g0:g1], resid_gate_rows=T)
        else:
            ops.norm_modulate(x2, norm=NORM_NONE, out=ws["xb"], resid=val, resid_gate=sl(2), resid_gate_rows=T)
        if r1 > r0:
            ops.gemm(ws["xb"][r0:r1], W["cq_w"], out=ws["q"][r0:r1], head_norm=W.get("cq_norm"), head_norm_sec_cols=D)
            ops.fmha(q3[g0:g1], k[g0:g1], v[g0:g1], heads, out=attc3[g0:g1])
            ops.gemm(attc[r0:r1], W["co_w"], W["co_b"], out=val[r0:r1])
        # x += cross_attn (no gate) ; a = modulate(norm(x)).  Identical-token samples take the closed form.
        norm_a(**_pre_norm(W, "n2_w"), shift=sl(3), scale=sl(4), mod_rows=T, resid=val,
               resid_bcast=oconst[l] if oconst is not None else None, resid_bcast_rows=T,
               resid_rows=(r0, r1) if oconst is not None else None,
               resid_out_gate=sl(2) if split else None, resid_out_gate_rows=T)
        if fp8:
            ops.gemm_fp8(ws["a8"], ws["a8s"], W["fc1_q"], W["fc1_s"], W["fc1_b"], act=ops.ACT_GELU_ERF,
                         out_kind=ops.OUT_FP8, out=ws["h8"], out_scale=ws["h8s"])
            ops.gemm_fp8(ws["h8"], ws["h8s"], W["fc2_q"], W["fc2_s"], W["fc2_b"], out=val)
        else:
            ops.gemm(ws["a"], W["fc1_w"], W["fc1_b"], act=ops.ACT_GELU_ERF, out=ws["h"])
            ops.gemm(ws["h"], W["fc2_w"], W["fc2_b"], out=val)
        pend_gate = sl(5)
    ops.norm_modulate(x2, norm=NORM_NONE, resid=val, resid_gate=pend_gate, resid_gate_rows=T, want_out=False)


def _bf16(dev):
    return lambda w: w.detach().to(dev, torch.bfloat16).contiguous()


def _fp32(dev):
    return lambda w: w.detach().to(dev, torch.float32).contiguous()


class DenoiserMixin:
    """Derived state of a DiT denoiser: the repacked weights (`_prep`), per-batch workspaces, the step-invariant
    conditioning cache with its model-owned static buffers, and the CUDA graphs of a forward (see dit/_graph.py).
    A family provides `_pack` (its model-level weights), optionally `_pack_block`, `_context` (the cached
    conditioning of a context), `_mod_workspace` (its modulation buffers) and `_forward_impl`."""

    _ln3_fused_in_scale = False  # forward(..., in_scale=) folds the denoiser's c_in into the patch embed
    _gemm_precision = "bf16"     # "fp8": see set_gemm_precision

    def set_gemm_precision(self, precision: str):
        """Operand precision of every block's qkv / fc1 / fc2 GEMMs: "bf16" (the default, held to the reference's
        parity tolerance) or "fp8" (e4m3 operands with 1x128 activation block scales and per-channel weight scales
        on the fp8 tensor cores, format in include/ln3b200.h -- faster, and OUTSIDE the parity tolerance).  The
        parameters and state_dict are untouched; the derived state (repacks, workspaces, conditioning cache, CUDA
        graphs) is dropped and rebuilt for the new precision on the next forward.  Returns self."""
        if precision not in ("bf16", "fp8"):
            raise ValueError(f"gemm precision must be 'bf16' or 'fp8', got {precision!r}")
        if precision != self.gemm_precision:
            self._gemm_precision = precision
            self._invalidate()
        return self

    @property
    def gemm_precision(self) -> str:
        return self._gemm_precision

    def initialize_weights(self, zeroed=()):
        """reference dit_models_xformers.py:786-819: xavier-uniform Linears with zero bias, the patch embed as a
        Linear, N(0, 0.02) timestep MLP -- in this order, which seeded builds' weights depend on -- then the
        family's zero-initialised Linears `zeroed` and the 3-plane sin-cos position table."""
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
        for m in (self.final_layer.linear, *zeroed):
            nn.init.constant_(m.weight, 0)
            nn.init.constant_(m.bias, 0)
        self.init_PE_3D_aware()

    def init_PE_3D_aware(self):
        p = int(self.x_embedder.num_patches ** 0.5)
        D = self.pos_embed.shape[-1]
        pe = get_2d_sincos_pos_embed(D, (self.plane_n, p * p)).reshape(self.plane_n * p * p, D)
        self.pos_embed.data.copy_(torch.from_numpy(pe).float().unsqueeze(0))

    def _invalidate(self):
        """Drop everything derived from the parameters: repacks, workspaces, the cached conditioning
        and its static buffers, and the captured graphs (they hold raw pointers into all of those)."""
        self._prep = None
        self._ws = {}
        self._ctx_cache = ContextCache()
        self._ctx_static = {}
        self._graphs = {}

    def _apply(self, fn, *a, **kw):
        self._invalidate()
        return super()._apply(fn, *a, **kw)

    def load_state_dict(self, *a, **kw):
        self._invalidate()
        return super().load_state_dict(*a, **kw)

    @torch.no_grad()
    def prepare(self):
        """One-time repack of the weights onto the model's device: bf16 GEMM operands, fp32 for the rest.
        Owned by the module, rebuilt after load_state_dict / .to()."""
        dev = self.pos_embed.device
        if dev.type != "cuda":
            raise RuntimeError("ln3diff_b200 DiT runs on CUDA only (no CPU fallback)")
        bf, f32 = _bf16(dev), _fp32(dev)
        P = dict(t0_w=bf(self.t_embedder.mlp[0].weight), t0_b=f32(self.t_embedder.mlp[0].bias),
                 t2_w=bf(self.t_embedder.mlp[2].weight), t2_b=f32(self.t_embedder.mlp[2].bias),
                 pe_w=f32(self.x_embedder.proj.weight), pe_b=f32(self.x_embedder.proj.bias), pos=f32(self.pos_embed),
                 fin_w=f32(self.final_layer.linear.weight), fin_b=f32(self.final_layer.linear.bias),
                 **self._pack(bf, f32))
        P["blocks"] = [dict(
            qkv_w=bf(b.attn.qkv.weight), qkv_b=f32(b.attn.qkv.bias),
            proj_w=bf(b.attn.proj.weight), proj_b=f32(b.attn.proj.bias),
            cq_w=bf(b.cross_attn.to_q.weight),
            co_w=bf(b.cross_attn.to_out[0].weight), co_b=f32(b.cross_attn.to_out[0].bias),
            fc1_w=bf(b.mlp.mlp[0].weight), fc1_b=f32(b.mlp.mlp[1].bias),
            fc2_w=bf(b.mlp.mlp[2].weight), fc2_b=f32(b.mlp.mlp[3].bias),
            **self._pack_block(b, bf, f32)) for b in self.blocks]
        if self.gemm_precision == "fp8":
            self._check_fp8_shapes()
            for W, b in zip(P["blocks"], self.blocks):
                for key, lin in (("qkv", b.attn.qkv), ("fc1", b.mlp.mlp[0]), ("fc2", b.mlp.mlp[2])):
                    W[key + "_q"], W[key + "_s"] = ops.quantize_weight_fp8(lin.weight.to(dev))
        self._invalidate()
        self._prep = P
        return P

    def _pack_block(self, b, bf, f32) -> dict:
        return {}

    def _check_fp8_shapes(self):
        """The fp8 kernels' shape rules (include/ln3b200.h), checked once so that an unsupported model fails in
        prepare() with the reason rather than in the middle of a forward."""
        D = self.embed_dim
        H = int(self.mlp_ratio) * D
        if D % 256 != 0 or D > 1536 or H % 128 != 0:
            raise RuntimeError(f"fp8 GEMM precision needs embed_dim % 256 == 0, embed_dim <= 1536 and an MLP width "
                               f"% 128 == 0 (embed_dim {D}, MLP width {H}); use set_gemm_precision('bf16')")

    def _static(self, key, make):
        st = self._ctx_static.get(key)
        if st is None:
            st = self._ctx_static[key] = make()
        return st

    def _workspace(self, B):
        ws = self._ws.get(B)
        if ws is None:
            dev = self.pos_embed.device
            D, T = self.embed_dim, self.pos_embed.shape[1]
            M = B * T
            e = lambda *s, dt=torch.bfloat16: torch.empty(*s, device=dev, dtype=dt)
            ws = self._ws[B] = dict(tfeat=e(B, 256), th=e(B, D), st=e(B, D), x=e(B, T, D, dt=torch.float32),
                                    xb=e(M, D), a=e(M, D), v=e(M, D), qkv=e(M, 3 * D), att=e(M, D),
                                    q=e(M, self.blocks[0].cross_attn.to_q.out_features),
                                    h=e(M, int(self.mlp_ratio) * D), **self._mod_workspace(B, e))
            if self.gemm_precision == "fp8":
                H = int(self.mlp_ratio) * D
                ws.update(a8=e(M, D, dt=ops.FP8), a8s=e(M, D // 128, dt=torch.float32),
                          h8=e(M, H, dt=ops.FP8), h8s=e(M, H // 128, dt=torch.float32))
        return ws

    def _graph(self, B, cx, shared_mod: bool = False) -> ForwardGraph:
        """The captured forward for batch B and the launch sequence `cx` implies (context length, closed-form
        row split, shared modulation row); captured on first use, then cached on the model."""
        key = (B, cx["kv"][0][0].shape[1], cx["rows"], cx["oconst"] is not None, bool(shared_mod))
        g = self._graphs.get(key)
        if g is None:
            dev = self.pos_embed.device
            g = ForwardGraph()
            g.key, g.cross_attention_rows = key, cx["rows"]
            g.x = torch.zeros(B, 3 * self.in_channels, self.input_size, self.input_size, device=dev)
            g.t = torch.zeros(B, device=dev)
            if self._ln3_fused_in_scale:
                g.in_scale = torch.ones(B, device=dev)
            # shared_mod: the caller writes one modulation_table() row per step into g.mod (g.t is then unused)
            if shared_mod:
                g.mod = torch.zeros(1, self._prep["ada_w"].shape[0], device=dev)
            self._workspace(B)   # allocated on the caller's stream, not in the side-stream warm-up of the capture
            capture_forward(g, lambda: self._forward_impl(g.x, g.t, cx, g.in_scale, g.mod), dev)
            self._graphs[key] = g
        return g

    def _run(self, x, t, cx, in_scale=None):
        """One forward: a replay of the cached CUDA graph (captured on first use; the result leaves the static
        buffer), or the eager launch sequence under LN3_CUDA_GRAPH=0 / inside a caller's own capture."""
        if graphs_enabled() and not torch.cuda.is_current_stream_capturing():
            g = self._graph(x.shape[0], cx)
            g.load(x, t, 1.0 if in_scale is None else in_scale)
            g.replay()
            return g.out.clone()
        return self._forward_impl(x.float().contiguous(), t, cx, in_scale, None)

    def step_forward(self, rows: int, context, t: torch.Tensor, in_scale=None) -> StepForward:
        """The forwards of a sampling loop over a fixed `rows`-sample batch conditioned on `context`: write the batch
        into `.x` (rows, 3C, S, S) fp32, then `(k)` runs step k's forward and returns the output buffer, which the
        next call overwrites.  t (steps, rows) fp32: every step's timesteps; in_scale (steps, rows) or None (1.0):
        every step's c_in, for the families that set `_ln3_fused_in_scale`.

        Each step is a replay of the cached CUDA graph (`_graph`), or the eager launch sequence on `.x` under
        LN3_CUDA_GRAPH=0 / inside a caller's own capture.  A graph replay of a family with `modulation_table` reads
        one shared adaLN row per step, all steps' rows computed from t[:, 0] in one pass (every sample of a step
        shares its timestep), unless LN3_SHARED_MODULATION=0."""
        return StepForward(self, rows, context, t, in_scale)

    @torch.no_grad()
    def forward(self, x, timesteps=None, context=None, y=None, get_attr="", in_scale=None, **kwargs):
        """x (B, 3*C, S, S) fp32; timesteps (B,) int64 index / float; context as the family's `_context` takes it
        -> (B, 3*C_out, S, S) fp32 contiguous.  `in_scale` (B,) folds the denoiser's c_in into the patch embed
        in the families that set `_ln3_fused_in_scale`; the others ignore it."""
        if get_attr != "":
            return getattr(self, get_attr)
        if not x.is_cuda:
            raise RuntimeError("ln3diff_b200 DiT runs on CUDA only (no CPU fallback)")
        if self._prep is None:
            self.prepare()
        cx = self._context(context)
        t = timesteps.to(device=x.device, dtype=torch.float32).contiguous()
        return self._run(x, t, cx, in_scale)

    @torch.no_grad()
    def forward_with_cfg(self, x, t, context, cfg_scale):
        """reference dit_trilatent.py:249-262, dit_i23d.py:155-168 (cond first, uncond second; returns
        cat([half, half]))."""
        eps = self.forward(x, t, context)
        cond_eps, uncond_eps = torch.split(eps, len(eps) // 2, dim=0)
        half = uncond_eps + cfg_scale * (cond_eps - uncond_eps)
        return torch.cat([half, half], dim=0)


class StepForward:
    """See DenoiserMixin.step_forward."""

    def __init__(self, den, rows, context, t, in_scale):
        if den._prep is None:
            den.prepare()
        self.den, self.cx, self.t, self.in_scale = den, den._context(context), t, in_scale
        self.g = self.mod = None
        if graphs_enabled() and not torch.cuda.is_current_stream_capturing():
            shared = hasattr(den, "modulation_table") and os.environ.get("LN3_SHARED_MODULATION", "1") != "0"
            self.g = den._graph(rows, self.cx, shared)
            if shared:
                self.mod = den.modulation_table(t[:, 0])
            if in_scale is None:
                self.g.load(in_scale=1.0)
            self.x = self.g.x
        else:
            self.x = torch.empty(rows, 3 * den.in_channels, den.input_size, den.input_size,
                                 device=den.pos_embed.device, dtype=torch.float32)

    def __call__(self, k: int) -> torch.Tensor:
        in_scale = None if self.in_scale is None else self.in_scale[k]
        if self.g is None:
            return self.den._forward_impl(self.x, self.t[k], self.cx, in_scale, None)
        if self.mod is not None:
            self.g.load(mod=self.mod[k:k + 1], in_scale=in_scale)
        else:
            self.g.load(t=self.t[k], in_scale=in_scale)
        self.g.replay()
        return self.g.out


class PixArtMixin(DenoiserMixin):
    """The PixArt-style denoisers' prologue and final layer: one shared adaLN on t = t_emb + pooled embedding
    (cx['cls']) plus each block's scale_shift_table, and the T2IFinalLayer.  A family provides `_pack_context`,
    its conditioning weights."""

    def _pack(self, bf, f32) -> dict:
        return dict(ada_w=bf(self.adaLN_modulation[1].weight), ada_b=f32(self.adaLN_modulation[1].bias),
                    fin_tab=f32(self.final_layer.scale_shift_table),
                    tables=f32(torch.stack([b.scale_shift_table.detach().reshape(-1) for b in self.blocks], 0)),
                    **self._pack_context(bf, f32))

    def _mod_workspace(self, B, e) -> dict:
        D = self.embed_dim
        return dict(t=e(B, D, dt=torch.float32), t0=e(B, 6 * D, dt=torch.float32),
                    mod=e(self.depth, B, 6 * D, dt=torch.float32))

    def _forward_impl(self, x, t, cx, in_scale=None, mod_row=None):
        """x (B, 3C, S, S) fp32, t (B,) fp32; cx from `_context`.  `in_scale` and `mod_row` are DiT_TriLatent's
        inputs and unused here."""
        P, B = self._prep, x.shape[0]
        D, T = self.embed_dim, self.pos_embed.shape[1]
        ws = self._workspace(B)
        ops.timestep_embedding(t, out=ws["tfeat"])
        ops.gemm(ws["tfeat"], P["t0_w"], P["t0_b"], act=ops.ACT_SILU, out=ws["th"])
        ws["t"].copy_(cx["cls"])                                                       # t = t_emb + pooled embedding
        ops.gemm(ws["th"], P["t2_w"], P["t2_b"], out_kind=ops.OUT_RESID_F32, out=ws["t"])
        ops.norm_modulate(ws["t"], norm=NORM_NONE, act=ops.ACT_SILU, out=ws["st"])
        ops.gemm(ws["st"], P["ada_w"], P["ada_b"], out_kind=ops.OUT_F32, out=ws["t0"])  # shared adaLN (B, 6D)
        torch.add(P["tables"][:, None, :], ws["t0"][None], out=ws["mod"])              # + per-block tables
        xs = ops.patch_embed(x, P["pe_w"], P["pe_b"], P["pos"], out=ws["x"])
        run_blocks(P["blocks"], cx, ws, xs.view(B * T, D), ws["mod"], self.num_heads, T)
        # T2IFinalLayer: shift = table[0] + t, scale = table[1] + t
        return ops.final_layer(xs, ws["t"], ws["t"], P["fin_w"], P["fin_b"], self.input_size,
                               shift_tab=P["fin_tab"][0].contiguous(), scale_tab=P["fin_tab"][1].contiguous())
