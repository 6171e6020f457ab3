"""GPU (-m gpu): every kernel launch of a DiT denoiser forward, element by element against float64.

The per-kernel tests check the arithmetic of each kernel; this file checks how the denoisers call them: the views,
offsets, chunks, layers, sub-batches and buffers of `run_blocks` (dit/_denoiser.py) and of each family's context,
prologue and final layer.  A tracer wraps the ops the denoisers call (ops.gemm, gemm_fp8, fmha, norm_modulate,
norm_modulate_fp8, timestep_embedding, patch_embed, final_layer) and hands every launch of an eager forward to an
auditor that

  * matches it against the written-down launch sequence of the family and configuration (`expected_launches`):
    the op of every launch and their count;
  * recomputes what the launch should have written in float64 from two inputs only: the nn.Module's own parameters
    (bf16 GEMM weights, fp32 otherwise; for fp8 the per-channel e4m3 codes restated from quantize_weight_fp8's rule)
    and the recorded outputs of the semantically preceding launches, chosen by the model's definition (layer l's
    gate_msa is chunk 2 of layer l's modulation, the cross-attention K/V of layer l and sample b come from sample b's
    context).  The launch's own arguments are never used for the reference, so a wrong view is an O(1) mismatch,
    while errors never compound: each check carries exactly one kernel's bound (kernel_bounds.py);
  * for every check kind, recomputes the reference once with a mapping deliberately slipped (the neighbouring
    layer's weights or K/V, mod chunk j +- 1, the other CFG half, q_norm and k_norm swapped, the row range shifted by
    one sample, ...) and asserts the slip moves the affected elements by >= 100x the bound (the median; the fp8 and
    attention kinds by FP8_FACTOR / FMHA_FACTOR, where the derived bound is itself a sizeable share of |y|);
  * asserts that every traced launch was checked.

The closed-form rows of identical-token samples are checked against real float64 softmax attention over their
context tokens, element-wise.  Stale rows of the workspace (att / q / xb outside the attended rows) are not
compared; instead every consumer's view is asserted to cover exactly the attended rows.  Seeded slips injected
through the tracer (a view argument shifted within its storage) must make the audit fail, naming the step, the
layer and the worst element.  Finally the CUDA-graph replay of the same forward must be bit-identical to the
audited eager forward."""
from __future__ import annotations

import pytest
import torch

import kernel_bounds as kb
import mv23d_oracle as mo
from launch_audit import FMHA_FACTOR, Step, _report, traced
from launch_audit import Audit as LaunchAudit

pytestmark = pytest.mark.gpu

TRACED = ("gemm", "gemm_fp8", "fmha", "norm_modulate", "norm_modulate_fp8", "timestep_embedding", "patch_embed",
          "final_layer")
B = 4                 # batch of every audited forward
SEP_L = 1             # the layer whose checks also run the separation (slipped-mapping) assertions
NORM_NONE, NORM_LAYER, NORM_RMS = 0, 1, 2
ACT_GELU_ERF, ACT_GELU_TANH, ACT_SILU = 1, 2, 3
# The fp8 bounds are relative to the operands, not to the result: the GEMM's assumed in-block accumulation
# (kernel_bounds.fp8_acc_bound) is 2^-6 sum|a w|, about 0.3 |y| at K = 768, and an e4m3 output is good to 2^-4
# relative.  A slip of an fp8 check kind therefore cannot move its elements by 100x the bound; it must still put the
# median affected element outside it (the check then fails on most of them), with margin.
FP8_FACTOR = 2.0


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


# ------------------------------------------------------------------ models (seeded, non-zero adaLN and gates)
def _seeded(m, sd_fn):
    """The seeded weights, with the head-norm weights spread to 1 + N(0, 2^2) (the fixtures draw 1 + N(0, 0.02^2)):
    q_norm and k_norm must differ by more than the bound for their exchange to be visible."""
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = sd_fn(shapes, m.state_dict()["pos_embed"])
    for k in sd:
        if k.endswith(("q_norm.weight", "k_norm.weight")):
            sd[k] = 1 + 100 * (sd[k] - 1)
    m.load_state_dict(sd)
    return m


def _build(family):
    from oracle import dit as odit
    from oracle import fixtures as fx
    from ln3diff_b200.utils import build_i23d, build_mv23d, build_t23d
    if family == "t23d":
        return _seeded(build_t23d("DiT-B/2"), lambda s, pe: odit.synth_state_dict(s, seed=7, keep={"pos_embed": pe}))
    if family == "t23d_pixart":
        from ln3diff_b200.dit.dit_trilatent import DiT_models
        m = DiT_models["DiT-PixelArt-B/2"](input_size=32, num_classes=0, learn_sigma=False, in_channels=4,
                                          context_dim=768, roll_out=True)
        return _seeded(m.eval(), fx.i23d_state_dict)
    if family == "i23d":
        return _seeded(build_i23d("DiT-PixArt-B/2"), fx.i23d_state_dict)
    return _seeded(build_mv23d(depth=mo.MV_DEPTH, hidden_size=mo.MV_HIDDEN, num_heads=mo.MV_HEADS), mo.mv_state_dict)


_MODELS = {}


def model(family, dev):
    if family not in _MODELS:
        _MODELS[family] = _build(family).to(dev)
    return _MODELS[family]


LAYOUTS = {"cond-zero": (0, 2), "zero-cond": (2, 4), "distinct": None}   # uncond (zero-token) samples -> rows


def inputs(family, layout, dev, seed=5):
    """x, t, context, in_scale for batch B; the zero-token samples are the unconditional half of CFG."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 12, 32, 32, generator=g)
    zero = {"cond-zero": [2, 3], "zero-cond": [0, 1], "distinct": []}[layout]
    if family == "t23d":
        t = torch.tensor([12.0, 250.0, 603.0, 871.0])
        c = torch.randn(B, 77, 768, generator=g)
        c[zero] = 0
        ctx = c
    elif family == "mv23d":
        t = torch.tensor([0.1, 0.35, 0.6, 0.9])
        c = torch.randn(B, mo.MV_VIEWS, 256, mo.MV_CONTEXT, generator=g)
        c[zero] = 0
        ctx = {"concat": c}
    else:
        t = torch.tensor([12.0, 250.0, 603.0, 871.0]) if family == "t23d_pixart" else torch.tensor([0.1, 0.35, 0.6, 0.9])
        L, C = (77, 768) if family == "t23d_pixart" else (256, 2048)
        v, c = torch.randn(B, 768, generator=g), torch.randn(B, L, C, generator=g)
        v[zero], c[zero] = 0, 0
        ctx = {"vector": v, "crossattn": c}
    in_scale = torch.tensor([0.71, 1.3, 0.05, 2.2]) if family == "t23d" else None
    to = lambda a: a.to(dev) if a is not None else None
    ctx = {k: to(v) for k, v in ctx.items()} if isinstance(ctx, dict) else to(ctx)
    return to(x), to(t), ctx, to(in_scale)


# ------------------------------------------------------------------ the expected launch sequence
CONTEXT = {   # the cached conditioning of a context: (op, step) model-level, and per layer
    "t23d": ([("norm_modulate", "ctx_cast"), ("gemm", "ctx_fc1"), ("gemm", "ctx_fc2"), ("gemm", "ctx_kv_all")], []),
    "t23d_pixart": ([("norm_modulate", "cap_ln"), ("gemm", "cap")],
                    [("norm_modulate", "ctx_ynorm"), ("gemm", "ctx_kv")]),
    "i23d": ([("norm_modulate", "cap_ln"), ("gemm", "cap"), ("norm_modulate", "ctx_clip_norm"),
              ("norm_modulate", "ctx_dino_cast"), ("gemm", "ctx_dino_fc1"), ("gemm", "ctx_dino_fc2")],
             [("gemm", "ctx_kv"), ("gemm", "ctx_dkv")]),
    "mv23d": ([("norm_modulate", "ctx_cast")], [("gemm", "ctx_kv")]),
}
PROLOGUE_T23D = [("timestep_embedding", "t_freq"), ("gemm", "t_mlp0"), ("gemm", "t_mlp2"), ("gemm", "adaLN")]
PROLOGUE_PIXART = [("timestep_embedding", "t_freq"), ("gemm", "t_mlp0"), ("gemm", "t_plus_cls"),
                   ("norm_modulate", "t_silu"), ("gemm", "adaLN")]


def expected_launches(family, depth, fp8, rows, split, mod_row=False):
    """The launch sequence of one traced call: [modulation_table] -> context -> prologue -> patch embed -> blocks ->
    final residual pass -> final layer.  rows: the attended samples (g0, g1) when identical-token samples take the
    closed form, else None; split: the split residual pass (LN3_SPLIT_RESID_PASS)."""
    seq = [Step(op, k, None) for op, k in PROLOGUE_T23D] if mod_row else []
    glob, per_layer = CONTEXT[family]
    seq += [Step(op, k, None) for op, k in glob]
    seq += [Step(op, k, l) for l in range(depth) for op, k in per_layer]
    if rows is not None:
        seq += [Step("gemm", "ctx_oconst", l) for l in range(depth)]
    if not mod_row:
        seq += [Step(op, k, None) for op, k in (PROLOGUE_T23D if family == "t23d" else PROLOGUE_PIXART)]
    seq.append(Step("patch_embed", "patch_embed", None))
    nm, gm = ("norm_modulate_fp8", "gemm_fp8") if fp8 else ("norm_modulate", "gemm")
    g0, g1 = rows if rows is not None else (0, B)
    for l in range(depth):
        seq += [Step(nm, "norm1", l), Step(gm, "qkv", l), Step("fmha", "self_attn", l), Step("gemm", "proj", l)]
        if not split or g1 > g0:
            seq.append(Step("norm_modulate", "resid_xb", l))
        if g1 > g0:
            seq += [Step("gemm", "cross_q", l), Step("fmha", "cross_attn", l), Step("gemm", "cross_out", l)]
        seq += [Step(nm, "norm2", l), Step(gm, "fc1", l), Step(gm, "fc2", l)]
    seq += [Step("norm_modulate", "final_resid", None), Step("final_layer", "final_layer", None)]
    return seq


# ------------------------------------------------------------------ the auditor
class Audit(LaunchAudit):
    """Checks each launch as it happens (block by block: only the values later launches read are kept)."""

    def __init__(self, m, family, seq, x, t, ctx, in_scale, rows, split, table_t=None, table_row=None):
        super().__init__(seq)
        self.m, self.family = m, family
        self.D, self.T, self.H, self.depth = m.embed_dim, m.pos_embed.shape[1], m.num_heads, m.depth
        self.M = B * self.T
        self.dev = x.device
        self.x_in, self.t_in, self.ctx, self.in_scale = x, t, ctx, in_scale
        self.rows, self.split = rows, split
        self.g0, self.g1 = rows if rows is not None else (0, B)
        self.r0, self.r1 = self.g0 * self.T, self.g1 * self.T
        self.table_t, self.table_row = table_t, table_row
        self.fp8 = m.gemm_precision == "fp8"
        self.pixart = family != "t23d"
        self.idx = torch.arange(self.M, device=self.dev) // self.T
        self.rec = {}
        self.kv, self.dkv, self.oc = {}, {}, {}
        self.wcache = {}

    # ---- weights from the module, rounded as the precision contract says
    def bf(self, p):
        return p.detach().to(self.dev, torch.bfloat16).double()

    def fp(self, p):
        return p.detach().to(self.dev, torch.float32).double()

    def q8(self, p):
        q, s = kb.restated_weight_fp8(p.detach().to(self.dev))
        return q, s

    def W(self, l):
        if l not in self.wcache:
            for k in [k for k in self.wcache if abs(k - l) > 1]:
                del self.wcache[k]
            b = self.m.blocks[l]
            mlp = b.mlp.mlp
            w = dict(qkv_w=b.attn.qkv.weight, qkv_b=self.fp(b.attn.qkv.bias), proj_w=self.bf(b.attn.proj.weight),
                     proj_b=self.fp(b.attn.proj.bias), cq_w=self.bf(b.cross_attn.to_q.weight),
                     co_w=self.bf(b.cross_attn.to_out[0].weight), co_b=self.fp(b.cross_attn.to_out[0].bias),
                     fc1_w=mlp[0].weight, fc1_b=self.fp(mlp[1].bias), fc2_w=mlp[2].weight, fc2_b=self.fp(mlp[3].bias),
                     kv_w=self.bf(torch.cat([b.cross_attn.to_k.weight, b.cross_attn.to_v.weight], 0)))
            for key in ("qkv_w", "fc1_w", "fc2_w"):
                w[key] = self.q8(w[key]) if self.fp8 else self.bf(w[key])
            if self.pixart:
                w.update(n1=self.fp(b.norm1.weight), n2=self.fp(b.norm2.weight), tab=self.fp(b.scale_shift_table))
            if b.attn.qk_norm:
                w.update(qn=self.fp(b.attn.q_norm.weight), kn=self.fp(b.attn.k_norm.weight),
                         cqn=self.fp(b.cross_attn.q_norm.weight), ckn=self.fp(b.cross_attn.k_norm.weight))
            self.wcache[l] = w
        return self.wcache[l]

    def mod(self, l):
        """Layer l's (B, 6D) shift / scale / gate rows, from the recorded adaLN output (and the block's table)."""
        D = self.D
        if self.pixart:
            return kb.f32(self.W(l)["tab"].reshape(1, 6 * D) + self.rec["t0"])
        return self.rec["ada"][:, l * 6 * D:(l + 1) * 6 * D]

    def chunk(self, l, j):
        return self.mod(l)[:, j * self.D:(j + 1) * self.D]

    # ---- assertions
    def check_x(self, got, ref):
        """fp32 residual stream: at most 1 ulp (double-rounding ties only), bit-exact almost everywhere."""
        self.within("residual stream x", got, ref, kb.ulp_f32(ref))
        exact = float((got.double() == ref).double().mean())
        assert exact >= 0.99, f"step {self.step.kind} layer {self.step.layer}: only {exact:.4f} of x is bit-exact"

    # ---- check kinds
    def gemm_ref(self, a64, w, b64, act=0, head=None):
        """(ref, tol) before the output rounding; w bf16 (fp64 values) or (codes, scales) with a64 = (codes, scales)."""
        if isinstance(w, tuple):
            (aq, as_), (wq, ws) = a64, w
            y, Tm = kb.fp8_reference(aq, as_, wq, ws, b64)
            E = kb.fp8_acc_bound(Tm, aq.shape[1], b64)
            if head is not None:
                return kb.fp8_head_norm_ref(y, E, head, head.shape[0], self.D)
            if act:
                v, ferr = kb.gelu_ref(y)
                return v, kb.SLOPE * E + ferr
            return y, E
        y = a64 @ w.T
        if b64 is not None:
            y = y + b64
        tau = kb.gemm_tau(a64, w, b64)
        if head is not None:
            return kb.head_rmsnorm_ref(y, tau, head, self.D, 1e-5)
        ref, act_err = kb.act_ref(act, y)
        return ref, (kb.SLOPE * tau + act_err if act else tau)

    def gemm_check(self, got, a64, w, b64, act=0, head=None, out="bf16", x0=None):
        ref, tol = self.gemm_ref(a64, w, b64, act, head)
        if out == "fp8":
            q, s = got
            sratio, _, ok, s_ok = kb.fp8_out_check(q, s, ref, tol)
            self.ratio[self.step.kind + " (scales)"] = max(self.ratio[self.step.kind + " (scales)"], sratio)
            assert bool(s_ok.all()), f"step {self.step.kind} layer {self.step.layer}: block scales off ({sratio:.3f})"
            if not bool(ok.all()):
                deq = q.double() * s.double().repeat_interleave(128, dim=1)
                raise AssertionError(self.fail_msg("fp8 codes", deq, ref, tol + (ref.abs() + tol) * 2.0 ** -4, ~ok))
            return ref, tol
        if out == "f32":
            bound = tol
        elif out == "resid":
            ref = x0 + ref
            bound = tol + kb.ulp(ref.abs() + tol, 23) / 2
        elif isinstance(w, tuple):
            bound = kb.fp8_bf16_bound(ref, tol)
        else:
            bound = kb.gemm_bf16_bound(ref, tol)
        self.within("output", got, ref, bound)
        return ref, bound

    def fmha_check(self, got, q, k, v):
        ref, tol = kb.fmha_reference(q, k, v, self.H, 64 ** -0.5, False)
        bound = kb.gemm_bf16_bound(ref, tol)
        self.within("attention", got, ref, bound)
        return ref, bound

    def norm_out_ref(self, xg, norm, eps, weight, l, js):
        """(y, bound) of the modulated output from the kernel's own updated x; bf16 or fp8 bound."""
        shift, scale = self.chunk(l, js[0]), self.chunk(l, js[1])
        idx = self.idx[:xg.shape[0]]
        y, tau = kb.nm_out_ref(xg, norm, eps, 0, weight=weight, shift=shift, scale=scale, mod_idx=idx)
        if not self.fp8:
            return y, kb.bf16_bound(y, tau)
        from oracle import dit as odit
        n = odit.layer_norm(xg, eps) if norm == NORM_LAYER else odit.rms_norm(xg, None, eps)
        if weight is not None:
            n = n * weight
        # the fp32 error of the modulated value before the quantisation: test_gpu_norm_modulate_fp8.py's 64 u term,
        # or the glue kernels' tau where it is larger -- tau carries the LayerNorm's mean cancellation
        # (rstd * gamma * mean|x|), which a residual stream with a large mean makes the larger of the two
        e64 = 64 * 2.0 ** -24 * (n.abs() * (1 + scale[idx].abs()) + shift[idx].abs())
        return y, torch.maximum(e64, tau)

    def norm_out_check(self, got, xg, norm, eps, weight, l, js=(0, 1)):
        y, b = self.norm_out_ref(xg, norm, eps, weight, l, js)
        if self.fp8:
            q, s = got
            err, bound = kb.nm_fp8_error(q, s, y, b)
            deq = q.double() * s.double().repeat_interleave(128, dim=1)
            self.within("fp8 output (dequantised)", deq, y, bound)
            bound_y = bound
        else:
            self.within("bf16 output", got, y, b)
            bound_y = b
        if l == SEP_L:
            wrong, _ = self.norm_out_ref(xg, norm, eps, weight, l, (js[0] + 1, js[1] + 1))
            # an e4m3 code is only good to 2^-4 relative: the fp8 output separates by ~16x a relative change of one
            self.separated("norm_modulate_fp8 output" if self.fp8 else "norm_modulate output", y, wrong, bound_y,
                           factor=FP8_FACTOR if self.fp8 else 100.0)
        return y

    # ---- context
    def do_ctx_cast(self, l, args, kw, ret):
        if self.family == "t23d":
            c = self.ctx
        else:
            c = self.ctx["concat"].reshape(B, -1, self.ctx["concat"].shape[-1])
        c = c.reshape(-1, c.shape[-1]).double()
        self.within("bf16 cast", ret, c, kb.ulp_bf16(c) / 2)
        self.rec["cb"] = ret

    def do_ctx_fc1(self, l, args, kw, ret):
        p = self.m.clip_text_proj.y_proj.fc1
        self.gemm_check(ret, self.rec["cb"].double(), self.bf(p.weight), self.fp(p.bias), ACT_GELU_TANH)
        self.rec["c1"] = ret

    def do_ctx_fc2(self, l, args, kw, ret):
        p = self.m.clip_text_proj.y_proj.fc2
        self.gemm_check(ret, self.rec["c1"].double(), self.bf(p.weight), self.fp(p.bias))
        self.rec["c2"] = ret

    def _store_kv(self, l, kv, store):
        D = self.D
        kv = kv.view(B, -1, 2 * D)
        store[l] = (kv[:, :, :D], kv[:, :, D:])

    def do_ctx_kv_all(self, l, args, kw, ret):
        """T23D: one GEMM for every layer's K|V of the projected context: columns [2 D l, 2 D (l + 1))."""
        D, a = self.D, self.rec["c2"].double()
        for layer in range(self.depth):
            self.step = Step(self.step.op, "ctx_kv_all", layer)
            cols = ret[:, 2 * D * layer:2 * D * (layer + 1)]
            ref, bound = self.gemm_check(cols, a, self.W(layer)["kv_w"], None)
            if layer == SEP_L:
                wrong, _ = self.gemm_ref(a, self.W(layer + 1)["kv_w"], None)
                self.separated("gemm", ref, wrong, bound, self._live(a))
            self._store_kv(layer, cols, self.kv)

    def do_cap_ln(self, l, args, kw, ret):
        ln = self.m.cap_embedder[0]
        w, b = self.fp(ln.weight), self.fp(ln.bias)
        vec = self.ctx["vector"].double()
        zero = torch.zeros(B, dtype=torch.long, device=self.dev)
        y, tau = kb.nm_out_ref(vec, NORM_LAYER, 1e-5, 0, shift=b[None], scale=(w - 1)[None], mod_idx=zero)
        self.within("bf16 output", ret, y, kb.bf16_bound(y, tau))
        self.rec["vn"] = ret

    def do_cap(self, l, args, kw, ret):
        p = self.m.cap_embedder[1]
        self.gemm_check(ret, self.rec["vn"].double(), self.bf(p.weight), self.fp(p.bias), out="f32")
        self.rec["cls"] = ret

    def _rms_cast(self, ret, x, weight):
        y, tau = kb.nm_out_ref(x, NORM_RMS, 1e-5, 0, weight=weight)
        self.within("bf16 output", ret, y, kb.bf16_bound(y, tau))

    def do_ctx_ynorm(self, l, args, kw, ret):
        ca = self.ctx["crossattn"].double()
        self._rms_cast(ret, ca.reshape(-1, ca.shape[-1]), self.fp(self.m.blocks[l].attention_y_norm.weight))
        self.rec["y"] = ret

    def do_ctx_clip_norm(self, l, args, kw, ret):
        ca = self.ctx["crossattn"][..., :1024].double()
        self._rms_cast(ret, ca.reshape(-1, 1024), self.fp(self.m.attention_y_norm.weight))
        self.rec["y"] = ret

    def do_ctx_dino_cast(self, l, args, kw, ret):
        c = self.ctx["crossattn"][..., 1024:].double()
        c = c.reshape(-1, c.shape[-1])
        self.within("bf16 cast", ret, c, kb.ulp_bf16(c) / 2)
        self.rec["cb"] = ret

    def do_ctx_dino_fc1(self, l, args, kw, ret):
        p = self.m.dino_proj.y_proj.fc1
        self.gemm_check(ret, self.rec["cb"].double(), self.bf(p.weight), self.fp(p.bias), ACT_GELU_TANH)
        self.rec["c1"] = ret

    def do_ctx_dino_fc2(self, l, args, kw, ret):
        p = self.m.dino_proj.y_proj.fc2
        self.gemm_check(ret, self.rec["c1"].double(), self.bf(p.weight), self.fp(p.bias))
        self.rec["dino"] = ret

    def do_ctx_kv(self, l, args, kw, ret):
        """Layer l's cross-attention K|V: PixArt T23D of its own RMS-normed tokens; I23D / MV23D with the K half
        head-normed by cross_attn.k_norm and the V half untouched."""
        w = self.W(l)
        a = (self.rec["y"] if self.family in ("t23d_pixart", "i23d") else self.rec["cb"]).double()
        head = w["ckn"][None] if "ckn" in w else None
        ref, bound = self.gemm_check(ret, a, w["kv_w"], None, head=head)
        if l == SEP_L:
            wrong, _ = self.gemm_ref(a, self.W(l + 1)["kv_w"], None, head=head)
            self.separated("gemm", ref, wrong, bound, self._live(a))
        self._store_kv(l, ret, self.kv)

    def do_ctx_dkv(self, l, args, kw, ret):
        """I23D: layer l's second self-attention K/V source, the DINO tokens through the K|V rows of attn.qkv, the
        K half head-normed by attn.k_norm."""
        b, D, w = self.m.blocks[l], self.D, self.W(l)
        kv_w, kv_b = self.bf(b.attn.qkv.weight[D:]), self.fp(b.attn.qkv.bias[D:])
        a = self.rec["dino"].double()
        ref, bound = self.gemm_check(ret, a, kv_w, kv_b, head=w["kn"][None])
        if l == SEP_L:
            wrong, _ = self.gemm_ref(a, kv_w, kv_b, head=w["qn"][None])
            self.separated("gemm head-norm", ref, wrong, bound, self._k_cols(ref))
        self._store_kv(l, ret, self.dkv)

    @staticmethod
    def _live(a):
        """Rows of an operand that are not all zero (the zero-token samples give zero K/V without a bias)."""
        return (a.abs().sum(1) > 0)[:, None]

    def _k_cols(self, ref):
        m = torch.zeros_like(ref, dtype=torch.bool)
        m[:, :self.D] = True
        return m

    def do_ctx_oconst(self, l, args, kw, ret):
        """The closed form of identical-token samples: to_out of real float64 softmax attention over the sample's own
        context K/V (any query gives the same result there).  Rows of the attended samples are never read."""
        k, v = self.kv[l]
        g = torch.Generator(device=self.dev).manual_seed(l)
        q = torch.randn(B, 2, self.D, device=self.dev, generator=g, dtype=torch.float64)
        attn = torch.nn.functional.scaled_dot_product_attention(
            kb.heads(q, self.H), kb.heads(k, self.H), kb.heads(v, self.H)).transpose(1, 2).flatten(2)
        out = [b for b in range(B) if not self.g0 <= b < self.g1]
        assert torch.equal(attn[out, 0], attn[out, 1]), "identical context tokens: the query cannot matter"
        w = self.W(l)
        ref, bound = self.gemm_check(ret[out], attn[out, 0], w["co_w"], w["co_b"])
        if l == SEP_L:
            wrong, _ = self.gemm_ref(attn[out, 0], self.W(l + 1)["co_w"], self.W(l + 1)["co_b"])
            self.separated("gemm", ref, wrong, bound)
        self.oc[l] = ret

    # ---- prologue
    def do_t_freq(self, l, args, kw, ret):
        t = self.table_t if self.table_t is not None and "ada" not in self.rec else self.t_in
        ref, bound = kb.timestep_embedding_ref(t.float())
        self.within("[cos | sin]", ret, ref, bound)
        self.separated("timestep_embedding (cos and sin halves swapped)", ref, ref.roll(128, 1), bound)
        self.rec["tfeat"] = ret

    def do_t_mlp0(self, l, args, kw, ret):
        p = self.m.t_embedder.mlp[0]
        self.gemm_check(ret, self.rec["tfeat"].double(), self.bf(p.weight), self.fp(p.bias), ACT_SILU)
        self.rec["th"] = ret

    def do_t_mlp2(self, l, args, kw, ret):
        p = self.m.t_embedder.mlp[2]
        self.gemm_check(ret, self.rec["th"].double(), self.bf(p.weight), self.fp(p.bias), ACT_SILU)
        self.rec["st"] = ret

    def do_t_plus_cls(self, l, args, kw, ret):
        """t = t_emb + the pooled embedding of the context (zero for MV23D), the GEMM's in-place residual epilogue."""
        p = self.m.t_embedder.mlp[2]
        cls = self.rec["cls"].double() if "cls" in self.rec else torch.zeros(B, self.D, device=self.dev,
                                                                             dtype=torch.float64)
        a, w, b = self.rec["th"].double(), self.bf(p.weight), self.fp(p.bias)
        ref, bound = self.gemm_check(ret, a, w, b, out="resid", x0=cls)
        if "cls" in self.rec:
            self.separated("gemm resid", ref, ref - cls + cls.roll(1, 0), bound)
        self.rec["t"] = ret

    def do_t_silu(self, l, args, kw, ret):
        y, tau = kb.nm_out_ref(self.rec["t"].double(), NORM_NONE, 0, ACT_SILU)
        self.within("bf16 output", ret, y, kb.bf16_bound(y, tau))
        self.rec["st"] = ret

    def do_adaLN(self, l, args, kw, ret):
        a = self.rec["st"].double()
        if self.pixart:
            p = self.m.adaLN_modulation[1]
            self.gemm_check(ret, a, self.bf(p.weight), self.fp(p.bias), out="f32")
            self.rec["t0"] = ret
            return
        lins = [b.adaLN_modulation[1] for b in self.m.blocks] + [self.m.final_layer.adaLN_modulation[1]]
        w = self.bf(torch.cat([p.weight for p in lins], 0))
        ref, bound = self.gemm_check(ret, a, w, self.fp(torch.cat([p.bias for p in lins], 0)), out="f32")
        if self.table_t is not None and "ada" not in self.rec:     # modulation_table: the step's row, every sample
            self.rec["ada"] = ret[self.table_row:self.table_row + 1].expand(B, -1)
        else:
            self.rec["ada"] = ret
        self.separated("gemm f32 (chunk j + 1)", ref, ref.roll(-self.D, 1), bound)

    def do_patch_embed(self, l, args, kw, ret):
        p = self.m.x_embedder.proj
        a = dict(x=self.x_in.double(), in_scale=self.in_scale.double() if self.in_scale is not None else None,
                 W=self.fp(p.weight), bias=self.fp(p.bias), pos=self.fp(self.m.pos_embed[0]))
        ref, bound = kb.patch_embed_ref(**a)
        self.within("tokens", ret, ref, bound)
        self.separated("patch_embed", ref, kb.patch_embed_ref(**a, roll_plane=True)[0], bound)
        self.rec["x"] = ret.view(self.M, self.D)

    # ---- blocks
    def pre_norm(self, l, key):
        return (NORM_RMS, 1e-5, self.W(l)[key]) if self.pixart else (NORM_LAYER, 1e-6, None)

    def cur_x(self, args):
        """The whole residual stream after the launch (the launch may have updated a row slice of it)."""
        return self.m._ws[B]["x"].view(self.M, self.D).clone()

    def do_norm1(self, l, args, kw, ret):
        xb_ = self.rec["x"].double()
        xg = self.cur_x(args)
        if l == 0:
            assert kw.get("resid") is None
            ref = xb_
            self.check_x(xg, ref)
        else:
            val, gate = self.rec["val_mlp"].double(), self.chunk(l - 1, 5)
            ref = kb.nm_resid_ref(xb_, val, gate, self.idx)
            self.check_x(xg, ref)
            if l == SEP_L + 1:
                wrong = kb.nm_resid_ref(xb_, val, self.chunk(l - 1, 4), self.idx)           # mod chunk 5 - 1
                self.separated("residual update", ref, wrong, kb.ulp_f32(ref))
                wrong = kb.nm_resid_ref(xb_, self.rec["val_attn"].double(), gate, self.idx)  # an earlier val
                self.separated("residual update (stale val)", ref, wrong, kb.ulp_f32(ref))
        norm, eps, w = self.pre_norm(l, "n1")
        self.norm_out_check(ret, xg.double(), norm, eps, w, l, (0, 1))
        self.rec["x"], self.rec["a"] = xg, ret

    def do_qkv(self, l, args, kw, ret):
        w = self.W(l)
        head = torch.stack([w["qn"], w["kn"]]) if "qn" in w else None
        a = self.rec["a"] if self.fp8 else self.rec["a"].double()
        ref, bound = self.gemm_check(ret, a, w["qkv_w"], w["qkv_b"], head=head)
        if l == SEP_L:
            qk = torch.zeros_like(ref, dtype=torch.bool)
            qk[:, :2 * self.D] = True
            if head is not None and not self.fp8:      # fp8: the head-norm bound carries the whole head's error
                wrong, _ = self.gemm_ref(a, w["qkv_w"], w["qkv_b"], head=head.flip(0))
                self.separated("gemm head-norm (q_norm and k_norm swapped)", ref, wrong, bound, qk)
            wrong, _ = self.gemm_ref(a, self.W(l + 1)["qkv_w"], self.W(l + 1)["qkv_b"], head=head)
            if self.fp8:
                self.separated("gemm_fp8", ref, wrong, bound, ~qk if head is not None else None, factor=FP8_FACTOR)
            else:
                self.separated("gemm", ref, wrong, bound)
        self.rec["qkv"] = ret

    def do_self_attn(self, l, args, kw, ret):
        """Self-attention over the block's own tokens, followed (I23D) by layer l's DINO K/V."""
        D = self.D
        qkv = self.rec["qkv"].view(B, self.T, 3 * D)
        q, k, v = qkv[:, :, :D], qkv[:, :, D:2 * D], qkv[:, :, 2 * D:]
        if l in self.dkv:
            k2, v2 = self.dkv[l]
            kk, vv = torch.cat([k, k2], 1), torch.cat([v, v2], 1)
        else:
            kk, vv = k, v
        ref, bound = self.fmha_check(ret, q, kk, vv)
        if l == SEP_L:
            if l in self.dkv:
                k2, v2 = self.dkv[l + 1]
                wrong, _ = kb.fmha_reference(q, torch.cat([k, k2], 1), torch.cat([v, v2], 1), self.H, 0.125, False)
                # the DINO keys are 256 of the 1024: their source moves the output by about a quarter as much
                self.separated("fmha (dkv of layer l + 1)", ref, wrong, bound, factor=FMHA_FACTOR / 4)
            wrong, _ = kb.fmha_reference(q, kk.roll(1, 0), vv.roll(1, 0), self.H, 0.125, False)
            self.separated("fmha (neighbouring sample's K/V)", ref, wrong, bound, factor=FMHA_FACTOR)
        self.rec["att"] = ret.reshape(self.M, D)

    def do_proj(self, l, args, kw, ret):
        w = self.W(l)
        ref, bound = self.gemm_check(ret, self.rec["att"].double(), w["proj_w"], w["proj_b"])
        if l == SEP_L:
            wrong, _ = self.gemm_ref(self.rec["att"].double(), self.W(l + 1)["proj_w"], self.W(l + 1)["proj_b"])
            self.separated("gemm", ref, wrong, bound)
        self.rec["val_attn"] = ret

    def _rows_view(self, t, what):
        """A consumer of the attended rows must read exactly rows [r0, r1) of its buffer."""
        rows = t.shape[0] * (t.shape[1] if t.dim() == 3 else 1)
        assert rows == self.r1 - self.r0 and t.storage_offset() == self.r0 * self.D, \
            f"step {self.step.kind} layer {self.step.layer}: {what} covers {rows} rows from offset {t.storage_offset()}"

    def do_resid_xb(self, l, args, kw, ret):
        x0, xg = self.rec["x"].double(), self.cur_x(args)
        r0, r1 = (self.r0, self.r1) if self.split else (0, self.M)
        if self.split:
            self._rows_view(args[0], "x")
        gate = self.chunk(l, 2)
        val = self.rec["val_attn"].double()
        ref = x0.clone()
        ref[r0:r1] = kb.nm_resid_ref(x0[r0:r1], val[r0:r1], gate, self.idx[r0:r1])
        self.check_x(xg, ref)          # rows outside [r0, r1) unchanged
        if l == SEP_L:
            wrong = kb.nm_resid_ref(x0[r0:r1], val[r0:r1], self.chunk(l, 1), self.idx[r0:r1])
            self.separated("residual update", ref[r0:r1], wrong, kb.ulp_f32(ref[r0:r1]))
        xr = xg[r0:r1].double()
        self.within("xb = bf16(x)", ret, xr, kb.ulp_bf16(xr) / 2)
        self.rec["x"], self.rec["xb"] = xg, ret

    def do_cross_q(self, l, args, kw, ret):
        w = self.W(l)
        self._rows_view(args[0], "xb")
        xb = self.rec["xb"] if self.rec["xb"].shape[0] == self.r1 - self.r0 else self.rec["xb"][self.r0:self.r1]
        head = w["cqn"][None] if "cqn" in w else None
        ref, bound = self.gemm_check(ret, xb.double(), w["cq_w"], None, head=head)
        if l == SEP_L and head is not None:
            wrong, _ = self.gemm_ref(xb.double(), w["cq_w"], None, head=w["ckn"][None])
            self.separated("gemm head-norm (k_norm for q_norm)", ref, wrong, bound)
        self.rec["q"] = ret

    def do_cross_attn(self, l, args, kw, ret):
        """Samples [g0, g1) attend to their own context's K/V of layer l."""
        g0, g1 = self.g0, self.g1
        self._rows_view(args[0], "q")
        q = self.rec["q"].view(g1 - g0, self.T, self.D)
        k, v = self.kv[l]
        ref, bound = self.fmha_check(ret, q, k[g0:g1], v[g0:g1])
        if l == SEP_L:
            k1, v1 = self.kv[l + 1]
            wrong, _ = kb.fmha_reference(q, k1[g0:g1], v1[g0:g1], self.H, 0.125, False)
            live = (v[g0:g1].abs().sum((1, 2)) > 0)[:, None, None]        # zero-token samples without a bias: V = 0
            self.separated("fmha (K/V of layer l + 1)", ref, wrong, bound, live, factor=FMHA_FACTOR)
            o = [(b + 2) % B for b in range(g0, g1)]                          # the other CFG half
            wrong, _ = kb.fmha_reference(q, k[o], v[o], self.H, 0.125, False)
            self.separated("fmha (the other CFG half's context)", ref, wrong, bound, factor=FMHA_FACTOR)
        self.rec["att_c"] = ret.reshape(-1, self.D)

    def do_cross_out(self, l, args, kw, ret):
        w = self.W(l)
        self._rows_view(args[0], "att")
        ref, bound = self.gemm_check(ret, self.rec["att_c"].double(), w["co_w"], w["co_b"])
        self.rec["val_cross"] = ret

    def do_norm2(self, l, args, kw, ret):
        """x += cross-attention (ungated); closed-form samples add their broadcast row and, in the split pass, first
        their own gate_msa * attention projection, which their val rows still hold."""
        x0, xg = self.rec["x"].double(), self.cur_x(args)
        val = self.rec["val_attn"].double().clone()
        if self.r1 > self.r0:
            val[self.r0:self.r1] = self.rec["val_cross"].double()
        if self.rows is not None:
            oc = self.oc[l].double()
            inside = (self.idx >= self.g0) & (self.idx < self.g1)
            og = self.chunk(l, 2) if self.split else None
            ref = kb.nm_resid_ref(x0, val, None, None, bcast=oc, bcast_idx=self.idx, inside=inside, ogate=og,
                                  ogate_idx=self.idx)
            if l == SEP_L:
                sh = torch.clamp(self.idx - 1, 0, B) if self.g0 > 0 else self.idx + 1
                ins_w = (sh >= self.g0) & (sh < self.g1)
                wrong = kb.nm_resid_ref(x0, val, None, None, bcast=oc, bcast_idx=self.idx, inside=ins_w, ogate=og,
                                        ogate_idx=self.idx)
                self.separated("residual update (rows shifted by one sample)", ref, wrong, kb.ulp_f32(ref),
                               (ins_w != inside)[:, None])
        else:
            ref = kb.nm_resid_ref(x0, val, None, None)
        self.check_x(xg, ref)
        norm, eps, w = self.pre_norm(l, "n2")
        self.norm_out_check(ret, xg.double(), norm, eps, w, l, (3, 4))
        self.rec["x"], self.rec["a"] = xg, ret

    def do_fc1(self, l, args, kw, ret):
        w = self.W(l)
        a = self.rec["a"] if self.fp8 else self.rec["a"].double()
        self.gemm_check(ret, a, w["fc1_w"], w["fc1_b"], ACT_GELU_ERF, out="fp8" if self.fp8 else "bf16")
        self.rec["h"] = ret

    def do_fc2(self, l, args, kw, ret):
        w = self.W(l)
        a = self.rec["h"] if self.fp8 else self.rec["h"].double()
        ref, bound = self.gemm_check(ret, a, w["fc2_w"], w["fc2_b"])
        if l == SEP_L and self.fp8:
            wrong, _ = self.gemm_ref(a, self.W(l + 1)["fc2_w"], self.W(l + 1)["fc2_b"])
            self.separated("gemm_fp8 (fc2 of layer l + 1)", ref, wrong, bound, factor=FP8_FACTOR)
        self.rec["val_mlp"] = ret

    def do_final_resid(self, l, args, kw, ret):
        L = self.depth - 1
        ref = kb.nm_resid_ref(self.rec["x"].double(), self.rec["val_mlp"].double(), self.chunk(L, 5), self.idx)
        xg = self.cur_x(args)
        self.check_x(xg, ref)
        self.rec["x"] = xg

    def do_final_layer(self, l, args, kw, ret):
        D, fl = self.D, self.m.final_layer
        x = self.rec["x"].double().view(B, self.T, D)
        W, b = self.fp(fl.linear.weight), self.fp(fl.linear.bias)
        if self.pixart:
            t, tab = self.rec["t"].double(), self.fp(fl.scale_shift_table)
            sh = sc = t
            tabs = dict(shift_tab=tab[0], scale_tab=tab[1])
        else:
            f0 = self.depth * 6 * D
            ada = self.rec["ada"]
            sh, sc = ada[:, f0:f0 + D].double(), ada[:, f0 + D:f0 + 2 * D].double()
            tabs = {}
        ref, bound = kb.final_layer_ref(x, sh, sc, W, b, 32, 4, **tabs)
        self.within("output", ret, ref, bound)
        wrong, _ = kb.final_layer_ref(x, sh, sc, W, b, 32, 4, swap_pq=True, **tabs)
        pq = torch.zeros(1, 1, 32, 32, dtype=torch.bool, device=self.dev)
        pq[..., 0::2, 1::2] = True
        pq[..., 1::2, 0::2] = True                                 # p != q: the elements the swap moves
        self.separated("final_layer (unpatchify p and q swapped)", ref, wrong, bound, pq)
        self.rec["out"] = ret


# ------------------------------------------------------------------ one audited forward
def run_audit(family, prec, variant, dev, monkeypatch, slip=None, graph=True):
    m = model(family, dev)
    m.set_gemm_precision(prec)
    m._invalidate()
    layout = variant if variant in LAYOUTS else "cond-zero"
    monkeypatch.setenv("LN3_SPLIT_RESID_PASS", "0" if variant == "no-split" else "1")
    monkeypatch.setenv("LN3_UNCOND_CLOSED_FORM", "0" if variant == "full-attention" else "1")
    monkeypatch.setenv("LN3_CUDA_GRAPH", "0")
    x, t, ctx, in_scale = inputs(family, layout, dev)
    rows = LAYOUTS[layout] if variant != "full-attention" else None
    split = rows is not None and variant != "no-split"
    mod_row = variant == "mod-row"
    m.prepare()
    seq = expected_launches(family, m.depth, prec == "fp8", rows, split, mod_row)
    table_t = torch.tensor([12.0, 250.0, 603.0, 871.0], device=dev) if mod_row else None
    audit = Audit(m, family, seq, x, t, ctx, in_scale, rows, split, table_t=table_t, table_row=2)
    with torch.no_grad(), traced(audit, monkeypatch, TRACED, slip):
        if mod_row:
            table = m.modulation_table(table_t)
            cx = m._context(ctx)
            out = m._forward_impl(x, t, cx, in_scale, table[2:3]).clone()
        else:
            out = m(x, t, ctx, in_scale=in_scale)
    assert audit.n_checked == audit.n_traced == len(seq), (audit.n_checked, audit.n_traced, len(seq))
    assert torch.equal(out, audit.rec["out"])
    if graph:
        # the CUDA-graph replay runs the audited launch sequence: bit-identical output
        monkeypatch.setenv("LN3_CUDA_GRAPH", "1")
        with torch.no_grad():
            if mod_row:
                g = m.capture_graph(B, ctx, shared_mod=True)
                g.x.copy_(x)
                g.in_scale.copy_(in_scale)
                g.mod.copy_(table[2:3])
                g.replay()
                rep = g.out.clone()
            else:
                rep = m(x, t, ctx, in_scale=in_scale)
        assert torch.equal(rep, out), f"graph replay differs from the audited eager forward ({family} {prec} {variant})"
    return audit


FAMILIES = ["t23d", "t23d_pixart", "i23d", "mv23d"]
VARIANTS = ["cond-zero", "zero-cond", "distinct", "no-split", "full-attention"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("prec", ["bf16", "fp8"])
@pytest.mark.parametrize("family", FAMILIES)
def test_denoiser_launch_audit(dev, monkeypatch, family, prec, variant):
    audit = run_audit(family, prec, variant, dev, monkeypatch)
    _report(audit, f"{family} {prec} {variant}")
    kinds = {"gemm", "fmha (neighbouring sample's K/V)", "residual update",
             "timestep_embedding (cos and sin halves swapped)", "patch_embed",
             "final_layer (unpatchify p and q swapped)",
             "norm_modulate_fp8 output" if prec == "fp8" else "norm_modulate output"}
    if variant in ("cond-zero", "zero-cond", "no-split"):
        kinds.add("residual update (rows shifted by one sample)")
    if family in ("i23d", "mv23d"):
        kinds.add("gemm head-norm (k_norm for q_norm)")
        if prec == "bf16":
            kinds.add("gemm head-norm (q_norm and k_norm swapped)")
    if prec == "fp8":
        kinds |= {"gemm_fp8", "gemm_fp8 (fc2 of layer l + 1)"}
    missing = kinds - set(audit.sep)
    assert not missing, f"check kinds without a separation assertion: {missing}"


@pytest.mark.parametrize("prec", ["bf16", "fp8"])
def test_t23d_shared_modulation_row_audit(dev, monkeypatch, prec):
    """The sampler's path: modulation_table() for every step at once, one row shared by the batch, in_scale folded
    into the patch embed."""
    audit = run_audit("t23d", prec, "mod-row", dev, monkeypatch)
    _report(audit, f"t23d {prec} shared modulation row")


# ------------------------------------------------------------------ seeded slips: the audit must catch them
def _shift(t, elems):
    return t.as_strided(t.shape, t.stride(), t.storage_offset() + elems)


def _slip_gate(args, kw):                     # resid gate one chunk over (D columns): gate_msa row of the next chunk
    kw["resid_gate"] = _shift(kw["resid_gate"], kw["resid_gate"].shape[1])
    return args, kw


def _slip_next_layer_kv(args, kw):            # T23D K|V buffer (B Lc, depth 2D): layer l + 1 sits 2D columns further
    D = args[1].shape[2]
    args[1], args[2] = _shift(args[1], 2 * D), _shift(args[2], 2 * D)
    return args, kw


def _slip_sub_batch(args, kw):                # cross-attention K/V of samples [g0 + 1, g1 + 1)
    args[1], args[2] = _shift(args[1], args[1].stride(0)), _shift(args[2], args[2].stride(0))
    return args, kw


def _slip_swap_head_norm(args, kw):           # q_norm and k_norm exchanged
    kw["head_norm"] = kw["head_norm"].flip(0).contiguous()
    return args, kw


SLIPS = {   # id: (family, prec, variant, step, layer, rewrite, step named in the failure)
    "resid-gate-next-chunk": ("t23d", "bf16", "cond-zero", "norm1", 3, _slip_gate, "norm1 layer 3"),
    "kv-of-layer-l+1": ("t23d", "bf16", "cond-zero", "cross_attn", 3, _slip_next_layer_kv, "cross_attn layer 3"),
    "cross-sub-batch-shifted": ("t23d_pixart", "bf16", "cond-zero", "cross_attn", 2, _slip_sub_batch,
                                "cross_attn layer 2"),
    "qk-head-norm-swapped": ("i23d", "bf16", "distinct", "qkv", 4, _slip_swap_head_norm, "qkv layer 4"),
}


@pytest.mark.parametrize("case", list(SLIPS) + ["fc2-stale-fp8-scales"])
def test_seeded_slip_is_caught(dev, monkeypatch, case):
    if case == "fc2-stale-fp8-scales":
        # fc2 reads the block scales of the previous layer's fc1 (a stale copy of the h8 scale buffer)
        stale = {}

        def slip(args, kw):
            args[1] = stale["h8s"]
            return args, kw

        family, prec, variant, step, layer, named = "mv23d", "fp8", "cond-zero", "fc2", 2, "fc2 layer 2"
        orig = Audit.do_fc2

        def keep(self, l, args, kw, ret):
            if l == layer - 1:
                stale["h8s"] = args[1].clone()
            return orig(self, l, args, kw, ret)
        monkeypatch.setattr(Audit, "do_fc2", keep)
    else:
        family, prec, variant, step, layer, slip, named = SLIPS[case]
    with pytest.raises(AssertionError) as e:
        run_audit(family, prec, variant, dev, monkeypatch, slip=(step, layer, slip), graph=False)
    msg = str(e.value)
    print(f"{case}: {msg[:400]}")
    assert f"step {named}" in msg and "worst at index" in msg, msg
