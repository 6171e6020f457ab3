"""GPU (-m gpu): the per-launch float64 audit of test_gpu_denoiser_launches.py on DiT-XL/2 blocks.

DiT-XL/2 is the one denoiser whose widths differ inside a block: hidden D = 1152 with 16 self-attention heads of 72,
and a cross-attention that keeps the reference's 64-wide heads, inner width E = 1024.  Its cross-attention output is
an (M, E) view at the start of the self-attention output buffer, and its context K/V cache is (B Lc, depth 2 E).  The
audit runs the T23D launch sequence, checks, and slipped-mapping separations of test_gpu_denoiser_launches.py on an
XL-width model of depth 3 (the separations run at layer 1 and read layer 2), with these width-dependent checks:
  * self-attention against the float64 reference at head width 72, cross-attention at 64 (fmha_reference_hd);
  * the context K|V GEMM's per-layer columns [2 E l, 2 E (l + 1)), the cross-attention query and output as E-wide rows
    at offset r0 E of their buffers, and the closed-form rows over E-wide K/V.
fp8 is refused at 1152 (embed_dim % 256), so every configuration runs in bf16."""
import pytest
import torch

import kernel_bounds as kb
import test_gpu_denoiser_launches as dl
from fmha_reference_hd import fmha_reference_hd
from launch_audit import FMHA_FACTOR, Step, _report

pytestmark = pytest.mark.gpu

B, SEP_L = dl.B, dl.SEP_L
XL_DEPTH = 3


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def xl_model(dev):
    from ln3diff_b200.dit.dit_models_xformers import TextCondDiTBlock
    from ln3diff_b200.dit.dit_trilatent import DiT_TriLatent
    from oracle import dit as odit
    m = DiT_TriLatent(depth=XL_DEPTH, hidden_size=1152, patch_size=2, num_heads=16, input_size=32, num_classes=0,
                      learn_sigma=False, in_channels=4, context_dim=768, roll_out=True, vit_blk=TextCondDiTBlock)
    m = dl._seeded(m.eval(), lambda s, pe: odit.synth_state_dict(s, seed=7, keep={"pos_embed": pe}))
    return m.to(dev)


class XLAudit(dl.Audit):
    """dl.Audit with the cross-attention width E and the head width of each attention taken from its operands."""

    def __init__(self, m, *a, **kw):
        super().__init__(m, *a, **kw)
        self.E = m.blocks[0].cross_attn.to_q.out_features

    def attn_ref(self, q, k, v):
        hd = q.shape[-1] // self.H
        if hd == 64:
            return kb.fmha_reference(q, k, v, self.H, 64 ** -0.5, False)
        return fmha_reference_hd(q, k, v, self.H, hd, hd ** -0.5, False)

    def fmha_check(self, got, q, k, v):
        ref, tol = self.attn_ref(q, k, v)
        bound = kb.gemm_bf16_bound(ref, tol)
        self.within("attention", got, ref, bound)
        return ref, bound

    def _rows_view_e(self, t, what):
        rows = t.shape[0] * (t.shape[1] if t.dim() == 3 else 1)
        assert rows == self.r1 - self.r0 and t.storage_offset() == self.r0 * self.E, \
            f"step {self.step.kind} layer {self.step.layer}: {what} covers {rows} rows from offset {t.storage_offset()}"

    def _store_kv(self, l, kv, store):
        E = self.E
        kv = kv.view(B, -1, 2 * E)
        store[l] = (kv[:, :, :E], kv[:, :, E:])

    def do_ctx_kv_all(self, l, args, kw, ret):
        E, a = self.E, self.rec["c2"].double()
        for layer in range(self.depth):
            self.step = Step(self.step.op, "ctx_kv_all", layer)
            cols = ret[:, 2 * E * layer:2 * E * (layer + 1)]
            ref, bound = self.gemm_check(cols, a, self.W(layer)["kv_w"], None)
            if layer == SEP_L:
                wrong, _ = self.gemm_ref(a, self.W(layer + 1)["kv_w"], None)
                self.separated("gemm", ref, wrong, bound, self._live(a))
            self._store_kv(layer, cols, self.kv)

    def do_ctx_oconst(self, l, args, kw, ret):
        k, v = self.kv[l]
        g = torch.Generator(device=self.dev).manual_seed(l)
        q = torch.randn(B, 2, self.E, device=self.dev, generator=g, dtype=torch.float64)
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

    def do_self_attn(self, l, args, kw, ret):
        D = self.D
        qkv = self.rec["qkv"].view(B, self.T, 3 * D)
        q, k, v = qkv[:, :, :D], qkv[:, :, D:2 * D], qkv[:, :, 2 * D:]
        ref, bound = self.fmha_check(ret, q, k, v)
        if l == SEP_L:
            wrong, _ = self.attn_ref(q, k.roll(1, 0), v.roll(1, 0))
            self.separated("fmha (neighbouring sample's K/V)", ref, wrong, bound, factor=FMHA_FACTOR)
            # the same columns read as 18 heads of 64: a 64-wide head shares most of its products with the 72-wide
            # head it overlaps, so this moves the output by 13-14x the bound (H100, every variant), not 20x
            wrong, _ = fmha_reference_hd(q, k, v, D // 64, 64, 72 ** -0.5)
            self.separated("fmha (heads read 64 wide)", ref, wrong, bound, factor=FMHA_FACTOR / 4)
        self.rec["att"] = ret.reshape(self.M, D)

    def do_cross_q(self, l, args, kw, ret):
        w = self.W(l)
        self._rows_view(args[0], "xb")
        xb = self.rec["xb"] if self.rec["xb"].shape[0] == self.r1 - self.r0 else self.rec["xb"][self.r0:self.r1]
        ref, bound = self.gemm_check(ret, xb.double(), w["cq_w"], None)
        if l == SEP_L:
            wrong, _ = self.gemm_ref(xb.double(), self.W(l + 1)["cq_w"], None)
            self.separated("gemm (cross q of layer l + 1)", ref, wrong, bound)
        self.rec["q"] = ret

    def do_cross_attn(self, l, args, kw, ret):
        g0, g1 = self.g0, self.g1
        self._rows_view_e(args[0], "q")
        self._rows_view_e(kw["out"], "out")
        q = self.rec["q"].view(g1 - g0, self.T, self.E)
        k, v = self.kv[l]
        ref, bound = self.fmha_check(ret, q, k[g0:g1], v[g0:g1])
        if l == SEP_L:
            k1, v1 = self.kv[l + 1]
            wrong, _ = self.attn_ref(q, k1[g0:g1], v1[g0:g1])
            live = (v[g0:g1].abs().sum((1, 2)) > 0)[:, None, None]
            self.separated("fmha (K/V of layer l + 1)", ref, wrong, bound, live, factor=FMHA_FACTOR)
            o = [(b + 2) % B for b in range(g0, g1)]
            wrong, _ = self.attn_ref(q, k[o], v[o])
            self.separated("fmha (the other CFG half's context)", ref, wrong, bound, factor=FMHA_FACTOR)
        self.rec["att_c"] = ret.reshape(-1, self.E)

    def do_cross_out(self, l, args, kw, ret):
        w = self.W(l)
        self._rows_view_e(args[0], "att")
        ref, bound = self.gemm_check(ret, self.rec["att_c"].double(), w["co_w"], w["co_b"])
        if l == SEP_L:
            wrong, _ = self.gemm_ref(self.rec["att_c"].double(), self.W(l + 1)["co_w"], self.W(l + 1)["co_b"])
            self.separated("gemm (cross out of layer l + 1)", ref, wrong, bound)
        self.rec["val_cross"] = ret


def run_xl_audit(variant, dev, monkeypatch, xl_model, slip=None, graph=True):
    monkeypatch.setitem(dl._MODELS, "t23d", xl_model)
    monkeypatch.setattr(dl, "Audit", XLAudit)
    return dl.run_audit("t23d", "bf16", variant, dev, monkeypatch, slip=slip, graph=graph)


@pytest.mark.parametrize("variant", dl.VARIANTS + ["mod-row"])
def test_xl_launch_audit(dev, monkeypatch, xl_model, variant):
    audit = run_xl_audit(variant, dev, monkeypatch, xl_model)
    _report(audit, f"DiT-XL/2 width, depth {XL_DEPTH}, {variant}")
    kinds = {"gemm", "fmha (neighbouring sample's K/V)", "fmha (heads read 64 wide)", "residual update",
             "norm_modulate output", "patch_embed", "final_layer (unpatchify p and q swapped)",
             "timestep_embedding (cos and sin halves swapped)", "fmha (K/V of layer l + 1)",
             "fmha (the other CFG half's context)", "gemm (cross q of layer l + 1)", "gemm (cross out of layer l + 1)"}
    if variant in ("cond-zero", "zero-cond", "no-split", "mod-row"):
        kinds.add("residual update (rows shifted by one sample)")
    missing = kinds - set(audit.sep)
    assert not missing, f"check kinds without a separation assertion: {missing}"


@pytest.mark.parametrize("case,rewrite", [("kv-of-layer-l+1", dl._slip_next_layer_kv),
                                          ("cross-sub-batch-shifted", dl._slip_sub_batch)])
def test_xl_seeded_slip_is_caught(dev, monkeypatch, xl_model, case, rewrite):
    """Layer 1's cross-attention reading layer 2's K/V (2 E columns further in the cache), and the attended samples'
    K/V shifted by one sample: the audit fails at that launch and names it."""
    with pytest.raises(AssertionError) as e:
        run_xl_audit("cond-zero", dev, monkeypatch, xl_model, slip=("cross_attn", 1, rewrite), graph=False)
    msg = str(e.value)
    print(f"{case}: {msg[:400]}")
    assert "step cross_attn layer 1" in msg and "worst at index" in msg, msg
