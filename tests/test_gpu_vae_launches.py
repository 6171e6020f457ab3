"""GPU (-m gpu): every kernel launch of the VAE, element by element against float64 -- the DiT2 decoder and its conv_sr
upsampler, the MVEncoder and MVEncoderGSDynamicInp trunks with their mid-block transformer, fusion conv and view-mean
pooling, and the posterior.

The per-kernel tests check the arithmetic of each kernel; this file checks how the VAE's host code calls them: the
two alternating modulation buffers of the decoder and its deferred MLP residual, the in-plane / global attention
views, the token grouping of the encoder's attn1 / attn2, the folded LayerNorm affines, the GEGLU epilogue, the
view-major channel order of the fusion conv and the torch.chunk boundaries of the pooling.  The tracer of
launch_audit.py wraps the ops these modules call and hands every launch to an auditor that

  * matches it against the launch sequence written down from the model's definition: the op of every launch and
    their count;
  * recomputes what the launch should have written in float64 from the module's own parameters (bf16 GEMM weights,
    fp32 otherwise; the conv references carry the TF32 term when conv_tf32 is set) and the recorded outputs of the
    semantically preceding launches, never from the launch's own arguments.  Each check carries exactly one kernel's
    bound (kernel_bounds.py); the decoder's fp32 residual stream is held to <= 1 ulp and >= 99 % bit-exact, the
    encoder's (updated in a GEMM epilogue) to that GEMM's residual bound;
  * for every check kind, recomputes the reference once with a mapping deliberately slipped and asserts the slip
    moves the affected elements by >= 100x the bound (the median).  The TF32 conv and the attention bounds are
    themselves a sizeable share of |y|, so those kinds take a smaller factor, stated where it is defined.

Each audited entry point then runs a second time untraced and must give the same bits.  Seeded slips injected
through the tracer must make the audit fail, naming the step and the block or layer."""
from __future__ import annotations

import pytest
import torch

import kernel_bounds as kb
import vae_encoder_oracle as vo
from launch_audit import FMHA_FACTOR, Audit, Step, _report, traced

pytestmark = pytest.mark.gpu

TRACED = ("patch_embed_triplane", "gemm", "norm_modulate", "fmha", "conv_nhwc", "groupnorm_stats", "attn_single_head",
          "downsample_nhwc", "view_mean_nhwc", "vae_posterior")
SEP_L = 1             # the decoder block whose checks also run the separation (slipped-mapping) assertions
NORM_LAYER, ACT_GELU_ERF = 1, 1
# A TF32 conv's bound is 2^-10 sum|w x|, only ~2^10 / sqrt(K) below a typical output (K = 9 Cin terms): a wrong weight
# or channel order moves the output by 20-40x that bound at the VAE's channel counts, not 100x (the per-kernel tests
# use the same factor for the same reason).
TF32_FACTOR = 10.0
# The VAE attends over 256 to 6144 keys at once (an in-plane block over 256, a global block over 768, the encoder's
# attn1 over 4096 or 6144).  Under such diffuse attention y is a mean over that many keys while the 2^-8 term of the
# attention bound does not shrink with it: a wrong key set or grouping moved the output by 8.6-37x the bound on an H100
# 80GB HBM3, below even the denoiser's FMHA_FACTOR.  The attention kinds here take a quarter of it, as the denoiser's
# DINO kind does.
VAE_FMHA_FACTOR = FMHA_FACTOR / 4
IN_MUL = 0.96806      # the release scripts' triplane_scaling_divider, folded into the patch embed


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


# ------------------------------------------------------------------ models (seeded)
_MODELS = {}


def decoder(arch, dev):
    """The AE decoder with every weight key-seeded as oracle.fixtures.decoder_state_dict draws it: the adaLN weights
    are N(0, 1/D) there, so the gates are O(1) (derandomize_zero_init alone gives N(0, 0.02^2) and gates of ~1e-2)."""
    if arch not in _MODELS:
        from ln3diff_b200.utils import build_ae_decoder
        from oracle import fixtures as fx
        m = build_ae_decoder(arch)
        sd = m.state_dict()
        sd.update(fx.decoder_state_dict({k: tuple(v.shape) for k, v in sd.items()}))
        m.load_state_dict(sd)
        _MODELS[arch] = m.to(dev)
    return _MODELS[arch]


def encoder(kind, dev):
    """vae_encoder_oracle's seeded weights, with the transformer's LayerNorm affines widened to weight 1 + N(0, 1) and
    bias N(0, 1) (the seeding draws 1 + N(0, 0.1^2) and N(0, 0.1^2)): exchanging two LayerNorms' pairs must move the
    bf16 output by more than 100x half a bf16 ulp."""
    if kind not in _MODELS:
        from ln3diff_b200.utils import build_ae_encoder
        enc = build_ae_encoder(dino_version="mv-sd-dit" if kind == "mv" else "mv-sd-dit-dynaInp-trilatent")
        sd = vo.enc_state_dict({k: tuple(v.shape) for k, v in enc.state_dict().items()})
        for k in sd:
            if ".transformer_blocks.0.norm" in k:
                sd[k] = 1 + 10 * (sd[k] - 1) if k.endswith("weight") else 10 * sd[k]
        enc.load_state_dict(sd)
        _MODELS[kind] = enc.to(dev)
    return _MODELS[kind]


def posterior_decoder(dev):
    """A DiT2-S/2 decoder with vae_encoder_oracle's quant_conv: the posterior half of encode_latents."""
    if "post" not in _MODELS:
        from ln3diff_b200.utils import build_ae_decoder
        dec = build_ae_decoder("DiT2-S/2")
        qw, qb = vo.quant_conv_params()
        dec.superresolution["quant_conv"].weight.data.copy_(qw)
        dec.superresolution["quant_conv"].bias.data.copy_(qb)
        _MODELS["post"] = dec.to(dev)
    return _MODELS["post"]


def enc_inputs(n_views, res, seed):
    """(n_views, 10, res, res): RGB and Plücker channels in [-1, 1], depth in [0.5, 2]."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n_views, 10, res, res, generator=g) * 2 - 1
    x[:, 9] = 0.5 + 0.75 * (x[:, 9] + 1)
    return x


# ------------------------------------------------------------------ the launch sequences, from the model definitions
def res_steps(layer, rb):
    """ResnetBlock: norm1 -> swish -> conv1, [nin_shortcut], norm2 -> swish -> conv2 + shortcut."""
    s = [Step("groupnorm_stats", "gn1", layer), Step("conv_nhwc", "conv1", layer)]
    if hasattr(rb, "nin_shortcut"):
        s.append(Step("conv_nhwc", "nin", layer))
    return s + [Step("groupnorm_stats", "gn2", layer), Step("conv_nhwc", "conv2", layer)]


def decoder_launches(m):
    """PatchEmbedTriplane -> depth x DiT block (adaLN, norm1 with the previous block's gated MLP residual, qkv,
    attention, proj, gated residual + norm2, fc1, fc2) -> the last block's MLP residual -> conv_sr (ldm Decoder)."""
    vd, sr = m.vit_decoder, m.superresolution["conv_sr"]
    seq = [Step("patch_embed_triplane", "patch_embed", None)]
    for l in range(vd.depth):
        seq += [Step("gemm", "ada", l), Step("norm_modulate", "norm1", l), Step("gemm", "qkv", l),
                Step("fmha", "attn", l), Step("gemm", "proj", l), Step("norm_modulate", "norm2", l),
                Step("gemm", "fc1", l), Step("gemm", "fc2", l)]
    seq.append(Step("norm_modulate", "final_resid", None))
    seq.append(Step("conv_nhwc", "conv_in", "conv_in"))
    seq += res_steps("mid.block_1", sr.mid.block_1)
    seq += [Step("groupnorm_stats", "attn_gn", "mid.attn_1")] + [Step("conv_nhwc", f"attn_{n}", "mid.attn_1")
                                                                  for n in "qkv"]
    seq += [Step("attn_single_head", "attn_core", "mid.attn_1"), Step("conv_nhwc", "attn_out", "mid.attn_1")]
    seq += res_steps("mid.block_2", sr.mid.block_2)
    for lvl in reversed(range(len(sr.up))):
        for bi, rb in enumerate(sr.up[lvl].block):
            seq += res_steps(f"up.{lvl}.block.{bi}", rb)
        if hasattr(sr.up[lvl], "upsample"):
            seq.append(Step("conv_nhwc", "upsample", f"up.{lvl}.upsample"))
    return seq + [Step("groupnorm_stats", "norm_out", "norm_out"), Step("conv_nhwc", "conv_out", "conv_out")]


def encoder_launches(enc, n_views, pool_frames=None, posterior=False):
    """Encoder.forward: conv_in -> down levels (res blocks, Downsample) -> mid.block_1 -> SpatialTransformer3D
    (GroupNorm, proj_in, norm1 -> attn1 over an object's views, norm2 -> attn2 per view, norm3 -> GEGLU feed-forward,
    proj_out + x) -> mid.block_2 -> norm_out, swish, conv_out; then MVEncoder's fusion conv or MVEncoderGSDynamicInp's
    mean over each torch.chunk(N // num_frames) of the views (equal chunks of ceil(N / chunks), a shorter last one);
    then the posterior."""
    seq = [Step("conv_nhwc", "conv_in", "conv_in")]
    for i, d in enumerate(enc.down):
        for bi, rb in enumerate(d.block):
            seq += res_steps(f"down.{i}.block.{bi}", rb)
        if hasattr(d, "downsample"):
            seq.append(Step("downsample_nhwc", "downsample", f"down.{i}.downsample"))
    seq += res_steps("mid.block_1", enc.mid.block_1)
    st = "mid.attn_1"
    seq += [Step("groupnorm_stats", "st_gn", st), Step("conv_nhwc", "proj_in", st)]
    for j in (1, 2):
        seq += [Step("norm_modulate", f"ln{j}", st), Step("gemm", f"qkv{j}", st), Step("fmha", f"attn{j}", st),
                Step("gemm", f"to_out{j}", st)]
    seq += [Step("norm_modulate", "ln3", st), Step("gemm", "ff_gate", st), Step("gemm", "ff_value", st),
            Step("gemm", "ff_out", st), Step("conv_nhwc", "proj_out", st)]
    seq += res_steps("mid.block_2", enc.mid.block_2)
    seq += [Step("groupnorm_stats", "norm_out", "norm_out"), Step("conv_nhwc", "conv_out", "conv_out")]
    if hasattr(enc, "fusion_layer"):
        seq.append(Step("conv_nhwc", "fusion", "fusion_layer"))
    else:
        chunks = torch.arange(n_views).chunk(n_views // pool_frames)
        seq.append(Step("view_mean_nhwc", "pool", "chunks"))
        if chunks[-1].numel() != chunks[0].numel():
            seq.append(Step("view_mean_nhwc", "pool_tail", "chunks"))
    if posterior:
        seq.append(Step("vae_posterior", "posterior", "quant_conv"))
    return seq


# ------------------------------------------------------------------ the auditors
class ConvAudit(Audit):
    """The GEMM, conv, GroupNorm and single-head attention checks shared by the decoder and the encoder; `root` is the
    module the conv steps' layer paths resolve in."""

    def __init__(self, seq, root, tf32, dev):
        super().__init__(seq)
        self.root, self.tf32, self.dev = root, tf32, dev
        self.rec = {}

    def bf(self, p):
        return p.detach().to(self.dev, torch.bfloat16).double()

    def fp(self, p):
        return p.detach().to(self.dev, torch.float32).double()

    def mod_(self, layer):
        return self.root.get_submodule(layer)

    # ---- GEMM (bf16 operands, fp32 accumulation)
    @staticmethod
    def gemm_ref(a64, w, b64, act=0):
        y = a64 @ w.T
        if b64 is not None:
            y = y + b64
        tau = kb.gemm_tau(a64, w, b64)
        ref, act_err = kb.act_ref(act, y)
        return ref, (kb.SLOPE * tau + act_err if act else tau)

    def gemm_check(self, got, a64, w, b64, act=0, out="bf16", x0=None):
        ref, tol = self.gemm_ref(a64, w, b64, act)
        if out == "f32":
            bound = tol
        elif out == "resid":                       # x += val in the epilogue: one more fp32 rounding
            ref = x0 + ref
            bound = tol + kb.ulp(ref.abs() + tol, 23) / 2
        else:
            bound = kb.gemm_bf16_bound(ref, tol)
        self.within("output", got, ref, bound)
        return ref, bound

    def fmha_check(self, got, q, k, v, H):
        ref, tol = kb.fmha_reference(q, k, v, H, 64 ** -0.5, False)
        bound = kb.gemm_bf16_bound(ref, tol)
        self.within("attention", got.reshape(ref.shape), ref, bound)
        return ref, bound

    # ---- NHWC conv / GroupNorm
    def conv_ref(self, x, conv, ksize, gn=None, swish=False, res=None, up=False, w=None, b=None):
        sc, sh = gn if gn is not None else (None, None)
        w = conv.weight.float() if w is None else w
        b = conv.bias.float() if b is None else b
        return kb.conv_reference(x, w, b, ksize=ksize, up=up, sc=sc, sh=sh, swish=swish, res=res,
                                 tf32=self.tf32 and ksize == 3)

    def conv_check(self, got, x, conv, ksize, **kw):
        ref, tol = self.conv_ref(x, conv, ksize, **kw)
        self.within("output", got.permute(0, 3, 1, 2), ref, tol)
        return ref, tol

    def conv_factor(self, ksize):
        return TF32_FACTOR if self.tf32 and ksize == 3 else 100.0

    def gn_check(self, ret, x, norm):
        sc_r, sh_r, tol_sc, tol_sh, _, _ = kb.gn_reference(x, norm.weight.float(), norm.bias.float(), 32)
        self.within("scale", ret[0], sc_r, tol_sc)
        self.within("shift", ret[1], sh_r, tol_sh)
        # image n's statistics in image n's row
        self.separated("groupnorm_stats (the neighbouring image's statistics)", sc_r, sc_r.roll(1, 0), tol_sc)
        return ret

    # ---- ResnetBlock
    def do_gn1(self, layer, args, kw, ret):
        self.rec["blk_in"] = self.rec["h"]
        self.rec["gn"] = self.gn_check(ret, self.rec["h"], self.mod_(layer).norm1)

    def do_conv1(self, layer, args, kw, ret):
        rb = self.mod_(layer)
        ref, tol = self.conv_check(ret, self.rec["blk_in"], rb.conv1, 3, gn=self.rec["gn"], swish=True)
        if layer == "mid.block_2":
            other = self.mod_("mid.block_1").conv1
            wrong, _ = self.conv_ref(self.rec["blk_in"], rb.conv1, 3, gn=self.rec["gn"], swish=True,
                                     w=other.weight.float(), b=other.bias.float())
            self.separated("conv_nhwc (mid.block_1's weights for mid.block_2's)", ref, wrong, tol,
                           factor=self.conv_factor(3))
        self.rec["h1"] = ret

    def do_nin(self, layer, args, kw, ret):
        self.conv_check(ret, self.rec["blk_in"], self.mod_(layer).nin_shortcut, 1)
        self.rec["sc"] = ret

    def do_gn2(self, layer, args, kw, ret):
        self.rec["gn"] = self.gn_check(ret, self.rec["h1"], self.mod_(layer).norm2)

    def do_conv2(self, layer, args, kw, ret):
        res = self.rec.pop("sc", self.rec["blk_in"])
        self.conv_check(ret, self.rec["h1"], self.mod_(layer).conv2, 3, gn=self.rec["gn"], swish=True, res=res)
        self.rec["h"] = ret

    def do_norm_out(self, layer, args, kw, ret):
        self.rec["gn"] = self.gn_check(ret, self.rec["h"], self.mod_(layer))

    def do_conv_out(self, layer, args, kw, ret):
        self.conv_check(ret, self.rec["h"], self.mod_(layer), 3, gn=self.rec["gn"], swish=True)
        self.rec["h"] = ret


class DecoderAudit(ConvAudit):
    """decode_to_channels_last: PatchEmbedTriplane, the DiT2 blocks with per-token adaLN, then conv_sr."""

    def __init__(self, m, seq, latent, tf32, dev):
        super().__init__(seq, m.superresolution["conv_sr"], tf32, dev)
        self.m, self.vd, self.latent = m, m.vit_decoder, latent
        self.B = latent.shape[0]
        self.D, self.H, self.depth = self.vd.embed_dim, self.vd.num_heads, self.vd.depth
        self.T = 3 * m.token_size ** 2
        self.M = self.B * self.T
        self.idx = torch.arange(self.M, device=dev)          # mod_rows = 1: row r is modulated by its own token's row
        self.mods = {}
        self.xbuf = None
        self.gate_min = float("inf")

    def blk(self, l):
        return self.vd.blocks[l]

    def chunk(self, l, j):
        return self.mods[l][:, j * self.D:(j + 1) * self.D].double()

    def check_x(self, got, ref):
        """fp32 residual stream: at most 1 ulp (double-rounding ties only), bit-exact almost everywhere."""
        self.within("residual stream x", got, ref, kb.ulp_f32(ref))
        exact = float((got.double() == ref).double().mean())
        assert exact >= 0.99, f"step {self.step.kind} layer {self.step.layer}: only {exact:.4f} of x is bit-exact"

    def norm_out(self, got, xg, l, js):
        """bf16(LayerNorm(x) (1 + scale) + shift) with layer l's chunks js, per token."""
        y, tau = kb.nm_out_ref(xg, NORM_LAYER, 1e-6, 0, shift=self.chunk(l, js[0]), scale=self.chunk(l, js[1]),
                               mod_idx=self.idx)
        bound = kb.bf16_bound(y, tau)
        self.within("bf16 output", got, y, bound)
        if l == SEP_L:
            wrong, _ = kb.nm_out_ref(xg, NORM_LAYER, 1e-6, 0, shift=self.chunk(l, js[0] + 1),
                                     scale=self.chunk(l, js[1] + 1), mod_idx=self.idx)
            self.separated("norm_modulate output (mod chunks j + 1)", y, wrong, bound)

    def do_patch_embed(self, l, args, kw, ret):
        p = self.m.superresolution["ldm_upsample"].proj
        y, tol, silu, tol_s = kb.pet_reference(self.latent, p.weight.float(), p.bias.float(), IN_MUL)
        self.within("tokens", ret[0], y, tol)
        self.within("silu bf16", ret[1].float(), silu, tol_s)
        self.separated("patch_embed_triplane (objects shifted by one)", y, y.roll(1, 0), tol)
        self.rec["c"] = ret[1].view(self.M, self.D)

    def do_ada(self, l, args, kw, ret):
        lin = self.blk(l).adaLN_modulation[1]
        assert float((lin.weight != 0).double().mean()) > 0.999, f"block {l}: adaLN weights hold zeros"
        a = self.rec["c"].double()
        ref, bound = self.gemm_check(ret, a, self.bf(lin.weight), self.fp(lin.bias), out="f32")
        if l == SEP_L:
            nxt = self.blk(l + 1).adaLN_modulation[1]
            wrong, _ = self.gemm_ref(a, self.bf(nxt.weight), self.fp(nxt.bias))
            self.separated("gemm f32 (block l + 1's adaLN)", ref, wrong, bound)
        self.mods[l] = ret
        self.mods.pop(l - 2, None)
        gates = torch.cat([self.chunk(l, 2), self.chunk(l, 5)], 1)
        self.gate_min = min(self.gate_min, float(gates.abs().mean()))

    def do_norm1(self, l, args, kw, ret):
        if l == 0:
            self.xbuf = args[0]                     # the residual stream, updated in place from here on
            ref = self.fp(self.vd.pos_embed[0]).repeat(self.B, 1)
        else:
            x0, val = self.rec["x"].double(), self.rec["val_mlp"].double()
            ref = kb.nm_resid_ref(x0, val, self.chunk(l - 1, 5), self.idx)         # block l-1's gate_mlp
            if l == SEP_L + 1:
                wrong = kb.nm_resid_ref(x0, val, self.chunk(l, 5), self.idx)
                self.separated("residual update (block l's gate_mlp for block l-1's)", ref, wrong, kb.ulp_f32(ref))
                wrong = kb.nm_resid_ref(x0, val, self.chunk(l - 1, 4), self.idx)
                self.separated("residual update (mod chunk 5 - 1)", ref, wrong, kb.ulp_f32(ref))
        xg = self.xbuf.clone()
        self.check_x(xg, ref)
        self.norm_out(ret, xg.double(), l, (0, 1))
        self.rec["x"], self.rec["a"] = xg, ret

    def do_qkv(self, l, args, kw, ret):
        b, a = self.blk(l), self.rec["a"].double()
        ref, bound = self.gemm_check(ret, a, self.bf(b.attn.qkv.weight), self.fp(b.attn.qkv.bias))
        if l == SEP_L:
            n = self.blk(l + 1)
            wrong, _ = self.gemm_ref(a, self.bf(n.attn.qkv.weight), self.fp(n.attn.qkv.bias))
            self.separated("gemm (block l + 1's weights)", ref, wrong, bound)
        self.rec["qkv"] = ret

    def grouped(self, in_plane):
        """q, k, v of the block's tokens: in-plane blocks attend within each (object, plane), 'b (n l) c -> (b n) l c';
        the others over the 3 planes of an object."""
        G = 3 * self.B if in_plane else self.B
        D = self.D
        qkv = self.rec["qkv"].view(G, self.M // G, 3 * D)
        return qkv[:, :, :D], qkv[:, :, D:2 * D], qkv[:, :, 2 * D:]

    def do_attn(self, l, args, kw, ret):
        in_plane = l % 2 == 0
        q, k, v = self.grouped(in_plane)
        ref, bound = self.fmha_check(ret, q, k, v, self.H)
        flat = lambda t: t.reshape(self.M, self.D)
        if l in (0, 1):
            # the other grouping: a wrong query / key set for every token
            qo, ko, vo_ = self.grouped(not in_plane)
            wrong, _ = kb.fmha_reference(qo, ko, vo_, self.H, 0.125, False)
            what = "global grouping for an in-plane block" if in_plane else "in-plane grouping for a global block"
            self.separated(f"fmha ({what})", flat(ref), flat(wrong), flat(bound), factor=VAE_FMHA_FACTOR)
        if l == SEP_L:
            wrong, _ = kb.fmha_reference(q, k.roll(1, 0), v.roll(1, 0), self.H, 0.125, False)
            self.separated("fmha (the neighbouring object's K/V)", ref, wrong, bound, factor=VAE_FMHA_FACTOR)
        self.rec["att"] = ret.reshape(self.M, self.D)

    def do_proj(self, l, args, kw, ret):
        b, a = self.blk(l), self.rec["att"].double()
        ref, bound = self.gemm_check(ret, a, self.bf(b.attn.proj.weight), self.fp(b.attn.proj.bias))
        if l == SEP_L:
            n = self.blk(l + 1)
            wrong, _ = self.gemm_ref(a, self.bf(n.attn.proj.weight), self.fp(n.attn.proj.bias))
            self.separated("gemm (proj of block l + 1)", ref, wrong, bound)
        self.rec["val_attn"] = ret

    def do_norm2(self, l, args, kw, ret):
        x0, val = self.rec["x"].double(), self.rec["val_attn"].double()
        ref = kb.nm_resid_ref(x0, val, self.chunk(l, 2), self.idx)                  # gate_msa
        xg = self.xbuf.clone()
        self.check_x(xg, ref)
        if l == SEP_L:
            wrong = kb.nm_resid_ref(x0, val, self.chunk(l, 1), self.idx)
            self.separated("residual update (mod chunk 2 - 1)", ref, wrong, kb.ulp_f32(ref))
        self.norm_out(ret, xg.double(), l, (3, 4))
        self.rec["x"], self.rec["a"] = xg, ret

    def do_fc1(self, l, args, kw, ret):
        mlp = self.blk(l).mlp.mlp
        self.gemm_check(ret, self.rec["a"].double(), self.bf(mlp[0].weight), self.fp(mlp[1].bias), ACT_GELU_ERF)
        self.rec["h"] = ret

    def do_fc2(self, l, args, kw, ret):
        mlp, a = self.blk(l).mlp.mlp, self.rec["h"].double()
        ref, bound = self.gemm_check(ret, a, self.bf(mlp[2].weight), self.fp(mlp[3].bias))
        if l == SEP_L:
            n = self.blk(l + 1).mlp.mlp
            wrong, _ = self.gemm_ref(a, self.bf(n[2].weight), self.fp(n[3].bias))
            # fc2 sums K = 4 D products: its bound (K + 1) 2^-23 sum|a w| is ~1/30 of a typical |y| at D = 1024, so
            # a wrong block's weights move it by ~57x the bound there (DiT2-L/2 on an H100), not 100x
            self.separated("gemm (fc2 of block l + 1)", ref, wrong, bound, factor=20.0)
        self.rec["val_mlp"] = ret

    def do_final_resid(self, l, args, kw, ret):
        L = self.depth - 1
        ref = kb.nm_resid_ref(self.rec["x"].double(), self.rec["val_mlp"].double(), self.chunk(L, 5), self.idx)
        xg = self.xbuf.clone()
        self.check_x(xg, ref)
        ts = self.m.token_size
        self.rec["h"] = xg.view(3 * self.B, ts, ts, self.D)          # tokens (B, 3 16 16, D) are NHWC (3B, 16, 16, D)

    # ---- conv_sr
    def do_conv_in(self, layer, args, kw, ret):
        self.conv_check(ret, self.rec["h"], self.mod_(layer), 3)
        self.rec["h"] = ret

    def do_attn_gn(self, layer, args, kw, ret):
        self.rec["blk_in"] = self.rec["h"]
        self.rec["gn"] = self.gn_check(ret, self.rec["h"], self.mod_(layer).norm)

    def _attn_1x1(self, n, layer, ret):
        at = self.mod_(layer)
        x = self.rec["blk_in"]
        ref, tol = self.conv_check(ret, x, getattr(at, n), 1, gn=self.rec["gn"])
        if n == "q":
            wrong, _ = self.conv_ref(x, at.q, 1, gn=self.rec["gn"], w=at.k.weight.float(), b=at.k.bias.float())
            self.separated("conv_nhwc 1x1 (k's weights for q's)", ref, wrong, tol)
        self.rec[n] = ret

    def do_attn_q(self, layer, args, kw, ret):
        self._attn_1x1("q", layer, ret)

    def do_attn_k(self, layer, args, kw, ret):
        self._attn_1x1("k", layer, ret)

    def do_attn_v(self, layer, args, kw, ret):
        self._attn_1x1("v", layer, ret)

    def do_attn_core(self, layer, args, kw, ret):
        N, Hh, Ww, C = self.rec["q"].shape
        q, k, v = (self.rec[n].view(N, Hh * Ww, C) for n in "qkv")
        y, tol = kb.attn_reference(q, k, v)
        self.within("attention", ret.view(N, Hh * Ww, C), y, tol)
        wrong, _ = kb.attn_reference(q, k.roll(1, 0), v.roll(1, 0))
        self.separated("attn_single_head (the neighbouring image's K/V)", y, wrong, tol)
        self.rec["att"] = ret

    def do_attn_out(self, layer, args, kw, ret):
        self.conv_check(ret, self.rec["att"], self.mod_(layer).proj_out, 1, res=self.rec["blk_in"])
        self.rec["h"] = ret

    def do_upsample(self, layer, args, kw, ret):
        self.conv_check(ret, self.rec["h"], self.mod_(layer).conv, 3, up=True)
        self.rec["h"] = ret

    def do_conv_out(self, layer, args, kw, ret):
        super().do_conv_out(layer, args, kw, ret)
        self.rec["out"] = ret


class EncoderAudit(ConvAudit):
    """The encoder trunk, then the fusion conv or the view-mean pooling, then (encode_latents) the posterior."""

    def __init__(self, enc, seq, x, tf32, dev, pool_frames=None, post=None, noise=None):
        super().__init__(seq, enc, tf32, dev)
        self.enc, self.x_in = enc, x
        st = enc.mid.attn_1
        self.heads, self.inner = st.n_heads, st.n_heads * st.d_head
        self.F = enc.num_frames                              # attn1 groups the views by the module's num_frames
        self.pool_frames, self.post, self.noise = pool_frames, post, noise
        self.pooled = []

    def do_conv_in(self, layer, args, kw, ret):
        x = self.x_in.float().permute(0, 2, 3, 1).contiguous()
        self.conv_check(ret, x, self.mod_(layer), 3)
        self.rec["h"] = ret

    def do_downsample(self, layer, args, kw, ret):
        conv = self.mod_(layer).conv
        ref, tol = kb.downsample_reference(self.rec["h"], conv.weight.float(), conv.bias.float(), self.tf32)
        self.within("output", ret.permute(0, 3, 1, 2), ref, tol)
        self.rec["h"] = ret

    # ---- SpatialTransformer3D
    def tb(self):
        return self.enc.mid.attn_1.transformer_blocks[0]

    def do_st_gn(self, layer, args, kw, ret):
        self.rec["st_in"] = self.rec["h"]
        self.rec["gn"] = self.gn_check(ret, self.rec["h"], self.mod_(layer).norm)

    def do_proj_in(self, layer, args, kw, ret):
        self.conv_check(ret, self.rec["st_in"], self.mod_(layer).proj_in, 1, gn=self.rec["gn"])
        self.shape = ret.shape
        self.rec["xs"] = ret.view(-1, self.inner)                     # the fp32 residual stream (tokens, inner)

    def ln_ref(self, j):
        """LayerNorm(eps 1e-5) with norm_j's affine, as one modulation row: shift = bias, scale = weight - 1 (fp32)."""
        ln = getattr(self.tb(), f"norm{j}")
        xs = self.rec["xs"].double()
        zero = torch.zeros(xs.shape[0], dtype=torch.long, device=self.dev)
        return kb.nm_out_ref(xs, NORM_LAYER, 1e-5, 0, shift=self.fp(ln.bias)[None],
                             scale=kb.f32(self.fp(ln.weight) - 1)[None], mod_idx=zero)

    def _ln(self, j, ret):
        y, tau = self.ln_ref(j)
        bound = kb.bf16_bound(y, tau)
        self.within("bf16 output", ret, y, bound)
        o = j % 3 + 1
        self.separated(f"norm_modulate (ln{o}'s pair for ln{j}'s)", y, self.ln_ref(o)[0], bound)
        self.rec["a"] = ret

    def do_ln1(self, layer, args, kw, ret):
        self._ln(1, ret)

    def do_ln2(self, layer, args, kw, ret):
        self._ln(2, ret)

    def do_ln3(self, layer, args, kw, ret):
        self._ln(3, ret)

    def qkv_w(self, j):
        at = getattr(self.tb(), f"attn{j}")
        return self.bf(torch.cat([at.to_q.weight, at.to_k.weight, at.to_v.weight], 0))

    def _qkv(self, j, ret):
        a = self.rec["a"].double()
        ref, bound = self.gemm_check(ret, a, self.qkv_w(j), None)
        if j == 1:
            wrong, _ = self.gemm_ref(a, self.qkv_w(2), None)
            self.separated("gemm (attn2's to_q/k/v for attn1's)", ref, wrong, bound)
        self.rec["qkv"] = ret

    def do_qkv1(self, layer, args, kw, ret):
        self._qkv(1, ret)

    def do_qkv2(self, layer, args, kw, ret):
        self._qkv(2, ret)

    def grouped(self, groups):
        rows, i = self.rec["qkv"].shape[0], self.inner
        qkv = self.rec["qkv"].view(groups, rows // groups, 3 * i)
        return qkv[:, :, :i], qkv[:, :, i:2 * i], qkv[:, :, 2 * i:]

    def _attn(self, j, ret):
        """attn1: the tokens of all views of one object, '(b f) l c -> b (f l) c'; attn2: each view's own tokens."""
        N = self.shape[0]
        groups = N // self.F if j == 1 else N
        q, k, v = self.grouped(groups)
        ref, bound = self.fmha_check(ret, q, k, v, self.heads)
        flat = lambda t: t.reshape(-1, self.inner)
        wrong, _ = kb.fmha_reference(q, k.roll(1, 0), v.roll(1, 0), self.heads, 0.125, False)
        self.separated(f"fmha attn{j} (the neighbouring {'object' if j == 1 else 'view'}'s K/V)", ref, wrong, bound,
                       factor=VAE_FMHA_FACTOR)
        if j == 1:
            qv, kv, vv = self.grouped(N)
            wrong, _ = kb.fmha_reference(qv, kv, vv, self.heads, 0.125, False)
            self.separated("fmha attn1 (grouped per view instead of per object)", flat(ref), flat(wrong), flat(bound),
                           factor=VAE_FMHA_FACTOR)
        self.rec["att"] = ret.reshape(-1, self.inner)

    def do_attn1(self, layer, args, kw, ret):
        self._attn(1, ret)

    def do_attn2(self, layer, args, kw, ret):
        self._attn(2, ret)

    def _to_out(self, j, ret):
        """x += to_out(attention), in the GEMM's OUT_RESID_F32 epilogue."""
        o = getattr(self.tb(), f"attn{j}").to_out[0]
        a, x0 = self.rec["att"].double(), self.rec["xs"].double()
        ref, bound = self.gemm_check(ret, a, self.bf(o.weight), self.fp(o.bias), out="resid", x0=x0)
        if j == 1:
            o2 = self.tb().attn2.to_out[0]
            wrong = x0 + self.gemm_ref(a, self.bf(o2.weight), self.fp(o2.bias))[0]
            self.separated("gemm resid (attn2's to_out for attn1's)", ref, wrong, bound)
        self.rec["xs"] = ret

    def do_to_out1(self, layer, args, kw, ret):
        self._to_out(1, ret)

    def do_to_out2(self, layer, args, kw, ret):
        self._to_out(2, ret)

    def geglu_w(self, half):
        """GEGLU: proj(x).chunk(2, -1) = (value, gate): value rows [0, 4 inner), gate rows after them."""
        p, n = self.tb().ff.net[0].proj, 4 * self.inner
        s = slice(0, n) if half == "value" else slice(n, 2 * n)
        return self.bf(p.weight[s]), self.fp(p.bias[s])

    def do_ff_gate(self, layer, args, kw, ret):
        a = self.rec["a"].double()
        ref, bound = self.gemm_check(ret, a, *self.geglu_w("gate"), ACT_GELU_ERF, out="f32")
        wrong, _ = self.gemm_ref(a, *self.geglu_w("value"), ACT_GELU_ERF)
        self.separated("gemm f32 gelu (GEGLU value half for the gate half)", ref, wrong, bound)
        self.rec["gate"] = ret

    def do_ff_value(self, layer, args, kw, ret):
        """prod = 0 + gate * value: the gated-residual epilogue onto zeros, one fp32 rounding of the product of the
        recorded gate and the value GEMM; its bf16 copy (out2) is that product rounded to nearest."""
        a, g = self.rec["a"].double(), self.rec["gate"].double()
        y, tau = self.gemm_ref(a, *self.geglu_w("value"))
        ref = g * y
        bound = g.abs() * tau + kb.ulp(ref.abs() + g.abs() * tau, 23) / 2
        self.within("gate * value", ret, ref, bound)
        self.separated("gemm gated resid (the neighbouring token's gate)", ref, g.roll(1, 0) * y, bound)
        assert torch.equal(kw["out2"], ret.to(torch.bfloat16)), "GEGLU bf16 copy differs from bf16(gate * value)"
        self.rec["prod_bf"] = kw["out2"].clone()

    def do_ff_out(self, layer, args, kw, ret):
        o = self.tb().ff.net[2]
        self.gemm_check(ret, self.rec["prod_bf"].double(), self.bf(o.weight), self.fp(o.bias), out="resid",
                        x0=self.rec["xs"].double())
        self.rec["xs"] = ret

    def do_proj_out(self, layer, args, kw, ret):
        self.conv_check(ret, self.rec["xs"].view(self.shape), self.mod_(layer).proj_out, 1, res=self.rec["st_in"])
        self.rec["h"] = ret

    # ---- fusion / pooling / posterior
    def do_fusion(self, layer, args, kw, ret):
        """fusion_layer(cat(feat.chunk(F), dim=1)) per object: input channel v Z + c is channel c of view v."""
        h = self.rec["h"]
        N, S, _, Z = h.shape
        F_ = self.F
        v = h.view(N // F_, F_, S, S, Z)
        fused = v.permute(0, 2, 3, 1, 4).reshape(N // F_, S, S, F_ * Z)
        conv = self.mod_(layer)
        ref, tol = self.conv_check(ret, fused, conv, 3)
        wrong, _ = self.conv_ref(v.permute(0, 2, 3, 4, 1).reshape(N // F_, S, S, F_ * Z).contiguous(), conv, 3)
        self.separated("conv_nhwc (fusion channels in c F + v order)", ref, wrong, tol, factor=self.conv_factor(3))
        self.rec["mom"] = ret

    def _pool(self, ret, tail):
        h = self.rec["h"]
        chunks = h.chunk(h.shape[0] // self.pool_frames)
        sel = [c for c in chunks if (c.shape[0] != chunks[0].shape[0]) == tail]
        xv = torch.stack(sel)
        ref, tol = xv.double().mean(1), kb.view_mean_tol(xv)
        self.within("view mean", ret, ref, tol)
        # the chunk boundaries one view later
        size = chunks[0].shape[0]
        hr = h.roll(-1, 0)
        first = 0 if not tail else size * (len(chunks) - 1)
        wrong = torch.stack([hr[first + i * size:first + i * size + c.shape[0]].double().mean(0)
                             for i, c in enumerate(sel)])
        self.separated("view_mean_nhwc (torch.chunk boundary one view off)", ref, wrong, tol)
        self.pooled.append(ret)
        self.rec["mom"] = torch.cat(self.pooled)

    def do_pool(self, layer, args, kw, ret):
        self._pool(ret, False)

    def do_pool_tail(self, layer, args, kw, ret):
        self._pool(ret, True)

    def do_posterior(self, layer, args, kw, ret):
        """quant_conv (groups 3) of the encoder's moments, the soft-clamped logvar and z = mean + std noise, the noise
        the CPU generator's randn(B, 12, S, S) after the caller's seed."""
        qc = self.post.superresolution["quant_conv"]
        qw, qb = self.fp(qc.weight), self.fp(qc.bias)
        mom = self.rec["mom"].double().permute(0, 3, 1, 2)
        noise = self.noise.to(self.dev).double() if self.noise is not None else torch.zeros_like(mom[:, :12])
        m64, lv64, z64 = vo.posterior(qw, qb, mom, noise if self.noise is not None else None)
        tols = kb._posterior_tol(qw, qb, mom, m64, lv64, z64, noise)
        for what, got, ref, tol in zip(("mean", "logvar", "z"), ret, (m64, lv64, z64), tols):
            self.within(what, got, ref, tol)
        wrong, _, _ = vo.posterior(qw, qb, mom.roll(1, 1))
        self.separated("vae_posterior (moments one channel over)", m64, wrong, tols[0])
        self.separated("vae_posterior (objects shifted by one)", m64, m64.roll(1, 0), tols[0])
        self.rec["z"] = ret[2]


# ------------------------------------------------------------------ audited runs
def run_decoder(arch, B, tf32, dev, monkeypatch, slip=None):
    m = decoder(arch, dev)
    lat = torch.randn(B, 12, 32, 32, generator=torch.Generator().manual_seed(40 + B)).to(dev)
    seq = decoder_launches(m)
    audit = DecoderAudit(m, seq, lat, tf32, dev)
    m.conv_tf32 = tf32
    try:
        with torch.no_grad(), traced(audit, monkeypatch, TRACED, slip):
            out = m.decode_to_channels_last(lat, IN_MUL)
        assert audit.n_checked == audit.n_traced == len(seq), (audit.n_checked, audit.n_traced, len(seq))
        assert torch.equal(out.view(audit.rec["out"].shape), audit.rec["out"])
        assert torch.equal(m.decode_to_channels_last(lat, IN_MUL), out), "a second decode gives other bits"
    finally:
        m.conv_tf32 = True
    # the adaLN gates are O(1): a gate from the wrong block or chunk is an O(1) change
    assert audit.gate_min > 0.05, audit.gate_min
    return audit


def run_encoder(kind, n_views, res, dev, monkeypatch, num_frames=None, sample_posterior=None, slip=None):
    """kind 'mv' (MVEncoder) or 'xl' (MVEncoderGSDynamicInp); sample_posterior None enters through the encoder's
    forward, True / False through pipeline.encode_latents."""
    from ln3diff_b200 import pipeline
    enc = encoder(kind, dev)
    x = enc_inputs(n_views, res, seed=70 + n_views).to(dev)
    pool = None if kind == "mv" else (num_frames or enc.num_frames)
    post = posterior_decoder(dev) if sample_posterior is not None else None
    noise = None
    if sample_posterior:
        noise = torch.randn(n_views // enc.num_frames, 12, res // 8, res // 8,
                            generator=torch.Generator().manual_seed(71))
    seq = encoder_launches(enc, n_views, pool, posterior=post is not None)
    audit = EncoderAudit(enc, seq, x, enc.conv_tf32, dev, pool, post, noise)

    def call():
        if post is None:
            return enc(x, num_frames) if num_frames is not None else enc(x)
        torch.manual_seed(71)
        return pipeline.encode_latents(enc, post, x, sample_posterior=sample_posterior)["latent_normalized_2Ddiffusion"]

    with torch.no_grad(), traced(audit, monkeypatch, TRACED, slip):
        out = call()
    assert audit.n_checked == audit.n_traced == len(seq), (audit.n_checked, audit.n_traced, len(seq))
    if post is None:
        assert torch.equal(out, audit.rec["mom"].permute(0, 3, 1, 2))
    else:
        assert torch.equal(out, audit.rec["z"])
    assert torch.equal(call(), out), "a second run gives other bits"
    return audit


# ------------------------------------------------------------------ the audits
DEC_KINDS = {"patch_embed_triplane (objects shifted by one)", "gemm f32 (block l + 1's adaLN)",
             "residual update (block l's gate_mlp for block l-1's)", "residual update (mod chunk 5 - 1)",
             "residual update (mod chunk 2 - 1)", "norm_modulate output (mod chunks j + 1)",
             "gemm (block l + 1's weights)", "gemm (proj of block l + 1)", "gemm (fc2 of block l + 1)",
             "fmha (global grouping for an in-plane block)", "fmha (in-plane grouping for a global block)",
             "fmha (the neighbouring object's K/V)", "groupnorm_stats (the neighbouring image's statistics)",
             "conv_nhwc (mid.block_1's weights for mid.block_2's)", "conv_nhwc 1x1 (k's weights for q's)",
             "attn_single_head (the neighbouring image's K/V)"}
ENC_KINDS = {"groupnorm_stats (the neighbouring image's statistics)",
             "conv_nhwc (mid.block_1's weights for mid.block_2's)", "norm_modulate (ln2's pair for ln1's)",
             "norm_modulate (ln3's pair for ln2's)", "norm_modulate (ln1's pair for ln3's)",
             "gemm (attn2's to_q/k/v for attn1's)", "fmha attn1 (the neighbouring object's K/V)",
             "fmha attn1 (grouped per view instead of per object)", "fmha attn2 (the neighbouring view's K/V)",
             "gemm resid (attn2's to_out for attn1's)", "gemm f32 gelu (GEGLU value half for the gate half)",
             "gemm gated resid (the neighbouring token's gate)"}


def _kinds_separated(audit, kinds):
    missing = kinds - set(audit.sep)
    assert not missing, f"check kinds without a separation assertion: {missing}"


@pytest.mark.parametrize("arch,B,tf32", [("DiT2-L/2", 2, True), ("DiT2-L/2", 2, False), ("DiT2-S/2", 3, True)],
                         ids=["L2-B2-tf32", "L2-B2-fp32", "S2-B3-tf32"])
def test_decoder_launch_audit(dev, monkeypatch, arch, B, tf32):
    audit = run_decoder(arch, B, tf32, dev, monkeypatch)
    _report(audit, f"decoder {arch} B={B} conv_tf32={tf32}")
    _kinds_separated(audit, DEC_KINDS)


@pytest.mark.parametrize("kind,n_views,res,num_frames,sample_posterior", [
    ("mv", 8, 256, None, True),            # 2 objects x 4 views, encode_latents with a posterior sample
    ("xl", 12, 256, None, False),          # 2 objects x 6 views, encode_latents with the posterior mode
    ("xl", 30, 64, 7, None),               # 5 objects x 6 views; pooling chunks of 8, 8, 8 and 6
], ids=["mv-2x4-256-sample", "xl-2x6-256-mode", "xl-30v-64-nf7"])
def test_encoder_launch_audit(dev, monkeypatch, kind, n_views, res, num_frames, sample_posterior):
    audit = run_encoder(kind, n_views, res, dev, monkeypatch, num_frames, sample_posterior)
    _report(audit, f"encoder {kind} {n_views} views {res}^2 num_frames={num_frames} posterior={sample_posterior}")
    kinds = set(ENC_KINDS)
    if kind == "mv":
        kinds.add("conv_nhwc (fusion channels in c F + v order)")
    else:
        kinds.add("view_mean_nhwc (torch.chunk boundary one view off)")
    if sample_posterior is not None:
        kinds |= {"vae_posterior (moments one channel over)", "vae_posterior (objects shifted by one)"}
    _kinds_separated(audit, kinds)
    if num_frames == 7:
        assert [s.kind for s in audit.seq[-2:]] == ["pool", "pool_tail"]


# ------------------------------------------------------------------ seeded slips: the audit must catch them
def _shift(t, elems):
    return t.as_strided(t.shape, t.stride(), t.storage_offset() + elems)


def _slip_own_gate(args, kw):                 # block l's gate_mlp (chunk 5 of its own modulation) for block l-1's
    kw["resid_gate"] = _shift(kw["shift"], 5 * kw["shift"].shape[1])
    return args, kw


def _slip_global_view(args, kw):              # an in-plane block's attention on the (B, T) view of the same buffers
    def glob(t):
        return t.as_strided((t.shape[0] // 3, 3 * t.shape[1], t.shape[2]), (3 * t.stride(0), t.stride(1), 1),
                            t.storage_offset())
    args[0], args[1], args[2] = glob(args[0]), glob(args[1]), glob(args[2])
    kw["out"] = glob(kw["out"])
    return args, kw


def _slip_block1_weights(enc):                # mid.block_2's conv1 with mid.block_1's packed weights
    def f(args, kw):
        args[1], args[2] = enc._prep["mid1"]["c1"]
        return args, kw
    return f


def _slip_attn1_view(tokens_per_view):        # attn1's K/V taken one view later (a copy, rolled over the tokens)
    def f(args, kw):
        for i in (1, 2):
            t = args[i]
            args[i] = t.reshape(-1, t.shape[2]).roll(-tokens_per_view, 0).view(t.shape)
        return args, kw
    return f


def _slip_fusion_transposed(views):           # the fusion conv's input in c F + v channel order
    def f(args, kw):
        x = args[0]
        B, S, _, FZ = x.shape
        args[0] = x.view(B, S, S, views, FZ // views).transpose(3, 4).reshape(x.shape).contiguous()
        return args, kw
    return f


SLIPS = ["dec-block5-own-gate", "dec-inplane-on-global-view", "enc-mid2-block1-weights", "enc-attn1-view-shift",
         "enc-fusion-transposed"]


@pytest.mark.parametrize("case", SLIPS)
def test_seeded_slip_is_caught(dev, monkeypatch, case):
    with pytest.raises(AssertionError) as e:
        if case == "dec-block5-own-gate":
            named = "norm1 layer 5"
            run_decoder("DiT2-S/2", 3, True, dev, monkeypatch, slip=("norm1", 5, _slip_own_gate))
        elif case == "dec-inplane-on-global-view":
            named = "attn layer 2"
            run_decoder("DiT2-S/2", 3, True, dev, monkeypatch, slip=("attn", 2, _slip_global_view))
        elif case == "enc-mid2-block1-weights":
            named = "conv1 layer mid.block_2"
            enc = encoder("xl", dev)
            run_encoder("xl", 30, 64, dev, monkeypatch, 7,
                        slip=("conv1", "mid.block_2", _slip_block1_weights(enc)))
        elif case == "enc-attn1-view-shift":
            named = "attn1 layer mid.attn_1"
            run_encoder("xl", 30, 64, dev, monkeypatch, 7, slip=("attn1", "mid.attn_1", _slip_attn1_view(8 * 8)))
        else:
            named = "fusion layer fusion_layer"
            run_encoder("mv", 8, 64, dev, monkeypatch, slip=("fusion", "fusion_layer", _slip_fusion_transposed(4)))
    msg = str(e.value)
    print(f"{case}: {msg[:400]}")
    assert f"step {named}" in msg and "worst at index" in msg, msg
