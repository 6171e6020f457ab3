"""GPU (-m gpu): the fp8 GEMM precision of the DiT denoisers (DenoiserMixin.set_gemm_precision("fp8")) at full size:
T23D DiT-L/2, I23D DiT-PixArt-L/2 and MV23D DiT-PixArt-MV-L/2 with seeded weights.

fp8 is outside the reference's parity tolerance; what is checked here:
  * each fp8 GEMM of block 0 (qkv with the head-norm of PixArt, fc1 -> GELU -> fp8, fc2), on the operands the
    block's own launch sequence produces, against float64 on the dequantised operands, within the accumulation
    bound derived in test_gpu_gemm_fp8.py;
  * the whole forward against the bf16 forward on the same inputs: rel-L2 below REL_L2_MAX, fixed before any fp8 run.
    Justification: e4m3 keeps 3 mantissa bits, so one rounding moves a value by at most 2^-4 relative and, for
    values spread over a binade, by about 2^-4 / sqrt(12) = 1.8 % rms.  Each of the three GEMMs quantises two
    operands (about 2.5 % rms on its output) and 24 blocks add their contributions to the residual stream with
    independent errors, while the skip path and the bf16 GEMMs (proj, cross-attention) carry no fp8 error: the
    final layer's output should move by a few percent.  REL_L2_MAX = 0.1 leaves room for the attention softmax
    amplifying its logits' error and is still far below an unrelated output (rel-L2 about 1.4).
  * eager and CUDA-graph-replay fp8 forwards are bit-identical; switching back to bf16 reproduces the bf16 output
    bit for bit; the state_dict is untouched."""
import pytest
import torch

pytestmark = pytest.mark.gpu

FP8 = torch.float8_e4m3fn
REL_L2_MAX = 0.1
U_ACC = 2.0 ** -13


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _model_and_inputs(family, dev):
    from ln3diff_b200.utils import build_i23d, build_mv23d, build_t23d
    g = torch.Generator().manual_seed(61)
    if family == "t23d":
        m = build_t23d("DiT-L/2", device=dev)
        B = 16
        ctx = torch.randn(B, 77, 768, generator=g)
        ctx[B // 2:] = 0
        ctx = ctx.to(dev)
    elif family == "i23d":
        m = build_i23d("DiT-PixArt-L/2", device=dev)
        B = 8
        ctx = {"vector": torch.randn(B, 768, generator=g), "crossattn": torch.randn(B, 256, 2048, generator=g)}
        ctx = {k: v.to(dev) for k, v in ctx.items()}
    else:
        m = build_mv23d("DiT-PixArt-MV-L/2", device=dev)
        B = 8
        c = torch.randn(B, 6, 256, 768, generator=g)
        c[B // 2:] = 0
        ctx = {"concat": c.to(dev)}
    x = torch.randn(B, 12, 32, 32, generator=g).to(dev)
    t = (torch.rand(B, generator=g) * (900.0 if family == "t23d" else 1.0)).to(dev)
    return m, x, t, ctx


def _gemm_check(what, a_q, a_s, w_q, w_s, b, got, act=None):
    """got (bf16 or (codes, scales)) against float64 on the dequantised operands."""
    import math
    M, K = a_q.shape
    A = (a_q.double().view(M, K // 128, 128) * a_s.double()[:, :, None]).view(M, K)
    W = w_q.double() * w_s.double()[:, None]
    y = A @ W.T + b.double()
    E = 128 * U_ACC * (A.abs() @ W.abs().T) + (K // 128 + 2) * 2.0 ** -23 * ((A.abs() @ W.abs().T) + b.double().abs())
    if act == "gelu":
        y = 0.5 * y * (1 + torch.special.erf(y / math.sqrt(2)))
        E = 1.13 * E + 1.1e-5 + 3.2e-5 * y.abs()
    if isinstance(got, tuple):
        q, s = got
        deq = q.double() * s.double().repeat_interleave(128, dim=1)
        # dequantised within half an e4m3 ulp (2^-4 relative, or 2^-10 s below the normal range) of a value within E
        bound = E + torch.maximum((y.abs() + E) * 2.0 ** -4, s.double().repeat_interleave(128, dim=1) * 2.0 ** -10)
        err = (deq - y).abs()
    else:
        bound = E + (y.abs() + E) * 2.0 ** -8
        err = (got.double() - y).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max())
    assert ratio <= 1.0, f"{what}: max error / bound {ratio:.3f}"
    return ratio


def _block0_gemms(m, x, t, ctx):
    """Block 0's fp8 launch sequence by hand (norm1 -> qkv, fc1 -> fc2 on the same operand) with the model's fp8
    weights on a seeded residual stream, and a check of its three GEMMs."""
    from ln3diff_b200 import ops
    from ln3diff_b200.dit._denoiser import _pre_norm
    m.set_gemm_precision("fp8")
    P = m.prepare()
    W = P["blocks"][0]
    D = m.embed_dim
    g = torch.Generator(device=x.device).manual_seed(3)
    M = x.shape[0] * m.pos_embed.shape[1]
    x2 = torch.randn(M, D, device=x.device, generator=g) * 2
    mod = torch.randn(x.shape[0], 2 * D, device=x.device, generator=g) * 0.3
    a_q, a_s = ops.norm_modulate_fp8(x2, **_pre_norm(W, "n1_w"), shift=mod[:, :D], scale=mod[:, D:],
                                     mod_rows=m.pos_embed.shape[1])
    hn = W.get("qk_norm")
    qkv = ops.gemm_fp8(a_q, a_s, W["qkv_q"], W["qkv_s"], W["qkv_b"], head_norm=hn, head_norm_sec_cols=D)
    r = {}
    if hn is None:
        r["qkv"] = _gemm_check("qkv", a_q, a_s, W["qkv_q"], W["qkv_s"], W["qkv_b"], qkv)
    else:   # the v section carries no head norm: check it directly
        r["qkv_v"] = _gemm_check("qkv v", a_q, a_s, W["qkv_q"][2 * D:], W["qkv_s"][2 * D:], W["qkv_b"][2 * D:],
                                 qkv[:, 2 * D:])
    h_q, h_s = ops.gemm_fp8(a_q, a_s, W["fc1_q"], W["fc1_s"], W["fc1_b"], act=ops.ACT_GELU_ERF, out_kind=ops.OUT_FP8)
    r["fc1"] = _gemm_check("fc1", a_q, a_s, W["fc1_q"], W["fc1_s"], W["fc1_b"], (h_q, h_s), act="gelu")
    out = ops.gemm_fp8(h_q, h_s, W["fc2_q"], W["fc2_s"], W["fc2_b"])
    r["fc2"] = _gemm_check("fc2", h_q, h_s, W["fc2_q"], W["fc2_s"], W["fc2_b"], out)
    return r


@pytest.mark.parametrize("family", ["t23d", "i23d", "mv23d"])
def test_fp8_denoiser_forward(dev, family, monkeypatch):
    m, x, t, ctx = _model_and_inputs(family, dev)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    ref = m(x, t, ctx)                                          # bf16, graph replay
    assert m.set_gemm_precision("fp8") is m and m._prep is None and not m._graphs
    out = m(x, t, ctx)                                          # fp8, graph replay
    assert "qkv_q" in m._prep["blocks"][0] and m._prep["blocks"][0]["qkv_q"].dtype == FP8
    monkeypatch.setenv("LN3_CUDA_GRAPH", "0")
    eager = m(x, t, ctx)
    monkeypatch.delenv("LN3_CUDA_GRAPH")
    assert torch.equal(out, eager), "fp8 graph replay and eager forward differ"
    rel = _rel(out, ref)
    print(f"{family}: fp8 vs bf16 forward rel-L2 {rel:.4e}")
    assert bool(torch.isfinite(out).all()) and rel < REL_L2_MAX, rel
    ratios = _block0_gemms(m, x, t, ctx)
    print(f"{family}: block-0 fp8 GEMM max error / bound {ratios}")
    m.set_gemm_precision("bf16")
    assert torch.equal(m(x, t, ctx), ref), "bf16 after fp8 differs from the first bf16 forward"
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_fp8_t23d_sampler_runs_through_the_pipeline(dev):
    """pipeline.sample_t23d with the shared-modulation graph path, fp8 vs bf16 on the same noise (DiT-B/2)."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_t23d
    m = build_t23d("DiT-B/2", device=dev)
    g = torch.Generator().manual_seed(9)
    x0 = torch.randn(2, 12, 32, 32, generator=g).to(dev)
    c = {"crossattn": torch.randn(2, 77, 768, generator=g).to(dev)}
    uc = {"crossattn": torch.zeros(2, 77, 768, device=dev)}
    ref = pipeline.sample_t23d(m, x0, c, uc, 4, 6.5)
    m.set_gemm_precision("fp8")
    out = pipeline.sample_t23d(m, x0, c, uc, 4, 6.5)
    rel = _rel(out, ref)
    print(f"sample_t23d 4 steps DiT-B/2: fp8 vs bf16 rel-L2 {rel:.4e}")
    assert bool(torch.isfinite(out).all()) and rel < REL_L2_MAX


def test_fp8_unsupported_width_raises(dev):
    from ln3diff_b200.dit.dit_models_xformers import TextCondDiTBlock
    from ln3diff_b200.dit.dit_trilatent import DiT_TriLatent
    m = DiT_TriLatent(input_size=32, patch_size=2, in_channels=4, hidden_size=384, depth=1, num_heads=6, num_classes=0,
                      learn_sigma=False, context_dim=768, roll_out=True, vit_blk=TextCondDiTBlock).to(dev)
    m.set_gemm_precision("fp8")                      # embed_dim 384: not a multiple of 256
    with pytest.raises(RuntimeError, match="fp8 GEMM precision needs"):
        m(torch.zeros(1, 12, 32, 32, device=dev), torch.zeros(1, device=dev), torch.zeros(1, 77, 768, device=dev))
