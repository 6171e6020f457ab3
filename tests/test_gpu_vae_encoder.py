"""GPU: the stage-1 VAE encoder path -- ln3_downsample_nhwc and ln3_vae_posterior element by element against float64,
the mid-block transformer and its GEGLU, the whole MVEncoder against the reference's golden in both conv modes, and
`reconstruct` end to end against the oracle chain."""
import json
import os
import tempfile

import pytest
import torch
import torch.nn.functional as F

import vae_encoder_oracle as vo
from kernel_bounds import _posterior_tol, downsample_reference

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).norm() / b.norm())


def _pack(w):
    """Conv2d weight (Cout, Cin, 3, 3) -> the kernels' [9, Cin, Cout]."""
    return w.permute(2, 3, 1, 0).reshape(9, w.shape[1], w.shape[0]).contiguous()


def _golden_encoder(dev, golden, tf32: bool):
    from ln3diff_b200.utils import build_ae_encoder
    g = golden("vae_encoder.npz")
    enc = build_ae_encoder()
    enc.load_state_dict(vo.enc_state_dict(json.loads(str(g["encoder_shapes"]))))
    enc.conv_tf32 = tf32
    return enc.to(dev), g


def _golden_decoder(dev, arch="DiT2-S/2"):
    from ln3diff_b200.utils import build_ae_decoder
    dec = build_ae_decoder(arch)
    qw, qb = vo.quant_conv_params()
    dec.superresolution["quant_conv"].weight.data.copy_(qw)
    dec.superresolution["quant_conv"].bias.data.copy_(qb)
    return dec.to(dev)


# ------------------------------------------------------------------ ln3_downsample_nhwc
@pytest.mark.parametrize("N,H,W,Cin,Cout", [
    (1, 18, 34, 16, 32),      # ragged tiles: 9 x 17 outputs on 8 x 8 tiles
    (2, 16, 16, 32, 40),      # Cout tail: 32 + 8 channels
    (3, 22, 14, 10, 24),      # Cin = 10 (conv_in's count): one partial chunk
    (1, 12, 20, 24, 64),      # Cin not a multiple of 16
    (4, 256, 256, 64, 64),    # production: level 0 (per 4 views)
    (4, 128, 128, 128, 128),  # production: level 1
    (4, 64, 64, 256, 256),    # production: level 2
])
@pytest.mark.parametrize("tf32", [False, True])
def test_downsample_elementwise(dev, N, H, W, Cin, Cout, tf32):
    """Against F.conv2d(F.pad(x, (0,1,0,1)), stride=2) in float64, within kernel_bounds.downsample_reference's bound."""
    from ln3diff_b200 import ops
    g = torch.Generator().manual_seed(N * 1000 + H + Cin + Cout)
    x = torch.randn(N, H, W, Cin, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / (3 * Cin ** 0.5)
    b = 0.1 * torch.randn(Cout, generator=g)
    Ho, Wo = H // 2, W // 2
    n_out, pad = N * Ho * Wo * Cout, 4096
    buf = torch.full((n_out + 2 * pad,), float("nan"), device=dev)
    out = buf[pad:pad + n_out].view(N, Ho, Wo, Cout)
    xd, wd, bd = x.to(dev), _pack(w).to(dev), b.to(dev)
    ops.downsample_nhwc(xd, wd, bd, out=out, tf32=tf32)
    first = out.clone()
    ops.downsample_nhwc(xd, wd, bd, out=out, tf32=tf32)
    torch.cuda.synchronize()
    assert torch.equal(first, out)                                              # two launches bit-identical
    assert bool(buf[:pad].isnan().all()) and bool(buf[pad + n_out:].isnan().all())
    assert not bool(out.isnan().any())
    xc = x.to(dev, torch.float64).permute(0, 3, 1, 2)
    ref, tol = downsample_reference(x.to(dev), w.to(dev), b.to(dev), tf32)
    err = (out.double().permute(0, 3, 1, 2) - ref).abs()
    assert bool((err <= tol).all()), float((err / tol).max())
    # the pad is on the bottom / right only: a one-pixel shift of the input moves the result far beyond the bound
    # (by >= 100x the fp32 bound; the TF32 bound, 2^-10 T, sits only ~2^10 / sqrt(K) below a typical output)
    ref_shift = F.conv2d(F.pad(xc, (1, 0, 1, 0)), w.to(dev, torch.float64), b.to(dev, torch.float64), stride=2)
    assert float(((ref_shift - ref).abs() / tol).median()) > (10 if tf32 else 100)


# ------------------------------------------------------------------ ln3_vae_posterior
def test_vae_posterior_elementwise_and_channel_mapping(dev):
    from ln3diff_b200 import ops
    g = torch.Generator().manual_seed(51)
    B, S = 3, 32
    mom = 3 * torch.randn(B, 24, S, S, generator=g)
    qw, qb = vo.quant_conv_params()
    noise = torch.randn(B, 12, S, S, generator=g)
    mean, lv, z = ops.vae_posterior(mom.permute(0, 2, 3, 1).contiguous().to(dev), qw.reshape(24, 8).to(dev), qb.to(dev),
                                    noise.to(dev))
    _, _, zm = ops.vae_posterior(mom.permute(0, 2, 3, 1).contiguous().to(dev), qw.reshape(24, 8).to(dev), qb.to(dev))
    m64, lv64, z64 = vo.posterior(qw.double(), qb.double(), mom.double(), noise.double())
    tols = _posterior_tol(qw.double(), qb.double(), mom.double(), m64, lv64, z64, noise.double())
    for got, ref, tol in zip((mean, lv, z), (m64, lv64, z64), tols):
        err = (got.cpu().double() - ref).abs()
        assert bool((err <= tol).all()), float((err / tol).max())
    assert torch.equal(zm, mean)                                   # noise NULL: z = mean
    assert float(lv.abs().max()) <= 20.0 and float(lv.abs().max()) > 0.5   # the soft clamp is exercised
    # channel i*3 + n of the reference's reshape: a one-channel slip of the moments moves mean / logvar by >= 100x tol
    for slip in (1, -1):
        mom_s = torch.roll(mom.double(), slip, dims=1)
        ms, lvs, _ = vo.posterior(qw.double(), qb.double(), mom_s, noise.double())
        qs = F.conv2d(mom.double(), qw.double(), qb.double(), groups=3)
        ms2 = torch.roll(qs, slip, dims=1)[:, :12]                     # or a slip of the output channels
        for alt in (ms, ms2):
            assert float(((alt - m64).abs() / tols[0]).median()) > 100
        assert float(((lvs - lv64).abs() / tols[1]).median()) > 100


def test_vae_reparameterization_draws_cpu_noise_like_the_reference(dev):
    """Under one torch.manual_seed, the decoder's vae_reparameterization gives the z of the reference formula
    mean + std * torch.randn(mean.shape) (CPU generator), and posterior.sample() draws the same noise."""
    dec = _golden_decoder(dev)
    g = torch.Generator().manual_seed(52)
    mom = (2 * torch.randn(2, 24, 32, 32, generator=g)).to(dev)
    torch.manual_seed(123)
    ret = dec.vae_reparameterization(mom, True)
    post = ret["posterior"]
    assert set(ret) == {"normal_entropy", "latent_normalized", "latent_normalized_2Ddiffusion", "log_q_2Ddiffusion",
                        "log_q", "posterior"}
    assert ret["latent_normalized_2Ddiffusion"].shape == (2, 12, 32, 32) and ret["latent_normalized"].shape == (2, 3072, 4)
    assert post.mean.shape == (2, 4, 3, 1024)
    torch.manual_seed(123)
    noise = torch.randn(post.mean.shape).to(dev)
    ref = post.mean + post.std * noise
    z = ret["latent_normalized_2Ddiffusion"].reshape(ref.shape)
    # the kernel's expf and torch's exp may differ by a few ulps of std; products and sums by one ulp each
    tol = 8 * U * (ref.abs() + post.std * noise.abs())
    assert float(((z - ref).abs() / tol).max()) <= 1.0
    torch.manual_seed(123)
    assert float(((post.sample() - z).abs() / tol).max()) <= 1.0
    mode = dec.vae_reparameterization(mom, False)
    assert torch.equal(mode["latent_normalized_2Ddiffusion"].reshape(ref.shape), post.mean)
    # log_q divides by var (the reference's quirk), entropy from the clamped logvar
    lq = -0.5 * ((z - post.mean) / post.var) ** 2 - 0.5 * torch.log(torch.tensor(2 * torch.pi)) - post.logvar
    assert torch.allclose(ret["log_q"], lq)


# ------------------------------------------------------------------ mid block
def test_geglu_epilogue_elementwise(dev):
    """value * gelu_erf(gate) through the gated-residual epilogue, with bf16-exact operands so that only the fp32
    accumulation (<= (K + 2) 2^-24 T per GEMM) and the epilogue's erf-GELU (|err| <= 1e-6 |g|: the erfc fit of
    1.5e-7 plus the approximate rcp / ex2) separate the kernel from float64:
        |p - p64| <= |gelu(g)| tol_v + |v| (1.13 tol_g + 1e-6 |g|) + 2^-24 |p|       (gelu' <= 1.13)
    and the bf16 copy is the round-to-nearest of the fp32 product."""
    from ln3diff_b200.ldm.modules.diffusionmodules.model import MVEncoder
    g = torch.Generator().manual_seed(53)
    M, K, Nh = 1024, 512, 2048
    a = torch.randn(M, K, generator=g).bfloat16()
    wv, wg = ((torch.randn(Nh, K, generator=g) / K ** 0.5).bfloat16() for _ in range(2))
    bv, bg = (0.1 * torch.randn(Nh, generator=g) for _ in range(2))
    P = dict(ff_v=(wv.to(dev), bv.to(dev)), ff_g=(wg.to(dev), bg.to(dev)))
    prod, prod_bf = MVEncoder._geglu(a.to(dev), P)
    a64 = a.double()
    v, gt = a64 @ wv.double().T + bv.double(), a64 @ wg.double().T + bg.double()
    gelu = F.gelu(gt)
    p64 = v * gelu
    tol_v = (K + 2) * U * (a64.abs() @ wv.double().abs().T + bv.double().abs())
    tol_g = (K + 2) * U * (a64.abs() @ wg.double().abs().T + bg.double().abs())
    tol = gelu.abs() * tol_v + v.abs() * (1.13 * tol_g + 1e-6 * gt.abs()) + U * p64.abs() + 1e-30
    err = (prod.cpu().double() - p64).abs()
    assert bool((err <= tol).all()), float((err / tol).max())
    assert torch.equal(prod_bf.cpu(), prod.cpu().bfloat16())
    # value and gate halves are not swapped: the swapped product is far outside the bound
    assert float(((gt * F.gelu(v) - p64).abs() / tol).median()) > 100


def test_mid_block_transformer_vs_oracle(dev, golden):
    """SpatialTransformer3D on the GPU (bf16 GEMM operands, fp32 accumulate and residual stream) against the float64
    oracle.  Derived bf16 bound on the transformer branch (output - x_in): every GEMM rounds both operands to bf16
    (relative 2^-9 each), so each of the five GEMM stages in sequence (qkv, P.V, to_out, GEGLU in, ff out) contributes
    at most 2^-8 of its output's scale, and the softmax and the LayerNorms are computed in fp32: <= 5 * 2^-8 = 2e-2
    rel-L2 of the branch; rounding errors of random sign typically stay near a tenth of that."""
    enc, g = _golden_encoder(dev, golden, tf32=False)
    P = enc.prepare()
    gen = torch.Generator().manual_seed(54)
    h = torch.randn(8, 32, 32, 256, generator=gen)
    out = enc._spatial_transformer(h.to(dev), P["st"], 4)
    sd = {k: v.double().to(dev) for k, v in vo.enc_state_dict(json.loads(str(g["encoder_shapes"]))).items()}
    ref = vo.spatial_transformer3d(sd, "mid.attn_1.", h.to(dev).double().permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    branch, branch_ref = out.double() - h.to(dev).double(), ref - h.to(dev).double()
    e = _rel(branch, branch_ref)
    print(f"mid-block transformer branch rel-L2 vs float64: {e:.3e}")
    assert e < 2e-2, e
    # attn1 really mixes the 4 views of an object: running it per view (num_frames = 1) is far off
    per_view = enc._spatial_transformer(h.to(dev), P["st"], 1)
    assert _rel(per_view.double() - h.to(dev).double(), branch_ref) > 10 * e


# ------------------------------------------------------------------ the whole encoder
@pytest.mark.parametrize("tf32", [False, True])
def test_encoder_vs_reference_golden(dev, golden, tf32):
    """MVEncoder + posterior on 2 objects x 4 views at 256^2 against the reference's recorded fp32 output.
    Bound: the bf16 mid-block branch carries <= 2e-2 of its own scale (test above), and that branch is a fraction of the
    mid-block output; TF32 convs add per layer a relative error ~2^-11 sqrt(2) (operand rounding of random sign), over
    ~20 conv layers renormalised by GroupNorm ~20 * 7e-4 = 1.4e-2 in the worst case of aligned errors.  So: exact convs
    < 1e-2, TF32 convs < 2e-2; the measured values are printed."""
    from ln3diff_b200 import pipeline
    enc, g = _golden_encoder(dev, golden, tf32)
    dec = _golden_decoder(dev)
    x = vo.enc_inputs().to(dev)
    torch.manual_seed(vo.NOISE_SEED)
    ret = pipeline.encode_latents(enc, dec, x, sample_posterior=True)
    moments = enc(x)
    assert moments.shape == (2, 24, 32, 32) and moments.dtype == torch.float32
    e_m = _rel(moments, g["moments"])
    e_z = _rel(ret["latent_normalized_2Ddiffusion"][:1], g["z_obj0"])
    e_mean = _rel(ret["posterior"].mean[:1].reshape(1, 12, 32, 32), g["mean_obj0"])
    print(f"encoder ({'TF32' if tf32 else 'fp32'} convs) vs reference: moments rel-L2 {e_m:.3e}, mean {e_mean:.3e}, "
          f"z {e_z:.3e}")
    bound = 2e-2 if tf32 else 1e-2
    assert e_m < bound and e_z < bound and e_mean < bound, (e_m, e_mean, e_z)
    assert set(ret) == set(json.loads(str(g["ret_keys"])))
    # the objects differ, and the encoder is deterministic
    assert _rel(moments[0], moments[1]) > 0.1 and torch.equal(enc(x), moments)


def test_encoder_runs_the_new_kernels(dev, golden):
    """Which kernels one encode_latents call runs, and how many.

    The count is exact from the library's own launch counter: conv_in; 4 launches per res block (two GroupNorm
    statistics, two 3x3 convs) plus a 1x1 shortcut where the channel count changes (levels 1 and 2), over 4 levels and
    the 2 mid blocks; 3 Downsample convs; 15 for the mid-block transformer (GroupNorm, proj_in, 3 LayerNorms, qkv /
    attention / to_out twice, the GEGLU gate and value GEMMs, ff.net.2, proj_out); norm_out statistics, conv_out,
    fusion_layer and the posterior: 1 + 18 + 3 + 8 + 15 + 4 = 49.

    The kernel kinds come from torch.profiler over three calls.  In a process that has already run several profiling
    sessions, CUPTI drops activity records: on an H100, after the rest of the GPU suite, the trace of one call held 41 of
    the 49 library kernels that the launch counter saw.  A trace never invents a kernel, so the per-kind counts are upper
    bounds, every kind must appear at least once in three calls, and a complete trace must match them exactly."""
    from torch.profiler import ProfilerActivity, profile
    from ln3diff_b200 import _lib, pipeline
    enc, _ = _golden_encoder(dev, golden, tf32=True)
    dec = _golden_decoder(dev)
    x = vo.enc_inputs(1).to(dev)
    pipeline.encode_latents(enc, dec, x)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    pipeline.encode_latents(enc, dec, x)
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 == 49
    reps = 3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            pipeline.encode_latents(enc, dec, x)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            names = [e.get("name", "") for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    count = lambda *parts: sum(all(p in n for p in parts) for n in names)
    # per call: the three stride-2 Downsample convs on the TF32 instance (DOWN = true), 18 TF32 3x3 convs in all
    # (conv_in, 2 per res block, conv_out, fusion_layer and the Downsample convs), 7 GEMMs, 2 attentions, 1 posterior
    per_call = {("conv3x3_tf32_kernel", "true"): 3, ("conv3x3_tf32_kernel",): 18, ("gemm_bf16_kernel",): 7,
                ("fmha_fwd_kernel",): 2, ("vae_posterior_kernel",): 1}
    got = {k: count(*k) for k in per_call}
    print(f"library launches {reps} x 49, ln3 kernels in the trace {count('ln3::')}; per kind {got}")
    if count("ln3::") == reps * 49:
        assert got == {k: reps * v for k, v in per_call.items()}, names
    else:
        assert count("ln3::") < reps * 49
        assert all(1 <= got[k] <= reps * v for k, v in per_call.items()), (got, names)
    # TF32 mode runs no exact-fp32 3x3 conv, strided or not
    assert count("conv_nhwc_kernel", "true") == 0 and count("conv_nhwc_kernel", ", 3, false") == 0


# ------------------------------------------------------------------ end to end
def test_reconstruct_end_to_end_vs_oracle_chain(dev, golden):
    """reconstruct at render resolution 32: encoder -> posterior sample -> decode -> render, against the oracle chain
    (the encoder oracle in float64, the decoder and renderer oracles in fp32) with the same CPU-drawn posterior noise and
    explicit renderer noise, within the decoder path's pixel tolerance (3e-2 rel-L2: bf16 DiT2 features)."""
    from ln3diff_b200 import pipeline
    from oracle import decoder as odec
    from oracle import fixtures as fx
    from oracle import render as orender
    from ln3diff_b200.utils import build_ae_decoder
    enc, g = _golden_encoder(dev, golden, tf32=True)
    dec = build_ae_decoder(fx.DECODER_ARCH, image_size=32)
    qw, qb = vo.quant_conv_params()
    dec.superresolution["quant_conv"].weight.data.copy_(qw)
    dec.superresolution["quant_conv"].bias.data.copy_(qb)
    sd_dec = {k: v.clone() for k, v in dec.state_dict().items()}
    dec = dec.to(dev)
    x = vo.enc_inputs(1)
    cams = torch.from_numpy(golden("cameras.npz")["objv_eval_pose"])[[2, 9]]
    res, V = 32, 2
    gen = torch.Generator().manual_seed(56)
    nc, nf = torch.rand(V, res * res, 64, generator=gen), torch.rand(V, res * res, 64, generator=gen)
    torch.manual_seed(57)
    ret, out = pipeline.reconstruct(enc, dec, x.to(dev), cams.to(dev), resolution=res, noise=(nc.to(dev), nf.to(dev)))
    assert out["image_raw"].shape == (1, V, 3, res, res)
    assert {"normal_entropy", "latent_normalized", "latent_normalized_2Ddiffusion", "log_q_2Ddiffusion", "log_q",
            "posterior"} == set(ret)
    # oracle chain
    sd_enc = {k: v.double().to(dev) for k, v in vo.enc_state_dict(json.loads(str(g["encoder_shapes"]))).items()}
    with torch.no_grad():
        mom = vo.mv_encoder(sd_enc, x.to(dev).double()).cpu()
    torch.manual_seed(57)
    noise = torch.randn(1, 4, 3, 1024).reshape(1, 12, 32, 32)
    _, _, z = vo.posterior(qw.double(), qb.double(), mom, noise.double())
    assert _rel(ret["latent_normalized_2Ddiffusion"], z) < 2e-2
    with torch.no_grad():
        planes = odec.vae_decode(sd_dec, fx.DECODER_ARCH, z.float(), 1.0).reshape(3, 32, 128, 128)
    osg = tuple(sd_dec[f"triplane_decoder.decoder.net.{i}.{n}"] for i, n in ((0, "weight"), (0, "bias"), (2, "weight"),
                                                                              (2, "bias")))
    for v in range(V):
        ref = orender.render_view(planes, osg, cams[v], res, orender.OBJAVERSE_OPTS, nc[v], nf[v])
        e = _rel(out["image_raw"][0, v], ref["image_raw"])
        print(f"reconstruct view {v}: image rel-L2 {e:.3e}")
        assert e < 3e-2 and _rel(out["image_mask"][0, v], ref["image_mask"]) < 3e-2
