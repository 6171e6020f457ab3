"""GPU: the multi-view-to-3D (MV23D) path -- ln3_plucker_patchify element by element, the 9-channel DINOv2 conditioner
against transformers' port, the DiT-PixArt-MV-L/2 denoiser against the reference's golden, and mv_to_3d end to end."""
import json
import os
import random
import tempfile

import numpy as np
import pytest
import torch

import mv23d_oracle as mo

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).norm() / b.norm())


def _ulp_bf16(v: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |v| (8 significand bits): 2^(floor(log2|v|) - 7), floored at the smallest normal."""
    a = v.abs().double().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def _cams(N: int, bf16_valued: bool) -> torch.Tensor:
    """N camera rows cycling through the translated / rotated / skewed / identity-pose cameras of the oracle, each
    perturbed so that no two views are equal."""
    base = mo.ray_cameras()
    g = torch.Generator().manual_seed(N)
    c = base[torch.arange(N) % base.shape[0]].clone()
    c[:, [3, 7, 11]] += 0.1 * torch.randn(N, 3, generator=g)
    c[:, [16, 20]] *= 1 + 0.05 * torch.rand(N, 2, generator=g)
    return mo.bf16(c) if bf16_valued else c


def _run_patchify(dev, image, cams, ldo=1792, pad_rows=3):
    """The operand written into the middle of a NaN-filled buffer; returns (view, whole buffer, row offset)."""
    from ln3diff_b200 import ops
    N = image.shape[0]
    buf = torch.full(((N * 256 + 2 * pad_rows) * ldo,), float("nan"), device=dev, dtype=torch.bfloat16)
    out = buf[pad_rows * ldo:(pad_rows + N * 256) * ldo].view(N * 256, ldo)
    ops.plucker_patchify(image.to(dev), cams.to(dev), out=out)
    torch.cuda.synchronize()
    return out.cpu(), buf.cpu(), pad_rows * ldo


def _f32_emulation(image: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """The kernel's arithmetic step by step in IEEE fp32 (numpy rounds every operation; no FMA), with the release
    rounding points: the exact value each output element must hold."""
    f = np.float32
    c = c.numpy().astype(f)
    N = c.shape[0]
    ar = ((np.arange(224, dtype=f) + f(0.5)) / f(224)).astype(f)
    v, u = np.meshgrid(ar, ar, indexing="ij")
    bf = lambda x: torch.from_numpy(np.ascontiguousarray(x, dtype=f)).bfloat16().float().numpy()
    rays = np.empty((N, 6, 224, 224), dtype=f)
    for n in range(N):
        cn = c[n]
        a = (u - cn[18]) / cn[16]
        b = (v - cn[21]) / cn[20]
        nrm = np.sqrt((a * a + b * b) + f(1))
        e = [bf(a / nrm), bf(b / nrm), bf(f(1) / nrm)]
        d = []
        for i in range(3):
            r = [bf(cn[4 * i + j]) for j in range(3)]
            d.append(bf((r[0] * e[0] + r[1] * e[1]) + r[2] * e[2]))
        o = cn[[3, 7, 11]]
        rays[n, 0] = o[1] * d[2] - o[2] * d[1]
        rays[n, 1] = o[2] * d[0] - o[0] * d[2]
        rays[n, 2] = o[0] * d[1] - o[1] * d[0]
        rays[n, 3:] = np.stack(d)
    x = torch.cat([image, torch.from_numpy(rays)], 1)
    return mo.im2col(x).bfloat16()


@pytest.mark.parametrize("N", [1, 6, 7])
@pytest.mark.parametrize("bf16_cams", [False, True])
def test_plucker_patchify_elementwise(dev, N, bf16_cams):
    g = torch.Generator().manual_seed(100 + N)
    image = torch.randn(N, 3, 224, 224, generator=g) * 1.5
    cams = _cams(N, bf16_cams)
    out, buf, off = _run_patchify(dev, image, cams)
    # bytes outside the view are untouched (still NaN), every byte of the view is written
    assert bool(buf[:off].isnan().all()) and bool(buf[off + out.numel():].isnan().all())
    assert not bool(out.isnan().any())
    # padding columns [1764, 1792): exactly zero
    assert bool((out[:, 1764:] == 0).all())
    # RGB columns: the kernel's only operation is the round-to-nearest-even cast, so bit-identical to bf16(x)
    assert torch.equal(out[:, :588], mo.im2col(image).bfloat16())
    # every column bit-identical to the fp32 emulation of the same rounding order
    assert torch.equal(out[:, :1764], _f32_emulation(image, cams))
    # ray columns against float64 with the same rounding points.  d = bf16(R_b . e_b): the kernel's e_b can differ from
    # float64's by one bf16 ulp when fp32 dir (relative error <= 4 * 2^-24) falls next to a bf16 rounding boundary, its
    # fp32 3-term sum adds <= 2 * 2^-24 * sum|R e|, and the two final roundings may land one bf16 ulp apart:
    #   |d_k - d_64| <= ulp(d_64) + sum_j |R_ij| ulp(e_j) + 2^-23 sum_j |R_ij e_j|                 (tol_d)
    # o x d in fp32: two products and a difference (<= 2^-23 (|o_a d_b| + |o_b d_a|)), the d error above times |o|, and
    # the final rounding (one ulp of the result):
    #   |m_k - m_64| <= ulp(m_64) + |o_a| tol_d,b + |o_b| tol_d,a + 2^-23 (|o_a d_b| + |o_b d_a|)
    r = mo.plucker_rays_f64(cams.double())
    R, e, o, d, m = r["R"], r["e"], r["o"], r["d"], r["m"]
    tol_d = _ulp_bf16(d) + torch.einsum("nij,njhw->nihw", R.abs(), _ulp_bf16(e)) \
        + 2.0 ** -23 * torch.einsum("nij,njhw->nihw", R.abs(), e.abs())
    idx = [(1, 2), (2, 0), (0, 1)]
    tol_m = torch.stack([_ulp_bf16(m[:, k]) + o[:, a].abs() * tol_d[:, b] + o[:, b].abs() * tol_d[:, a]
                         + 2.0 ** -23 * (o[:, a] * d[:, b]).abs() + 2.0 ** -23 * (o[:, b] * d[:, a]).abs()
                         for k, (a, b) in enumerate(idx)], 1)
    got = out[:, 588:1764].double()
    ref = mo.im2col(torch.cat([m, d], 1))
    tol = mo.im2col(torch.cat([tol_m, tol_d], 1))
    assert bool(((got - ref).abs() <= tol).all()), float(((got - ref).abs() / tol).max())
    assert float((got == mo.bf16(ref)).double().mean()) > 0.99


def test_plucker_patchify_matches_torch_under_cuda_autocast(dev):
    """The rounding order in the header, checked against the reference's op sequence run by torch on the GPU under the
    engine's bf16 autocast (plucker_rays restates gen_rays / get_plucker_ray op for op) and the final `.to(bf16)`.
    Measured on an H100: 99.998 % of the ray elements bit-identical; the rest are pixels where cuBLAS rounded a
    partial sum of R . dir (up to 32 bf16 ulps of a nearly cancelling d, 136 of its cross product)."""
    N = 6
    cams = _cams(N, True)
    image = torch.zeros(N, 3, 224, 224)
    out, _, _ = _run_patchify(dev, image, cams)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        rays = mo.plucker_rays(cams.to(dev))
    ref = mo.im2col(rays.to(torch.bfloat16).float().cpu()).double()
    got = out[:, 588:1764].double()
    mcols, dcols = slice(0, 588), slice(588, 1176)
    ulps = ((got - ref).abs() / _ulp_bf16(ref)).nan_to_num(0)
    exact_m, exact_d = (float((got[:, s] == ref[:, s]).double().mean()) for s in (mcols, dcols))
    print(f"kernel vs torch CUDA bf16 autocast: rays dtype {rays.dtype}; bit-identical o x d {exact_m:.6f}, "
          f"d {exact_d:.6f}; max |diff| in bf16 ulps: o x d {float(ulps[:, mcols].max()):.2f}, "
          f"d {float(ulps[:, dcols].max()):.2f}")
    assert rays.dtype == torch.float32          # cat of the fp32 cross product with the bf16 d: promoted
    # Where they differ, cuBLAS's bf16 batched matmul did not round the 3-term sum once (torch allows reduced-precision
    # reductions for bf16 GEMMs): a partial sum rounded to bf16 moves d by at most one bf16 ulp of the largest partial
    # sum, <= 2^-8 sum_j |R_ij e_j|, on top of the final rounding.  The cross product inherits |o| times that.
    r = mo.plucker_rays_f64(cams.double())
    tol_d = _ulp_bf16(r["d"]) + 2.0 ** -8 * torch.einsum("nij,njhw->nihw", r["R"].abs(), r["e"].abs())
    o = r["o"]
    tol_m = torch.stack([_ulp_bf16(r["m"][:, k]) + o[:, a].abs() * tol_d[:, b] + o[:, b].abs() * tol_d[:, a]
                         for k, (a, b) in enumerate([(1, 2), (2, 0), (0, 1)])], 1)
    tol = mo.im2col(torch.cat([tol_m, tol_d], 1))
    assert bool(((got - ref).abs() <= tol).all()), float(((got - ref).abs() / tol).max())
    assert min(exact_m, exact_d) > 0.999


# ------------------------------------------------------------------ conditioner
def test_mv_conditioner_matches_transformers_port_and_general_conditioner(dev):
    from ln3diff_b200.sgm.modules.encoders.modules import FrozenDinov2ImageEmbedderMVPlucker, GeneralConditioner
    V, W = 3, 256
    hf, sd = mo.dinov2_reg9(depth=2, width=W)
    emb = FrozenDinov2ImageEmbedderMVPlucker(arch="vitb", device=dev, n_cond_frames=V, enable_bf16=True, aug_c=False,
                                             state_dict=sd)
    g = torch.Generator().manual_seed(6)
    img = torch.rand(1, V, 3, 224, 224, generator=g) * 2 - 1       # 224 input: the resize is the identity
    cams = _cams(V, False)[None]
    tokens = emb({"img": img.to(dev), "c": cams.to(dev)})
    assert tokens.shape == (1, V, 256, W) and tokens.dtype == torch.float32
    pix = emb.preprocess(img[0].to(dev)).cpu()
    r = mo.plucker_rays_f64(cams[0].double())
    x9 = torch.cat([pix, r["m"].float(), r["d"].float()], 1).bfloat16().float()   # the operand's bf16 values
    with torch.no_grad():
        ref = hf(pixel_values=x9).last_hidden_state[:, 5:]
    assert _rel(tokens[0], ref) < 1.5e-2
    # the rays matter: the same images with other cameras give other tokens
    t2 = emb({"img": img.to(dev), "c": _cams(V, True)[None].flip(1).to(dev)})
    assert _rel(t2, tokens) > 1e-2
    # GeneralConditioner, as sgm/configs/mv23d-plucker-clipl-compat-fm-lognorm-noclip.yaml builds it (aug_c on)
    emb.aug_c = True
    emb._emb_config = {"input_key": "img-c", "ucg_rate": 0.1}
    cond = GeneralConditioner([emb])
    cam_t = cams.clone().to(dev)
    random.seed(0)
    np.random.seed(0)
    c, uc = cond.get_unconditional_conditioning({"img-c": {"img": img.to(dev), "c": cam_t}},
                                                force_uc_zero_embeddings=["img-c"])
    assert c["concat"].shape == (1, V, 256, W) and float(uc["concat"].abs().max()) == 0.0
    assert bool(torch.isfinite(c["concat"]).all()) and emb.ucg_rate == 0.1
    assert not torch.equal(cam_t.cpu(), cams)                     # aug_c rotated the caller's cameras in place


# ------------------------------------------------------------------ denoiser
def _golden_model(dev):
    from ln3diff_b200.utils import build_mv23d
    m = build_mv23d(depth=mo.MV_DEPTH, hidden_size=mo.MV_HIDDEN, num_heads=mo.MV_HEADS)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    m.load_state_dict(mo.mv_state_dict(shapes, m.state_dict()["pos_embed"]))
    return m.to(dev)


def test_mv_denoiser_matches_reference_golden(dev, golden, monkeypatch):
    g = golden("mv23d.npz")
    m = _golden_model(dev)
    x, t, ctx = mo.mv_inputs()
    x, t, cd = x.to(dev), t.to(dev), {"concat": ctx["concat"].to(dev)}
    out = m(x, t, cd)
    assert out.dtype == torch.float32 and out.shape == (2, 12, 32, 32)
    assert _rel(out, g["out"]) < 2e-2
    assert _rel(m.forward_with_cfg(x, t, cd, 4.0), g["out_cfg"]) < 3e-2
    assert m._ctx_cache.value["rows"] == (0, 1)                  # the zero row takes the closed-form cross-attention
    # the replayed CUDA graph is bit-identical to the eager launch sequence
    monkeypatch.setenv("LN3_CUDA_GRAPH", "0")
    assert torch.equal(m(x, t, cd), out)
    # closed-form unconditional rows vs full attention over the all-zero tokens: the same function; the split residual
    # passes add the same fp32 terms in another order, which bf16 operands downstream amplify to ~1e-4
    monkeypatch.setenv("LN3_UNCOND_CLOSED_FORM", "0")
    full = _golden_model(dev)(x, t, {"concat": cd["concat"].clone()})
    assert _rel(full, out) < 2e-3


def test_mv_l2_full_size_runs_the_wgmma_kernels(dev, monkeypatch):
    """DiT-PixArt-MV-L/2 at B' = 8 (4 conditional + 4 zero rows) with 6 views (1536 context tokens)."""
    from torch.profiler import ProfilerActivity, profile
    from ln3diff_b200.utils import build_mv23d
    m = build_mv23d("DiT-PixArt-MV-L/2", device=dev)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(8, 12, 32, 32, generator=g).to(dev)
    ctx = torch.randn(8, 6, 256, 768, generator=g)
    ctx[4:] = 0
    cd = {"concat": ctx.to(dev)}
    t = torch.full((8,), 0.3, device=dev)
    out = m(x, t, cd)
    assert out.shape == (8, 12, 32, 32) and bool(torch.isfinite(out).all())
    monkeypatch.setenv("LN3_CUDA_GRAPH", "0")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m(x, t, cd)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    gemms = [e for e in events if "gemm_bf16_kernel" in e.get("name", "")]
    fmhas = [e for e in events if "fmha_fwd_kernel" in e.get("name", "")]
    assert len(gemms) >= 24 * 5 and {tuple(e["args"]["block"]) for e in gemms} == {(384, 1, 1)}
    assert len(fmhas) >= 24 * 2


# ------------------------------------------------------------------ end to end
def test_mv_to_3d_end_to_end_small(dev):
    """eval_cldm for 'img-c' at small size: the pipeline's latents equal sample_flow on a hand-built context (the
    conditioner's tokens repeated, zeros for the unconditional half), and the renders are finite."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.sgm.modules.encoders.modules import FrozenDinov2ImageEmbedderMVPlucker, GeneralConditioner
    from ln3diff_b200.utils import build_ae_decoder, build_mv23d, orbit_cameras
    V, W, S = 3, 256, 2
    emb = FrozenDinov2ImageEmbedderMVPlucker(arch="vitb", device=dev, n_cond_frames=V, enable_bf16=True, aug_c=False,
                                             random_init=True, width=W, depth=2, mlp_dim=4 * W, seed=3)
    emb._emb_config = {"input_key": "img-c", "ucg_rate": 0.1}
    cond = GeneralConditioner([emb])
    m = build_mv23d(depth=2, hidden_size=384, num_heads=6, context_dim=W, device=dev)
    dec = build_ae_decoder("DiT2-S/2", device=dev)
    g = torch.Generator().manual_seed(12)
    imgs = torch.rand(1, V, 3, 256, 256, generator=g) * 2 - 1
    mv_cams = orbit_cameras(V)[None]
    cams = orbit_cameras(30).to(dev)
    lat, out = pipeline.mv_to_3d(cond, m, dec, imgs, mv_cams, cams, num_samples=S, num_steps=4,
                                 sampling_method="euler", resolution=32)
    assert lat.shape == (S, 12, 32, 32) and out["image_raw"].shape == (S, 24, 3, 32, 32)
    assert bool(torch.isfinite(out["image_raw"]).all()) and bool(torch.isfinite(lat).all())
    emb.ucg_rate = 0.0                            # a direct call, outside get_unconditional_conditioning
    tok = emb({"img": imgs.to(dev), "c": mv_cams.to(dev)})
    c = {"concat": tok.repeat_interleave(S, 0)}
    uc = {"concat": torch.zeros_like(c["concat"])}
    lat2 = pipeline.sample_flow(m, c, uc, S, seed=42, num_steps=4, sampling_method="euler")
    assert torch.equal(lat, lat2)
    assert float((lat[0] - lat[1]).abs().max()) > 0.0             # same condition, different noise per sample
