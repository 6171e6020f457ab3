"""GPU (-m gpu): oracle comparisons at the sizes bench.py runs (DiT-L/2 denoiser forward, DiT2-L/2 VAE decode),
and the measured latents -> pixels error next to the error of the reference's OWN GPU arithmetic (its modules
under bf16 autocast, restated by the oracle run on the GPU).  The measured numbers are written to
ln3_parity.json in $LN3_PARITY_DIR (default: the system temporary directory), never into the source tree.

Tolerances: one bf16 tensor-core forward <= 2e-2 rel-L2 against the fp32 oracle (section 8 / north_star: bf16
compute); rendered pixels 1e-3 from identical TRI-PLANES (tests/test_gpu_parity.py); from identical LATENTS the
pixels inherit the bf16 decoder's error, bounded here by 1.5x the error the reference's own bf16-autocast path makes
on the same latent."""
import json
import os
import tempfile
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _record(**kw):
    path = os.path.join(os.environ.get("LN3_PARITY_DIR", tempfile.gettempdir()), "ln3_parity.json")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    cur = {}
    if os.path.exists(path):
        try:
            cur = json.load(open(path))
        except Exception:
            cur = {}
    cur.update(kw)
    json.dump(cur, open(path, "w"), indent=1, sort_keys=True)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def test_dit_L2_forward_vs_oracle(dev):
    """BASELINE configs[1] model size: DiT-L/2 T23D forward of 2 samples (one zero-embedding uncond row, one
    conditioned row -- the CFG pair) against oracle.dit.dit_t23d_forward in fp32 on the host cores."""
    from ln3diff_b200.utils import build_t23d
    from oracle import dit as odit
    m = build_t23d("DiT-L/2")
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(31)
    x = torch.randn(2, 12, 32, 32, generator=g)
    t = torch.tensor([17.0, 803.0])
    ctx = torch.cat([torch.zeros(1, 77, 768), torch.randn(1, 77, 768, generator=g)])
    t0 = time.perf_counter()
    with torch.no_grad():
        ref = odit.dit_t23d_forward(sd, "DiT-L/2", x, t, ctx)
    cpu_s = time.perf_counter() - t0
    m = m.to(dev)
    out = m(x.to(dev), t.to(dev), ctx.to(dev))
    r = _rel(out, ref)
    _record(dit_L2_forward_rel_l2=r, dit_L2_oracle_cpu_seconds=cpu_s)
    assert out.shape == (2, 12, 32, 32) and r < 2e-2, r
    # per-sample too: the closed-form uncond row and the attended row each within tolerance
    assert _rel(out[0], ref[0]) < 2e-2 and _rel(out[1], ref[1]) < 2e-2


def test_dit2_L2_decode_and_pixels_vs_oracle(dev, golden):
    """Release decoder size: DiT2-L/2 VAE decode of one latent vs oracle.decoder.vae_decode (fp32, CPU); then the
    pixels of one 64x64 view rendered from OUR tri-plane vs from the fp32 oracle's (identical latent, identical
    sampling noise).  The same two errors are measured for the reference's own GPU arithmetic -- the oracle's
    module-for-module restatement run on the GPU under torch.autocast(bf16), which is how the reference runs its
    decoder (nsr/train_util_diffusion.py:177-206 under the engine's autocast) -- to show what tolerance identical
    latents can support at all."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_ae_decoder
    from oracle import decoder as odec
    from oracle import render as orender
    m = build_ae_decoder("DiT2-L/2", image_size=64)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    # random-init weights give a near-empty volume (white image, vacuous pixel error): a density bias of +3 fills
    # ~80 % of the pixels of this view with partially transparent, coloured matter
    sd["triplane_decoder.decoder.net.2.bias"][0] += 3.0
    m.load_state_dict(sd)
    g = torch.Generator().manual_seed(32)
    lat = 0.96806 ** -1 * torch.randn(1, 12, 32, 32, generator=g)
    with torch.no_grad():
        planes_ref = odec.vae_decode(sd, "DiT2-L/2", lat, 0.96806)                       # (1, 96, 128, 128) fp32
        sd_gpu = {k: v.to(dev) for k, v in sd.items() if v.is_floating_point()}
        with torch.autocast("cuda", dtype=torch.bfloat16):
            planes_refbf16 = _vae_decode_autocast(odec, sd_gpu, "DiT2-L/2", lat.to(dev), 0.96806).float().cpu()
    m = m.to(dev)
    cl = m.decode_to_channels_last(lat.to(dev), in_mul=0.96806)
    planes = cl.permute(0, 1, 4, 2, 3).reshape(1, 96, 128, 128)
    e_planes, e_planes_ref = _rel(planes, planes_ref), _rel(planes_refbf16, planes_ref)

    cam = torch.from_numpy(golden("cameras.npz")["objv_eval_pose"])[3]
    res = 64
    gen = torch.Generator().manual_seed(33)
    nc, nf = torch.rand(1, res * res, 64, generator=gen), torch.rand(1, res * res, 64, generator=gen)
    osg = tuple(sd[f"triplane_decoder.decoder.net.{i}.{n}"] for i, n in ((0, "weight"), (0, "bias"), (2, "weight"), (2, "bias")))
    px_ref = orender.render_view(planes_ref.reshape(3, 32, 128, 128), osg, cam, res, orender.OBJAVERSE_OPTS, nc[0], nf[0])
    px_refbf16 = orender.render_view(planes_refbf16.reshape(3, 32, 128, 128), osg, cam, res, orender.OBJAVERSE_OPTS, nc[0], nf[0])
    out = pipeline.decode_and_render(m, lat.to(dev), cam[None].to(dev), res, 0.96806, noise=(nc.to(dev), nf.to(dev)),
                                     mlp_tf32=False)
    e_px = _rel(out["image_raw"][0, 0], px_ref["image_raw"])
    e_px_ref = _rel(px_refbf16["image_raw"], px_ref["image_raw"])
    _record(dit2_L2_planes_rel_l2=e_planes, dit2_L2_planes_rel_l2_reference_bf16_autocast=e_planes_ref,
            latent_to_pixels_rel_l2=e_px, latent_to_pixels_rel_l2_reference_bf16_autocast=e_px_ref)
    occupied = float((px_ref["weights_samples"] > 0.05).float().mean())
    _record(latent_to_pixels_occupied_fraction=occupied)
    print(f"planes: ours {e_planes:.3e} / reference-bf16 {e_planes_ref:.3e}; pixels: ours {e_px:.3e} / "
          f"reference-bf16 {e_px_ref:.3e}; occupied pixels {occupied:.2f}")
    assert occupied > 0.1, "vacuous render: nothing in the volume"
    assert e_planes < 3e-2, e_planes          # 24 bf16 DiT2 blocks + conv tail on random-init weights
    assert e_px < 3e-2, e_px
    assert e_planes < 1.5 * e_planes_ref + 1e-3 and e_px < 1.5 * e_px_ref + 1e-3


def _vae_decode_autocast(odec, sd, arch, latent, scaling_divider):
    """oracle.decoder.vae_decode without its fp32 casts of the state dict / input dtype changes (autocast decides)."""
    lat = latent.float() * scaling_divider
    tok = odec.patch_embed_triplane(sd, lat)
    tok = odec.dit2_forward(sd, arch, tok)
    B, L, C = tok.shape
    hw = int(round((L // 3) ** 0.5))
    z = tok.reshape(B, 3, hw, hw, C).permute(0, 1, 4, 2, 3).reshape(B * 3, C, hw, hw)
    y = odec.ldm_decoder(sd, z.float())
    return y.reshape(B, 3 * y.shape[1], y.shape[2], y.shape[3])


def test_sampling_trajectory_vs_oracle_short(dev):
    """The fused Euler-EDM+CFG loop on DiT-B/2 for the first steps of the 250-step schedule, against the oracle
    loop on the host: the rel-L2 of the state after every step stays within the per-forward tolerance."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_t23d
    from oracle import dit as odit
    from oracle import samplers as osmp
    m = build_t23d("DiT-B/2")
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(41)
    x0 = torch.randn(1, 12, 32, 32, generator=g)
    c = {"crossattn": torch.randn(1, 77, 768, generator=g)}
    uc = {"crossattn": torch.zeros(1, 77, 768)}
    net = lambda xin, idx, cond: odit.dit_t23d_forward(sd, "DiT-B/2", xin, idx, cond["crossattn"])
    n = 12
    m = m.to(dev)
    cd, ucd = {"crossattn": c["crossattn"].to(dev)}, {"crossattn": uc["crossattn"].to(dev)}
    with torch.no_grad():
        ref = osmp.euler_edm_cfg_sample(net, x0, c, uc, n, 6.5)
    out = pipeline.sample_t23d(m, x0.to(dev), cd, ucd, n, 6.5)
    r = _rel(out, ref)
    _record(sampling_12step_B2_rel_l2=r)
    assert r < 2e-2, r
