"""CPU: the oracle restatements against fixtures produced by the REFERENCE's own code
(oracle/make_golden.py, run in the build container)."""
import numpy as np
import torch

from oracle import dit as odit
from oracle import fixtures as fx
from oracle import render as orender
from oracle import samplers as osmp


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).norm() / b.norm()).item()


def test_dit_t23d_forward_matches_reference(golden):
    from ln3diff_b200.dit.dit_models_xformers import TextCondDiTBlock
    from ln3diff_b200.dit.dit_trilatent import DiT_models
    m = DiT_models["DiT-B/2"](input_size=32, num_classes=0, learn_sigma=False, in_channels=4,
                              context_dim=768, roll_out=True, vit_blk=TextCondDiTBlock)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    g = golden("dit_t23d.npz")
    # the analytic 3D-aware pos_embed of the mirror must equal the reference's
    assert abs(m.state_dict()["pos_embed"].double().sum().item() - float(g["pos_embed_checksum"])) < 1e-6
    sd = odit.synth_state_dict(shapes, seed=7, keep={"pos_embed": m.state_dict()["pos_embed"]})
    x, t, ctx = fx.dit_inputs()
    with torch.no_grad():
        y = odit.dit_t23d_forward(sd, "DiT-B/2", x, t, ctx)
    assert y.shape == (2, 12, 32, 32)
    assert _rel(y, g["out"]) < 2e-6          # fp32 vs fp32, different summation orders only


def test_sampler_engines_match_reference(golden):
    g = golden("samplers.npz")
    toy = fx.toy_network()
    x0, c, uc, noise, step_noise, z = fx.sampler_inputs()
    assert torch.equal(osmp.legacy_ddpm_sigmas(10), torch.from_numpy(g["sigmas10"]))
    assert torch.equal(osmp.legacy_ddpm_sigmas(250), torch.from_numpy(g["sigmas250"]))
    assert torch.equal(osmp.legacy_ddpm_sigmas(1000, append_zero=False, flip=True),
                       torch.from_numpy(g["denoiser_sigmas"]))
    out = osmp.euler_edm_cfg_sample(toy, x0.clone(), c, uc, 10, 6.5)
    assert torch.equal(out, torch.from_numpy(g["sgm"]))           # bit-exact: same op sequence
    tab = osmp.DDPMTables(osmp.linear_betas(1000), osmp.space_timesteps(1000, "10"))
    assert np.array_equal(tab.betas, g["ddpm_betas10"])
    assert tab.timestep_map == list(g["ddpm_timestep_map"])
    out = osmp.ddpm_p_sample_loop(lambda xx, tt, cc: toy(xx, tt * 1000, cc), (2, 12, 32, 32), tab, noise,
                                  step_noise, cond=c["crossattn"])
    assert torch.equal(out, torch.from_numpy(g["ddpm"]))
    ctx2 = {"crossattn": torch.cat([c["crossattn"], uc["crossattn"]])}
    out = osmp.flow_ode_cfg_sample(lambda xx, tt, cc: toy(xx, tt * 1000, cc), z, ctx2, 4.0, 10)
    assert torch.equal(out, torch.from_numpy(g["flow"]))


def test_renderer_matches_reference(golden):
    g, cams = golden("render.npz"), torch.from_numpy(golden("cameras.npz")["objv_eval_pose"])
    assert cams.shape == (40, 25)
    res = 24
    planes, osg, nc, nf = fx.render_inputs(res)
    for vi, row in enumerate(fx.RENDER_CAM_ROWS):
        cam = cams[row]
        o, d = orender.generate_rays(cam[:16].reshape(1, 4, 4), cam[16:].reshape(1, 3, 3), res)
        assert torch.equal(o[0], torch.from_numpy(g[f"ray_o_{vi}"]))
        assert (d[0] - torch.from_numpy(g[f"ray_d_{vi}"])).abs().max() < 2e-7
        # same rays as the reference -> isolates the renderer
        r = orender.render_rays(planes, osg, torch.from_numpy(g[f"ray_o_{vi}"]), torch.from_numpy(g[f"ray_d_{vi}"]),
                                orender.OBJAVERSE_OPTS, nc[vi], nf[vi])
        assert _rel(r["rgb"], g[f"rgb_{vi}"]) < 5e-6
        assert _rel(r["depth"], g[f"depth_{vi}"]) < 5e-6
        assert _rel(r["weights"], g[f"weights_{vi}"]) < 5e-6
        w = torch.from_numpy(g[f"weights_{vi}"])
        assert 0.05 < float(w.mean()) < 0.95          # the fixture is not vacuous (alpha spans (0,1))


def test_render_edge_cases():
    """All rays missing the box (degenerate (-1,-2) limits) and a camera inside the box."""
    res = 8
    planes, osg, nc, nf = fx.render_inputs(res, n_views=1)
    o = torch.tensor([[3.0, 3.0, 3.0]]).repeat(res * res, 1)
    d = torch.nn.functional.normalize(torch.tensor([[1.0, 0.2, 0.1]]), dim=1).repeat(res * res, 1)
    r = orender.render_rays(planes, osg, o, d, orender.OBJAVERSE_OPTS, nc[0], nf[0], return_debug=True)
    assert not bool(r["valid"].any())
    assert torch.isfinite(r["rgb"]).all() and torch.allclose(r["weights"], torch.zeros_like(r["weights"]))
    assert torch.allclose(r["rgb"], torch.ones_like(r["rgb"]))       # white background, nothing hit
    o2 = torch.zeros(res * res, 3)
    g = torch.Generator().manual_seed(3)
    d2 = torch.nn.functional.normalize(torch.randn(res * res, 3, generator=g), dim=1)
    r2 = orender.render_rays(planes, osg, o2, d2, orender.OBJAVERSE_OPTS, nc[0], nf[0], return_debug=True)
    assert bool(r2["valid"].all()) and torch.isfinite(r2["rgb"]).all()


def test_render_group_matches_reference(golden):
    """oracle.render.render_group vs one batch-3 ImportanceRenderer.forward call (render_group.npz): shared start
    range and depth clamp across the views, NaN slab tests (origin on a face, zero direction component) invalid."""
    g = golden("render_group.npz")
    planes, osg, o, d, nc, nf = fx.render_group_inputs()
    assert torch.equal(o, torch.from_numpy(g["ray_o"])) and torch.equal(d, torch.from_numpy(g["ray_d"]))
    r = orender.render_group(planes, osg, o, d, nc, nf, orender.OBJAVERSE_OPTS)
    for k in ("rgb", "depth", "weights"):
        assert (r[k] - torch.from_numpy(g[k])).abs().max() < 2e-6, k    # fp32 vs fp32, summation order only
    assert r["valid"][0, :5].tolist() == [False, False, True, False, False]
    assert bool(r["valid"][1].all()) and not bool(r["valid"][2].any())
    # the fixture tells one batched call from three per-view calls: the NaN rays of view 0 march the shared
    # start range, and the all-miss view's depth is clamped to the shared range
    for v, k in ((0, "rgb"), (2, "depth")):
        one = orender.render_rays(planes[v], osg, o[v], d[v], orender.OBJAVERSE_OPTS, nc[v], nf[v])
        assert (one[k] - torch.from_numpy(g[k][v])).abs().max() > 1e-2, (v, k)


def test_vae_decoder_matches_reference(golden):
    from oracle import decoder as odec
    from ln3diff_b200.utils import build_ae_decoder
    g = golden("decoder.npz")
    m = build_ae_decoder(fx.DECODER_ARCH)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()
              if k.startswith(("superresolution.ldm_upsample", "superresolution.conv_sr", "vit_decoder"))}
    sd = fx.decoder_state_dict(shapes)
    with torch.no_grad():
        y = odec.vae_decode(sd, fx.DECODER_ARCH, fx.decoder_latent(), fx.SCALING_DIVIDER)
    assert y.shape == (1, 96, 128, 128)
    assert _rel(y[:, :, 40:56, 40:56], g["crop"]) < 1e-5
    assert _rel(y.mean(dim=(0, 2, 3)), g["chan_mean"]) < 1e-4
    assert _rel(y.abs().mean(dim=(0, 2, 3)), g["chan_absmean"]) < 1e-5


def test_dit_i23d_forward_matches_reference(golden):
    from ln3diff_b200.utils import build_i23d
    g = golden("dit_i23d.npz")
    m = build_i23d(fx.I23D_ARCH)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = fx.i23d_state_dict(shapes, m.state_dict()["pos_embed"])
    x, t, ctx = fx.i23d_inputs()
    with torch.no_grad():
        y = odit.dit_i23d_pixart_forward(sd, fx.I23D_ARCH, x, t, ctx)
    assert _rel(y, g["out"]) < 2e-6
    c, u = y.chunk(2)
    half = u + 4.0 * (c - u)
    assert _rel(torch.cat([half, half]), g["out_cfg"]) < 2e-6


def test_point_queries_match_reference(golden):
    """oracle.render.run_model_points / grid_points vs ImportanceRenderer._run_model (points.npz)."""
    g = golden("points.npz")
    planes, osg, _, _ = fx.render_inputs(8)
    rgb, sigma = orender.run_model_points(planes, osg, torch.from_numpy(g["points"]), 0.9)
    assert _rel(rgb, g["rgb"]) < 2e-6 and _rel(sigma, g["sigma"]) < 2e-6
    G = int(g["grid_size"])
    pts = orender.grid_points([-0.45] * 3, [0.45] * 3, G)
    rgb, sigma = orender.run_model_points(planes, osg, pts, 0.9)
    assert _rel(rgb, g["grid_rgb"]) < 2e-6 and _rel(sigma, g["grid_sigma"]) < 2e-6
    # about a fifth of the random points fall outside the planes' support (zeros padding): both sides agree
    outside = (torch.from_numpy(g["points"]).abs() > 0.45).any(-1)
    assert 0.1 < outside.float().mean() < 0.7


def test_dit_t23d_pixart_forward_matches_reference(golden):
    """oracle.dit.dit_t23d_pixart_forward vs the reference's DiT_TriLatent_PixelArt (dit_t23d_pixart.npz)."""
    from ln3diff_b200.dit.dit_trilatent import DiT_models
    g = golden("dit_t23d_pixart.npz")
    m = DiT_models[fx.T23D_PIXART_ARCH](input_size=32, num_classes=0, learn_sigma=False, in_channels=4,
                                        context_dim=768, roll_out=True)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes["blocks.0.attention_y_norm.weight"] == (768,) and "clip_text_proj.y_proj.fc1.weight" not in shapes
    sd = fx.i23d_state_dict(shapes, m.state_dict()["pos_embed"])
    x, t, ctx = fx.t23d_pixart_inputs()
    with torch.no_grad():
        y = odit.dit_t23d_pixart_forward(sd, fx.T23D_PIXART_ARCH, x, t, ctx)
    assert _rel(y, g["out"]) < 2e-6
    c, u = y.chunk(2)
    half = u + 6.5 * (c - u)
    assert _rel(torch.cat([half, half]), g["out_cfg"]) < 2e-6
