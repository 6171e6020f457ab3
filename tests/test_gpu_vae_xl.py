"""GPU: reconstruction with the DiT2-L/2 VAE -- ln3_view_mean_nhwc element by element, the MVEncoderGSDynamicInp mirror
against the reference's golden in both conv modes and its pooling semantics, the F = 6 mid-block, the fused renderer at
96 + 96 samples per ray against float64 on every dispatch path and against the reference's golden, batched
decode_and_render, and `reconstruct` end to end with a DiT2-L/2 decoder at 192^2."""
import ctypes as C
import json

import pytest
import torch

import test_gpu_render_conformance as rc
import vae_encoder_oracle as vo
from kernel_bounds import _chunk_mean, view_mean_tol
from oracle import fixtures as fx
from oracle import render as orender
from test_vae_xl_host import NUM_FRAMES, dyna_encoder, xl_inputs

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
S96 = 96


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).norm() / b.norm())


# ------------------------------------------------------------------ ln3_view_mean_nhwc
@pytest.mark.parametrize("B,F,S,C", [(3, 5, 7, 13), (2, 6, 32, 24), (1, 8, 9, 5), (4, 6, 11, 1)])
def test_view_mean_elementwise(dev, B, F, S, C):
    """Bit-exact against the header's order (fp32 sum over the views in order, then one division by F), and within
    (F + 1) u sum|x| / F of the float64 mean; nothing outside the output is written."""
    from ln3diff_b200 import ops
    g = torch.Generator().manual_seed(B * 100 + F * 10 + S + C)
    x = 3 * torch.randn(B * F, S, S, C, generator=g) + 0.5
    n, pad = B * S * S * C, 1024
    buf = torch.full((n + 2 * pad,), float("nan"), device=dev)
    out = buf[pad:pad + n].view(B, S, S, C)
    from ln3diff_b200 import _lib
    _lib.check(_lib.lib().ln3_view_mean_nhwc(_lib.ptr(x.to(dev)), _lib.ptr(out), B, F, S, C, _lib.current_stream()))
    got = out.cpu()
    assert bool(buf[:pad].isnan().all()) and bool(buf[pad + n:].isnan().all())
    xv = x.view(B, F, S, S, C)
    s = xv[:, 0].clone()
    for f in range(1, F):
        s = s + xv[:, f]
    assert torch.equal(got, s / F)
    ref = xv.double().mean(1)
    tol = view_mean_tol(xv)
    assert bool(((got.double() - ref).abs() <= tol).all())
    assert torch.equal(ops.view_mean_nhwc(x.to(dev), F).cpu(), got)


def test_view_mean_error_returns(dev):
    from ln3diff_b200 import _lib, ops
    lib = _lib.lib()
    x = torch.zeros(12, 4, 4, 8, device=dev)
    p = _lib.ptr(x)
    for args in ((p, p, 2, 0, 4, 8), (p, p, 2, -6, 4, 8), (p, p, -1, 6, 4, 8), (p, p, 2, 6, 0, 8), (p, p, 2, 6, 4, 0),
                 (C.c_void_p(0), p, 2, 6, 4, 8), (p, C.c_void_p(0), 2, 6, 4, 8)):
        assert lib.ln3_view_mean_nhwc(*args, _lib.current_stream()) == -1, args
    n0 = _lib.launch_count()
    assert lib.ln3_view_mean_nhwc(p, p, 0, 6, 4, 8, _lib.current_stream()) == 0
    assert _lib.launch_count() == n0
    with pytest.raises(ValueError):
        ops.view_mean_nhwc(x, 5)                       # 12 views are not a multiple of 5
    with pytest.raises(ValueError, match="CUDA"):
        ops.view_mean_nhwc(x.cpu(), 6)


# ------------------------------------------------------------------ the encoder
def _golden_xl_encoder(dev, golden, tf32: bool):
    from ln3diff_b200.utils import build_ae_encoder
    g = golden("vae_xl.npz")
    enc = build_ae_encoder(dino_version="mv-sd-dit-dynaInp-trilatent")
    enc.load_state_dict(vo.enc_state_dict(json.loads(str(g["encoder_shapes"]))))
    enc.conv_tf32 = tf32
    return enc.to(dev), g


@pytest.mark.parametrize("tf32", [False, True])
def test_xl_encoder_vs_reference_golden(dev, golden, tf32):
    """MVEncoderGSDynamicInp on 2 objects x 6 views at 256^2 against the reference's recorded fp32 moments.  The
    bounds of test_gpu_vae_encoder.test_encoder_vs_reference_golden hold unchanged: the bf16 mid-block branch carries
    <= 2e-2 of its own scale, TF32 convs ~20 * 7e-4 in the worst case of aligned errors, and the view mean of 6
    moments adds a few fp32 roundings and averages the per-view errors down.  Exact convs < 1e-2, TF32 convs < 2e-2."""
    enc, g = _golden_xl_encoder(dev, golden, tf32)
    x = xl_inputs().to(dev)
    moments = enc(x)
    assert moments.shape == (2, 24, 32, 32) and moments.dtype == torch.float32
    e = _rel(moments, g["moments"])
    print(f"XL encoder ({'TF32' if tf32 else 'fp32'} convs) vs reference: moments rel-L2 {e:.3e}")
    assert e < (2e-2 if tf32 else 1e-2), e
    assert _rel(moments[0], moments[1]) > 0.05 and torch.equal(enc(x), moments)
    # the pooling is the mean of the per-view trunk outputs (not a sum, not one view)
    per_view = enc._trunk_nhwc(x, NUM_FRAMES)
    assert torch.equal(enc.forward_nhwc(x), _chunk_mean(per_view, NUM_FRAMES))


def test_xl_encoder_num_frames_argument_follows_the_reference(dev):
    """forward(x, num_frames): the mid-block groups views by self.num_frames whatever the argument; the pooling
    chunks by the argument (torch.chunk sizes, including a shorter last chunk); num_frames <= 4 fails the assert."""
    from ln3diff_b200.utils import build_ae_encoder
    enc = build_ae_encoder(dino_version="mv-sd-dit-dynaInp-trilatent", seed=3).to(dev)
    x = torch.rand(30, 10, 64, 64, generator=torch.Generator().manual_seed(5)).to(dev) * 2 - 1
    h = enc._trunk_nhwc(x, 6)                                  # 30 views = 5 objects of 6 for the attention
    # h.chunk(30 // nf): chunks of ceil(30 / (30 // nf)) views; nf = 7 gives 4 chunks of 8, 8, 8 and 6
    for nf, n_chunks in ((6, 5), (5, 6), (7, 4), (10, 3), (30, 1)):
        got = enc(x, num_frames=nf)
        ref = _chunk_mean(h, nf).permute(0, 3, 1, 2)
        assert got.shape[0] == n_chunks and got.shape == ref.shape and torch.equal(got, ref), nf
    assert torch.equal(enc(x), enc(x, num_frames=6))
    with pytest.raises(AssertionError):
        enc(x, num_frames=4)
    # the attention really groups by self.num_frames: grouping by 5 gives a different trunk
    assert not torch.equal(enc._trunk_nhwc(x, 5), h)


def test_mid_block_transformer_f6_vs_oracle(dev, golden):
    """SpatialTransformer3D with attn1 over 6 views (6144 tokens per object) against float64: the bf16 bound of
    test_gpu_vae_encoder.test_mid_block_transformer_vs_oracle (5 * 2^-8 = 2e-2 rel-L2 of the branch)."""
    enc, g = _golden_xl_encoder(dev, golden, tf32=False)
    P = enc.prepare()
    h = torch.randn(12, 32, 32, 256, generator=torch.Generator().manual_seed(64))
    out = enc._spatial_transformer(h.to(dev), P["st"], NUM_FRAMES)
    sd = {k: v.double().to(dev) for k, v in vo.enc_state_dict(json.loads(str(g["encoder_shapes"]))).items()}
    ref = vo.spatial_transformer3d(sd, "mid.attn_1.", h.to(dev).double().permute(0, 3, 1, 2),
                                   NUM_FRAMES).permute(0, 2, 3, 1)
    branch, branch_ref = out.double() - h.to(dev).double(), ref - h.to(dev).double()
    e = _rel(branch, branch_ref)
    print(f"F=6 mid-block transformer branch rel-L2 vs float64: {e:.3e}")
    assert e < 2e-2, e
    # attn1 really mixes the 6 views of an object: running it per view (num_frames = 1) is far off
    per_view = enc._spatial_transformer(h.to(dev), P["st"], 1)
    assert _rel(per_view.double() - h.to(dev).double(), branch_ref) > 10 * e


# ------------------------------------------------------------------ renderer at 96 + 96
def _noise96(V, M, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(V, M, S96, generator=g), torch.rand(V, M, S96, generator=g)


def _simple96(name, V, w, h, seed, *, n_obj=1, view_obj=None, **kw):
    o, d = rc._pinhole_rays(V, w, h, seed)
    nc, nf = _noise96(V, w * h, seed + 1)
    vo_ = view_obj if view_obj is not None else [v * n_obj // V for v in range(V)]
    return rc.Case(name, rc._planes(n_obj, seed + 2), o, d, nc, nf, vo_, **kw)


def _group96(gs):
    o, d = rc._pinhole_rays(5, 8, 8, 170)
    o[1], d[1] = rc._miss_rays(64, 171)
    o[3], d[3] = rc._inside_rays(64, 172)
    nc, nf = _noise96(5, 64, 173)
    return rc.Case(f"groups96_gs{gs}", rc._planes(5, 174), o, d, nc, nf, list(range(5)), group_size=gs, tiled=True)


def _edge96(golden):
    g = golden("vae_xl.npz")
    planes, _, o, d, _, _ = fx.render_group_inputs()
    assert torch.equal(o, torch.from_numpy(g["render_ray_o"])) and torch.equal(d, torch.from_numpy(g["render_ray_d"]))
    return rc.Case("edge96", planes, o, d, torch.from_numpy(g["render_noise_coarse"]),
                   torch.from_numpy(g["render_noise_fine"]), [0, 1, 2], group_size=3)


CASES96 = {
    "square8": lambda: _simple96("square8", 2, 8, 8, 110, tiled=True),
    "side6_v3": lambda: _simple96("side6_v3", 3, 6, 6, 112),                       # linear, partial last item
    "wide20x12": lambda: _simple96("wide20x12", 2, 20, 12, 115, image_width=20, tiled=True),
    "objects_3x2": lambda: _simple96("objects_3x2", 6, 8, 8, 117, n_obj=3, tiled=True),
    "view_obj_perm": lambda: _simple96("view_obj_perm", 6, 8, 8, 118, n_obj=3, view_obj=[2, 0, 1, 1, 0, 2],
                                       explicit_map=True, tiled=True),
    "groups_gs2": lambda: _group96(2),
    "groups_gs5": lambda: _group96(5),
}


def _opts96(c):
    o = rc._opts(c.box_warp, c.bbox, c.white_back)
    o.update(depth_resolution=S96, depth_resolution_importance=S96)
    return o


def _reference96(c):
    opts, osg = _opts96(c), tuple(t.double() for t in rc._OSG)
    outs = []
    for v0 in range(0, c.V, c.group_size):
        vs = list(range(v0, min(v0 + c.group_size, c.V)))
        planes = torch.stack([c.planes[c.view_obj[v]] for v in vs]).double()
        outs.append(orender.render_group(planes, osg, c.ray_o[vs].double(), c.ray_d[vs].double(),
                                         c.nc[vs].double(), c.nf[vs].double(), opts))
    return {k: torch.cat([o[k] for o in outs]).reshape(c.V, c.M, -1).squeeze(-1) for k in ("rgb", "depth", "weights")}


def _run96(dev, c, tf32, image_width=-1, debug=False):
    from ln3diff_b200 import ops
    pcl = ops.planes_to_channels_last(c.planes.contiguous().to(dev))
    kw = dict(view_obj=torch.tensor(c.view_obj, dtype=torch.int32, device=dev)) if c.explicit_map else \
        dict(views_per_obj=c.V // c.planes.shape[0])
    out = ops.render_views(pcl, c.ray_o.contiguous().to(dev), c.ray_d.contiguous().to(dev), c.nc.contiguous().to(dev),
                           c.nf.contiguous().to(dev), tuple(t.to(dev) for t in rc._OSG), group_size=c.group_size,
                           box_warp=c.box_warp, bbox_min=-c.bbox, bbox_max=c.bbox, white_back=c.white_back,
                           mlp_tf32=tf32, debug=debug, samples_per_ray=S96,
                           image_width=c.image_width if image_width == -1 else image_width, **kw)
    torch.cuda.synchronize()
    return {"rgb": out["rgb"].permute(0, 2, 1).cpu(), "depth": out["depth"][:, 0].cpu(),
            "weights": out["weights"][:, 0].cpu(), **({"dbg": out} if debug else {})}


def _check_debug(c, dbg, over):
    """Debug outputs at the 96-sample shapes, per view against the float64 render_rays of a one-view call: every
    ray's sort permutation is a permutation of 0..191 and its importance indices lie in 0..94; rays that took the
    reference's discrete decisions (importance index, sort order, in-box test) have fine depths within 1e-5 of it, and
    every ray past the exact bound took a different one (test_gpu_render_conformance's rule)."""
    M = c.M
    assert dbg["inbox"].shape == (c.V * M, 2 * S96) and dbg["order"].shape == (c.V * M, 2 * S96)
    assert dbg["inds"].shape == (c.V * M, S96) and dbg["z_fine"].shape == (c.V * M, S96)
    order = dbg["order"].cpu().long()
    assert torch.equal(order.sort(1)[0], torch.arange(2 * S96).expand_as(order))
    inds = dbg["inds"].cpu().long()
    assert int(inds.min()) >= 0 and int(inds.max()) <= S96 - 2
    if c.group_size != 1:
        return
    opts, osg = _opts96(c), tuple(t.double() for t in rc._OSG)
    n_same = 0
    for v in range(c.V):
        r = orender.render_rays(c.planes[c.view_obj[v]].double(), osg, c.ray_o[v].double(), c.ray_d[v].double(),
                                opts, c.nc[v].double(), c.nf[v].double(), return_debug=True)
        sl = slice(v * M, (v + 1) * M)
        inbox = torch.cat([r["inbox_coarse"], r["inbox_fine"]], 1)
        flip = ((inds[sl] != r["inds"]).any(1) | (order[sl] != r["order"]).any(1)
                | (dbg["inbox"][sl].cpu().bool() != inbox).any(1))
        same = ~flip
        n_same += int(same.sum())
        err = (dbg["z_fine"][sl].cpu().double() - r["z_fine"]).abs().amax(1)
        assert bool((err[same] <= 1e-5 * r["z_fine"].abs().amax(1)[same].clamp_min(1)).all()), float(err[same].max())
        rays = torch.nonzero(over[v])[:, 0]
        assert bool(flip[rays].all()), (v, rays[~flip[rays]].tolist())
    assert n_same >= 0.9 * c.V * M


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
@pytest.mark.parametrize("name", list(CASES96))
def test_render96_matches_fp64_reference(dev, name, tf32):
    """The element-wise bounds of test_gpu_render_conformance (fp32: 2e-5, discrete-decision flips up to 1e-4 on at
    most 0.5 % of the rays of one-view groups; TF32: 2e-3 / 1e-3 and 1e-3 per-view rgb rel-L2) at 96 + 96 samples."""
    c = CASES96[name]()
    got = _run96(dev, c, tf32, debug=not tf32)
    over = rc._check(f"{name} S=96", got, _reference96(c), tf32, flips_allowed=c.group_size == 1)
    if not tf32:
        _check_debug(c, got["dbg"], over)


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
@pytest.mark.parametrize("name", ["square8", "objects_3x2", "groups_gs2"])
def test_render96_tiled_and_linear_schedules_are_bit_identical(dev, name, tf32):
    c = CASES96[name]()
    a, b = _run96(dev, c, tf32), _run96(dev, c, tf32, image_width=0)
    for k in ("rgb", "depth", "weights"):
        assert torch.equal(a[k], b[k]), (name, k)


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
def test_render96_matches_reference_golden(dev, golden, tf32):
    """The reference's own ImportanceRenderer.forward with its resolved 96_96 options on the batch-3 edge-ray call
    (NaN slab tests, an all-miss view), noise injected, and the float64 oracle of the same call."""
    g = golden("vae_xl.npz")
    c = _edge96(golden)
    got = _run96(dev, c, tf32, debug=True)
    ref = {"rgb": torch.from_numpy(g["render_rgb"]).double(), "depth": torch.from_numpy(g["render_depth"])[..., 0].double(),
           "weights": torch.from_numpy(g["render_weights"])[..., 0].double()}
    rc._check("edge rays S=96 vs reference golden", got, ref, tf32)
    rc._check("edge rays S=96 vs float64", got, _reference96(c), tf32)
    # 64 samples would not pass: the kernel really took 96
    ref64 = orender.render_group(c.planes.double(), tuple(t.double() for t in rc._OSG), c.ray_o.double(),
                                 c.ray_d.double(), c.nc[..., :64].double(), c.nf[..., :64].double(),
                                 orender.OBJAVERSE_OPTS)
    assert float((ref64["rgb"] - ref["rgb"]).abs().max()) > 1e-3


def test_render_views_rejects_other_sample_counts(dev):
    from ln3diff_b200 import _lib, ops
    c = CASES96["square8"]()
    with pytest.raises(ValueError, match="64 or 96"):
        ops.render_views(torch.zeros(1, 3, 16, 16, 32, device=dev), c.ray_o.to(dev), c.ray_d.to(dev),
                         c.nc.to(dev), c.nf.to(dev), tuple(t.to(dev) for t in rc._OSG), views_per_obj=2,
                         samples_per_ray=128)
    with pytest.raises(ValueError, match="V\\*M\\*64"):     # 96-sample noise with the default count
        ops.render_views(torch.zeros(1, 3, 16, 16, 32, device=dev), c.ray_o.to(dev), c.ray_d.to(dev),
                         c.nc.to(dev), c.nf.to(dev), tuple(t.to(dev) for t in rc._OSG), views_per_obj=2)
    # the C boundary: S != S_importance and S = 80 are LN3_EUNSUPPORTED (-3) before any launch
    for s, si in ((96, 64), (80, 80), (128, 128)):
        a = _lib.RenderArgs()
        a.V, a.M, a.C, a.S, a.S_importance, a.hidden_dim, a.decoder_output_dim = 1, 16, 32, s, si, 64, 3
        assert _lib.lib().ln3_render_views(C.byref(a), _lib.current_stream()) == -3
        assert b"96+96" in _lib.lib().ln3_last_error()


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
def test_decode_and_render_96_object_batches(dev, tf32):
    """pipeline.decode_and_render with the 96 preset (rendering_kwargs depth_resolution 96), B=3 in launches of 2
    then 1 objects: every object equals a single-object 96-sample render_views, bit for bit."""
    from ln3diff_b200 import ops, pipeline
    from ln3diff_b200.utils import orbit_cameras
    B, V, res = 3, 2, 16
    M = res * res
    planes_cl = ops.planes_to_channels_last(rc._planes(B, 130).to(dev))
    osg = tuple(t.to(dev) for t in rc._OSG)

    class Decoder:
        rendering_kwargs = dict(box_warp=0.9, sampler_bbox_min=-0.45, sampler_bbox_max=0.45, white_back=True,
                                depth_resolution=96, depth_resolution_importance=96)

        class triplane_decoder:
            class decoder:
                @staticmethod
                def raw_parameters():
                    return osg

        @staticmethod
        def decode_to_channels_last(latents, in_mul):
            return planes_cl

    cams = orbit_cameras(V)
    nc, nf = (t.to(dev) for t in _noise96(B * V, M, 131))
    out = pipeline.decode_and_render(Decoder(), torch.zeros(B, 12, 32, 32, device=dev), cams, resolution=res,
                                     noise=(nc, nf), mlp_tf32=tf32, max_views_per_launch=2 * V)
    o, d = ops.generate_rays(cams.to(dev).contiguous(), res)
    for b in range(B):
        one = ops.render_views(planes_cl[b:b + 1].contiguous(), o, d, nc[b * V:(b + 1) * V].contiguous(),
                               nf[b * V:(b + 1) * V].contiguous(), osg, views_per_obj=V, mlp_tf32=tf32,
                               samples_per_ray=96)
        assert torch.equal(out["image_raw"][b], one["rgb"].view(V, 3, res, res)), b
        assert torch.equal(out["image_depth"][b], one["depth"].view(V, 1, res, res)), b
        assert torch.equal(out["weights_samples"][b], one["weights"].view(V, 1, res, res)), b
    # without explicit noise the pipeline draws (B*V, M, 96) itself
    out2 = pipeline.decode_and_render(Decoder(), torch.zeros(B, 12, 32, 32, device=dev), cams, resolution=res)
    assert out2["image_raw"].shape == (B, V, 3, res, res) and bool(out2["image_raw"].isfinite().all())


# ------------------------------------------------------------------ end to end
def test_reconstruct_xl_end_to_end_vs_oracle_chain(dev, golden):
    """reconstruct with the XL encoder (2 objects x 6 views at 256^2) and a DiT2-L/2 decoder rendering 192^2 at
    96 + 96 samples, against the oracle chain (the encoder oracle in float64, the decoder and renderer oracles in fp32)
    with the same CPU-drawn posterior noise and explicit renderer noise, within the decoder path's pixel tolerance of
    test_gpu_vae_encoder (3e-2 rel-L2: bf16 DiT2 features)."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_ae_decoder
    from oracle import decoder as odec
    enc, g = _golden_xl_encoder(dev, golden, tf32=True)
    arch = "DiT2-L/2"
    dec = build_ae_decoder(arch, image_size=192, depth_resolution=96)
    qw, qb = vo.quant_conv_params()
    dec.superresolution["quant_conv"].weight.data.copy_(qw)
    dec.superresolution["quant_conv"].bias.data.copy_(qb)
    sd_dec = {k: v.clone() for k, v in dec.state_dict().items()}
    dec = dec.to(dev)
    x = xl_inputs()
    cams = torch.from_numpy(golden("cameras.npz")["objv_eval_pose"])[[2, 9]]
    res, V, B = 192, 2, 2
    gen = torch.Generator().manual_seed(66)
    nc, nf = torch.rand(B * V, res * res, S96, generator=gen), torch.rand(B * V, res * res, S96, generator=gen)
    torch.manual_seed(67)
    ret, out = pipeline.reconstruct(enc, dec, x.to(dev), cams.to(dev), resolution=res, noise=(nc.to(dev), nf.to(dev)))
    assert out["image_raw"].shape == (B, V, 3, res, res)
    sd_enc = {k: v.double().to(dev) for k, v in vo.enc_state_dict(json.loads(str(g["encoder_shapes"]))).items()}
    with torch.no_grad():
        mom = dyna_encoder(sd_enc, x.to(dev).double()).cpu()
    torch.manual_seed(67)
    noise = torch.randn(B, 4, 3, 1024).reshape(B, 12, 32, 32)
    _, _, z = vo.posterior(qw.double(), qb.double(), mom, noise.double())
    assert _rel(ret["latent_normalized_2Ddiffusion"], z) < 2e-2
    opts = dict(orender.OBJAVERSE_OPTS, depth_resolution=S96, depth_resolution_importance=S96)
    osg = tuple(sd_dec[f"triplane_decoder.decoder.net.{i}.{n}"] for i, n in ((0, "weight"), (0, "bias"), (2, "weight"),
                                                                              (2, "bias")))
    for b in range(B):
        with torch.no_grad():
            planes = odec.vae_decode(sd_dec, arch, z[b:b + 1].float(), 1.0).reshape(3, 32, 128, 128)
        for v in range(V):
            ref = orender.render_view(planes, osg, cams[v], res, opts, nc[b * V + v], nf[b * V + v])
            e = _rel(out["image_raw"][b, v], ref["image_raw"])
            print(f"reconstruct XL object {b} view {v}: image rel-L2 {e:.3e}")
            assert e < 3e-2 and _rel(out["image_mask"][b, v], ref["image_mask"]) < 3e-2
