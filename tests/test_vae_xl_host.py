"""CPU: the DiT2-L/2 VAE's reconstruction path -- the MVEncoderGSDynamicInp mirror's checkpoint layout and
construction, a float64 restatement of that encoder and the float64 renderer oracle at 96 + 96 samples per ray against
the reference's recorded output (tests/golden/vae_xl.npz, tools/make_golden_vae_xl.py), the 96_96 rendering options
and the reference's create_3DAE_model under the overlay."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

import vae_encoder_oracle as vo
from oracle import fixtures as fx
from oracle import render as orender
from oracle.decoder import _gn, _resblock, _swish

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NUM_FRAMES = 6


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


def dyna_encoder(sd, x, num_frames=NUM_FRAMES, return_mid=False):
    """MVEncoderGSDynamicInp.forward (model.py:611-623) in the dtype of its inputs: the Encoder trunk with the mid-block
    attention over groups of num_frames views, then the mean of each object's num_frames per-view moments."""
    h = F.conv2d(x, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    for lvl in range(len(vo.CH_MULT)):
        for b in range(vo.NUM_RES_BLOCKS):
            h = _resblock(sd, f"down.{lvl}.block.{b}.", h)
        if lvl != len(vo.CH_MULT) - 1:
            h = vo.downsample(sd, f"down.{lvl}.downsample.", h)
    h = _resblock(sd, "mid.block_1.", h)
    h = vo.spatial_transformer3d(sd, "mid.attn_1.", h, num_frames)
    mid = h
    h = _resblock(sd, "mid.block_2.", h)
    h = F.conv2d(_swish(_gn(h, sd["norm_out.weight"], sd["norm_out.bias"])), sd["conv_out.weight"], sd["conv_out.bias"],
                 padding=1)
    out = torch.cat([f.mean(keepdim=True, dim=0) for f in h.chunk(h.shape[0] // num_frames)], 0)
    return (out, mid) if return_mid else out


def xl_inputs():
    """The golden's 2 objects x 6 views (tools/make_golden_vae_xl.py): the first 12 views of enc_inputs."""
    return vo.enc_inputs(n_obj=2 * NUM_FRAMES // vo.VIEWS)


def _xl_encoder(**kw):
    from ln3diff_b200.ldm.modules.diffusionmodules.model import MVEncoderGSDynamicInp
    args = dict(double_z=True, resolution=256, in_channels=vo.IN_CH, ch=vo.CH, ch_mult=list(vo.CH_MULT),
                num_res_blocks=vo.NUM_RES_BLOCKS, dropout=0.0, attn_resolutions=[], out_ch=3, z_channels=vo.Z_CH,
                attn_kwargs={"n_heads": vo.HEADS, "d_head": vo.D_HEAD})
    args.update(kw)
    return MVEncoderGSDynamicInp(**args)


# ------------------------------------------------------------------ mirror construction
def test_mirror_state_dict_matches_reference_keys_and_shapes(golden):
    g = golden("vae_xl.npz")
    ref = json.loads(str(g["encoder_shapes"]))
    enc = _xl_encoder(num_frames=NUM_FRAMES)
    assert {k: list(v.shape) for k, v in enc.state_dict().items()} == ref
    assert not any(k.startswith("fusion_layer") for k in ref)
    from ln3diff_b200.utils import build_ae_encoder
    built = build_ae_encoder(dino_version="mv-sd-dit-dynaInp-trilatent")
    assert type(built).__name__ == "MVEncoderGSDynamicInp" and built.num_frames == 6
    assert {k: list(v.shape) for k, v in built.state_dict().items()} == ref
    assert type(build_ae_encoder()).__name__ == "MVEncoder"
    assert build_ae_encoder(dino_version="mv-sd-dit-dynaInp-trilatent", num_frames=8).num_frames == 8


def test_missing_num_frames_is_both_not_implemented_and_type_error():
    with pytest.raises(NotImplementedError, match="num_frames") as ei:
        _xl_encoder()
    assert isinstance(ei.value, TypeError)
    from ln3diff_b200.ldm.modules.diffusionmodules import model as M
    with pytest.raises(NotImplementedError):
        M.MVEncoderGS(ch=64, out_ch=3, num_res_blocks=1, attn_resolutions=[], in_channels=10, resolution=256,
                      z_channels=12)


def test_cpu_tensors_are_refused():
    enc = _xl_encoder(num_frames=NUM_FRAMES)
    with pytest.raises(RuntimeError, match="CUDA only"):
        enc(torch.zeros(6, 10, 64, 64))
    with pytest.raises(RuntimeError, match="CUDA only"):
        enc(torch.zeros(6, 10, 64, 64), num_frames=6)


def test_check_options_accepts_64_and_96_only():
    from ln3diff_b200.nsr.volumetric_rendering.renderer import ImportanceRenderer
    base = dict(orender.OBJAVERSE_OPTS)
    for s in (64, 96):
        ImportanceRenderer._check_options(dict(base, depth_resolution=s, depth_resolution_importance=s))
    for s, si in ((80, 80), (128, 128), (96, 64), (64, 96), (32, 32)):
        with pytest.raises(NotImplementedError):
            ImportanceRenderer._check_options(dict(base, depth_resolution=s, depth_resolution_importance=si))


def test_golden_rendering_options_are_the_96_preset(golden):
    """The reference resolved cfg objverse_tuneray_aug_resolution_96_96_auto to the 64_64 preset with 96 samples."""
    from ln3diff_b200.utils import OBJAVERSE_RENDERING_KWARGS, build_ae_decoder
    ref = json.loads(str(golden("vae_xl.npz")["rendering_options"]))
    assert ref["depth_resolution"] == ref["depth_resolution_importance"] == 96
    keys = ("ray_start", "ray_end", "box_warp", "white_back", "sampler_bbox_min", "sampler_bbox_max",
            "filter_out_of_bbox", "clamp_mode", "disparity_space_sampling")
    assert {k: ref[k] for k in keys} == {k: OBJAVERSE_RENDERING_KWARGS[k] for k in keys}
    dec = build_ae_decoder("DiT2-S/2", depth_resolution=96)
    kw = dec.rendering_kwargs
    assert kw["depth_resolution"] == kw["depth_resolution_importance"] == 96
    assert build_ae_decoder("DiT2-S/2").rendering_kwargs["depth_resolution"] == 64


# ------------------------------------------------------------------ oracles against the reference golden
@pytest.fixture(scope="module")
def oracle_obj0(golden):
    """float64 restatement on object 0 (6 views: its mid-block attention is self-contained)."""
    g = golden("vae_xl.npz")
    sd = {k: v.double() for k, v in vo.enc_state_dict(json.loads(str(g["encoder_shapes"]))).items()}
    with torch.no_grad():
        m64, mid64 = dyna_encoder(sd, xl_inputs()[:NUM_FRAMES].double(), return_mid=True)
    return g, m64, mid64


def test_dyna_encoder_restatement_matches_reference_golden(oracle_obj0):
    """The golden is the reference's fp32 evaluation; against the exact (float64) result it carries its own fp32
    rounding, bounded as in test_vae_encoder_host (6e-5 for ~20 renormalised layers of dot products of <= 2304
    terms).  The view mean adds 6 fp32 additions and a division: a few ulps more."""
    g, m64, mid64 = oracle_obj0
    ref, ref_mid = torch.from_numpy(g["moments"][:1]), torch.from_numpy(g["mid_obj0_strided"])
    s = vo.MID_STRIDE
    assert ref.shape == (1, 24, 32, 32) and g["moments"].shape == (2, 24, 32, 32)
    assert _rel(ref, m64) < 6e-5, _rel(ref, m64)
    assert _rel(ref_mid, mid64[:, :, ::s, ::s]) < 6e-5
    # the second object is not a copy of the first, and the mid-block transformer is not the identity
    assert _rel(g["moments"][1], g["moments"][0]) > 0.05
    assert _rel(mid64[:, :, ::s, ::s], torch.zeros_like(mid64[:, :, ::s, ::s]) + 1e-30) > 0.5


def test_render_group_at_96_samples_matches_reference_golden(golden):
    """oracle.render.render_group in fp32 at 96 + 96 samples against ImportanceRenderer.forward of the reference on
    the same batch-3 call (edge rays whose slab test yields NaN, a view whose rays all miss), noise injected.  Both
    are fp32 torch evaluations of the same expressions."""
    g = golden("vae_xl.npz")
    opts = json.loads(str(g["rendering_options"]))
    planes, osg, _, _, _, _ = fx.render_group_inputs()
    o, d = torch.from_numpy(g["render_ray_o"]), torch.from_numpy(g["render_ray_d"])
    nc, nf = torch.from_numpy(g["render_noise_coarse"]), torch.from_numpy(g["render_noise_fine"])
    assert nc.shape == nf.shape == (3, o.shape[1], 96)
    r = orender.render_group(planes, osg, o, d, nc, nf, opts)
    for k, gk in (("rgb", "render_rgb"), ("depth", "render_depth"), ("weights", "render_weights")):
        err = float((r[k] - torch.from_numpy(g[gk])).abs().max())
        assert err < 1e-5, (k, err)
    assert not bool(r["valid"][2].any()) and not bool(r["valid"][0, [0, 1, 3, 4]].any())
    # 96 samples differ from 64: the 64-sample render of the same call is measurably different
    r64 = orender.render_group(planes, osg, o, d, nc[..., :64].contiguous(), nf[..., :64].contiguous(),
                               dict(opts, depth_resolution=64, depth_resolution_importance=64))
    assert float((r64["rgb"] - r["rgb"]).abs().max()) > 1e-3


# ------------------------------------------------------------------ overlay
def test_reference_create_3dae_model_builds_the_xl_mirrors_under_the_overlay():
    """The reference's unmodified create_3DAE_model with the XL script's arguments (dino_version
    'mv-sd-dit-dynaInp-trilatent', num_frames 6, DiT2-L/2) returns the MVEncoderGSDynamicInp mirror and the decoder
    mirror, the rendering options of cfg objverse_tuneray_aug_resolution_96_96_auto resolved by the reference's own
    nsr/script_util; the mirror renderer accepts them."""
    import importlib
    import sys
    from oracle._stubs import REFERENCE_ROOT
    if not os.path.isdir(os.path.join(REFERENCE_ROOT, "nsr")):
        pytest.skip("reference checkout not present")
    prefixes = ("dit", "sgm", "nsr", "guided_diffusion", "transport", "vit", "ldm", "xformers", "timm", "torchdiffeq",
                "omegaconf", "blobfile")
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k.split(".")[0] in prefixes}
    saved_path = list(sys.path)
    from oracle import _stubs
    from ln3diff_b200 import overlay
    _stubs.install()
    overlay.install()
    try:
        n = importlib.import_module("nsr.script_util")
        opts = dict(cfg="objverse_tuneray_aug_resolution_96_96_auto", density_reg=0.25, density_reg_p_dist=0.004,
                    reg_type="l1", c_scale=1, patch_rendering_resolution=45)
        rk = n.rendering_options_defaults(type("Opts", (), opts)())
        cls = "vit.vit_triplane.RodinSR_256_fusionv6_ConvQuant_liteSR_dinoInit3DAttn_SD_B_3L_C_withrollout_withSD_D_ditDecoder_S"
        with torch.device("meta"):
            ae = n.create_3DAE_model(arch_encoder="vits", arch_decoder="vitb", dino_version="mv-sd-dit-dynaInp-trilatent",
                                     img_size=[256], encoder_in_channels=10, sd_E_ch=64, sd_E_num_res_blocks=1,
                                     z_channels=12, num_frames=6, ae_classname=cls, arch_dit_decoder="DiT2-L/2",
                                     embed_dim=1024, vae_p=2, ldm_z_channels=4, ldm_embed_dim=4, out_chans=96,
                                     decoder_in_chans=32, decoder_output_dim=3, image_size=192, rendering_kwargs=rk,
                                     no_dim_up_mlp=True)
        assert type(ae.encoder).__module__ == "ln3diff_b200.ldm.modules.diffusionmodules.model"
        assert type(ae.encoder).__name__ == "MVEncoderGSDynamicInp" and ae.encoder.num_frames == 6
        assert not hasattr(ae.encoder, "fusion_layer")
        assert type(ae.decoder).__module__ == "ln3diff_b200.vit.vit_triplane"
        kw = ae.decoder.rendering_kwargs
        assert kw["depth_resolution"] == kw["depth_resolution_importance"] == 96
        ae.decoder.triplane_decoder.renderer._check_options(kw)
    finally:
        overlay.uninstall()
        for k in list(sys.modules):
            if k.split(".")[0] in prefixes:
                del sys.modules[k]
        sys.modules.update(saved)
        sys.path[:] = saved_path


# ------------------------------------------------------------------ the C boundary
def test_view_mean_refusals_without_a_gpu():
    """ln3_view_mean_nhwc validates before any CUDA call: bad sizes and NULL pointers are LN3_EINVAL, B == 0 is a
    no-op."""
    import ctypes as C
    from ln3diff_b200 import _lib
    lib = _lib.lib()
    p = C.c_void_p(16)
    EINVAL = -1   # LN3_EINVAL
    for args in ((p, p, 1, 0, 4, 4), (p, p, 1, -2, 4, 4), (p, p, -1, 6, 4, 4), (p, p, 1, 6, 0, 4), (p, p, 1, 6, 4, 0),
                 (C.c_void_p(0), p, 1, 6, 4, 4), (p, C.c_void_p(0), 1, 6, 4, 4), (C.c_void_p(0), p, 0, 6, 4, 4)):
        rc = lib.ln3_view_mean_nhwc(*args, C.c_void_p(0))
        assert rc == EINVAL, (args, rc)
        assert b"view_mean_nhwc" in lib.ln3_last_error()
    assert lib.ln3_view_mean_nhwc(p, p, 0, 6, 4, 4, C.c_void_p(0)) == 0
