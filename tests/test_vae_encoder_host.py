"""CPU: the stage-1 VAE encoder path -- the oracle restatement against the reference's recorded output
(tests/golden/vae_encoder.npz, tools/make_golden_vae_encoder.py), the mirror's checkpoint layout, the reference's
create_3DAE_model under the overlay, and the host-side checks of ln3_downsample_nhwc and ln3_vae_posterior."""
import ctypes as C
import json
import os

import pytest
import torch

import vae_encoder_oracle as vo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def oracle_run(golden):
    """The oracle on object 0 (4 views) in fp32 and float64, and the posterior of the golden moments."""
    g = golden("vae_encoder.npz")
    sd = vo.enc_state_dict(json.loads(str(g["encoder_shapes"])))
    x = vo.enc_inputs()[:vo.VIEWS]
    with torch.no_grad():
        m32, mid32 = vo.mv_encoder(sd, x, return_mid=True)
        sd64 = {k: v.double() for k, v in sd.items()}
        m64, mid64 = vo.mv_encoder(sd64, x.double(), return_mid=True)
    return g, m32, mid32, m64, mid64


def test_oracle_encoder_matches_reference_golden(oracle_run):
    """fp32 reorder tolerance.  The reference (golden) and the oracle evaluate the same fp32 network with differently
    ordered sums, so each differs from the exact (float64) result by its own rounding and
        |oracle32 - ref32| <= |oracle32 - f64| + |ref32 - f64|      (triangle inequality, also for the L2 norm).
    Each conv / linear output is a dot product of K <= 2304 terms: fp32 rounding contributes a relative error of
    about sqrt(K) 2^-24 ~ 3e-6 in the RMS sense (random-sign rounding errors), and the ~20 layers in sequence, each
    renormalised by GroupNorm / LayerNorm, add these errors rather than compound them: 20 * 3e-6 = 6e-5 bounds either
    fp32 evaluation against float64, hence 1.2e-4 the two against each other.  Measured: ~1e-6."""
    g, m32, mid32, m64, mid64 = oracle_run
    ref, ref_mid = torch.from_numpy(g["moments"][:1]), torch.from_numpy(g["mid_obj0_strided"])
    s = vo.MID_STRIDE
    mid32_s, mid64_s = mid32[:, :, ::s, ::s], mid64[:, :, ::s, ::s]
    e_ref, e_or = _rel(ref, m64), _rel(m32, m64)
    assert e_ref < 6e-5 and e_or < 6e-5, (e_ref, e_or)
    assert _rel(m32, ref) <= e_ref + e_or + 1e-12
    assert _rel(mid32_s, ref_mid) < 1.2e-4 and _rel(ref_mid, mid64_s) < 6e-5
    # the mid-block transformer is not the identity (proj_out is seeded, not zero) and the views are fused
    assert _rel(mid64_s, torch.zeros_like(mid64_s) + 1e-30) > 0.5
    assert ref.shape == (1, 24, 32, 32) and g["moments"].shape == (2, 24, 32, 32)


def test_oracle_posterior_matches_reference_golden(golden):
    """mean / logvar / z of object 0 for the noise the reference drew after manual_seed(NOISE_SEED).  The posterior is
    element-wise after an 8-term dot product, so fp32 vs fp32 differ by at most (8 + 1) 2^-24 sum|terms| in the
    moments, carried through tanh (slope <= 1) and exp (relative error = absolute error of 0.5 logvar) -- a few ulps."""
    g = golden("vae_encoder.npz")
    qw, qb = vo.quant_conv_params()
    mom = torch.from_numpy(g["moments"])
    noise = vo.posterior_noise()
    mean, lv, z = vo.posterior(qw, qb, mom, noise)
    terms = vo.conv_terms_abs(mom, qw, pad=(0, 0, 0, 0), groups=3) + qb.abs()[None, :, None, None]
    tol_m = 9 * 2.0 ** -24 * terms[:, :12] + 2.0 ** -24 * mean.abs()
    tol_lv = 9 * 2.0 ** -24 * terms[:, 12:] + 4 * 2.0 ** -24 * lv.abs()
    std = torch.exp(0.5 * lv.double())
    tol_z = tol_m + std * (0.5 * tol_lv + 4 * 2.0 ** -24) * noise.abs() + 2 * 2.0 ** -24 * z.abs()
    for got, ref, tol in ((mean, g["mean_obj0"], tol_m), (lv, g["logvar_obj0"], tol_lv), (z, g["z_obj0"], tol_z)):
        d = (got[:1].double() - torch.from_numpy(ref).double()).abs()
        assert bool((d <= tol[:1]).all()), float((d / tol[:1]).max())
    assert set(json.loads(str(g["ret_keys"]))) == {"normal_entropy", "latent_normalized", "latent_normalized_2Ddiffusion",
                                                   "log_q_2Ddiffusion", "log_q", "posterior"}
    # log_q divides by var, not std (the reference's quirk): check the golden against both readings
    var = torch.exp(lv[:1].double())
    lq = -0.5 * ((z[:1].double() - mean[:1]) / var) ** 2 - 0.5 * torch.log(torch.tensor(2 * torch.pi)) - lv[:1]
    assert _rel(torch.from_numpy(g["log_q_obj0"]), lq) < 1e-5


def test_mirror_state_dicts_match_reference_layout(golden):
    """MVEncoder and the `_S` decoder (DiT2-B/2, DiT2-L/2): every key and shape of the reference's modules."""
    from ln3diff_b200.dit.dit_decoder import DiT2_models
    from ln3diff_b200.nsr.triplane import Triplane
    from ln3diff_b200.utils import OBJAVERSE_RENDERING_KWARGS, build_ae_encoder
    from ln3diff_b200.vit import vit_triplane as vt
    g = golden("vae_encoder.npz")
    enc = build_ae_encoder()
    assert {k: list(v.shape) for k, v in enc.state_dict().items()} == json.loads(str(g["encoder_shapes"]))
    assert float(enc.mid.attn_1.proj_out.weight.detach().abs().max()) > 0          # derandomised: not the reference's zeros
    S = vt.RodinSR_256_fusionv6_ConvQuant_liteSR_dinoInit3DAttn_SD_B_3L_C_withrollout_withSD_D_ditDecoder_S
    for arch, D, tag in (("DiT2-B/2", 768, "B"), ("DiT2-L/2", 1024, "L")):
        with torch.device("meta"):
            vd = DiT2_models[arch](input_size=16, num_classes=0, learn_sigma=False, in_channels=D, mixed_prediction=False,
                                   context_dim=None, roll_out=True, plane_n=3, return_all_layers=False)
            tri = Triplane(c_dim=25, img_resolution=128, img_channels=3, out_chans=96, triplane_size=224,
                           rendering_kwargs=dict(OBJAVERSE_RENDERING_KWARGS), decoder_in_chans=32, decoder_output_dim=3)
            dec = S(vd, tri, False, vae_p=2, ldm_z_channels=4, ldm_embed_dim=4)
        assert {k: list(v.shape) for k, v in dec.state_dict().items()} == json.loads(str(g["decoder_shapes_" + tag]))


def test_encoder_has_no_cpu_fallback_and_unbuilt_branches_raise():
    from ln3diff_b200.ldm.modules.diffusionmodules import model as M
    from ln3diff_b200.utils import build_ae_decoder, build_ae_encoder
    enc = build_ae_encoder()
    with pytest.raises(RuntimeError, match="CUDA only"):
        enc(torch.zeros(4, 10, 64, 64))
    dec = build_ae_decoder("DiT2-S/2")
    with pytest.raises(RuntimeError, match="CUDA only"):
        dec.vae_reparameterization(torch.zeros(1, 24, 32, 32), True)
    for cls in (M.MVEncoderGS, M.MVEncoderGSDynamicInp):
        with pytest.raises(NotImplementedError):
            cls(ch=64, out_ch=3, num_res_blocks=1, attn_resolutions=[], in_channels=10, resolution=256, z_channels=12)
    with pytest.raises(NotImplementedError):
        M.MVEncoder(ch=64, out_ch=3, num_res_blocks=1, attn_resolutions=[32], in_channels=10, resolution=256,
                    z_channels=12, attn_kwargs={"n_heads": 8, "d_head": 64})


def test_prepare_is_invalidated_by_load_state_dict_and_to():
    from ln3diff_b200.utils import build_ae_encoder
    enc = build_ae_encoder()
    enc._prep = {"stale": True}
    enc.load_state_dict(enc.state_dict())
    assert enc._prep is None
    enc._prep = {"stale": True}
    enc.to(torch.float32)
    assert enc._prep is None


def test_reference_create_3dae_model_builds_the_encoder_mirror_under_the_overlay():
    """The reference's unmodified create_3DAE_model(dino_version='mv-sd-dit', encoder_in_channels=10, ...) returns an AE
    whose encoder is the MVEncoder mirror and whose decoder is the `_S` mirror; AE.forward(behaviour='encoder_vae')
    reaches the mirror (which refuses CPU tensors)."""
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
    from ln3diff_b200.utils import OBJAVERSE_RENDERING_KWARGS
    _stubs.install()
    overlay.install()
    try:
        n = importlib.import_module("nsr.script_util")
        cls = "vit.vit_triplane.RodinSR_256_fusionv6_ConvQuant_liteSR_dinoInit3DAttn_SD_B_3L_C_withrollout_withSD_D_ditDecoder_S"
        ae = n.create_3DAE_model(arch_encoder="vits", arch_decoder="vitb", dino_version="mv-sd-dit", img_size=[256],
                                 encoder_in_channels=10, sd_E_ch=64, sd_E_num_res_blocks=1, z_channels=12, num_frames=4,
                                 ae_classname=cls, arch_dit_decoder="DiT2-B/2", embed_dim=768, vae_p=2, ldm_z_channels=4,
                                 ldm_embed_dim=4, out_chans=96, decoder_in_chans=32, decoder_output_dim=3,
                                 image_size=128, rendering_kwargs=dict(OBJAVERSE_RENDERING_KWARGS), no_dim_up_mlp=True)
        assert type(ae.encoder).__module__ == "ln3diff_b200.ldm.modules.diffusionmodules.model"
        assert type(ae.encoder).__name__ == "MVEncoder" and ae.encoder.num_frames == 4
        assert type(ae.decoder).__module__ == "ln3diff_b200.vit.vit_triplane"
        with pytest.raises(RuntimeError, match="CUDA only"):
            ae(img=torch.zeros(4, 10, 256, 256), behaviour="encoder_vae")
    finally:
        overlay.uninstall()
        for k in list(sys.modules):
            if k.split(".")[0] in prefixes:
                del sys.modules[k]
        sys.modules.update(saved)
        sys.path[:] = saved_path


def test_bench_flop_count_matches_the_shapes():
    """tools/vae_encode_bench.py's algorithmic count: ~234 GFLOP per object at 4 x 256^2 (36 GF of convs per view,
    ~22 GF of transformer per view, the 4096-token attn1 core 34 GF per object), linear in the object count."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("vae_encode_bench", os.path.join(ROOT, "tools", "vae_encode_bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    per_obj = bench.encoder_flops(1)
    assert 2.2e11 < per_obj < 2.5e11, per_obj
    assert bench.encoder_flops(8) == 8 * per_obj


# ------------------------------------------------------------------ the C boundary
def test_vae_posterior_ctypes_struct_matches_header():
    import re
    from ln3diff_b200 import _lib
    src = open(os.path.join(ROOT, "include", "ln3b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    body = re.search(r"typedef struct ln3_vae_posterior_args\s*\{(.*?)\}\s*ln3_vae_posterior_args;", src,
                     flags=re.S).group(1)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            decl = re.sub(r"^(const\s+)?[A-Za-z_0-9]+\s*\**", "", decl, count=1)
            names += [n.strip().lstrip("*") for n in decl.split(",")]
    assert names == [f[0] for f in _lib.VaePosteriorArgs._fields_]


EINVAL, ECUDA = -1, -2
BASE = 1 << 36


def _addr(i: int) -> int:
    return BASE + i * (1 << 24)


@pytest.fixture
def lib(built_lib):
    if torch.cuda.is_available():
        pytest.skip("fabricated addresses: the control call must not reach a real device")
    from ln3diff_b200 import _lib
    return _lib.lib()


def _call(lib, fn, args):
    rc = getattr(lib, fn)(C.byref(args), C.c_void_p(0))
    return rc, lib.ln3_last_error().decode(errors="replace")


def _ds_args(**over):
    from ln3diff_b200._lib import MLP_TF32, ConvArgs
    a = ConvArgs()
    a.x, a.w, a.bias, a.out = _addr(1), _addr(2), _addr(3), _addr(4)
    a.N, a.H, a.W, a.Cin, a.Cout, a.ksize, a.precision = 4, 256, 256, 64, 64, 3, MLP_TF32
    for k, v in over.items():
        setattr(a, k, v)
    return a


def test_downsample_control_calls_pass_validation(lib):
    from ln3diff_b200._lib import MLP_FP32
    for over in ({}, dict(precision=MLP_FP32), dict(H=2, W=2), dict(Cin=10, Cout=24), dict(H=18, W=34), dict(bias=None)):
        rc, msg = _call(lib, "ln3_downsample_nhwc", _ds_args(**over))
        assert rc == ECUDA, (over, rc, msg)


@pytest.mark.parametrize("over,match", [
    (dict(H=255), "even"),
    (dict(W=17), "even"),
    (dict(ksize=1), "ksize"),
    (dict(upsample=1), "upsample"),
    (dict(in_scale=_addr(5), in_shift=_addr(6)), "in_scale"),
    (dict(in_shift=_addr(6)), "in_scale"),
    (dict(residual=_addr(7)), "residual"),
    (dict(precision=2), "precision"),
    (dict(Cin=0), "positive"),
    (dict(Cout=-1), "positive"),
    (dict(H=0), "positive"),
    (dict(N=-1), "N >= 0"),
    (dict(x=None), "null"),
    (dict(w=None), "null"),
    (dict(out=None), "null"),
])
def test_downsample_rejects_bad_arguments(lib, over, match):
    rc, msg = _call(lib, "ln3_downsample_nhwc", _ds_args(**over))
    assert rc == EINVAL and match in msg, (over, rc, msg)


def _vp_args(**over):
    from ln3diff_b200._lib import VaePosteriorArgs
    a = VaePosteriorArgs()
    for i, name in enumerate(("moments", "w", "bias", "noise", "mean", "logvar", "z")):
        setattr(a, name, _addr(i + 1))
    a.B, a.S = 2, 32
    for k, v in over.items():
        setattr(a, k, v)
    return a


def test_vae_posterior_control_calls_pass_validation(lib):
    for over in ({}, dict(noise=None), dict(B=1, S=1)):
        rc, msg = _call(lib, "ln3_vae_posterior", _vp_args(**over))
        assert rc == ECUDA, (over, rc, msg)


@pytest.mark.parametrize("over,match", [
    (dict(B=-1), "B >= 0"),
    (dict(S=0), "S > 0"),
    (dict(moments=None), "null"),
    (dict(w=None), "null"),
    (dict(bias=None), "null"),
    (dict(mean=None), "null"),
    (dict(logvar=None), "null"),
    (dict(z=None), "null"),
])
def test_vae_posterior_rejects_bad_arguments(lib, over, match):
    rc, msg = _call(lib, "ln3_vae_posterior", _vp_args(**over))
    assert rc == EINVAL and match in msg, (over, rc, msg)


def test_python_checks_reject_cpu_and_odd_inputs():
    from ln3diff_b200 import ops
    with pytest.raises(ValueError, match="CUDA"):
        ops.downsample_nhwc(torch.zeros(1, 8, 8, 16), torch.zeros(9, 16, 16), None)
    with pytest.raises(ValueError, match="CUDA"):
        ops.vae_posterior(torch.zeros(1, 32, 32, 24), torch.zeros(24, 8), torch.zeros(24))
