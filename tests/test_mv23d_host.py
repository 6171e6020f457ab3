"""CPU: the multi-view-to-3D (MV23D) path -- the oracle restatements against the reference's recorded output
(tests/golden/mv23d.npz, tools/make_golden_mv23d.py), the DiT-PixArt-MV-L/2 mirror's checkpoint layout and registry,
the conditioner's camera augmentation, and the host-side checks of ln3_plucker_patchify."""
import ctypes as C
import json
import os
import random
import re

import numpy as np
import pytest
import torch

import mv23d_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


def _mirror_mv(**kw):
    from ln3diff_b200.dit.dit_i23d import DiT_I23D_PixelArt_MVCond_noClip
    return DiT_I23D_PixelArt_MVCond_noClip(input_size=32, patch_size=2, in_channels=4, num_classes=0, learn_sigma=False,
                                           context_dim=768, pooling_ctx_dim=768, roll_out=True, **kw)


def test_oracle_mv_forward_matches_reference_golden(golden):
    g = golden("mv23d.npz")
    m = _mirror_mv(hidden_size=mo.MV_HIDDEN, depth=mo.MV_DEPTH, num_heads=mo.MV_HEADS)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = mo.mv_state_dict(shapes, m.state_dict()["pos_embed"])
    x, t, ctx = mo.mv_inputs()
    out = mo.mv_noclip_forward(sd, x, t, ctx, mo.MV_HEADS)
    assert _rel(out, g["out"]) < 1e-5
    cond, unc = out.chunk(2)
    half = unc + 4.0 * (cond - unc)
    assert _rel(torch.cat([half, half]), g["out_cfg"]) < 1e-5
    # the conditional and the zero-context rows really differ: the cross-attention is exercised
    assert _rel(cond, unc) > 1e-2


def test_oracle_plucker_rays_match_reference_golden(golden):
    """The torch restatement of gen_rays / get_plucker_ray (CPU: fp32, as the reference runs without autocast) and the
    float64 restatement agree with the reference's own rays on translated, rotated and skewed cameras."""
    g = golden("mv23d.npz")
    cams = torch.from_numpy(g["ray_cams"])
    ref = torch.from_numpy(g["rays_strided"]).double()
    rays = mo.plucker_rays(cams)[:, :, ::7, ::7]
    assert torch.allclose(rays.double(), ref, rtol=0, atol=2e-6)
    # float64 without the bf16 rounding points (R and dir exact): fp32 rounding only
    c = cams.double()
    f64 = mo.plucker_rays_f64(c)
    assert (f64["d"][:, :, ::7, ::7] - ref[:, 3:]).abs().max() < 2 ** -7       # bf16 rounding of |d| <= 1
    assert ref.shape == (4, 6, 32, 32) and float(ref[:, 3:].norm(dim=1).sub(1).abs().max()) < 1e-5


def test_camera_augmentation_matches_reference_draws(golden):
    """aug_c: the mirror rotates the same cameras with the same angles and axes as the reference, in place, and leaves
    both Python `random` and NumPy's global generator where the reference leaves them."""
    from ln3diff_b200.sgm.modules.encoders.modules import FrozenDinov2ImageEmbedderMVPlucker as E
    g = golden("mv23d.npz")
    c = torch.from_numpy(g["aug_in"]).clone()
    ptr = c.data_ptr()
    random.seed(1234)
    np.random.seed(4321)
    out = E.augment_cameras(c)
    assert out is c and c.data_ptr() == ptr
    assert torch.allclose(c, torch.from_numpy(g["aug_out"]), rtol=0, atol=1e-6)
    assert [random.random() for _ in range(4)] == g["aug_next_py"].tolist()
    assert np.random.uniform(size=4).tolist() == g["aug_next_np"].tolist()
    changed = (torch.from_numpy(g["aug_in"]) != c).any(-1)
    assert 0 < int(changed.sum()) < 12
    assert torch.equal(c[..., 16:], torch.from_numpy(g["aug_in"])[..., 16:])   # intrinsics untouched


def test_mirror_state_dict_matches_reference_layout(golden):
    """Every key and shape of the reference's DiT-PixArt-MV-L/2, including the unused attention_y_norm tensors."""
    from ln3diff_b200.dit.dit_i23d import DiT_models
    ref = json.loads(str(golden("mv23d.npz")["mv_l2_shapes"]))
    with torch.device("meta"):
        m = DiT_models["DiT-PixArt-MV-L/2"](input_size=32, num_classes=0, learn_sigma=False, in_channels=4,
                                            context_dim=768, pooling_ctx_dim=768, roll_out=True)
    mine = {k: list(v.shape) for k, v in m.state_dict().items()}
    assert mine == ref
    assert "blocks.0.attention_y_norm.weight" in mine and "attention_y_norm.weight" in mine
    assert not any(k.startswith(("cap_embedder", "dino_proj", "clip_spatial_proj")) for k in mine)


def test_registry_builds_mv_l2_and_keeps_other_mv_keys_unbuilt():
    from ln3diff_b200.dit.dit_i23d import (DiT_I23D_PixelArt_MVCond_noClip, DiT_models,
                                           ImageCondDiTBlockPixelArtRMSNormNoClip)
    with torch.device("meta"):
        m = DiT_models["DiT-PixArt-MV-L/2"](input_size=32, num_classes=0, learn_sigma=False, in_channels=4,
                                            context_dim=768, pooling_ctx_dim=768, roll_out=True)
    assert type(m) is DiT_I23D_PixelArt_MVCond_noClip and type(m.blocks[0]) is ImageCondDiTBlockPixelArtRMSNormNoClip
    assert (m.depth, m.embed_dim, m.num_heads) == (24, 1024, 16)
    for k in ("DiT-PixArt-MV-B/2", "DiT-PixArt-MV-XL/2", "DiT-PixArt-MV-PCD-L"):
        with pytest.raises(NotImplementedError):
            DiT_models[k](input_size=32, num_classes=0, learn_sigma=False, in_channels=4, context_dim=768, roll_out=True)


def test_mv_denoiser_has_no_cpu_fallback():
    m = _mirror_mv(hidden_size=128, depth=1, num_heads=2)
    x, t, _ = mo.mv_inputs()
    with pytest.raises(RuntimeError, match="CUDA only"):
        m(x, t, {"concat": torch.zeros(2, 1, 256, 768)})


def test_conditioner_rejects_training_augmentation_and_unreachable_weights(monkeypatch):
    from ln3diff_b200.sgm.modules.encoders import modules as M
    with pytest.raises(RuntimeError, match="pretrained loader failed"):
        monkeypatch.setattr(torch.hub, "load", lambda *a, **k: (_ for _ in ()).throw(OSError("no network")))
        M.FrozenDinov2ImageEmbedderMVPlucker(arch="vitb", n_cond_frames=6, enable_bf16=True, aug_c=True, device="cpu")
    e = M.FrozenDinov2ImageEmbedderMVPlucker.__new__(M.FrozenDinov2ImageEmbedderMVPlucker)
    torch.nn.Module.__init__(e)
    e._ucg_rate = 0.1
    with pytest.raises(NotImplementedError, match="training-time augmentation"):
        e.preprocess(torch.zeros(1, 3, 256, 256))


def test_nine_channel_patch_embed_surgery():
    """A 3-channel (hub) patch embedding becomes the reference's zero-padded 9-channel one; 9-channel weights pass."""
    from ln3diff_b200.sgm.modules.encoders.modules import _nine_channel_patch_embed
    w3 = torch.randn(8, 3, 14, 14)
    sd = _nine_channel_patch_embed({"model.patch_embed.proj.weight": w3, "model.patch_embed.proj.bias": torch.ones(8)})
    w9 = sd["model.patch_embed.proj.weight"]
    assert w9.shape == (8, 9, 14, 14) and torch.equal(w9[:, :3], w3) and not w9[:, 3:].any()
    assert torch.equal(sd["model.patch_embed.proj.bias"], torch.ones(8))
    w = torch.randn(8, 9, 14, 14)
    assert _nine_channel_patch_embed({"patch_embed.proj.weight": w})["patch_embed.proj.weight"] is w


def test_reference_factory_builds_the_mv_mirror_under_the_overlay():
    """The reference's unmodified create_model_and_diffusion(i23d=True, dit_model_arch='DiT-PixArt-MV-L/2',
    context_dim=768, ...) returns the mirror class when the overlay is installed."""
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
        g = importlib.import_module("guided_diffusion.script_util")
        d = g.model_and_diffusion_defaults()
        d.update(dict(create_dit=True, i23d=True, dit_model_arch="DiT-PixArt-MV-L/2", context_dim=768,
                      pooling_ctx_dim=768, roll_out=True, denoise_in_channels=4, denoise_out_channels=4,
                      diffusion_input_size=32, learn_sigma=False, mixed_prediction=False, timestep_respacing="10"))
        with torch.device("meta"):
            model, _ = g.create_model_and_diffusion(**d)
        assert type(model).__module__ == "ln3diff_b200.dit.dit_i23d"
        assert type(model).__name__ == "DiT_I23D_PixelArt_MVCond_noClip" and model.depth == 24
    finally:
        overlay.uninstall()
        for k in list(sys.modules):
            if k.split(".")[0] in prefixes:
                del sys.modules[k]
        sys.modules.update(saved)
        sys.path[:] = saved_path


# ------------------------------------------------------------------ ln3_plucker_patchify at the C boundary
def test_plucker_patchify_ctypes_struct_matches_header():
    from ln3diff_b200 import _lib
    src = open(os.path.join(ROOT, "include", "ln3b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    body = re.search(r"typedef struct ln3_plucker_patchify_args\s*\{(.*?)\}\s*ln3_plucker_patchify_args;", src,
                     flags=re.S).group(1)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if not decl:
            continue
        decl = re.sub(r"^(const\s+)?(unsigned\s+)?[A-Za-z_0-9]+(\s+long)?\s*\**", "", decl, count=1)
        names += [re.sub(r"\[.*?\]", "", n).strip().lstrip("*") for n in decl.split(",")]
    assert names == [f[0] for f in _lib.PluckerPatchifyArgs._fields_]


EINVAL, ECUDA = -1, -2
BASE = 1 << 36


def _pp_args(**over):
    from ln3diff_b200._lib import PluckerPatchifyArgs
    a = PluckerPatchifyArgs()
    a.image, a.cams, a.out = BASE + (1 << 24), BASE + 2 * (1 << 24), BASE + 3 * (1 << 24)
    a.N, a.ldo = 6, 1792
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.fixture
def lib(built_lib):
    if torch.cuda.is_available():
        pytest.skip("fabricated addresses: the control call must not reach a real device")
    from ln3diff_b200 import _lib
    return _lib.lib()


def _call(lib, args):
    rc = lib.ln3_plucker_patchify(C.byref(args), C.c_void_p(0))
    return rc, lib.ln3_last_error().decode(errors="replace")


def test_plucker_patchify_control_call_passes_validation(lib):
    for over in ({}, dict(ldo=1768), dict(ldo=2048), dict(N=1)):
        rc, msg = _call(lib, _pp_args(**over))
        assert rc == ECUDA, (over, rc, msg)


@pytest.mark.parametrize("over,match", [
    (dict(ldo=1760), "ldo"),              # narrower than the 1764 operand columns
    (dict(ldo=1796), "ldo"),              # wide enough, not a multiple of 8
    (dict(ldo=0), "ldo"),
    (dict(N=-1), "N < 0"),
    (dict(image=None), "null"),
    (dict(cams=None), "null"),
    (dict(out=None), "null"),
    (dict(image=BASE + (1 << 24) + 4), "16-byte aligned"),
    (dict(cams=BASE + 2 * (1 << 24) + 8), "16-byte aligned"),
    (dict(out=BASE + 3 * (1 << 24) + 2), "16-byte aligned"),
])
def test_plucker_patchify_rejects_bad_arguments(lib, over, match):
    rc, msg = _call(lib, _pp_args(**over))
    assert rc == EINVAL and match in msg, (over, rc, msg)


def test_plucker_patchify_python_checks():
    """ops.plucker_patchify validates before any device call (CPU tensors are rejected first)."""
    from ln3diff_b200 import ops
    with pytest.raises(ValueError, match="CUDA"):
        ops.plucker_patchify(torch.zeros(1, 3, 224, 224), torch.zeros(1, 25))
