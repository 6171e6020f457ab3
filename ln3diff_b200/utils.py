"""Small host utilities shared by bench.py, smoke() and the tests (no oracle imports here)."""
from __future__ import annotations

import torch


def host_cores() -> int:
    """Threads this process may actually use: the scheduler affinity mask capped by the cgroup CPU quota
    (os.cpu_count() reports the whole node; oversubscribing a 16-core lease with 128 threads is ~20x slower)."""
    import os
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period))))
    except Exception:
        pass
    return max(1, n)


def derandomize_zero_init(module: torch.nn.Module, std: float = 0.02, seed: int = 1234) -> None:
    """adaLN-Zero + the zero-initialised final layer make a freshly constructed DiT output exactly
    0 (reference dit/dit_models_xformers.py:807-819).  There are no checkpoints offline, so
    benchmarks / tests replace every all-zero floating parameter by N(0, std^2), in sorted key
    order from a CPU generator (identical to oracle.dit.derandomize_zero_init)."""
    g = torch.Generator().manual_seed(seed)
    sd = module.state_dict()
    new = {}
    for k in sorted(sd.keys()):
        v = sd[k]
        if v.is_floating_point() and v.numel() > 0 and float(v.abs().max()) == 0.0:
            new[k] = (torch.randn(v.shape, generator=g, dtype=torch.float32) * std).to(v.device, v.dtype)
    if new:
        sd.update(new)
        module.load_state_dict(sd)


def build_t23d(arch: str = "DiT-L/2", seed: int = 0, device: str | None = None):
    """DiT as the reference's create_model_and_diffusion builds it for T23D
    (guided_diffusion/script_util.py:407-415), random-init + derandomised zero tensors."""
    from .dit.dit_models_xformers import TextCondDiTBlock
    from .dit.dit_trilatent import DiT_models
    torch.manual_seed(seed)
    m = DiT_models[arch](input_size=32, num_classes=0, learn_sigma=False, in_channels=4,
                         context_dim=768, roll_out=True, vit_blk=TextCondDiTBlock)
    derandomize_zero_init(m)
    m.eval()
    return m.to(device) if device else m


def build_i23d(arch: str = "DiT-PixArt-L/2", seed: int = 0, device: str | None = None):
    """I23D denoiser as the release builds it (DiT_models_i23d[arch](..., context_dim=1024,
    pooling_ctx_dim=768), guided_diffusion/script_util.py:152-252)."""
    from .dit.dit_i23d import DiT_models
    torch.manual_seed(seed)
    m = DiT_models[arch](input_size=32, num_classes=0, learn_sigma=False, in_channels=4, context_dim=1024,
                         pooling_ctx_dim=768, roll_out=True)
    derandomize_zero_init(m)
    m.eval()
    return m.to(device) if device else m


def build_mv23d(arch: str = "DiT-PixArt-MV-L/2", seed: int = 0, device: str | None = None, **kwargs):
    """Multi-view denoiser as the MV23D release builds it (DiT_models_i23d['DiT-PixArt-MV-L/2'](...,
    context_dim=768, pooling_ctx_dim=768, learn_sigma=False), guided_diffusion/script_util.py:397-406);
    `kwargs` override the registry sizes (depth, hidden_size, num_heads) for reduced test models."""
    from .dit.dit_i23d import DiT_I23D_PixelArt_MVCond_noClip, DiT_models
    torch.manual_seed(seed)
    args = dict(input_size=32, num_classes=0, learn_sigma=False, in_channels=4, context_dim=768, pooling_ctx_dim=768,
                roll_out=True)
    if kwargs:
        m = DiT_I23D_PixelArt_MVCond_noClip(patch_size=2, **{**args, **kwargs})
    else:
        m = DiT_models[arch](**args)
    derandomize_zero_init(m)
    m.eval()
    return m.to(device) if device else m


def orbit_cameras(V: int, radius: float = 1.7, focal: float = 1.3889) -> torch.Tensor:
    """(V, 25) synthetic camera rows in the layout of the reference's assets/objv_eval_pose.pt:
    16 row-major cam2world (OpenCV convention, looking at the origin) + 9 normalised intrinsics
    (fx = fy = 1.3889, cx = cy = 0.5)."""
    import math
    cams = []
    for v in range(V):
        az = 2 * math.pi * v / max(V, 1) + 0.3
        el = 0.35 + 0.2 * ((v % 3) - 1)
        eye = torch.tensor([radius * math.cos(el) * math.cos(az), radius * math.cos(el) * math.sin(az),
                            radius * math.sin(el)])
        fwd = -eye / eye.norm()
        right = torch.linalg.cross(fwd, torch.tensor([0.0, 0.0, 1.0]))
        right = right / right.norm()
        down = torch.linalg.cross(fwd, right)
        c2w = torch.eye(4)
        c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = right, down, fwd, eye
        K = torch.tensor([focal, 0, 0.5, 0, focal, 0.5, 0, 0, 1.0])
        cams.append(torch.cat([c2w.reshape(-1), K]))
    return torch.stack(cams).float()


OBJAVERSE_RENDERING_KWARGS = dict(  # nsr/script_util.py:433-465,761-797 (resolved preset, SURVEY appendix C)
    image_resolution=256, disparity_space_sampling=False, clamp_mode="softplus", c_gen_conditioning_zero=True,
    c_scale=1, superresolution_noise_mode="none", density_reg=0.25, density_reg_p_dist=0.004, reg_type="l1",
    decoder_lr_mul=1, decoder_activation="sigmoid", sr_antialias=True, return_triplane_features=False,
    return_sampling_details_flag=True, depth_resolution=64, depth_resolution_importance=64, ray_start="auto",
    ray_end="auto", box_warp=0.9, white_back=True, radius_range=[1.5, 2], sampler_bbox_min=-0.45,
    sampler_bbox_max=0.45, filter_out_of_bbox=True, PatchRaySampler=True, patch_rendering_resolution=45,
    z_near=1.05, z_far=2.45)


def build_ae_decoder(arch: str = "DiT2-L/2", image_size: int = 128, seed: int = 0, device: str | None = None,
                     depth_resolution: int = 64):
    """The AE decoder as create_3DAE_model assembles it for the Objaverse release
    (nsr/script_util.py:1355-1429): Triplane renderer + DiT2 backbone + SD conv upsampler.  depth_resolution sets
    the coarse and the importance samples per ray: 64 (objaverse_tuneray_aug_resolution_64_64_auto) or 96 (the
    96_96 preset of the DiT2-L/2 VAE's reconstruction script, nsr/script_util.py:838-870)."""
    from .dit.dit_decoder import DiT2_models
    from .nsr.triplane import Triplane
    from .vit.vit_triplane import (
        RodinSR_256_fusionv6_ConvQuant_liteSR_dinoInit3DAttn_SD_B_3L_C_withrollout_withSD_D_ditDecoder as AEDec)
    torch.manual_seed(seed)
    D = {"DiT2-L/2": 1024, "DiT2-L/2-half": 1024, "DiT2-B/2": 768, "DiT2-S/2": 384}[arch]
    vd = DiT2_models[arch](input_size=16, num_classes=0, learn_sigma=False, in_channels=D, mixed_prediction=False,
                           context_dim=None, roll_out=True, plane_n=3, return_all_layers=False)
    tri = Triplane(c_dim=25, img_resolution=image_size, img_channels=3, out_chans=96, triplane_size=224,
                   rendering_kwargs=dict(OBJAVERSE_RENDERING_KWARGS, depth_resolution=depth_resolution,
                                         depth_resolution_importance=depth_resolution),
                   decoder_in_chans=32, decoder_output_dim=3)
    m = AEDec(vd, tri, False, vae_p=2, ldm_z_channels=4, ldm_embed_dim=4)
    derandomize_zero_init(m)
    m.eval()
    return m.to(device) if device else m


def build_ae_encoder(seed: int = 0, device: str | None = None, ch: int = 64, num_res_blocks: int = 1,
                     in_channels: int = 10, dino_version: str = "mv-sd-dit", num_frames: int | None = None):
    """The stage-1 encoder as create_3DAE_model builds it (nsr/script_util.py:1294-1339) with the release scripts'
    sd_E_ch=64, sd_E_num_res_blocks=1: encoder_cls(double_z=True, resolution=256, in_channels=10, ch_mult=[1,2,4,4],
    z_channels=12, attn_kwargs={'n_heads': 8, 'd_head': 64}).  encoder_cls is MVEncoder for dino_version 'mv-sd-dit'
    (4 views) and MVEncoderGSDynamicInp for 'mv-sd-dit-dynaInp-trilatent' (the DiT2-L/2 VAE; num_frames defaults to
    the release scripts' 6).  Random init; the zero-initialised proj_out of the mid-block transformer is re-randomised
    (derandomize_zero_init), otherwise the whole transformer would be multiplied by zero."""
    from .ldm.modules.diffusionmodules.model import MVEncoder, MVEncoderGSDynamicInp
    if dino_version == "mv-sd-dit":
        cls, num_frames = MVEncoder, 4 if num_frames is None else num_frames
    elif dino_version == "mv-sd-dit-dynaInp-trilatent":
        cls, num_frames = MVEncoderGSDynamicInp, 6 if num_frames is None else num_frames
    else:
        raise NotImplementedError(f"dino_version {dino_version!r}: only the release VAE encoders are built")
    torch.manual_seed(seed)
    m = cls(double_z=True, resolution=256, in_channels=in_channels, ch=ch, ch_mult=[1, 2, 4, 4],
            num_res_blocks=num_res_blocks, num_frames=num_frames, dropout=0.0, attn_resolutions=[], out_ch=3,
            z_channels=12, attn_kwargs={"n_heads": 8, "d_head": 64})
    derandomize_zero_init(m)
    m.eval()
    return m.to(device) if device else m
