"""TEST INFRASTRUCTURE ONLY -- CPU restatements for the multi-view-to-3D (MV23D) path, shared by
tests/test_mv23d_host.py, tests/test_gpu_mv23d.py and tools/make_golden_mv23d.py.  The product package never
imports this module.

  mv_noclip_forward    DiT_I23D_PixelArt_MVCond_noClip.forward (dit/dit_i23d.py:392-492) with
                       ImageCondDiTBlockPixelArtRMSNormNoClip blocks (dit/dit_models_xformers.py:541-601,621-635), fp32
  plucker_rays         FrozenDinov2ImageEmbedderMVPlucker.gen_rays + get_plucker_ray
                       (sgm/modules/encoders/modules.py:955-1005), op for op in torch: run on the CPU it is the
                       reference's fp32 arithmetic; run on CUDA under torch.autocast(bf16) it takes the reference's
                       release rounding (the engine's use_amp autocast)
  plucker_rays_f64     the same rays in float64 with the bf16 rounding points of the release configuration
  dinov2_reg9          transformers' Dinov2WithRegistersModel with num_channels=9, renamed to the hub key layout
Pinned against the reference's own code by tests/golden/mv23d.npz (tools/make_golden_mv23d.py).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

MV_DEPTH, MV_HIDDEN, MV_HEADS, MV_CONTEXT = 3, 768, 12, 768    # reduced denoiser of the golden
MV_VIEWS = 3


def mv_inputs():
    """Seeded inputs of the MV golden: x (2,12,32,32), t (2,), concat (2, V, 256, 768) whose second (unconditional)
    row is all zero, as GeneralConditioner's force_uc_zero_embeddings makes it."""
    g = torch.Generator().manual_seed(23)
    x = torch.randn(2, 12, 32, 32, generator=g)
    t = torch.tensor([0.2, 0.2])
    concat = torch.randn(2, MV_VIEWS, 256, MV_CONTEXT, generator=g)
    concat[1] = 0
    return x, t, {"concat": concat}


def mv_state_dict(shapes: dict, pos_embed: torch.Tensor) -> dict:
    from oracle import fixtures as fx
    return fx.i23d_state_dict(shapes, pos_embed)


def mv_noclip_forward(sd: dict, x: torch.Tensor, timesteps: torch.Tensor, context: dict, heads: int) -> torch.Tensor:
    """fp32 forward of DiT_I23D_PixelArt_MVCond_noClip: t = t_embedder(t) (no pooled embedding), shared adaLN +
    per-block scale_shift_table, RMSNorm pre-norms, q/k-normed self-attention over the latent tokens only, q/k-normed
    cross-attention to the flattened DINO tokens (no attention_y_norm), T2IFinalLayer."""
    from oracle import dit as odit
    sd = {k: v.float() for k, v in sd.items()}
    depth = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))
    x = x.float()
    B = x.shape[0]
    ctx = context["concat"].float()
    dino = ctx.reshape(B, -1, ctx.shape[-1])                            # 'b v l c -> b (v l) c'
    t = odit.timestep_embedding(timesteps.float())
    t = F.linear(F.silu(F.linear(t, sd["t_embedder.mlp.0.weight"], sd["t_embedder.mlp.0.bias"])),
                 sd["t_embedder.mlp.2.weight"], sd["t_embedder.mlp.2.bias"])
    t0 = F.linear(F.silu(t), sd["adaLN_modulation.1.weight"], sd["adaLN_modulation.1.bias"])
    h = odit.patch_embed_rollout(sd, x) + sd["pos_embed"]
    for i in range(depth):
        p = f"blocks.{i}."
        mod = sd[p + "scale_shift_table"][None] + t0.reshape(B, 6, -1)
        sh_a, sc_a, g_a, sh_m, sc_m, g_m = mod.chunk(6, dim=1)
        a_in = odit.rms_norm(h, sd[p + "norm1.weight"], 1e-5) * (1 + sc_a) + sh_a
        h = h + g_a * odit.self_attention(sd, p + "attn.", a_in, heads, qk_norm=True)
        h = h + odit.cross_attention(sd, p + "cross_attn.", h, dino, heads, qk_norm=True)
        h = h + g_m * odit.fused_mlp(sd, p + "mlp.", odit.rms_norm(h, sd[p + "norm2.weight"], 1e-5) * (1 + sc_m) + sh_m)
    shift, scale = (sd["final_layer.scale_shift_table"][None] + t[:, None]).chunk(2, dim=1)
    h = odit.layer_norm(h) * (1 + scale) + shift
    h = F.linear(h, sd["final_layer.linear.weight"], sd["final_layer.linear.bias"])
    return odit.unpatchify_rollout(h, sd["final_layer.linear.weight"].shape[0] // 4).contiguous()


# ------------------------------------------------------------------ cameras and rays
def ray_cameras() -> torch.Tensor:
    """(4, 25) camera rows exercising every term of the ray formula: an orbit camera, a translated and rotated one,
    one with skewed intrinsics (fx != fy, off-centre principal point) and an identity pose."""
    from ln3diff_b200.utils import orbit_cameras
    cams = orbit_cameras(3).double()
    rot = cams[1].clone()
    a = 0.7
    Rz = torch.tensor([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]], dtype=torch.float64)
    c2w = rot[:16].reshape(4, 4)
    c2w[:3, :3] = Rz @ c2w[:3, :3]
    c2w[:3, 3] += torch.tensor([0.31, -0.17, 0.05], dtype=torch.float64)
    rot[:16] = c2w.reshape(-1)
    skew = cams[2].clone()
    skew[16], skew[20], skew[18], skew[21] = 1.91, 1.23, 0.43, 0.58
    ident = torch.cat([torch.eye(4, dtype=torch.float64).reshape(-1),
                       torch.tensor([1.3889, 0, 0.5, 0, 1.3889, 0.5, 0, 0, 1], dtype=torch.float64)])
    ident[3], ident[7], ident[11] = 0.2, -0.4, 1.7
    return torch.stack([cams[0], rot, skew, ident]).float()


def plucker_rays(c: torch.Tensor, res: int = 224) -> torch.Tensor:
    """(N, 25) cameras -> (N, 6, res, res) Plücker rays [o x d, d], the reference's op sequence."""
    out = []
    for cam in c:
        intrinsics, c2w = cam[16:], cam[:16].reshape(4, 4)
        yy, xx = torch.meshgrid(torch.arange(res, dtype=torch.float32, device=c.device) + 0.5,
                                torch.arange(res, dtype=torch.float32, device=c.device) + 0.5, indexing="ij")
        yy, xx = yy / res, xx / res
        cx, cy, fx, fy = intrinsics[2], intrinsics[5], intrinsics[0], intrinsics[4]
        c2w = c2w.float()
        xx = (xx - cx) / fx
        yy = (yy - cy) / fy
        dirs = torch.stack((xx, yy, torch.ones_like(xx)), dim=-1)
        dirs /= torch.norm(dirs, dim=-1, keepdim=True)
        dirs = (c2w[None, :3, :3] @ dirs.reshape(-1, 3, 1))[..., 0]
        o = c2w[None, :3, 3].expand(res * res, -1).contiguous().view(res, res, 3)
        d = dirs.view(res, res, 3)
        out.append(torch.cat([torch.cross(o, d, dim=-1), d], dim=-1).permute(2, 0, 1))
    return torch.stack(out, 0)


def bf16(v: torch.Tensor) -> torch.Tensor:
    return v.to(torch.bfloat16).to(v.dtype)


def plucker_rays_f64(c: torch.Tensor, res: int = 224) -> dict:
    """float64 rays with the release rounding points: bf16 dir and R, bf16 d = R dir, o x d exact, bf16 at the end.
    Returns the rounded channels and the intermediates the tolerances are derived from."""
    c = c.double()
    N = c.shape[0]
    ar = (torch.arange(res, dtype=torch.float64) + 0.5) / res
    v, u = torch.meshgrid(ar, ar, indexing="ij")
    fx, fy, cx, cy = (c[:, k, None, None] for k in (16, 20, 18, 21))
    a, b = (u - cx) / fx, (v - cy) / fy
    nrm = torch.sqrt(a * a + b * b + 1)
    e = torch.stack([a / nrm, b / nrm, 1 / nrm], 1)                       # (N, 3, res, res)
    eb = bf16(e)
    R = bf16(c[:, :16].reshape(N, 4, 4)[:, :3, :3])
    d_exact = torch.einsum("nij,njhw->nihw", R, eb)
    d = bf16(d_exact)
    o = c[:, :16].reshape(N, 4, 4)[:, :3, 3][:, :, None, None].expand_as(d)
    m = torch.linalg.cross(o, d, dim=1)
    return dict(m=m, d=d, d_exact=d_exact, R=R, e=eb, o=o)


def im2col(x: torch.Tensor) -> torch.Tensor:
    """(N, C, 224, 224) -> (N*256, C*196) in Conv2d.weight.reshape(D, -1) column order."""
    N, C = x.shape[:2]
    return x.reshape(N, C, 16, 14, 16, 14).permute(0, 2, 4, 1, 3, 5).reshape(N * 256, C * 196)


def dinov2_reg9(depth=2, width=256, seed=0, init_scale=3.0):
    """transformers' Dinov2WithRegistersModel with a 9-channel patch embedding (RGB + Plücker) -> (HF model,
    state dict in the dinov2 hub layout with the `model.` prefix), as oracle/conditioners.dinov2_reg renames it."""
    from transformers import Dinov2WithRegistersConfig, Dinov2WithRegistersModel
    from oracle.conditioners import _randomize_norms
    torch.manual_seed(seed)
    cfg = Dinov2WithRegistersConfig(hidden_size=width, num_hidden_layers=depth, num_attention_heads=width // 64,
                                    mlp_ratio=4, image_size=224, patch_size=14, num_channels=9, num_register_tokens=4,
                                    layer_norm_eps=1e-6, hidden_act="gelu", initializer_range=0.02 * init_scale,
                                    layerscale_value=1.0)
    m = _randomize_norms(Dinov2WithRegistersModel(cfg).eval().float(), seed)
    h = m.state_dict()
    sd = {"cls_token": h["embeddings.cls_token"], "register_tokens": h["embeddings.register_tokens"],
          "pos_embed": h["embeddings.position_embeddings"],
          "patch_embed.proj.weight": h["embeddings.patch_embeddings.projection.weight"],
          "patch_embed.proj.bias": h["embeddings.patch_embeddings.projection.bias"],
          "norm.weight": h["layernorm.weight"], "norm.bias": h["layernorm.bias"]}
    for i in range(depth):
        s, d = f"encoder.layer.{i}.", f"blocks.{i}."
        sd[d + "attn.qkv.weight"] = torch.cat([h[s + f"attention.attention.{n}.weight"] for n in ("query", "key", "value")])
        sd[d + "attn.qkv.bias"] = torch.cat([h[s + f"attention.attention.{n}.bias"] for n in ("query", "key", "value")])
        for a, b in (("attention.output.dense", "attn.proj"), ("norm1", "norm1"), ("norm2", "norm2"),
                     ("mlp.fc1", "mlp.fc1"), ("mlp.fc2", "mlp.fc2")):
            sd[d + b + ".weight"], sd[d + b + ".bias"] = h[s + a + ".weight"], h[s + a + ".bias"]
        sd[d + "ls1.gamma"], sd[d + "ls2.gamma"] = h[s + "layer_scale1.lambda1"], h[s + "layer_scale2.lambda1"]
    return m, {"model." + k: t for k, t in sd.items()}
