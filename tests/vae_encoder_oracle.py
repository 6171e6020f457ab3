"""Plain torch restatement of the stage-1 VAE encoder path (test infrastructure; runs in the dtype it is given, fp32 or
float64, on any device):

  MVEncoder                ldm/modules/diffusionmodules/model.py:459-577 (ResnetBlock :94-153, Downsample :72-91)
  SpatialTransformer3D     ldm/modules/attention.py:390-463 (BasicTransformerBlock3D, GEGLU FeedForward :54-81)
  vae_encode + posterior   vit/vit_triplane.py:912-933, 1152-1199; utils/torch_utils/distributions/distributions.py

plus the seeded weights and inputs that tools/make_golden_vae_encoder.py feeds the reference's own modules.  Pinned to
tests/golden/vae_encoder.npz on the CPU."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle.decoder import _gn, _resblock, _swish

CH, CH_MULT, NUM_RES_BLOCKS, IN_CH, Z_CH, HEADS, D_HEAD, VIEWS = 64, (1, 2, 4, 4), 1, 10, 12, 8, 64, 4
N_OBJ, RES = 2, 256
NOISE_SEED = 31                      # torch.manual_seed before the reference's posterior.sample()
MID_STRIDE = 8                       # the golden keeps every 8th pixel of the mid-block transformer output


def enc_state_dict(shapes: dict, seed: int = 7) -> dict:
    """Seeded weights for every key of the encoder (sorted key order, one CPU generator): conv / linear weights
    N(0, 1/fan_in), biases N(0, 0.02^2), norm weights 1 + N(0, 0.1^2), norm biases N(0, 0.1^2).  Nothing is zero, so
    the reference's zero-initialised proj_out is covered."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k in sorted(shapes):
        shp = tuple(shapes[k])
        norm = "norm" in k and len(shp) == 1
        if norm and k.endswith("weight"):
            v = 1 + 0.1 * torch.randn(shp, generator=g)
        elif norm or k.endswith("bias"):
            v = (0.1 if norm else 0.02) * torch.randn(shp, generator=g)
        else:
            fan_in = int(torch.tensor(shp[1:]).prod())
            v = torch.randn(shp, generator=g) / math.sqrt(fan_in)
        sd[k] = v
    return sd


def quant_conv_params(seed: int = 8):
    """quant_conv = Conv2d(24, 24, 1, groups=3) weights (24, 8, 1, 1) and bias (24,)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(24, 8, 1, 1, generator=g) / math.sqrt(8), 0.1 * torch.randn(24, generator=g)


def enc_inputs(n_obj: int = N_OBJ, res: int = RES, seed: int = 9) -> torch.Tensor:
    """img_to_encoder-like input (n_obj*4, 10, res, res): RGB in [-1, 1], six ray channels in [-1, 1], depth in
    [0.5, 2]."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n_obj * VIEWS, IN_CH, res, res, generator=g) * 2 - 1
    x[:, 9] = 0.5 + 0.75 * (x[:, 9] + 1)
    return x


def posterior_noise(n_obj: int = N_OBJ, S: int = 32) -> torch.Tensor:
    """The draw of the reference's sample() after torch.manual_seed(NOISE_SEED): randn(mean.shape), (B, 4, 3, L)."""
    g = torch.Generator().manual_seed(NOISE_SEED)
    return torch.randn(n_obj, Z_CH // 3, 3, S * S, generator=g).reshape(n_obj, Z_CH, S, S)


# ------------------------------------------------------------------ encoder
def downsample(sd, p, x):
    return F.conv2d(F.pad(x, (0, 1, 0, 1)), sd[p + "conv.weight"], sd[p + "conv.bias"], stride=2)


def _ln(x, sd, p):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], eps=1e-5)


def attention(sd, p, x, heads=HEADS):
    """CrossAttention self-attention: (B, L, C) -> to_out(softmax(q k^T / sqrt(d)) v)."""
    B, L, _ = x.shape
    q, k, v = (F.linear(x, sd[p + n + ".weight"]) for n in ("to_q", "to_k", "to_v"))
    q, k, v = (t.reshape(B, L, heads, -1).transpose(1, 2) for t in (q, k, v))
    a = torch.softmax(q @ k.transpose(-1, -2) * q.shape[-1] ** -0.5, dim=-1) @ v
    return F.linear(a.transpose(1, 2).reshape(B, L, -1), sd[p + "to_out.0.weight"], sd[p + "to_out.0.bias"])


def geglu_ff(sd, p, x):
    h, gate = F.linear(x, sd[p + "net.0.proj.weight"], sd[p + "net.0.proj.bias"]).chunk(2, dim=-1)
    return F.linear(h * F.gelu(gate), sd[p + "net.2.weight"], sd[p + "net.2.bias"])


def spatial_transformer3d(sd, p, x, num_frames=VIEWS, heads=HEADS):
    N, C, H, W = x.shape
    h = F.conv2d(_gn(x, sd[p + "norm.weight"], sd[p + "norm.bias"]), sd[p + "proj_in.weight"], sd[p + "proj_in.bias"])
    D = h.shape[1]
    t = h.reshape(N, D, H * W).transpose(1, 2)                         # 'b c h w -> b (h w) c'
    b = p + "transformer_blocks.0."
    t = t.reshape(N // num_frames, num_frames * H * W, D)              # '(b f) l c -> b (f l) c'
    t = t + attention(sd, b + "attn1.", _ln(t, sd, b + "norm1"), heads)
    t = t.reshape(N, H * W, D)
    t = t + attention(sd, b + "attn2.", _ln(t, sd, b + "norm2"), heads)
    t = t + geglu_ff(sd, b + "ff.", _ln(t, sd, b + "norm3"))
    t = t.transpose(1, 2).reshape(N, D, H, W)
    return F.conv2d(t, sd[p + "proj_out.weight"], sd[p + "proj_out.bias"]) + x


def mv_encoder(sd, x, num_frames=VIEWS, return_mid=False):
    """(B*4, 10, R, R) -> moments (B, 24, R/8, R/8); with return_mid also the mid-block transformer output."""
    h = F.conv2d(x, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    for lvl in range(len(CH_MULT)):
        for b in range(NUM_RES_BLOCKS):
            h = _resblock(sd, f"down.{lvl}.block.{b}.", h)
        if lvl != len(CH_MULT) - 1:
            h = downsample(sd, f"down.{lvl}.downsample.", h)
    h = _resblock(sd, "mid.block_1.", h)
    h = spatial_transformer3d(sd, "mid.attn_1.", h, num_frames)
    mid = h
    h = _resblock(sd, "mid.block_2.", h)
    h = F.conv2d(_swish(_gn(h, sd["norm_out.weight"], sd["norm_out.bias"])), sd["conv_out.weight"], sd["conv_out.bias"],
                 padding=1)
    h = torch.cat([torch.cat(f.chunk(num_frames), dim=1) for f in h.chunk(h.shape[0] // num_frames)], 0)
    out = F.conv2d(h, sd["fusion_layer.weight"], sd["fusion_layer.bias"], padding=1)
    return (out, mid) if return_mid else out


# ------------------------------------------------------------------ posterior
def posterior(qw, qb, moments, noise=None):
    """quant_conv -> reshape (B, 8, 3, H, W) -> chunk -> 20 tanh(lv/20) -> z = mean + exp(0.5 lv) * noise.
    Returns mean, logvar, z in the (B, 12, S, S) layout of latent_normalized_2Ddiffusion."""
    q = F.conv2d(moments, qw, qb, groups=3)
    B, C2, H, W = q.shape
    mean, lv = q.reshape(B, C2 // 3, 3, H, W).chunk(2, dim=1)
    lv = lv.div(20.0).tanh().mul(20.0)
    mean, lv = mean.reshape(B, -1, H, W), lv.reshape(B, -1, H, W)
    z = mean if noise is None else mean + torch.exp(0.5 * lv) * noise.to(mean.dtype)
    return mean, lv, z


def conv_terms_abs(x, w, stride=1, pad=(1, 1, 1, 1), groups=1):
    """sum_k |w_k x_k| per output element (the scale of a dot product's rounding error)."""
    return F.conv2d(F.pad(x.abs(), pad), w.abs(), stride=stride, groups=groups)

