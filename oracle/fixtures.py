"""TEST INFRASTRUCTURE ONLY -- seeded inputs shared by oracle/make_golden.py (which runs the real
reference on them) and the tests (which run the oracle / the CUDA path on the same inputs)."""
from __future__ import annotations

import torch

RENDER_CAM_ROWS = (3, 17)  # rows of assets/objv_eval_pose.pt used by the render fixture


def dit_inputs():
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 12, 32, 32, generator=g)
    t = torch.tensor([10, 500])
    ctx = torch.randn(2, 77, 768, generator=g)
    return x, t, ctx


def toy_network():
    """Closed-form stand-in for the denoiser: pins the sampler engines without DiT cost."""
    g = torch.Generator().manual_seed(0)
    Wt = torch.randn(12, 12, generator=g) * 0.2

    def net(x, t, cond):
        c = cond["crossattn"] if isinstance(cond, dict) else cond
        return torch.tanh(torch.einsum("oc,bchw->bohw", Wt.to(x.device), x)
                          + 0.001 * t.float()[:, None, None, None]
                          + c.mean(dim=(1, 2))[:, None, None, None])
    return net


def sampler_inputs():
    g = torch.Generator().manual_seed(21)
    x0 = torch.randn(2, 12, 32, 32, generator=g)
    c = {"crossattn": torch.randn(2, 77, 16, generator=g)}
    uc = {"crossattn": torch.zeros(2, 77, 16)}
    noise = torch.randn(2, 12, 32, 32, generator=g)
    step_noise = [torch.randn(2, 12, 32, 32, generator=g) for _ in range(10)]
    z = torch.randn(2, 12, 32, 32, generator=g)
    return x0, c, uc, noise, step_noise, z


def render_inputs(res: int, n_views: int = len(RENDER_CAM_ROWS), plane_res: int = 16):
    """Small tri-plane (3,32,plane_res,plane_res) with scale 5 and an OSG sigma bias of +2 so that
    alpha spans (0,1) and in-box masks are mixed (random planes alone give sigma ~ 0: SURVEY 7.2)."""
    g = torch.Generator().manual_seed(31)
    planes = 5 * torch.randn(3, 32, plane_res, plane_res, generator=g)
    w1 = torch.randn(64, 32, generator=g)
    b1 = torch.randn(64, generator=g) * 0.1
    w2 = torch.randn(4, 64, generator=g)
    b2 = torch.randn(4, generator=g) * 0.1
    b2[0] += 2.0
    M = res * res
    nc = torch.rand(n_views, M, 64, generator=g)
    nf = torch.rand(n_views, M, 64, generator=g)
    return planes, (w1, b1, w2, b2), nc, nf


def render_group_inputs(res: int = 6):
    """Three objects, one view each, rendered as ONE reference call (batch 3), with edge rays:
      view 0  rays from z = 2 that hit the box, except rays 0-4: origins on a box face with the matching direction
              component +0.0 or -0.0 (t = 0 * inf = NaN: the reference marks them invalid), and ray 2 with zero
              x / y components strictly inside those slabs (valid)
      view 1  origins inside the box, two of them axis-aligned
      view 2  every ray misses: only the call's shared start range and depth clamp give it depths.
    Returns planes (3,3,32,16,16) (object n for view n), osg, ray_o / ray_d (3,res*res,3), noise (3,res*res,64) x2."""
    planes0, osg, _, _ = render_inputs(res, n_views=1)
    g = torch.Generator().manual_seed(51)
    planes = torch.stack([planes0, 5 * torch.randn(planes0.shape, generator=g),
                          5 * torch.randn(planes0.shape, generator=g)])
    M = res * res
    n = torch.nn.functional.normalize
    o0 = torch.randn(M, 3, generator=g) * 0.1 + torch.tensor([0.0, 0.0, 2.0])
    d0 = n(-o0 + 0.05 * torch.randn(M, 3, generator=g), dim=1)
    edge = [((-0.45, 0.0, 2.0), (0.0, 0.0, -1.0)),     # on the x = lo face, d_x = +0
            ((0.45, 0.1, 2.0), (-0.0, 0.0, -1.0)),     # on the x = hi face, d_x = -0
            ((0.1, 0.0, 2.0), (0.0, 0.0, -1.0)),       # d_x = d_y = 0 inside the slabs: valid
            ((0.2, 0.45, -2.0), (0.0, 0.0, 1.0)),      # on the y = hi face, d_y = +0
            ((-0.45, -0.45, 2.0), (0.0, -0.0, -1.0))]  # on an edge: two NaN slabs
    for i, (oo, dd) in enumerate(edge):
        o0[i], d0[i] = torch.tensor(oo), torch.tensor(dd)
    o1 = (torch.rand(M, 3, generator=g) - 0.5) * 0.6
    d1 = n(torch.randn(M, 3, generator=g), dim=1)
    d1[0], d1[1] = torch.tensor([1.0, 0.0, 0.0]), torch.tensor([0.0, -1.0, 0.0])
    o2 = torch.tensor([3.0, 3.0, 3.0]) + 0.1 * torch.randn(M, 3, generator=g)
    d2 = n(torch.tensor([1.0, 0.2, 0.1]) + 0.05 * torch.randn(M, 3, generator=g), dim=1)
    nc = torch.rand(3, M, 64, generator=g)
    nf = torch.rand(3, M, 64, generator=g)
    return planes, osg, torch.stack([o0, o1, o2]), torch.stack([d0, d1, d2]), nc, nf


DECODER_ARCH, DECODER_DIM = "DiT2-S/2", 384
SCALING_DIVIDER = 0.96806  # --triplane_scaling_divider of the release scripts


def decoder_state_dict(shapes: dict) -> dict:
    """Key-seeded synthetic AE-decoder weights; GroupNorm / norm scales are centred at 1."""
    from .dit import synth_state_dict
    sd = synth_state_dict(shapes, seed=9)
    for k in sd:
        if "norm" in k and k.endswith("weight") and sd[k].dim() == 1:
            sd[k] = 1 + sd[k]
    return sd


def decoder_latent():
    return torch.randn(1, 12, 32, 32, generator=torch.Generator().manual_seed(3))


I23D_ARCH = "DiT-PixArt-B/2"


def i23d_inputs():
    g = torch.Generator().manual_seed(13)
    x = torch.randn(2, 12, 32, 32, generator=g)
    t = torch.tensor([0.1, 0.7])
    ctx = {"vector": torch.randn(2, 768, generator=g), "crossattn": torch.randn(2, 256, 2048, generator=g)}
    return x, t, ctx


def i23d_state_dict(shapes: dict, pos_embed: torch.Tensor) -> dict:
    from .dit import synth_state_dict
    sd = synth_state_dict(shapes, seed=5, keep={"pos_embed": pos_embed})
    for k in sd:
        if (k.endswith("norm.weight") or "norm1.weight" in k or "norm2.weight" in k
                or k == "cap_embedder.0.weight" or k.endswith("attention_y_norm.weight")):
            sd[k] = 1 + sd[k]
    return sd


T23D_PIXART_ARCH = "DiT-PixelArt-B/2"


def t23d_pixart_inputs():
    g = torch.Generator().manual_seed(17)
    x = torch.randn(2, 12, 32, 32, generator=g)
    t = torch.tensor([12.0, 871.0])
    ctx = {"vector": torch.randn(2, 768, generator=g), "crossattn": torch.randn(2, 77, 768, generator=g)}
    return x, t, ctx

