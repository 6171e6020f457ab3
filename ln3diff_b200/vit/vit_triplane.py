"""Mirror of reference vit/vit_triplane.py for the Objaverse release decoder class
`RodinSR_256_fusionv6_ConvQuant_liteSR_dinoInit3DAttn_SD_B_3L_C_withrollout_withSD_D_ditDecoder`
(resolved from `--ae_classname` by dotted path, nsr/script_util.py:1418-1429).

Decode path (train_util_diffusion.py:188-206 -> nsr/script_util.py:243-259):
  vit_decode_backbone   (vit_triplane.py:996-1011, :2126-2132)  latent -> PatchEmbedTriplane -> DiT2
  vit_decode_postprocess (:1913-1977)                           tokens -> conv_sr -> (B, 96, 128, 128)
  triplane_decode       (:1013-1041)                            Triplane.forward(planes, c)
Device work: wgmma GEMM / attention kernels for the 24 DiT2 blocks (per-token adaLN as one GEMM
per block), NHWC fp32 conv kernels for the SD decoder.  The DiT2 token stream is consumed by conv_in
in place (tokens are NHWC) and conv_out writes the channels-last tri-plane the ray marcher reads."""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from .. import ops
from .._lib import NORM_LAYER
from ..ldm.modules.diffusionmodules.model import Decoder


class PatchEmbedTriplane(nn.Module):
    """vit_triplane.py:58-108 parameters: Conv2d(in_chans -> 3*embed_dim, k = s = patch, groups = 3)."""

    def __init__(self, img_size=32, patch_size=2, in_chans=4, embed_dim=768, norm_layer=None, flatten=True,
                 bias=True):
        super().__init__()
        assert patch_size == 2 and norm_layer is None and flatten
        self.img_size, self.patch_size = (img_size, img_size), (patch_size, patch_size)
        self.num_patches = (img_size // patch_size) ** 2
        self.proj = nn.Conv2d(in_chans, embed_dim * 3, kernel_size=patch_size, stride=patch_size, bias=bias, groups=3)


class DiagonalGaussianDistribution:
    """utils/torch_utils/distributions/distributions.py:29-113: the VAE posterior over the tri-plane latent.
    mean / logvar are (B, z, 3, L); logvar is soft-clamped to 20 tanh(lv / 20) when soft_clamp (the release setting).
    `sample()` draws its noise from the CPU generator, `torch.randn(mean.shape)`, and moves it to the device, exactly as
    the reference does, so the same `torch.manual_seed` gives the same latent on any device."""

    def __init__(self, parameters, deterministic=False, soft_clamp=False):
        self.parameters = parameters
        self.mean, logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = logvar.div(20.0).tanh().mul(20.0) if soft_clamp else torch.clamp(logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self._finish()

    @classmethod
    def from_kernel(cls, mean, logvar):
        """The posterior whose mean and (already clamped) logvar ln3_vae_posterior wrote."""
        self = cls.__new__(cls)
        self.parameters, self.mean, self.logvar, self.deterministic = None, mean, logvar, False
        self._finish()
        return self

    def _finish(self):
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if self.deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self):
        return self.mean + self.std * torch.randn(self.mean.shape).to(device=self.mean.device)

    def mode(self):
        return self.mean

    def log_p(self, samples):
        # the reference divides by var, not std (distributions.py:72-78); kept
        normalized_samples = (samples - self.mean) / self.var
        return -0.5 * normalized_samples * normalized_samples - 0.5 * math.log(2 * math.pi) - self.logvar

    def normal_entropy(self):
        return self.logvar + 0.5 * (math.log(2 * math.pi) + 1)

    def kl(self, other=None):
        if self.deterministic:
            return torch.Tensor([0.0])
        if other is None:
            return 0.5 * torch.sum(torch.pow(self.mean, 2) + self.var - 1.0 - self.logvar, dim=[1, 2, 3])
        return 0.5 * torch.sum(torch.pow(self.mean - other.mean, 2) / other.var + self.var / other.var - 1.0
                               - self.logvar + other.logvar, dim=[1, 2, 3])


class RodinSR_256_fusionv6_ConvQuant_liteSR_dinoInit3DAttn_SD_B_3L_C_withrollout_withSD_D_ditDecoder(nn.Module):
    def __init__(self, vit_decoder, triplane_decoder, cls_token=False, normalize_feat=True, sr_ratio=2,
                 use_fusion_blk=True, fusion_blk_depth=2, fusion_blk=None, channel_multiplier=4, ldm_z_channels=4,
                 ldm_embed_dim=4, vae_p=2, **kwargs):
        super().__init__()
        assert not cls_token, "cls_token decoders are outside the release configuration"
        self.vit_decoder, self.triplane_decoder, self.cls_token = vit_decoder, triplane_decoder, cls_token
        self.vae_p, self.ldm_z_channels, self.ldm_embed_dim = vae_p, ldm_z_channels, ldm_embed_dim
        self.token_size = 16
        self.rendering_kwargs = getattr(triplane_decoder, "rendering_kwargs", {})
        D = vit_decoder.embed_dim
        # ViTTriplaneDecomposed replaces the DiT pos_embed by a 3-plane one (vit_triplane.py:210)
        vit_decoder.pos_embed = nn.Parameter(torch.zeros(1, 3 * self.token_size ** 2, D))
        self.register_buffer("w_avg", torch.zeros([512]))
        self.superresolution = nn.ModuleDict(dict(
            ldm_upsample=PatchEmbedTriplane(vae_p * self.token_size, vae_p, 3 * ldm_embed_dim, D, bias=True),
            quant_conv=nn.Conv2d(2 * 3 * ldm_z_channels, 2 * ldm_embed_dim * 3, kernel_size=1, groups=3),
            conv_sr=Decoder(resolution=128, in_channels=3, ch=32, ch_mult=[1, 2, 2, 4], num_res_blocks=1, dropout=0.0,
                            attn_resolutions=[], out_ch=32, z_channels=D)))
        self.decoder_pred = None
        self.D_roll_out_input = False
        self.plane_n = 3
        self.reparameterization_soft_clamp = True
        self._prep = None

    # ------------------------------------------------------------------ weight repack
    def _apply(self, fn, *a, **kw):
        self._prep = None
        return super()._apply(fn, *a, **kw)

    def load_state_dict(self, *a, **kw):
        self._prep = None
        return super().load_state_dict(*a, **kw)

    @torch.no_grad()
    def prepare(self):
        dev = self.w_avg.device
        if dev.type != "cuda":
            raise RuntimeError("ln3diff_b200 decoder runs on CUDA only (no CPU fallback)")
        bf = lambda w: w.detach().to(dev, torch.bfloat16).contiguous()
        f32 = lambda w: w.detach().to(dev, torch.float32).contiguous()
        pk = lambda conv: (f32(conv.weight.permute(2, 3, 1, 0).reshape(-1, conv.weight.shape[1], conv.weight.shape[0])),
                           f32(conv.bias))
        P = {"up_w": f32(self.superresolution["ldm_upsample"].proj.weight),
             "up_b": f32(self.superresolution["ldm_upsample"].proj.bias),
             "pos": f32(self.vit_decoder.pos_embed)}
        P["blocks"] = [dict(ada_w=bf(b.adaLN_modulation[1].weight), ada_b=f32(b.adaLN_modulation[1].bias),
                            qkv_w=bf(b.attn.qkv.weight), qkv_b=f32(b.attn.qkv.bias),
                            proj_w=bf(b.attn.proj.weight), proj_b=f32(b.attn.proj.bias),
                            fc1_w=bf(b.mlp.mlp[0].weight), fc1_b=f32(b.mlp.mlp[1].bias),
                            fc2_w=bf(b.mlp.mlp[2].weight), fc2_b=f32(b.mlp.mlp[3].bias))
                       for b in self.vit_decoder.blocks]
        sr = self.superresolution["conv_sr"]

        def res(rb):
            d = dict(n1=(f32(rb.norm1.weight), f32(rb.norm1.bias)), c1=pk(rb.conv1),
                     n2=(f32(rb.norm2.weight), f32(rb.norm2.bias)), c2=pk(rb.conv2))
            if hasattr(rb, "nin_shortcut"):
                d["nin"] = pk(rb.nin_shortcut)
            return d

        at = sr.mid.attn_1
        qc = self.superresolution["quant_conv"]
        P["quant"] = (f32(qc.weight.reshape(qc.weight.shape[0], -1)), f32(qc.bias))
        P["sr"] = dict(conv_in=pk(sr.conv_in), mid1=res(sr.mid.block_1), mid2=res(sr.mid.block_2),
                       attn=dict(n=(f32(at.norm.weight), f32(at.norm.bias)), q=pk(at.q), k=pk(at.k), v=pk(at.v),
                                 o=pk(at.proj_out)),
                       up=[dict(blocks=[res(b) for b in u.block],
                                upsample=pk(u.upsample.conv) if hasattr(u, "upsample") else None) for u in sr.up],
                       nout=(f32(sr.norm_out.weight), f32(sr.norm_out.bias)), conv_out=pk(sr.conv_out))
        self._prep = P
        return P

    # ------------------------------------------------------------------ fused decode
    # 3x3 convolutions of the SD upsampler on the tensor cores (TF32 operands, fp32 accumulate); set to False
    # for exact fp32 arithmetic
    conv_tf32 = True

    def _res(self, x, W):
        tf = self.conv_tf32
        h = ops.conv_nhwc(x, *W["c1"], ksize=3, gn=ops.groupnorm_stats(x, *W["n1"]), swish=True, tf32=tf)
        sc = ops.conv_nhwc(x, *W["nin"], ksize=1) if "nin" in W else x
        return ops.conv_nhwc(h, *W["c2"], ksize=3, gn=ops.groupnorm_stats(h, *W["n2"]), swish=True, residual=sc, tf32=tf)

    @torch.no_grad()
    def decode_to_channels_last(self, latent, in_mul: float = 1.0):
        """latent (B, 12, 32, 32) -> channels-last tri-plane (B, 3, 128, 128, 32) fp32 (what the ray
        marcher consumes).  `in_mul` folds `planes *= triplane_scaling_divider`."""
        if isinstance(latent, dict):
            latent = latent["latent_normalized_2Ddiffusion"]
        if not latent.is_cuda:
            raise RuntimeError("ln3diff_b200 decoder runs on CUDA only (no CPU fallback)")
        if self._prep is None:
            self.prepare()
        P = self._prep
        vd = self.vit_decoder
        B, D, H = latent.shape[0], vd.embed_dim, vd.num_heads
        T = 3 * self.token_size ** 2
        M = B * T
        _, sc_bf = ops.patch_embed_triplane(latent.float().contiguous(), P["up_w"], P["up_b"], in_mul)
        sc2 = sc_bf.view(M, D)                                   # SiLU(c), the adaLN operand of every block
        x = P["pos"].expand(B, T, D).clone()   # the residual stream is updated in place: never alias the weights
        x2 = x.view(M, D)
        dev = latent.device
        # two modulation buffers, alternating per block: the deferred MLP residual of block i-1 is applied by block i's
        # first pass with block i-1's per-token gate, which then still sits in the other buffer (no copy)
        mods = (torch.empty(M, 6 * D, device=dev, dtype=torch.float32), torch.empty(M, 6 * D, device=dev, dtype=torch.float32))
        a = torch.empty(M, D, device=dev, dtype=torch.bfloat16)
        qkv = torch.empty(M, 3 * D, device=dev, dtype=torch.bfloat16)
        att = torch.empty(M, D, device=dev, dtype=torch.bfloat16)
        hbuf = torch.empty(M, int(vd.mlp_ratio) * D, device=dev, dtype=torch.bfloat16)
        val = torch.empty(M, D, device=dev, dtype=torch.bfloat16)
        mod = mods[0]
        for i, W in enumerate(P["blocks"]):
            gate_prev = mod[:, 5 * D:6 * D]      # gate_mlp of the previous block (its buffer is not rewritten until block i+1)
            mod = mods[i & 1]
            ops.gemm(sc2, W["ada_w"], W["ada_b"], out_kind=ops.OUT_F32, out=mod)   # per-token adaLN (B*768, 6D)
            sl = lambda j: mod[:, j * D:(j + 1) * D]
            ops.norm_modulate(x2, norm=NORM_LAYER, shift=sl(0), scale=sl(1), mod_rows=1, out=a,
                              resid=val if i > 0 else None, resid_gate=gate_prev if i > 0 else None, resid_gate_rows=1)
            ops.gemm(a, W["qkv_w"], W["qkv_b"], out=qkv)
            if i % 2 == 0:   # attention within each plane: 'b (n l) c -> (b n) l c'
                q3 = qkv.view(B * 3, T // 3, 3 * D)
                ops.fmha(q3[:, :, :D], q3[:, :, D:2 * D], q3[:, :, 2 * D:], H, out=att.view(B * 3, T // 3, D))
            else:            # global attention over the 3 planes
                q3 = qkv.view(B, T, 3 * D)
                ops.fmha(q3[:, :, :D], q3[:, :, D:2 * D], q3[:, :, 2 * D:], H, out=att.view(B, T, D))
            ops.gemm(att, W["proj_w"], W["proj_b"], out=val)
            ops.norm_modulate(x2, norm=NORM_LAYER, shift=sl(3), scale=sl(4), mod_rows=1, out=a,
                              resid=val, resid_gate=sl(2), resid_gate_rows=1)
            ops.gemm(a, W["fc1_w"], W["fc1_b"], act=ops.ACT_GELU_ERF, out=hbuf)
            ops.gemm(hbuf, W["fc2_w"], W["fc2_b"], out=val)
        ops.norm_modulate(x2, norm=NORM_LAYER, resid=val, resid_gate=mod[:, 5 * D:6 * D], resid_gate_rows=1, want_out=False)
        # tokens (B, 3*16*16, D) are already NHWC (3B, 16, 16, D)
        ts = self.token_size
        out = self._conv_sr(x.view(B * 3, ts, ts, D))
        return out.view(B, 3, out.shape[1], out.shape[2], out.shape[3])

    @torch.no_grad()
    def _conv_sr(self, h):
        """superresolution['conv_sr'] (the ldm Decoder) on NHWC fp32 tokens (3B, 16, 16, D) -> the channels-last
        planes (3B, 128, 128, 32)."""
        if self._prep is None:
            self.prepare()
        S = self._prep["sr"]
        tf = self.conv_tf32
        h = ops.conv_nhwc(h, *S["conv_in"], ksize=3, tf32=tf)
        h = self._res(h, S["mid1"])
        A = S["attn"]
        gn = ops.groupnorm_stats(h, *A["n"])
        q, k, v = (ops.conv_nhwc(h, *A[n_], ksize=1, gn=gn) for n_ in ("q", "k", "v"))
        h = ops.conv_nhwc(ops.attn_single_head(q, k, v), *A["o"], ksize=1, residual=h)
        h = self._res(h, S["mid2"])
        for lvl in reversed(range(len(S["up"]))):
            for W in S["up"][lvl]["blocks"]:
                h = self._res(h, W)
            if S["up"][lvl]["upsample"] is not None:
                h = ops.conv_nhwc(h, *S["up"][lvl]["upsample"], ksize=3, upsample=True, tf32=tf)
        return ops.conv_nhwc(h, *S["conv_out"], ksize=3, gn=ops.groupnorm_stats(h, *S["nout"]), swish=True, tf32=tf)

    # ------------------------------------------------------------------ VAE posterior (encoder side)
    @torch.no_grad()
    def _posterior(self, moments, sample_posterior: bool):
        """moments (B, 24, S, S) -> (posterior, latent (B, 4, 3, S*S)) on ln3_vae_posterior.  A channels-last view (what
        the encoder mirror returns) reaches the kernel without a copy."""
        if not moments.is_cuda:
            raise RuntimeError("ln3diff_b200 decoder runs on CUDA only (no CPU fallback)")
        assert self.reparameterization_soft_clamp and self.plane_n == 3 and self.vae_p > 1
        if self._prep is None:
            self.prepare()
        B, C2, H, W = moments.shape
        assert C2 == 6 * self.ldm_z_channels == 24 and H == W, "moments must be (B, 24, S, S)"
        nhwc = moments.float().permute(0, 2, 3, 1).contiguous()
        # sample(): the CPU generator's randn(mean.shape), as the reference draws it
        noise = torch.randn(B, 12, H, W).to(moments.device) if sample_posterior else None
        mean, logvar, z = ops.vae_posterior(nhwc, *self._prep["quant"], noise)
        shp = (B, self.ldm_z_channels, self.plane_n, H * W)          # the reference's (B, C, 3, L)
        return DiagonalGaussianDistribution.from_kernel(mean.view(shp), logvar.view(shp)), z.view(shp)

    def vae_encode(self, h):
        """vit_triplane.py:912-933: quant_conv + DiagonalGaussianDistribution(soft_clamp=True) of the encoder moments."""
        return self._posterior(h, False)[0]

    def vae_reparameterization(self, latent, sample_posterior):
        """vit_triplane.py:1152-1199: encoder moments (B, 24, 32, 32) -> the reference's dict (posterior sample or mode,
        log_q with its division by var, the (B, 12, 32, 32) diffusion latent)."""
        posterior, latent = self._posterior(latent, sample_posterior)
        log_q = posterior.log_p(latent)
        S = self.token_size * self.vae_p
        B = latent.shape[0]
        return dict(normal_entropy=posterior.normal_entropy(),
                    latent_normalized=latent.permute(0, 2, 3, 1).reshape(B, -1, latent.shape[1]),
                    latent_normalized_2Ddiffusion=latent.reshape(B, -1, S, S),
                    log_q_2Ddiffusion=log_q.reshape(B, -1, S, S),
                    log_q=log_q,
                    posterior=posterior)

    def vit_decode(self, latent, img_size, sample_posterior=True, **kwargs):
        """vit_triplane.py:879-885: reparameterise the encoder moments, then decode to the tri-plane."""
        ret_dict = self.vae_reparameterization(latent, sample_posterior)
        return self.vit_decode_postprocess(self.vit_decode_backbone(ret_dict, img_size), ret_dict)

    # ------------------------------------------------------------------ reference-named entry points
    def vit_decode_backbone(self, latent, img_size=None):
        """Returns a handle consumed by vit_decode_postprocess (the fused decode runs there)."""
        return latent["latent_normalized_2Ddiffusion"] if isinstance(latent, dict) else latent

    def vit_decode_postprocess(self, latent_from_vit, ret_dict: dict):
        cl = self.decode_to_channels_last(latent_from_vit)
        B = cl.shape[0]
        planes = cl.permute(0, 1, 4, 2, 3).reshape(B, 3 * cl.shape[4], cl.shape[2], cl.shape[3]).contiguous()
        ret_dict.update(dict(cls_token=None, latent_after_vit=planes))   # 'b (n c) h w'
        return ret_dict

    def triplane_decode(self, vit_decode_out, c, return_raw_only=False, **kwargs):
        latent_after_vit = vit_decode_out.get("latent_after_vit") if isinstance(vit_decode_out, dict) else vit_decode_out
        if not isinstance(vit_decode_out, dict):
            vit_decode_out = dict(latent_normalized=latent_after_vit)
        ret = self.triplane_decoder(latent_after_vit, c, return_raw_only=return_raw_only, **kwargs)
        ret.update({"latent_after_vit": latent_after_vit, **vit_decode_out})
        return ret

    # ------------------------------------------------------------------ mesh-extraction queries
    @torch.no_grad()
    def forward_points(self, planes, points: torch.Tensor, chunk_size: int = 2 ** 16):
        """reference vit_triplane.py:2009-2050.  One launch for all points: `chunk_size` (the reference's
        guard against its own (N,P,3,32) feature temporaries + empty_cache() per chunk) is accepted and
        ignored.  Returns {'rgb': (N,P,3), 'sigma': (N,P,1)}."""
        return self.triplane_decoder.renderer._run_model(
            planes=planes, decoder=self.triplane_decoder.decoder, sample_coordinates=points,
            sample_directions=None, options=self.rendering_kwargs)

    @torch.no_grad()
    def triplane_decode_grid(self, vit_decode_out, grid_size, aabb: torch.Tensor = None, **kwargs):
        """reference vit_triplane.py:2052-2120: density / colour on a grid_size^3 lattice over the sampler
        bbox (or `aabb` (N,2,3)).  The lattice is generated inside the kernel with torch.linspace's
        arithmetic; no coordinate tensor exists.  Returns {'rgb': (N,G,G,G,3), 'sigma': (N,G,G,G,1)}."""
        assert isinstance(vit_decode_out, dict)
        planes = vit_decode_out["latent_after_vit"]
        kw = self.rendering_kwargs
        ren = self.triplane_decoder.renderer
        planes_cl = ren._as_channels_last(planes)
        N = planes_cl.shape[0]
        if aabb is None:
            if "sampler_bbox_min" in kw:
                lo, hi = [kw["sampler_bbox_min"]] * 3, [kw["sampler_bbox_max"]] * 3
            else:
                lo, hi = [-kw["box_warp"] / 2] * 3, [kw["box_warp"] / 2] * 3
            boxes = [(lo, hi)] * N
            uniform = True
        else:
            assert planes_cl.shape[0] == aabb.shape[0], "Batch size mismatch for planes and aabb"
            ab = aabb.detach().float().cpu()
            boxes = [(ab[i, 0].tolist(), ab[i, 1].tolist()) for i in range(N)]
            uniform = all(b == boxes[0] for b in boxes)
        osg = self.triplane_decoder.decoder.raw_parameters()
        if uniform:
            sigma, rgb = ops.query_points(planes_cl, osg, grid_size=grid_size, aabb_min=boxes[0][0],
                                          aabb_max=boxes[0][1], box_warp=kw["box_warp"],
                                          mlp_tf32=kw.get("osg_mlp_tf32", True))
        else:
            parts = [ops.query_points(planes_cl[i:i + 1], osg, grid_size=grid_size, aabb_min=boxes[i][0],
                                      aabb_max=boxes[i][1], box_warp=kw["box_warp"],
                                      mlp_tf32=kw.get("osg_mlp_tf32", True)) for i in range(N)]
            sigma, rgb = torch.cat([p_[0] for p_ in parts]), torch.cat([p_[1] for p_ in parts])
        G = grid_size
        return {"rgb": rgb.reshape(N, G, G, G, -1), "sigma": sigma.reshape(N, G, G, G, -1)}



# `vae_reconstruction.sh` names the `_S` variant (vit_triplane.py:1517-1837).  Its decode and reparameterisation compute
# what the class above computes and its state_dict has the same keys and shapes (DiT2-B/2 and DiT2-L/2).
RodinSR_256_fusionv6_ConvQuant_liteSR_dinoInit3DAttn_SD_B_3L_C_withrollout_withSD_D_ditDecoder_S = \
    RodinSR_256_fusionv6_ConvQuant_liteSR_dinoInit3DAttn_SD_B_3L_C_withrollout_withSD_D_ditDecoder
