"""Fused generation pipelines over the mirrored modules (the calls the reference's engines make).

`sample_t23d` is `DiffusionEngineLSGM.sample` (nsr/lsgm/sgm_DiffusionEngine.py:385-407):
EulerEDMSampler(num_steps) + DiscreteDenoiser(EpsScaling, 1000 idx) + VanillaCFG(scale) around the
T23D DiT.  Everything that is step-invariant is hoisted out of the loop -- the sigma schedule, the
nearest-of-1000 quantisation (two (1000, 2B) abs-diff argmins per step in the reference,
denoiser.py:64-78), c_in / c_out, the update coefficients -- into small device tables, so one step is
    DiT forward (2B samples, c_in folded into the patch embed)  +  1 fused update launch:
    x' = x + (dt/s) * sq * [(1-g) net_u + g net_c]        (sq = quantised sigma, c_out = -sq)
which is algebraically the reference's  D = x - sq*net;  x' = x + (x - cfg(D))/s * dt.
"""
from __future__ import annotations

import os

import torch

from . import ops
from .dit._graph import graphs_enabled
from .sgm.modules.diffusionmodules.discretizer import LegacyDDPMDiscretization


@torch.no_grad()
def edm_cfg_tables(num_steps: int, scale: float, B: int, device, dtype=torch.float32):
    """Per-step device tables for the fused Euler-EDM + CFG loop (float32 arithmetic in the same
    order as the reference's scalar tensors)."""
    disc = LegacyDDPMDiscretization()
    sigmas = disc(num_steps, device="cpu")                       # (num_steps+1,), last = 0
    table = disc(1000, do_append_zero=False, flip=True)          # ascending, DiscreteDenoiser.sigmas
    s = sigmas[:-1]
    idx = (s[None, :] - table[:, None]).abs().argmin(dim=0)      # sigma_to_idx
    sq = table[idx]                                              # quantised sigma
    idx2 = (sq[None, :] - table[:, None]).abs().argmin(dim=0)    # possibly_quantize_c_noise
    c_in = 1 / (sq ** 2 + 1.0) ** 0.5
    r = (sigmas[1:] - s) / s                                     # dt / sigma
    w_u = r * sq * (1 - scale)
    w_c = r * sq * scale
    coef = torch.stack([torch.ones_like(r), w_u, w_c, torch.zeros_like(r)], 1)  # (steps, 4)
    return dict(
        init_scale=float(torch.sqrt(1.0 + sigmas[0] ** 2.0)),
        t_idx=idx2.to(device=device, dtype=torch.float32)[:, None].repeat(1, 2 * B).contiguous(),
        c_in=c_in.to(device)[:, None].repeat(1, 2 * B).contiguous(),
        coef=coef.to(device)[:, None, :].repeat(1, B, 1).contiguous(),
        sigmas=sigmas,
    )


@torch.no_grad()
def sample_t23d(model, randn: torch.Tensor, c: dict, uc: dict, num_steps: int = 250,
                scale: float = 6.5, tables: dict | None = None, use_graph: bool = True) -> torch.Tensor:
    """randn (B, 12, 32, 32) fp32 on the GPU (the reference draws it on the CPU generator and moves
    it, sgm_DiffusionEngine.py:395); c / uc = {'crossattn': (B, 77, ctx_dim)}.  Returns the
    denoised latents (B, 12, 32, 32) fp32."""
    if not randn.is_cuda:
        raise RuntimeError("sample_t23d runs on CUDA only (no CPU fallback)")
    B = randn.shape[0]
    if tables is None:
        tables = edm_cfg_tables(num_steps, scale, B, randn.device)
    ctx = torch.cat((uc["crossattn"], c["crossattn"]), 0).contiguous()   # VanillaCFG order: (uc, c)
    x = (randn.float() * tables["init_scale"]).contiguous()
    xa, xb = x, torch.empty_like(x)
    if use_graph and graphs_enabled() and hasattr(model, "capture_graph"):
        # one CUDA graph = one DiT forward of the 2B CFG batch; replayed every step.  The graph is cached on
        # the model per launch-sequence shape: this call computes the prompt batch's step-invariant
        # conditioning into the model's static buffers and captures only the first time a shape is seen.
        # every sample of a step shares its timestep: the adaLN modulations of all steps in one pass
        shared = hasattr(model, "modulation_table") and os.environ.get("LN3_SHARED_MODULATION", "1") != "0"
        g = model.capture_graph(2 * B, ctx, shared_mod=shared)
        mod_table = model.modulation_table(tables["t_idx"][:num_steps, 0]) if shared else None
        for i in range(num_steps):
            g.x[:B].copy_(xa)
            g.x[B:].copy_(xa)
            if shared:
                g.mod.copy_(mod_table[i:i + 1])
            else:
                g.t.copy_(tables["t_idx"][i])
            g.in_scale.copy_(tables["c_in"][i])
            g.replay()
            ops.sampler_affine_update(xa, tables["coef"][i], g.out[:B], g.out[B:], out=xb)
            xa, xb = xb, xa
        return xa.clone()
    x2 = torch.empty((2 * B,) + tuple(x.shape[1:]), device=x.device, dtype=torch.float32)
    for i in range(num_steps):
        x2[:B].copy_(xa)
        x2[B:].copy_(xa)
        net = model(x2, tables["t_idx"][i], ctx, in_scale=tables["c_in"][i])
        ops.sampler_affine_update(xa, tables["coef"][i], net[:B], net[B:], out=xb)
        xa, xb = xb, xa
    return xa


@torch.no_grad()
def decode_and_render(decoder, latents: torch.Tensor, cameras: torch.Tensor, resolution: int = 128,
                      scaling_divider: float = 0.96806, noise: tuple | None = None, mlp_tf32: bool = True,
                      max_views_per_launch: int | None = None):
    """`TrainLoopDiffusionWithRec.render_video_given_triplane` (nsr/train_util_diffusion.py:176-382)
    without the host round trips: latents (B,12,32,32) -> tri-planes (decoded ONCE; the reference
    decodes twice, :204-206 and :268-270) -> every camera of `cameras` (V,25) for every latent in
    fused renderer launches.  Per-view global reductions (group_size=1) reproduce the reference's
    one-view-per-call loop (:292-302).  Returns image_raw (B,V,3,H,W) in [-1,1], image_depth
    (B,V,1,H,W), image_mask (B,V,1,H,W).  `noise` = (coarse, fine) tensors of shape (B*V, H*W, 64) to
    override the device RNG (tests).  The sampling noise costs 512 B per ray, so the views are rendered in
    launches of whole objects with at most `max_views_per_launch` views (default: ~2 GiB of noise)."""
    if not latents.is_cuda:
        raise RuntimeError("decode_and_render runs on CUDA only (no CPU fallback)")
    B, V = latents.shape[0], cameras.shape[0]
    H = W = resolution
    M = resolution * resolution
    dev = latents.device
    planes_cl = decoder.decode_to_channels_last(latents, in_mul=scaling_divider)     # (B,3,128,128,32)
    cams1 = cameras.to(dev, torch.float32).contiguous()                               # (V, 25)
    ray_o1, ray_d1 = ops.generate_rays(cams1, resolution)                              # shared by every object
    if max_views_per_launch is None:
        max_views_per_launch = max(V, (2 << 30) // (2 * M * 64 * 4))
    obj_per_launch = max(1, min(B, max_views_per_launch // V))
    kw = decoder.rendering_kwargs
    osg = decoder.triplane_decoder.decoder.raw_parameters()
    rgb = torch.empty(B, V, 3, H, W, device=dev)
    depth = torch.empty(B, V, 1, H, W, device=dev)
    wts = torch.empty(B, V, 1, H, W, device=dev)
    for b0 in range(0, B, obj_per_launch):
        nb = min(obj_per_launch, B - b0)
        if noise is None:
            nz = (torch.rand(nb * V, M, 64, device=dev), torch.rand(nb * V, M, 64, device=dev))
        else:
            nz = (noise[0][b0 * V:(b0 + nb) * V].contiguous(), noise[1][b0 * V:(b0 + nb) * V].contiguous())
        out = ops.render_views(planes_cl[b0:b0 + nb], ray_o1.repeat(nb, 1, 1), ray_d1.repeat(nb, 1, 1), nz[0], nz[1],
                               osg, views_per_obj=V, group_size=1,
                               box_warp=kw.get("box_warp", 0.9), bbox_min=kw.get("sampler_bbox_min", -0.45),
                               bbox_max=kw.get("sampler_bbox_max", 0.45), white_back=kw.get("white_back", True),
                               mlp_tf32=mlp_tf32)
        rgb[b0:b0 + nb].copy_(out["rgb"].view(nb, V, 3, H, W))
        depth[b0:b0 + nb].copy_(out["depth"].view(nb, V, 1, H, W))
        wts[b0:b0 + nb].copy_(out["weights"].view(nb, V, 1, H, W))
    return dict(image_raw=rgb, image_depth=depth, weights_samples=wts, image_mask=wts * (1 + 2 * 0.001) - 0.001)


@torch.no_grad()
def generate_t23d(model, decoder, randn, c, uc, cameras, num_steps: int = 250, scale: float = 6.5,
                  resolution: int = 128):
    """Text-to-3D end to end on one GPU: sample -> decode -> render (the body of
    DiffusionEngineLSGM.eval_cldm, nsr/lsgm/sgm_DiffusionEngine.py:410-523, minus conditioner + video sink)."""
    latents = sample_t23d(model, randn, c, uc, num_steps, scale)
    return latents, decode_and_render(decoder, latents, cameras, resolution)


@torch.no_grad()
def condition_prompt(conditioner, cond_key: str, prompt, num_samples: int, device=None, dtype=torch.float32):
    """The conditioner call of DiffusionEngineLSGM.eval_cldm (nsr/lsgm/sgm_DiffusionEngine.py:443-477): ONE prompt
    (a caption string / token-id row for T23D, an image (1,3,H,W) for I23D) -> (c, uc) with the unconditional half
    forced to zero embeddings, every tensor repeated to `num_samples` rows (`repeat_interleave`, :473-477)."""
    ucg_keys = [cond_key]
    batch_c = {cond_key: prompt}
    c, uc = conditioner.get_unconditional_conditioning(
        batch_c, force_uc_zero_embeddings=ucg_keys if len(conditioner.embedders) > 0 else [])
    for k in c:
        if isinstance(c[k], torch.Tensor):
            assert c[k].shape[0] == 1, "eval_cldm conditions on one prompt at a time"
            c[k], uc[k] = (y[k].repeat_interleave(num_samples, 0).to(dtype) for y in (c, uc))
            if device is not None:
                c[k], uc[k] = c[k].to(device), uc[k].to(device)
    return c, uc


@torch.no_grad()
def text_to_3d(conditioner, model, decoder, prompt, cameras, num_samples: int = 1, num_steps: int = 250,
               scale: float = 6.5, resolution: int = 128, seed: int = 41):
    """eval_cldm for one caption end to end (:410-523): conditioner -> `th.manual_seed(41)` CPU noise draw (:457-466,
    395-398) -> Euler-EDM + CFG sampling -> decode -> render.  Returns (latents, render dict)."""
    dev = next(model.parameters()).device
    c, uc = condition_prompt(conditioner, "caption", prompt, num_samples, device=dev)
    g = torch.Generator().manual_seed(seed)
    C = model.in_channels if not model.roll_out else 3 * model.in_channels
    randn = torch.randn(num_samples, C, 32, 32, generator=g).to(dev)
    return generate_t23d(model, decoder, randn, c, uc, cameras, num_steps, scale, resolution)


@torch.no_grad()
def sample_flow(model, c: dict, uc: dict, num_samples: int, seed: int = 42, num_steps: int = 250,
                cfg_scale: float = 4.0, sampling_method: str = "dopri5", dtype=torch.float32) -> torch.Tensor:
    """`FlowMatchingEngine.sample` (nsr/lsgm/flow_matching_trainer.py:509-551) for the image-conditioned denoisers
    (I23D 'img', MV23D 'img-c'): global `torch.manual_seed(seed)` -- which also seeds the CUDA generators that the
    renderer's noise draws use afterwards -- then a CPU `randn(num_samples, 12, 32, 32)`, the CFG batch
    cat((cond, uc)) per conditioning key and cat([zs, zs]), `Sampler(create_transport(snr_type='lognorm'))
    .sample_ode(num_steps=..., sampling_method=...)` around `model.forward_with_cfg`, and `[-1].chunk(2)[0]`.

    Engine dtype: as on the existing I23D path, the ODE state and the context are carried in fp32 and the denoiser
    rounds its GEMM operands to bf16 itself.  The engine's `.to(self.dtype)` casts of the noise and the context
    (bf16 under `use_amp`) are applied as roundings to `dtype`; the default float32 leaves them exact.
    Returns the denoised latents (num_samples, 12, 32, 32) fp32."""
    from .transport import Sampler, create_transport
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("sample_flow runs on CUDA only (no CPU fallback)")
    torch.manual_seed(seed)
    C = 3 * model.in_channels if model.roll_out else model.in_channels
    zs = torch.randn(num_samples, C, model.input_size, model.input_size).to(dev).to(dtype).float()
    ctx = {}
    for k in c:
        if k in ("vector", "crossattn", "concat"):
            ctx[k] = torch.cat((c[k], uc[k]), 0).to(dev).to(dtype).float().contiguous()
        else:
            assert c[k] == uc[k]
            ctx[k] = c[k]
    fn = Sampler(create_transport(snr_type="lognorm")).sample_ode(sampling_method=sampling_method, num_steps=num_steps)
    samples = fn(torch.cat([zs, zs], 0), model.forward_with_cfg, context=ctx, cfg_scale=cfg_scale)[-1]
    return samples.chunk(2, dim=0)[0]


@torch.no_grad()
def _cond_to_3d(conditioner, model, decoder, cond_key, prompt, cameras, num_samples, seed, num_steps, cfg_scale,
                sampling_method, resolution, dtype):
    dev = next(model.parameters()).device
    c, uc = condition_prompt(conditioner, cond_key, prompt, num_samples, device=dev)
    latents = sample_flow(model, c, uc, num_samples, seed=seed, num_steps=num_steps, cfg_scale=cfg_scale,
                          sampling_method=sampling_method, dtype=dtype)
    return latents, decode_and_render(decoder, latents, cameras[:24].to(dev), resolution)


@torch.no_grad()
def mv_to_3d(conditioner, model, decoder, mv_images: torch.Tensor, mv_cameras: torch.Tensor, cameras: torch.Tensor,
             num_samples: int = 4, seed: int = 42, num_steps: int = 250, cfg_scale: float = 4.0,
             sampling_method: str = "dopri5", resolution: int = 192, dtype=torch.float32):
    """Multi-view-to-3D, `FlowMatchingEngine.eval_cldm` for cond_key 'img-c' (nsr/lsgm/flow_matching_trainer.py:
    553-678): the conditioner on {'img': mv_images (1, V, 3, H, W) in [-1, 1], 'c': mv_cameras (1, V, 25)} with the
    unconditional half forced to zero and every row repeated `num_samples` times, `sample_flow`, then decode and render
    of `cameras[:24]` at `resolution`.  The release (sample_obajverse_mv23d_dit.sh) runs 6 views, 4 samples, CFG 4.0,
    dopri5 with 250 output points and 192^2 renders.

    The engine casts the views and cameras to its dtype (bf16 under use_amp) before the conditioner sees them; they
    are cast to `dtype` here.  With `aug_c=True` the conditioner rotates cameras of that tensor in place -- the caller's
    own `mv_cameras` when it already has that dtype and device.  Returns (latents, render dict)."""
    dev = next(model.parameters()).device
    img_c = {"img": mv_images.to(dev).to(dtype), "c": mv_cameras.to(dev).to(dtype)}
    return _cond_to_3d(conditioner, model, decoder, "img-c", img_c, cameras, num_samples, seed, num_steps, cfg_scale,
                       sampling_method, resolution, dtype)


@torch.no_grad()
def image_to_3d(conditioner, model, decoder, image: torch.Tensor, cameras: torch.Tensor, num_samples: int = 4,
                seed: int = 42, num_steps: int = 250, cfg_scale: float = 4.0, sampling_method: str = "dopri5",
                resolution: int = 192, dtype=torch.float32):
    """Image-to-3D, `FlowMatchingEngine.eval_cldm` for cond_key 'img' (the I23D release): the conditioner on one image
    (1, 3, H, W) in [-1, 1], `sample_flow`, decode and render of `cameras[:24]`.  Returns (latents, render dict)."""
    dev = next(model.parameters()).device
    return _cond_to_3d(conditioner, model, decoder, "img", image.to(dev).to(dtype), cameras, num_samples, seed,
                       num_steps, cfg_scale, sampling_method, resolution, dtype)


# ---------------------------------------------------------------------------------------------- multi-GPU
def shard_range(n_total: int, world: int, rank: int) -> tuple[int, int, int]:
    """Contiguous block of ceil(P/G) prompts per rank (SURVEY.md section 8e): returns (lo, hi, per) with
    hi - lo <= per valid prompts on this rank (trailing ranks may hold fewer, or none)."""
    per = -(-n_total // world)
    lo = min(rank * per, n_total)
    return lo, min(lo + per, n_total), per


@torch.no_grad()
def generate_sharded(model, decoder, c_all: dict, uc_all: dict, cameras: torch.Tensor, *, seed: int = 41,
                     num_steps: int = 250, scale: float = 6.5, resolution: int = 256, batch: int = 32,
                     with_depth: bool = False, device=None, group=None, gather: bool = True,
                     sample_fn=None, render_fn=None, pack_fn=None) -> dict:
    """Text-to-3D for a list of P prompts sharded over the ranks of `group` (BASELINE configs[4], SURVEY 8e):

        one global CPU-generator noise draw `manual_seed(seed); randn(P, 12, 32, 32)` sliced per rank (the
        reference slices its own global draw the same way, nsr/lsgm/sgm_DiffusionEngine.py:395-398,456-470)
        -> sample_t23d -> decode_and_render at `resolution` for every camera -> uint8 HWC frames (frame sink)
        -> ONE NCCL all-gather of the frames per local batch, issued on a side stream so that it overlaps
        the next batch's sampling (nsr/train_util_diffusion.py:177-382 is the per-rank body it replaces).

    c_all / uc_all = {'crossattn': (P, 77, ctx_dim)} for ALL prompts on every rank (the reference's ranks all
    read the same caption list); each rank uses rows [lo, hi).  There is no collective inside the data path;
    ranks holding fewer than ceil(P/G) prompts contribute zero frames that are trimmed from the result.
    Returns {'latents': (n_local,12,32,32), 'frames': uint8 (n_local, V, H, Wout, 3), 'frames_all': uint8
    (P, V, H, Wout, 3) on every rank (None if not gathered), 'shard': (lo, hi), 'gather_bytes_per_rank': int}.
    `sample_fn / render_fn / pack_fn` replace the three CUDA stages (the world-size-2 gloo test drives the
    sharding, padding and gather logic of THIS function with CPU stand-ins)."""
    import torch.distributed as dist
    distributed = dist.is_available() and dist.is_initialized()
    world = dist.get_world_size(group) if distributed else 1
    rank = dist.get_rank(group) if distributed else 0
    P = c_all["crossattn"].shape[0]
    lo, hi, per = shard_range(P, world, rank)
    dev = torch.device(device) if device is not None else next(model.parameters()).device
    V = cameras.shape[0]
    g = torch.Generator().manual_seed(seed)
    randn_all = torch.randn(P, 12, 32, 32, generator=g)                      # identical on every rank
    if sample_fn is None:
        sample_fn = lambda x, c, uc: sample_t23d(model, x, c, uc, num_steps, scale)
    if render_fn is None:
        render_fn = lambda lat: decode_and_render(decoder, lat, cameras, resolution)
    if pack_fn is None:
        from .frames import FrameSink
        sink = FrameSink(dev)
        pack_fn = lambda r: sink.pack(r["image_raw"], r["image_depth"] if with_depth else None)
    Wout = resolution * (2 if with_depth else 1)
    frames = torch.zeros(per, V, resolution, Wout, 3, dtype=torch.uint8, device=dev)
    latents = torch.zeros(per, 12, 32, 32, device=dev)
    do_gather = gather and world > 1
    frames_all = torch.empty(world, per, V, resolution, Wout, 3, dtype=torch.uint8, device=dev) if do_gather else None
    cuda = dev.type == "cuda"
    side = torch.cuda.Stream(device=dev) if (do_gather and cuda) else None
    pending = []
    for b0 in range(0, per, batch):                                          # same trip count on every rank
        b1 = min(b0 + batch, per)
        n_valid = max(0, min(hi - lo, b1) - b0)
        if n_valid > 0:
            sl = slice(lo + b0, lo + b0 + n_valid)
            x = randn_all[sl].to(dev, non_blocking=True)
            c = {"crossattn": c_all["crossattn"][sl].to(dev, non_blocking=True)}
            uc = {"crossattn": uc_all["crossattn"][sl].to(dev, non_blocking=True)}
            lat = sample_fn(x, c, uc)
            latents[b0:b0 + n_valid].copy_(lat)
            frames[b0:b0 + n_valid].copy_(pack_fn(render_fn(lat)))
        if do_gather:
            if b0 == 0 and b1 == per:                                        # one batch: gather straight into place
                src, dst = frames, frames_all
            else:
                src = frames[b0:b1].contiguous()
                dst = torch.empty(world, b1 - b0, *frames.shape[1:], dtype=torch.uint8, device=dev)
            if side is not None:
                side.wait_stream(torch.cuda.current_stream(dev))
                with torch.cuda.stream(side):
                    dist.all_gather_into_tensor(dst.view(-1), src.view(-1), group=group)
                    if dst is not frames_all:
                        frames_all[:, b0:b1].copy_(dst)
                src.record_stream(side); dst.record_stream(side)
            else:
                dist.all_gather_into_tensor(dst.view(-1), src.view(-1), group=group)
                if dst is not frames_all:
                    frames_all[:, b0:b1].copy_(dst)
            pending.append((src, dst))
    if side is not None:
        torch.cuda.current_stream(dev).wait_stream(side)
    n_local = hi - lo
    out_all = frames_all.view(world * per, V, resolution, Wout, 3)[:P] if do_gather else (frames[:P] if gather else None)
    return dict(latents=latents[:n_local], frames=frames[:n_local], frames_all=out_all, shard=(lo, hi),
                gather_bytes_per_rank=int(frames.numel()) if do_gather else 0)
