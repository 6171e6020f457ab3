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

import torch

from . import ops
from .sgm.modules.diffusionmodules.discretizer import LegacyDDPMDiscretization


def _quantise(sigma: torch.Tensor, table: torch.Tensor):
    """DiscreteDenoiser(EpsScaling, 1000 idx) on float32 sigmas of any shape; `table` holds its ascending sigmas.
    Returns (timestep index, quantised sigma, c_in), each of sigma's shape."""
    sq = table[(sigma[..., None] - table).abs().argmin(-1)]      # sigma_to_idx, possibly_quantize_sigma
    idx = (sq[..., None] - table).abs().argmin(-1)               # possibly_quantize_c_noise
    return idx, sq, 1 / (sq ** 2 + 1.0) ** 0.5                   # EpsScaling's c_in


def _cfg_context(c: dict, uc: dict) -> dict:
    """VanillaCFG.prepare_inputs' context: cat((uc, c)) per tensor key, the other keys passed through."""
    return {k: torch.cat((uc[k], c[k]), 0) if k in ("vector", "crossattn", "concat") else c[k] for k in c}


@torch.no_grad()
def edm_cfg_tables(num_steps: int, scale: float, B: int, device, dtype=torch.float32):
    """Per-step device tables for the fused Euler-EDM + CFG loop (float32 arithmetic in the same
    order as the reference's scalar tensors)."""
    disc = LegacyDDPMDiscretization()
    sigmas = disc(num_steps, device="cpu")                       # (num_steps+1,), last = 0
    s = sigmas[:-1]
    idx2, sq, c_in = _quantise(s, disc(1000, do_append_zero=False, flip=True))
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


# ---------------------------------------------------------------------------------------------- sgm sampler family
# The reference's class names (sgm/inference/api.py:30-34) of the samplers sample_t23d runs.
SAMPLERS = ("EulerEDMSampler", "HeunEDMSampler", "EulerAncestralSampler", "DPMPP2SAncestralSampler",
            "DPMPP2MSampler", "LinearMultistepSampler")
_PLANS: dict = {}


def _plan_eval(plan, step, sigma, coef, *, kind, hist=(), hist_write=None, noise=False, draw=False, x_out=True):
    """Append one denoiser evaluation at `sigma` (a float32 scalar tensor).  kind 'D': e is the guided denoised D;
    kind 'd': e is the derivative (x_eval - D) / sigma.  coef holds the update part (a, b, c, h0, h1, h2, s)."""
    idx2, sq, c_in = _quantise(sigma, plan["_table"])
    g, sqd = plan["scale"], float(sq)
    if kind == "D":                                               # D = x_eval - sq net, CFG-combined
        k = (1.0, -sqd * (1 - g), -sqd * g)
    else:                                                         # d = (x_eval - D) / sigma = sq net / sigma
        k = (0.0, sqd * (1 - g) / float(sigma), sqd * g / float(sigma))
    row = list(k) + [float(coef.get(n, 0.0)) for n in ("a", "b", "c", "h0", "h1", "h2", "s")] + [0.0, 0.0]
    plan["evals"].append(dict(step=step, sigma=float(sigma), t_idx=int(idx2), c_in=float(c_in), coef=row,
                              hist=tuple(hist), hist_write=hist_write, noise=noise, draw=draw, x_out=x_out,
                              eval_out=True))


def edm_sampler_plan(sampler: str, num_steps: int, scale: float, eta: float = 1.0, s_noise: float = 1.0,
                     order: int = 4) -> dict:
    """The evaluation plan of one sgm sampler run with DiscreteDenoiser(EpsScaling, 1000) + VanillaCFG(scale) on
    the LegacyDDPM schedule (host-side, float32 scalar ops in the reference's order; cached).  One entry per
    denoiser evaluation: its sigma, timestep index and c_in, the ln3_sampler_step coefficient row
    (k0, k1, k2, a, b, c, h0, h1, h2, s, 0, 0) for the raw network halves, the history slots it reads (hist[j])
    and writes, whether it reads the step's noise / draws it, and which of x and the next forward's input it
    writes.  Reference: sgm/modules/diffusionmodules/sampling.py:133-362, sampling_utils.py:7-43."""
    from .sgm.modules.diffusionmodules.sampling_utils import get_ancestral_step, linear_multistep_coeff
    if sampler not in SAMPLERS[1:]:
        raise ValueError(f"unknown sampler {sampler!r}; expected one of {SAMPLERS}")
    if sampler == "LinearMultistepSampler" and not 1 <= order <= 4:
        raise ValueError("LinearMultistepSampler: the fused step keeps at most 3 past derivatives (order <= 4)")
    key = (sampler, int(num_steps), float(scale), float(eta), float(s_noise), int(order))
    plan = _PLANS.get(key)
    if plan is not None:
        return plan
    disc = LegacyDDPMDiscretization()
    sig = disc(num_steps, device="cpu")                           # (num_steps+1,) float32, last = 0
    plan = dict(sampler=sampler, num_steps=num_steps, scale=scale, evals=[], sigmas=sig, n_slots=0,
                init_scale=float(torch.sqrt(1.0 + sig[0] ** 2.0)),
                _table=disc(1000, do_append_zero=False, flip=True))
    ancestral = sampler in ("EulerAncestralSampler", "DPMPP2SAncestralSampler")
    nlog = lambda s: s.log().neg()                                # to_neg_log_sigma
    tsig = lambda t: t.neg().exp()                                # to_sigma
    sig_np = sig.numpy()
    for i in range(num_steps):
        s, sn = sig[i], sig[i + 1]
        if ancestral:
            sd, su = get_ancestral_step(s, sn, eta=eta)
            su = torch.as_tensor(su, dtype=torch.float32)
            # ancestral_step: x + noise * s_noise * sigma_up where next_sigma > 0 (one draw per step regardless)
            ns = dict(s=float(s_noise * su) if float(sn) > 0.0 else 0.0)
            nread = float(sn) > 0.0
        if sampler == "EulerAncestralSampler":
            r = (sd - s) / s                                      # x + (sd - s) (x - D) / s
            _plan_eval(plan, i, s, dict(a=1 + r, c=-r, **ns), kind="D", noise=nread, draw=True)
        elif sampler == "DPMPP2SAncestralSampler":
            if float(sd) < 1e-14:
                r = (sd - s) / s
                _plan_eval(plan, i, s, dict(a=1 + r, c=-r, **ns), kind="D", noise=nread, draw=True)
            else:
                t, tn = nlog(s), nlog(sd)
                h = tn - t
                sm = t + 0.5 * h
                m1, m2 = tsig(sm) / tsig(t), (-0.5 * h).expm1()
                m3, m4 = tsig(tn) / tsig(t), (-h).expm1()
                _plan_eval(plan, i, s, dict(a=m1, c=-m2), kind="D", x_out=False)           # x2 -> next input
                _plan_eval(plan, i, tsig(sm), dict(a=m3, c=-m4, **ns), kind="D", noise=nread, draw=True)
        elif sampler == "HeunEDMSampler":
            dt = sn - s
            if float(sn) < 1e-14:
                _plan_eval(plan, i, s, dict(a=1.0, c=dt), kind="d")
            else:
                plan["n_slots"] = 1
                _plan_eval(plan, i, s, dict(a=1.0, c=dt), kind="d", hist_write=0, x_out=False)   # x_euler, d
                _plan_eval(plan, i, sn, dict(a=1.0, c=dt / 2.0, h0=dt / 2.0), kind="d", hist=(0,))
        elif sampler == "DPMPP2MSampler":
            t, tn = nlog(s), nlog(sn)
            h = tn - t
            m1, m2 = tsig(tn) / tsig(t), (-h).expm1()
            plan["n_slots"] = 2
            if i == 0 or float(sn) < 1e-14:
                _plan_eval(plan, i, s, dict(a=m1, c=-m2), kind="D", hist_write=i % 2)
            else:
                rr = (t - nlog(sig[i - 1])) / h
                m3, m4 = 1 + 1 / (2 * rr), 1 / (2 * rr)
                _plan_eval(plan, i, s, dict(a=m1, c=-float(m2) * float(m3), h0=float(m2) * float(m4)), kind="D",
                           hist=((i - 1) % 2,), hist_write=i % 2)
        else:                                                     # LinearMultistepSampler
            cur = min(i + 1, order)
            cf = [linear_multistep_coeff(cur, sig_np, i, j) for j in range(cur)]
            plan["n_slots"] = order
            hist = tuple((i - 1 - j) % order for j in range(cur - 1))
            _plan_eval(plan, i, s, dict(a=1.0, c=cf[0], **{f"h{j}": cf[j + 1] for j in range(cur - 1)}), kind="d",
                       hist=hist, hist_write=i % order)
    plan["evals"][-1]["eval_out"] = False                         # nothing reads the input after the last forward
    if plan["evals"][-1]["hist_write"] is not None:
        plan["evals"][-1]["hist_write"] = None
    E = len(plan["evals"])
    plan["coef"] = torch.tensor([e["coef"] for e in plan["evals"]], dtype=torch.float32).reshape(E, 12)
    plan["t_idx"] = torch.tensor([float(e["t_idx"]) for e in plan["evals"]], dtype=torch.float32)
    plan["c_in"] = torch.tensor([e["c_in"] for e in plan["evals"]], dtype=torch.float32)
    del plan["_table"]
    _PLANS[key] = plan
    return plan


@torch.no_grad()
def _sample_t23d_plan(model, randn, c, uc, plan, noise):
    """The evaluation plan's loop: one DiT forward of the 2B CFG batch per entry (a graph replay), then one
    ln3_sampler_step that writes the state, both halves of the next forward's input and the history slot."""
    B, dev = randn.shape[0], randn.device
    if noise is not None and (tuple(noise.shape) != (plan["num_steps"],) + tuple(randn.shape) or not noise.is_cuda):
        raise ValueError(f"noise must be a CUDA tensor of shape {(plan['num_steps'],) + tuple(randn.shape)}")
    tabs = plan.setdefault("_device", {}).get((B, dev))
    if tabs is None:
        tabs = plan["_device"][(B, dev)] = dict(
            t_idx=plan["t_idx"].to(dev)[:, None].repeat(1, 2 * B).contiguous(),
            c_in=plan["c_in"].to(dev)[:, None].repeat(1, 2 * B).contiguous(),
            coef=plan["coef"].to(dev)[:, None, :].repeat(1, B, 1).contiguous())
    fw = model.step_forward(2 * B, _cfg_context(c, uc), tabs["t_idx"], tabs["c_in"])
    xs = (randn.float() * plan["init_scale"]).contiguous()
    slots = [torch.empty_like(xs) for _ in range(plan["n_slots"])]
    xin = fw.x
    xin[:B].copy_(xs)
    xin[B:].copy_(xs)
    for k, ev in enumerate(plan["evals"]):
        net = fw(k)
        nz = None
        if ev["draw"]:
            nz = noise[ev["step"]] if noise is not None else torch.randn_like(xs)
        ops.sampler_step(xs, xin[:B], tabs["coef"][k], net[:B], net[B:], [slots[j] for j in ev["hist"]],
                         nz if ev["noise"] else None, x_out=xs if ev["x_out"] else None,
                         eval_out=xin if ev["eval_out"] else None,
                         hist_out=slots[ev["hist_write"]] if ev["hist_write"] is not None else None)
    return xs


@torch.no_grad()
def sample_t23d(model, randn: torch.Tensor, c: dict, uc: dict, num_steps: int = 250,
                scale: float = 6.5, tables: dict | None = None,
                sampler: str = "EulerEDMSampler", eta: float = 1.0, s_noise: float = 1.0, order: int = 4,
                noise: torch.Tensor | None = None, s_churn: float = 0.0) -> torch.Tensor:
    """randn (B, 12, 32, 32) fp32 on the GPU (the reference draws it on the CPU generator and moves
    it, sgm_DiffusionEngine.py:395); c / uc = {'crossattn': (B, 77, ctx_dim)} (and 'vector' (B, ctx_dim) for the
    PixArt-style denoiser).  Returns the denoised latents (B, 12, 32, 32) fp32.

    Every denoiser evaluation is one forward of the 2B-sample CFG batch (uc rows first) through the model's
    `step_forward`: a replay of its cached CUDA graph, or eager launches under LN3_CUDA_GRAPH=0.

    `sampler` is one of the reference's sgm class names (SAMPLERS): 'EulerEDMSampler' (the default, the
    engine's) or HeunEDMSampler, EulerAncestralSampler, DPMPP2SAncestralSampler, DPMPP2MSampler and
    LinearMultistepSampler with the reference's parameters eta / s_noise (ancestral), order (LMS).  The ancestral
    samplers draw one `torch.randn_like` of the state per step on the device generator, in the reference's order;
    `noise` (num_steps, B, 12, 32, 32) replaces those draws.  `tables` (edm_cfg_tables) is Euler-only.  Stochastic
    churn (s_churn > 0) is not fused: use the mirrored sampler classes for it."""
    if not randn.is_cuda:
        raise RuntimeError("sample_t23d runs on CUDA only (no CPU fallback)")
    if s_churn > 0:
        raise ValueError("sample_t23d does not fuse stochastic churn (s_churn > 0); use the sgm sampler classes")
    if sampler != "EulerEDMSampler":
        if tables is not None:
            raise ValueError("tables= holds Euler-EDM coefficients; it cannot be used with sampler=" + repr(sampler))
        plan = edm_sampler_plan(sampler, num_steps, scale, eta, s_noise, order)
        return _sample_t23d_plan(model, randn, c, uc, plan, noise)
    if noise is not None:
        raise ValueError("EulerEDMSampler draws no noise; noise= is for the ancestral samplers")
    B = randn.shape[0]
    if tables is None:
        tables = edm_cfg_tables(num_steps, scale, B, randn.device)
    fw = model.step_forward(2 * B, _cfg_context(c, uc), tables["t_idx"][:num_steps], tables["c_in"][:num_steps])
    xa = (randn.float() * tables["init_scale"]).contiguous()
    xb = torch.empty_like(xa)
    for i in range(num_steps):
        fw.x[:B].copy_(xa)
        fw.x[B:].copy_(xa)
        net = fw(i)
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
    (B,V,1,H,W), image_mask (B,V,1,H,W).  The samples per ray S (coarse = importance, 64 or 96) come from
    decoder.rendering_kwargs['depth_resolution'].  `noise` = (coarse, fine) tensors of shape (B*V, H*W, S) to
    override the device RNG (tests).  The sampling noise costs 8*S bytes per ray, so the views are rendered in
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
    kw = decoder.rendering_kwargs
    S = kw.get("depth_resolution", 64)
    if max_views_per_launch is None:
        max_views_per_launch = max(V, (2 << 30) // (2 * M * S * 4))
    obj_per_launch = max(1, min(B, max_views_per_launch // V))
    osg = decoder.triplane_decoder.decoder.raw_parameters()
    rgb = torch.empty(B, V, 3, H, W, device=dev)
    depth = torch.empty(B, V, 1, H, W, device=dev)
    wts = torch.empty(B, V, 1, H, W, device=dev)
    for b0 in range(0, B, obj_per_launch):
        nb = min(obj_per_launch, B - b0)
        if noise is None:
            nz = (torch.rand(nb * V, M, S, device=dev), torch.rand(nb * V, M, S, device=dev))
        else:
            nz = (noise[0][b0 * V:(b0 + nb) * V].contiguous(), noise[1][b0 * V:(b0 + nb) * V].contiguous())
        out = ops.render_views(planes_cl[b0:b0 + nb], ray_o1.repeat(nb, 1, 1), ray_d1.repeat(nb, 1, 1), nz[0], nz[1],
                               osg, views_per_obj=V, group_size=1,
                               box_warp=kw.get("box_warp", 0.9), bbox_min=kw.get("sampler_bbox_min", -0.45),
                               bbox_max=kw.get("sampler_bbox_max", 0.45), white_back=kw.get("white_back", True),
                               mlp_tf32=mlp_tf32, samples_per_ray=S)
        rgb[b0:b0 + nb].copy_(out["rgb"].view(nb, V, 3, H, W))
        depth[b0:b0 + nb].copy_(out["depth"].view(nb, V, 1, H, W))
        wts[b0:b0 + nb].copy_(out["weights"].view(nb, V, 1, H, W))
    return dict(image_raw=rgb, image_depth=depth, weights_samples=wts, image_mask=wts * (1 + 2 * 0.001) - 0.001)


@torch.no_grad()
def generate_t23d(model, decoder, randn, c, uc, cameras, num_steps: int = 250, scale: float = 6.5,
                  resolution: int = 128, sampler: str = "EulerEDMSampler", **sampler_kwargs):
    """Text-to-3D end to end on one GPU: sample -> decode -> render (the body of
    DiffusionEngineLSGM.eval_cldm, nsr/lsgm/sgm_DiffusionEngine.py:410-523, minus conditioner + video sink).
    `sampler` and `sampler_kwargs` (eta, s_noise, order, noise) go to sample_t23d."""
    latents = sample_t23d(model, randn, c, uc, num_steps, scale, sampler=sampler, **sampler_kwargs)
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
               scale: float = 6.5, resolution: int = 128, seed: int = 41, sampler: str = "EulerEDMSampler",
               **sampler_kwargs):
    """eval_cldm for one caption end to end (:410-523): conditioner -> `th.manual_seed(41)` CPU noise draw (:457-466,
    395-398) -> Euler-EDM + CFG sampling (or `sampler`, see sample_t23d) -> decode -> render.
    Returns (latents, render dict)."""
    dev = next(model.parameters()).device
    c, uc = condition_prompt(conditioner, "caption", prompt, num_samples, device=dev)
    g = torch.Generator().manual_seed(seed)
    C = model.in_channels if not model.roll_out else 3 * model.in_channels
    randn = torch.randn(num_samples, C, 32, 32, generator=g).to(dev)
    return generate_t23d(model, decoder, randn, c, uc, cameras, num_steps, scale, resolution, sampler, **sampler_kwargs)


@torch.no_grad()
def sample_flow(model, c: dict, uc: dict, num_samples: int, seed: int = 42, num_steps: int = 250,
                cfg_scale: float = 4.0, sampling_method: str = "dopri5", dtype=torch.float32,
                sde: dict | None = None) -> torch.Tensor:
    """`FlowMatchingEngine.sample` (nsr/lsgm/flow_matching_trainer.py:509-551) for the image-conditioned denoisers
    (I23D 'img', MV23D 'img-c'): global `torch.manual_seed(seed)` -- which also seeds the CUDA generators that the
    renderer's noise draws use afterwards -- then a CPU `randn(num_samples, 12, 32, 32)`, the CFG batch
    cat((cond, uc)) per conditioning key and cat([zs, zs]), `Sampler(create_transport(snr_type='lognorm'))
    .sample_ode(num_steps=..., sampling_method=...)` around `model.forward_with_cfg`, and `[-1].chunk(2)[0]`.

    Engine dtype: as on the existing I23D path, the ODE state and the context are carried in fp32 and the denoiser
    rounds its GEMM operands to bf16 itself.  The engine's `.to(self.dtype)` casts of the noise and the context
    (bf16 under `use_amp`) are applied as roundings to `dtype`; the default float32 leaves them exact.

    `sde`: a dict of `sample_sde` keywords samples with the SDE instead of the ODE (see `sample_flow_sde`).
    Returns the denoised latents (num_samples, 12, 32, 32) fp32."""
    from .transport import Sampler, create_transport
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("sample_flow runs on CUDA only (no CPU fallback)")
    _check_sde_method(sde, sampling_method)
    C = 3 * model.in_channels if model.roll_out else model.in_channels
    zs = flow_batch_noise(1, num_samples, (C, model.input_size, model.input_size), seed).to(dev).to(dtype).float()
    ctx = flow_batch_context(c, uc, dev, dtype)
    if sde is not None:
        return sample_flow_sde(model, zs, ctx, num_samples, num_steps, cfg_scale, sde)[0][:num_samples]
    fn = Sampler(create_transport(snr_type="lognorm")).sample_ode(sampling_method=sampling_method, num_steps=num_steps)
    samples = fn(torch.cat([zs, zs], 0), model.forward_with_cfg, context=ctx, cfg_scale=cfg_scale)[-1]
    return samples.chunk(2, dim=0)[0]


# ---------------------------------------------------------------------------------------------- flow SDE
# parse_sde_args' defaults (transport/train_utils.py:23-33); num_steps comes from the sampling function.
SDE_DEFAULTS = dict(sampling_method="Euler", diffusion_form="sigma", diffusion_norm=1.0, last_step="Mean",
                    last_step_size=0.04)


def sde_options(sde: dict) -> dict:
    """`sde=` of the flow pipelines completed with SDE_DEFAULTS."""
    unknown = set(sde) - set(SDE_DEFAULTS)
    if unknown:
        raise ValueError(f"sde= takes the sample_sde keywords {sorted(SDE_DEFAULTS)} (num_steps comes from the "
                         f"function), got {sorted(unknown)}")
    return {**SDE_DEFAULTS, **sde}


def _check_sde_method(sde, sampling_method):
    if sde is not None and sampling_method != "dopri5":
        raise ValueError(f"sampling_method={sampling_method!r} selects an ODE solver; with sde= the SDE method is "
                         "sde['sampling_method']")


class _PinnedNoise:
    """Step noise on the global CPU generator, `randn(shape)` per call as the reference draws it, moved to the device
    through a ring of pinned buffers and non-blocking copies: the host waits only for the copy made `depth` draws
    earlier, never for the stream.  Returns one device buffer that every call overwrites in stream order."""

    def __init__(self, shape, device, depth: int = 3):
        self.host = [torch.empty(shape).pin_memory() for _ in range(depth)]
        self.copied = [None] * depth
        self.dev = torch.empty(shape, device=device)
        self.k = 0

    def __call__(self, step: int) -> torch.Tensor:
        i = self.k % len(self.host)
        self.k += 1
        if self.copied[i] is not None:
            self.copied[i].synchronize()
        torch.randn(self.host[i].shape, out=self.host[i])
        self.dev.copy_(self.host[i], non_blocking=True)
        self.copied[i] = torch.cuda.Event()
        self.copied[i].record()
        return self.dev


@torch.no_grad()
def sample_flow_sde(model, zs: torch.Tensor, ctx: dict, num_samples: int, num_steps: int, cfg_scale: float,
                    sde: dict):
    """`Sampler(create_transport(snr_type='lognorm')).sample_sde(**sde, num_steps=num_steps)` on cat([zs, zs]) around
    `model.forward_with_cfg`, keeping only the running state (transport/transport.py:sde_fused): per drift evaluation
    one forward of the 2R-row CFG batch (a CUDA-graph replay) and one ln3_flow_sde_step.  zs (R, ...) CUDA fp32 holds
    R / num_samples conditions of num_samples rows; ctx is the CFG context cat((c, uc)).  Each step draws the
    reference's randn(2 * num_samples, ...) on the global CPU generator, which every condition shares.
    Returns (final state (2R, ...), the evaluation plan)."""
    from .transport.transport import sde_fused, sde_plan
    o = sde_options(sde)
    plan = sde_plan(o["sampling_method"], o["diffusion_form"], o["diffusion_norm"], o["last_step"],
                    o["last_step_size"], num_steps)
    draw = _PinnedNoise((2 * num_samples,) + tuple(zs.shape[1:]), zs.device)
    return sde_fused(plan, model, torch.cat([zs, zs], 0), ctx, cfg_scale, draw), plan


def flow_batch_row_groups(P: int, num_samples: int) -> torch.Tensor:
    """The condition of every row of the batched CFG state cat([zs, zs]) of P conditions x num_samples samples
    (condition-major): rows [gN, (g+1)N) and [PN + gN, PN + (g+1)N) are condition g.  int32 (2PN,)."""
    g = torch.arange(P, dtype=torch.int32).repeat_interleave(num_samples)
    return torch.cat([g, g])


def flow_batch_noise(P: int, num_samples: int, shape: tuple, seed: int = 42) -> torch.Tensor:
    """The initial noise of P conditions, (P*N, *shape) condition-major: each condition gets the draw `sample_flow`
    makes, `torch.manual_seed(seed); randn(N, *shape)` on the CPU (so all conditions get the same noise, as P
    sequential calls would).  Seeds the global generators as sample_flow does."""
    torch.manual_seed(seed)
    zs = torch.randn(num_samples, *shape)
    return zs.repeat(P, *([1] * len(shape)))


def flow_batch_context(c: dict, uc: dict, dev=None, dtype=torch.float32) -> dict:
    """The CFG context of `sample_flow` for stacked conditions: cat((c, uc)) per tensor key (conditional rows first),
    rounded to `dtype` and carried in fp32; other keys must agree between c and uc and are passed through."""
    ctx = {}
    for k in c:
        if k in ("vector", "crossattn", "concat"):
            ctx[k] = torch.cat((c[k], uc[k]), 0).to(dev).to(dtype).float().contiguous()
        else:
            assert c[k] == uc[k]
            ctx[k] = c[k]
    return ctx


@torch.no_grad()
def sample_flow_batched(model, c: dict, uc: dict, num_samples: int, seed: int = 42, num_steps: int = 250,
                        cfg_scale: float = 4.0, dtype=torch.float32, sde: dict | None = None,
                        sampling_method: str = "dopri5"):
    """`sample_flow` for P conditions in one denoiser batch.  c / uc hold P conditions stacked condition-major, each
    repeated `num_samples` times as `condition_prompt` returns it ((P*N, ...) per key).  The batch is cat([zs, zs])
    of 2PN rows with context cat((c, uc)); the noise is `flow_batch_noise` (sample_flow's draw for every condition).
    num_steps is the output grid of sample_ode.

    `sampling_method`: an adaptive method (dopri5, bosh3, fehlberg2, adaptive_heun) runs every condition on its own
    trajectory (transport/rk.py:odeint_rk_adaptive_grouped), so its latents do not depend on the other conditions in
    the batch; it only uses the grid's last point, t = 1.  A fixed-grid method (euler, midpoint, heun, rk4) steps the
    whole batch on the grid, which every condition shares.  Any other name raises NotImplementedError.
    Returns (latents (P, N, 12, 32, 32) fp32, stats) with per-condition lists nfe (and, for an adaptive method,
    accepted / rejected) and the batch's forward count batch_nfe.

    With `sde` (a dict of `sample_sde` keywords, see `sample_flow_sde`) the P conditions instead run the SDE on the
    shared fixed grid of num_steps points; every condition reads the noise draw its own `sample_flow(..., sde=)` call
    would make, so its latents are that call's up to the rounding of the batched GEMMs.  stats then hold nfe (per
    condition) and batch_nfe, both the forward count."""
    from .transport import rk
    _check_sde_method(sde, sampling_method)
    if sampling_method not in rk.FIXED_GRID_METHODS:
        rk.tableau(sampling_method)                   # NotImplementedError naming the built methods
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("sample_flow_batched runs on CUDA only (no CPU fallback)")
    N = num_samples
    rows = next(v for k, v in c.items() if k in ("vector", "crossattn", "concat")).shape[0]
    assert rows % N == 0, "c must hold num_samples rows per condition"
    P = rows // N
    C = 3 * model.in_channels if model.roll_out else model.in_channels
    shape = (C, model.input_size, model.input_size)
    zs = flow_batch_noise(P, N, shape, seed).to(dev).to(dtype).float()
    ctx = flow_batch_context(c, uc, dev, dtype)
    if sde is not None:
        x, plan = sample_flow_sde(model, zs, ctx, N, num_steps, cfg_scale, sde)
        return x[:P * N].reshape(P, N, *shape), dict(nfe=[plan["forwards"]] * P, batch_nfe=plan["forwards"])
    if sampling_method in rk.FIXED_GRID_METHODS:
        from .transport import Sampler, create_transport
        fn = Sampler(create_transport(snr_type="lognorm")).sample_ode(sampling_method=sampling_method,
                                                                       num_steps=num_steps)
        y = fn(torch.cat([zs, zs], 0), model.forward_with_cfg, context=ctx, cfg_scale=cfg_scale)[-1]
        nfe = rk.FIXED_GRID_FORWARDS[sampling_method] * (num_steps - 1)
        return y[:P * N].reshape(P, N, *shape), dict(nfe=[nfe] * P, batch_nfe=nfe)
    grid = torch.linspace(0, 1, num_steps)            # sample_ode's grid: the solver integrates to its last point
    fn = lambda t, x: model.forward_with_cfg(x, t, ctx, cfg_scale)
    if sampling_method == "dopri5":
        from .transport.dopri5 import odeint_dopri5_grouped
        y, stats = odeint_dopri5_grouped(fn, torch.cat([zs, zs], 0), flow_batch_row_groups(P, N), P,
                                         t0=float(grid[0]), t1=float(grid[-1]), rtol=1e-3, atol=1e-6)
    else:
        y, stats = rk.odeint_rk_adaptive_grouped(fn, torch.cat([zs, zs], 0), flow_batch_row_groups(P, N), P,
                                                 t0=float(grid[0]), t1=float(grid[-1]), method=sampling_method,
                                                 rtol=1e-3, atol=1e-6)
    return y[:P * N].reshape(P, N, *shape), stats


def _condition_list(conditioner, cond_key, prompts, num_samples, dev):
    """condition_prompt once per prompt, in order, stacked condition-major: (c, uc) with (P*N, ...) per tensor key."""
    cs, ucs = zip(*(condition_prompt(conditioner, cond_key, p, num_samples, device=dev) for p in prompts))
    c = {k: torch.cat([ci[k] for ci in cs]) if isinstance(cs[0][k], torch.Tensor) else cs[0][k] for k in cs[0]}
    uc = {k: torch.cat([ui[k] for ui in ucs]) if isinstance(ucs[0][k], torch.Tensor) else ucs[0][k] for k in ucs[0]}
    return c, uc


def _own(x, dev, dtype):
    """A condition's own copy on `dev` in `dtype` (a tensor, or a dict of them): the conditioner's kernels want
    16-byte aligned rows, and aug_c rotates the cameras of this copy in place."""
    if isinstance(x, dict):
        return {k: _own(v, dev, dtype) for k, v in x.items()}
    return x.to(dev).to(dtype).clone()


@torch.no_grad()
def _conds_to_3d(conditioner, model, decoder, cond_key, prompts, cameras, num_samples, seed, num_steps, cfg_scale,
                 resolution, dtype, sde, sampling_method):
    """`_cond_to_3d` for a list of conditions: the conditioner once per condition, in order, one batched sample,
    then decode and render of every latent.  The render noise is one device draw for the batch."""
    dev = next(model.parameters()).device
    c, uc = _condition_list(conditioner, cond_key, prompts, num_samples, dev)
    latents, stats = sample_flow_batched(model, c, uc, num_samples, seed=seed, num_steps=num_steps,
                                         cfg_scale=cfg_scale, dtype=dtype, sde=sde, sampling_method=sampling_method)
    P, N = latents.shape[:2]
    out = decode_and_render(decoder, latents.reshape(P * N, *latents.shape[2:]), cameras[:24].to(dev), resolution)
    return latents, {k: v.reshape(P, N, *v.shape[1:]) for k, v in out.items()}, stats


@torch.no_grad()
def images_to_3d(conditioner, model, decoder, images: torch.Tensor, cameras: torch.Tensor, num_samples: int = 4,
                 seed: int = 42, num_steps: int = 250, cfg_scale: float = 4.0, resolution: int = 192,
                 dtype=torch.float32, sde: dict | None = None, sampling_method: str = "dopri5"):
    """`image_to_3d` for P images (P, 3, H, W) in [-1, 1] in one denoiser batch.  Each image's latents are those
    `image_to_3d` gives for it alone up to the rounding of the batched GEMMs; the renders use one device noise draw
    for the whole batch, so they are not bit-identical to sequential calls.  `sde`, `sampling_method`: see
    sample_flow_batched.
    Returns (latents (P, N, 12, 32, 32), render dict with (P, N, 24, ...) tensors, per-image stats)."""
    dev = next(model.parameters()).device
    imgs = [_own(images[i:i + 1], dev, dtype) for i in range(images.shape[0])]
    return _conds_to_3d(conditioner, model, decoder, "img", imgs, cameras, num_samples, seed, num_steps, cfg_scale,
                        resolution, dtype, sde, sampling_method)


@torch.no_grad()
def mvs_to_3d(conditioner, model, decoder, mv_images: torch.Tensor, mv_cameras: torch.Tensor, cameras: torch.Tensor,
              num_samples: int = 4, seed: int = 42, num_steps: int = 250, cfg_scale: float = 4.0,
              resolution: int = 192, dtype=torch.float32, sde: dict | None = None, sampling_method: str = "dopri5"):
    """`mv_to_3d` for P multi-view conditions, mv_images (P, V, 3, H, W) and mv_cameras (P, V, 25), in one
    denoiser batch.  The conditioner runs once per condition in order, so its `aug_c` camera draws follow the same
    sequence as P sequential `mv_to_3d` calls.  Every condition gets its own copy of its views and cameras (the
    conditioner's kernels want 16-byte aligned rows), so with `aug_c=True` the rotations apply to those copies and the
    caller's `mv_cameras` is left as it is.  `sde`, `sampling_method`: see sample_flow_batched.  Returns as
    `images_to_3d`."""
    dev = next(model.parameters()).device
    prompts = [_own({"img": mv_images[i:i + 1], "c": mv_cameras[i:i + 1]}, dev, dtype)
               for i in range(mv_images.shape[0])]
    return _conds_to_3d(conditioner, model, decoder, "img-c", prompts, cameras, num_samples, seed, num_steps,
                        cfg_scale, resolution, dtype, sde, sampling_method)


@torch.no_grad()
def _conds_to_3d_sharded(conditioner, model, decoder, cond_key, P, host_prompt, cameras, *, num_samples, seed,
                         num_steps, cfg_scale, resolution, dtype, sde, sampling_method, batch, with_depth, device,
                         group, gather, sample_fn, render_fn, pack_fn):
    """The body of images_to_3d_sharded / mvs_to_3d_sharded; host_prompt(i) is condition i as the caller holds it."""
    dev = torch.device(device) if device is not None else next(model.parameters()).device
    N = num_samples
    lo, hi, per = shard_range(P, *_world_rank(group))
    if sample_fn is None:
        sample_fn = lambda c, uc: sample_flow_batched(model, c, uc, N, seed=seed, num_steps=num_steps,
                                                      cfg_scale=cfg_scale, dtype=dtype, sde=sde,
                                                      sampling_method=sampling_method)
    if render_fn is None:
        cams = cameras[:24].to(dev)
        render_fn = lambda lat: decode_and_render(decoder, lat, cams, resolution)
    if pack_fn is None:
        pack_fn = _frame_packer(dev, with_depth)
    frame_shape = (N, min(cameras.shape[0], 24), resolution, resolution * (2 if with_depth else 1), 3)
    latents = torch.zeros(per, N, 12, 32, 32, device=dev)
    stats: dict = {}

    def run_batch(i0, i1):
        c, uc = _condition_list(conditioner, cond_key, [_own(host_prompt(i), dev, dtype) for i in range(i0, i1)], N,
                                dev)
        lat, st = sample_fn(c, uc)
        latents[i0 - lo:i1 - lo].copy_(lat)
        for k, v in st.items():
            if isinstance(v, list):                   # per-condition counts; batch_nfe belongs to one batch only
                stats.setdefault(k, []).extend(v)
        return pack_fn(render_fn(lat.reshape(-1, *lat.shape[2:]))).reshape(i1 - i0, *frame_shape)

    # every rank draws the host RNG of all P conditions in order (aug_c), and applies only its own shard's draws
    for i in range(lo):
        conditioner.skip_unconditional_conditioning({cond_key: host_prompt(i)})
    out = _sharded_frames(P, batch, frame_shape, dev, group, gather, run_batch)
    for i in range(hi, P):
        conditioner.skip_unconditional_conditioning({cond_key: host_prompt(i)})
    return dict(latents=latents[:hi - lo], stats=stats, **out)


@torch.no_grad()
def images_to_3d_sharded(conditioner, model, decoder, images: torch.Tensor, cameras: torch.Tensor,
                         num_samples: int = 4, seed: int = 42, num_steps: int = 250, cfg_scale: float = 4.0,
                         resolution: int = 192, dtype=torch.float32, sde: dict | None = None,
                         sampling_method: str = "dopri5", *, batch: int = 8, with_depth: bool = False, device=None,
                         group=None, gather: bool = True, sample_fn=None, render_fn=None, pack_fn=None) -> dict:
    """`images_to_3d` for P images (P, 3, H, W) sharded over the ranks of `group` (SURVEY 8d configuration 4).

    Every rank holds all P images and owns the contiguous block [lo, hi) of shard_range(P, world, rank).  It works
    through its block in local batches of at most `batch` images; a batch runs the conditioner once per image, in
    order (only on this rank's images), sample_flow_batched (`sampling_method`, `sde` as in images_to_3d),
    decode_and_render of `cameras[:24]` at `resolution`, and FrameSink.pack (image | colour-mapped depth side by side
    with `with_depth`).  Each batch ends with ONE all_gather_into_tensor of its uint8 frames on a side stream, so the
    gather overlaps the next batch; every rank makes the same number of trips, and ranks holding fewer images
    contribute zero frames that are trimmed from the result.

    Equal to one process: each image's initial noise is the draw sample_flow makes (flow_batch_noise), so nothing is
    sliced across ranks, and its latents equal those of images_to_3d over the same image list up to the rounding of
    the batched GEMMs (an adaptive solve is per image, so only the batch size can change them).  With world == 1
    and batch >= P this is images_to_3d, bit for bit, renders included.  The renders of a run with several batches
    use one device noise draw per batch, so they differ from images_to_3d's.

    Returns {'latents': (n_local, N, 12, 32, 32), 'frames': uint8 (n_local, N, V, H, Wout, 3), 'frames_all': uint8
    (P, N, V, H, Wout, 3) in image order on every rank (None with gather=False), 'shard': (lo, hi),
    'gather_bytes_per_rank': int, 'stats': the per-image solver lists (nfe; accepted / rejected for an adaptive
    method) of this rank's images}; V = min(24, len(cameras)), Wout = resolution (2 resolution with depth).
    `sample_fn(c, uc) -> (latents, stats)`, `render_fn(latents (n*N, ...)) -> render dict` and `pack_fn(render dict)`
    replace the three CUDA stages, and `device` the model's device (the gloo test drives this function's sharding,
    condition order and gather with CPU stand-ins)."""
    return _conds_to_3d_sharded(conditioner, model, decoder, "img", images.shape[0], lambda i: images[i:i + 1],
                                cameras, num_samples=num_samples, seed=seed, num_steps=num_steps, cfg_scale=cfg_scale,
                                resolution=resolution, dtype=dtype, sde=sde, sampling_method=sampling_method,
                                batch=batch, with_depth=with_depth, device=device, group=group, gather=gather,
                                sample_fn=sample_fn, render_fn=render_fn, pack_fn=pack_fn)


@torch.no_grad()
def mvs_to_3d_sharded(conditioner, model, decoder, mv_images: torch.Tensor, mv_cameras: torch.Tensor,
                      cameras: torch.Tensor, num_samples: int = 4, seed: int = 42, num_steps: int = 250,
                      cfg_scale: float = 4.0, resolution: int = 192, dtype=torch.float32, sde: dict | None = None,
                      sampling_method: str = "dopri5", *, batch: int = 8, with_depth: bool = False, device=None,
                      group=None, gather: bool = True, sample_fn=None, render_fn=None, pack_fn=None) -> dict:
    """`mvs_to_3d` for P multi-view conditions, mv_images (P, V, 3, H, W) and mv_cameras (P, V, 25), sharded over the
    ranks of `group` as images_to_3d_sharded shards images; arguments and results as there.

    aug_c: the release conditioner (FrozenDinov2ImageEmbedderMVPlucker, aug_c=True) rotates cameras with draws from
    Python `random` and `np.random`, per (condition, view) and in condition order.  So every rank makes the draws of
    ALL P conditions in order -- conditioner.skip_unconditional_conditioning for each condition another rank owns --
    and applies only those of its own conditions, on the device copy of their cameras, in `dtype`.  Each condition
    therefore sees the rotations a single mvs_to_3d call gives it after the same seeds, and every rank leaves both
    generators where that call leaves them.  The caller's `mv_cameras` is never rotated."""
    return _conds_to_3d_sharded(conditioner, model, decoder, "img-c", mv_images.shape[0],
                                lambda i: {"img": mv_images[i:i + 1], "c": mv_cameras[i:i + 1]}, cameras,
                                num_samples=num_samples, seed=seed, num_steps=num_steps, cfg_scale=cfg_scale,
                                resolution=resolution, dtype=dtype, sde=sde, sampling_method=sampling_method,
                                batch=batch, with_depth=with_depth, device=device, group=group, gather=gather,
                                sample_fn=sample_fn, render_fn=render_fn, pack_fn=pack_fn)


@torch.no_grad()
def _cond_to_3d(conditioner, model, decoder, cond_key, prompt, cameras, num_samples, seed, num_steps, cfg_scale,
                sampling_method, resolution, dtype, sde):
    dev = next(model.parameters()).device
    c, uc = condition_prompt(conditioner, cond_key, prompt, num_samples, device=dev)
    latents = sample_flow(model, c, uc, num_samples, seed=seed, num_steps=num_steps, cfg_scale=cfg_scale,
                          sampling_method=sampling_method, dtype=dtype, sde=sde)
    return latents, decode_and_render(decoder, latents, cameras[:24].to(dev), resolution)


@torch.no_grad()
def mv_to_3d(conditioner, model, decoder, mv_images: torch.Tensor, mv_cameras: torch.Tensor, cameras: torch.Tensor,
             num_samples: int = 4, seed: int = 42, num_steps: int = 250, cfg_scale: float = 4.0,
             sampling_method: str = "dopri5", resolution: int = 192, dtype=torch.float32, sde: dict | None = None):
    """Multi-view-to-3D, `FlowMatchingEngine.eval_cldm` for cond_key 'img-c' (nsr/lsgm/flow_matching_trainer.py:
    553-678): the conditioner on {'img': mv_images (1, V, 3, H, W) in [-1, 1], 'c': mv_cameras (1, V, 25)} with the
    unconditional half forced to zero and every row repeated `num_samples` times, `sample_flow`, then decode and render
    of `cameras[:24]` at `resolution`.  The release (sample_obajverse_mv23d_dit.sh) runs 6 views, 4 samples, CFG 4.0,
    dopri5 with 250 output points and 192^2 renders.

    The engine casts the views and cameras to its dtype (bf16 under use_amp) before the conditioner sees them; they
    are cast to `dtype` here.  With `aug_c=True` the conditioner rotates cameras of that tensor in place -- the caller's
    own `mv_cameras` when it already has that dtype and device.  `sde`: see sample_flow.  Returns (latents, render
    dict)."""
    dev = next(model.parameters()).device
    img_c = {"img": mv_images.to(dev).to(dtype), "c": mv_cameras.to(dev).to(dtype)}
    return _cond_to_3d(conditioner, model, decoder, "img-c", img_c, cameras, num_samples, seed, num_steps, cfg_scale,
                       sampling_method, resolution, dtype, sde)


@torch.no_grad()
def image_to_3d(conditioner, model, decoder, image: torch.Tensor, cameras: torch.Tensor, num_samples: int = 4,
                seed: int = 42, num_steps: int = 250, cfg_scale: float = 4.0, sampling_method: str = "dopri5",
                resolution: int = 192, dtype=torch.float32, sde: dict | None = None):
    """Image-to-3D, `FlowMatchingEngine.eval_cldm` for cond_key 'img' (the I23D release): the conditioner on one image
    (1, 3, H, W) in [-1, 1], `sample_flow`, decode and render of `cameras[:24]`.  `sde`: see sample_flow.
    Returns (latents, render dict)."""
    dev = next(model.parameters()).device
    return _cond_to_3d(conditioner, model, decoder, "img", image.to(dev).to(dtype), cameras, num_samples, seed,
                       num_steps, cfg_scale, sampling_method, resolution, dtype, sde)


@torch.no_grad()
def encode_latents(encoder, decoder, img_to_encoder: torch.Tensor, sample_posterior: bool = True) -> dict:
    """`AE.forward(img=img_to_encoder, behaviour='encoder_vae')` (nsr/script_util.py:326-329), the first step of
    `eval_novelview_loop` (nsr/train_nv_util.py:1177-1219): img_to_encoder (B*F, 10, 256, 256) fp32 with
    F = encoder.num_frames views per object (4 for MVEncoder, 6 for the DiT2-L/2 VAE's MVEncoderGSDynamicInp) -- per
    view RGB in [-1, 1], the Plücker rays o x d and d, and depth -- through the encoder to the moments (B, 24, 32, 32),
    then the decoder's vae_reparameterization.  Returns the reference's dict; `latent_normalized_2Ddiffusion` (B, 12, 32, 32) is
    the latent every stage-2 DiT is trained on (what `--save_latent True` writes).  sample_posterior draws the noise
    from the CPU generator, as the reference does."""
    if not img_to_encoder.is_cuda:
        raise RuntimeError("encode_latents runs on CUDA only (no CPU fallback)")
    return decoder.vae_reparameterization(encoder(img_to_encoder), sample_posterior)


@torch.no_grad()
def reconstruct(encoder, decoder, img_to_encoder: torch.Tensor, cameras: torch.Tensor, resolution: int = 128,
                scaling_divider: float = 1.0, sample_posterior: bool = True, noise: tuple | None = None,
                mlp_tf32: bool = True):
    """3D reconstruction from multi-view images, the body of `eval_novelview_loop`: `encode_latents` of img_to_encoder
    (B*F, 10, 256, 256), F = encoder.num_frames, then decode and render of every camera of `cameras` (V, 25) for every
    object at the decoder's samples per ray.  The reconstruction trainer renders the posterior
    latent with `triplane_scaling_divider = 1.0` (TrainLoop3DRec, nsr/train_util.py:565, applied at :580).
    Returns (the encoder_vae dict, the render dict of `decode_and_render`)."""
    ret = encode_latents(encoder, decoder, img_to_encoder, sample_posterior)
    out = decode_and_render(decoder, ret["latent_normalized_2Ddiffusion"], cameras, resolution,
                            scaling_divider=scaling_divider, noise=noise, mlp_tf32=mlp_tf32)
    return ret, out


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
    P = c_all["crossattn"].shape[0]
    dev = torch.device(device) if device is not None else next(model.parameters()).device
    g = torch.Generator().manual_seed(seed)
    randn_all = torch.randn(P, 12, 32, 32, generator=g)                      # identical on every rank
    if sample_fn is None:
        sample_fn = lambda x, c, uc: sample_t23d(model, x, c, uc, num_steps, scale)
    if render_fn is None:
        render_fn = lambda lat: decode_and_render(decoder, lat, cameras, resolution)
    if pack_fn is None:
        pack_fn = _frame_packer(dev, with_depth)
    lo, hi, per = shard_range(P, *_world_rank(group))
    latents = torch.zeros(per, 12, 32, 32, device=dev)

    def run_batch(i0, i1):
        sl = slice(i0, i1)
        x = randn_all[sl].to(dev, non_blocking=True)
        c = {"crossattn": c_all["crossattn"][sl].to(dev, non_blocking=True)}
        uc = {"crossattn": uc_all["crossattn"][sl].to(dev, non_blocking=True)}
        lat = sample_fn(x, c, uc)
        latents[i0 - lo:i1 - lo].copy_(lat)
        return pack_fn(render_fn(lat))

    out = _sharded_frames(P, batch, (cameras.shape[0], resolution, resolution * (2 if with_depth else 1), 3), dev,
                          group, gather, run_batch)
    return dict(latents=latents[:hi - lo], **out)


def _world_rank(group) -> tuple[int, int]:
    """(world size, rank) of `group`, or (1, 0) without an initialised process group."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


def _frame_packer(dev, with_depth: bool):
    """The default pack stage of the sharded pipelines: FrameSink.pack of image_raw (and image_depth)."""
    from .frames import FrameSink
    sink = FrameSink(dev)
    return lambda r: sink.pack(r["image_raw"], r["image_depth"] if with_depth else None)


def _sharded_frames(P: int, batch: int, frame_shape: tuple, dev, group, gather: bool, run_batch) -> dict:
    """The batch loop and frame gather that every sharded pipeline shares.  This rank of `group` owns the contiguous
    block [lo, hi) of shard_range(P, world, rank) and works through it in local batches of at most `batch` items:
    run_batch(i0, i1) runs the global items [i0, i1) and returns their uint8 frames (i1 - i0, *frame_shape).  Every
    rank makes ceil(per / batch) trips, including ranks that own fewer items or none; each trip ends with ONE
    all_gather_into_tensor of the batch's frame rows (zeros past the rank's last item), issued on a side stream so
    that it overlaps the next batch.  The padding rows are trimmed from the result.
    Returns {'frames': (n_local, *frame_shape), 'frames_all': (P, *frame_shape) in item order on every rank (None if
    not gathered), 'shard': (lo, hi), 'gather_bytes_per_rank': int}."""
    import torch.distributed as dist
    world, rank = _world_rank(group)
    lo, hi, per = shard_range(P, world, rank)
    frames = torch.zeros(per, *frame_shape, dtype=torch.uint8, device=dev)
    do_gather = gather and world > 1
    frames_all = torch.empty(world, per, *frame_shape, dtype=torch.uint8, device=dev) if do_gather else None
    cuda = dev.type == "cuda"
    side = torch.cuda.Stream(device=dev) if (do_gather and cuda) else None
    pending = []
    for b0 in range(0, per, batch):                                          # same trip count on every rank
        b1 = min(b0 + batch, per)
        n_valid = max(0, min(hi - lo, b1) - b0)
        if n_valid > 0:
            frames[b0:b0 + n_valid].copy_(run_batch(lo + b0, lo + b0 + n_valid))
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
    out_all = frames_all.view(world * per, *frame_shape)[:P] if do_gather else (frames[:P] if gather else None)
    return dict(frames=frames[:n_local], frames_all=out_all, shard=(lo, hi),
                gather_bytes_per_rank=int(frames.numel()) if do_gather else 0)
