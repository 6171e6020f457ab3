"""TEST INFRASTRUCTURE ONLY -- restatements of the transport's SDE samplers (reference transport/transport.py:246-372,
integrators.py:9-75, path.py:18-110 for the Linear path with velocity prediction) that the tests hold the library
against:

  sample_sde   plain fp32 torch around any CFG velocity callable, with the noise draws passed in explicitly;
  emulate      the library's evaluation plan (transport.sde_plan) applied in float64 with the ln3_flow_sde_step
               formula around the raw (un-guided) network, i.e. what the fused pipeline computes;
  toy_cfg      a CFG-shaped closed-form network built like oracle.fixtures.toy_network (tests/golden/flow_sde.npz).
"""
from __future__ import annotations

import math

import torch

SEED, N, CFG, STEPS = 7, 2, 4.0, 10
SHAPE = (12, 8, 8)
FORMS = ("sigma", "linear", "decreasing", "inccreasing-decreasing")
LASTS = (None, "Mean", "Tweedie", "Euler")


def toy_raw():
    """The raw network (2R rows, conditional first) -> (2R rows): tanh(W x + 0.001 t + mean(context))."""
    from oracle import fixtures as fx
    return fx.toy_network()


def toy_cfg(raw=None):
    """forward_with_cfg around `raw` (dit_i23d.py:155-168): guided half g = u + s (c - u), returns cat([g, g]).
    `.calls` counts the model calls."""
    raw = raw or toy_raw()

    def model(x, t, context, cfg_scale):
        model.calls += 1
        out = raw(x, t, context)
        c, u = torch.split(out, len(out) // 2, dim=0)
        half = u + cfg_scale * (c - u)
        return torch.cat([half, half], dim=0)
    model.calls = 0
    return model


def inputs():
    """(zs (N, 12, 8, 8) drawn after manual_seed(SEED), CFG context {'crossattn': cat(cond, zeros)}).  Seeds the global
    generator, as the engine does before its draws."""
    g = torch.Generator().manual_seed(19)
    cond = torch.randn(N, 77, 16, generator=g)
    ctx = {"crossattn": torch.cat([cond, torch.zeros_like(cond)], 0)}
    torch.manual_seed(SEED)
    zs = torch.randn(N, *SHAPE)
    return zs, ctx


def noises(num_steps: int, rows: int = 2 * N) -> list:
    """The draws `sample_sde` makes after `inputs()`: one randn(rows, 12, 8, 8) per step but the last."""
    return [torch.randn(rows, *SHAPE) for _ in range(num_steps - 1)]


def _diffusion(t, form, norm):
    if form in ("sigma", "linear"):
        return norm * (1 - t)
    if form == "decreasing":
        return 0.25 * (norm * torch.cos(math.pi * t) + 1) ** 2
    if form == "inccreasing-decreasing":
        return norm * torch.sin(math.pi * t) ** 2
    raise NotImplementedError(form)


def _score(v, x, t):
    sig = 1 - t
    return (t * v - x) / (sig ** 2 + t * sig)


def sample_sde(model, init, context, cfg_scale, noise: list, *, sampling_method="Euler", diffusion_form="sigma",
               diffusion_norm=1.0, last_step="Mean", last_step_size=0.04, num_steps=STEPS):
    """The reference's sample_sde list semantics in plain fp32 torch: returns the final state (2N rows).  Two model
    calls per SDE drift, as the reference makes them."""
    size = 0.0 if last_step is None else last_step_size
    ts = torch.linspace(0, 1 - size, num_steps)
    dt = ts[1] - ts[0]
    col = lambda t: torch.ones(init.shape[0], 1, 1, 1) * t
    vel = lambda x, t: model(x, col(t).flatten(), context, cfg_scale)
    drift = lambda x, t: vel(x, t) + _diffusion(col(t), diffusion_form, diffusion_norm) * _score(vel(x, t), x, col(t))
    x = init
    for i in range(num_steps - 1):
        t, w = ts[i], noise[i]
        sq = torch.sqrt(2 * _diffusion(col(t), diffusion_form, diffusion_norm))
        if sampling_method == "Euler":
            x = x + drift(x, t) * dt + sq * (w * torch.sqrt(dt))
        else:
            xh = x + sq * (w * torch.sqrt(dt))
            k1 = drift(xh, t)
            k2 = drift(xh + dt * k1, t + dt)
            x = xh + 0.5 * dt * (k1 + k2)
    t1 = torch.tensor(1 - size, dtype=torch.float32)
    if last_step == "Mean":
        x = x + drift(x, t1) * size
    elif last_step == "Euler":
        x = x + vel(x, t1) * size
    elif last_step == "Tweedie":
        x = x / t1 + (1 - t1) ** 2 / t1 * _score(vel(x, t1), x, col(t1))
    return x


def emulate(plan: dict, raw, init, context, cfg_scale, noise: list):
    """Apply transport.sde_plan's entries in float64 with the kernel's formula around the raw network (evaluated in
    fp32 on the rounded input, as the denoiser sees it).  noise[k] has 2N rows; R / N conditions share it.
    Returns the final state (2R rows, float64)."""
    R2 = init.shape[0]
    y = init.double().clone()
    x = torch.zeros_like(y)
    hist = torch.zeros_like(y)
    rep = lambda w: w.double().view(2, 1, w.shape[0] // 2, -1).expand(2, R2 // w.shape[0], -1, -1).reshape(y.shape)
    if plan["pre_sigma"] is not None:
        y = y + plan["pre_sigma"] * rep(noise[0])
    for e in plan["evals"]:
        f = raw(y.float(), torch.full((R2,), e["t"]), context).double()
        c, u = f[:R2 // 2], f[R2 // 2:]
        v = u + cfg_scale * (c - u)
        v = torch.cat([v, v])
        sc = (e["t"] * v - y) / e["var"]
        d = (v + e["diffusion"] * sc, v, sc)[e["mode"]]
        w = rep(noise[e["noise"]]) if e["noise"] is not None else torch.zeros_like(y)
        xin = x if e["x_in"] else torch.zeros_like(y)
        hin = hist if e["hist_in"] else torch.zeros_like(y)
        o = lambda k: k[0] * xin + k[1] * y + k[2] * d + k[3] * hin + k[4] * w
        x_new = o(e["cx"])
        y = o(e["cy"]) if e["cy"] is not None else y
        if e["hist_out"]:
            hist = d
        x = x_new
    return x
