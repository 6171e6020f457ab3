"""TEST INFRASTRUCTURE ONLY (oracle) -- fp32 CPU restatements of the five sgm samplers beyond Euler-EDM, and a
float64 emulator of the pipeline's evaluation plans.  Only tests/ and tools/ may import this module.

  HeunEDMSampler, EulerAncestralSampler, DPMPP2SAncestralSampler, DPMPP2MSampler, LinearMultistepSampler
      sgm/modules/diffusionmodules/sampling.py:93-362, sampling_utils.py:7-43
  around DiscreteDenoiser(EpsScaling, 1000) + VanillaCFG(scale) on the LegacyDDPM schedule (the shipped T23D
  denoiser: denoiser.py:13-78, denoiser_scaling.py:29-37, guiders.py:24-42), as oracle.samplers restates Euler.
Pinned by oracle/make_golden_edm_samplers.py against the reference's own classes (tests/golden/edm_samplers.npz).
`network(x_in, idx, cond_dict)` is any callable; ancestral noise is taken from a list, one entry per step.
The LMS coefficients are Gauss-Legendre quadratures (exact for the degree <= 3 integrand), no scipy.
"""
from __future__ import annotations

import numpy as np
import torch

from .samplers import legacy_ddpm_sigmas, sigma_to_idx

SAMPLERS = ("HeunEDMSampler", "EulerAncestralSampler", "DPMPP2SAncestralSampler", "DPMPP2MSampler",
            "LinearMultistepSampler")
SCALE = 6.5
NOISE_SEED = 71


def inputs():
    """x0 (2, 12, 8, 8), cond, uc: the 8x8 corner of oracle.fixtures.sampler_inputs() (the toy network is per pixel)."""
    from .fixtures import sampler_inputs
    x0, c, uc, _, _, _ = sampler_inputs()
    return x0[..., :8, :8].contiguous(), c, uc


def step_noise(num_steps: int, shape=(2, 12, 8, 8)) -> list:
    """The seeded ancestral noise of the golden runs: entry k is the k-th `randn_like` draw of the sampler."""
    g = torch.Generator().manual_seed(NOISE_SEED)
    return [torch.randn(*shape, generator=g) for _ in range(num_steps)]


def lms_coeff(order: int, t, i: int, j: int) -> float:
    """linear_multistep_coeff: the integral of the j-th Lagrange basis polynomial over [t[i], t[i+1]] (float64)."""
    if order - 1 > i:
        raise ValueError(f"Order {order} too high for step {i}")
    t = np.asarray(t, dtype=np.float64)
    xg, wg = np.polynomial.legendre.leggauss(4)
    a, b = t[i], t[i + 1]
    tau = 0.5 * (b - a) * xg + 0.5 * (b + a)
    prod = np.ones_like(tau)
    for k in range(order):
        if k != j:
            prod = prod * (tau - t[i - k]) / (t[i - j] - t[i - k])
    return float(0.5 * (b - a) * np.sum(wg * prod))


def ancestral_step(sigma_from, sigma_to, eta=1.0):
    sigma_up = torch.minimum(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    return (sigma_to ** 2 - sigma_up ** 2) ** 0.5, sigma_up


def _nls(s):
    return s.log().neg()


def _sig(t):
    return t.neg().exp()


def _v(s):
    return s[:, None, None, None]


def edm_sample(sampler: str, network, x: torch.Tensor, cond: dict, uc: dict, num_steps: int, scale: float = SCALE,
               noise: list | None = None, eta: float = 1.0, s_noise: float = 1.0, order: int = 4):
    """`sampler(num_steps)(denoiser, x, cond, uc)` of the reference in its op order (fp32).  Returns (x, draws)."""
    table = legacy_ddpm_sigmas(1000, append_zero=False, flip=True)
    sig = legacy_ddpm_sigmas(num_steps)
    c_cat = {k: torch.cat((uc[k], cond[k]), 0) for k in cond}
    draws = [0]

    def draw():
        draws[0] += 1
        return noise[draws[0] - 1]

    def denoise(xx, sigma):
        xin, sin = torch.cat([xx] * 2), torch.cat([sigma] * 2)
        sq = table[sigma_to_idx(sin, table)]
        sq4 = _v(sq)
        c_in = 1 / (sq4 ** 2 + 1.0) ** 0.5
        den = network(xin * c_in, sigma_to_idx(sq, table), c_cat) * (-sq4) + xin * torch.ones_like(sq4)
        x_u, x_c = den.chunk(2)
        return x_u + scale * (x_c - x_u)

    def noised(xx, nxt, su):
        return torch.where(_v(nxt) > 0.0, xx + draw() * s_noise * _v(su), xx)

    x = x * torch.sqrt(1.0 + sig[0] ** 2.0)
    s_in = x.new_ones([x.shape[0]])
    old, ds = None, []
    for i in range(num_steps):
        sigma, nxt = s_in * sig[i], s_in * sig[i + 1]
        if sampler == "HeunEDMSampler":
            sh = sigma * (0.0 + 1.0)
            d = (x - denoise(x, sh)) / _v(sh)
            dt = _v(nxt - sh)
            xe = x + dt * d
            if torch.sum(nxt) < 1e-14:
                x = xe
            else:
                dn = (xe - denoise(xe, nxt)) / _v(nxt)
                x = torch.where(_v(nxt) > 0.0, x + (d + dn) / 2.0 * dt, xe)
        elif sampler == "EulerAncestralSampler":
            sd, su = ancestral_step(sigma, nxt, eta)
            d = (x - denoise(x, sigma)) / _v(sigma)
            x = noised(x + _v(sd - sigma) * d, nxt, su)
        elif sampler == "DPMPP2SAncestralSampler":
            sd, su = ancestral_step(sigma, nxt, eta)
            den = denoise(x, sigma)
            xe = x + _v(sd - sigma) * ((x - den) / _v(sigma))
            if torch.sum(sd) < 1e-14:
                x = xe
            else:
                t, tn = _nls(sigma), _nls(sd)
                h = tn - t
                s = t + 0.5 * h
                m1, m2, m3, m4 = (_v(m) for m in (_sig(s) / _sig(t), (-0.5 * h).expm1(), _sig(tn) / _sig(t),
                                                  (-h).expm1()))
                x2 = m1 * x - m2 * den
                x = torch.where(_v(sd) > 0.0, m3 * x - m4 * denoise(x2, _sig(s)), xe)
            x = noised(x, nxt, su)
        elif sampler == "DPMPP2MSampler":
            den = denoise(x, sigma)
            t, tn = _nls(sigma), _nls(nxt)
            h = tn - t
            m1, m2 = _v(_sig(tn) / _sig(t)), _v((-h).expm1())
            xs = m1 * x - m2 * den
            if old is None or torch.sum(nxt) < 1e-14:
                x = xs
            else:
                r = (t - _nls(s_in * sig[i - 1])) / h
                dd = _v(1 + 1 / (2 * r)) * den - _v(1 / (2 * r)) * old
                x = torch.where(_v(nxt) > 0.0, m1 * x - m2 * dd, xs)
            old = den
        elif sampler == "LinearMultistepSampler":
            d = (x - denoise(x, sigma)) / _v(sigma)
            ds.append(d)
            if len(ds) > order:
                ds.pop(0)
            cur = min(i + 1, order)
            coeffs = [lms_coeff(cur, sig.numpy(), i, j) for j in range(cur)]
            x = x + sum(cf * dd for cf, dd in zip(coeffs, reversed(ds)))
        else:
            raise ValueError(sampler)
    return x, draws[0]


def apply_plan(plan: dict, network, x0: torch.Tensor, cond: dict, uc: dict, noise: list | None = None):
    """Run a pipeline evaluation plan (ln3diff_b200.pipeline.edm_sampler_plan) in float64 with the
    ln3_sampler_step formula per entry:
        e = k0 x_eval + k1 net_u + k2 net_c
        v = a x + b x_eval + c e + sum_j h_j hist[j] + s noise;   x <- v, next input <- (v, v), hist slot <- e
    around `network(x_in, idx, cond)` (called in fp32 on fp32(x_eval * c_in), as the DiT is).  Returns x (float64)."""
    B = x0.shape[0]
    c_cat = {k: torch.cat((uc[k], cond[k]), 0) for k in cond}
    x = x0.double() * plan["init_scale"]
    xe = x.clone()
    slots = {}
    for ev in plan["evals"]:
        idx = torch.full((2 * B,), ev["t_idx"], dtype=torch.int64)
        xin = torch.cat([xe, xe]) * ev["c_in"]
        net = network(xin.float(), idx, c_cat).double()
        k0, k1, k2, a, b, c, h0, h1, h2, s = ev["coef"][:10]
        e = k0 * xe + k1 * net[:B] + k2 * net[B:]
        v = a * x + b * xe + c * e
        for j, slot in enumerate(ev["hist"]):
            v = v + (h0, h1, h2)[j] * slots[slot]
        if ev["noise"]:
            v = v + s * noise[ev["step"]].double()
        if ev["x_out"]:
            x = v
        if ev["eval_out"]:
            xe = v
        if ev["hist_write"] is not None:
            slots[ev["hist_write"]] = e
    return x
