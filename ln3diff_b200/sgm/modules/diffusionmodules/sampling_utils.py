"""Mirror of reference sgm/modules/diffusionmodules/sampling_utils.py:7-43 (host-side scalar helpers of the sgm
samplers; no kernel).

`linear_multistep_coeff` integrates the Lagrange basis polynomial exactly in float64 (numpy.polynomial) where the
reference calls `scipy.integrate.quad(fn, t[i], t[i+1], epsrel=epsrel)`: the integrand is a polynomial of degree
order - 1 <= 3, so the closed form is what the quadrature approximates, and the package needs no scipy.  `epsrel` is
kept for the reference's signature and unused.
"""
import numpy as np
import torch
from numpy.polynomial import polynomial as P

from ...util import append_dims


def linear_multistep_coeff(order, t, i, j, epsrel=1e-4):
    if order - 1 > i:
        raise ValueError(f"Order {order} too high for step {i}")
    tt = np.asarray(t, dtype=np.float64)
    poly = np.array([1.0])
    for k in range(order):
        if j == k:
            continue
        poly = P.polymul(poly, np.array([-tt[i - k], 1.0]) / (tt[i - j] - tt[i - k]))
    prim = P.polyint(poly)
    return float(P.polyval(tt[i + 1], prim) - P.polyval(tt[i], prim))


def get_ancestral_step(sigma_from, sigma_to, eta=1.0):
    if not eta:
        return sigma_to, 0.0
    sigma_up = torch.minimum(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
    return sigma_down, sigma_up


def to_d(x, sigma, denoised):
    return (x - denoised) / append_dims(sigma, x.ndim)


def to_neg_log_sigma(sigma):
    return sigma.log().neg()


def to_sigma(neg_log_sigma):
    return neg_log_sigma.neg().exp()
