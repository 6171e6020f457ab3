"""Adaptive Dormand-Prince 5(4) solver: the `sampling_method='dopri5'` default of the reference's
`Sampler.sample_ode` (transport/transport.py:374-421 -> transport/integrators.py:112-119 ->
`torchdiffeq.odeint(fn, x, t, method='dopri5', atol=[1e-6], rtol=[1e-3])`).

torchdiffeq (0.2.3, environment_ln3diff.yml:297) is an un-vendored third-party dependency that is absent from
the image, so transport/rk.py restates its PUBLISHED algorithm -- "parity unpinned" (SURVEY.md 8c); dopri5 is the
"dopri5" tableau of its explicit Runge-Kutta solvers:
  * Dormand-Prince tableau (alpha, beta, c_sol = last beta row (FSAL), c_error = c_sol - 4th-order weights);
  * initial step selection (Hairer, Norsett, Wanner, "Solving ODEs I", II.4) with order 4;
  * error ratio = rms( err / (atol + rtol * max(|y0|, |y1|)) ), accept iff <= 1;
  * step controller dt' = dt * min(ifactor=10, max(safety=0.9 / ratio^(1/5), dfactor)), dfactor = 0.2 on a rejected
    step and 1 on an accepted one (the step never shrinks after an accept), ratio == 0 -> dt * 10;
  * dense output: quartic fit through (y0, f0, y_mid, y1, f1) with the DPS_C_MID mid-point weights; the outputs at
    the caller's time grid are interpolated, the solver never steps to them exactly.
"""
from __future__ import annotations

import torch as th

from .rk import (TABLEAUS, Dopri5GroupError, _initial_step, _interp_eval, _lincomb, _rms,  # noqa: F401
                 odeint_rk_adaptive, odeint_rk_adaptive_grouped)

_ALPHA = TABLEAUS["dopri5"].alpha
_BETA = TABLEAUS["dopri5"].beta
_C_ERROR = TABLEAUS["dopri5"].c_error
_C_MID = TABLEAUS["dopri5"].mid


def odeint_dopri5(fn, y0: th.Tensor, t, rtol: float = 1e-3, atol: float = 1e-6, first_step: float | None = None,
                  safety: float = 0.9, ifactor: float = 10.0, dfactor: float = 0.2, max_num_steps: int = 2 ** 31 - 1,
                  stats: dict | None = None) -> th.Tensor:
    """fn(t: float, y) -> dy/dt; `t` an increasing 1-D grid (tensor or sequence); returns the stacked solution
    (len(t), *y0.shape) with solution[0] = y0.  `stats` (optional dict) receives nfe / accepted / rejected."""
    return odeint_rk_adaptive(fn, y0, t, "dopri5", rtol=rtol, atol=atol, first_step=first_step, safety=safety,
                              ifactor=ifactor, dfactor=dfactor, max_num_steps=max_num_steps, stats=stats)


def odeint_dopri5_grouped(fn, y0: th.Tensor, row_group, n_groups: int, t0: float = 0.0, t1: float = 1.0,
                          rtol: float = 1e-3, atol: float = 1e-6, safety: float = 0.9, ifactor: float = 10.0,
                          dfactor: float = 0.2, max_num_steps: int = 2 ** 31 - 1):
    """`odeint_dopri5` for `n_groups` independent problems in one batch, its control logic on the device:
    `odeint_rk_adaptive_grouped(method='dopri5')` (see there).  At most one attempt (6 forwards) runs after the last
    group ends.  Returns (y(t1) (B, ...), stats) with per-group lists nfe / accepted / rejected and batch_nfe.
    Raises Dopri5GroupError naming the groups that failed."""
    return odeint_rk_adaptive_grouped(fn, y0, row_group, n_groups, t0, t1, "dopri5", rtol=rtol, atol=atol,
                                      safety=safety, ifactor=ifactor, dfactor=dfactor, max_num_steps=max_num_steps)
