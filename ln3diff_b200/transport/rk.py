"""Explicit Runge-Kutta ODE solvers for `Sampler.sample_ode(sampling_method=...)` (reference transport/transport.py:
374-421 -> transport/integrators.py:101-120 -> `torchdiffeq.odeint(fn, x, t, method=...)`): the adaptive `dopri5`,
`bosh3`, `fehlberg2` and `adaptive_heun`, and the fixed-grid `rk4`.

torchdiffeq (0.2.3, environment_ln3diff.yml:297) is an un-vendored third-party dependency that is absent from the
image, so this file restates its PUBLISHED algorithms -- "parity unpinned" (SURVEY.md 8c): there is no copy of
torchdiffeq here to pin the data-dependent step sequence against; tests check the solvers against closed-form ODE
solutions, their observed orders of convergence and their documented controller behaviour.  Restated pieces
(torchdiffeq rk_common.py, misc.py, dopri5.py, bosh3.py, fehlberg2.py, adaptive_heun.py, fixed_grid.py):
  * the Butcher tableaus (alpha, beta, c_sol, c_error) and dense-output mid weights of TABLEAUS;
  * initial step selection (Hairer, Norsett, Wanner, "Solving ODEs I", II.4) with `order - 1`;
  * error ratio = rms( err / (atol + rtol * max(|y0|, |y1|)) ), accept iff <= 1;
  * step controller dt' = dt * min(ifactor=10, max(safety=0.9 / ratio^(1/order), dfactor)), dfactor = 0.2 on a
    rejected step and 1 on an accepted one (the step never shrinks after an accept), ratio == 0 -> dt * 10;
  * a tableau that is not FSAL (c_sol is not the last beta row with a trailing 0: fehlberg2, adaptive_heun)
    recomputes y1 = y0 + dt (c_sol . k) but keeps f1 = k[-1], the derivative at the last stage's input, which the
    next step reuses as its f0 (torchdiffeq's _runge_kutta_step does exactly this);
  * dense output: quartic fit through (y0, f0, y_mid, y1, f1), y_mid = y0 + dt (mid . k); the outputs at the
    caller's time grid are interpolated, the solver never steps to them exactly;
  * rk4: torchdiffeq's `rk4_alt_step_func` (the 3/8 rule) on the output grid.
Time-like quantities are float64 on the host (torchdiffeq keeps them in float64 tensors); the state keeps its dtype.
One error-norm reduction per attempted step is read back by the host (the accept / reject branch is host control
flow in torchdiffeq as well).  Every function evaluation is one `forward_with_cfg` = one CUDA-graph replay.
"""
from __future__ import annotations

from typing import NamedTuple

import torch as th


class Tableau(NamedTuple):
    """An explicit Runge-Kutta pair: stage i (1-based) evaluates f at t + alpha[i-1] dt and y + dt (beta[i-1] . k),
    k = (f0, k_1, ..); c_sol weighs the solution, c_error the embedded error estimate, mid the dense-output
    mid-point."""
    alpha: tuple
    beta: tuple
    c_sol: tuple
    c_error: tuple
    mid: tuple
    order: int

    @property
    def fsal(self) -> bool:
        """torchdiffeq's test: the last stage's input is the solution (c_sol = last beta row + trailing 0)."""
        return self.c_sol[-1] == 0 and tuple(self.c_sol[:-1]) == tuple(self.beta[-1])


TABLEAUS = {
    # Dormand-Prince 5(4), torchdiffeq dopri5.py (c_error: a 4th-order solution of its own, not scipy RK45's E)
    "dopri5": Tableau(
        alpha=(1 / 5, 3 / 10, 4 / 5, 8 / 9, 1.0, 1.0),
        beta=((1 / 5,),
              (3 / 40, 9 / 40),
              (44 / 45, -56 / 15, 32 / 9),
              (19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729),
              (9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656),
              (35 / 384, 0.0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84)),
        c_sol=(35 / 384, 0.0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84, 0.0),
        c_error=(35 / 384 - 1951 / 21600, 0.0, 500 / 1113 - 22642 / 50085, 125 / 192 - 451 / 720,
                 -2187 / 6784 - -12231 / 42400, 11 / 84 - 649 / 6300, -1.0 / 60.0),
        mid=(6025192743 / 30085553152 / 2, 0.0, 51252292925 / 65400821598 / 2, -2691868925 / 45128329728 / 2,
             187940372067 / 1594534317056 / 2, -1776094331 / 19743644256 / 2, 11237099 / 235043384 / 2),
        order=5),
    # Bogacki-Shampine 3(2), torchdiffeq bosh3.py
    "bosh3": Tableau(
        alpha=(1 / 2, 3 / 4, 1.0),
        beta=((1 / 2,), (0.0, 3 / 4), (2 / 9, 1 / 3, 4 / 9)),
        c_sol=(2 / 9, 1 / 3, 4 / 9, 0.0),
        c_error=(2 / 9 - 7 / 24, 1 / 3 - 1 / 4, 4 / 9 - 1 / 3, -1 / 8),
        mid=(0.0, 0.5, 0.0, 0.0),
        order=3),
    # Runge-Kutta-Fehlberg 2(1), torchdiffeq fehlberg2.py
    "fehlberg2": Tableau(
        alpha=(1 / 2, 1.0),
        beta=((1 / 2,), (1 / 256, 255 / 256)),
        c_sol=(1 / 512, 255 / 256, 1 / 512),
        c_error=(-1 / 512, 0.0, 1 / 512),
        mid=(0.0, 0.5, 0.0),
        order=2),
    # Heun-Euler 2(1), torchdiffeq adaptive_heun.py
    "adaptive_heun": Tableau(
        alpha=(1.0,),
        beta=((1.0,),),
        c_sol=(1 / 2, 1 / 2),
        c_error=(1 / 2, -1 / 2),
        mid=(1 / 2, 0.0),
        order=2),
}
ADAPTIVE_METHODS = tuple(TABLEAUS)
FIXED_GRID_METHODS = ("euler", "midpoint", "heun", "rk4")
FIXED_GRID_FORWARDS = {"euler": 1, "midpoint": 2, "heun": 2, "rk4": 4}   # forwards per grid step
BUILT_METHODS = ADAPTIVE_METHODS + FIXED_GRID_METHODS


def tableau(method: str) -> Tableau:
    """The tableau of an adaptive method; NotImplementedError naming the built methods for any other name."""
    if method not in TABLEAUS:
        raise NotImplementedError(f"sampling_method={method!r} is not built (it needs torchdiffeq, an un-vendored "
                                  f"dependency of the reference); built: {', '.join(BUILT_METHODS)}")
    return TABLEAUS[method]


def _rms(t: th.Tensor) -> float:
    return float(t.float().pow(2).mean().sqrt())


def _lincomb(y0, ks, coefs, dt):
    out = y0
    for k, c in zip(ks, coefs):
        if c != 0.0:
            out = out + k * (c * dt)
    return out


def _initial_step(fn, t0, y0, f0, order, rtol, atol):
    scale = atol + y0.abs() * rtol
    d0, d1 = _rms(y0 / scale), _rms(f0 / scale)
    h0 = 1e-6 if (d0 < 1e-5 or d1 < 1e-5) else 0.01 * d0 / d1
    f1 = fn(t0 + h0, y0 + h0 * f0)
    d2 = _rms((f1 - f0) / scale) / h0
    if d1 <= 1e-15 and d2 <= 1e-15:
        h1 = max(1e-6, h0 * 1e-3)
    else:
        h1 = (0.01 / max(d1, d2)) ** (1.0 / float(order + 1))
    return min(100 * h0, h1)


def _interp_eval(coef, t0, t1, t):
    x = (t - t0) / (t1 - t0)
    total = coef[0] + x * coef[1]
    xp = x
    for c in coef[2:]:
        xp = xp * x
        total = total + xp * c
    return total


def _next_dt(dt, ratio, order, safety, ifactor, dfactor):
    """torchdiffeq's _optimal_step_size."""
    if ratio == 0:
        return dt * ifactor
    df = 1.0 if ratio < 1 else dfactor
    return dt * min(ifactor, max(safety / ratio ** (1.0 / order), df))


def rk_attempt(f, tab: Tableau, t, y, f0, dt, rtol, atol):
    """One attempted step from (t, y) with derivative f0: (y1, f1, ks, error ratio)."""
    ks = [f0]
    for alpha, beta in zip(tab.alpha, tab.beta):
        yi = _lincomb(y, ks, beta, dt)
        ks.append(f(t + alpha * dt, yi))
    # FSAL: the last stage's input is the solution; otherwise it is recomputed, and f1 stays k[-1] either way
    y1 = yi if tab.fsal else _lincomb(y, ks, tab.c_sol, dt)
    err = _lincomb(th.zeros_like(y), ks, tab.c_error, dt)
    tol = atol + rtol * th.max(y.abs(), y1.abs())
    return y1, ks[-1], ks, _rms(err / tol)


def odeint_rk_adaptive(fn, y0: th.Tensor, t, method: str = "dopri5", rtol: float = 1e-3, atol: float = 1e-6,
                       first_step: float | None = None, safety: float = 0.9, ifactor: float = 10.0,
                       dfactor: float = 0.2, max_num_steps: int = 2 ** 31 - 1, stats: dict | None = None) -> th.Tensor:
    """torchdiffeq's adaptive `method` (one of ADAPTIVE_METHODS).  fn(t: float, y) -> dy/dt; `t` an increasing 1-D
    grid (tensor or sequence); returns the stacked solution (len(t), *y0.shape) with solution[0] = y0.  `stats`
    (optional dict) receives nfe / accepted / rejected."""
    tab = tableau(method)
    ts = [float(v) for v in (t.tolist() if isinstance(t, th.Tensor) else t)]
    assert all(b > a for a, b in zip(ts, ts[1:])), "t must be strictly increasing"
    nfe = [0]

    def f(tt, yy):
        nfe[0] += 1
        return fn(tt, yy)

    f0 = f(ts[0], y0)
    dt = first_step if first_step is not None else _initial_step(f, ts[0], y0, f0, tab.order - 1, rtol, atol)
    y, t0, t1 = y0, ts[0], ts[0]
    interp = [y0] * 5
    sol = [y0]
    accepted = rejected = 0
    for t_out in ts[1:]:
        n = 0
        while t_out > t1:
            assert n < max_num_steps, f"max_num_steps exceeded ({n}>={max_num_steps})"
            assert t1 + dt > t1, f"underflow in dt {dt}"
            y1, f1, ks, ratio = rk_attempt(f, tab, t1, y, f0, dt, rtol, atol)
            if ratio <= 1.0:
                y_mid = _lincomb(y, ks, tab.mid, dt)
                a = 2 * dt * (f1 - f0) - 8 * (y1 + y) + 16 * y_mid
                b = dt * (5 * f0 - 3 * f1) + 18 * y + 14 * y1 - 32 * y_mid
                c = dt * (f1 - 4 * f0) - 11 * y - 5 * y1 + 16 * y_mid
                interp = [y, dt * f0, c, b, a]
                t0, t1, y, f0 = t1, t1 + dt, y1, f1
                accepted += 1
            else:
                rejected += 1
            dt = _next_dt(dt, ratio, tab.order, safety, ifactor, dfactor)
            n += 1
        sol.append(_interp_eval(interp, t0, t1, t_out))
    if stats is not None:
        stats.update(nfe=nfe[0], accepted=accepted, rejected=rejected)
    return th.stack(sol, 0)


class RKGroupError(RuntimeError):
    """Raised by `odeint_rk_adaptive_grouped` when a group exceeds max_num_steps or its step underflows.  `groups`
    lists the failed groups; `y` and `stats` hold the result of the solve, in which every other group is complete."""

    def __init__(self, msg, groups, y, stats):
        super().__init__(msg)
        self.groups, self.y, self.stats = groups, y, stats


class Dopri5GroupError(RKGroupError):
    """RKGroupError of a dopri5 solve."""


def odeint_rk_adaptive_grouped(fn, y0: th.Tensor, row_group, n_groups: int, t0: float = 0.0, t1: float = 1.0,
                               method: str = "dopri5", rtol: float = 1e-3, atol: float = 1e-6, safety: float = 0.9,
                               ifactor: float = 10.0, dfactor: float = 0.2, max_num_steps: int = 2 ** 31 - 1):
    """`odeint_rk_adaptive(method=...)` for `n_groups` independent problems in one batch, its control logic on the
    device (ln3_ode_rk_*).

    Row r of y0 (B, ...) fp32 on CUDA belongs to group row_group[r] (int sequence or tensor, every group non-empty).
    Each group follows exactly the steps `odeint_rk_adaptive(fn_g, y0_g, [t0, ..., t1], method)` takes for its rows
    alone (the interior points of a grid never change the step sequence; only the last is an output): its own error
    norm, step size, accept / reject, counters and end.  fn(t_rows, y) -> dy/dt takes the per-row fp32 time (B,) and
    returns a new (B, ...) tensor; rows of finished groups keep flowing through it with their state frozen, so the
    batch shape never changes.  max_num_steps bounds the attempts of a group from t0 to t1.

    The host enqueues attempt n + 2 only after it has read the status of attempt n (copied to pinned memory behind an
    event), so the GPU never waits on the host and at most one attempt (S forwards, S the method's stage count) runs
    after the last group ends.  Returns (y(t1) (B, ...), stats) with per-group lists nfe / accepted / rejected and
    batch_nfe, the forwards the batch ran.  Raises RKGroupError (Dopri5GroupError for dopri5) naming the groups
    that failed."""
    from .. import _lib, ops
    tableau(method)
    m = _lib.ODE_METHODS[method]
    name = "odeint_dopri5_grouped" if method == "dopri5" else f"odeint_rk_adaptive_grouped({method!r})"
    if not y0.is_cuda:
        raise RuntimeError(f"{name} runs on CUDA only (no CPU fallback)")
    assert t1 > t0, "t1 must be greater than t0"
    S = ops.ode_stages(m)
    dev, B = y0.device, y0.shape[0]
    y = y0.float().contiguous().clone()
    t_rows = th.full((B,), float(t0), device=dev, dtype=th.float32)
    f0 = fn(t_rows, y).float().contiguous().clone()
    y_stage, out = th.empty_like(y), th.full_like(y, float("nan"))
    state = ops.ode_state(n_groups, t0, dev)
    rg = th.as_tensor(row_group, dtype=th.int32)
    a = ops.ode_args(y, f0, y_stage, t_rows, out, rg, state, t_end=float(t1), rtol=rtol, atol=atol, safety=safety,
                     ifactor=ifactor, dfactor=dfactor, max_num_steps=max_num_steps)
    ops.ode_initial_step(a, 0, method=m)
    ops.ode_stage(a, 0, method=m)
    ops.ode_initial_step(a, 1, fn(t_rows, y_stage).float().contiguous(), method=m)
    batch_nfe = 2
    pinned = th.empty((2,) + tuple(state.shape), dtype=th.uint8, pin_memory=True)
    events = [th.cuda.Event(), th.cuda.Event()]
    n = 0
    while True:
        ks = []
        for i in range(1, S + 1):
            ops.ode_stage(a, i, ks, method=m)
            ks.append(fn(t_rows, y_stage).float().contiguous())
        ops.ode_step(a, ks, method=m)
        batch_nfe += S
        pinned[n % 2].copy_(state, non_blocking=True)
        events[n % 2].record()
        if n >= 1:                        # attempt n is in flight while the host reads attempt n - 1
            events[(n - 1) % 2].synchronize()
            if not bool((ops.ode_state_fields(pinned[(n - 1) % 2])["status"] == 0).any()):
                break
        n += 1
    events[n % 2].synchronize()
    f = ops.ode_state_fields(pinned[n % 2])
    stats = dict(nfe=f["nfe"].tolist(), accepted=f["accepted"].tolist(), rejected=f["rejected"].tolist(),
                 batch_nfe=batch_nfe)
    failed = [g for g, s in enumerate(f["status"].tolist()) if s < 0]
    if failed:
        why = {-1: "max_num_steps exceeded", -2: "underflow in dt"}
        msg = "; ".join(f"group {g}: {why[int(f['status'][g])]} (t={float(f['t'][g])}, dt={float(f['dt'][g])})"
                        for g in failed)
        error = Dopri5GroupError if method == "dopri5" else RKGroupError
        raise error(f"{name}: {msg}", failed, out, stats)
    return out, stats


# ---------------------------------------------------------------------------------------------- fixed grid rk4
_ONE_THIRD, _TWO_THIRDS = 1 / 3, 2 / 3


def rk4_alt_step(fn, t0, dt, t1, y0, k1=None):
    """torchdiffeq's rk4_alt_step_func (the 3/8 rule), in its tensor arithmetic: returns y0 + dy.  t0, dt, t1 are
    the grid's float32 0-dim tensors; fn(t, y) -> dy/dt; `k1`: f(t0, y0) when the caller already has it."""
    if k1 is None:
        k1 = fn(t0, y0)
    k2 = fn(t0 + dt * _ONE_THIRD, y0 + dt * k1 * _ONE_THIRD)
    k3 = fn(t0 + dt * _TWO_THIRDS, y0 + dt * (k2 - k1 * _ONE_THIRD))
    k4 = fn(t1, y0 + dt * (k1 - k2 + k3))
    return y0 + (k1 + 3 * (k2 + k3) + k4) * dt * 0.125


def odeint_rk4(fn, y0: th.Tensor, t) -> th.Tensor:
    """torchdiffeq's fixed-grid `rk4` on the output grid `t` (a 1-D tensor: sample_ode passes its float32 grid; a
    sequence becomes float64): one rk4_alt_step per interval, 4 forwards each, fn(t: 0-dim tensor, y).  Returns the
    stacked solution (len(t), *y0.shape)."""
    t = t if isinstance(t, th.Tensor) else th.tensor(t, dtype=th.float64)
    ys = [y0]
    for i in range(len(t) - 1):
        ys.append(rk4_alt_step(fn, t[i], t[i + 1] - t[i], t[i + 1], ys[-1]))
    return th.stack(ys, 0)
