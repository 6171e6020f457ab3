"""Adaptive Dormand-Prince 5(4) solver: the `sampling_method='dopri5'` default of the reference's
`Sampler.sample_ode` (transport/transport.py:374-421 -> transport/integrators.py:112-119 ->
`torchdiffeq.odeint(fn, x, t, method='dopri5', atol=[1e-6], rtol=[1e-3])`).

torchdiffeq (0.2.3, environment_ln3diff.yml:297) is an un-vendored third-party dependency that is absent from
the image, so this file restates its PUBLISHED algorithm -- "parity unpinned" (SURVEY.md 8c): the accepted-step
sequence is data dependent and there is no copy of torchdiffeq here to pin it against; tests check the
solver against closed-form ODE solutions and its documented controller behaviour.  Restated pieces:
  * Dormand-Prince tableau (alpha, beta, c_sol = last beta row (FSAL), c_error = c_sol - 4th-order weights);
  * initial step selection (Hairer, Norsett, Wanner, "Solving ODEs I", II.4) with order 4;
  * error ratio = rms( err / (atol + rtol * max(|y0|, |y1|)) ), accept iff <= 1;
  * step controller dt' = dt * min(ifactor=10, max(safety=0.9 / ratio^(1/5), dfactor)), dfactor = 0.2 on a rejected
    step and 1 on an accepted one (the step never shrinks after an accept), ratio == 0 -> dt * 10;
  * dense output: quartic fit through (y0, f0, y_mid, y1, f1) with the DPS_C_MID mid-point weights; the outputs at
    the caller's time grid are interpolated, the solver never steps to them exactly.
Time-like quantities are float64 on the host (torchdiffeq keeps them in float64 tensors); the state keeps its dtype.
One error-norm reduction per attempted step is read back by the host (the accept / reject branch is host control
flow in torchdiffeq as well).  Every function evaluation is one `forward_with_cfg` = one CUDA-graph replay.
"""
from __future__ import annotations

import torch as th

_ALPHA = (1 / 5, 3 / 10, 4 / 5, 8 / 9, 1.0, 1.0)
_BETA = ((1 / 5,),
         (3 / 40, 9 / 40),
         (44 / 45, -56 / 15, 32 / 9),
         (19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729),
         (9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656),
         (35 / 384, 0.0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84))
_C_ERROR = (35 / 384 - 1951 / 21600, 0.0, 500 / 1113 - 22642 / 50085, 125 / 192 - 451 / 720,
            -2187 / 6784 - -12231 / 42400, 11 / 84 - 649 / 6300, -1.0 / 60.0)
_C_MID = (6025192743 / 30085553152 / 2, 0.0, 51252292925 / 65400821598 / 2, -2691868925 / 45128329728 / 2,
          187940372067 / 1594534317056 / 2, -1776094331 / 19743644256 / 2, 11237099 / 235043384 / 2)


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


def odeint_dopri5(fn, y0: th.Tensor, t, rtol: float = 1e-3, atol: float = 1e-6, first_step: float | None = None,
                  safety: float = 0.9, ifactor: float = 10.0, dfactor: float = 0.2, max_num_steps: int = 2 ** 31 - 1,
                  stats: dict | None = None) -> th.Tensor:
    """fn(t: float, y) -> dy/dt; `t` an increasing 1-D grid (tensor or sequence); returns the stacked solution
    (len(t), *y0.shape) with solution[0] = y0.  `stats` (optional dict) receives nfe / accepted / rejected."""
    ts = [float(v) for v in (t.tolist() if isinstance(t, th.Tensor) else t)]
    assert all(b > a for a, b in zip(ts, ts[1:])), "t must be strictly increasing"
    nfe = [0]

    def f(tt, yy):
        nfe[0] += 1
        return fn(tt, yy)

    f0 = f(ts[0], y0)
    dt = first_step if first_step is not None else _initial_step(f, ts[0], y0, f0, 4, rtol, atol)
    y, t0, t1 = y0, ts[0], ts[0]
    interp = [y0] * 5
    sol = [y0]
    accepted = rejected = 0
    for t_out in ts[1:]:
        n = 0
        while t_out > t1:
            assert n < max_num_steps, f"max_num_steps exceeded ({n}>={max_num_steps})"
            assert t1 + dt > t1, f"underflow in dt {dt}"
            ks = [f0]
            for alpha, beta in zip(_ALPHA, _BETA):
                yi = _lincomb(y, ks, beta, dt)
                ks.append(f(t1 + alpha * dt, yi))
            y1, f1 = yi, ks[-1]                                     # FSAL: the last stage is the solution
            err = _lincomb(th.zeros_like(y), ks, _C_ERROR, dt)
            tol = atol + rtol * th.max(y.abs(), y1.abs())
            ratio = _rms(err / tol)
            accept = ratio <= 1.0
            if accept:
                y_mid = _lincomb(y, ks, _C_MID, dt)
                a = 2 * dt * (f1 - f0) - 8 * (y1 + y) + 16 * y_mid
                b = dt * (5 * f0 - 3 * f1) + 18 * y + 14 * y1 - 32 * y_mid
                c = dt * (f1 - 4 * f0) - 11 * y - 5 * y1 + 16 * y_mid
                interp = [y, dt * f0, c, b, a]
                t0, t1, y, f0 = t1, t1 + dt, y1, f1
                accepted += 1
            else:
                rejected += 1
            if ratio == 0:
                dt = dt * ifactor
            else:
                df = 1.0 if ratio < 1 else dfactor
                dt = dt * min(ifactor, max(safety / ratio ** 0.2, df))
            n += 1
        sol.append(_interp_eval(interp, t0, t1, t_out))
    if stats is not None:
        stats.update(nfe=nfe[0], accepted=accepted, rejected=rejected)
    return th.stack(sol, 0)


class Dopri5GroupError(RuntimeError):
    """Raised by `odeint_dopri5_grouped` when a group exceeds max_num_steps or its step underflows.  `groups` lists
    the failed groups; `y` and `stats` hold the result of the solve, in which every other group is complete."""

    def __init__(self, msg, groups, y, stats):
        super().__init__(msg)
        self.groups, self.y, self.stats = groups, y, stats


def odeint_dopri5_grouped(fn, y0: th.Tensor, row_group, n_groups: int, t0: float = 0.0, t1: float = 1.0,
                          rtol: float = 1e-3, atol: float = 1e-6, safety: float = 0.9, ifactor: float = 10.0,
                          dfactor: float = 0.2, max_num_steps: int = 2 ** 31 - 1):
    """`odeint_dopri5` for `n_groups` independent problems in one batch, its control logic on the device.

    Row r of y0 (B, ...) fp32 on CUDA belongs to group row_group[r] (int sequence or tensor, every group non-empty).
    Each group follows exactly the steps `odeint_dopri5(fn_g, y0_g, [t0, ..., t1])` takes for its rows alone (the
    interior points of a grid never change the step sequence; only the last is an output): its own error norm, step
    size, accept / reject, counters and end.  fn(t_rows, y) -> dy/dt takes the per-row fp32 time (B,) and returns a
    new (B, ...) tensor; rows of finished groups keep flowing through it with their state frozen, so the batch shape
    never changes.  max_num_steps bounds the attempts of a group from t0 to t1.

    The host enqueues attempt n + 2 only after it has read the status of attempt n (copied to pinned memory behind an
    event), so the GPU never waits on the host and at most one attempt (6 forwards) runs after the last group ends.
    Returns (y(t1) (B, ...), stats) with per-group lists nfe / accepted / rejected and batch_nfe, the forwards the
    batch ran.  Raises Dopri5GroupError naming the groups that failed."""
    from .. import ops
    if not y0.is_cuda:
        raise RuntimeError("odeint_dopri5_grouped runs on CUDA only (no CPU fallback)")
    assert t1 > t0, "t1 must be greater than t0"
    dev, B = y0.device, y0.shape[0]
    y = y0.float().contiguous().clone()
    t_rows = th.full((B,), float(t0), device=dev, dtype=th.float32)
    f0 = fn(t_rows, y).float().contiguous().clone()
    y_stage, out = th.empty_like(y), th.full_like(y, float("nan"))
    state = ops.ode_state(n_groups, t0, dev)
    rg = th.as_tensor(row_group, dtype=th.int32)
    a = ops.ode_args(y, f0, y_stage, t_rows, out, rg, state, t_end=float(t1), rtol=rtol, atol=atol, safety=safety,
                     ifactor=ifactor, dfactor=dfactor, max_num_steps=max_num_steps)
    ops.ode_initial_step(a, 0)
    ops.ode_stage(a, 0)
    ops.ode_initial_step(a, 1, fn(t_rows, y_stage).float().contiguous())
    batch_nfe = 2
    pinned = th.empty((2,) + tuple(state.shape), dtype=th.uint8, pin_memory=True)
    events = [th.cuda.Event(), th.cuda.Event()]
    n = 0
    while True:
        ks = []
        for i in range(1, 7):
            ops.ode_stage(a, i, ks)
            ks.append(fn(t_rows, y_stage).float().contiguous())
        ops.ode_step(a, ks)
        batch_nfe += 6
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
        raise Dopri5GroupError(f"odeint_dopri5_grouped: {msg}", failed, out, stats)
    return out, stats
