import enum

import numpy as np
import torch as th

from .. import ops


class ModelType(enum.Enum):
    NOISE = enum.auto()
    SCORE = enum.auto()
    VELOCITY = enum.auto()


class PathType(enum.Enum):
    LINEAR = enum.auto()
    GVP = enum.auto()
    VP = enum.auto()


class WeightType(enum.Enum):
    NONE = enum.auto()
    VELOCITY = enum.auto()
    LIKELIHOOD = enum.auto()


class SNRType(enum.Enum):
    UNIFORM = enum.auto()
    LOGNORM = enum.auto()


class Transport:
    """reference transport/transport.py:48-72: only the Linear path with velocity prediction (the
    I23D release configuration, nsr/lsgm/flow_matching_trainer.py:160-192) is on the hot path."""

    def __init__(self, *, model_type, path_type, loss_type, train_eps, sample_eps, snr_type):
        if path_type != PathType.LINEAR or model_type != ModelType.VELOCITY:
            raise NotImplementedError("ln3diff_b200 implements the Linear path / velocity prediction")
        self.loss_type, self.model_type, self.path_type = loss_type, model_type, path_type
        self.train_eps, self.sample_eps, self.snr_type = train_eps, sample_eps, snr_type
        assert self.snr_type == SNRType.LOGNORM, "use lognorm schedule plz."

    def check_interval(self, train_eps, sample_eps, *, diffusion_form="SBDM", sde=False, reverse=False,
                       eval=False, last_step_size=0.0):
        t0, t1 = 0, 1  # velocity & Linear ODE: stable everywhere (transport.py:85-112)
        if sde:          # the first step is semi-implicit: SBDM starts at eps, and t1 leaves room for the last step
            eps = train_eps if not eval else sample_eps
            t0 = eps if diffusion_form == "SBDM" else 0
            t1 = 1 - eps if last_step_size == 0 else 1 - last_step_size
        return (1 - t0, 1 - t1) if reverse else (t0, t1)

    def get_drift(self):
        def velocity_ode(x, t, model, **model_kwargs):
            out = model(x, t, **model_kwargs)
            assert out.shape == x.shape, "Output shape from ODE solver must match input shape"
            return out
        return velocity_ode

    def get_score(self):
        """reference transport.py:231-245 for velocity prediction: path.py get_score_from_velocity."""
        return lambda x, t, model, **kw: score_from_velocity(model(x, t, **kw), x, t)


def create_transport(path_type="Linear", prediction="velocity", loss_weight=None, train_eps=None,
                     sample_eps=None, snr_type="uniform"):
    """reference transport/__init__.py:3-72."""
    model_type = {"noise": ModelType.NOISE, "score": ModelType.SCORE}.get(prediction, ModelType.VELOCITY)
    loss_type = {"velocity": WeightType.VELOCITY, "likelihood": WeightType.LIKELIHOOD}.get(loss_weight, WeightType.NONE)
    if snr_type == "lognorm":
        snr = SNRType.LOGNORM
    elif snr_type == "uniform":
        snr = SNRType.UNIFORM
    else:
        raise ValueError(f"Invalid snr type {snr_type}")
    ptype = {"Linear": PathType.LINEAR, "GVP": PathType.GVP, "VP": PathType.VP}[path_type]
    return Transport(model_type=model_type, path_type=ptype, loss_type=loss_type, train_eps=0, sample_eps=0,
                     snr_type=snr)


class ode:
    """reference transport/integrators.py:78-120 with the fixed-grid solvers of torchdiffeq."""

    def __init__(self, drift, *, t0, t1, sampler_type, num_steps, atol, rtol):
        assert t0 < t1, "ODE sampler has to be in forward time"
        self.drift = drift
        self.t = th.linspace(t0, t1, num_steps)
        self.atol, self.rtol, self.sampler_type = atol, rtol, sampler_type

    def _axpy(self, x, dt, k, coef=None):
        """x + dt * k as one fused launch on CUDA (`coef`: the step's device-resident (B, 4) row block)."""
        if coef is not None:
            return ops.sampler_affine_update(x.contiguous(), coef, k.float().contiguous())
        return x + dt * k

    def sample(self, x, model, **model_kwargs):
        device = x.device
        B = x.size(0)

        def _fn(t, x):
            # `th.ones(B).to(device) * t` of the reference (integrators.py:104-107) without the H2D copy / sync
            tt = th.full((B,), float(t), device=device, dtype=th.float32)
            return self.drift(x, tt, model, **model_kwargs)

        t = self.t                                                 # float32 grid, kept on the HOST
        if self.sampler_type in ("euler", "heun", "midpoint"):
            n = len(t) - 1
            dts = t[1:] - t[:-1]                                   # float32 arithmetic as the reference's tensors
            halves = 0.5 * dts
            fused = x.is_cuda and x.dtype == th.float32
            tab = None
            if fused:   # every step's update coefficients in one upload: [:, 0] = dt, [:, 1] = dt / 2
                tab = th.zeros(n, 2, B, 4)
                tab[..., 0] = 1.0
                tab[:, 0, :, 1] = dts[:, None]
                tab[:, 1, :, 1] = halves[:, None]
                tab = tab.to(device)
            ys = [x]
            for i in range(n):
                t0, t1, dt, half = t[i], t[i + 1], dts[i], halves[i]
                cf = tab[i, 0] if fused else None
                ch = tab[i, 1] if fused else None
                y = ys[-1]
                if self.sampler_type == "euler":
                    y = self._axpy(y, dt, _fn(t0, y), cf)
                elif self.sampler_type == "midpoint":
                    y = self._axpy(y, dt, _fn(t0 + half, self._axpy(y, half, _fn(t0, y), ch)), cf)
                else:
                    k1 = _fn(t0, y)
                    k2 = _fn(t1, self._axpy(y, dt, k1, cf))
                    y = self._axpy(self._axpy(y, half, k1, ch), half, k2, ch)
                ys.append(y)
            return th.stack(ys, 0)
        if self.sampler_type == "rk4":
            return self._rk4(x, _fn, B, device)
        try:
            from torchdiffeq import odeint  # the reference's own third-party solver, when it is installed
        except ImportError:
            odeint = None
        if odeint is not None:
            return odeint(_fn, x, t.to(device), method=self.sampler_type, atol=[self.atol], rtol=[self.rtol])
        if self.sampler_type == "dopri5":
            # the shipped I23D default (transport.py:374-381): restated solver, see transport/dopri5.py
            from .dopri5 import odeint_dopri5
            self.last_stats = {}
            return odeint_dopri5(_fn, x, t, rtol=self.rtol, atol=self.atol, stats=self.last_stats)
        from .rk import odeint_rk_adaptive, tableau
        tableau(self.sampler_type)     # NotImplementedError naming the built methods for any other name
        self.last_stats = {}           # bosh3 / fehlberg2 / adaptive_heun: restated solvers, see transport/rk.py
        return odeint_rk_adaptive(_fn, x, t, self.sampler_type, rtol=self.rtol, atol=self.atol,
                                  stats=self.last_stats)

    def _rk4(self, x, _fn, B, device):
        """torchdiffeq's fixed-grid rk4 (rk4_alt_step_func, the 3/8 rule) on the output grid.  CUDA fp32 states take
        each stage input and the update through ln3_sampler_affine_update (five launches per step, coefficients
        uploaded once); any other state runs transport/rk.py:odeint_rk4's tensor arithmetic."""
        from .rk import _ONE_THIRD, _TWO_THIRDS, odeint_rk4
        t = self.t
        if not (x.is_cuda and x.dtype == th.float32):
            return odeint_rk4(_fn, x, t)
        n = len(t) - 1
        dts = t[1:] - t[:-1]
        third, eighth = dts * _ONE_THIRD, dts * 0.125
        # per step (x, m0, m1, noise) weights of: y + dt/3 k1 | y + dt k2 - dt/3 k1 | y + dt k1 - dt k2 + dt k3 |
        # acc = y + dt/8 k1 + 3dt/8 k2 + 3dt/8 k3 | acc + dt/8 k4
        w = th.zeros(n, 5, 4)
        w[:, :, 0] = 1.0
        w[:, 0, 1] = third
        w[:, 1, 1], w[:, 1, 2] = dts, -third
        w[:, 2, 1], w[:, 2, 2], w[:, 2, 3] = dts, -dts, dts
        w[:, 3, 1], w[:, 3, 2], w[:, 3, 3] = eighth, 3 * eighth, 3 * eighth
        w[:, 4, 1] = eighth
        tab = w[:, :, None, :].expand(n, 5, B, 4).contiguous().to(device)
        upd = ops.sampler_affine_update
        ys = [x]
        for i in range(n):
            t0, dt, c = t[i], dts[i], tab[i]
            y = ys[-1].contiguous()
            k1 = _fn(t0, y).float().contiguous()
            k2 = _fn(t0 + dt * _ONE_THIRD, upd(y, c[0], k1)).float().contiguous()
            k3 = _fn(t0 + dt * _TWO_THIRDS, upd(y, c[1], k2, k1)).float().contiguous()
            k4 = _fn(t[i + 1], upd(y, c[2], k1, k2, k3)).float().contiguous()
            ys.append(upd(upd(y, c[3], k1, k2, k3), c[4], k4))
        return th.stack(ys, 0)


class Sampler:
    """reference transport/transport.py:246-259,374-421."""

    def __init__(self, transport):
        self.transport = transport
        self.drift = self.transport.get_drift()

    def sample_ode(self, *, sampling_method="dopri5", num_steps=50, atol=1e-6, rtol=1e-3, reverse=False,
                   cfg=False):
        if reverse:
            drift = lambda x, t, model, **kw: self.drift(x, th.ones_like(t) * (1 - t), model, **kw)
        else:
            drift = self.drift
        t0, t1 = self.transport.check_interval(self.transport.train_eps, self.transport.sample_eps, sde=False,
                                               eval=True, reverse=reverse, last_step_size=0.0)
        return ode(drift=drift, t0=t0, t1=t1, sampler_type=sampling_method, num_steps=num_steps, atol=atol,
                   rtol=rtol).sample

    def sample_sde(self, *, sampling_method="Euler", diffusion_form="SBDM", diffusion_norm=1.0, last_step="Mean",
                   last_step_size=0.04, num_steps=250):
        """reference transport.py:313-372: returns `_sample(init, model, **model_kwargs)`, the list of `num_steps`
        states of the Euler-Maruyama or Heun SDE solver, the last one from `last_step`.  Every noise draw is the
        reference's `randn(x.size())` on the global CPU generator.

        With `init` CUDA fp32 and `model` a library denoiser's bound `forward_with_cfg`, each drift evaluation is one
        forward of the 2N-row CFG batch (a replay of the denoiser's CUDA graph) and one ln3_flow_sde_step; the
        reference runs the model twice per SDE drift.  Any other model runs the reference's torch arithmetic.

        Raises what the reference raises for an unknown method, diffusion form or last step, NotImplementedError for
        the `constant` form (the reference cannot run it either: it takes the square root of a Python float), and
        ValueError where the reference returns NaN: `SBDM` (its diffusion is infinite at t0 = 0 on this transport)
        and `Heun` with `last_step=None` (its last stage evaluates the score at t = 1, where the variance is 0)."""
        if last_step is None:
            last_step_size = 0.0
        plan = sde_plan(sampling_method, diffusion_form, diffusion_norm, last_step, last_step_size, num_steps,
                        self.transport)
        _sde = sde(plan, self.transport)

        def _sample(init, model, **model_kwargs):
            if init.is_cuda and init.dtype == th.float32 and _is_library_cfg(model):
                xs = []
                sde_fused(plan, model.__self__, init, model_kwargs["context"], model_kwargs["cfg_scale"],
                          lambda k: th.randn(init.size()).to(init), record=xs.append)
            else:
                xs = _sde.sample(init, model, **model_kwargs)
                ts = th.ones(init.size(0), device=init.device) * plan["t1"]
                xs.append(_sde.last_step(xs[-1], ts, model, **model_kwargs))
            assert len(xs) == num_steps, "Samples does not match the number of steps"
            return xs
        return _sample


# ---------------------------------------------------------------------------------------------- SDE sampling
# The Linear path (alpha_t = t, sigma_t = 1 - t) with velocity prediction: reference path.py:18-110,
# integrators.py:9-75, transport.py:260-372.
DIFFUSION_FORMS = ("constant", "SBDM", "sigma", "linear", "decreasing", "inccreasing-decreasing")  # sic, path.py:56
SDE_METHODS = ("Euler", "Heun")
LAST_STEPS = (None, "Mean", "Tweedie", "Euler")


def _expand(t, x):
    return t.view(t.size(0), *([1] * (x.dim() - 1)))


def score_from_velocity(v, x, t):
    """path.py:67-82 (ICPlan): (t v - x) / var, var = sigma_t^2 - t * d_sigma_t * sigma_t, in the reference's order."""
    t = _expand(t, x)
    sigma_t = 1 - t
    var = sigma_t ** 2 - t * -1 * sigma_t
    return (t * v - x) / var


def diffusion_coefficient(t, form, norm):
    """path.py:45-65 (ICPlan.compute_diffusion) for one form; `t` is a float32 tensor."""
    if form not in DIFFUSION_FORMS:
        raise NotImplementedError(f"Diffusion form {form} not implemented")
    if form == "constant":
        raise NotImplementedError("diffusion_form='constant' is not supported: the reference returns a Python float "
                                  "there and its th.sqrt(2 * diffusion) raises TypeError")
    if form == "SBDM":
        sigma_t = 1 - t
        return norm * ((1 / t) * (sigma_t ** 2) - sigma_t * -1)
    if form in ("sigma", "linear"):
        return norm * (1 - t)
    if form == "decreasing":
        return 0.25 * (norm * th.cos(np.pi * t) + 1) ** 2
    return norm * th.sin(np.pi * t) ** 2


class sde:
    """reference integrators.py:9-75 and transport.py:260-311 in torch arithmetic (two model calls per SDE drift)."""

    def __init__(self, plan, transport):
        self.plan, self.t, self.dt = plan, plan["grid"], plan["dt"]
        form, norm = plan["diffusion_form"], plan["diffusion_norm"]
        self.diffusion = lambda x, t: diffusion_coefficient(_expand(t, x), form, norm)
        self.drift = transport.get_drift()
        self.score = transport.get_score()

    def sde_drift(self, x, t, model, **kw):
        return self.drift(x, t, model, **kw) + self.diffusion(x, t) * self.score(x, t, model, **kw)

    def _euler(self, x, t, model, **kw):
        w_cur = th.randn(x.size()).to(x)
        t = th.ones(x.size(0)).to(x) * t
        dw = w_cur * th.sqrt(self.dt)
        drift = self.sde_drift(x, t, model, **kw)
        diffusion = self.diffusion(x, t)
        mean_x = x + drift * self.dt
        return mean_x + th.sqrt(2 * diffusion) * dw

    def _heun(self, x, t, model, **kw):
        w_cur = th.randn(x.size()).to(x)
        dw = w_cur * th.sqrt(self.dt)
        t_cur = th.ones(x.size(0)).to(x) * t
        diffusion = self.diffusion(x, t_cur)
        xhat = x + th.sqrt(2 * diffusion) * dw
        K1 = self.sde_drift(xhat, t_cur, model, **kw)
        xp = xhat + self.dt * K1
        K2 = self.sde_drift(xp, t_cur + self.dt, model, **kw)
        return xhat + 0.5 * self.dt * (K1 + K2)   # the last point is not skipped (integrators.py:49)

    def sample(self, init, model, **kw):
        step = self._euler if self.plan["sampling_method"] == "Euler" else self._heun
        x, samples = init, []
        with th.no_grad():
            for ti in self.t[:-1]:
                x = step(x, ti, model, **kw)
                samples.append(x)
        return samples

    def last_step(self, x, t, model, **kw):
        kind, size = self.plan["last_step"], self.plan["last_step_size"]
        if kind is None:
            return x
        if kind == "Mean":
            return x + self.sde_drift(x, t, model, **kw) * size
        if kind == "Euler":
            return x + self.drift(x, t, model, **kw) * size
        alpha, sigma = t[0], 1 - t[0]                  # Tweedie: x / alpha + sigma^2 / alpha * score
        return x / alpha + (sigma ** 2) / alpha * self.score(x, t, model, **kw)


def sde_plan(sampling_method, diffusion_form, diffusion_norm, last_step, last_step_size, num_steps, transport=None):
    """The drift evaluations of one `sample_sde` run as ln3_flow_sde_step arguments, computed on the host in the
    reference's float32 arithmetic.  Every entry: the forward time `t` and the kernel's `var`, `diffusion`, `mode`,
    output coefficients `cx` / `cy` (a, b, c, h, sigma; None: not written), whether it reads the state `x_in` and the
    history `hist_in`, writes the history `hist_out`, which step's noise it reads (`noise`, or None) and whether its
    x_out is one of the returned states (`record`).  `pre_sigma`: Heun's first xhat = init + pre_sigma * w_0, before
    the first forward.  Euler-Maruyama keeps the state in the forward input; Heun keeps xhat in the state."""
    from .. import ops
    if sampling_method not in SDE_METHODS:
        raise NotImplementedError("Smapler type not implemented.")   # integrators.py:61 (sic)
    if last_step not in LAST_STEPS:
        raise NotImplementedError(f"last_step={last_step!r}: expected one of {LAST_STEPS}")
    if num_steps < 2:
        raise ValueError("sample_sde needs num_steps >= 2 (its step size is t[1] - t[0])")
    if last_step is None:
        last_step_size = 0.0
    if diffusion_form == "SBDM":
        raise ValueError("diffusion_form='SBDM' is non-finite on this transport: sample_eps = 0 puts the first step at "
                         "t = 0, where the SBDM diffusion is infinite; use 'sigma' (the command-line default), "
                         "'linear', 'decreasing' or 'inccreasing-decreasing'")
    if sampling_method == "Heun" and last_step is None:
        raise ValueError("sampling_method='Heun' with last_step=None is non-finite: the grid then ends at t1 = 1 and "
                         "Heun's last stage evaluates the score where its variance is 0; choose a last step")
    transport = transport or create_transport(snr_type="lognorm")
    t0, t1 = transport.check_interval(transport.train_eps, transport.sample_eps, diffusion_form=diffusion_form,
                                      sde=True, eval=True, reverse=False, last_step_size=last_step_size)
    grid = th.linspace(t0, t1, num_steps)
    dt = grid[1] - grid[0]
    sdt = th.sqrt(dt)
    half = 0.5 * dt

    def at(t):   # t: float32 0-dim tensor -> (t, var, D) as the kernel takes them
        tt = t.reshape(1)
        sigma_t = 1 - tt
        var = sigma_t ** 2 - tt * -1 * sigma_t
        return dict(t=float(tt), var=float(var), diffusion=float(diffusion_coefficient(tt, diffusion_form,
                                                                                      diffusion_norm)))

    def noise_scale(t):   # sqrt(2 D(t)) * sqrt(dt)
        return float(th.sqrt(2 * diffusion_coefficient(t.reshape(1), diffusion_form, diffusion_norm)) * sdt)

    evals = []

    def ev(t, mode, cx, cy=None, *, x_in=False, hist_in=False, hist_out=False, noise=None, record=False):
        evals.append(dict(at(t), mode=mode, cx=tuple(float(c) for c in cx),
                          cy=None if cy is None else tuple(float(c) for c in cy), x_in=x_in, hist_in=hist_in,
                          hist_out=hist_out, noise=noise, record=record))

    S, D, dtf, hf = num_steps - 1, ops.SDE_DRIFT, float(dt), float(half)
    for i in range(S):
        if sampling_method == "Euler":               # x <- x + dt (v + D sc) + sqrt(2D) sqrt(dt) w_i
            c = (0.0, 1.0, dtf, 0.0, noise_scale(grid[i]))
            ev(grid[i], D, c, c, noise=i, record=True)
        else:
            # stage 1 at xhat: K1 -> hist, xhat -> state, xp = xhat + dt K1 -> next input
            ev(grid[i], D, (0.0, 1.0, 0.0, 0.0, 0.0), (0.0, 1.0, dtf, 0.0, 0.0), hist_out=True)
            # stage 2 at xp, t + dt in float32: x = xhat + dt/2 (K1 + K2); the next input is the next step's xhat
            nxt = i + 1 < S
            cy = (1.0, 0.0, hf, hf, noise_scale(grid[i + 1]) if nxt else 0.0)
            ev(grid[i] + dt, D, (1.0, 0.0, hf, hf, 0.0), cy, x_in=True, hist_in=True, noise=i + 1 if nxt else None,
               record=True)
    t_last = th.ones(1) * t1
    size = float(th.ones(1) * last_step_size)
    if last_step == "Mean":
        ev(t_last, D, (0.0, 1.0, size, 0.0, 0.0), record=True)
    elif last_step == "Euler":
        ev(t_last, ops.SDE_VELOCITY, (0.0, 1.0, size, 0.0, 0.0), record=True)
    elif last_step == "Tweedie":
        alpha, sigma = t_last, 1 - t_last
        ev(t_last, ops.SDE_SCORE, (0.0, 1 / alpha, (sigma ** 2) / alpha, 0.0, 0.0), record=True)
    return dict(sampling_method=sampling_method, diffusion_form=diffusion_form, diffusion_norm=diffusion_norm,
                last_step=last_step, last_step_size=last_step_size, num_steps=num_steps, t0=t0, t1=t1, grid=grid,
                dt=dt, evals=evals, pre_sigma=noise_scale(grid[0]) if sampling_method == "Heun" else None,
                forwards=len(evals))


def _is_library_cfg(model) -> bool:
    """`model` is a library denoiser's bound forward_with_cfg (the fused path's precondition)."""
    from ..dit._denoiser import DenoiserMixin
    owner = getattr(model, "__self__", None)
    return isinstance(owner, DenoiserMixin) and getattr(model, "__func__", None) is type(owner).forward_with_cfg


def sde_fused(plan, den, init, context, cfg_scale, draw, record=None):
    """Run `plan` (sde_plan) on the CUDA fp32 2R-row CFG state `init` around denoiser `den`: one forward (the
    denoiser's `step_forward`, conditional rows first) and one ln3_flow_sde_step per entry.  `draw(k)` returns step k's
    noise, a CUDA fp32 (2N, ...) draw (N divides R), and is called once per step in step order; `record(x)` receives
    every returned state as a new tensor (and, with last_step=None, the last one again).  Returns the final state
    buffer (2R rows)."""
    from .. import ops
    rows = init.shape[0]
    t_rows = th.tensor([e["t"] for e in plan["evals"]], dtype=th.float32)[:, None].repeat(1, rows).to(init.device)
    fw = den.step_forward(rows, context, t_rows)
    state = th.empty_like(fw.x)
    hist = th.empty_like(fw.x) if plan["sampling_method"] == "Heun" else None
    noise, drawn = None, -1
    fw.x.copy_(init)
    if plan["pre_sigma"] is not None:               # Heun's first xhat, before the first forward
        noise, drawn = draw(0), 0
        P = rows // noise.shape[0]
        th.add(init.view(2, P, noise.shape[0] // 2, -1), noise.view(2, 1, noise.shape[0] // 2, -1),
               alpha=plan["pre_sigma"], out=fw.x.view(2, P, noise.shape[0] // 2, -1))
    last = None
    for k, e in enumerate(plan["evals"]):
        f = fw(k)
        if e["noise"] is not None and e["noise"] > drawn:
            noise, drawn = draw(e["noise"]), e["noise"]
        x_out = state if record is None or not e["record"] else th.empty_like(state)
        ops.flow_sde_step(fw.x, f, cfg_scale=cfg_scale, t=e["t"], var=e["var"], diffusion=e["diffusion"],
                          mode=e["mode"], x=state if e["x_in"] else None, hist=hist if e["hist_in"] else None,
                          noise=noise if e["noise"] is not None else None, x_out=x_out, cx=e["cx"],
                          y_out=fw.x if e["cy"] is not None else None, cy=e["cy"] or (0.0,) * 5,
                          hist_out=hist if e["hist_out"] else None)
        if x_out is not state:
            record(x_out)
            last = x_out
    if record is not None and plan["last_step"] is None:
        record(last)
    return state
