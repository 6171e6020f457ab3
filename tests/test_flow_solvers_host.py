"""CPU: the explicit Runge-Kutta flow solvers of transport/rk.py (restated torchdiffeq 0.2.3 dopri5, bosh3,
fehlberg2, adaptive_heun and rk4; parity unpinned) -- tableau consistency and the scipy cross-check, observed orders of
convergence on closed-form ODEs, the step controller, the non-FSAL f1 rule, refusals and argument checks, and
dopri5's host results against the parent revision's."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADAPTIVE = ("dopri5", "bosh3", "fehlberg2", "adaptive_heun")
FSAL = {"dopri5": True, "bosh3": True, "fehlberg2": False, "adaptive_heun": False}
ORDER = {"dopri5": 5, "bosh3": 3, "fehlberg2": 2, "adaptive_heun": 2}


def _rk():
    from ln3diff_b200.transport import rk
    return rk


@pytest.mark.parametrize("method", ADAPTIVE)
def test_tableau_consistency(method):
    """Row sums of beta equal alpha, sum(c_sol) = 1, sum(c_error) = 0, one weight per k, FSAL as torchdiffeq tests
    it."""
    tab = _rk().TABLEAUS[method]
    S = len(tab.alpha)
    assert len(tab.beta) == S and [len(b) for b in tab.beta] == list(range(1, S + 1))
    for a, b in zip(tab.alpha, tab.beta):
        assert abs(sum(b) - a) <= 1e-15, (a, b)
    assert len(tab.c_sol) == len(tab.c_error) == len(tab.mid) == S + 1
    assert abs(sum(tab.c_sol) - 1.0) <= 1e-15 and abs(sum(tab.c_error)) <= 1e-15
    assert tab.fsal == FSAL[method] and tab.order == ORDER[method]


def test_tableaus_against_scipy():
    """bosh3 is scipy's RK23 (C, A, B, E = -c_error); dopri5's alpha / beta / c_sol are RK45's C / A / B.  dopri5's
    error weights are not compared with RK45.E: torchdiffeq embeds a different 4th-order solution."""
    from scipy.integrate import RK23, RK45
    rk = _rk()
    b3 = rk.TABLEAUS["bosh3"]
    # scipy lists the stages before the FSAL one; that last stage (alpha 1) evaluates f at the solution B
    np.testing.assert_allclose(b3.alpha[:2], RK23.C[1:], rtol=0, atol=1e-15)
    for i, row in enumerate(b3.beta[:2]):
        np.testing.assert_allclose(row, RK23.A[i + 1, :i + 1], rtol=0, atol=1e-15)
    assert b3.alpha[2] == 1.0
    np.testing.assert_allclose(b3.beta[2], RK23.B, rtol=0, atol=1e-15)
    np.testing.assert_allclose(b3.c_sol[:-1], RK23.B, rtol=0, atol=1e-15)
    np.testing.assert_allclose(b3.c_error, -RK23.E, rtol=0, atol=1e-15)
    d5 = rk.TABLEAUS["dopri5"]
    np.testing.assert_allclose(d5.alpha[:5], RK45.C[1:], rtol=0, atol=1e-15)
    assert d5.alpha[5] == 1.0
    for i, row in enumerate(d5.beta[:5]):
        np.testing.assert_allclose(row, RK45.A[i + 1, :i + 1], rtol=0, atol=1e-15)
    np.testing.assert_allclose(d5.beta[5], RK45.B, rtol=0, atol=1e-15)
    np.testing.assert_allclose(d5.c_sol[:6], RK45.B, rtol=0, atol=1e-15)
    assert abs(d5.c_error[0] - (35 / 384 - 1951 / 21600)) <= 1e-17 and abs(RK45.E[0] - -71 / 57600) <= 1e-17


# ------------------------------------------------------------------ observed order of convergence
PROBLEMS = {   # f(t, y), y0, exact y(T), T
    "linear": (lambda t, y: -1.3 * y, 1.0, lambda T: math.exp(-1.3 * T), 1.0),
    "gauss": (lambda t, y: -t * y, 1.0, lambda T: math.exp(-T * T / 2), 2.0),
}


def _fixed_step_error(method, prob, n):
    """Global error at T of n equal steps of the tableau, its f1 (k[-1]) chained into the next step's f0."""
    rk = _rk()
    f, y0, exact, T = PROBLEMS[prob]
    tab = rk.TABLEAUS[method]
    y = torch.full((1,), y0, dtype=torch.float64)
    dt, t = T / n, 0.0
    f0 = f(t, y)
    for i in range(n):
        y, f0, _, _ = rk.rk_attempt(f, tab, t, y, f0, dt, 1e-3, 1e-6)
        t = (i + 1) * dt
    return abs(float(y[0]) - exact(T))


def _rk4_error(prob, n):
    rk = _rk()
    f, y0, exact, T = PROBLEMS[prob]
    y = rk.odeint_rk4(lambda t, y: f(float(t), y), torch.full((1,), y0, dtype=torch.float64),
                      torch.linspace(0, T, n + 1, dtype=torch.float64))
    return abs(float(y[-1, 0]) - exact(T))


@pytest.mark.parametrize("prob", sorted(PROBLEMS))
@pytest.mark.parametrize("method", ADAPTIVE + ("rk4",))
def test_observed_order_of_convergence(method, prob):
    """log2(e(h) / e(h/2)) on y' = lambda y and y' = -t y is within 0.3 of the nominal order."""
    err = _rk4_error if method == "rk4" else (lambda p, n: _fixed_step_error(method, p, n))
    nominal = 4 if method == "rk4" else ORDER[method]
    n = 16
    e1, e2 = err(prob, n), err(prob, 2 * n)
    observed = math.log2(e1 / e2)
    assert abs(observed - nominal) <= 0.3, (method, prob, e1, e2, observed)


@pytest.mark.parametrize("method", ADAPTIVE)
def test_adaptive_solver_meets_tolerance_on_closed_forms(method):
    rk = _rk()
    for prob in sorted(PROBLEMS):
        f, y0, exact, T = PROBLEMS[prob]
        st = {}
        y = rk.odeint_rk_adaptive(f, torch.full((2,), y0, dtype=torch.float64), [0.0, T / 2, T], method,
                                  rtol=1e-6, atol=1e-9, stats=st)
        assert y.shape == (3, 2)
        assert abs(float(y[1, 0]) - exact(T / 2)) < 1e-4 and abs(float(y[2, 0]) - exact(T)) < 1e-4, (prob, y)
        S = len(rk.TABLEAUS[method].alpha)
        assert st["nfe"] == 2 + S * (st["accepted"] + st["rejected"])


# ------------------------------------------------------------------ step controller
def test_controller_rules():
    """ratio 0 -> 10 dt; an accepted ratio below 1 never shrinks dt; a rejected one always does, bounded by dfactor.
    At exactly ratio == 1 the step is accepted but dfactor still applies (torchdiffeq sets dfactor = 1 only for
    ratio < 1), so dt becomes 0.9 dt."""
    rk = _rk()
    for order in (2, 3, 5):
        assert rk._next_dt(0.1, 0.0, order, 0.9, 10.0, 0.2) == 0.1 * 10.0
        assert rk._next_dt(0.1, 1.0, order, 0.9, 10.0, 0.2) == 0.1 * 0.9
        for ratio in (1e-12, 1e-3, 0.2, 0.5, 0.9, 0.999):
            new = rk._next_dt(0.1, ratio, order, 0.9, 10.0, 0.2)
            assert 0.1 <= new <= 1.0 + 1e-15, (order, ratio, new)
        for ratio in (1.0001, 1.5, 10.0, 1e6):
            new = rk._next_dt(0.1, ratio, order, 0.9, 10.0, 0.2)
            assert 0.1 * 0.2 - 1e-17 <= new < 0.1, (order, ratio, new)
        assert rk._next_dt(0.1, 0.5, order, 0.9, 10.0, 0.2) == 0.1 * min(10.0, max(0.9 / 0.5 ** (1.0 / order), 1.0))


@pytest.mark.parametrize("method", ADAPTIVE)
def test_rejected_step_is_retried_smaller_and_accepted_steps_never_shrink(method, monkeypatch):
    """A too-large first step on a stiff problem is rejected, retried from the same t with a smaller dt; across the
    whole solve every accepted attempt is followed by a dt at least as large."""
    rk = _rk()
    attempts = []
    real = rk.rk_attempt

    def spy(f, tab, t, y, f0, dt, rtol, atol):
        out = real(f, tab, t, y, f0, dt, rtol, atol)
        attempts.append((t, dt, out[3]))
        return out
    monkeypatch.setattr(rk, "rk_attempt", spy)
    st = {}
    rk.odeint_rk_adaptive(lambda t, y: -20.0 * y + torch.cos(5 * torch.tensor(t)), torch.ones(3, dtype=torch.float64),
                          [0.0, 1.0], method, first_step=0.5, stats=st)
    assert attempts[0][2] > 1.0 and st["rejected"] >= 1
    for (t, dt, ratio), (t2, dt2, _) in zip(attempts, attempts[1:]):
        if ratio < 1.0:
            assert t2 == t + dt and dt2 >= dt
        else:
            assert t2 == t and dt2 < dt
    assert st["accepted"] + st["rejected"] == len(attempts)


# ------------------------------------------------------------------ the non-FSAL f1 rule
@pytest.mark.parametrize("method", ("fehlberg2", "adaptive_heun"))
def test_non_fsal_step_returns_the_last_stage_derivative(method):
    """y1 = y0 + dt (c_sol . k) is recomputed, but f1 = k[-1] -- not f(t1, y1) -- and the next attempt starts from that
    f1 without evaluating f at (t1, y1)."""
    rk = _rk()
    tab = rk.TABLEAUS[method]
    f = lambda t, y: y * y + t
    y0 = torch.tensor([0.5, -0.25], dtype=torch.float64)
    dt = 0.2
    y1, f1, ks, _ = rk.rk_attempt(f, tab, 0.0, y0, f(0.0, y0), dt, 1e-3, 1e-6)
    assert f1 is ks[-1]
    assert torch.equal(y1, rk._lincomb(y0, ks, tab.c_sol, dt))
    assert not torch.equal(y1, rk._lincomb(y0, ks[:-1], tab.beta[-1], dt))
    assert float((f(dt, y1) - f1).abs().max()) > 1e-4
    calls = []

    def rec(t, y):
        calls.append((t, y.clone()))
        return f(t, y)
    st = {}
    rk.odeint_rk_adaptive(rec, y0, [0.0, 0.5], method, first_step=dt, rtol=0.1, atol=0.1, stats=st)
    S = len(tab.alpha)
    assert st["nfe"] == 1 + S * (st["accepted"] + st["rejected"]) and st["rejected"] == 0
    # the second attempt's first stage input is y1 + dt2 * alpha_1 * f1 with the first attempt's f1 = k[-1]
    t2, y_in = calls[1 + S]
    dt2 = (t2 - dt) / tab.alpha[0]
    ref = y1 + f1 * (tab.beta[0][0] * dt2)
    assert torch.allclose(y_in, ref, rtol=0, atol=1e-12)
    assert not torch.allclose(y_in, y1 + f(dt, y1) * (tab.beta[0][0] * dt2), rtol=0, atol=1e-6)


# ------------------------------------------------------------------ refusals and argument checks
@pytest.mark.parametrize("method", ("dopri8", "explicit_adams", "implicit_adams", "fixed_adams", "scipy_solver"))
def test_unbuilt_methods_raise_naming_the_built_ones(method):
    from ln3diff_b200 import pipeline
    from ln3diff_b200.transport import Sampler, create_transport
    fn = Sampler(create_transport(snr_type="lognorm")).sample_ode(sampling_method=method, num_steps=5)
    with pytest.raises(NotImplementedError, match="built: dopri5, bosh3, fehlberg2, adaptive_heun, euler, midpoint, "
                                                  "heun, rk4"):
        fn(torch.zeros(2, 4), lambda x, t, **kw: -x)
    with pytest.raises(NotImplementedError, match=method):
        _rk().odeint_rk_adaptive(lambda t, y: -y, torch.ones(2), [0.0, 1.0], method)
    m = torch.nn.Linear(1, 1)
    with pytest.raises(NotImplementedError, match="built:"):
        pipeline.sample_flow_batched(m, {"crossattn": torch.zeros(2, 1, 1)}, {"crossattn": torch.zeros(2, 1, 1)}, 1,
                                     sampling_method=method)


@pytest.mark.parametrize("method", ("bosh3", "rk4", "euler"))
def test_sde_with_an_ode_method_is_refused(method):
    from ln3diff_b200 import pipeline
    m = torch.nn.Linear(1, 1)
    with pytest.raises(ValueError, match="selects an ODE solver"):
        pipeline.sample_flow_batched(m, {"crossattn": torch.zeros(2, 1, 1)}, {"crossattn": torch.zeros(2, 1, 1)}, 1,
                                     sde={}, sampling_method=method)


@pytest.mark.parametrize("method", ("bosh3", "rk4"))
def test_batched_new_methods_refuse_the_cpu(method):
    from ln3diff_b200 import pipeline
    m = torch.nn.Linear(1, 1)
    with pytest.raises(RuntimeError, match="CUDA only"):
        pipeline.sample_flow_batched(m, {"crossattn": torch.zeros(2, 1, 1)}, {"crossattn": torch.zeros(2, 1, 1)}, 1,
                                     sampling_method=method)
    if method != "rk4":
        with pytest.raises(RuntimeError, match="CUDA only"):
            _rk().odeint_rk_adaptive_grouped(lambda t, y: -y, torch.zeros(2, 8), [0, 0], 1, method=method)


@pytest.mark.parametrize("method", ("bosh3", "fehlberg2", "adaptive_heun"))
def test_sample_ode_dispatches_the_adaptive_methods(method):
    """Sampler.sample_ode(sampling_method=...) runs the restated solver and records its stats."""
    from ln3diff_b200.transport import Sampler, create_transport
    from ln3diff_b200.transport import transport as tr
    sampler = tr.ode(drift=Sampler(create_transport(snr_type="lognorm")).drift, t0=0, t1=1, sampler_type=method,
                     num_steps=50, atol=1e-6, rtol=1e-3)
    x0 = torch.randn(2, 3, generator=torch.Generator().manual_seed(0))
    traj = sampler.sample(x0, lambda x, t, **kw: -x * t[:, None])
    assert traj.shape == (50, 2, 3) and sampler.last_stats["accepted"] > 0
    # fehlberg2's error estimate is that of its very accurate 1st-order solution: it takes few, long steps and is
    # the least accurate of the three at rtol = 1e-3 (6 steps, 3% relative error here)
    assert torch.allclose(traj[-1], x0 * math.exp(-0.5), rtol=5e-2 if method == "fehlberg2" else 2e-3, atol=0)


def test_sample_ode_rk4_is_odeint_rk4_on_the_float32_grid():
    from ln3diff_b200.transport import Sampler, create_transport
    fn = Sampler(create_transport(snr_type="lognorm")).sample_ode(sampling_method="rk4", num_steps=11)
    x0 = torch.randn(2, 3, generator=torch.Generator().manual_seed(1))
    vel = lambda x, t, **kw: -x * t[:, None]
    traj = fn(x0, vel)
    ref = _rk().odeint_rk4(lambda t, y: vel(y, torch.full((2,), float(t))), x0, torch.linspace(0, 1, 11))
    assert traj.shape == (11, 2, 3) and torch.equal(traj, ref)
    assert torch.allclose(traj[-1], x0 * math.exp(-0.5), atol=1e-5)


def test_ode_stage_counts_and_unknown_methods(built_lib):
    from ln3diff_b200 import _lib, ops
    L = _lib.lib()
    assert [L.ln3_ode_stages(m) for m in range(4)] == [6, 3, 2, 1]
    assert [ops.ode_stages(_lib.ODE_METHODS[m]) for m in ADAPTIVE] == [len(_rk().TABLEAUS[m].alpha) for m in ADAPTIVE]
    assert L.ln3_ode_stages(4) == -3 and L.ln3_ode_stages(-1) == -3
    assert b"unknown method" in L.ln3_last_error()
    with pytest.raises(RuntimeError, match="code -3"):
        ops.ode_stages(9)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_rk_entry_points_check_arguments_without_a_gpu(built_lib):
    """ln3_ode_rk_*: an unknown method is LN3_EUNSUPPORTED, a stage past the method's last LN3_EINVAL, and the step
    needs exactly the method's k[0 .. S-1]; valid arguments fail with LN3_ECUDA here.  (The pointers are never
    dereferenced: every call fails before a kernel runs.)"""
    from ln3diff_b200 import _lib
    L = _lib.lib()
    rg = (ctypes.c_int * 4)(0, 1, 1, 0)
    a = _lib.OdeArgs()
    fake = 1 << 20
    a.y = a.f0 = a.y_stage = a.t_rows = a.out = a.row_group = a.state = a.workspace = fake
    a.row_group_host = ctypes.cast(rg, ctypes.c_void_p)
    a.workspace_bytes = 1 << 20
    a.B, a.G, a.n_per_sample, a.max_num_steps = 4, 2, 64, 100
    for m, S in ((1, 3), (2, 2), (3, 1)):
        for i in range(6):
            a.k[i] = fake if i < S else None
        assert L.ln3_ode_rk_step(ctypes.byref(a), m, None) == -2, m
        assert L.ln3_ode_rk_stage(ctypes.byref(a), m, S, None) == -2, m
        assert L.ln3_ode_rk_stage(ctypes.byref(a), m, S + 1, None) == -1, m
        assert L.ln3_ode_rk_initial_step(ctypes.byref(a), m, 1, None) == -2, m
        a.k[S - 1] = None
        assert L.ln3_ode_rk_step(ctypes.byref(a), m, None) == -1, m
        assert b"k[%d]" % (S - 1) in L.ln3_last_error()
    for m in (-1, 4, 99):
        assert L.ln3_ode_rk_step(ctypes.byref(a), m, None) == -3
        assert L.ln3_ode_rk_stage(ctypes.byref(a), m, 1, None) == -3
        assert L.ln3_ode_rk_initial_step(ctypes.byref(a), m, 0, None) == -3


# ------------------------------------------------------------------ dopri5 unchanged
def test_dopri5_host_results_equal_the_parent_revision():
    """tests/golden/flow_solvers_dopri5_host.npz holds odeint_dopri5's solution and stats on this seeded problem as
    computed before the solver became one tableau of odeint_rk_adaptive; both must be bit-identical."""
    from ln3diff_b200.transport.dopri5 import odeint_dopri5
    gold = np.load(os.path.join(ROOT, "tests", "golden", "flow_solvers_dopri5_host.npz"))
    g = torch.Generator().manual_seed(7)
    y0 = torch.randn(3, 256, generator=g)
    w = torch.rand(3, 256, generator=g) * 4
    st = {}
    sol = odeint_dopri5(lambda t, y: -4.0 * y + 3 * math.sin(25 * t) * torch.cos(w * y), y0, [0.0, 0.3, 1.0],
                        rtol=1e-4, atol=1e-6, stats=st)
    assert [st["nfe"], st["accepted"], st["rejected"]] == gold["dopri5_host_stats"].tolist()
    assert st["rejected"] > 0
    assert torch.equal(sol, torch.from_numpy(gold["dopri5_host_sol"]))
