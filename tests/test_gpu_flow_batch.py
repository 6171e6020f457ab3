"""GPU: batched image- and multi-view-to-3D on the grouped dopri5 solver -- the ln3_ode_* kernels against float64
torch element by element, the solver against the host solver per group, the independence of a condition's result
from the other conditions in its batch, the equivalence with sequential `sample_flow` calls, and the two pipelines
end to end at small size."""
import math
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ALPHA = (1 / 5, 3 / 10, 4 / 5, 8 / 9, 1.0, 1.0)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).norm() / b.norm())


class Problem:
    """Buffers and an argument block for B rows of n elements in the groups `rg`, with per-group t / dt set."""

    def __init__(self, dev, rg, n, t, dt, status=None, t_end=1.0, rtol=1e-3, atol=1e-6, seed=0, max_num_steps=100):
        from ln3diff_b200 import ops
        g = torch.Generator().manual_seed(seed)
        self.rg = torch.tensor(rg, dtype=torch.int32)
        B, G = len(rg), len(t)
        self.B, self.G, self.n = B, G, n
        r = lambda: torch.randn(B, n, generator=g).to(dev)
        self.y, self.f0, self.ks = r(), r(), [r() for _ in range(6)]
        self.y_stage = torch.full((B, n), float("nan"), device=dev)
        self.out = torch.full((B, n), float("nan"), device=dev)
        self.t_rows = torch.full((B,), -7.0, device=dev)
        st = ops.ode_state(G, 0.0, "cpu")
        f, i = st.view(torch.float64), st.view(torch.int32)
        f[:, 0] = torch.tensor(t, dtype=torch.float64)
        f[:, 2] = torch.tensor(t, dtype=torch.float64)
        f[:, 1] = torch.tensor(dt, dtype=torch.float64)
        if status is not None:
            i[:, 15] = torch.tensor(status, dtype=torch.int32)
        self.state = st.to(dev)
        self.t, self.dt = list(t), list(dt)
        self.rtol, self.atol, self.t_end = rtol, atol, t_end
        self.args = ops.ode_args(self.y, self.f0, self.y_stage, self.t_rows, self.out, self.rg, self.state,
                                 t_end=t_end, rtol=rtol, atol=atol, max_num_steps=max_num_steps)

    def fields(self):
        from ln3diff_b200 import ops
        torch.cuda.synchronize()
        return ops.ode_state_fields(self.state)


def _beta():
    from ln3diff_b200.transport import dopri5 as d5
    return d5._BETA, d5._C_ERROR, d5._C_MID


# ------------------------------------------------------------------ kernels vs float64
def test_stage_combination_every_tableau_row(dev):
    """y_stage = y + dt_g sum_j beta_ij k_j and t_rows = fp32(t_g + alpha_i dt_g) for stages 1..6 and the initial-step
    probe (stage 0); rows of a finished group are left untouched.  n = 1100 is not a multiple of the 1024-element
    chunk."""
    from ln3diff_b200 import ops
    BETA, _, _ = _beta()
    rg = [0, 1, 2, 0, 1, 2, 2]
    pb = Problem(dev, rg, 1100, t=[0.0, 0.25, 0.5], dt=[0.125, 0.03, 0.3], status=[0, 0, 1])
    y, k = pb.y.double().cpu(), [pb.f0.double().cpu()] + [x.double().cpu() for x in pb.ks]
    running = torch.tensor([g != 2 for g in rg])
    for stage in range(7):
        ops.ode_stage(pb.args, stage, pb.ks)
        torch.cuda.synchronize()
        ys, tr = pb.y_stage.cpu(), pb.t_rows.cpu()
        for r, g in enumerate(rg):
            if not running[r]:
                assert bool(torch.isnan(ys[r]).all()) and float(tr[r]) == -7.0, "finished rows must stay untouched"
                continue
            dt = pb.dt[g]
            if stage == 0:
                ref, tref, terms = y[r] + dt * k[0][r], pb.t[g] + dt, (dt * k[0][r]).abs()
            else:
                ref, terms = y[r].clone(), torch.zeros_like(y[r])
                for j, b in enumerate(BETA[stage - 1]):
                    ref += b * dt * k[j][r]
                    terms += (b * dt * k[j][r]).abs()
                tref = pb.t[g] + ALPHA[stage - 1] * dt
            bound = 8 * 2.0 ** -24 * (y[r].abs() + terms)
            assert bool(((ys[r].double() - ref).abs() <= bound).all()), (stage, r)
            assert float(tr[r]) == float(torch.tensor(tref, dtype=torch.float32)), (stage, r)
        pb.y_stage.fill_(float("nan"))
        pb.t_rows.fill_(-7.0)


def test_error_ratio_per_group(dev):
    """ratio = rms(err / (atol + rtol max(|y|, |y1|))) over each group's rows, err = dt sum_j c_err_j k_j."""
    from ln3diff_b200 import ops
    _, C_ERROR, _ = _beta()
    rg = [0, 1, 0, 2, 1, 2, 0]
    pb = Problem(dev, rg, 2048 + 12, t=[0.0, 0.1, 0.2], dt=[1e-3, 2e-3, 4e-3], rtol=1e-2, atol=1e-3, t_end=10.0)
    pb.y_stage.copy_(pb.y + 0.01 * torch.randn_like(pb.y))
    y, y1 = pb.y.double().cpu(), pb.y_stage.double().cpu()
    k = [pb.f0.double().cpu()] + [x.double().cpu() for x in pb.ks]
    ops.ode_step(pb.args, pb.ks)
    f = pb.fields()
    for g in range(3):
        rows = [r for r, gg in enumerate(rg) if gg == g]
        err = sum(c * pb.dt[g] * kj[rows] for c, kj in zip(C_ERROR, k))
        tol = 1e-3 + 1e-2 * torch.maximum(y[rows].abs(), y1[rows].abs())
        ref = float((err / tol).pow(2).mean().sqrt())
        assert abs(float(f["ratio"][g]) - ref) <= 1e-5 * ref, (g, float(f["ratio"][g]), ref)
        assert int(f["nfe"][g]) == 6 and int(f["accepted"][g]) + int(f["rejected"][g]) == 1


def test_controller_decisions_on_crafted_ratios(dev):
    """ratio 0, just below 1, just above 1 and one deep in the dfactor branch (safety / ratio^(1/5) < dfactor):
    y = y1 = 0 and k_0..k_5 = 0 except k_6 = f1 = c_g make err = -dt c_g / 60 and tol = atol, so ratio = dt c_g /
    (60 atol).  Checked: accept iff ratio <= 1, the next dt, the counters, t, and FSAL (f0 <- f1 on accept only)."""
    from ln3diff_b200 import ops
    targets = [0.0, 0.999, 1.001, 5000.0]
    rg = [0, 1, 2, 3, 3, 2, 1, 0]
    dt, atol = 0.1, 1e-6
    pb = Problem(dev, rg, 64, t=[0.0] * 4, dt=[dt] * 4, atol=atol, rtol=1e-3, t_end=1.0)
    for x in [pb.y, pb.f0, pb.y_stage] + pb.ks[:5]:
        x.zero_()
    cg = torch.tensor([targets[g] * 60 * atol / dt for g in rg], device=dev)
    pb.ks[5].copy_(cg[:, None].expand(-1, 64))
    ops.ode_step(pb.args, pb.ks)
    f = pb.fields()
    f0 = pb.f0.cpu()
    for g, tgt in enumerate(targets):
        ratio = float(f["ratio"][g])
        assert (ratio == 0.0) if tgt == 0 else abs(ratio - tgt) <= 1e-5 * tgt
        accept = ratio <= 1.0
        assert (ratio <= 1.0) == (tgt <= 1.0)
        if ratio == 0:
            dt_ref = dt * 10.0
        else:
            df = 1.0 if ratio < 1 else 0.2
            dt_ref = dt * min(10.0, max(0.9 / ratio ** 0.2, df))
        assert abs(float(f["dt"][g]) - dt_ref) <= 1e-14 * dt_ref, (g, float(f["dt"][g]), dt_ref)
        assert int(f["accepted"][g]) == int(accept) and int(f["rejected"][g]) == int(not accept)
        assert float(f["t"][g]) == (dt if accept else 0.0) and int(f["event"][g]) == int(accept)
        assert int(f["status"][g]) == 0
        for r in (r for r, gg in enumerate(rg) if gg == g):
            assert torch.equal(f0[r], pb.ks[5][r].cpu() if accept else torch.zeros(64)), (g, r)
    assert float(f["dt"][3]) == dt * 0.2                                   # the dfactor branch


def test_final_interpolation_at_t_end(dev):
    """An accepted step that crosses t_end writes the quartic dense output at t_end (_interp_eval of the host solver)
    into `out`, commits y <- y1, f0 <- f1 and marks the group done; a group that does not reach t_end leaves `out`
    untouched."""
    from ln3diff_b200 import ops
    _, _, C_MID = _beta()
    rg = [0, 1, 1, 0]
    n = 1024 + 256
    pb = Problem(dev, rg, n, t=[0.9, 0.1], dt=[0.15, 0.15], t_end=1.0, seed=3)
    base = pb.f0.clone()
    for x in pb.ks:                                   # nearly equal stage derivatives: a small error ratio
        x.copy_(base + 1e-3 * torch.randn_like(base))
    pb.y_stage.copy_(pb.y + 0.15 * base)
    y, f0, y1 = pb.y.double().cpu(), pb.f0.double().cpu(), pb.y_stage.double().cpu()
    k = [f0] + [x.double().cpu() for x in pb.ks]
    ops.ode_step(pb.args, pb.ks)
    fl = pb.fields()
    assert fl["ratio"].max() < 1.0 and fl["status"].tolist() == [1, 0] and fl["event"].tolist() == [2, 1]
    out = pb.out.cpu()
    dt = 0.15
    f1 = k[6]
    y_mid = y + sum(c * dt * kj for c, kj in zip(C_MID, k))
    a = 2 * dt * (f1 - f0) - 8 * (y1 + y) + 16 * y_mid
    b = dt * (5 * f0 - 3 * f1) + 18 * y + 14 * y1 - 32 * y_mid
    c = dt * (f1 - 4 * f0) - 11 * y - 5 * y1 + 16 * y_mid
    from ln3diff_b200.transport.dopri5 import _interp_eval
    t_new = float(fl["t"][0])
    assert t_new == 0.9 + 0.15
    ref = _interp_eval([y, dt * f0, c, b, a], 0.9, t_new, 1.0)
    scale = 256 * (y.abs() + y1.abs() + y_mid.abs() + dt * (f0.abs() + f1.abs()))
    for r, g in enumerate(rg):
        if g == 0:
            assert bool(((out[r].double() - ref[r]).abs() <= 2.0 ** -24 * scale[r]).all()), r
        else:
            assert bool(torch.isnan(out[r]).all()), r
        assert torch.equal(pb.y[r].cpu(), y1[r].float()) and torch.equal(pb.f0[r].cpu(), pb.ks[5][r].cpu())


def test_group_map_out_of_range_is_einval(dev):
    from ln3diff_b200 import ops
    pb = Problem(dev, [0, 1, 1, 0], 64, t=[0.0, 0.0], dt=[0.1, 0.1])
    pb.args.tensors[6][2] = 2                        # the host copy the entry points validate
    with pytest.raises(RuntimeError, match=r"code -1\).*row_group\[2\] = 2"):
        ops.ode_stage(pb.args, 1, pb.ks)
    pb.args.tensors[6][1:3] = 0                      # group 1 now has no row
    with pytest.raises(RuntimeError, match=r"code -1\).*group 1 has no rows"):
        ops.ode_step(pb.args, pb.ks)
    pb.args.tensors[6][2] = -1
    with pytest.raises(RuntimeError, match="code -1"):
        ops.ode_initial_step(pb.args, 0)


# ------------------------------------------------------------------ solver vs host solver
LAM, OMEGA = (0.5, 6.0, 60.0), (1.0, 3.0, 12.0)


def _linear_problem(dev, rows_per_group=2, n=64):
    g = torch.Generator().manual_seed(5)
    G = len(LAM)
    rg = [gg for gg in range(G) for _ in range(rows_per_group)]
    y0 = torch.randn(len(rg), n, generator=g).to(dev)
    lam = torch.tensor([LAM[gg] for gg in rg], device=dev)[:, None]
    om = torch.tensor([OMEGA[gg] for gg in rg], device=dev)[:, None]
    fn = lambda t, y: -lam * y + torch.cos(om * t[:, None])          # t: the per-row fp32 time
    return rg, y0, fn, lam, om


def _closed_form(y0, lam, om, t):
    A = lam / (lam ** 2 + om ** 2)
    return (y0 - A) * math.exp(-lam * t) + (lam * math.cos(om * t) + om * math.sin(om * t)) / (lam ** 2 + om ** 2)


def _host_group(fn, y0, rg, g, t1=1.0, **kw):
    from ln3diff_b200.transport.dopri5 import odeint_dopri5
    rows = [r for r, gg in enumerate(rg) if gg == g]
    st = {}
    sel = torch.tensor(rows, device=y0.device)

    def fg(t, y):
        full = torch.zeros_like(y0)
        full[sel] = y
        tt = torch.full((y0.shape[0],), float(t), device=y0.device, dtype=torch.float32)
        return fn(tt, full)[sel]
    sol = odeint_dopri5(fg, y0[sel].clone(), [0.0, 0.5, t1], stats=st, **kw)
    return rows, sol[-1], st


def test_grouped_solver_matches_host_solver_per_group(dev):
    """dy/dt = -lambda_g y + cos(omega_g t) with a different stiffness per group: each group takes exactly the steps
    odeint_dopri5 takes for it alone (nfe, accepted, rejected), ends within 1e-6 relative of it, and within the
    tolerance of test_dopri5_restatement_solves_known_odes of the closed form."""
    from ln3diff_b200.transport.dopri5 import odeint_dopri5_grouped
    rg, y0, fn, lam, om = _linear_problem(dev)
    y, st = odeint_dopri5_grouped(fn, y0, rg, len(LAM), rtol=1e-3, atol=1e-6)
    steps = []
    for g in range(len(LAM)):
        rows, ref, hst = _host_group(fn, y0, rg, g, rtol=1e-3, atol=1e-6)
        assert (st["nfe"][g], st["accepted"][g], st["rejected"][g]) == (hst["nfe"], hst["accepted"], hst["rejected"]), g
        # both solvers carry an fp32 state; their error ratios differ in the last bits (reduction order), so dt and
        # every later rounding differ, and the quartic dense output at t1 amplifies fp32 roundings up to ~32x
        rel = _rel(y[rows], ref)
        print(f"group {g}: {hst['accepted']} accepted, {hst['rejected']} rejected, rel-L2 to the host solver {rel:.2e}")
        assert rel <= 4e-6, g
        exact = _closed_form(y0[rows].double().cpu(), LAM[g], OMEGA[g], 1.0)
        assert float((y[rows].double().cpu() - exact).abs().max()) < 1e-2, g
        steps.append(hst["accepted"] + hst["rejected"])
    assert st["batch_nfe"] >= max(st["nfe"]) and st["batch_nfe"] <= max(st["nfe"]) + 6
    assert len(set(steps)) > 1, "the groups must take different step sequences"


def test_group_over_max_num_steps_raises_naming_it(dev):
    """The stiffest group exceeds max_num_steps: a RuntimeError names it, and the other groups' results and counters
    are those of an unlimited solve."""
    from ln3diff_b200.transport.dopri5 import Dopri5GroupError, odeint_dopri5_grouped
    rg, y0, fn, _, _ = _linear_problem(dev)
    y, st = odeint_dopri5_grouped(fn, y0, rg, len(LAM))
    steps = [a + r for a, r in zip(st["accepted"], st["rejected"])]
    worst = max(range(len(steps)), key=lambda g: steps[g])
    limit = steps[worst] - 1
    assert all(s <= limit for g, s in enumerate(steps) if g != worst)
    with pytest.raises(RuntimeError, match=f"group {worst}: max_num_steps") as ei:
        odeint_dopri5_grouped(fn, y0, rg, len(LAM), max_num_steps=limit)
    e = ei.value
    assert isinstance(e, Dopri5GroupError) and e.groups == [worst]
    for g in range(len(LAM)):
        if g == worst:
            continue
        rows = [r for r, gg in enumerate(rg) if gg == g]
        assert torch.equal(e.y[rows], y[rows])
        assert (e.stats["nfe"][g], e.stats["accepted"][g]) == (st["nfe"][g], st["accepted"][g])


# ------------------------------------------------------------------ denoiser: independence and equivalence
@pytest.fixture(scope="module")
def i23d(dev):
    from ln3diff_b200.utils import build_i23d
    return build_i23d("DiT-PixArt-B/2", device=dev)


def _i23d_conditions(P, N, seed):
    """P I23D conditions shaped like the conditioner's output (pooled (768,), tokens (256, 2048)), each repeated N
    times; the unconditional half is zero, as force_uc_zero_embeddings gives it."""
    g = torch.Generator().manual_seed(seed)
    vec, tok = torch.randn(P, 768, generator=g), torch.randn(P, 256, 2048, generator=g)
    c = {"vector": vec.repeat_interleave(N, 0), "crossattn": tok.repeat_interleave(N, 0)}
    return c, {k: torch.zeros_like(v) for k, v in c.items()}


def _cat(*cs):
    return {k: torch.cat([c[k] for c in cs]) for k in cs[0]}


def _sl(c, i, N):
    return {k: v[i * N:(i + 1) * N] for k, v in c.items()}


def test_condition_result_is_independent_of_its_batch(dev, i23d):
    """Batches [A, B] and [A, C] run the same launch sequence; A's latents and stats are bitwise equal."""
    from ln3diff_b200 import pipeline
    N = 2
    c, uc = _i23d_conditions(3, N, seed=11)
    A, B, C = (_sl(c, i, N) for i in range(3))
    UA = _sl(uc, 0, N)
    lat_ab, st_ab = pipeline.sample_flow_batched(i23d, _cat(A, B), _cat(UA, UA), N)
    lat_ac, st_ac = pipeline.sample_flow_batched(i23d, _cat(A, C), _cat(UA, UA), N)
    assert torch.equal(lat_ab[0], lat_ac[0])
    for k in ("nfe", "accepted", "rejected"):
        assert st_ab[k][0] == st_ac[k][0], k
    assert not torch.equal(lat_ab[1], lat_ac[1])


def _sequential(monkeypatch, model, c, uc, N):
    """pipeline.sample_flow(dopri5) with the host solver's stats captured."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.transport import dopri5 as d5
    seen = []
    real = d5.odeint_dopri5

    def spy(*a, **kw):
        out = real(*a, **kw)
        seen.append(dict(kw["stats"]))
        return out
    monkeypatch.setattr(d5, "odeint_dopri5", spy)
    lat = pipeline.sample_flow(model, c, uc, N, sampling_method="dopri5")
    monkeypatch.setattr(d5, "odeint_dopri5", real)
    return lat, seen[-1]


def test_single_condition_matches_sample_flow_dopri5(dev, i23d, monkeypatch):
    """P = 1: the same accepted / rejected counts as sample_flow(dopri5) and latents within 1e-3 relative L2 (the only
    intended difference is the order of the error-norm reduction)."""
    from ln3diff_b200 import pipeline
    N = 2
    c, uc = _i23d_conditions(1, N, seed=21)
    ref, hst = _sequential(monkeypatch, i23d, c, uc, N)
    lat, st = pipeline.sample_flow_batched(i23d, c, uc, N)
    rel = _rel(lat[0], ref)
    print(f"P=1: rel-L2 {rel:.3e}, host (acc, rej) = ({hst['accepted']}, {hst['rejected']}), "
          f"batched = ({st['accepted'][0]}, {st['rejected'][0]})")
    assert (st["accepted"][0], st["rejected"][0], st["nfe"][0]) == (hst["accepted"], hst["rejected"], hst["nfe"])
    assert rel <= 1e-3


def test_four_conditions_match_four_sequential_calls(dev, i23d, monkeypatch):
    """P = 4 in one batch vs four sequential sample_flow(dopri5) calls: per condition rel-L2 <= 1e-2 and NFE within
    one attempt (the batch size can change the GEMM tile schedule and with it the bf16 roundings)."""
    from ln3diff_b200 import pipeline
    P, N = 4, 2
    c, uc = _i23d_conditions(P, N, seed=31)
    lat, st = pipeline.sample_flow_batched(i23d, c, uc, N)
    for i in range(P):
        ref, hst = _sequential(monkeypatch, i23d, _sl(c, i, N), _sl(uc, i, N), N)
        rel = _rel(lat[i], ref)
        print(f"P=4 condition {i}: rel-L2 {rel:.3e}, nfe batched {st['nfe'][i]} vs sequential {hst['nfe']}")
        assert rel <= 1e-2, i
        assert abs(st["nfe"][i] - hst["nfe"]) <= 6, i


# ------------------------------------------------------------------ end to end
def _stub_image_embedder(dev):
    """A deterministic stand-in for the I23D image conditioner: (1, 3, H, W) -> tokens (1, 256, 2048) and a pooled
    (1, 768) embedding, both functions of the image."""
    from ln3diff_b200.sgm.modules.encoders.modules import AbstractEmbModel

    class Stub(AbstractEmbModel):
        def __init__(self):
            super().__init__()
            g = torch.Generator().manual_seed(4)
            self.wt = torch.randn(48, 256 * 8, generator=g).to(dev)
            self.wp = torch.randn(48, 768, generator=g).to(dev)

        def forward(self, img):
            feat = torch.nn.functional.adaptive_avg_pool2d(img.float(), 4).flatten(1)       # (B, 48)
            tok = torch.sin(feat @ self.wt).reshape(-1, 256, 8).repeat(1, 1, 256)
            return tok, torch.cos(feat @ self.wp)

    emb = Stub()
    emb._emb_config = {"input_key": "img", "ucg_rate": 0.0}
    return emb


def test_images_to_3d_end_to_end_small(dev, i23d):
    """P = 3 images: shapes of latents and renders; each condition's latents equal sample_flow_batched on the hand-built
    context (the conditioner's tokens repeated, zeros for the unconditional half)."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.sgm.modules.encoders.modules import GeneralConditioner
    from ln3diff_b200.utils import build_ae_decoder, orbit_cameras
    P, S = 3, 2
    emb = _stub_image_embedder(dev)
    cond = GeneralConditioner([emb])
    dec = build_ae_decoder("DiT2-S/2", device=dev)
    g = torch.Generator().manual_seed(13)
    imgs = torch.rand(P, 3, 64, 64, generator=g) * 2 - 1
    cams = orbit_cameras(30).to(dev)
    lat, out, st = pipeline.images_to_3d(cond, i23d, dec, imgs, cams, num_samples=S, resolution=32)
    assert lat.shape == (P, S, 12, 32, 32) and out["image_raw"].shape == (P, S, 24, 3, 32, 32)
    assert out["image_depth"].shape == (P, S, 24, 1, 32, 32) and len(st["nfe"]) == P
    assert bool(torch.isfinite(out["image_raw"]).all()) and bool(torch.isfinite(lat).all())
    tv = [emb(imgs[i:i + 1].to(dev)) for i in range(P)]                  # one image per call, as the pipeline
    c = {"vector": torch.cat([v for _, v in tv]).repeat_interleave(S, 0),
         "crossattn": torch.cat([t for t, _ in tv]).repeat_interleave(S, 0)}
    uc = {k: torch.zeros_like(v) for k, v in c.items()}
    lat2, _ = pipeline.sample_flow_batched(i23d, c, uc, S)
    assert torch.equal(lat, lat2)


def test_mvs_to_3d_end_to_end_small_with_camera_augmentation(dev):
    """P = 3 multi-view conditions with aug_c: the conditioner runs once per condition in order, so with the same
    seeds the augmented cameras -- and hence the latents -- equal those of sequential condition_prompt calls."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.sgm.modules.encoders.modules import FrozenDinov2ImageEmbedderMVPlucker, GeneralConditioner
    from ln3diff_b200.utils import build_ae_decoder, build_mv23d, orbit_cameras
    P, V, W, S = 3, 3, 256, 2
    emb = FrozenDinov2ImageEmbedderMVPlucker(arch="vitb", device=dev, n_cond_frames=V, enable_bf16=True, aug_c=True,
                                             random_init=True, width=W, depth=2, mlp_dim=4 * W, seed=3)
    emb._emb_config = {"input_key": "img-c", "ucg_rate": 0.0}
    cond = GeneralConditioner([emb])
    m = build_mv23d(depth=2, hidden_size=384, num_heads=6, context_dim=W, device=dev)
    dec = build_ae_decoder("DiT2-S/2", device=dev)
    g = torch.Generator().manual_seed(12)
    imgs = torch.rand(P, V, 3, 256, 256, generator=g) * 2 - 1
    mv_cams = torch.stack([orbit_cameras(V + i)[:V] for i in range(P)])
    cams = orbit_cameras(30).to(dev)
    random.seed(5); np.random.seed(5)
    lat, out, st = pipeline.mvs_to_3d(cond, m, dec, imgs, mv_cams.clone(), cams, num_samples=S, resolution=32)
    assert lat.shape == (P, S, 12, 32, 32) and out["image_raw"].shape == (P, S, 24, 3, 32, 32)
    assert bool(torch.isfinite(out["image_raw"]).all()) and bool(torch.isfinite(lat).all())
    random.seed(5); np.random.seed(5)
    cam_d = [mv_cams[i:i + 1].clone().to(dev) for i in range(P)]            # one (1, V, 25) tensor per call
    cs = [pipeline.condition_prompt(cond, "img-c", {"img": imgs[i:i + 1].to(dev), "c": cam_d[i]}, S, device=dev)
          for i in range(P)]
    c, uc = _cat(*[x[0] for x in cs]), _cat(*[x[1] for x in cs])
    assert not torch.equal(torch.cat(cam_d).cpu(), mv_cams), "aug_c must have rotated some cameras"
    lat2, _ = pipeline.sample_flow_batched(m, c, uc, S)
    assert torch.equal(lat, lat2)
