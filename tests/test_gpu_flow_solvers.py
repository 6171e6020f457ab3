"""GPU: the batched flow solvers beyond dopri5 -- the grouped bosh3 / fehlberg2 / adaptive_heun solves against the host
solver per group, each condition of a batch against its solo `sample_flow` run (adaptive methods and the fixed-grid
rk4), CUDA-graph against eager forwards, `images_to_3d` end to end with rk4 and bosh3, and the default dopri5
`images_to_3d` latents against the parent revision's."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_ADAPTIVE = ("bosh3", "fehlberg2", "adaptive_heun")
STAGES = {"dopri5": 6, "bosh3": 3, "fehlberg2": 2, "adaptive_heun": 1}
GOLDEN_DOPRI5 = os.path.join(ROOT, "tests", "golden", "flow_dopri5_images_to_3d.npz")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).norm() / b.norm())


# ------------------------------------------------------------------ grouped solver vs host solver
LAM, OMEGA = (0.5, 6.0, 60.0), (1.0, 3.0, 12.0)


def _linear_problem(dev, rows_per_group=2, n=64, LAM=LAM, OMEGA=OMEGA):
    """dy/dt = -lambda_g y + cos(omega_g t), a different stiffness per group."""
    g = torch.Generator().manual_seed(5)
    rg = [gg for gg in range(len(LAM)) for _ in range(rows_per_group)]
    y0 = torch.randn(len(rg), n, generator=g).to(dev)
    lam = torch.tensor([LAM[gg] for gg in rg], device=dev)[:, None]
    om = torch.tensor([OMEGA[gg] for gg in rg], device=dev)[:, None]
    return rg, y0, (lambda t, y: -lam * y + torch.cos(om * t[:, None]))


def _closed_form(y0, lam, om, t):
    A = lam / (lam ** 2 + om ** 2)
    return (y0 - A) * math.exp(-lam * t) + (lam * math.cos(om * t) + om * math.sin(om * t)) / (lam ** 2 + om ** 2)


def _host_group(fn, y0, rg, g, method, **kw):
    from ln3diff_b200.transport.rk import odeint_rk_adaptive
    rows = [r for r, gg in enumerate(rg) if gg == g]
    sel = torch.tensor(rows, device=y0.device)
    st = {}

    def fg(t, y):
        full = torch.zeros_like(y0)
        full[sel] = y
        return fn(torch.full((y0.shape[0],), float(t), device=y0.device, dtype=torch.float32), full)[sel]
    sol = odeint_rk_adaptive(fg, y0[sel].clone(), [0.0, 0.5, 1.0], method, stats=st, **kw)
    return rows, sol[-1], st


@pytest.mark.parametrize("method", NEW_ADAPTIVE)
def test_grouped_solver_matches_host_solver_per_group(dev, method):
    """Each group takes exactly the steps odeint_rk_adaptive takes for it alone (nfe, accepted, rejected) and ends
    within 4e-6 relative L2 of it -- the bound of the dopri5 test: the error-norm reduction order is the only
    intended difference, and last-bit ratio differences change dt.  fehlberg2's stiffest group is lambda = 20: at 60
    it runs on its stability limit, where its error ratios come within 3e-4 of 1 and any last-bit difference in the
    trajectory can flip an accept / reject decision."""
    from ln3diff_b200.transport.rk import odeint_rk_adaptive_grouped
    lams, oms = ((0.5, 6.0, 20.0), (1.0, 3.0, 6.0)) if method == "fehlberg2" else (LAM, OMEGA)
    rg, y0, fn = _linear_problem(dev, LAM=lams, OMEGA=oms)
    y, st = odeint_rk_adaptive_grouped(fn, y0, rg, len(LAM), method=method, rtol=1e-3, atol=1e-6)
    S = STAGES[method]
    steps = []
    for g in range(len(LAM)):
        rows, ref, hst = _host_group(fn, y0, rg, g, method, rtol=1e-3, atol=1e-6)
        assert (st["nfe"][g], st["accepted"][g], st["rejected"][g]) == (hst["nfe"], hst["accepted"], hst["rejected"])
        assert hst["nfe"] == 2 + S * (hst["accepted"] + hst["rejected"])
        rel = _rel(y[rows], ref)
        print(f"{method} group {g}: {hst['accepted']} accepted, {hst['rejected']} rejected, rel-L2 to the host "
              f"solver {rel:.2e}")
        assert rel <= 4e-6, g
        exact = _closed_form(y0[rows].double().cpu(), lams[g], oms[g], 1.0)   # a sanity bound: the low-order
        assert float((y[rows].double().cpu() - exact).abs().max()) < 1e-1, g    # pairs are loose at rtol 1e-3
        steps.append(hst["accepted"] + hst["rejected"])
    assert max(st["nfe"]) <= st["batch_nfe"] <= max(st["nfe"]) + S
    assert len(set(steps)) > 1, "the groups must take different step sequences"


def test_grouped_failure_names_the_group(dev):
    from ln3diff_b200.transport.rk import RKGroupError, odeint_rk_adaptive_grouped
    rg, y0, fn = _linear_problem(dev)
    _, st = odeint_rk_adaptive_grouped(fn, y0, rg, len(LAM), method="bosh3")
    steps = [a + r for a, r in zip(st["accepted"], st["rejected"])]
    worst = max(range(len(steps)), key=lambda g: steps[g])
    with pytest.raises(RKGroupError, match=f"group {worst}: max_num_steps") as ei:
        odeint_rk_adaptive_grouped(fn, y0, rg, len(LAM), method="bosh3", max_num_steps=steps[worst] - 1)
    assert worst in ei.value.groups


# ------------------------------------------------------------------ denoiser: batch vs solo, graph vs eager
@pytest.fixture(scope="module")
def i23d(dev):
    from ln3diff_b200.utils import build_i23d
    return build_i23d("DiT-PixArt-B/2", device=dev)


def _i23d_conditions(P, N, seed):
    g = torch.Generator().manual_seed(seed)
    vec, tok = torch.randn(P, 768, generator=g), torch.randn(P, 256, 2048, generator=g)
    c = {"vector": vec.repeat_interleave(N, 0), "crossattn": tok.repeat_interleave(N, 0)}
    return c, {k: torch.zeros_like(v) for k, v in c.items()}


def _sl(c, i, N):
    return {k: v[i * N:(i + 1) * N] for k, v in c.items()}


def _solo(monkeypatch, model, c, uc, N, method, num_steps):
    """pipeline.sample_flow(method) with the host solver's stats captured (adaptive methods)."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.transport import rk
    seen = []
    real = rk.odeint_rk_adaptive

    def spy(*a, **kw):
        out = real(*a, **kw)
        seen.append(dict(kw["stats"]))
        return out
    monkeypatch.setattr(rk, "odeint_rk_adaptive", spy)
    lat = pipeline.sample_flow(model, c, uc, N, sampling_method=method, num_steps=num_steps)
    monkeypatch.setattr(rk, "odeint_rk_adaptive", real)
    return lat, (seen[-1] if seen else None)


@pytest.mark.parametrize("method", NEW_ADAPTIVE + ("rk4",))
def test_three_conditions_match_their_solo_runs(dev, i23d, monkeypatch, method):
    """P = 3 in one batch vs three sample_flow calls: per condition rel-L2 <= 1e-2 (the batch size can change the GEMM
    tile schedule and with it the bf16 roundings) and, for an adaptive method, NFE within one attempt or 10 %: those
    roundings move accept / reject decisions, and the low-order pairs take many short attempts."""
    from ln3diff_b200 import pipeline
    P, N, steps = 3, 2, 8
    c, uc = _i23d_conditions(P, N, seed=41)
    lat, st = pipeline.sample_flow_batched(i23d, c, uc, N, num_steps=steps, sampling_method=method)
    assert lat.shape == (P, N, 12, 32, 32) and bool(torch.isfinite(lat).all())
    for i in range(P):
        ref, hst = _solo(monkeypatch, i23d, _sl(c, i, N), _sl(uc, i, N), N, method, steps)
        rel = _rel(lat[i], ref)
        print(f"{method} P=3 condition {i}: rel-L2 {rel:.3e}, nfe batched {st['nfe'][i]}"
              + (f" vs solo {hst['nfe']}" if hst else ""))
        assert rel <= 1e-2, i
        if method == "rk4":
            assert hst is None and st["nfe"][i] == st["batch_nfe"] == 4 * (steps - 1)
        else:
            assert abs(st["nfe"][i] - hst["nfe"]) <= max(STAGES[method], 0.1 * hst["nfe"]), i


@pytest.mark.parametrize("method", ("bosh3", "fehlberg2", "rk4"))
def test_graph_and_eager_forwards_give_identical_latents(dev, i23d, monkeypatch, method):
    from ln3diff_b200 import pipeline
    N = 1
    c, uc = _i23d_conditions(2, N, seed=51)
    a, sa = pipeline.sample_flow_batched(i23d, c, uc, N, num_steps=6, sampling_method=method)
    monkeypatch.setenv("LN3_CUDA_GRAPH", "0")
    b, sb = pipeline.sample_flow_batched(i23d, c, uc, N, num_steps=6, sampling_method=method)
    monkeypatch.delenv("LN3_CUDA_GRAPH")
    assert torch.equal(a, b) and sa == sb


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
            feat = torch.nn.functional.adaptive_avg_pool2d(img.float(), 4).flatten(1)
            tok = torch.sin(feat @ self.wt).reshape(-1, 256, 8).repeat(1, 1, 256)
            return tok, torch.cos(feat @ self.wp)

    emb = Stub()
    emb._emb_config = {"input_key": "img", "ucg_rate": 0.0}
    return emb


@pytest.mark.parametrize("method", ("rk4", "bosh3"))
def test_images_to_3d_end_to_end_128(dev, i23d, method):
    """P = 2 images at 128^2 on random weights: shapes, finite renders, and latents equal to sample_flow_batched on
    the hand-built context."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.sgm.modules.encoders.modules import GeneralConditioner
    from ln3diff_b200.utils import build_ae_decoder, orbit_cameras
    P, S, steps = 2, 1, 10
    emb = _stub_image_embedder(dev)
    cond = GeneralConditioner([emb])
    dec = build_ae_decoder("DiT2-S/2", device=dev)
    imgs = torch.rand(P, 3, 64, 64, generator=torch.Generator().manual_seed(13)) * 2 - 1
    cams = orbit_cameras(30).to(dev)
    lat, out, st = pipeline.images_to_3d(cond, i23d, dec, imgs, cams, num_samples=S, num_steps=steps,
                                         resolution=128, sampling_method=method)
    assert lat.shape == (P, S, 12, 32, 32) and out["image_raw"].shape == (P, S, 24, 3, 128, 128)
    assert bool(torch.isfinite(out["image_raw"]).all()) and bool(torch.isfinite(lat).all())
    assert len(st["nfe"]) == P
    tv = [emb(imgs[i:i + 1].to(dev)) for i in range(P)]
    c = {"vector": torch.cat([v for _, v in tv]).repeat_interleave(S, 0),
         "crossattn": torch.cat([t for t, _ in tv]).repeat_interleave(S, 0)}
    uc = {k: torch.zeros_like(v) for k, v in c.items()}
    lat2, _ = pipeline.sample_flow_batched(i23d, c, uc, S, num_steps=steps, sampling_method=method)
    assert torch.equal(lat, lat2)


def dopri5_images_to_3d_case(dev):
    """The seeded default-solver case of test_default_dopri5_latents_equal_the_parent_revision: images_to_3d with no
    sampling_method on DiT-PixArt-B/2 (seed 0) and the stub conditioner, P = 2 images, N = 1.  Returns
    (latents, stats)."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.sgm.modules.encoders.modules import GeneralConditioner
    from ln3diff_b200.utils import build_ae_decoder, build_i23d, orbit_cameras
    model = build_i23d("DiT-PixArt-B/2", seed=0, device=dev)
    cond = GeneralConditioner([_stub_image_embedder(dev)])
    dec = build_ae_decoder("DiT2-S/2", device=dev)
    imgs = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(23)) * 2 - 1
    lat, _, st = pipeline.images_to_3d(cond, model, dec, imgs, orbit_cameras(30).to(dev), num_samples=1,
                                       resolution=32)
    return lat, st


def test_default_dopri5_latents_equal_the_parent_revision(dev):
    """tests/golden/flow_dopri5_images_to_3d.npz holds this case's latents and stats as the library computed them on
    an H100 before the grouped solver became tableau-driven; the default call must reproduce them bit for bit."""
    gold = np.load(GOLDEN_DOPRI5)
    lat, st = dopri5_images_to_3d_case(dev)
    for k in ("nfe", "accepted", "rejected"):
        assert st[k] == gold[k].tolist(), k
    assert torch.equal(lat.cpu(), torch.from_numpy(gold["latents"]))
