"""GPU: flow-matching SDE sampling (Euler-Maruyama, Heun) for image- and multi-view-to-3D.

  - ops.flow_sde_step element-wise: the drift d bit-equal to the reference's fp32 tensor ops, every output within
    8 * 2^-24 * sum|terms| of float64, in every mode, with P > 1 conditions sharing a noise draw, in place and out of
    place; and its refusals;
  - on DiT-PixArt-B/2: the pipeline against the fp32 oracle around the oracle DiT (rel-L2 < 2e-2, bf16 GEMMs), the
    mirror's fused Sampler.sample_sde against the pipeline, LN3_CUDA_GRAPH=0 against the graph (bit-identical), the
    forward counts, the CPU generator's draw sequence and the untouched CUDA generator;
  - four batched conditions against four sequential calls, a condition independent of its batch mates, and
    images_to_3d(..., sde=) end to end."""
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def _rel(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    return float((a - b).norm() / b.norm())


# ------------------------------------------------------------------ ops.flow_sde_step element-wise
@pytest.mark.parametrize("R,N,n", [(1, 1, 4), (3, 1, 12), (3, 3, 12), (16, 4, 12288)])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("inplace", [False, True])
def test_flow_sde_step_elementwise(dev, R, N, n, mode, inplace):
    from ln3diff_b200 import ops
    g = torch.Generator().manual_seed(R * 100 + n + mode)
    r = lambda rows: torch.randn(rows, n, generator=g).to(dev)
    x, y, f, hist, noise = r(2 * R), r(2 * R), r(2 * R), r(2 * R), r(2 * N)
    s, t, var, D = 4.0, 0.37, 0.5338, 0.63
    cx = (0.9, -1.1, 0.25, 0.125, 0.0)
    cy = (0.3, 1.0, -0.04, 0.5, 0.07)
    x0, y0 = x.clone(), y.clone()
    outs = dict(x_out=x if inplace else torch.empty_like(x), y_out=y if inplace else torch.empty_like(y),
                hist_out=torch.empty_like(y))
    ops.flow_sde_step(y, f, cfg_scale=s, t=t, var=var, diffusion=D, mode=mode, x=x, hist=hist, noise=noise, cx=cx,
                      cy=cy, **outs)
    torch.cuda.synchronize()
    # d as the reference's separate fp32 tensor ops on the CPU (var a broadcast tensor: a true division)
    f32 = lambda a: torch.full((2 * R, 1), a, dtype=torch.float32)
    fh, yh = f.cpu(), y0.cpu()
    fc, fu = fh[:R].repeat(2, 1), fh[R:].repeat(2, 1)
    v = fu + f32(s) * (fc - fu)
    sc = (f32(t) * v - yh) / f32(var)
    d = (v + f32(D) * sc, v, sc)[mode]
    assert torch.equal(outs["hist_out"].cpu(), d)
    d = d.to(dev)
    w = noise.view(2, 1, N, n).expand(2, R // N, N, n).reshape(2 * R, n)
    terms = [x0.double(), y0.double(), d.double(), hist.double(), w.double()]
    for name, k in (("x_out", cx), ("y_out", cy)):
        ref = sum(float(c) * tm for c, tm in zip(torch.tensor(k).tolist(), terms))
        bound = 8 * U * sum(abs(float(c)) * tm.abs() for c, tm in zip(torch.tensor(k).tolist(), terms)) + 1e-30
        err = (outs[name].double() - ref).abs()
        assert bool((err <= bound).all()), (name, float((err / bound).max()))


def test_flow_sde_step_optional_terms_and_outputs(dev):
    """NULL x / hist / noise drop their terms; only the requested outputs are written."""
    from ln3diff_b200 import ops
    R, n = 2, 16
    y, f = torch.randn(2 * R, n, device=dev), torch.randn(2 * R, n, device=dev)
    yo = torch.full_like(y, float("nan"))
    ops.flow_sde_step(y, f, cfg_scale=1.0, t=0.0, var=1.0, mode=ops.SDE_VELOCITY, y_out=yo, cy=(5.0, 1.0, 2.0, 7.0, 9.0))
    torch.cuda.synchronize()
    v = torch.cat([f[:R], f[:R]])                                     # s = 1: the conditional rows
    assert torch.allclose(yo, y + 2.0 * v, rtol=1e-6, atol=1e-6)


def test_flow_sde_step_refusals(dev):
    from ln3diff_b200 import ops
    y, f = torch.randn(4, 8, device=dev), torch.randn(4, 8, device=dev)
    kw = dict(cfg_scale=4.0, t=0.5, var=0.5)
    with pytest.raises(ValueError, match="at least one"):
        ops.flow_sde_step(y, f, **kw)
    with pytest.raises(RuntimeError, match="output y_out overlaps input f"):
        ops.flow_sde_step(y, f, y_out=f, **kw)
    with pytest.raises(RuntimeError, match="output x_out overlaps input y"):
        ops.flow_sde_step(y, f, x_out=y, **kw)
    y3, f3 = torch.randn(6, 8, device=dev), torch.randn(6, 8, device=dev)
    with pytest.raises(RuntimeError, match=r"R % N == 0 \(N = 2, R = 3\)"):
        ops.flow_sde_step(y3, f3, noise=torch.randn(4, 8, device=dev), y_out=y3, **kw)
    with pytest.raises(RuntimeError, match=r"N <= R .*\(N = 3, R = 2\)"):
        ops.flow_sde_step(y, f, noise=torch.randn(6, 8, device=dev), y_out=y, **kw)
    with pytest.raises(ValueError, match="multiple of 4"):
        ops.flow_sde_step(torch.randn(4, 6, device=dev), torch.randn(4, 6, device=dev), y_out=y, **kw)
    with pytest.raises(ValueError, match="mode"):
        ops.flow_sde_step(y, f, mode=3, y_out=y.clone(), **kw)


# ------------------------------------------------------------------ the pipeline on DiT-PixArt-B/2
STEPS, N = 5, 1
CASES = [("Euler", "sigma", "Mean"), ("Euler", "linear", None), ("Heun", "decreasing", "Tweedie"),
         ("Heun", "inccreasing-decreasing", "Euler")]


@pytest.fixture(scope="module")
def i23d(dev):
    from ln3diff_b200.utils import build_i23d
    m = build_i23d("DiT-PixArt-B/2")
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    return m.to(dev), sd


def _conditions(P, n, seed):
    g = torch.Generator().manual_seed(seed)
    vec, tok = torch.randn(P, 768, generator=g), torch.randn(P, 256, 2048, generator=g)
    c = {"vector": vec.repeat_interleave(n, 0), "crossattn": tok.repeat_interleave(n, 0)}
    return c, {k: torch.zeros_like(v) for k, v in c.items()}


def _sde(case):
    return dict(sampling_method=case[0], diffusion_form=case[1], last_step=case[2])


def _forwards(case, steps):
    return (1 if case[0] == "Euler" else 2) * (steps - 1) + (case[2] is not None)


@pytest.mark.parametrize("case", CASES)
def test_pipeline_vs_oracle_mirror_eager_and_rng(dev, i23d, case, monkeypatch):
    from ln3diff_b200 import ops, pipeline
    from ln3diff_b200.dit._graph import ForwardGraph
    from ln3diff_b200.transport import Sampler, create_transport
    from oracle import dit as odit
    from oracle import flow_sde as ofs
    m, sd = i23d
    c, uc = _conditions(1, N, seed=3)
    replays = [0]
    orig = ForwardGraph.replay

    def counting(self):
        replays[0] += 1
        return orig(self)
    monkeypatch.setattr(ForwardGraph, "replay", counting)
    out = pipeline.sample_flow(m, c, uc, N, seed=42, num_steps=STEPS, sde=_sde(case))
    cpu_after, cuda_after = torch.get_rng_state(), torch.cuda.get_rng_state(dev)
    assert replays[0] == _forwards(case, STEPS), replays[0]
    monkeypatch.setattr(ForwardGraph, "replay", orig)
    # the reference's draw sequence: manual_seed(seed), randn(N, ...), then randn(2N, ...) per step but the last;
    # manual_seed also seeds the CUDA generator, which the sampler must leave as seeded
    torch.manual_seed(42)
    assert torch.equal(torch.cuda.get_rng_state(dev), cuda_after), "the SDE draws on the CPU generator only"
    zs = torch.randn(N, 12, 32, 32)
    noise = [torch.randn(2 * N, 12, 32, 32) for _ in range(STEPS - 1)]
    assert torch.equal(torch.get_rng_state(), cpu_after)

    ctx = {k: torch.cat([c[k], uc[k]]) for k in c}
    raw = lambda x, t, cc: odit.dit_i23d_pixart_forward(sd, "DiT-PixArt-B/2", x, t, cc)
    ref = ofs.sample_sde(ofs.toy_cfg(raw), torch.cat([zs, zs]), ctx, 4.0, noise, num_steps=STEPS, **_sde(case))
    rel = _rel(out, ref[:N])
    print(f"{case}: pipeline vs oracle rel-L2 {rel:.3e}")
    assert rel < 2e-2, rel

    monkeypatch.setenv("LN3_CUDA_GRAPH", "0")
    eager = pipeline.sample_flow(m, c, uc, N, seed=42, num_steps=STEPS, sde=_sde(case))
    monkeypatch.delenv("LN3_CUDA_GRAPH")
    assert torch.equal(out, eager), _rel(eager, out)

    launches = []
    orig_step = ops.flow_sde_step
    monkeypatch.setattr(ops, "flow_sde_step", lambda *a, **k: (launches.append(1), orig_step(*a, **k))[1])
    ctxd = {k: v.to(dev) for k, v in ctx.items()}
    torch.manual_seed(42)
    zd = torch.randn(N, 12, 32, 32).to(dev)
    fn = Sampler(create_transport(snr_type="lognorm")).sample_sde(num_steps=STEPS, **_sde(case))
    xs = fn(torch.cat([zd, zd]), m.forward_with_cfg, context=ctxd, cfg_scale=4.0)
    assert len(xs) == STEPS and len(launches) == _forwards(case, STEPS)
    rel2 = _rel(xs[-1].chunk(2)[0], out)
    print(f"{case}: mirror (fused) vs pipeline rel-L2 {rel2:.3e}")
    assert rel2 <= 1e-3, rel2


def test_sde_none_keeps_the_ode_path(dev, i23d):
    from ln3diff_b200 import pipeline
    m, _ = i23d
    c, uc = _conditions(1, 2, seed=5)
    a = pipeline.sample_flow(m, c, uc, 2, num_steps=4, sampling_method="euler")
    b = pipeline.sample_flow(m, c, uc, 2, num_steps=4, sampling_method="euler", sde=None)
    assert torch.equal(a, b)
    with pytest.raises(ValueError, match="sampling_method"):
        pipeline.sample_flow(m, c, uc, 2, num_steps=4, sampling_method="euler", sde={})
    with pytest.raises(ValueError, match="SBDM"):
        pipeline.sample_flow(m, c, uc, 2, num_steps=4, sde={"diffusion_form": "SBDM"})


def _cat(*cs):
    return {k: torch.cat([c[k] for c in cs]) for k in cs[0]}


def _sl(c, i, n):
    return {k: v[i * n:(i + 1) * n] for k, v in c.items()}


@pytest.mark.parametrize("case", [("Euler", "sigma", "Mean"), ("Heun", "linear", "Tweedie")])
def test_four_conditions_match_four_sequential_calls(dev, i23d, case):
    from ln3diff_b200 import pipeline
    m, _ = i23d
    P, n, steps = 4, 2, 6
    c, uc = _conditions(P, n, seed=31)
    lat, st = pipeline.sample_flow_batched(m, c, uc, n, num_steps=steps, sde=_sde(case))
    assert lat.shape == (P, n, 12, 32, 32)
    assert st["batch_nfe"] == _forwards(case, steps) and st["nfe"] == [_forwards(case, steps)] * P
    for i in range(P):
        ref = pipeline.sample_flow(m, _sl(c, i, n), _sl(uc, i, n), n, num_steps=steps, sde=_sde(case))
        rel = _rel(lat[i], ref)
        print(f"{case} P=4 condition {i}: rel-L2 {rel:.3e}")
        assert rel <= 1e-2, (i, rel)


def test_condition_result_is_independent_of_its_batch(dev, i23d):
    from ln3diff_b200 import pipeline
    m, _ = i23d
    n = 2
    c, uc = _conditions(3, n, seed=11)
    A, B, C = (_sl(c, i, n) for i in range(3))
    UA = _sl(uc, 0, n)
    sde = dict(sampling_method="Heun", diffusion_form="sigma")
    lat_ab, _ = pipeline.sample_flow_batched(m, _cat(A, B), _cat(UA, UA), n, num_steps=4, sde=sde)
    lat_ac, _ = pipeline.sample_flow_batched(m, _cat(A, C), _cat(UA, UA), n, num_steps=4, sde=sde)
    assert torch.equal(lat_ab[0], lat_ac[0])
    assert not torch.equal(lat_ab[1], lat_ac[1])


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


def test_images_to_3d_sde_end_to_end_small(dev, i23d):
    from ln3diff_b200 import pipeline
    from ln3diff_b200.sgm.modules.encoders.modules import GeneralConditioner
    from ln3diff_b200.utils import build_ae_decoder, orbit_cameras
    m, _ = i23d
    P, S = 2, 2
    emb = _stub_image_embedder(dev)
    cond = GeneralConditioner([emb])
    dec = build_ae_decoder("DiT2-S/2", device=dev)
    g = torch.Generator().manual_seed(13)
    imgs = torch.rand(P, 3, 64, 64, generator=g) * 2 - 1
    cams = orbit_cameras(30).to(dev)
    sde = dict(sampling_method="Euler", last_step="Euler")
    lat, out, st = pipeline.images_to_3d(cond, m, dec, imgs, cams, num_samples=S, num_steps=6, resolution=32, sde=sde)
    assert lat.shape == (P, S, 12, 32, 32) and out["image_raw"].shape == (P, S, 24, 3, 32, 32)
    assert bool(torch.isfinite(out["image_raw"]).all()) and bool(torch.isfinite(lat).all())
    assert st["batch_nfe"] == 6
    tv = [emb(imgs[i:i + 1].to(dev)) for i in range(P)]
    c = {"vector": torch.cat([v for _, v in tv]).repeat_interleave(S, 0),
         "crossattn": torch.cat([t for t, _ in tv]).repeat_interleave(S, 0)}
    uc = {k: torch.zeros_like(v) for k, v in c.items()}
    lat2, _ = pipeline.sample_flow_batched(m, c, uc, S, num_steps=6, sde=sde)
    assert torch.equal(lat, lat2)
