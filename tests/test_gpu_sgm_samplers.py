"""GPU (-m gpu): the sgm sampler family beyond Euler-EDM on the device.

  - ops.sampler_step element-wise against a float64 restatement, |err| <= 16 * 2^-24 * sum|terms| per element, for
    every output subset, 0-3 history operands, with and without net_c and noise, B in {1, 3, 16},
    n_per_sample in {4, 12, 12288}, and both in-place aliases;
  - pipeline.sample_t23d(sampler=...) on DiT-B/2, 4 steps, against the fp32 oracle restatement around the oracle DiT
    (rel-L2 < 2e-2, the Euler pipeline's bound), the mirrored class on its fused CUDA path (< 1e-2), the eager
    launch sequence (bit-identical), the forward count per sampler, and the device generator's state after an
    ancestral run;
  - the Euler loop on DiT-B/2 and DiT-PixelArt-B/2, bit-identical to a hand-written loop of public forwards;
  - DPM++ 2M with fp8 GEMMs against bf16 (rel-L2 < 0.1, the fp8 denoiser tests' limit)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

NAMES = ("HeunEDMSampler", "EulerAncestralSampler", "DPMPP2SAncestralSampler", "DPMPP2MSampler",
         "LinearMultistepSampler")
ANCESTRAL = ("EulerAncestralSampler", "DPMPP2SAncestralSampler")
FORWARDS = {"EulerAncestralSampler": lambda n: n, "DPMPP2MSampler": lambda n: n, "LinearMultistepSampler": lambda n: n,
            "HeunEDMSampler": lambda n: 2 * n - 1, "DPMPP2SAncestralSampler": lambda n: 2 * n - 1}
STEPS = 4


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).norm() / b.norm()).item()


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


# ------------------------------------------------------------------ ops.sampler_step element-wise
OUTS = [(xo, eo, ho) for xo in (0, 1) for eo in (0, 1) for ho in (0, 1) if xo or eo or ho]


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("net_c", [False, True])
@pytest.mark.parametrize("nh", [0, 1, 2, 3])
@pytest.mark.parametrize("B,n", [(1, 4), (3, 12), (16, 12288), (3, 12288), (16, 4), (1, 12)])
def test_sampler_step_elementwise(dev, B, n, nh, net_c, noise):
    from ln3diff_b200 import ops
    g = torch.Generator().manual_seed(B * 1000 + n + 10 * nh + 2 * net_c + noise)
    r = lambda *s: torch.randn(*s, generator=g) * 3
    x, xe, nu, nc, nz = r(B, n), r(B, n), r(B, n), r(B, n), r(B, n)
    hs = [r(B, n) for _ in range(nh)]
    coef = torch.randn(B, 12, generator=g)
    coef[:, 10:] = 0
    k0, k1, k2, a, b, c, h0, h1, h2, s = (coef[:, j:j + 1].double() for j in range(10))
    et = [k0 * xe.double(), k1 * nu.double()] + ([k2 * nc.double()] if net_c else [])
    e = sum(et)
    vt = [a * x.double(), b * xe.double(), c * e] + [(h0, h1, h2)[j] * hs[j].double() for j in range(nh)]
    vt += [s * nz.double()] if noise else []
    v = sum(vt)
    bound_e = 16 * 2.0 ** -24 * sum(t.abs() for t in et)
    bound_v = 16 * 2.0 ** -24 * (sum(t.abs() for t in vt[:2] + vt[3:]) + c.abs() * sum(t.abs() for t in et))
    d = lambda t: t.to(dev).contiguous()
    dx, dxe, dnu, dnc, dnz, dhs, dcoef = d(x), d(xe), d(nu), d(nc) if net_c else None, d(nz) if noise else None, \
        [d(h) for h in hs], d(coef)

    def check(out, ref, bound, what):
        err = (out.double().cpu() - ref).abs()
        assert bool((err <= bound).all()), (what, float((err - bound).max()))

    for xo, eo, ho in OUTS:
        outs = dict(x_out=torch.full((B, n), float("nan"), device=dev) if xo else None,
                    eval_out=torch.full((2 * B, n), float("nan"), device=dev) if eo else None,
                    hist_out=torch.full((B, n), float("nan"), device=dev) if ho else None)
        ops.sampler_step(dx, dxe, dcoef, dnu, dnc, dhs, dnz, **outs)
        if xo:
            check(outs["x_out"], v, bound_v, "x_out")
        if eo:
            check(outs["eval_out"][:B], v, bound_v, "eval_out[:B]")
            assert torch.equal(outs["eval_out"][:B], outs["eval_out"][B:])
        if ho:
            check(outs["hist_out"], e, bound_e, "hist_out")
    # the in-place aliases: x_out is x, eval_out starts at x_eval
    xa = dx.clone()
    ev = torch.empty(2 * B, n, device=dev)
    ev[:B].copy_(dxe)
    ops.sampler_step(xa, ev[:B], dcoef, dnu, dnc, dhs, dnz, x_out=xa, eval_out=ev)
    check(xa, v, bound_v, "x_out aliased to x")
    check(ev[:B], v, bound_v, "eval_out aliased to x_eval")
    assert torch.equal(ev[:B], ev[B:]) and torch.equal(ev[:B], xa)


def test_sampler_step_refusals(dev):
    from ln3diff_b200 import ops
    x = torch.zeros(2, 16, device=dev)
    coef = torch.zeros(2, 12, device=dev)
    ev = torch.zeros(4, 16, device=dev)
    with pytest.raises(ValueError, match="overlaps"):
        ops.sampler_step(x, x, coef, x, hist_out=x)
    with pytest.raises(ValueError, match="overlaps"):
        ops.sampler_step(x, ev[:2], coef, x, eval_out=ev, x_out=ev[2:])
    with pytest.raises(ValueError, match="at least one"):
        ops.sampler_step(x, x, coef, x)
    with pytest.raises(ValueError, match="multiple of 4"):
        y = torch.zeros(2, 6, device=dev)
        ops.sampler_step(y, y, coef, y, x_out=torch.zeros(2, 6, device=dev))


# ------------------------------------------------------------------ the pipeline on DiT-B/2
@pytest.fixture(scope="module")
def setup(dev):
    from ln3diff_b200.utils import build_t23d
    m = build_t23d("DiT-B/2")
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(43)
    x0 = torch.randn(2, 12, 32, 32, generator=g)
    c = {"crossattn": torch.randn(2, 77, 768, generator=g)}
    uc = {"crossattn": torch.zeros(2, 77, 768)}
    noise = torch.randn(STEPS, 2, 12, 32, 32, generator=g)
    m = m.to(dev)
    cd, ucd = {"crossattn": c["crossattn"].to(dev)}, {"crossattn": uc["crossattn"].to(dev)}
    return dict(m=m, sd=sd, x0=x0, c=c, uc=uc, noise=noise, cd=cd, ucd=ucd)


@pytest.mark.parametrize("name", NAMES)
def test_pipeline_vs_oracle_mirror_and_eager(dev, setup, name, monkeypatch):
    from ln3diff_b200 import pipeline
    from ln3diff_b200.dit._graph import ForwardGraph
    from ln3diff_b200.sgm.modules.diffusionmodules import sampling as smp
    from ln3diff_b200.sgm.modules.diffusionmodules.denoiser import DiscreteDenoiser
    from oracle import dit as odit
    from oracle import edm_samplers as oes
    S = setup
    m, x0 = S["m"], S["x0"]
    kw = dict(noise=S["noise"].to(dev)) if name in ANCESTRAL else {}
    replays = [0]
    orig = ForwardGraph.replay

    def counting(self):
        replays[0] += 1
        return orig(self)
    monkeypatch.setattr(ForwardGraph, "replay", counting)
    out = pipeline.sample_t23d(m, x0.to(dev), S["cd"], S["ucd"], STEPS, 6.5, sampler=name, **kw)
    assert replays[0] == FORWARDS[name](STEPS), (name, replays[0])
    monkeypatch.setattr(ForwardGraph, "replay", orig)

    ref, _ = oes.edm_sample(name, lambda xi, ti, cc: odit.dit_t23d_forward(S["sd"], "DiT-B/2", xi, ti, cc["crossattn"]),
                            x0.clone(), S["c"], S["uc"], STEPS, 6.5, noise=list(S["noise"]))
    rel = _rel(out, ref)
    print(f"{name}: pipeline vs oracle rel-L2 {rel:.3e}")
    assert rel < 2e-2, rel

    monkeypatch.setenv("LN3_CUDA_GRAPH", "0")
    eager = pipeline.sample_t23d(m, x0.to(dev), S["cd"], S["ucd"], STEPS, 6.5, sampler=name, **kw)
    monkeypatch.delenv("LN3_CUDA_GRAPH")
    assert torch.equal(out, eager), _rel(eager, out)

    disc = {"target": "sgm.modules.diffusionmodules.discretizer.LegacyDDPMDiscretization"}
    s = getattr(smp, name)(discretization_config=disc, num_steps=STEPS, device=str(dev), guider_config={
        "target": "sgm.modules.diffusionmodules.guiders.VanillaCFG", "params": {"scale": 6.5}})
    d = DiscreteDenoiser(scaling_config={"target": "sgm.modules.diffusionmodules.denoiser_scaling.EpsScaling"},
                         num_idx=1000, discretization_config=disc).to(dev)
    if name in ANCESTRAL:
        it = iter(S["noise"].to(dev))
        s.noise_sampler = lambda v: next(it)
    launches = []
    orig_step = smp.ops.sampler_step
    monkeypatch.setattr(smp.ops, "sampler_step", lambda *a, **k: (launches.append(1), orig_step(*a, **k))[1])
    out2 = s(lambda i, sg, cc: d(m, i, sg, cc), x0.clone().to(dev), S["cd"], S["ucd"])
    assert len(launches) == FORWARDS[name](STEPS)                 # the fused tail ran once per evaluation
    rel2 = _rel(out2, out)
    print(f"{name}: mirror class (fused) vs pipeline rel-L2 {rel2:.3e}")
    assert rel2 < 1e-2, rel2


def test_euler_default_is_unchanged(dev, setup):
    from ln3diff_b200 import pipeline
    S = setup
    a = pipeline.sample_t23d(S["m"], S["x0"].to(dev), S["cd"], S["ucd"], STEPS, 6.5)
    b = pipeline.sample_t23d(S["m"], S["x0"].to(dev), S["cd"], S["ucd"], STEPS, 6.5, sampler="EulerEDMSampler")
    assert torch.equal(a, b)
    with pytest.raises(ValueError, match="tables"):
        pipeline.sample_t23d(S["m"], S["x0"].to(dev), S["cd"], S["ucd"], STEPS, 6.5, sampler="DPMPP2MSampler",
                             tables=pipeline.edm_cfg_tables(STEPS, 6.5, 2, dev))
    with pytest.raises(ValueError, match="churn"):
        pipeline.sample_t23d(S["m"], S["x0"].to(dev), S["cd"], S["ucd"], STEPS, 6.5, sampler="HeunEDMSampler",
                             s_churn=1.0)


@pytest.mark.parametrize("arch", ["DiT-B/2", "DiT-PixelArt-B/2"])
def test_euler_is_a_loop_of_public_forwards(dev, arch):
    """The Euler loop, bit for bit, as a hand-written loop of the model's public forward: per step the two halves of
    the CFG input, model(x2, t_idx, ctx, in_scale=c_in), then the affine update.  DiT-B/2 runs its shared adaLN rows
    in the pipeline; the PixArt-style denoiser has no such table and ignores in_scale."""
    from ln3diff_b200 import ops, pipeline
    from ln3diff_b200.utils import build_t23d
    m = build_t23d(arch, device=dev)
    B = 2
    g = torch.Generator().manual_seed(17)
    x0 = torch.randn(B, 12, 32, 32, generator=g).to(dev)
    c = {"crossattn": torch.randn(B, 77, 768, generator=g).to(dev)}
    if arch == "DiT-PixelArt-B/2":
        c["vector"] = torch.randn(B, 768, generator=g).to(dev)
    uc = {k: torch.zeros_like(v) for k, v in c.items()}
    out = pipeline.sample_t23d(m, x0, c, uc, STEPS, 6.5)

    tabs = pipeline.edm_cfg_tables(STEPS, 6.5, B, dev)
    ctx = {k: torch.cat((uc[k], c[k])) for k in c}
    x = x0 * tabs["init_scale"]
    x2 = torch.empty(2 * B, 12, 32, 32, device=dev)
    for i in range(STEPS):
        x2[:B].copy_(x)
        x2[B:].copy_(x)
        net = m(x2, tabs["t_idx"][i], ctx, in_scale=tabs["c_in"][i])
        x = ops.sampler_affine_update(x, tabs["coef"][i], net[:B], net[B:])
    assert torch.isfinite(out).all()
    assert torch.equal(out, x), _rel(out, x)


@pytest.mark.parametrize("name", ANCESTRAL)
def test_ancestral_rng_follows_the_reference(dev, setup, name):
    """One device randn_like of the (B, 12, 32, 32) fp32 state per step, the last step included."""
    from ln3diff_b200 import pipeline
    S = setup
    torch.manual_seed(5)
    pipeline.sample_t23d(S["m"], S["x0"].to(dev), S["cd"], S["ucd"], STEPS, 6.5, sampler=name)
    after = torch.cuda.get_rng_state(dev)
    torch.manual_seed(5)
    x = torch.empty(2, 12, 32, 32, device=dev)
    for _ in range(STEPS):
        torch.randn_like(x)
    assert torch.equal(after, torch.cuda.get_rng_state(dev))


def test_dpmpp2m_fp8_vs_bf16(dev):
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_t23d
    m = build_t23d("DiT-B/2", device=dev)
    g = torch.Generator().manual_seed(9)
    x0 = torch.randn(2, 12, 32, 32, generator=g).to(dev)
    c = {"crossattn": torch.randn(2, 77, 768, generator=g).to(dev)}
    uc = {"crossattn": torch.zeros(2, 77, 768, device=dev)}
    ref = pipeline.sample_t23d(m, x0, c, uc, 10, 6.5, sampler="DPMPP2MSampler")
    m.set_gemm_precision("fp8")
    out = pipeline.sample_t23d(m, x0, c, uc, 10, 6.5, sampler="DPMPP2MSampler")
    rel = _rel(out, ref)
    print(f"DPM++ 2M 10 steps DiT-B/2: fp8 vs bf16 rel-L2 {rel:.4e}")
    assert bool(torch.isfinite(out).all()) and rel < 0.1
