"""CPU: the transport's SDE samplers (Euler-Maruyama, Heun) against the reference's own outputs
(tests/golden/flow_sde.npz, oracle/make_golden_flow_sde.py), and the host side of ln3_flow_sde_step.

  - the mirror's torch path (Sampler.sample_sde on CPU tensors) and the fp32 oracle: bit-equal to the golden states
    (or rel-L2 <= 1e-6), the same model-call counts, list length and CPU generator state afterwards;
  - the float64 emulator of the fused evaluation plan: rel-L2 <= 1e-5, and the plan's forward counts;
  - the SDE interval and grid, Heun's float32 t + dt, and every refusal with its message;
  - the ctypes struct against the header, the export, and the LN3_EINVAL refusals of the C entry (fabricated
    addresses that are never dereferenced, so those run only without a GPU);
  - the pipeline and the ops entry refusing CPU tensors."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, ECUDA = -1, -2
BASE = 1 << 36
no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="fabricated addresses must not reach a real device")
CELLS = [(m, f, l) for m in ("Euler", "Heun") for f in ("sigma", "linear", "decreasing", "inccreasing-decreasing")
         for l in (None, "Mean", "Tweedie", "Euler") if not (m == "Heun" and l is None)]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "flow_sde.npz"))


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


def _key(m, f, l):
    return f"{m}_{f}_{l}"


@pytest.mark.parametrize("method,form,last", CELLS)
def test_mirror_torch_path_matches_reference(golden, method, form, last):
    from ln3diff_b200.transport import Sampler, create_transport
    from oracle import flow_sde as ofs
    zs, ctx = ofs.inputs()
    model = ofs.toy_cfg()
    fn = Sampler(create_transport(snr_type="lognorm")).sample_sde(sampling_method=method, diffusion_form=form,
                                                                 last_step=last, num_steps=ofs.STEPS)
    xs = fn(torch.cat([zs, zs], 0), model, context=ctx, cfg_scale=ofs.CFG)
    k = _key(method, form, last)
    assert len(xs) == int(golden[k + "_len"]) == ofs.STEPS
    assert model.calls == int(golden[k + "_calls"])
    assert torch.equal(torch.get_rng_state(), torch.from_numpy(golden["rng_after"]))
    ref = torch.from_numpy(golden[k])
    assert torch.equal(xs[-1], ref) or _rel(xs[-1], ref) <= 1e-6
    half = ref.shape[0] // 2
    assert not torch.equal(ref[:half], ref[half:]), "the two CFG halves draw their own noise and must diverge"


@pytest.mark.parametrize("method,form,last", CELLS)
def test_oracle_and_emulator_match_reference(golden, method, form, last):
    from ln3diff_b200.transport import sde_plan
    from oracle import flow_sde as ofs
    zs, ctx = ofs.inputs()
    noise = ofs.noises(ofs.STEPS)
    ref = torch.from_numpy(golden[_key(method, form, last)])
    init = torch.cat([zs, zs], 0)
    out = ofs.sample_sde(ofs.toy_cfg(), init, ctx, ofs.CFG, noise, sampling_method=method, diffusion_form=form,
                         last_step=last)
    assert torch.equal(out, ref) or _rel(out, ref) <= 1e-6, _rel(out, ref)
    plan = sde_plan(method, form, 1.0, last, 0.04, ofs.STEPS)
    em = ofs.emulate(plan, ofs.toy_raw(), init, ctx, ofs.CFG, noise)
    assert _rel(em, ref) <= 1e-5, _rel(em, ref)
    per_step = 1 if method == "Euler" else 2
    assert plan["forwards"] == per_step * (ofs.STEPS - 1) + (last is not None)


def test_emulator_maps_the_noise_of_batched_conditions():
    """R = P * N rows per half: every condition reads the same (2N, ...) draw, so P = 3 stacked copies of one
    condition give three copies of its result."""
    from ln3diff_b200.transport import sde_plan
    from oracle import flow_sde as ofs
    zs, ctx = ofs.inputs()
    noise = ofs.noises(ofs.STEPS)
    plan = sde_plan("Heun", "sigma", 1.0, "Mean", 0.04, ofs.STEPS)
    one = ofs.emulate(plan, ofs.toy_raw(), torch.cat([zs, zs]), ctx, ofs.CFG, noise)
    P = 3
    ctx3 = {"crossattn": torch.cat([ctx["crossattn"][:ofs.N].repeat(P, 1, 1), ctx["crossattn"][ofs.N:].repeat(P, 1, 1)])}
    three = ofs.emulate(plan, ofs.toy_raw(), torch.cat([zs.repeat(P, 1, 1, 1)] * 2), ctx3, ofs.CFG, noise)
    for g in range(P):
        assert torch.equal(three[g * ofs.N:(g + 1) * ofs.N], one[:ofs.N])
        assert torch.equal(three[P * ofs.N + g * ofs.N:P * ofs.N + (g + 1) * ofs.N], one[ofs.N:])


# ------------------------------------------------------------------ interval, grid and refusals
def test_interval_and_grid():
    from ln3diff_b200.transport import create_transport, sde_plan
    tr = create_transport(snr_type="lognorm")
    assert tr.check_interval(0, 0, sde=True, eval=True, last_step_size=0.04) == (0, 0.96)
    assert tr.check_interval(0, 0, sde=True, eval=True, last_step_size=0.0) == (0, 1)
    assert tr.check_interval(0, 0, sde=True, eval=True, diffusion_form="SBDM", last_step_size=0.04) == (0, 0.96)
    assert tr.check_interval(0, 0, sde=False) == (0, 1)
    p = sde_plan("Heun", "sigma", 1.0, "Mean", 0.04, 10)
    grid = torch.linspace(0, 0.96, 10)
    assert torch.equal(p["grid"], grid) and torch.equal(p["dt"], grid[1] - grid[0])
    for i in range(9):
        s1, s2 = p["evals"][2 * i], p["evals"][2 * i + 1]
        assert s1["t"] == float(grid[i])
        assert s2["t"] == float(grid[i] + (grid[1] - grid[0]))          # float32 t + dt, not the grid point
    assert p["evals"][-1]["t"] == float(torch.ones(1) * 0.96)
    p = sde_plan("Euler", "linear", 1.0, None, 0.04, 10)
    assert p["t1"] == 1 and p["last_step_size"] == 0.0 and len(p["evals"]) == 9


@pytest.mark.parametrize("kw,exc,match", [
    (dict(diffusion_form="SBDM"), ValueError, "SBDM"),
    (dict(sampling_method="Heun", last_step=None), ValueError, "Heun"),
    (dict(diffusion_form="constant"), NotImplementedError, "constant"),
    (dict(diffusion_form="increasing-decreasing"), NotImplementedError, "not implemented"),
    (dict(sampling_method="euler"), NotImplementedError, "Smapler"),
    (dict(last_step="mean"), NotImplementedError, "last_step"),
    (dict(num_steps=1), ValueError, "num_steps"),
])
def test_refusals(golden, kw, exc, match):
    from ln3diff_b200.transport import Sampler, create_transport
    args = dict(sampling_method="Euler", diffusion_form="sigma", last_step="Mean", num_steps=10)
    args.update(kw)
    with pytest.raises(exc, match=match):
        Sampler(create_transport(snr_type="lognorm")).sample_sde(**args)
    # what the reference does in those cells
    assert float(golden["sbdm_diffusion"][0]) == float("inf") and not bool(golden["sbdm_finite"])
    assert not any(bool(golden[f"heun_none_finite_{f}"]) for f in ("sigma", "linear", "decreasing",
                                                                    "inccreasing-decreasing"))
    assert str(golden["constant_error"]) == "TypeError"
    assert str(golden["increasing_decreasing_error"]) == "NotImplementedError"


def test_default_sde_form_is_the_reference_signature():
    import inspect
    from ln3diff_b200.transport import Sampler
    sig = inspect.signature(Sampler.sample_sde).parameters
    assert {k: v.default for k, v in sig.items() if k != "self"} == dict(
        sampling_method="Euler", diffusion_form="SBDM", diffusion_norm=1.0, last_step="Mean", last_step_size=0.04,
        num_steps=250)


# ------------------------------------------------------------------ ln3_flow_sde_step: ABI and refusals
def _fields(cname: str) -> list:
    src = open(os.path.join(ROOT, "include", "ln3b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    body = re.search(r"typedef struct " + cname + r"\s*\{(.*?)\}\s*" + cname + ";", src, flags=re.S).group(1)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            decl = re.sub(r"^(const\s+)?[A-Za-z_0-9]+(\s+long)?\s*\**", "", decl, count=1)
            names += [re.sub(r"\[\d+\]", "", n.strip().lstrip("*")) for n in decl.split(",")]
    return names


def test_ctypes_struct_matches_header(built_lib):
    from ln3diff_b200 import _lib, ops
    assert _fields("ln3_flow_sde_step_args") == [f[0] for f in _lib.FlowSdeStepArgs._fields_]
    assert _lib.FlowSdeStepArgs.cx.size == _lib.FlowSdeStepArgs.cy.size == 5 * C.sizeof(C.c_float)
    assert hasattr(C.CDLL(str(built_lib)), "ln3_flow_sde_step")
    src = open(os.path.join(ROOT, "include", "ln3b200.h")).read()
    assert "LN3_SDE_DRIFT = 0, LN3_SDE_VELOCITY = 1, LN3_SDE_SCORE = 2" in src
    assert (ops.SDE_DRIFT, ops.SDE_VELOCITY, ops.SDE_SCORE) == (0, 1, 2)


PTRS = ("x", "y", "f", "hist", "noise", "x_out", "y_out", "hist_out")
R_, N_, n_ = 6, 3, 12288
ROWS = 4 * 2 * R_ * n_


def _addr(i: int) -> int:
    return BASE + i * (1 << 24)


def _args(**over):
    from ln3diff_b200._lib import FlowSdeStepArgs
    a = FlowSdeStepArgs()
    for i, name in enumerate(PTRS):
        setattr(a, name, _addr(i + 1))
    a.R, a.N, a.n, a.mode = R_, N_, n_, 0
    for k, v in over.items():
        setattr(a, k, v)
    return a


@pytest.fixture(scope="module")
def lib(built_lib):
    from ln3diff_b200 import _lib
    return _lib.lib()


def _call(lib, a):
    rc = lib.ln3_flow_sde_step(C.byref(a), C.c_void_p(0))
    return rc, lib.ln3_last_error().decode(errors="replace")


@no_gpu
def test_flow_sde_step_valid_arguments_reach_the_launch(lib):
    for over in ({}, dict(x=None, hist=None, noise=None, N=0), dict(x_out=None, y_out=None), dict(mode=1),
                 dict(mode=2), dict(x_out=_addr(1)), dict(y_out=_addr(2)), dict(x_out=_addr(1), y_out=_addr(2)),
                 dict(N=6), dict(N=1), dict(R=1, N=1, n=4)):
        rc, msg = _call(lib, _args(**over))
        assert rc == ECUDA, (over, rc, msg)
    assert _call(lib, _args(R=0, noise=None))[0] == 0


@pytest.mark.parametrize("name", PTRS)
@no_gpu
def test_flow_sde_step_rejects_misaligned_pointer(lib, name):
    rc, msg = _call(lib, _args(**{name: _addr(PTRS.index(name) + 1) + 4}))
    assert rc == EINVAL and "16-byte aligned" in msg, (name, rc, msg)


@pytest.mark.parametrize("over,match", [
    (dict(n=12286), "% 4"),
    (dict(R=-1), "negative"),
    (dict(R=40000), "32767"),
    (dict(mode=3), "mode"),
    (dict(mode=-1), "mode"),
    (dict(y=None), "null"),
    (dict(f=None), "null"),
    (dict(x_out=None, y_out=None, hist_out=None), "no output"),
    # the noise row mapping
    (dict(N=0), "N <= R"),
    (dict(N=4), "R % N"),
    (dict(N=7), "N <= R"),
    # every overlap but the in-place updates
    (dict(x_out=_addr(2)), "output x_out overlaps input y"),
    (dict(x_out=_addr(1) + 16), "output x_out overlaps input x"),
    (dict(y_out=_addr(1)), "output y_out overlaps input x"),
    (dict(y_out=_addr(3) - ROWS + 16), "output y_out overlaps input f"),
    (dict(y_out=_addr(2) + 16), "output y_out overlaps input y"),
    (dict(hist_out=_addr(4)), "output hist_out overlaps input hist"),
    (dict(hist_out=_addr(5)), "output hist_out overlaps input noise"),
    (dict(x_out=_addr(3)), "output x_out overlaps input f"),
    (dict(x_out=_addr(7)), "outputs x_out and y_out overlap"),
    (dict(y_out=_addr(8)), "outputs y_out and hist_out overlap"),
    (dict(x_out=_addr(8) - 16), "outputs x_out and hist_out overlap"),
    (dict(R=0, y=None), "null"),
])
@no_gpu
def test_flow_sde_step_rejects_bad_arguments(lib, over, match):
    rc, msg = _call(lib, _args(**over))
    assert rc == EINVAL and match in msg, (over, rc, msg)


def test_ops_flow_sde_step_refuses_before_the_call():
    from ln3diff_b200 import ops
    x = torch.zeros(4, 8)
    with pytest.raises(ValueError, match="CUDA"):
        ops.flow_sde_step(x, x, cfg_scale=4.0, t=0.1, var=1.0, y_out=x)


def test_pipeline_sde_refusals_without_gpu():
    """The pipeline's CUDA check comes first; its argument checks are pure host logic."""
    from ln3diff_b200 import pipeline
    from ln3diff_b200.utils import build_i23d
    m = build_i23d("DiT-PixArt-B/2")
    with pytest.raises(RuntimeError, match="CUDA"):
        pipeline.sample_flow(m, {}, {}, 1, sde={})
    with pytest.raises(ValueError, match="sampling_method"):
        pipeline.sde_options({"num_steps": 5})
    with pytest.raises(ValueError, match="sampling_method"):
        pipeline.sde_options({"unknown": 1})
    assert pipeline.sde_options({}) == dict(sampling_method="Euler", diffusion_form="sigma", diffusion_norm=1.0,
                                            last_step="Mean", last_step_size=0.04)
