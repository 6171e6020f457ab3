"""CPU: the sgm sampler family beyond Euler-EDM (Heun, Euler-ancestral, DPM++ 2S-a, DPM++ 2M, LMS) against the
reference's own outputs (tests/golden/edm_samplers.npz, oracle/make_golden_edm_samplers.py), and the host side of
ln3_sampler_step.

  - the mirrored classes on CPU tensors run the reference's torch arithmetic: bit-equal to the golden outputs, and
    they draw the same number of ancestral noises; LMS within rel-L2 1e-6 (its coefficients are integrated exactly
    instead of by scipy's quadrature);
  - the fp32 oracle restatements, within the same limits;
  - linear_multistep_coeff against the reference's scipy values;
  - pipeline.edm_sampler_plan applied by the float64 plan emulator (the kernel's formula per evaluation) around the
    toy network: rel-L2 <= 1e-5 for every sampler and both schedules, and the forward counts;
  - the ctypes struct against the header, the export, and every LN3_EINVAL refusal of the C entry (fabricated
    addresses that are never dereferenced, as in test_abi_validation.py, so those run only without a GPU)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("HeunEDMSampler", "EulerAncestralSampler", "DPMPP2SAncestralSampler", "DPMPP2MSampler",
         "LinearMultistepSampler")
EINVAL, ECUDA = -1, -2
BASE = 1 << 36
no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="fabricated addresses must not reach a real device")


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


def _toy_denoiser():
    from ln3diff_b200.sgm.modules.diffusionmodules.denoiser import DiscreteDenoiser
    from oracle import fixtures as fx
    disc = {"target": "sgm.modules.diffusionmodules.discretizer.LegacyDDPMDiscretization"}
    den = DiscreteDenoiser(scaling_config={"target": "sgm.modules.diffusionmodules.denoiser_scaling.EpsScaling"},
                           num_idx=1000, discretization_config=disc)
    toy = fx.toy_network()
    return disc, lambda inp, sig, cc: den(toy, inp, sig, cc)


def _run_mirror(name, S):
    from ln3diff_b200.sgm.modules.diffusionmodules import sampling as smp
    from oracle import edm_samplers as oes
    disc, fn = _toy_denoiser()
    s = getattr(smp, name)(discretization_config=disc, num_steps=S, device="cpu", guider_config={
        "target": "sgm.modules.diffusionmodules.guiders.VanillaCFG", "params": {"scale": oes.SCALE}})
    x0, c, uc = oes.inputs()
    noise = oes.step_noise(S)
    n = [0]

    def draw(v):
        n[0] += 1
        return noise[n[0] - 1]
    if hasattr(s, "noise_sampler"):
        s.noise_sampler = draw
    return s(fn, x0.clone(), c, uc), n[0]


@pytest.mark.parametrize("S", [10, 3])
@pytest.mark.parametrize("name", NAMES)
def test_mirror_classes_match_reference_golden(golden, name, S):
    g = golden("edm_samplers.npz")
    out, draws = _run_mirror(name, S)
    ref = torch.from_numpy(g[f"{name}_{S}"])
    if name == "LinearMultistepSampler":
        assert _rel(out, ref) <= 1e-6, _rel(out, ref)
    else:
        assert torch.equal(out, ref), _rel(out, ref)
    assert draws == int(g[f"{name}_{S}_draws"])


@pytest.mark.parametrize("S", [10, 3])
@pytest.mark.parametrize("name", NAMES)
def test_oracle_restatements_match_reference_golden(golden, name, S):
    from oracle import edm_samplers as oes
    from oracle import fixtures as fx
    g = golden("edm_samplers.npz")
    x0, c, uc = oes.inputs()
    out, draws = oes.edm_sample(name, fx.toy_network(), x0.clone(), c, uc, S, noise=oes.step_noise(S))
    ref = torch.from_numpy(g[f"{name}_{S}"])
    if name == "LinearMultistepSampler":
        assert _rel(out, ref) <= 1e-6, _rel(out, ref)
    else:
        assert torch.equal(out, ref), _rel(out, ref)
    assert draws == int(g[f"{name}_{S}_draws"])


@pytest.mark.parametrize("S", [10, 3])
def test_linear_multistep_coeff_matches_reference(golden, S):
    """The exact integral against scipy's quadrature of the same float64 integrand (1e-10), and against the
    coefficients the reference's sampler uses, whose integrand numpy evaluates in float32 (float32 sigma nodes)."""
    from ln3diff_b200.sgm.modules.diffusionmodules.sampling_utils import linear_multistep_coeff
    from oracle import edm_samplers as oes
    g = golden("edm_samplers.npz")
    sig = g[f"sigmas_{S}"]
    for i in range(S):
        cur = min(i + 1, 4)
        for j in range(cur):
            ours = linear_multistep_coeff(cur, sig, i, j)
            assert abs(ours - g[f"lms_coeff64_{S}"][i, j]) <= 1e-10 * abs(g[f"lms_coeff64_{S}"][i, j]), (i, j)
            assert abs(ours - g[f"lms_coeff_{S}"][i, j]) <= 1e-5 * abs(g[f"lms_coeff_{S}"][i, j]), (i, j)
            assert abs(oes.lms_coeff(cur, sig, i, j) - ours) <= 1e-12 * abs(ours), (i, j)
    with pytest.raises(ValueError):
        linear_multistep_coeff(3, sig, 1, 0)


@pytest.mark.parametrize("S", [10, 3])
def test_get_ancestral_step_matches_reference(golden, S):
    from ln3diff_b200.sgm.modules.diffusionmodules.sampling_utils import get_ancestral_step
    g = golden("edm_samplers.npz")
    sig = torch.from_numpy(g[f"sigmas_{S}"])
    sd, su = get_ancestral_step(sig[:-1], sig[1:], eta=1.0)
    assert torch.equal(sd, torch.from_numpy(g[f"sigma_down_{S}"]))
    assert torch.equal(su, torch.from_numpy(g[f"sigma_up_{S}"]))


FORWARDS = {"EulerAncestralSampler": lambda n: n, "DPMPP2MSampler": lambda n: n, "LinearMultistepSampler": lambda n: n,
            "HeunEDMSampler": lambda n: 2 * n - 1, "DPMPP2SAncestralSampler": lambda n: 2 * n - 1}


@pytest.mark.parametrize("S", [10, 3])
@pytest.mark.parametrize("name", NAMES)
def test_pipeline_plan_reproduces_reference(golden, name, S):
    from ln3diff_b200 import pipeline
    from oracle import edm_samplers as oes
    from oracle import fixtures as fx
    g = golden("edm_samplers.npz")
    plan = pipeline.edm_sampler_plan(name, S, oes.SCALE)
    assert len(plan["evals"]) == FORWARDS[name](S)
    assert sum(e["draw"] for e in plan["evals"]) == int(g[f"{name}_{S}_draws"])
    x0, c, uc = oes.inputs()
    out = oes.apply_plan(plan, fx.toy_network(), x0, c, uc, noise=oes.step_noise(S))
    assert _rel(out, g[f"{name}_{S}"]) <= 1e-5, _rel(out, g[f"{name}_{S}"])


def test_pipeline_plan_forward_counts_and_refusals():
    from ln3diff_b200 import pipeline
    for name, f in FORWARDS.items():
        for n in (1, 2, 25, 50):
            assert len(pipeline.edm_sampler_plan(name, n, 6.5)["evals"]) == f(n), (name, n)
    with pytest.raises(ValueError, match="unknown sampler"):
        pipeline.edm_sampler_plan("DDIMSampler", 10, 6.5)
    with pytest.raises(ValueError, match="order"):
        pipeline.edm_sampler_plan("LinearMultistepSampler", 10, 6.5, order=5)


def test_sample_t23d_argument_refusals():
    from ln3diff_b200 import pipeline
    x = torch.zeros(1, 12, 32, 32)
    with pytest.raises(RuntimeError, match="CUDA"):
        pipeline.sample_t23d(None, x, {}, {}, 4, sampler="DPMPP2MSampler")


def test_overlay_mirrors_sampling_utils():
    from ln3diff_b200 import overlay
    assert overlay.MIRRORED["sgm.modules.diffusionmodules.sampling_utils"] == \
        "ln3diff_b200.sgm.modules.diffusionmodules.sampling_utils"


# ------------------------------------------------------------------ ln3_sampler_step: ABI and refusals
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
    from ln3diff_b200 import _lib
    assert _fields("ln3_sampler_step_args") == [f[0] for f in _lib.SamplerStepArgs._fields_]
    assert _lib.SamplerStepArgs.hist.size == 3 * C.sizeof(C.c_void_p)
    assert hasattr(C.CDLL(str(built_lib)), "ln3_sampler_step")


PTRS = ("x", "x_eval", "net_u", "net_c", "hist0", "hist1", "hist2", "noise", "coef", "x_out", "eval_out", "hist_out")


def _addr(i: int) -> int:
    return BASE + i * (1 << 24)


def _args(**over):
    from ln3diff_b200._lib import SamplerStepArgs
    a = SamplerStepArgs()
    for i, name in enumerate(PTRS):
        if name.startswith("hist") and name != "hist_out":
            a.hist[int(name[4])] = _addr(i + 1)
        else:
            setattr(a, name, _addr(i + 1))
    a.B, a.n_per_sample = 3, 12288
    for k, v in over.items():
        if k.startswith("hist") and k != "hist_out":
            a.hist[int(k[4])] = v
        else:
            setattr(a, k, v)
    return a


@pytest.fixture(scope="module")
def lib(built_lib):
    from ln3diff_b200 import _lib
    return _lib.lib()


def _call(lib, a):
    rc = lib.ln3_sampler_step(C.byref(a), C.c_void_p(0))
    return rc, lib.ln3_last_error().decode(errors="replace")


@no_gpu
def test_sampler_step_control_and_aliases_pass_validation(lib):
    for over in ({}, dict(net_c=None, hist0=None, hist1=None, hist2=None, noise=None),
                 dict(x_out=None, eval_out=None), dict(hist_out=None, eval_out=None),
                 dict(x_out=_addr(1)), dict(eval_out=_addr(2)), dict(x_out=_addr(1), eval_out=_addr(2)),
                 dict(x_eval=_addr(1)), dict(B=1, n_per_sample=4)):
        rc, msg = _call(lib, _args(**over))
        assert rc == ECUDA, (over, rc, msg)
    assert _call(lib, _args(B=0))[0] == 0


@pytest.mark.parametrize("name", PTRS)
@no_gpu
def test_sampler_step_rejects_misaligned_pointer(lib, name):
    rc, msg = _call(lib, _args(**{name: _addr(PTRS.index(name) + 1) + 4}))
    assert rc == EINVAL and "16-byte aligned" in msg, (name, rc, msg)


ROW = 4 * 3 * 12288


@pytest.mark.parametrize("over,match", [
    (dict(n_per_sample=12286), "% 4"),
    (dict(n_per_sample=6), "% 4"),
    (dict(B=-1), "negative"),
    (dict(x=None), "null"),
    (dict(x_eval=None), "null"),
    (dict(net_u=None), "null"),
    (dict(coef=None), "null"),
    (dict(x_out=None, eval_out=None, hist_out=None), "no output"),
    # every overlap but the two in-place aliases
    (dict(x_out=_addr(2)), "overlaps input x_eval"),                  # x_out onto x_eval
    (dict(x_out=_addr(1) + 16), "overlaps input x"),                  # x_out inside x, other start
    (dict(eval_out=_addr(1)), "overlaps input x"),                    # eval_out onto x
    (dict(eval_out=_addr(2) + 16), "overlaps input x_eval"),
    (dict(eval_out=_addr(3) - ROW), "overlaps input net_u"),          # second half lands on net_u
    (dict(hist_out=_addr(5)), "overlaps input hist[0]"),              # hist_out onto a history input
    (dict(hist_out=_addr(7) + 16), "overlaps input hist[2]"),
    (dict(hist_out=_addr(1)), "overlaps input x"),
    (dict(hist_out=_addr(2)), "overlaps input x_eval"),
    (dict(hist_out=_addr(4)), "overlaps input net_c"),
    (dict(hist_out=_addr(8)), "overlaps input noise"),
    (dict(x_out=_addr(9)), "overlaps input coef"),
    (dict(x_out=_addr(11)), "outputs x_out and eval_out overlap"),
    (dict(eval_out=_addr(12) - ROW), "outputs eval_out and hist_out overlap"),
    (dict(x_out=_addr(12)), "outputs x_out and hist_out overlap"),
    # a bad struct is refused even when there is nothing to compute
    (dict(B=0, x=None), "null"),
    (dict(B=0, x_out=None, eval_out=None, hist_out=None), "no output"),
])
@no_gpu
def test_sampler_step_rejects_bad_arguments(lib, over, match):
    rc, msg = _call(lib, _args(**over))
    assert rc == EINVAL and match in msg, (over, rc, msg)


def test_ops_sampler_step_refuses_before_the_call():
    """ops.sampler_step checks CUDA placement first: CPU tensors never reach the library."""
    from ln3diff_b200 import ops
    x = torch.zeros(2, 8)
    with pytest.raises(ValueError, match="CUDA"):
        ops.sampler_step(x, x, torch.zeros(2, 12), x, x_out=x)
