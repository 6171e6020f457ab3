"""CPU: the host-side argument checks of the glue kernels (norm_modulate, final_layer, sampler_affine_update).

Every call goes through the C ABI with fabricated device addresses that are never dereferenced: a rejected call
must return LN3_EINVAL with a matching ln3_last_error(), and the aligned control call must get past validation,
which without a GPU means LN3_ECUDA.  With a GPU the control call would launch a kernel on those addresses, so
these tests only run where there is none."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(),
                                reason="fabricated addresses: the control call must not reach a real device")

EINVAL, ECUDA = -1, -2
BASE = 1 << 36        # fabricated 4 KB-aligned region; buffer i starts at BASE + i * 2^24


def _addr(i: int) -> int:
    return BASE + i * (1 << 24)


@pytest.fixture(scope="module")
def lib(built_lib):
    from ln3diff_b200 import _lib
    return _lib.lib()


def _call(lib, fn: str, args) -> tuple[int, str]:
    rc = getattr(lib, fn)(C.byref(args), C.c_void_p(0))
    return rc, lib.ln3_last_error().decode(errors="replace")


# ------------------------------------------------------------------ norm_modulate
NM_PTRS = ("x", "out", "shift", "scale", "shift_tab", "scale_tab", "weight", "resid", "resid_gate",
           "resid_bcast", "resid_out_gate")


def _nm_args(**over):
    """Every optional operand present (the closed-form CFG pass of a PixArt block, RMS with weight and tables)."""
    from ln3diff_b200._lib import NORM_RMS, NormModulateArgs
    a = NormModulateArgs()
    for i, name in enumerate(NM_PTRS):
        setattr(a, name, _addr(i + 1))
    D = 256
    a.rows, a.D, a.ldx, a.ldo, a.mod_ld, a.mod_rows = 8, D, D, D, 6 * D, 4
    a.norm, a.eps = NORM_RMS, 1e-5
    a.resid_ld, a.resid_gate_ld, a.resid_gate_rows = D, 6 * D, 4
    a.resid_bcast_ld, a.resid_bcast_rows, a.resid_row_begin, a.resid_row_end = D, 4, 0, 4
    a.resid_out_gate_ld, a.resid_out_gate_rows = 6 * D, 4
    for k, v in over.items():
        setattr(a, k, v)
    return a


def test_norm_modulate_aligned_control_passes_validation(lib):
    rc, msg = _call(lib, "ln3_norm_modulate", _nm_args())
    assert rc == ECUDA, (rc, msg)


@pytest.mark.parametrize("name", NM_PTRS)
@pytest.mark.parametrize("off", [4, 8])
def test_norm_modulate_rejects_misaligned_pointer(lib, name, off):
    """A column-offset view (mod[:, 1:1+D]) moves a base pointer by 4 bytes; 8 would do for the float4 kernel's
    64-bit bf16 accesses but not for the 256-bit kernel's 128-bit ones, so 16 is the one rule for all."""
    a = _nm_args(**{name: _addr(NM_PTRS.index(name) + 1) + off})
    rc, msg = _call(lib, "ln3_norm_modulate", a)
    assert rc == EINVAL, (name, off, rc, msg)
    assert "16-byte aligned" in msg, msg


# ------------------------------------------------------------------ final_layer
FL_PTRS = ("x", "shift", "scale", "shift_tab", "scale_tab", "weight", "bias", "out")


def _fl_args(**over):
    from ln3diff_b200._lib import FinalLayerArgs
    a = FinalLayerArgs()
    for i, name in enumerate(FL_PTRS):
        setattr(a, name, _addr(i + 1))
    a.B, a.S, a.D, a.Cout, a.mod_ld = 2, 32, 768, 4, 6 * 768
    for k, v in over.items():
        setattr(a, k, v)
    return a


def test_final_layer_aligned_control_passes_validation(lib):
    for over in ({}, dict(shift_tab=None, scale_tab=None), dict(bias=None), dict(D=1152, Cout=3, S=6)):
        rc, msg = _call(lib, "ln3_final_layer", _fl_args(**over))
        assert rc == ECUDA, (over, rc, msg)


@pytest.mark.parametrize("over,match", [
    (dict(S=7), "even S"),           # ops accepts S = 7 (T == 3 * 3**2): the last row / column were never written
    (dict(S=0), "even S"),
    (dict(Cout=0), "Cout > 0"),
    (dict(Cout=-1), "Cout > 0"),
    (dict(mod_ld=1), "mod_ld"),
    (dict(mod_ld=6 * 768 + 2), "mod_ld"),
    (dict(shift_tab=None), "given together"),
    (dict(scale_tab=None), "given together"),
])
def test_final_layer_rejects_bad_arguments(lib, over, match):
    rc, msg = _call(lib, "ln3_final_layer", _fl_args(**over))
    assert rc == EINVAL and match in msg, (over, rc, msg)


@pytest.mark.parametrize("name", ("x", "shift", "scale", "shift_tab", "scale_tab", "weight"))
def test_final_layer_rejects_misaligned_pointer(lib, name):
    rc, msg = _call(lib, "ln3_final_layer", _fl_args(**{name: _addr(FL_PTRS.index(name) + 1) + 4}))
    assert rc == EINVAL and "16-byte aligned" in msg, (name, rc, msg)


@pytest.mark.parametrize("name", ("bias", "out"))
def test_final_layer_accepts_scalar_operands_at_any_float_offset(lib, name):
    """bias and out are read / written one float at a time."""
    rc, msg = _call(lib, "ln3_final_layer", _fl_args(**{name: _addr(FL_PTRS.index(name) + 1) + 4}))
    assert rc == ECUDA, (name, rc, msg)


# ------------------------------------------------------------------ sampler_affine_update
SU_PTRS = ("x", "m0", "m1", "noise", "coef", "x_out")


def _su_args(**over):
    from ln3diff_b200._lib import SamplerUpdateArgs
    a = SamplerUpdateArgs()
    for i, name in enumerate(SU_PTRS):
        setattr(a, name, _addr(i + 1))
    a.B, a.n_per_sample = 3, 12288
    for k, v in over.items():
        setattr(a, k, v)
    return a


def test_sampler_update_aligned_control_passes_validation(lib):
    for over in ({}, dict(m1=None, noise=None)):
        rc, msg = _call(lib, "ln3_sampler_affine_update", _su_args(**over))
        assert rc == ECUDA, (over, rc, msg)


@pytest.mark.parametrize("name", SU_PTRS)
def test_sampler_update_rejects_misaligned_pointer(lib, name):
    rc, msg = _call(lib, "ln3_sampler_affine_update", _su_args(**{name: _addr(SU_PTRS.index(name) + 1) + 4}))
    assert rc == EINVAL and "16-byte aligned" in msg, (name, rc, msg)
