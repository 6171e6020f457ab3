"""CPU: the host-side argument checks of the glue kernels (norm_modulate, final_layer, sampler_affine_update) and of
the VAE decoder's conv tail (conv_nhwc, groupnorm_stats, attn_single_head, patch_embed_triplane).

Every call goes through the C ABI with fabricated device addresses that are never dereferenced: a rejected call
must return LN3_EINVAL with a matching ln3_last_error(), and the aligned control call must get past validation,
which without a GPU means LN3_ECUDA.  With a GPU the control call would launch a kernel on those addresses, so
these tests only run where there is none.  Sizes that divide on the host (groupnorm's C % G) must be rejected
before the division: G = 0 once killed the process with SIGFPE."""
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


# ------------------------------------------------------------------ conv_nhwc
def _conv_args(**over):
    """A 3x3 conv with fused GroupNorm-apply, upsample and residual: every optional operand present."""
    from ln3diff_b200._lib import MLP_FP32, ConvArgs
    a = ConvArgs()
    for i, name in enumerate(("x", "w", "bias", "in_scale", "in_shift", "residual", "out")):
        setattr(a, name, _addr(i + 1))
    a.N, a.H, a.W, a.Cin, a.Cout, a.ksize, a.upsample, a.in_swish, a.precision = 2, 16, 16, 32, 40, 3, 1, 1, MLP_FP32
    for k, v in over.items():
        setattr(a, k, v)
    return a


def test_conv_control_passes_validation(lib):
    from ln3diff_b200._lib import MLP_TF32
    for over in ({}, dict(precision=MLP_TF32), dict(ksize=1, upsample=0), dict(bias=None, residual=None),
                 dict(in_scale=None, in_shift=None), dict(H=7, W=9, upsample=0), dict(Cin=1, Cout=1)):
        rc, msg = _call(lib, "ln3_conv_nhwc", _conv_args(**over))
        assert rc == ECUDA, (over, rc, msg)


@pytest.mark.parametrize("over,match", [
    (dict(Cin=0), "positive H, W, Cin, Cout"),      # once launched and wrote the bias alone
    (dict(Cin=-3), "positive H, W, Cin, Cout"),
    (dict(H=0), "positive H, W, Cin, Cout"),
    (dict(W=-2), "positive H, W, Cin, Cout"),
    (dict(Cout=0), "positive H, W, Cin, Cout"),
    (dict(N=-1), "N >= 0"),
    (dict(precision=7), "precision"),               # once ran fp32 without a word
    (dict(precision=-1), "precision"),
    (dict(H=15), "even H, W"),
    (dict(in_shift=None), "given together"),
    (dict(x=None), "null"),
    (dict(w=None), "null"),
    (dict(out=None), "null"),
    # a bad struct is rejected even when there is nothing to compute
    (dict(N=0, Cin=0), "positive H, W, Cin, Cout"),
    (dict(N=0, precision=7), "precision"),
    (dict(N=0, out=None), "null"),
])
def test_conv_rejects_bad_arguments(lib, over, match):
    rc, msg = _call(lib, "ln3_conv_nhwc", _conv_args(**over))
    assert rc == EINVAL and match in msg, (over, rc, msg)


def test_conv_ksize_and_empty_batch(lib):
    rc, msg = _call(lib, "ln3_conv_nhwc", _conv_args(ksize=5))
    assert rc == -3 and "ksize" in msg, (rc, msg)                    # LN3_EUNSUPPORTED
    assert _call(lib, "ln3_conv_nhwc", _conv_args(N=0))[0] == 0      # valid and empty: no launch


def test_conv_cout_tile_query(lib):
    """Below 64 output channels the tile is always 32; otherwise 32 or 64 by the SM count; 0 for a bad size."""
    for Cout in (1, 5, 24, 32, 40, 63):
        assert lib.ln3_conv_cout_tile(8, 128, 128, Cout) == 32, Cout
    for dims in ((1, 16, 16, 64), (24, 128, 128, 64), (4, 256, 256, 512)):
        assert lib.ln3_conv_cout_tile(*dims) in (32, 64), dims
    for dims in ((0, 16, 16, 64), (1, 0, 16, 64), (1, 16, -1, 64), (1, 16, 16, 0)):
        assert lib.ln3_conv_cout_tile(*dims) == 0, dims


# ------------------------------------------------------------------ groupnorm_stats, attn_single_head, patch_embed_triplane
def _gn(lib, N=2, HW=64, Cc=128, G=32):
    a = [C.c_void_p(_addr(i)) for i in range(1, 6)]
    rc = lib.ln3_groupnorm_stats(a[0], a[1], a[2], N, HW, Cc, G, C.c_float(1e-6), a[3], a[4], C.c_void_p(0))
    return rc, lib.ln3_last_error().decode(errors="replace")


def test_groupnorm_control_passes_validation(lib):
    for over in ({}, dict(Cc=32, G=32), dict(Cc=256, G=1), dict(HW=1)):
        rc, msg = _gn(lib, **over)
        assert rc == ECUDA, (over, rc, msg)
    assert _gn(lib, N=0, G=0)[0] == 0 and _gn(lib, N=-1)[0] == 0     # N <= 0: nothing to do


@pytest.mark.parametrize("over,match", [
    (dict(G=0), "positive G, C, HW"),     # evaluated C % 0 on the host: SIGFPE
    (dict(G=-1), "positive G, C, HW"),
    (dict(Cc=0), "positive G, C, HW"),
    (dict(Cc=-32), "positive G, C, HW"),
    (dict(HW=0), "positive G, C, HW"),    # on a device: 0 / 0 mean, NaN scale / shift
    (dict(HW=-5), "positive G, C, HW"),
    (dict(Cc=100, G=32), "bad C / G"),
    (dict(Cc=512, G=1), "bad C / G"),      # 512 channels per group: more than the 256 threads of the block
])
def test_groupnorm_rejects_bad_arguments(lib, over, match):
    rc, msg = _gn(lib, **over)
    assert rc == EINVAL and match in msg, (over, rc, msg)


def _attn(lib, N, L, Cc):
    a = [C.c_void_p(_addr(i)) for i in range(1, 5)]
    rc = lib.ln3_attn_single_head(a[0], a[1], a[2], a[3], N, L, Cc, C.c_void_p(0))
    return rc, lib.ln3_last_error().decode(errors="replace")


def test_attn_single_head_validation(lib):
    for Cc in (32, 64, 128):
        assert _attn(lib, 3, 256, Cc)[0] == ECUDA
    assert _attn(lib, 0, 0, 128)[0] == 0
    for L in (0, -9):
        rc, msg = _attn(lib, 1, L, 128)
        assert rc == EINVAL and "L > 0" in msg, (L, rc, msg)
    rc, msg = _attn(lib, 1, 16, 48)
    assert rc == -3 and "C must be" in msg, (rc, msg)               # LN3_EUNSUPPORTED


def _pet(lib, B=1, Cz=4, S=32, E=384, bias=True, silu=True):
    rc = lib.ln3_patch_embed_triplane(C.c_void_p(_addr(1)), C.c_void_p(_addr(2)), C.c_void_p(_addr(3)) if bias else None,
                                      B, Cz, S, E, C.c_float(1.0), C.c_void_p(_addr(4)),
                                      C.c_void_p(_addr(5)) if silu else None, C.c_void_p(0))
    return rc, lib.ln3_last_error().decode(errors="replace")


def test_patch_embed_triplane_control_passes_validation(lib):
    for over in ({}, dict(bias=False, silu=False), dict(Cz=16, S=2, E=1), dict(Cz=1, E=1024)):
        rc, msg = _pet(lib, **over)
        assert rc == ECUDA, (over, rc, msg)
    assert _pet(lib, B=0, S=0, E=0)[0] == 0


@pytest.mark.parametrize("over,match", [
    (dict(E=0), "positive S, E"),
    (dict(E=-4), "positive S, E"),
    (dict(S=0), "positive S, E"),
    (dict(S=-2), "positive S, E"),
    (dict(S=33), "even S"),
    (dict(Cz=17), "Cz <= 16"),
    (dict(Cz=0), "Cz <= 16"),
])
def test_patch_embed_triplane_rejects_bad_arguments(lib, over, match):
    rc, msg = _pet(lib, **over)
    assert rc == EINVAL and match in msg, (over, rc, msg)
