"""ctypes binding of libln3b200.so -- the reference-side stub a maintainer would add.

The reference (pure PyTorch) has no FFI; this file is the whole "binding": argument structs
mirroring include/ln3b200.h field by field, and one checked call helper.  There is no CPU
fallback: if the shared library is missing or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libln3b200.so"

LN3_OK = 0
ACT_NONE, ACT_GELU_ERF, ACT_GELU_TANH, ACT_SILU, ACT_QUICK_GELU = 0, 1, 2, 3, 4
OUT_BF16, OUT_F32, OUT_RESID_F32 = 0, 1, 2

_lib = None


class GemmArgs(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("W", C.c_void_p), ("bias", C.c_void_p), ("out", C.c_void_p),
        ("out2", C.c_void_p), ("gate", C.c_void_p),
        ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
        ("lda", C.c_longlong), ("ldw", C.c_longlong), ("ldo", C.c_longlong),
        ("ldo2", C.c_longlong), ("gate_ld", C.c_longlong),
        ("gate_rows", C.c_int), ("act", C.c_int), ("out_kind", C.c_int),
        ("head_norm_w", C.c_void_p), ("head_norm_nsec", C.c_int), ("head_norm_sec_cols", C.c_int),
        ("head_norm_eps", C.c_float),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
    ]


class FmhaArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p),
        ("B", C.c_int), ("H", C.c_int), ("Lq", C.c_int), ("Lkv", C.c_int), ("head_dim", C.c_int),
        ("q_ld", C.c_longlong), ("q_bs", C.c_longlong), ("k_ld", C.c_longlong),
        ("k_bs", C.c_longlong), ("v_ld", C.c_longlong), ("v_bs", C.c_longlong),
        ("o_ld", C.c_longlong), ("o_bs", C.c_longlong),
        ("scale", C.c_float),
        ("k2", C.c_void_p), ("v2", C.c_void_p), ("Lkv2", C.c_int),
        ("k2_ld", C.c_longlong), ("k2_bs", C.c_longlong), ("v2_ld", C.c_longlong), ("v2_bs", C.c_longlong),
        ("causal", C.c_int),
    ]


class NormModulateArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("out", C.c_void_p), ("shift", C.c_void_p), ("scale", C.c_void_p),
        ("shift_tab", C.c_void_p), ("scale_tab", C.c_void_p), ("weight", C.c_void_p),
        ("rows", C.c_int), ("D", C.c_int),
        ("ldx", C.c_longlong), ("ldo", C.c_longlong), ("mod_ld", C.c_longlong),
        ("mod_rows", C.c_int), ("norm", C.c_int), ("act", C.c_int), ("eps", C.c_float),
        ("resid", C.c_void_p), ("resid_gate", C.c_void_p), ("resid_ld", C.c_longlong),
        ("resid_gate_ld", C.c_longlong), ("resid_gate_rows", C.c_int),
        ("resid_bcast", C.c_void_p), ("resid_bcast_ld", C.c_longlong), ("resid_bcast_rows", C.c_int),
        ("resid_row_begin", C.c_int), ("resid_row_end", C.c_int),
        ("resid_out_gate", C.c_void_p), ("resid_out_gate_ld", C.c_longlong), ("resid_out_gate_rows", C.c_int),
    ]


class PatchEmbedArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("in_scale", C.c_void_p), ("weight", C.c_void_p), ("bias", C.c_void_p),
        ("pos_embed", C.c_void_p), ("tokens", C.c_void_p),
        ("B", C.c_int), ("Cin", C.c_int), ("S", C.c_int), ("D", C.c_int),
    ]


class PluckerPatchifyArgs(C.Structure):
    _fields_ = [
        ("image", C.c_void_p), ("cams", C.c_void_p), ("out", C.c_void_p),
        ("N", C.c_int), ("ldo", C.c_longlong),
    ]


class FinalLayerArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("shift", C.c_void_p), ("scale", C.c_void_p), ("shift_tab", C.c_void_p),
        ("scale_tab", C.c_void_p), ("weight", C.c_void_p), ("bias", C.c_void_p), ("out", C.c_void_p),
        ("B", C.c_int), ("S", C.c_int), ("D", C.c_int), ("Cout", C.c_int),
        ("mod_ld", C.c_longlong),
    ]


class SamplerUpdateArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("m0", C.c_void_p), ("m1", C.c_void_p), ("noise", C.c_void_p),
        ("coef", C.c_void_p), ("x_out", C.c_void_p),
        ("B", C.c_int), ("n_per_sample", C.c_longlong),
    ]


class RenderArgs(C.Structure):
    _fields_ = [
        ("planes_cl", C.c_void_p), ("view_obj", C.c_void_p), ("ray_o", C.c_void_p),
        ("ray_d", C.c_void_p), ("noise_coarse", C.c_void_p), ("noise_fine", C.c_void_p),
        ("w1", C.c_void_p), ("b1", C.c_void_p), ("w2", C.c_void_p), ("b2", C.c_void_p),
        ("rgb", C.c_void_p), ("depth", C.c_void_p), ("weights", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
        ("dbg_inbox", C.c_void_p), ("dbg_inds", C.c_void_p), ("dbg_order", C.c_void_p),
        ("dbg_zfine", C.c_void_p),
        ("V", C.c_int), ("M", C.c_int), ("H", C.c_int), ("W", C.c_int), ("C", C.c_int),
        ("S", C.c_int), ("S_importance", C.c_int), ("hidden_dim", C.c_int),
        ("decoder_output_dim", C.c_int),
        ("group_size", C.c_int), ("views_per_obj", C.c_int), ("white_back", C.c_int),
        ("mlp_precision", C.c_int),
        ("box_warp", C.c_double), ("bbox_min", C.c_double), ("bbox_max", C.c_double),
        ("image_w", C.c_int),
    ]


class QueryPointsArgs(C.Structure):
    _fields_ = [
        ("planes_cl", C.c_void_p), ("points", C.c_void_p), ("w1", C.c_void_p), ("b1", C.c_void_p),
        ("w2", C.c_void_p), ("b2", C.c_void_p), ("sigma", C.c_void_p), ("rgb", C.c_void_p),
        ("P", C.c_longlong),
        ("n_obj", C.c_int), ("C", C.c_int), ("H", C.c_int), ("W", C.c_int), ("hidden_dim", C.c_int),
        ("decoder_output_dim", C.c_int), ("grid_size", C.c_int), ("mlp_precision", C.c_int),
        ("aabb_min_x", C.c_float), ("aabb_min_y", C.c_float), ("aabb_min_z", C.c_float),
        ("aabb_max_x", C.c_float), ("aabb_max_y", C.c_float), ("aabb_max_z", C.c_float),
        ("box_warp", C.c_double),
    ]


class PackFramesArgs(C.Structure):
    _fields_ = [
        ("image", C.c_void_p), ("depth", C.c_void_p), ("lut", C.c_void_p), ("out", C.c_void_p),
        ("workspace", C.c_void_p),
        ("N", C.c_int), ("H", C.c_int), ("W", C.c_int),
    ]


class MarchingCubesArgs(C.Structure):
    _fields_ = [
        ("grid", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("totals", C.c_void_p),
        ("vertices", C.c_void_p), ("faces", C.c_void_p),
        ("nx", C.c_int), ("ny", C.c_int), ("nz", C.c_int), ("max_vertices", C.c_int), ("max_faces", C.c_int),
        ("iso", C.c_float), ("scale", C.c_float * 3), ("offset", C.c_float * 3),
    ]


class ConvArgs(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("in_scale", C.c_void_p),
        ("in_shift", C.c_void_p), ("residual", C.c_void_p), ("out", C.c_void_p),
        ("N", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cin", C.c_int), ("Cout", C.c_int),
        ("ksize", C.c_int), ("upsample", C.c_int), ("in_swish", C.c_int), ("precision", C.c_int),
    ]


NORM_NONE, NORM_LAYER, NORM_RMS = 0, 1, 2
MLP_FP32, MLP_TF32 = 0, 1


def lib() -> C.CDLL:
    """Load libln3b200.so (once).  Raises if it has not been built -- no silent fallback."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise RuntimeError(
                f"{LIB_PATH} is missing: run `python -m ln3diff_b200.build` (or "
                "__graft_entry__.build()); the hot path has no CPU fallback")
        L = C.CDLL(str(LIB_PATH))
        L.ln3_abi_version.restype = C.c_int
        L.ln3_last_error.restype = C.c_char_p
        L.ln3_launch_count.restype = C.c_ulonglong
        L.ln3_add_launch_count.restype = None
        L.ln3_render_workspace_bytes.restype = C.c_size_t
        L.ln3_gemm_workspace_bytes.restype = C.c_size_t
        L.ln3_marching_cubes_workspace_bytes.restype = C.c_size_t
        _lib = L
    return _lib


def check(rc: int, what: str = "ln3") -> None:
    if rc != LN3_OK:
        msg = lib().ln3_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")


def launch_count() -> int:
    return int(lib().ln3_launch_count())


def add_launch_count(n: int) -> None:
    lib().ln3_add_launch_count(C.c_ulonglong(n))


def current_stream() -> C.c_void_p:
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t) -> C.c_void_p:
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)
