"""CPU: the C-ABI library builds for sm_90a, loads, and exports every symbol include/*.h declares.
No compute calls (there is no GPU here); compute entry points must fail loudly without one."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "ln3b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ln3_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_expected_surface():
    syms = declared_symbols()
    for must in ("ln3_abi_version", "ln3_last_error", "ln3_gemm_bf16", "ln3_fmha_fwd", "ln3_norm_modulate",
                 "ln3_sampler_affine_update", "ln3_render_views", "ln3_generate_rays"):
        assert must in syms


def test_library_builds_loads_and_exports_every_symbol(built_lib):
    lib = ctypes.CDLL(str(built_lib))
    for s in declared_symbols():
        assert hasattr(lib, s), f"{s} declared in include/ln3b200.h but not exported"
    lib.ln3_abi_version.restype = ctypes.c_int
    assert lib.ln3_abi_version() == 1


def test_ctypes_structs_match_header_field_order():
    """The ctypes mirrors must list the same fields in the same order as the C structs."""
    from ln3diff_b200 import _lib
    src = open(os.path.join(ROOT, "include", "ln3b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    pairs = {"ln3_gemm_args": _lib.GemmArgs, "ln3_fmha_args": _lib.FmhaArgs,
             "ln3_norm_modulate_args": _lib.NormModulateArgs, "ln3_patch_embed_args": _lib.PatchEmbedArgs,
             "ln3_final_layer_args": _lib.FinalLayerArgs, "ln3_sampler_update_args": _lib.SamplerUpdateArgs,
             "ln3_render_args": _lib.RenderArgs, "ln3_query_points_args": _lib.QueryPointsArgs,
             "ln3_pack_frames_args": _lib.PackFramesArgs, "ln3_marching_cubes_args": _lib.MarchingCubesArgs,
             "ln3_conv_args": _lib.ConvArgs}
    for cname, cls in pairs.items():
        body = re.search(r"typedef struct " + cname + r"\s*\{(.*?)\}\s*" + cname + ";", src, flags=re.S).group(1)
        names = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            decl = re.sub(r"^(const\s+)?(unsigned\s+)?[A-Za-z_0-9]+(\s+long)?\s*\**", "", decl, count=1)
            names += [re.sub(r"\[.*?\]", "", n).strip().lstrip("*") for n in decl.split(",")]
        assert names == [f[0] for f in cls._fields_], cname


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback(built_lib):
    from ln3diff_b200 import ops
    with pytest.raises(ValueError, match="CUDA"):
        ops.gemm(torch.zeros(128, 64, dtype=torch.bfloat16), torch.zeros(128, 64, dtype=torch.bfloat16))
    from ln3diff_b200.utils import build_t23d
    m = build_t23d("DiT-B/2")
    with pytest.raises(RuntimeError, match="CUDA only"):
        m(torch.zeros(1, 12, 32, 32), torch.zeros(1), torch.zeros(1, 77, 768))


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "ln3diff_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), os.path.join(dp, f)
