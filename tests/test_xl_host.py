"""CPU: DiT-XL/2 text-to-3D on the host side -- the registry entry builds with the reference's state_dict layout
(72-wide self-attention heads, a cross-attention that keeps 64-wide heads), the attention ABI's head-width rules,
fp8's width rule at 1152 and the XL entries that stay refused."""
import contextlib
import ctypes as C
import io

import pytest
import torch

EUNSUPPORTED = -3


def _xl(**kw):
    from ln3diff_b200.dit.dit_models_xformers import TextCondDiTBlock
    from ln3diff_b200.dit.dit_trilatent import DiT_models
    return DiT_models["DiT-XL/2"](input_size=32, num_classes=0, learn_sigma=False, in_channels=4, context_dim=768,
                                  roll_out=True, vit_blk=TextCondDiTBlock, **kw)


def test_xl_builds_with_72_wide_heads():
    with torch.device("meta"):
        m = _xl()
    assert (m.depth, m.embed_dim, m.num_heads) == (28, 1152, 16)
    assert m.embed_dim // m.num_heads == 72
    ca = m.blocks[0].cross_attn
    assert (ca.heads, ca.dim_head, ca.to_q.out_features) == (16, 64, 1024)


def test_xl_state_dict_matches_reference():
    """Keys and shapes against the reference's own DiT_TriLatent built by its DiT-XL/2 registry entry."""
    from oracle import _stubs
    _stubs.install()
    import dit.dit_models_xformers as dmx
    _stubs.patch_dit_namespace()
    import dit.dit_trilatent as dt
    with contextlib.redirect_stdout(io.StringIO()), torch.device("meta"):
        ref = dt.DiT_models["DiT-XL/2"](input_size=32, num_classes=0, learn_sigma=False, in_channels=4,
                                        context_dim=768, roll_out=True, vit_blk=dmx.TextCondDiTBlock)
        m = _xl()
    want = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == want


def test_other_head_widths_are_refused():
    from ln3diff_b200.dit.dit_models_xformers import TextCondDiTBlock
    from ln3diff_b200.dit.dit_trilatent import DiT_TriLatent
    for hidden, heads in ((1152, 12), (1024, 8), (1000, 16)):     # 96, 128 and a non-integral head width
        with pytest.raises(NotImplementedError, match="head_dim"), torch.device("meta"):
            DiT_TriLatent(hidden_size=hidden, num_heads=heads, depth=1, num_classes=0, learn_sigma=False,
                          in_channels=4, context_dim=768, roll_out=True, vit_blk=TextCondDiTBlock)


def test_fp8_width_rule_refuses_1152():
    """fp8 keeps its width rule (embed_dim a multiple of 256): the check prepare() runs raises at 1152 (prepare() itself
    needs the GPU; test_gpu_xl.py calls it)."""
    from ln3diff_b200.dit.dit_models_xformers import TextCondDiTBlock
    from ln3diff_b200.dit.dit_trilatent import DiT_TriLatent
    m = DiT_TriLatent(hidden_size=1152, num_heads=16, depth=1, num_classes=0, learn_sigma=False, in_channels=4,
                      context_dim=768, roll_out=True, vit_blk=TextCondDiTBlock)
    m.set_gemm_precision("fp8")
    with pytest.raises(RuntimeError, match="embed_dim % 256"):
        m._check_fp8_shapes()


def test_xl_entries_of_other_registries_stay_refused():
    from ln3diff_b200.dit.dit_decoder import DiT2_models
    from ln3diff_b200.dit.dit_i23d import DiT_models as I23D
    for k in ("DiT-XL/2", "DiT-PixArt-MV-XL/2"):
        with pytest.raises(NotImplementedError, match="not implemented"):
            I23D[k](input_size=32, num_classes=0, learn_sigma=False, in_channels=4, context_dim=1024, roll_out=True)
    assert "DiT2-XL/2" not in DiT2_models


# ------------------------------------------------------------------ the attention ABI's head-width rules
BASE = 1 << 40


@pytest.fixture(scope="module")
def lib(built_lib):
    from ln3diff_b200 import _lib
    return _lib.lib()


def _fmha(lib, **over):
    from ln3diff_b200._lib import FmhaArgs
    a = FmhaArgs()
    a.q, a.k, a.v, a.out = BASE, BASE + (1 << 24), BASE + (2 << 24), BASE + (3 << 24)
    a.B, a.H, a.Lq, a.Lkv, a.head_dim = 2, 16, 768, 768, 72
    for f in ("q_ld", "k_ld", "v_ld", "o_ld"):
        setattr(a, f, 3 * 16 * 72)
    for f in ("q_bs", "k_bs", "v_bs", "o_bs"):
        setattr(a, f, 768 * 3 * 16 * 72)
    a.scale = 72 ** -0.5
    for k, v in over.items():
        setattr(a, k, v)
    rc = lib.ln3_fmha_fwd(C.byref(a), C.c_void_p(0))
    return rc, lib.ln3_last_error().decode(errors="replace")


@pytest.mark.parametrize("hd", [0, 8, 32, 63, 65, 71, 73, 80, 96, 128])
def test_fmha_head_dim_outside_64_72_is_unsupported(lib, hd):
    rc, msg = _fmha(lib, head_dim=hd)
    assert rc == EUNSUPPORTED and "head_dim must be 64 or 72" in msg, (rc, msg)


def test_fmha_second_source_at_72_is_unsupported(lib):
    rc, msg = _fmha(lib, k2=BASE + (4 << 24), v2=BASE + (5 << 24), Lkv2=77, k2_ld=16 * 72, v2_ld=16 * 72,
                    k2_bs=77 * 16 * 72, v2_bs=77 * 16 * 72)
    assert rc == EUNSUPPORTED and "head_dim 64" in msg, (rc, msg)
