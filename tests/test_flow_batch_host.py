"""CPU: the host side of batched image- and multi-view-to-3D -- the row -> condition map of the CFG batch, the noise
and context layout against sequential `sample_flow` calls, the ctypes mirrors of the ln3_ode_* structs, and the
argument checks of the grouped dopri5 entry points, which fail loudly without a GPU."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("P,N", [(1, 1), (3, 1), (4, 4), (16, 4)])
def test_row_groups_follow_the_cfg_layout(P, N):
    """cat([zs, zs]) with P*N condition-major rows: rows gN..(g+1)N and PN+gN..PN+(g+1)N are condition g."""
    from ln3diff_b200.pipeline import flow_batch_row_groups
    rg = flow_batch_row_groups(P, N)
    assert rg.dtype == torch.int32 and rg.shape == (2 * P * N,)
    for g in range(P):
        assert rg[g * N:(g + 1) * N].eq(g).all() and rg[P * N + g * N:P * N + (g + 1) * N].eq(g).all()
    assert torch.bincount(rg.long()).tolist() == [2 * N] * P


def test_batched_noise_equals_sequential_draws():
    """Each condition gets the draw sample_flow makes for it alone: manual_seed(seed); randn(N, ...)."""
    from ln3diff_b200.pipeline import flow_batch_noise
    P, N, shape = 3, 4, (12, 32, 32)
    z = flow_batch_noise(P, N, shape, seed=42)
    after = torch.rand(1)                               # the global generator is left where sample_flow leaves it
    for g in range(P):
        torch.manual_seed(42)
        assert torch.equal(z[g * N:(g + 1) * N], torch.randn(N, *shape))
    assert torch.equal(after, torch.rand(1))


def test_context_is_all_conditional_rows_then_all_unconditional_rows():
    from ln3diff_b200.pipeline import flow_batch_context
    P, N = 3, 2
    c = {"crossattn": torch.arange(P * N, dtype=torch.float32)[:, None, None].expand(-1, 5, 8),
         "vector": torch.arange(P * N, dtype=torch.float32)[:, None].expand(-1, 4), "other": 7}
    uc = {"crossattn": -1 - c["crossattn"], "vector": -1 - c["vector"], "other": 7}
    ctx = flow_batch_context(c, uc)
    for k in ("crossattn", "vector"):
        assert ctx[k].shape[0] == 2 * P * N and ctx[k].is_contiguous() and ctx[k].dtype == torch.float32
        assert torch.equal(ctx[k][:P * N], c[k]) and torch.equal(ctx[k][P * N:], uc[k])
    assert ctx["other"] == 7
    bf = flow_batch_context(c, uc, dtype=torch.bfloat16)["vector"]
    assert bf.dtype == torch.float32 and torch.equal(bf, torch.cat([c["vector"], uc["vector"]]).bfloat16().float())


def _fields(cname: str) -> list:
    src = open(os.path.join(ROOT, "include", "ln3b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    body = re.search(r"typedef struct " + cname + r"\s*\{(.*?)\}\s*" + cname + ";", src, flags=re.S).group(1)
    names = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            decl = re.sub(r"^(const\s+)?(unsigned\s+)?[A-Za-z_0-9]+(\s+long)?\s*\**", "", decl, count=1)
            names += [re.sub(r"\[.*?\]", "", n).strip().lstrip("*") for n in decl.split(",")]
    return names


def test_ode_ctypes_structs_match_header_field_order():
    from ln3diff_b200 import _lib
    for cname, cls in (("ln3_ode_group", _lib.OdeGroup), ("ln3_ode_args", _lib.OdeArgs)):
        assert _fields(cname) == [f[0] for f in cls._fields_], cname
    assert ctypes.sizeof(_lib.OdeGroup) == 72 and ctypes.sizeof(_lib.OdeGroup) % 8 == 0


def test_ode_state_block_layout():
    from ln3diff_b200 import ops
    st = ops.ode_state(3, 0.25, "cpu")
    assert st.shape == (3, ops.ODE_GROUP_BYTES) and st.dtype == torch.uint8
    f = ops.ode_state_fields(st)
    assert f["t"].tolist() == [0.25] * 3 and f["t_prev"].tolist() == [0.25] * 3 and f["dt"].tolist() == [0.0] * 3
    assert f["status"].tolist() == [0] * 3 and f["nfe"].tolist() == [0] * 3
    from ln3diff_b200 import _lib
    g = _lib.OdeGroup.from_buffer_copy(bytes(st[1].numpy()))
    assert g.t == 0.25 and g.status == _lib.ODE_RUNNING


def test_ode_workspace_bytes(built_lib):
    from ln3diff_b200 import _lib
    L = _lib.lib()
    assert L.ln3_ode_workspace_bytes(8, 12288) == 8 * 12 * 2 * 8
    assert L.ln3_ode_workspace_bytes(3, 1028) == 3 * 2 * 2 * 8
    assert L.ln3_ode_workspace_bytes(0, 1024) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_ode_entry_points_fail_loudly_without_a_gpu(built_lib):
    """The checked Python wrappers refuse CPU tensors, the solver and the batched sampler refuse to run on the CPU,
    and the C entry points reject bad group maps with LN3_EINVAL before touching a device and otherwise fail with
    LN3_ECUDA.  (The pointers below are never dereferenced: every call fails before a kernel runs.)"""
    from ln3diff_b200 import _lib, ops, pipeline
    from ln3diff_b200.transport.dopri5 import odeint_dopri5_grouped
    x = torch.zeros(2, 8)
    with pytest.raises(ValueError, match="CUDA"):
        ops.ode_args(x, x, x, torch.zeros(2), x, torch.zeros(2, dtype=torch.int32), ops.ode_state(1, 0.0, "cpu"),
                     t_end=1.0, rtol=1e-3, atol=1e-6)
    with pytest.raises(RuntimeError, match="CUDA only"):
        odeint_dopri5_grouped(lambda t, y: -y, x, [0, 0], 1)
    m = torch.nn.Linear(1, 1)
    with pytest.raises(RuntimeError, match="CUDA only"):
        pipeline.sample_flow_batched(m, {"crossattn": torch.zeros(2, 1, 1)}, {"crossattn": torch.zeros(2, 1, 1)}, 1)
    L = _lib.lib()
    rg = (ctypes.c_int * 4)(0, 1, 1, 0)
    a = _lib.OdeArgs()
    fake = 1 << 20
    a.y = a.f0 = a.y_stage = a.t_rows = a.out = a.row_group = a.state = a.workspace = fake
    for i in range(6):
        a.k[i] = fake
    a.row_group_host = ctypes.cast(rg, ctypes.c_void_p)
    a.workspace_bytes = 1 << 20
    a.B, a.G, a.n_per_sample, a.max_num_steps = 4, 2, 64, 100
    assert L.ln3_ode_step(ctypes.byref(a), None) == -2                        # valid arguments: no device
    rg[2] = 2
    assert L.ln3_ode_stage(ctypes.byref(a), 1, None) == -1
    assert b"row_group[2] = 2" in L.ln3_last_error()
    rg[1] = rg[2] = 0
    assert L.ln3_ode_initial_step(ctypes.byref(a), 0, None) == -1
    assert b"group 1 has no rows" in L.ln3_last_error()
    rg[1] = rg[2] = 1
    a.n_per_sample = 6
    assert L.ln3_ode_step(ctypes.byref(a), None) == -1                        # not a multiple of 4
    a.n_per_sample = 64
    a.y = fake + 4
    assert L.ln3_ode_stage(ctypes.byref(a), 1, None) == -1                    # misaligned
    a.y = fake
    assert L.ln3_ode_stage(ctypes.byref(a), 7, None) == -1
    a.workspace_bytes = 8
    assert L.ln3_ode_initial_step(ctypes.byref(a), 0, None) == -1
