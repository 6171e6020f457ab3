"""GPU (-m gpu): the wgmma GEMM when its A operand is larger than the L2, element by element against float64 with the
references and tolerances of test_gpu_gemm_kernel.py.

Such a GEMM (the MLP's fc2 at bench.py's batch has a 100 MB A) walks its tiles N first instead of M first inside each
N panel; every output element must come out as on any other walk.  The cases have a partial last tile row and every
output kind."""
import pytest
import torch

from test_gpu_gemm_kernel import dev, run_case  # noqa: F401  (dev is a fixture)

pytestmark = pytest.mark.gpu

M, N, K = 12345, 384, 4096   # A: 101 MB of bf16; W: 3 MB


@pytest.fixture(scope="module")
def large_a(dev):  # noqa: F811
    l2 = torch.cuda.get_device_properties(dev).L2_cache_size
    assert 2 * M * K > l2 and 2 * N * K <= l2 // 2, "the case must take the N-first walk"
    return dev


def test_large_a_bf16(large_a):
    run_case(large_a, M, N, K)


def test_large_a_gelu(large_a):
    run_case(large_a, M, N, K, act=1, seed=1)


def test_large_a_f32_output(large_a):
    from ln3diff_b200 import ops
    run_case(large_a, M, N, K, out_kind=ops.OUT_F32, seed=2)


def test_large_a_gated_residual(large_a):
    from ln3diff_b200 import ops
    run_case(large_a, M, N, K, out_kind=ops.OUT_RESID_F32, gate_rows=768, out2=True, seed=3)
