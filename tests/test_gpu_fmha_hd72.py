"""GPU (-m gpu): the flash-attention kernel at head_dim 72 (DiT-XL/2: 1152 / 16 heads) element by element against a
float64 reference, on the XL self-attention shape (packed strided qkv), cross-attention to the 77 text tokens and the
edges of the tiling (ragged Lq / Lkv, one query, one key, a large B·H).

The bound is test_gpu_fmha_kernel.py's (see its docstring) with 72 products per S entry: the kernel pads the
contraction to 80 with exact zeros, which add exactly 0 to the fp32 sum, so d_j = c 72 2^-23 sum_d |q_d k_jd| + ...
Every output is a view inside a NaN-filled buffer whose bytes outside the view must keep their bits, and every case
is launched three times with bit-identical results."""
import pytest
import torch

from fmha_reference_hd import fmha_reference_hd
from kernel_bounds import ulp

pytestmark = pytest.mark.gpu

HD = 72
PAD = 256


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def guarded_out(B, Lq, D, ldo, bs, dev):
    flat = torch.full((2 * PAD + B * bs,), float("nan"), dtype=torch.bfloat16, device=dev)
    return flat, flat.as_strided((B, Lq, D), (bs, ldo, 1), PAD)


def make_inputs(dev, B, H, Lq, Lkv, layout, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    D = H * HD
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g).bfloat16()
    if layout == "packed":       # q / k / v column slices of one (B, L, 3 D) buffer: (B, N, 3, H, 72)
        qkv = rnd(B, max(Lq, Lkv), 3 * D)
        return qkv[:, :Lq, :D], qkv[:, :Lkv, D:2 * D], qkv[:, :Lkv, 2 * D:]
    kv = rnd(B, Lkv, 3, 2, D)    # K / V inside a wider per-layer cache
    return rnd(B, Lq, D), kv[:, :, 1, 0], kv[:, :, 1, 1]


def run(dev, q, k, v, H, *, causal=False, ldo=None, sub_batch=False):
    from ln3diff_b200 import ops
    B, Lq, D = q.shape
    ldo = D if ldo is None else ldo
    bs = Lq * ldo
    if sub_batch:
        flat, full = guarded_out(B + 2, Lq, D, ldo, bs, dev)
        out = full[1:B + 1]
    else:
        flat, out = guarded_out(B, Lq, D, ldo, bs, dev)
    before = flat.view(torch.int16).clone()
    results = []
    for _ in range(3):
        ops.fmha(q, k, v, H, out=out, causal=causal)
        torch.cuda.synchronize()
        results.append(out.clone())
    for r in results[1:]:
        assert torch.equal(r.view(torch.int16), results[0].view(torch.int16)), "launches differ"
    inside = torch.zeros(flat.numel(), dtype=torch.bool, device=dev)
    inside.as_strided(tuple(out.shape), out.stride(), out.storage_offset()).fill_(True)
    changed = (flat.view(torch.int16) != before) & ~inside
    assert not bool(changed.any()), f"{int(changed.sum())} elements outside the output view were written"
    return results[0]


def check(dev, B, H, Lq, Lkv, *, layout="cache", causal=False, ldo=None, sub_batch=False, seed=0):
    q, k, v = make_inputs(dev, B, H, Lq, Lkv, layout, seed)
    got = run(dev, q, k, v, H, causal=causal, ldo=ldo, sub_batch=sub_batch)
    ref, tol = fmha_reference_hd(q, k, v, H, HD, HD ** -0.5, causal)
    bound = ulp(ref.abs() + tol, 7) / 2 + tol
    err = (got.to(torch.float64) - ref).abs()
    bad = ~(err <= bound)
    what = f"B={B} H={H} Lq={Lq} Lkv={Lkv} causal={causal} layout={layout}"
    if bool(bad.any()):
        i = int(torch.where(bad, err / bound.clamp_min(1e-300), torch.zeros_like(err)).nan_to_num(float("inf"))
                .flatten().argmax())
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} out of bound; worst at flat {i}: got "
                             f"{got.flatten()[i].item()!r} expected {ref.flatten()[i].item()!r} "
                             f"bound {bound.flatten()[i].item():.3e}")
    return q, k, v, got


def test_xl_self_attention(dev):
    """DiT-XL/2 self-attention: 768 tokens x 16 heads of 72, q / k / v slices of the packed (B, N, 3, H, 72) qkv."""
    check(dev, 8, 16, 768, 768, layout="packed")


def test_cross_attention_77_tokens(dev):
    """Cross-attention to 77 tokens (one ragged key block), K / V strided inside a cache, output a sub-batch view."""
    check(dev, 4, 16, 768, 77, sub_batch=True)


@pytest.mark.parametrize("B,H,Lq,Lkv", [
    (2, 3, 1, 1),               # one query, one key
    (2, 3, 1, 300),             # one query
    (2, 3, 300, 1),             # one key
    (3, 4, 200, 333),           # neither a multiple of the tile
    (2, 4, 129, 129),           # one row / key past a tile
    (1, 2, 640, 1000),          # several query tiles and key blocks
])
def test_ragged(dev, B, H, Lq, Lkv):
    check(dev, B, H, Lq, Lkv)


@pytest.mark.parametrize("B,H,Lq,Lkv", [(4096, 1, 3, 5), (2, 2048, 2, 130), (300, 16, 130, 64)])
def test_large_batch_and_heads(dev, B, H, Lq, Lkv):
    check(dev, B, H, Lq, Lkv)


def test_causal(dev):
    check(dev, 2, 4, 300, 300, causal=True, seed=3)


def test_output_pitch(dev):
    """An output pitch wider than H 72 (a multiple of 8 elements)."""
    check(dev, 3, 16, 300, 200, ldo=16 * HD + 8)


def test_padding_does_not_read_the_next_head(dev):
    """Head h's tail step reads columns 64..71 of head h and exact zeros for 72..79: filling every other head's
    columns of q, k and v with huge values must leave head h's output bit for bit as it was."""
    from ln3diff_b200 import ops
    B, H, L, h = 2, 4, 200, 1
    q, k, v = make_inputs(dev, B, H, L, L, "packed", seed=9)
    base = run(dev, q, k, v, H)
    cols = torch.ones(H * HD, dtype=torch.bool, device=dev)
    cols[h * HD:(h + 1) * HD] = False
    q2, k2, v2 = (t.clone() for t in (q, k, v))
    for t in (q2, k2, v2):
        t[:, :, cols] = 3.0e4
    got = run(dev, q2, k2, v2, H)
    sl = slice(h * HD, (h + 1) * HD)
    assert torch.equal(got[:, :, sl].view(torch.int16), base[:, :, sl].view(torch.int16))
    assert not torch.equal(got, base)
    # and the same holds when the huge values sit in the very next head only
    q3, k3, v3 = (t.clone() for t in (q, k, v))
    for t in (q3, k3, v3):
        t[:, :, (h + 1) * HD:(h + 2) * HD] = -3.0e4
    got3 = ops.fmha(q3, k3, v3, H)
    assert torch.equal(got3[:, :, sl].view(torch.int16), base[:, :, sl].view(torch.int16))


def test_second_source_refused(dev):
    """A second K/V source is implemented for 64-wide heads only."""
    from ln3diff_b200 import ops
    q, k, v = make_inputs(dev, 1, 2, 10, 10, "cache", 0)
    with pytest.raises(RuntimeError, match="head_dim 64"):
        ops.fmha(q, k, v, 2, k2=k, v2=v)
