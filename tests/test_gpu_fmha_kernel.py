"""GPU (-m gpu): the wgmma flash-attention kernel (ops.fmha -> attention_wgmma.cu) element by element against a
float64 reference, on the shapes the project runs and the edges of the tiling (ragged Lq / Lkv, one query or one
key, causal block skip, a second K/V source, strided views, a large B·H).

The bound is derived from the kernel's arithmetic, per output element y = sum_j p_j v_j / sum_j p_j with
p_j = 2^(s_j c - m) (c = scale log2 e):
  e_j   relative error of the kernel's unrounded p_j: an absolute error d_j of the exponent gives ln2 d_j, where
        d_j = c 64 2^-23 sum_d |q_d k_jd| (fp32 accumulation of the 64 exact bf16 products of S)
            + 2^-22 (|s_j c| + |m|)    (the fp32 constant c, the rounded product s c and the subtraction of m:
                                        2^-24 (3 |s_j c| + 2 |m|))
        plus the ex2.approx error, taken as 2^-21 relative.  The running-max rescale multiplies numerator and
        denominator by the same factor alpha, so alpha's own error cancels in the ratio.
  num   P is rounded to bf16 before P V while the row sum l adds the unrounded values.  bf16 keeps 8 significant
        bits, so round-to-nearest is off by up to 2^-8 relative (half an ulp just above a power of two):
        |d num| <= sum_j p_j |v_j| (e_j + 2^-8 (1 + e_j)) + n_acc 2^-23 sum_j p_j |v_j| (1 + e_j + 2^-8)
  den   |d l| <= sum_j p_j e_j + n_acc 2^-23 sum_j p_j (1 + e_j)
        n_acc = Lkv_total + 2 nblocks: one fp32 add per key (one ulp: allows a tensor core that truncates) and
        one rescale product per 128-key block in each of the accumulators.
  y     (|d num| + |y| |d l|) / (l - |d l|), plus two roundings (1/l and the product: 2^-23 |y|), and the final
        bf16 rounding: half a bf16 ulp at |y| + tol.
Every output is a view inside a NaN-filled buffer whose bytes outside the view must keep their bits, and every
case is launched three times with bit-identical results."""
import pytest
import torch

from kernel_bounds import fmha_reference as reference
from kernel_bounds import ulp

pytestmark = pytest.mark.gpu

PAD = 256            # NaN elements before and after every output view (512 B of bf16 keeps 16-byte alignment)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def guarded_out(B, Lq, D, ldo, bs, dev):
    """(flat, view): a (B, Lq, D) view with row pitch ldo and batch stride bs inside a NaN-filled buffer."""
    flat = torch.full((2 * PAD + B * bs,), float("nan"), dtype=torch.bfloat16, device=dev)
    return flat, flat.as_strided((B, Lq, D), (bs, ldo, 1), PAD)


def run_case(dev, B, H, Lq, Lkv, *, Lkv2=0, causal=False, layout="packed", ldo=None, sub_batch=False,
             qscale=1.0, seed=0):
    from ln3diff_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    D = H * 64
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g).bfloat16()
    if layout == "packed":       # q / k / v column slices of one (B, L, 3 D) buffer (DiT self-attention)
        qkv = rnd(B, max(Lq, Lkv), 3 * D)
        if qscale != 1.0:
            qkv[:, :, :D] *= qscale
        q, k, v = qkv[:, :Lq, :D], qkv[:, :Lkv, D:2 * D], qkv[:, :Lkv, 2 * D:]
    else:                        # K / V of one layer inside a (B, Lkv, 3, 2, D) cache (DiT cross-attention)
        q = rnd(B, Lq, D) * qscale
        kv = rnd(B, Lkv, 3, 2, D)
        k, v = kv[:, :, 1, 0], kv[:, :, 1, 1]
    k2 = v2 = None
    if Lkv2:
        dkv = rnd(B, Lkv2, 2 * D)
        k2, v2 = dkv[:, :, :D], dkv[:, :, D:]
    ldo = D if ldo is None else ldo
    bs = Lq * ldo
    if sub_batch:                # att3[g0:g1]: the view starts one sample into a wider batch
        flat, full = guarded_out(B + 2, Lq, D, ldo, bs, dev)
        out = full[1:B + 1]
    else:
        flat, out = guarded_out(B, Lq, D, ldo, bs, dev)
    before = flat.view(torch.int16).clone()

    results = []
    for _ in range(3):
        ops.fmha(q, k, v, H, out=out, k2=k2, v2=v2, causal=causal)
        torch.cuda.synchronize()
        results.append(out.clone())
    what = f"B={B} H={H} Lq={Lq} Lkv={Lkv}+{Lkv2} causal={causal} layout={layout} ldo={ldo}"
    for r in results[1:]:
        assert torch.equal(r.view(torch.int16), results[0].view(torch.int16)), f"{what}: launches differ"
    inside = torch.zeros(flat.numel(), dtype=torch.bool, device=dev)
    inside.as_strided(tuple(out.shape), out.stride(), out.storage_offset()).fill_(True)
    changed = (flat.view(torch.int16) != before) & ~inside
    assert not bool(changed.any()), f"{what}: {int(changed.sum())} elements outside the output view were written"

    kk = torch.cat([k, k2], 1) if Lkv2 else k
    vv = torch.cat([v, v2], 1) if Lkv2 else v
    ref, tol = reference(q, kk, vv, H, 64 ** -0.5, causal)
    bound = ulp(ref.abs() + tol, 7) / 2 + tol
    got = results[0]
    err = (got.to(torch.float64) - ref).abs()
    bad = ~(err <= bound)                                  # NaN counts as out of bound
    if bool(bad.any()):
        i = int(torch.where(bad, err / bound.clamp_min(1e-300), torch.zeros_like(err)).nan_to_num(float("inf"))
                .flatten().argmax())
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} out of bound; worst at flat {i}: got "
                             f"{got.flatten()[i].item()!r} expected {ref.flatten()[i].item()!r} "
                             f"bound {bound.flatten()[i].item():.3e}")


# ------------------------------------------------------------------ the shapes the project runs
def test_bench_self_attention(dev):
    """dit_trilatent.py: 16 samples x 16 heads x 768 tokens, q / k / v slices of the packed qkv buffer."""
    run_case(dev, 16, 16, 768, 768)


def test_bench_cross_attention(dev):
    """The conditional half's cross-attention to 77 tokens: K / V strided per layer, output a sub-batch view."""
    run_case(dev, 8, 16, 768, 77, layout="cache", sub_batch=True)


@pytest.mark.parametrize("B,H,Lq,Lkv,Lkv2", [
    (8, 16, 768, 256, 0),       # PixArt cross-attention
    (8, 16, 768, 1536, 0),      # MV23D cross-attention
    (4, 16, 768, 768, 257),     # self-attention with a second K/V source (dit/_denoiser.py)
    (12, 16, 256, 256, 0),      # DiT2 decoder, in-plane attention (3 B x 256 tokens)
    (4, 16, 768, 768, 0),       # DiT2 decoder, global attention
])
def test_model_shapes(dev, B, H, Lq, Lkv, Lkv2):
    run_case(dev, B, H, Lq, Lkv, Lkv2=Lkv2, layout="cache" if Lkv != Lq else "packed")


def test_clip_causal(dev):
    """CLIP text tower: 8 prompts x 12 heads x 77 tokens, causal."""
    run_case(dev, 8, 12, 77, 77, causal=True)


# ------------------------------------------------------------------ edges of the tiling
@pytest.mark.parametrize("B,H,Lq,Lkv", [
    (2, 3, 1, 1),               # one query, one key
    (2, 3, 1, 300),             # one query
    (2, 3, 300, 1),             # one key
    (3, 4, 200, 333),           # neither a multiple of the tile
    (3, 4, 333, 100),           # Lkv < 128
    (2, 4, 129, 129),           # one row / key past a tile
    (1, 2, 640, 1000),          # several query tiles and key blocks, ragged last block
])
def test_ragged(dev, B, H, Lq, Lkv):
    run_case(dev, B, H, Lq, Lkv, layout="cache")


@pytest.mark.parametrize("B,H,L", [(2, 12, 77), (2, 4, 300), (1, 2, 640)])
def test_causal(dev, B, H, L):
    """Lq = Lkv = 77 (one block), and Lq > 128: rows of later tiles skip no block, earlier tiles skip the tail."""
    run_case(dev, B, H, L, L, causal=True, seed=L)


@pytest.mark.parametrize("L1,L2", [(200, 77), (77, 200), (1, 1), (256, 129)])
def test_second_kv_source(dev, L1, L2):
    """Both sources have ragged ends; the second source's blocks follow the first's."""
    run_case(dev, 2, 4, 300, L1, Lkv2=L2, layout="cache")


@pytest.mark.parametrize("ldo,sub_batch", [(1024 + 64, False), (1024 + 8, True)])
def test_output_views(dev, ldo, sub_batch):
    """An output pitch wider than H 64, and a sub-batch view inside a wider batch."""
    run_case(dev, 3, 16, 300, 200, ldo=ldo, sub_batch=sub_batch, layout="cache")


def test_peaked_scores(dev):
    """Large logits: the running max moves often and most probabilities underflow."""
    run_case(dev, 2, 4, 384, 700, qscale=6.0)


@pytest.mark.parametrize("B,H,Lq,Lkv", [(65535, 1, 3, 5), (2, 4096, 2, 130), (300, 16, 130, 64)])
def test_large_batch_and_heads(dev, B, H, Lq, Lkv):
    run_case(dev, B, H, Lq, Lkv, layout="cache")
