"""GPU (-m gpu): the kernels of decoder_conv.cu -- ln3_conv_nhwc (fp32 SIMT and TF32 mma.sync, both output-channel
tiles), ln3_groupnorm_stats, ln3_attn_single_head and ln3_patch_embed_triplane -- element by element against float64
references computed on the device, on the production shapes of the VAE decoder's conv tail and the MVEncoder and on
the edges of the tiling; then the whole conv_sr tail against the oracle's ldm Decoder.

Bounds are derived from each kernel's arithmetic with u = 2^-24 (an fp32 ulp is at most 2u of the value); each is
stated in the docstring of the function that computes it.  Every case launches at least twice with bit-identical
results, and every output lies inside a NaN-filled buffer whose bytes outside the output must keep their bits.  Every
case with an index mapping (image, pixel, group) also shows that a reference with the mapping wrong lands well outside
the bound, so the bound is tight enough to see that slip."""
import ctypes as C
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from kernel_bounds import _swish_tol, attn_reference, conv_reference, gn_reference, pet_reference

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
PAD = 1024                # guard elements before and after every output


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def _pack(w):
    """Conv2d weight (Cout, Cin, k, k) -> the kernels' [k*k, Cin, Cout]."""
    return w.permute(2, 3, 1, 0).reshape(-1, w.shape[1], w.shape[0]).contiguous()


def _guarded(n, dev, dtype=torch.float32):
    """(buf, flat view of n elements) inside a NaN-filled buffer."""
    buf = torch.full((n + 2 * PAD,), float("nan"), device=dev, dtype=dtype)
    return buf, buf[PAD:PAD + n]


def _guards_intact(buf, before):
    """The bytes outside the output are the NaN fill they started as."""
    iv, bv = buf.view(torch.int16), before.view(torch.int16)
    k = PAD * buf.element_size() // 2
    return torch.equal(iv[:k], bv[:k]) and torch.equal(iv[-k:], bv[-k:])


RATIOS = {}   # kernel / precision -> the largest error / bound ratio seen in this run


@pytest.fixture(scope="module", autouse=True)
def _report_ratios():
    yield
    for k, r in sorted(RATIOS.items()):
        print(f"largest error / bound: {k:28s} {r:.3e}")


def _check(got, ref, tol, what):
    err = (got.double() - ref).abs()
    ratio = float((err / tol).max())
    assert bool((err <= tol).all()), f"{what}: max err/bound {ratio:.3g}"
    RATIOS[what] = max(RATIOS.get(what, 0.0), ratio)
    return ratio


# ------------------------------------------------------------------ ln3_conv_nhwc
# (N, Hin, Win, Cin, Cout, ksize, upsample, gn, swish, bias, residual)
DEC = {                                                    # the conv_sr tail of the VAE decoder
    "conv_in384": (16, 16, 384, 128, 3, False, False, False, True, False),
    "conv_in1024": (16, 16, 1024, 128, 3, False, False, False, True, False),
    "res16": (16, 16, 128, 128, 3, False, True, True, True, False),
    "up16to32": (16, 16, 128, 128, 3, True, False, False, True, False),
    "res32_128to64": (32, 32, 128, 64, 3, False, True, True, True, False),
    "nin32_128to64": (32, 32, 128, 64, 1, False, False, False, True, False),
    "up64to128": (64, 64, 64, 64, 3, True, False, False, True, False),
    "res128_64to32": (128, 128, 64, 32, 3, False, True, True, True, True),
    "conv_out": (128, 128, 32, 32, 3, False, True, True, True, False),
    "qkv1x1": (16, 16, 128, 128, 1, False, True, False, True, False),
    "proj_out1x1": (16, 16, 128, 128, 1, False, False, False, True, True),
}
ENC = {                                                    # the MVEncoder, 4 views
    "enc_conv_in": (256, 256, 10, 64, 3, False, False, False, True, False),
    "enc_res256": (256, 256, 64, 64, 3, False, True, True, True, True),
    "enc_proj_in": (32, 32, 256, 512, 1, False, True, False, True, False),
    "enc_proj_out": (32, 32, 512, 256, 1, False, False, False, True, True),
    "enc_conv_out": (32, 32, 256, 24, 3, False, True, True, True, False),
    "enc_fusion": (32, 32, 96, 24, 3, False, False, False, True, False),
}
EDGE = {
    "1x1px": (3, 1, 1, 17, 40, 3, False, True, True, True, False),
    "1x1px_up": (2, 1, 1, 10, 72, 3, True, True, True, True, True),
    "7x9": (2, 7, 9, 48, 5, 3, False, True, True, False, False),
    "7x9_up": (3, 7, 9, 1, 24, 3, True, False, False, True, True),
    "20x24": (2, 20, 24, 48, 40, 3, False, True, True, True, True),
    "20x24_up": (2, 20, 24, 48, 40, 3, True, False, False, True, True),
    "20x24_cout32_nobias": (2, 20, 24, 48, 32, 3, False, False, False, False, False),
    "33x17": (3, 33, 17, 17, 72, 3, False, True, True, False, True),
    "33x17_cin1": (2, 33, 17, 1, 5, 3, False, False, False, True, False),
    "34x18_up": (2, 17, 9, 10, 72, 3, True, True, True, True, False),
    "1x1k_7x9": (3, 7, 9, 17, 72, 1, False, True, False, False, True),
    "1x1k_20x24_nobias": (2, 20, 24, 48, 40, 1, False, False, False, False, False),
    "1x1k_33x17_up": (2, 33, 17, 48, 5, 1, True, True, True, True, False),
}
CASES = ([(f"dec{n}_{k}", n) + v for n in (3, 24) for k, v in DEC.items()]
         + [(k, 4) + v for k, v in ENC.items()] + [(k,) + v for k, v in EDGE.items()])
CASES_3x3 = [c for c in CASES if c[6] == 3]


def _conv_operands(N, Hin, Win, Cin, Cout, ksize, up, gn, bias, residual, seed, zlow=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, Hin, Win, Cin, generator=g)
    w = torch.randn(Cout, Cin, ksize, ksize, generator=g) / math.sqrt(ksize * ksize * Cin)
    b = 0.1 * torch.randn(Cout, generator=g) if bias else None
    sc = sh = None
    if gn:                                                 # a different GroupNorm scale / shift for every image
        sc = 1 + 0.5 * torch.randn(N, Cin, generator=g)
        sh = torch.randn(N, Cin, generator=g)
        if zlow:                                           # pre-swish values down to about -100 (-> __expf overflow)
            sh = sh - 100 * torch.rand(N, Cin, generator=g)
            sh[:, 0] = -100.0
    H, W = (2 * Hin, 2 * Win) if up else (Hin, Win)
    res = torch.randn(N, H, W, Cout, generator=g) if residual else None
    return x, w, b, sc, sh, res


def _run_conv(dev, x, w, b, sc, sh, res, *, ksize, up, swish, tf32):
    """Two launches into a guarded buffer: (out NHWC, tile)."""
    from ln3diff_b200 import ops
    N, Hin, Win, _ = x.shape
    Cout = w.shape[0]
    H, W = (2 * Hin, 2 * Win) if up else (Hin, Win)
    n = N * H * W * Cout
    buf, flat = _guarded(n, dev)
    before = buf.clone()
    out = flat.view(N, H, W, Cout)
    args = (x.to(dev), _pack(w).to(dev), None if b is None else b.to(dev))
    kw = dict(ksize=ksize, upsample=up, gn=None if sc is None else (sc.to(dev), sh.to(dev)), swish=swish,
              residual=None if res is None else res.to(dev), out=out, tf32=tf32)
    ops.conv_nhwc(*args, **kw)
    first = out.clone()
    ops.conv_nhwc(*args, **kw)
    torch.cuda.synchronize()
    assert torch.equal(first, out)                                              # bit-identical launches
    assert _guards_intact(buf, before)
    assert not bool(out.isnan().any())
    return out, ops.conv_cout_tile(N, H, W, Cout)


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
@pytest.mark.parametrize("name,N,Hin,Win,Cin,Cout,ksize,up,gn,swish,bias,residual",
                         CASES, ids=[c[0] for c in CASES])
def test_conv_elementwise(dev, name, N, Hin, Win, Cin, Cout, ksize, up, gn, swish, bias, residual, tf32):
    if tf32 and ksize == 1:
        pytest.skip("ops.conv_nhwc runs 1x1 convs in fp32 whatever tf32 says")
    x, w, b, sc, sh, res = _conv_operands(N, Hin, Win, Cin, Cout, ksize, up, gn, bias, residual,
                                          seed=zlib.crc32(name.encode()) % 10007)
    out, _ = _run_conv(dev, x, w, b, sc, sh, res, ksize=ksize, up=up, swish=swish, tf32=tf32)
    d = lambda t: None if t is None else t.to(dev)
    ref, tol = conv_reference(x.to(dev), w.to(dev), d(b), ksize=ksize, up=up, sc=d(sc), sh=d(sh), swish=swish,
                              res=d(res), tf32=tf32)
    _check(out.permute(0, 3, 1, 2), ref, tol, f"conv {('tf32' if tf32 else 'fp32')}")
    # a reference that maps the pixels or the images wrong moves the outputs far beyond the bound (checked on the
    # first two images): by more than 10x for the median output (the fp32 bound of conv_in's K = 9216 terms is only
    # ~40x below a typical output)
    margin = 10
    first2 = lambda t: None if t is None else t[:2].to(dev)
    x2, sc2, sh2, res2 = x[:2], first2(sc), first2(sh), first2(res)
    ref2, tol2 = ref[:2], tol[:2]
    if Hin * Win > 1 and (up or ksize == 3):
        xs = torch.roll(x2, 1, dims=2) if Win > 1 else torch.roll(x2, 1, dims=1)    # input one pixel over
        ref_s, _ = conv_reference(xs.to(dev), w.to(dev), d(b), ksize=ksize, up=up, sc=sc2, sh=sh2, swish=swish,
                                  res=res2, tf32=tf32)
        assert float(((ref_s - ref2).abs() / tol2).median()) > margin, "pixel mapping"
    if gn and N > 1:
        sc0, sh0 = sc2[:1].expand_as(sc2).contiguous(), sh2[:1].expand_as(sh2).contiguous()   # image 0's sc / sh
        ref_0, _ = conv_reference(x2.to(dev), w.to(dev), d(b), ksize=ksize, up=up, sc=sc0, sh=sh0, swish=swish,
                                  res=res2, tf32=tf32)
        assert float(((ref_0 - ref2)[1:].abs() / tol2[1:]).median()) > margin, "per-image GroupNorm mapping"


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
@pytest.mark.parametrize("ksize,up", [(3, False), (3, True), (1, False)])
def test_conv_swish_deep_negative_preactivation(dev, ksize, up, tf32):
    """Pre-swish values down to about -100: __expf(-v) overflows below -88.7 and the kernel's swish returns -0."""
    if tf32 and ksize == 1:
        pytest.skip("ops.conv_nhwc runs 1x1 convs in fp32 whatever tf32 says")
    N, Hin, Win, Cin, Cout = 3, 12, 10, 24, 40
    x, w, b, sc, sh, res = _conv_operands(N, Hin, Win, Cin, Cout, ksize, up, True, True, False, seed=77, zlow=True)
    out, _ = _run_conv(dev, x, w, b, sc, sh, res, ksize=ksize, up=up, swish=True, tf32=tf32)
    z = x.double() * sc.double()[:, None, None, :] + sh.double()[:, None, None, :]
    assert float(z.min()) < -95 and float((z < -88.8).double().mean()) > 0.05       # the overflow branch is taken
    ref, tol = conv_reference(x.to(dev), w.to(dev), b.to(dev), ksize=ksize, up=up, sc=sc.to(dev), sh=sh.to(dev),
                              swish=True, tf32=tf32)
    _check(out.permute(0, 3, 1, 2), ref, tol, f"conv {('tf32' if tf32 else 'fp32')} (z to -100)")


def _tile_threshold_N(Cout, H, W):
    """The smallest N for which 64-channel CTAs give at least two per SM (conv_nhwc's rule)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per_image = ((H + 7) // 8) * ((W + 7) // 8) * ((Cout + 63) // 64)
    return -(-2 * sms // per_image)


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
@pytest.mark.parametrize("side", ["below", "at"])
def test_conv_tile_threshold(dev, side, tf32):
    """Shapes on both sides of the 2 x SM-count rule: 32-channel CTAs just below it, 64-channel CTAs at it; Cout = 72
    leaves a tail in both tiles."""
    Hin = Win = 16
    Cout = 72
    N = _tile_threshold_N(Cout, Hin, Win) - (1 if side == "below" else 0)
    x, w, b, sc, sh, res = _conv_operands(N, Hin, Win, 20, Cout, 3, False, True, True, True, seed=5)
    out, tile = _run_conv(dev, x, w, b, sc, sh, res, ksize=3, up=False, swish=True, tf32=tf32)
    assert tile == (32 if side == "below" else 64)
    ref, tol = conv_reference(x.to(dev), w.to(dev), b.to(dev), ksize=3, up=False, sc=sc.to(dev), sh=sh.to(dev),
                              swish=True, res=res.to(dev), tf32=tf32)
    _check(out.permute(0, 3, 1, 2), ref, tol, f"conv {('tf32' if tf32 else 'fp32')}")


def test_conv_cases_cover_both_tiles(dev):
    """The fp32 and the TF32 case lists each run both templates (32- and 64-channel CTAs) on this device."""
    from ln3diff_b200 import ops

    def tiles(cases):
        return {ops.conv_cout_tile(c[1], c[2] * (2 if c[7] else 1), c[3] * (2 if c[7] else 1), c[5]) for c in cases}
    assert tiles(CASES) == {32, 64}
    assert tiles(CASES_3x3) == {32, 64}
    assert tiles([c for c in CASES if c[6] == 1]) == {32, 64}


# ------------------------------------------------------------------ ln3_groupnorm_stats
def _gn_call(x, gamma, beta, G, eps=1e-6):
    """ln3_groupnorm_stats through the C ABI with scale / shift inside guarded buffers; two launches."""
    from ln3diff_b200 import _lib
    N, H, W, Cc = x.shape
    lib = _lib.lib()
    outs = []
    for _ in range(2):
        bsc, sc = _guarded(N * Cc, x.device)
        bsh, sh = _guarded(N * Cc, x.device)
        before = bsc.clone()
        rc = lib.ln3_groupnorm_stats(C.c_void_p(x.data_ptr()), C.c_void_p(gamma.data_ptr()),
                                     C.c_void_p(beta.data_ptr()), N, H * W, Cc, G, C.c_float(eps),
                                     C.c_void_p(sc.data_ptr()), C.c_void_p(sh.data_ptr()), _lib.current_stream())
        assert rc == 0, lib.ln3_last_error().decode()
        torch.cuda.synchronize()
        assert _guards_intact(bsc, before) and _guards_intact(bsh, before)
        outs.append((sc.view(N, Cc).clone(), sh.view(N, Cc).clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    return outs[0]


def _gn_operands(N, H, W, Cc, G, seed, dc=0.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, Cc, generator=g) * (0.5 + torch.rand(N, 1, 1, Cc, generator=g))
    x = x + 0.5 * torch.randn(N, 1, 1, Cc, generator=g)          # a different mean for every image and channel
    if dc:
        x = x + dc                                                # mean = dc x the standard deviation (~1)
    gamma = 1 + 0.3 * torch.randn(Cc, generator=g)
    beta = 0.3 * torch.randn(Cc, generator=g)
    return x, gamma, beta


GN_CASES = [   # (N, H, W, C, G, dc)
    pytest.param(2, 16, 16, 32, 32, 0.0, id="cpg1_cnt256"),
    pytest.param(3, 16, 16, 64, 32, 0.0, id="cpg2_cnt512"),
    pytest.param(3, 16, 16, 128, 32, 0.0, id="cpg4_dec16"),
    pytest.param(2, 32, 32, 128, 32, 0.0, id="cpg4_dec32"),
    pytest.param(2, 128, 128, 32, 32, 0.0, id="cpg1_dec128"),
    pytest.param(4, 256, 256, 64, 32, 0.0, id="cpg2_enc256"),
    pytest.param(3, 8, 8, 64, 8, 0.0, id="cpg8_cnt512"),
    pytest.param(2, 20, 24, 48, 8, 0.0, id="cpg6_20x24"),          # widths that are not powers of two
    pytest.param(3, 16, 16, 96, 32, 0.0, id="cpg3_dec16"),
    pytest.param(2, 7, 9, 240, 20, 1e3, id="dc1e3_cpg12"),
    pytest.param(2, 3, 5, 256, 1, 0.0, id="cpg256_cnt3840"),
    pytest.param(2, 1, 1, 256, 1, 0.0, id="cpg256_cnt256"),
    pytest.param(3, 5, 7, 32, 32, 0.0, id="cpg1_cnt35"),
    pytest.param(2, 1, 1, 64, 32, 0.0, id="cpg2_cnt2"),
    pytest.param(3, 16, 16, 128, 32, 1e3, id="dc1e3_dec16"),
    pytest.param(2, 7, 9, 256, 16, 1e3, id="dc1e3_cpg16"),
]


@pytest.mark.parametrize("N,H,W,Cc,G,dc", GN_CASES)
def test_groupnorm_stats_elementwise(dev, N, H, W, Cc, G, dc):
    x, gamma, beta = _gn_operands(N, H, W, Cc, G, seed=N * 100 + H + Cc + G, dc=dc)
    xd, gd, bd = x.to(dev), gamma.to(dev), beta.to(dev)
    sc, sh = _gn_call(xd, gd, bd, G)
    sc_r, sh_r, tol_sc, tol_sh, _, _ = gn_reference(xd, gd, bd, G)
    _check(sc, sc_r, tol_sc, "groupnorm scale")
    _check(sh, sh_r, tol_sh, "groupnorm shift")
    # image n's statistics land in image n's row: image 0's rows for every image are far outside the bound
    sc0 = sc_r[:1].expand_as(sc_r)
    assert float(((sc0 - sc_r)[1:].abs() / tol_sc[1:]).median()) > 100
    cpg = Cc // G
    if 1 < cpg < Cc:
        # group g holds channels [g C/G, (g + 1) C/G): a reference that groups the channels strided instead is wrong
        perm = torch.arange(Cc, device=dev).reshape(cpg, G).T.flatten()      # strided group g -> positions of g
        inv = torch.argsort(perm)
        sc_s, _, _, _, _, _ = gn_reference(xd[..., perm].contiguous(), gd[perm], bd[perm], G)
        assert float(((sc_s[:, inv] - sc_r).abs() / tol_sc).median()) > 100


# ------------------------------------------------------------------ GroupNorm -> conv, composed
@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
@pytest.mark.parametrize("N,Hin,Win,Cin,Cout,G,dc", [
    pytest.param(3, 16, 16, 128, 128, 32, 0.0, id="dec16_128"),
    pytest.param(3, 32, 32, 128, 64, 32, 0.0, id="dec32_128to64"),
    pytest.param(2, 20, 24, 48, 40, 8, 0.0, id="20x24_cin48_g8"),     # 6 channels per group
    pytest.param(2, 16, 16, 128, 40, 32, 1e3, id="dc1e3"),
])
def test_groupnorm_then_conv_composed(dev, N, Hin, Win, Cin, Cout, G, dc, tf32):
    """groupnorm_stats then conv_nhwc(gn=..., swish=True) against conv(swish(F.group_norm(x))) entirely in float64.
    The kernel's pre-activation z = fmaf(x, sc_hat, sh_hat) differs from the exact x sc + sh by
    |x| |d sc| + |d sh| + u |z|, where |d sh| holds u |mu sc|: the cancellation of x sc against beta - mu sc when the
    group's mean is large.  That error then goes through swish and the conv as in conv_reference.  Both kernels run
    twice into guarded buffers (_gn_call, _run_conv)."""
    x, gamma, beta = _gn_operands(N, Hin, Win, Cin, G, seed=91 + Cout, dc=dc)
    g = torch.Generator().manual_seed(92 + Cout)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin)
    b = 0.1 * torch.randn(Cout, generator=g)
    xd, gd, bd = x.to(dev), gamma.to(dev), beta.to(dev)
    sc, sh = _gn_call(xd, gd, bd, G)
    out, _ = _run_conv(dev, x, w, b, sc.cpu(), sh.cpu(), None, ksize=3, up=False, swish=True, tf32=tf32)
    sc_r, sh_r, tol_sc, tol_sh, _, _ = gn_reference(xd, gd, bd, G)
    x64 = xd.double()
    dz = x64.abs() * tol_sc[:, None, None, :] + tol_sh[:, None, None, :]
    _, tol = conv_reference(xd, w.to(dev), b.to(dev), ksize=3, up=False, sc=sc_r, sh=sh_r, swish=True, tf32=tf32,
                            dz=dz)
    gnx = F.group_norm(x64.permute(0, 3, 1, 2), G, gd.double(), bd.double(), eps=1e-6)
    ref_full = F.conv2d(gnx * torch.sigmoid(gnx), w.to(dev).double(), b.to(dev).double(), padding=1)
    _check(out.permute(0, 3, 1, 2), ref_full, tol, f"groupnorm -> conv {('tf32' if tf32 else 'fp32')}")


# ------------------------------------------------------------------ ln3_attn_single_head
def _attn_call(q, k, v):
    """ln3_attn_single_head through the C ABI into a guarded buffer; two launches."""
    from ln3diff_b200 import _lib
    N, L, Cc = q.shape
    lib = _lib.lib()
    outs = []
    for _ in range(2):
        buf, out = _guarded(N * L * Cc, q.device)
        before = buf.clone()
        rc = lib.ln3_attn_single_head(C.c_void_p(q.data_ptr()), C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()),
                                      C.c_void_p(out.data_ptr()), N, L, Cc, _lib.current_stream())
        assert rc == 0, lib.ln3_last_error().decode()
        torch.cuda.synchronize()
        assert _guards_intact(buf, before)
        outs.append(out.view(N, L, Cc).clone())
    assert torch.equal(outs[0], outs[1])
    return outs[0]


def _attn_operands(N, L, Cc, kind, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(N, L, Cc, generator=g) for _ in range(3))
    if kind == "peaky":          # one key per query row dominates by logit gaps of ~50
        j = torch.randint(0, L, (N, L), generator=g)
        q = q + 50 * Cc ** 0.5 * k.gather(1, j[..., None].expand(N, L, Cc)) / (k.norm(dim=-1, keepdim=True)
                                                                          .gather(1, j[..., None]) ** 2)
    elif kind == "late_max":     # the row maximum sits in the last, partial key block: every earlier block rescales
        k[:, -1] = 3 * k[:, -1] / k[:, -1].norm(dim=-1, keepdim=True) * Cc ** 0.5
        q = q + 4 * k[:, -1:] / Cc ** 0.5
    elif kind == "uniform":      # identical keys: a uniform softmax, y = mean of v
        k[:] = k[:, :1]
    return q, k, v


ATTN_CASES = ([pytest.param(N, L, Cc, "rand", id=f"N{N}_L{L}_C{Cc}")
               for (N, L, Cc) in [(1, 1, 32), (3, 7, 64), (1, 8, 128), (3, 9, 32), (1, 31, 64), (3, 32, 128),
                                  (3, 33, 32), (1, 37, 32), (2, 5, 128), (3, 200, 64), (3, 256, 128), (24, 256, 128),
                                  (24, 33, 64)]]
              + [pytest.param(3, 256, 128, "peaky", id="peaky_L256"), pytest.param(3, 200, 64, "peaky", id="peaky_L200"),
                 pytest.param(3, 200, 128, "late_max", id="late_max_L200"),
                 pytest.param(3, 33, 32, "late_max", id="late_max_L33"),
                 pytest.param(3, 256, 128, "uniform", id="uniform_L256"),
                 pytest.param(1, 9, 64, "uniform", id="uniform_L9")])


@pytest.mark.parametrize("N,L,Cc,kind", ATTN_CASES)
def test_attn_single_head_elementwise(dev, N, L, Cc, kind):
    q, k, v = _attn_operands(N, L, Cc, kind, seed=N * 1000 + L + Cc + len(kind))
    q, k, v = q.to(dev), k.to(dev), v.to(dev)
    out = _attn_call(q, k, v)
    from ln3diff_b200 import ops
    assert torch.equal(ops.attn_single_head(q, k, v), out)               # the product entry point: the same bits
    y, tol = attn_reference(q, k, v)
    _check(out, y, tol, "attn")
    if kind == "peaky":
        assert float(torch.softmax((q.double() @ k.double().transpose(1, 2)) * Cc ** -0.5, -1).amax(-1).min()) > 0.99
    if kind == "late_max":
        s = q.double() @ k.double().transpose(1, 2)
        assert bool((s.argmax(-1) == L - 1).all())
    if kind == "uniform":
        assert float((y - v.double().mean(1, keepdim=True)).abs().max()) < 1e-9
    if N > 1 and kind != "uniform":      # image 0's K / V for every image lands far outside the bound
        y0, _ = attn_reference(q, k[:1].expand_as(k), v[:1].expand_as(v))
        assert float(((y0 - y)[1:].abs() / tol[1:]).median()) > 100


def test_attn_single_head_rejects_unsupported_width(dev):
    from ln3diff_b200 import _lib
    q = torch.zeros(1, 16, 48, device=dev)
    lib = _lib.lib()
    rc = lib.ln3_attn_single_head(*(C.c_void_p(q.data_ptr()) for _ in range(4)), 1, 16, 48, _lib.current_stream())
    assert rc == -3 and "C must be" in lib.ln3_last_error().decode()          # LN3_EUNSUPPORTED


# ------------------------------------------------------------------ ln3_patch_embed_triplane
def _pet_call(lat, w, b, in_mul, want_silu):
    """ln3_patch_embed_triplane through the C ABI into guarded buffers; two launches."""
    from ln3diff_b200 import _lib
    B, C3, S, _ = lat.shape
    Cz, E = C3 // 3, w.shape[0] // 3
    n = B * 3 * (S // 2) ** 2 * E
    lib = _lib.lib()
    outs = []
    for _ in range(2):
        bt, tok = _guarded(n, lat.device)
        bs, sb = _guarded(n, lat.device, torch.bfloat16)
        bt0, bs0 = bt.clone(), bs.clone()
        rc = lib.ln3_patch_embed_triplane(C.c_void_p(lat.data_ptr()), C.c_void_p(w.data_ptr()),
                                          C.c_void_p(b.data_ptr()) if b is not None else None, B, Cz, S, E,
                                          C.c_float(in_mul), C.c_void_p(tok.data_ptr()),
                                          C.c_void_p(sb.data_ptr()) if want_silu else None, _lib.current_stream())
        assert rc == 0, lib.ln3_last_error().decode()
        torch.cuda.synchronize()
        assert _guards_intact(bt, bt0)
        if want_silu:
            assert _guards_intact(bs, bs0)
        else:
            assert torch.equal(bs.view(torch.int16), bs0.view(torch.int16))    # no copy asked for: nothing written
        outs.append((tok.view(B, -1, E).clone(), sb.view(B, -1, E).clone()))
    assert torch.equal(outs[0][0], outs[1][0])
    if want_silu:
        assert torch.equal(outs[0][1].view(torch.int16), outs[1][1].view(torch.int16))
    return outs[0]


@pytest.mark.parametrize("B,Cz,S,E,bias,want_silu,in_mul", [
    pytest.param(2, 4, 32, 384, True, True, 0.96806, id="prod_S384_B2"),
    pytest.param(3, 4, 16, 128, True, True, 0.5, id="S16_E128_B3"),
    pytest.param(3, 4, 32, 1024, True, True, 0.96806, id="prod_L1024_B3"),
    pytest.param(2, 1, 2, 1, True, True, 1.0, id="Cz1_S2_E1"),
    pytest.param(3, 16, 34, 100, False, True, 0.5, id="Cz16_S34_E100_nobias"),
    pytest.param(2, 4, 32, 256, True, False, 0.96806, id="E256_nosilu"),
    pytest.param(1, 16, 2, 257, True, True, 0.96806, id="Cz16_E257"),
    pytest.param(3, 1, 34, 384, False, False, 1.0, id="Cz1_S34_nobias_nosilu"),
])
def test_patch_embed_triplane_elementwise(dev, B, Cz, S, E, bias, want_silu, in_mul):
    g = torch.Generator().manual_seed(B * 100 + Cz * 10 + S + E)
    lat = 2 * torch.randn(B, 3 * Cz, S, S, generator=g)
    w = torch.randn(3 * E, Cz, 2, 2, generator=g) / math.sqrt(4 * Cz)
    b = 0.3 * torch.randn(3 * E, generator=g) if bias else None
    lat, w = lat.to(dev), w.to(dev)
    b = b.to(dev) if b is not None else None
    tok, sb = _pet_call(lat, w, b, in_mul, want_silu)
    y, tol, silu, tol_s = pet_reference(lat, w, b, in_mul)
    assert tok.shape == y.shape == (B, 3 * (S // 2) ** 2, E)
    _check(tok, y, tol, "patch_embed tokens")
    if want_silu:
        _check(sb.float(), silu, tol_s, "patch_embed silu bf16")
    # the product entry point gives the same bits, and the oracle's restatement of the reference module gives the
    # float64 reference this test uses
    from ln3diff_b200 import ops
    from oracle import decoder as odec
    tok2, sb2 = ops.patch_embed_triplane(lat, w, b, in_mul=in_mul, want_silu_bf16=want_silu)
    assert torch.equal(tok2, tok)
    assert (sb2 is None) if not want_silu else torch.equal(sb2.view(torch.int16), sb.view(torch.int16))
    pre = "superresolution.ldm_upsample."
    sd = {pre + "proj.weight": w.double(), pre + "proj.bias": b.double() if b is not None else w.new_zeros(3 * E).double()}
    assert float((odec.patch_embed_triplane(sd, (lat * in_mul).double()) - y).abs().max()) <= 1e-12 * float(y.abs().max())
    # output channel o = 3e + n reads conv group o // E; a reference that reads group o % 3 (the plane) instead is
    # wrong far beyond the bound wherever the two differ
    P = S // 2
    xp = (lat * in_mul).double().reshape(B, 3, Cz, P, 2, P, 2).permute(0, 3, 5, 1, 2, 4, 6).reshape(B, P * P, 3, 4 * Cz)
    o = torch.arange(3 * E, device=dev)

    def tokens_with_group(grp):
        yc = torch.einsum("blok,ok->bol", xp[:, :, grp], w.double().reshape(3 * E, 4 * Cz))
        if b is not None:
            yc = yc + b.double()[None, :, None]
        return yc.reshape(B, E, 3, P * P).flatten(2).transpose(1, 2)            # B (3 h w) E
    assert float((tokens_with_group(o // E) - y).abs().max()) <= 1e-9 * float(y.abs().max())
    differs = ((o // E) != (o % 3)).reshape(E, 3).T.repeat_interleave(P * P, 0)     # (3 h w, E)
    if bool(differs.any()):
        ratio = (tokens_with_group(o % 3) - y).abs() / tol
        assert float(ratio[:, differs].median()) > 100


# A chained bound through 31 convolutions, 22 GroupNorms and the attention is not simply derivable, so this one is
# measured: max |out - ref| / max |ref| of the tail was at most 2.45e-6 (fp32) and 9.79e-4 (TF32) over B = 1 and 8 on an
# H100 80GB HBM3 (SXM, 700 W power limit); the bounds sit >= 10x above.  Each wiring slip below must move the
# reference by >= 10x the bound (measured: 56x to 123x the TF32 bound).
CONV_SR_BOUND = {False: 3e-5, True: 1e-2}


@pytest.fixture(scope="module")
def conv_sr_decoder(dev):
    from ln3diff_b200.utils import build_ae_decoder
    from oracle import fixtures as fx
    m = build_ae_decoder(fx.DECODER_ARCH)
    sd = m.state_dict()
    shapes = {k: tuple(v.shape) for k, v in sd.items() if k.startswith("superresolution.conv_sr")}
    sd.update(fx.decoder_state_dict(shapes))
    m.load_state_dict(sd)
    m = m.to(dev)
    sd64 = {k: v.to(dev, torch.float64) for k, v in m.state_dict().items() if k.startswith("superresolution.conv_sr")}
    return m, sd64


def _rel_max(a, ref):
    return float((a - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
def test_conv_sr_tail_vs_oracle(dev, conv_sr_decoder, monkeypatch, B, tf32):
    """The decoder's _conv_sr on fp32 tokens (3B, 16, 16, D = 384, DiT2-S/2) against oracle.decoder.ldm_decoder run
    in float64 on the same tokens with the same (random, oracle.fixtures) weights."""
    from oracle import decoder as odec
    m, sd64 = conv_sr_decoder
    g = torch.Generator().manual_seed(400 + B)
    tok = torch.randn(3 * B, 16, 16, 384, generator=g).to(dev)
    m.conv_tf32 = tf32
    try:
        out = m._conv_sr(tok)
        again = m._conv_sr(tok)
    finally:
        m.conv_tf32 = True
    torch.cuda.synchronize()
    assert out.shape == (3 * B, 128, 128, 32) and torch.equal(out, again)
    z = tok.double().permute(0, 3, 1, 2)
    ref = odec.ldm_decoder(sd64, z)
    err = _rel_max(out.permute(0, 3, 1, 2), ref)
    bound = CONV_SR_BOUND[tf32]
    print(f"conv_sr B={B} tf32={tf32}: max err / max |ref| = {err:.3e} (bound {bound:.0e})")
    assert err <= bound
    if B != 1:
        return
    pre = "superresolution.conv_sr."
    swapped = dict(sd64)
    for k in [k for k in sd64 if k.startswith(pre + "mid.block_1.")]:
        k2 = k.replace("mid.block_1.", "mid.block_2.")
        swapped[k], swapped[k2] = sd64[k2], sd64[k]
    k_for_q = dict(sd64)
    for s in ("weight", "bias"):
        k_for_q[f"{pre}mid.attn_1.q.{s}"] = sd64[f"{pre}mid.attn_1.k.{s}"]
    slips = {"mid blocks swapped": odec.ldm_decoder(swapped, z), "k weights for q": odec.ldm_decoder(k_for_q, z)}
    attn = odec._attnblock
    monkeypatch.setattr(odec, "_attnblock", lambda sd, p, x: attn(sd, p, x) - x)
    slips["attention residual dropped"] = odec.ldm_decoder(sd64, z)
    for name, alt in slips.items():
        d = _rel_max(alt, ref)
        print(f"conv_sr slip '{name}': {d:.3e} = {d / bound:.1f} x bound")
        assert d >= 10 * bound, name
