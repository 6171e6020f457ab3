"""GPU (-m gpu): DiT-XL/2 text-to-3D -- 72-wide self-attention heads, cross-attention with 64-wide heads (inner 1024).
The depth-2 forward against the reference's own output (tests/golden/dit_t23d_xl.npz, oracle/make_golden_xl.py), the
full 28-layer forward against the fp32 oracle, 10-step sampling (graph replay vs eager launches, and against the
oracle sampler) and text-to-3D end to end.  Tolerances are the DiT-L/2 parity tests' (test_gpu_parity.py)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    return torch.device("cuda", 0)


def _seeded(m):
    from oracle import dit as odit
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    sd = odit.synth_state_dict(shapes, seed=7, keep={"pos_embed": m.state_dict()["pos_embed"]})
    m.load_state_dict(sd)
    return m, sd


@pytest.fixture(scope="module")
def xl(dev):
    """build_t23d("DiT-XL/2") with the oracle's key-seeded weights (non-zero adaLN and gates)."""
    from ln3diff_b200.utils import build_t23d
    m, sd = _seeded(build_t23d("DiT-XL/2"))
    return m.to(dev), sd


def test_depth2_forward_matches_reference_golden(dev, golden):
    from ln3diff_b200.dit.dit_models_xformers import TextCondDiTBlock
    from ln3diff_b200.dit.dit_trilatent import DiT_TriLatent
    from oracle import fixtures as fx
    m = DiT_TriLatent(depth=2, hidden_size=1152, patch_size=2, num_heads=16, input_size=32, num_classes=0,
                      learn_sigma=False, in_channels=4, context_dim=768, roll_out=True, vit_blk=TextCondDiTBlock)
    m, _ = _seeded(m)
    m = m.to(dev)
    x, t, ctx = fx.dit_inputs()
    out = m(x.to(dev), t.to(dev), {"crossattn": ctx.to(dev)})
    assert out.dtype == torch.float32 and out.is_contiguous() and out.shape == (2, 12, 32, 32)
    assert _rel(out, golden("dit_t23d_xl.npz")["out"]) < 2e-2


def test_full_forward_matches_fp32_oracle(dev, xl):
    from oracle import dit as odit
    from oracle import fixtures as fx
    m, sd = xl
    x, t, ctx = fx.dit_inputs()
    out = m(x.to(dev), t.to(dev), {"crossattn": ctx.to(dev)})
    sdd = {k: v.to(dev) for k, v in sd.items()}
    ref = odit.dit_t23d_forward(sdd, "DiT-XL/2", x.to(dev), t.to(dev), ctx.to(dev))
    assert _rel(out, ref) < 2e-2


def _cfg_inputs(dev, B=2):
    g = torch.Generator().manual_seed(41)
    x0 = torch.randn(B, 12, 32, 32, generator=g)
    c = {"crossattn": torch.randn(B, 77, 768, generator=g)}
    uc = {"crossattn": torch.zeros(B, 77, 768)}
    return x0, c, uc


@pytest.mark.parametrize("sampler", ["EulerEDMSampler", "DPMPP2MSampler"])
def test_sampling_graph_vs_eager_and_oracle(dev, xl, monkeypatch, sampler):
    from ln3diff_b200 import pipeline
    from oracle import dit as odit
    from oracle import edm_samplers as oes
    from oracle import samplers as osmp
    m, sd = xl
    x0, c, uc = _cfg_inputs(dev)
    cd, ucd = ({k: v.to(dev) for k, v in d.items()} for d in (c, uc))
    monkeypatch.delenv("LN3_CUDA_GRAPH", raising=False)
    out = pipeline.sample_t23d(m, x0.to(dev), cd, ucd, 10, 6.5, sampler=sampler)
    monkeypatch.setenv("LN3_CUDA_GRAPH", "0")
    eager = pipeline.sample_t23d(m, x0.to(dev), cd, ucd, 10, 6.5, sampler=sampler)
    assert torch.equal(out, eager), "graph replay and eager launches differ"
    # the oracle samplers run on the host; their fp32 network evaluations run on the GPU
    sdd = {k: v.to(dev) for k, v in sd.items()}
    net = lambda xi, ti, cc: odit.dit_t23d_forward(sdd, "DiT-XL/2", xi.to(dev), ti.to(dev),
                                                   cc["crossattn"].to(dev)).cpu()
    if sampler == "EulerEDMSampler":
        ref = osmp.euler_edm_cfg_sample(net, x0.clone(), c, uc, 10, 6.5)
    else:
        ref, _ = oes.edm_sample(sampler, net, x0.clone(), c, uc, 10, 6.5)
    assert _rel(out, ref) < 2e-2


def test_fp8_prepare_raises_at_1152(dev):
    from ln3diff_b200.dit.dit_models_xformers import TextCondDiTBlock
    from ln3diff_b200.dit.dit_trilatent import DiT_TriLatent
    m = DiT_TriLatent(depth=1, hidden_size=1152, num_heads=16, num_classes=0, learn_sigma=False, in_channels=4,
                      context_dim=768, roll_out=True, vit_blk=TextCondDiTBlock).to(dev)
    m.set_gemm_precision("fp8")
    with pytest.raises(RuntimeError, match="embed_dim % 256"):
        m.prepare()


def test_text_to_3d_end_to_end(dev, xl, tmp_path):
    """One prompt through the CLIP conditioner, 4 Euler steps of DiT-XL/2, decode with the released DiT2-L/2 VAE
    and render two views at 128^2; the latents are generate_t23d's / sample_t23d's for the same noise.  Then
    mesh.export_mesh writes an OBJ from those latents (random weights: the density threshold is the grid's median)."""
    from ln3diff_b200 import mesh, pipeline
    from ln3diff_b200.sgm.modules.encoders.modules import FrozenCLIPEmbedder, GeneralConditioner
    from ln3diff_b200.utils import build_ae_decoder, orbit_cameras
    m, _ = xl
    emb = FrozenCLIPEmbedder(device=dev, depth=2, seed=3, random_init=True)
    emb._emb_config = {"input_key": "caption", "ucg_rate": 0.1}
    cond = GeneralConditioner([emb])
    ids = torch.randint(3, 49000, (1, 77), generator=torch.Generator().manual_seed(1))
    ids[0, 9:] = 49407
    dec = build_ae_decoder("DiT2-L/2", device=dev)
    cams = orbit_cameras(2).to(dev)
    lat, out = pipeline.text_to_3d(cond, m, dec, ids, cams, num_samples=1, num_steps=4, resolution=128)
    assert lat.is_cuda and lat.shape == (1, 12, 32, 32) and bool(torch.isfinite(lat).all())
    img = out["image_raw"]
    assert img.is_cuda and img.shape == (1, 2, 3, 128, 128) and bool(torch.isfinite(img).all())
    c, uc = pipeline.condition_prompt(cond, "caption", ids, num_samples=1, device=dev)
    randn = torch.randn(1, 12, 32, 32, generator=torch.Generator().manual_seed(41)).to(dev)
    lat2, _ = pipeline.generate_t23d(m, dec, randn, c, uc, cams, num_steps=4, resolution=128)
    assert torch.equal(lat, lat2)
    planes = dec.vit_decode_postprocess(lat, {})
    thres = float(dec.triplane_decode_grid(planes, grid_size=64)["sigma"].median())
    path = mesh.export_mesh(dec, planes, str(tmp_path), "xl", mesh_size=64, mesh_thres=thres)
    with open(path) as f:
        lines = f.readlines()
    assert sum(ln.startswith("f ") for ln in lines) > 0 and sum(ln.startswith("v ") for ln in lines) > 0


def test_head_norm_and_fmha_width_refusals(dev):
    from ln3diff_b200 import ops
    a = torch.zeros(4, 64, dtype=torch.bfloat16, device=dev)
    w = torch.zeros(3 * 1152, 64, dtype=torch.bfloat16, device=dev)
    with pytest.raises(ValueError, match="64-wide heads only"):
        ops.gemm(a, w, head_norm=torch.ones(2, 72, device=dev), head_norm_sec_cols=1152)
    x = torch.zeros(1, 4, 3 * 2 * 48, dtype=torch.bfloat16, device=dev)
    with pytest.raises(ValueError, match="64 or 72"):
        ops.fmha(x[:, :, :96], x[:, :, 96:192], x[:, :, 192:], 2)
