"""GPU: device marching cubes vs the numpy oracle (bit-exact faces, fp32-rounded vertices) and, at the full
192^3 export size, through mesh invariants (SURVEY 8f-2; reference nsr/train_util_diffusion.py:208-249)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda", 0)


def _sphere(n, r, density=False):
    x = np.linspace(-1, 1, n)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    d = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    return ((10 * (r - d)) if density else (d - r)).astype(np.float32)


@pytest.mark.parametrize("case", ["sphere", "random", "ragged", "empty", "plane"])
def test_marching_cubes_matches_oracle(dev, case):
    from ln3diff_b200 import ops
    from oracle import mesh
    rng = np.random.default_rng(3)
    if case == "sphere":
        vol, iso = _sphere(32, 0.6), 0.0
    elif case == "random":
        vol, iso = rng.standard_normal((24, 24, 24)).astype(np.float32), 0.1
    elif case == "ragged":      # dimensions that are not multiples of anything, open surface at the border
        vol, iso = rng.standard_normal((7, 33, 18)).astype(np.float32), -0.2
    elif case == "empty":
        vol, iso = np.ones((9, 9, 9), np.float32), 10.0      # everything <= iso: no surface
    else:                         # values exactly equal to iso on a lattice plane (`<=` puts them inside)
        vol = np.broadcast_to(np.arange(12, dtype=np.float32)[:, None, None], (12, 10, 11)).copy()
        iso = 5.0
    v, f = ops.marching_cubes(torch.from_numpy(vol).to(dev), iso)
    vo, fo = mesh.marching_cubes(vol, iso)
    assert tuple(v.shape) == vo.shape and tuple(f.shape) == fo.shape
    if fo.shape[0]:
        assert np.array_equal(f.cpu().numpy().astype(np.int64), fo)          # index work: bit-exact
        assert np.abs(v.cpu().numpy().astype(np.float64) - vo).max() < 2e-5  # fp32 interpolation vs float64
    else:
        assert v.shape[0] == 0


def test_marching_cubes_full_size_invariants(dev):
    """192^3 (the reference's mesh_size): closed oriented 2-manifold, Euler characteristic 2, enclosed volume,
    affine fold of the reference's rescale; a second call gives the identical mesh (deterministic order)."""
    from ln3diff_b200 import ops
    from oracle import mesh
    G, r = 192, 0.7
    vol = torch.from_numpy(_sphere(G, r, density=True)).to(dev)
    s = 2.0 / (G - 1) * 0.45
    v, f = ops.marching_cubes(vol, 0.0, scale=(s, s, s), offset=(-0.45,) * 3)
    v2, f2 = ops.marching_cubes(vol, 0.0, scale=(s, s, s), offset=(-0.45,) * 3)
    assert torch.equal(v, v2) and torch.equal(f, f2)
    st = mesh.mesh_stats(v.cpu().numpy().astype(np.float64), f.cpu().numpy().astype(np.int64))
    assert st["closed"] and st["oriented"] and st["euler"] == 2
    rw = r * 0.45
    assert abs(st["volume"] / (4 / 3 * np.pi * rw ** 3) - 1) < 2e-3          # positive: outward normals for a density
    rad = v.norm(dim=1)
    assert float((rad - rw).abs().max()) < 1e-4
    # timing (reported, not asserted)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        ops.marching_cubes(vol, 0.0)
    e1.record()
    torch.cuda.synchronize()
    print(f"marching cubes 192^3: {e0.elapsed_time(e1) / 5:.3f} ms per call ({v.shape[0]} vertices, {f.shape[0]} faces)")


def test_extract_mesh_through_the_decoder_mirror(dev, tmp_path):
    """reference :208-247 end to end on a synthetic tri-plane: grid query -> marching cubes -> vertex colours -> OBJ."""
    from ln3diff_b200 import mesh as pmesh
    from ln3diff_b200.utils import build_ae_decoder
    torch.manual_seed(0)
    dec = build_ae_decoder("DiT2-S/2", device=dev)
    planes = (torch.randn(1, 96, 128, 128, device=dev) * 2.0)
    lat = {"latent_after_vit": planes}
    grid = dec.triplane_decode_grid(lat, grid_size=48)
    thres = float(grid["sigma"].median())
    m = pmesh.extract_mesh(dec, lat, mesh_size=48, mesh_thres=thres)
    assert m["vertices"].shape[0] > 0 and m["faces"].max() < m["vertices"].shape[0]
    assert m["vertex_colors"].dtype == np.uint8 and m["vertex_colors"].shape == m["vertices"].shape
    # vertices (before the export rotation) lie inside the sampler box, and the rotation is the reference's
    vd = m["vertices_device"].cpu().numpy()
    assert np.abs(vd).max() <= 0.45 + 1e-6
    assert np.allclose(m["vertices"], vd.astype(np.float64) @ pmesh.rotation_matrix_x(-90).T)
    # colours are the decoder's answer at the vertices
    rgb = dec.forward_points(planes, m["vertices_device"].unsqueeze(0))["rgb"].squeeze(0)
    assert np.array_equal(m["vertex_colors"], (rgb.clamp(0, 1) * 255).to(torch.uint8).cpu().numpy())
    p = pmesh.export_obj(str(tmp_path / "m.obj"), m["vertices"], m["faces"], m["vertex_colors"])
    assert sum(1 for ln in open(p) if ln.startswith("f ")) == m["faces"].shape[0]

