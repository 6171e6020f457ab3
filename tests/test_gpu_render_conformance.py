"""GPU (-m gpu): the fused renderer (render.cu) element by element against a float64 reference, on every dispatch
path: the 4x4 pixel-tile and the linear ray schedule (ragged shapes, partial last item, a single short item),
object batches through views_per_obj and through an explicit view -> object map, views that share the
reference's per-call reductions (group_size 1, 2, 3 and all of 5, a partial last group), production-size planes
with more work items than SMs, the rendering options, edge rays whose slab test yields NaN, and both MLP
precisions on every case.

The reference is oracle.render.render_group -- one ImportanceRenderer.forward call per group of views -- run in
float64 on the fp32 inputs the kernel saw (the box and bbox bounds rounded to fp32 as the kernel holds them).
Bounds are per element (depth relative to max(1, |ref|)); the observed maxima beside them were measured on an
H100 80GB HBM3 (SXM, 700 W power limit) over every case below.  No ray is exempt: on the exact path a ray may pass
TOL_EXACT only up to TOL_EXACT_FLIP, only when the kernel's debug outputs show it took a different discrete
decision (importance-sample index, sort order, in-box test) than the float64 reference, and only for at most
MAX_FLIP_FRACTION of the rays.  Each case whose point is a mapping (view -> object, view -> group, white_back) also asserts
that the reference with that mapping wrong differs by far more than the tolerance, so a slip cannot pass."""
from __future__ import annotations

import dataclasses
import math

import numpy as np
import pytest
import torch

from oracle import fixtures as fx
from oracle import render as orender

pytestmark = pytest.mark.gpu

TOL_EXACT = {"rgb": 2e-5, "weights": 2e-5, "depth": 2e-5}         # observed 3.9e-6, 2.8e-6, 3.5e-6
TOL_EXACT_FLIP = 1e-4                # observed 6.7e-5 (rgb), 6.2e-5 (weights): 128x128 planes only
MAX_FLIP_FRACTION = 5e-3
TOL_TF32 = {"rgb": 2e-3, "weights": 1e-3, "depth": 1e-3}           # observed 4.1e-4, 1.4e-4, 1.6e-4
TOL_TF32_REL = 1e-3                  # per-view rgb rel-L2; observed 2.0e-4
SENSITIVE = 1e-2          # a wrong mapping must move some element of every affected view by at least this


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


# ------------------------------------------------------------------ inputs
def _pinhole_rays(n_views: int, w: int, h: int, seed: int, radius: float = 2.0, fov: float = 0.9):
    """Rays of n_views cameras on a sphere around the box, looking at a jittered point near the origin, through a
    w x h pixel grid; ray m = y*w + x.  About half of every view's rays hit the [-0.45, 0.45]^3 box."""
    g = torch.Generator().manual_seed(seed)
    os_, ds = [], []
    for v in range(n_views):
        az = 2 * math.pi * (v + 0.37) / n_views
        el = 0.3 * math.sin(1.7 * v + 0.4)
        eye = radius * torch.tensor([math.cos(el) * math.cos(az), math.cos(el) * math.sin(az), math.sin(el)])
        fwd = torch.nn.functional.normalize(0.05 * torch.randn(3, generator=g) - eye, dim=0)
        right = torch.nn.functional.normalize(torch.linalg.cross(fwd, torch.tensor([0.0, 0.0, 1.0])), dim=0)
        up = torch.linalg.cross(right, fwd)
        xs = ((torch.arange(w) + 0.5) / w - 0.5) * fov * w / max(w, h)
        ys = ((torch.arange(h) + 0.5) / h - 0.5) * fov * h / max(w, h)
        d = fwd + xs[None, :, None] * right + ys[:, None, None] * up        # (h, w, 3)
        ds.append(torch.nn.functional.normalize(d.reshape(-1, 3), dim=1))
        os_.append(eye.expand(w * h, 3).clone())
    return torch.stack(os_), torch.stack(ds)


def _miss_rays(M: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    o = torch.tensor([3.0, 3.0, 3.0]) + 0.1 * torch.randn(M, 3, generator=g)
    d = torch.nn.functional.normalize(torch.tensor([1.0, 0.2, 0.1]) + 0.05 * torch.randn(M, 3, generator=g), dim=1)
    return o, d


def _inside_rays(M: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(M, 3, generator=g) - 0.5) * 0.6, torch.nn.functional.normalize(torch.randn(M, 3, generator=g), dim=1)


@dataclasses.dataclass
class Case:
    name: str
    planes: torch.Tensor            # (n_obj, 3, 32, H, W)
    ray_o: torch.Tensor             # (V, M, 3)
    ray_d: torch.Tensor
    nc: torch.Tensor                # (V, M, 64)
    nf: torch.Tensor
    view_obj: list                  # object of every view
    group_size: int = 1
    image_width: int | None = None  # None: ops.render_views' default (square side)
    tiled: bool = False             # the schedule the host is expected to select
    explicit_map: bool = False      # pass view_obj to the kernel instead of views_per_obj
    box_warp: float = 0.9
    bbox: float = 0.45
    white_back: bool = True

    @property
    def V(self):
        return self.ray_o.shape[0]

    @property
    def M(self):
        return self.ray_o.shape[1]

    @property
    def path(self):
        return f"{'tiled' if self.tiled else 'linear'}, group_size {self.group_size}"


_OSG = fx.render_inputs(1, n_views=1)[1]


def _planes(n_obj: int, seed: int, h: int = 16, w: int = 16):
    return 5 * torch.randn(n_obj, 3, 32, h, w, generator=torch.Generator().manual_seed(seed))


def _noise(V: int, M: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(V, M, 64, generator=g), torch.rand(V, M, 64, generator=g)


def _simple(name, V, w, h, seed, *, n_obj=1, view_obj=None, plane_hw=(16, 16), **kw):
    o, d = _pinhole_rays(V, w, h, seed)
    nc, nf = _noise(V, w * h, seed + 1)
    vo = view_obj if view_obj is not None else [v * n_obj // V for v in range(V)]
    return Case(name, _planes(n_obj, seed + 2, *plane_hw), o, d, nc, nf, vo, **kw)


def _group_case(gs: int):
    """5 views of 5 objects: hitting, all-miss, hitting, camera inside the box, hitting.  Group (0, 1) of
    group_size 2 holds the all-miss view beside a hitting one: its samples span the hitting view's start range
    and its depth is clamped to the hitting view's depth range."""
    M = 64
    o, d = _pinhole_rays(5, 8, 8, 70)
    o[1], d[1] = _miss_rays(M, 71)
    o[3], d[3] = _inside_rays(M, 72)
    nc, nf = _noise(5, M, 73)
    return Case(f"groups_gs{gs}", _planes(5, 74), o, d, nc, nf, list(range(5)), group_size=gs, tiled=True)


def _edge_case():
    planes, osg, o, d, nc, nf = fx.render_group_inputs()
    assert osg is _OSG or all(torch.equal(a, b) for a, b in zip(osg, _OSG))
    return Case("edge_rays", planes, o, d, nc, nf, [0, 1, 2], group_size=3, tiled=False)


def _production_case():
    o, d = _pinhole_rays(2, 64, 64, 90)
    nc, nf = _noise(2, 64 * 64, 91)
    return Case("production_128planes_64x64_2obj", _planes(2, 92, 128, 128), o, d, nc, nf, [0, 1], tiled=True)


CASE_BUILDERS = {
    "square8": lambda: _simple("square8", 2, 8, 8, 10, tiled=True),
    "side10": lambda: _simple("side10", 2, 10, 10, 11, tiled=False),                   # 100 rays / view
    "side6_v3": lambda: _simple("side6_v3", 3, 6, 6, 12, tiled=False),                 # V*M = 108 = 6*16 + 12
    "v1_m9": lambda: _simple("v1_m9", 1, 3, 3, 13, tiled=False),                       # less than one item
    "wide24x16": lambda: _simple("wide24x16", 2, 24, 16, 14, image_width=24, tiled=True),
    "wide20x12": lambda: _simple("wide20x12", 2, 20, 12, 15, image_width=20, tiled=True),
    "wide18x16": lambda: _simple("wide18x16", 2, 18, 16, 16, image_width=18, tiled=False),
    "objects_3x2": lambda: _simple("objects_3x2", 6, 8, 8, 17, n_obj=3, tiled=True),
    "view_obj_perm": lambda: _simple("view_obj_perm", 6, 8, 8, 18, n_obj=3, view_obj=[2, 0, 1, 1, 0, 2],
                                     explicit_map=True, tiled=True),
    "groups_gs1": lambda: _group_case(1),
    "groups_gs2": lambda: _group_case(2),
    "groups_gs3": lambda: _group_case(3),
    "groups_gs5": lambda: _group_case(5),
    "production": _production_case,
    "white_back_false": lambda: _simple("white_back_false", 2, 8, 8, 19, tiled=True, white_back=False),
    "box_warp_1.2": lambda: _simple("box_warp_1.2", 2, 8, 8, 20, tiled=True, box_warp=1.2, bbox=0.5),
    "narrow_bbox": lambda: _simple("narrow_bbox", 2, 8, 8, 21, tiled=True, bbox=0.3),
    "planes_16x24": lambda: _simple("planes_16x24", 2, 8, 8, 22, tiled=True, plane_hw=(16, 24)),
    "edge_rays": _edge_case,
}
CASES = {name: build() for name, build in CASE_BUILDERS.items()}


def _case(name: str) -> Case:
    return CASES[name]


# ------------------------------------------------------------------ reference
def _f32(x: float) -> float:
    return float(np.float32(x))


def _opts(box_warp: float, bbox: float, white_back: bool) -> dict:
    """Rendering options as the kernel holds them: box half-side and bbox bounds rounded to fp32."""
    o = dict(orender.OBJAVERSE_OPTS)
    o.update(box_warp=2 * _f32(box_warp / 2), sampler_bbox_min=_f32(-bbox), sampler_bbox_max=_f32(bbox),
             white_back=white_back)
    return o


def _reference(c: Case, view_obj=None, group_size=None, white_back=None) -> dict:
    """float64 render_group per group of consecutive views -> rgb (V,M,3), depth (V,M), weights (V,M)."""
    view_obj = c.view_obj if view_obj is None else view_obj
    gs = c.group_size if group_size is None else group_size
    opts = _opts(c.box_warp, c.bbox, c.white_back if white_back is None else white_back)
    osg = tuple(t.double() for t in _OSG)
    outs = []
    for v0 in range(0, c.V, gs):
        vs = list(range(v0, min(v0 + gs, c.V)))
        planes = torch.stack([c.planes[view_obj[v]] for v in vs]).double()
        outs.append(orender.render_group(planes, osg, c.ray_o[vs].double(), c.ray_d[vs].double(),
                                         c.nc[vs].double(), c.nf[vs].double(), opts))
    return {k: torch.cat([o[k] for o in outs]).reshape(c.V, c.M, -1).squeeze(-1) for k in ("rgb", "depth", "weights")}


_refs: dict = {}


def _ref(name: str) -> dict:
    if name not in _refs:
        _refs[name] = _reference(_case(name))
    return _refs[name]


# ------------------------------------------------------------------ kernel
def _run(dev, c: Case, tf32: bool, image_width=-1, debug=False) -> dict:
    from ln3diff_b200 import ops
    pcl = ops.planes_to_channels_last(c.planes.contiguous().to(dev))
    kw = dict(view_obj=torch.tensor(c.view_obj, dtype=torch.int32, device=dev)) if c.explicit_map else \
        dict(views_per_obj=c.V // c.planes.shape[0])
    if not c.explicit_map:
        assert c.view_obj == [v // kw["views_per_obj"] for v in range(c.V)]
    # poison free allocator blocks of the output and workspace sizes (best effort): a ray the kernel skips keeps
    # NaN, and a reduction slot it reads without writing holds 3.4e38, rather than a previous launch's values
    for shp in ((c.V, 3, c.M), (c.V, 1, c.M), (c.V, 1, c.M)):
        torch.full(shp, float("nan"), device=dev)
    torch.full((ops._lib.lib().ln3_render_workspace_bytes(c.V, c.M, c.group_size),), 0x7F, dtype=torch.uint8,
               device=dev)
    out = ops.render_views(pcl, c.ray_o.contiguous().to(dev), c.ray_d.contiguous().to(dev), c.nc.contiguous().to(dev),
                           c.nf.contiguous().to(dev), tuple(t.to(dev) for t in _OSG), group_size=c.group_size,
                           box_warp=c.box_warp, bbox_min=-c.bbox, bbox_max=c.bbox, white_back=c.white_back,
                           mlp_tf32=tf32, debug=debug,
                           image_width=c.image_width if image_width == -1 else image_width, **kw)
    torch.cuda.synchronize()
    return {"rgb": out["rgb"].permute(0, 2, 1).cpu(), "depth": out["depth"][:, 0].cpu(),
            "weights": out["weights"][:, 0].cpu(), **({"dbg": out} if debug else {})}


def _check(what: str, got: dict, ref: dict, tf32: bool, flips_allowed: bool = False) -> torch.Tensor:
    """Element-wise bounds of the module docstring (observed maxima printed with -s).  Returns the (V, M) mask of
    rays past TOL_EXACT but within TOL_EXACT_FLIP when flips_allowed (the caller must show they are flips)."""
    err = {"rgb": (got["rgb"].double() - ref["rgb"]).abs().amax(-1),
           "weights": (got["weights"].double() - ref["weights"]).abs(),
           "depth": (got["depth"].double() - ref["depth"]).abs() / ref["depth"].abs().clamp_min(1.0)}
    rel = max(float((got["rgb"][v].double() - ref["rgb"][v]).norm() / ref["rgb"][v].norm()) for v in range(len(ref["rgb"])))
    tol = TOL_TF32 if tf32 else TOL_EXACT
    over = torch.zeros_like(err["rgb"], dtype=torch.bool)
    for k, e in err.items():
        over |= ~(e <= tol[k])                                  # NaN counts as out of bound
    print(f"{what} [{'tf32' if tf32 else 'fp32'}]: " + ", ".join(f"{k} {float(e.max()):.3e}" for k, e in err.items())
          + f", rgb_rel {rel:.3e}, rays past the bound {int(over.sum())} of {over.numel()}")
    if flips_allowed and not tf32:
        for k, e in err.items():
            assert bool((e <= TOL_EXACT_FLIP).all()), (what, k, float(e.max()))
        assert int(over.sum()) <= MAX_FLIP_FRACTION * over.numel(), (what, int(over.sum()))
    else:
        assert not bool(over.any()), (what, {k: float(e.max()) for k, e in err.items()}, torch.nonzero(over)[:8].tolist())
    if tf32:
        assert rel <= TOL_TF32_REL, (what, rel)
    return over


def _assert_discrete_flips(c: Case, dbg: dict, over: torch.Tensor) -> None:
    """Every ray of `over` took a different discrete decision in the kernel than in the float64 reference."""
    assert c.group_size == 1     # the per-ray debug reference is render_rays: one view per reference call
    opts = _opts(c.box_warp, c.bbox, c.white_back)
    osg = tuple(t.double() for t in _OSG)
    for v in sorted(set(torch.nonzero(over)[:, 0].tolist())):
        r = orender.render_rays(c.planes[c.view_obj[v]].double(), osg, c.ray_o[v].double(), c.ray_d[v].double(),
                                opts, c.nc[v].double(), c.nf[v].double(), return_debug=True)
        sl = slice(v * c.M, (v + 1) * c.M)
        inbox = torch.cat([r["inbox_coarse"], r["inbox_fine"]], 1)
        flip = ((dbg["inds"][sl].cpu().long() != r["inds"]).any(1) | (dbg["order"][sl].cpu().long() != r["order"]).any(1)
                | (dbg["inbox"][sl].cpu().bool() != inbox).any(1))
        rays = torch.nonzero(over[v])[:, 0]
        print(f"view {v}: rays past TOL_EXACT {rays.tolist()}, discrete decision differs {flip[rays].tolist()}")
        assert bool(flip[rays].all()), (v, rays[~flip[rays]].tolist())


def _assert_sensitive(what: str, ref: dict, wrong: dict, views) -> None:
    for v in views:
        diff = max(float((ref[k][v] - wrong[k][v]).abs().max()) for k in ("rgb", "depth", "weights"))
        assert diff > SENSITIVE, f"{what}: view {v} moves only {diff:.2e}; the case cannot tell the mapping apart"


# ------------------------------------------------------------------ tests
@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
@pytest.mark.parametrize("name", [pytest.param(n, id=f"{n}-{c.path.replace(', ', '-').replace(' ', '')}")
                                  for n, c in CASES.items()])
def test_render_matches_fp64_reference(dev, name, tf32):
    c = _case(name)
    print(f"{name}: V={c.V} M={c.M} planes {tuple(c.planes.shape[-2:])}, {c.path}, {'tf32' if tf32 else 'fp32'} MLP")
    got = _run(dev, c, tf32, debug=not tf32)
    over = _check(name, got, _ref(name), tf32, flips_allowed=c.group_size == 1)
    if bool(over.any()):
        _assert_discrete_flips(c, got["dbg"], over)


def test_schedule_dispatch(dev):
    """The host picks the 4x4 tile schedule exactly for images whose width and height are multiples of 4."""
    from ln3diff_b200 import ops
    for name in CASE_BUILDERS:
        c = _case(name)
        w = ops.render_tile_width(c.M, c.image_width)
        assert (w > 0) == c.tiled, (name, c.M, c.image_width, w)
        assert w in (0, c.image_width or round(math.sqrt(c.M)))
    assert ops.render_tile_width(64, 0) == 0                   # image_width=0 forces the linear schedule


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
@pytest.mark.parametrize("name", [n for n in CASE_BUILDERS if n in ("square8", "wide24x16", "wide20x12",
                                                                     "objects_3x2", "groups_gs2", "production")])
def test_tiled_and_linear_schedules_are_bit_identical(dev, name, tf32):
    """A ray's arithmetic does not depend on the schedule that reached it."""
    c = _case(name)
    assert c.tiled
    a, b = _run(dev, c, tf32), _run(dev, c, tf32, image_width=0)
    for k in ("rgb", "depth", "weights"):
        assert torch.equal(a[k], b[k]), (name, k)


def test_cases_can_tell_the_mappings_apart():
    """Wrong view -> object maps, per-view reductions where views share them and a flipped white_back all move the
    float64 reference far beyond any tolerance above, in every view they affect."""
    for name in ("objects_3x2", "view_obj_perm"):
        c = _case(name)
        rot = [(o + 1) % c.planes.shape[0] for o in c.view_obj]
        _assert_sensitive(f"{name}: neighbouring object's planes", _ref(name), _reference(c, view_obj=rot), range(c.V))
        mod = [v % c.planes.shape[0] for v in range(c.V)]
        changed = [v for v in range(c.V) if mod[v] != c.view_obj[v]]
        assert changed
        _assert_sensitive(f"{name}: view % n_obj", _ref(name), _reference(c, view_obj=mod), changed)
    for gs in (2, 3, 5):
        name = f"groups_gs{gs}"
        _assert_sensitive(f"{name}: per-view reductions", _ref(name), _reference(_case(name), group_size=1), [1])
    c = _case("white_back_false")
    _assert_sensitive("white_back", _ref("white_back_false"), _reference(c, white_back=True), range(c.V))
    c = _case("edge_rays")
    _assert_sensitive("edge rays: per-view reductions", _ref("edge_rays"), _reference(c, group_size=1), [0, 2])


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
def test_edge_rays_match_reference_golden(dev, golden, tf32):
    """The batch-3 call of render_group.npz, made by the reference itself: rays whose slab test yields NaN are
    invalid there (torch.max / torch.min propagate NaN) and must be invalid in the kernel, which then marches them
    over the call's shared start range."""
    g = golden("render_group.npz")
    c = _case("edge_rays")
    got = _run(dev, c, tf32, debug=True)
    ref = {"rgb": torch.from_numpy(g["rgb"]).double(), "depth": torch.from_numpy(g["depth"])[..., 0].double(),
           "weights": torch.from_numpy(g["weights"])[..., 0].double()}
    _check("edge_rays vs reference golden", got, ref, tf32)
    # the NaN rays (0, 1, 3, 4 of view 0) sample the shared range [min valid start, max valid start]: the first
    # coarse depth is that minimum plus noise -- a ray marched over its own slab interval would start near 1.55
    valid = orender.render_group(c.planes, _OSG, c.ray_o, c.ray_d, c.nc, c.nf, orender.OBJAVERSE_OPTS)["valid"]
    smin = float(orender.ray_limits_box(c.ray_o, c.ray_d, 0.9)[0][..., 0][valid].min())
    z_fine = got["dbg"]["z_fine"].cpu()
    for m in (0, 1, 3, 4):
        assert float(z_fine[m].min()) < smin + 0.5 * (1.55 - smin), (m, float(z_fine[m].min()), smin)


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
def test_importance_renderer_mirror_batch3(dev, tf32):
    """nsr...ImportanceRenderer.forward with N=3 objects (views_per_obj=1, group_size=N, the device RNG draws of the
    reference) against the float64 render_group of the same draws."""
    from ln3diff_b200.nsr.volumetric_rendering.renderer import ImportanceRenderer
    c = _case("objects_3x2")
    planes = c.planes.to(dev)
    o, d = c.ray_o[::2].contiguous(), c.ray_d[::2].contiguous()       # one view per object
    N, M = 3, c.M

    class Dec:
        def raw_parameters(self):
            return tuple(t.to(dev) for t in _OSG)

    opts = dict(orender.OBJAVERSE_OPTS, osg_mlp_tf32=tf32)
    torch.cuda.manual_seed(1234)
    out = ImportanceRenderer()(planes, Dec(), o.to(dev), d.to(dev), opts)
    torch.cuda.manual_seed(1234)                                       # the same draws in the same order
    nc = torch.rand_like(torch.empty((N, M, 64, 1), device=dev, dtype=torch.float32)).reshape(N, M, 64).cpu()
    nf = torch.rand(N * M, 64, device=dev).reshape(N, M, 64).cpu()
    mc = Case("mirror", c.planes, o, d, nc, nf, [0, 1, 2], group_size=N)
    got = {"rgb": out["feature_samples"].cpu(), "depth": out["depth_samples"][..., 0].cpu(),
           "weights": out["weights_samples"][..., 0].cpu()}
    _check("ImportanceRenderer.forward N=3", got, _reference(mc), tf32)


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
def test_decode_and_render_object_batches(dev, tf32):
    """pipeline.decode_and_render with B=3 in launches of 2 then 1 objects: every object equals a single-object
    render_views of its own planes, bit for bit."""
    from ln3diff_b200 import ops, pipeline
    from ln3diff_b200.utils import orbit_cameras
    B, V, res = 3, 2, 16
    M = res * res
    planes_cl = ops.planes_to_channels_last(_planes(B, 30).to(dev))
    osg = tuple(t.to(dev) for t in _OSG)

    class Decoder:   # the three members decode_and_render reads; the planes stand in for decoded latents
        rendering_kwargs = dict(box_warp=0.9, sampler_bbox_min=-0.45, sampler_bbox_max=0.45, white_back=True)

        class triplane_decoder:
            class decoder:
                @staticmethod
                def raw_parameters():
                    return osg

        @staticmethod
        def decode_to_channels_last(latents, in_mul):
            return planes_cl

    cams = orbit_cameras(V)
    nc, nf = (t.reshape(B * V, M, 64).to(dev) for t in _noise(B * V, M, 31))
    out = pipeline.decode_and_render(Decoder(), torch.zeros(B, 12, 32, 32, device=dev), cams, resolution=res,
                                     noise=(nc, nf), mlp_tf32=tf32, max_views_per_launch=2 * V)
    o, d = ops.generate_rays(cams.to(dev).contiguous(), res)
    for b in range(B):
        one = ops.render_views(planes_cl[b:b + 1].contiguous(), o, d, nc[b * V:(b + 1) * V].contiguous(),
                               nf[b * V:(b + 1) * V].contiguous(), osg, views_per_obj=V, mlp_tf32=tf32)
        assert torch.equal(out["image_raw"][b], one["rgb"].view(V, 3, res, res)), b
        assert torch.equal(out["image_depth"][b], one["depth"].view(V, 1, res, res)), b
        assert torch.equal(out["weights_samples"][b], one["weights"].view(V, 1, res, res)), b
    assert not torch.equal(out["image_raw"][0], out["image_raw"][1])


def test_planes_to_channels_last_ragged(dev):
    """(n_obj=3, 96, 20, 12) -> (3, 3, 20, 12, 32): HW = 240 is not a multiple of the 32-pixel transpose tile."""
    from ln3diff_b200 import ops
    x = torch.randn(3, 96, 20, 12, generator=torch.Generator().manual_seed(40))
    got = ops.planes_to_channels_last(x.to(dev)).cpu()
    assert torch.equal(got, x.reshape(3, 3, 32, 20, 12).permute(0, 1, 3, 4, 2))
