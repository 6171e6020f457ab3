"""TEST INFRASTRUCTURE ONLY (oracle) -- fp32 CPU restatement of the reference's tri-plane
volumetric renderer.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs may import this module; the product path never does.

Restates, with basic torch ops and its own bilinear sampler (no F.grid_sample, no reference
imports):
  nsr/volumetric_rendering/ray_sampler.py:180-257   RaySampler.create_uv / forward          (R1)
  nsr/volumetric_rendering/math_utils.py:124-190    get_ray_limits_box                      (R2)
  nsr/volumetric_rendering/renderer.py:145-155      'auto' limits fix-up for invalid rays   (R2)
  nsr/volumetric_rendering/renderer.py:437-477      sample_stratified + math_utils.linspace (R3)
  nsr/volumetric_rendering/renderer.py:55-104,310-411  plane projection, bilinear gather,
                                                    in-box filter                            (R4)
  nsr/triplane.py:356-375 + nsr/networks_stylegan2.py:144-157  OSGDecoder / FullyConnectedLayer (R4)
  nsr/volumetric_rendering/ray_marcher.py:26-68     MipRayMarcher2                           (R5)
  nsr/volumetric_rendering/renderer.py:479-552      sample_importance / sample_pdf           (R6)
  nsr/volumetric_rendering/renderer.py:422-435      unify_samples (sort)                     (R7)
  nsr/triplane.py:612-672                            image reshape, image_mask               (R8)
Pinned by oracle/make_golden.py against the reference's own ImportanceRenderer / Triplane run in
the build container (tests/golden/render_*.npz).  Noise is an explicit input (the reference draws
torch.rand_like / torch.rand on the compute device: renderer.py:464,530).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

OBJAVERSE_OPTS = dict(  # nsr/script_util.py:433-465,761-797 (SURVEY.md appendix C)
    depth_resolution=64, depth_resolution_importance=64, ray_start="auto", ray_end="auto",
    box_warp=0.9, white_back=True, sampler_bbox_min=-0.45, sampler_bbox_max=0.45,
    filter_out_of_bbox=True, clamp_mode="softplus", disparity_space_sampling=False,
    decoder_activation="sigmoid")


def generate_rays(cam2world: torch.Tensor, intrinsics: torch.Tensor, res: int):
    """(V,4,4), (V,3,3) -> ray_o, ray_d (V, res*res, 3); ray m = y*res + x (x fastest)."""
    V = cam2world.shape[0]
    cam_loc = cam2world[:, :3, 3]
    fx, fy = intrinsics[:, 0, 0], intrinsics[:, 1, 1]
    cx, cy, sk = intrinsics[:, 0, 2], intrinsics[:, 1, 2], intrinsics[:, 0, 1]
    ar = torch.arange(res, dtype=torch.float32)
    c = ar * (1.0 / res) + (0.5 / res)
    y_cam = c[:, None].expand(res, res).reshape(1, -1).expand(V, -1)
    x_cam = c[None, :].expand(res, res).reshape(1, -1).expand(V, -1)
    z_cam = torch.ones_like(x_cam)
    u = lambda t: t.unsqueeze(-1)
    x_lift = (x_cam - u(cx) + u(cy) * u(sk) / u(fy) - u(sk) * y_cam / u(fy)) / u(fx) * z_cam
    y_lift = (y_cam - u(cy)) / u(fy) * z_cam
    pts = torch.stack((x_lift, y_lift, z_cam, torch.ones_like(z_cam)), dim=-1)  # (V,M,4)
    world = torch.einsum("vij,vmj->vmi", cam2world, pts)[:, :, :3]
    d = world - cam_loc[:, None, :]
    d = d / d.norm(dim=2, keepdim=True).clamp_min(1e-12)
    o = cam_loc[:, None, :].expand(-1, d.shape[1], -1).contiguous()
    return o, d


def ray_limits_box(o: torch.Tensor, d: torch.Tensor, side: float):
    """Slab test against [-side/2, side/2]^3; invalid rays -> (-1, -2).  (…,3) -> (…,1) x2."""
    shp = o.shape
    o = o.reshape(-1, 3)
    d = d.reshape(-1, 3)
    lo, hi = -side / 2, side / 2
    inv = 1 / d
    neg = inv < 0
    bmin = torch.where(neg, torch.full_like(inv, hi), torch.full_like(inv, lo))
    bmax = torch.where(neg, torch.full_like(inv, lo), torch.full_like(inv, hi))
    t0 = (bmin - o) * inv
    t1 = (bmax - o) * inv
    tmin, tmax = t0[:, 0], t1[:, 0]
    valid = ~((tmin > t1[:, 1]) | (t0[:, 1] > tmax))
    tmin = torch.max(tmin, t0[:, 1])
    tmax = torch.min(tmax, t1[:, 1])
    valid = valid & ~((tmin > t1[:, 2]) | (t0[:, 2] > tmax))
    tmin = torch.max(tmin, t0[:, 2])
    tmax = torch.min(tmax, t1[:, 2])
    tmin = torch.where(valid, tmin, torch.full_like(tmin, -1.0))
    tmax = torch.where(valid, tmax, torch.full_like(tmax, -2.0))
    return tmin.reshape(*shp[:-1], 1), tmax.reshape(*shp[:-1], 1)


def bilinear_zeros(plane: torch.Tensor, gx: torch.Tensor, gy: torch.Tensor) -> torch.Tensor:
    """grid_sample(bilinear, zeros, align_corners=False) for one plane.
    plane (C,H,W); gx, gy (P,) normalised to [-1,1] (gx indexes W) -> (P,C)."""
    C, H, W = plane.shape
    ix = ((gx + 1) * W - 1) / 2
    iy = ((gy + 1) * H - 1) / 2
    x0 = torch.floor(ix)
    y0 = torch.floor(iy)
    x1, y1 = x0 + 1, y0 + 1
    w_nw = (x1 - ix) * (y1 - iy)
    w_ne = (ix - x0) * (y1 - iy)
    w_sw = (x1 - ix) * (iy - y0)
    w_se = (ix - x0) * (iy - y0)
    flat = plane.reshape(C, H * W)

    def tap(xi, yi, w):
        ok = (xi >= 0) & (xi <= W - 1) & (yi >= 0) & (yi <= H - 1)
        idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long()
        return flat[:, idx].t() * (w * ok)[:, None]

    return tap(x0, y0, w_nw) + tap(x1, y0, w_ne) + tap(x0, y1, w_sw) + tap(x1, y1, w_se)


def osg_decoder(feat: torch.Tensor, w1, b1, w2, b2) -> tuple[torch.Tensor, torch.Tensor]:
    """feat (P,32) (already averaged over planes) -> rgb (P,3), sigma (P,1).
    FullyConnectedLayer: weight * (1/sqrt(in)), linear activation (networks_stylegan2.py:141-153)."""
    h = torch.addmm(b1.unsqueeze(0), feat, (w1 * (1.0 / math.sqrt(w1.shape[1]))).t())
    h = F.softplus(h)
    y = torch.addmm(b2.unsqueeze(0), h, (w2 * (1.0 / math.sqrt(w2.shape[1]))).t())
    rgb = torch.sigmoid(y[:, 1:]) * (1 + 2 * 0.001) - 0.001
    return rgb, y[:, 0:1]


def run_model(planes, osg, coords, opts):
    """planes (3,C,H,W); coords (P,3) -> rgb (P,3), sigma (P,1) with the out-of-box filter."""
    bmin, bmax = opts["sampler_bbox_min"], opts["sampler_bbox_max"]
    inbox = ((coords >= bmin) & (coords <= bmax)).all(-1)
    c = (2 / opts["box_warp"]) * coords
    f0 = bilinear_zeros(planes[0], c[:, 0], c[:, 1])  # plane 0 <- (x, y)
    f1 = bilinear_zeros(planes[1], c[:, 1], c[:, 2])  # plane 1 <- (y, z)
    f2 = bilinear_zeros(planes[2], c[:, 2], c[:, 0])  # plane 2 <- (z, x)
    feat = torch.stack([f0, f1, f2], 0).mean(0)
    rgb, sigma = osg_decoder(feat, *osg)
    if opts.get("filter_out_of_bbox", False):
        big = torch.nan_to_num(torch.tensor(-float("inf"))) / 3
        rgb = torch.where(inbox[:, None], rgb, torch.zeros_like(rgb))
        sigma = torch.where(inbox[:, None], sigma, big.expand_as(sigma))
    return rgb, sigma, inbox


def run_model_points(planes, osg, coords, box_warp: float):
    """ImportanceRenderer._run_model (renderer.py:310-322): planes (3,C,H,W); coords (P,3) ->
    rgb (P,3), sigma (P,1).  No in-box filter (that lives in _forward_pass, not here)."""
    rgb, sigma, _ = run_model(planes, osg, coords, {"box_warp": box_warp, "sampler_bbox_min": 0.0,
                                                    "sampler_bbox_max": 0.0, "filter_out_of_bbox": False})
    return rgb, sigma


def grid_points(aabb_min, aabb_max, grid_size: int) -> torch.Tensor:
    """The lattice of triplane_decode_grid (vit/vit_triplane.py:2092-2108): per-axis torch.linspace,
    meshgrid 'ij', stacked and flattened -> (G^3, 3)."""
    axes = [torch.linspace(float(aabb_min[d]), float(aabb_max[d]), grid_size) for d in range(3)]
    return torch.stack(torch.meshgrid(*axes, indexing="ij"), dim=-1).reshape(-1, 3)


def ray_march(colors, densities, depths, white_back=True, dmin=None, dmax=None):
    """MipRayMarcher2.run_forward on (R,S,3), (R,S,1), (R,S,1)."""
    deltas = depths[:, 1:] - depths[:, :-1]
    c_mid = (colors[:, :-1] + colors[:, 1:]) / 2
    s_mid = (densities[:, :-1] + densities[:, 1:]) / 2
    z_mid = (depths[:, :-1] + depths[:, 1:]) / 2
    s_mid = F.softplus(s_mid - 1)
    alpha = 1 - torch.exp(-(s_mid * deltas))
    shifted = torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], 1)
    T = torch.cumprod(shifted, 1)
    w = alpha * T[:, :-1]
    rgb = (w * c_mid).sum(1)
    wt = w.sum(1)
    depth = (w * z_mid).sum(1)
    depth = torch.nan_to_num(depth, float("inf"))
    depth = torch.clamp(depth, depths.min() if dmin is None else dmin,
                        depths.max() if dmax is None else dmax)
    if white_back:
        rgb = rgb + 1 - wt
    rgb = rgb * 2 - 1
    return rgb, depth, w


def sample_importance(z, w, n_imp, u):
    """z (R,S), w (R,S-1) coarse weights, u (R,n_imp) uniform noise -> (R,n_imp) fine depths."""
    w = F.max_pool1d(w.unsqueeze(1), 2, 1, padding=1)
    w = F.avg_pool1d(w, 2, 1).squeeze(1) + 0.01
    z_mid = 0.5 * (z[:, :-1] + z[:, 1:])
    bins, wts = z_mid, w[:, 1:-1]  # 63 bins for 61 weights -- reference quirk (renderer.py:497-501)
    eps = 1e-5
    n = wts.shape[1]
    wts = wts + eps
    pdf = wts / wts.sum(-1, keepdim=True)
    cdf = torch.cat([torch.zeros_like(pdf[:, :1]), torch.cumsum(pdf, -1)], -1)
    inds = torch.searchsorted(cdf, u.contiguous(), right=True)
    below = (inds - 1).clamp_min(0)
    above = inds.clamp_max(n)
    c0, c1 = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    b0, b1 = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    den = c1 - c0
    den = torch.where(den < eps, torch.ones_like(den), den)
    return b0 + (u - c0) / den * (b1 - b0), inds


def render_rays(planes, osg, ray_o, ray_d, opts, noise_coarse, noise_fine, return_debug=False):
    """One reference call of ImportanceRenderer.forward with batch 1.
    planes (3,C,H,W); ray_o/ray_d (M,3); noise_coarse (M,S); noise_fine (M,S_imp).
    Returns dict(rgb (M,3), depth (M,1), weights (M,1))."""
    S, S_imp = opts["depth_resolution"], opts["depth_resolution_importance"]
    M = ray_o.shape[0]
    assert opts["ray_start"] == opts["ray_end"] == "auto"
    start, end = ray_limits_box(ray_o, ray_d, opts["box_warp"])
    valid = end > start
    if bool(valid.any()):
        smin, smax = start[valid].min(), start[valid].max()
        start = torch.where(valid, start, smin.expand_as(start))
        end = torch.where(valid, end, smax.expand_as(end))  # max of valid *starts* (reference quirk)
    steps = torch.arange(S, dtype=torch.float32) / (S - 1)
    z_c = start + steps[None, :] * (end - start)  # (M,S)
    delta = (end - start) / (S - 1)
    z_c = z_c + noise_coarse * delta
    pts = ray_o[:, None, :] + z_c[:, :, None] * ray_d[:, None, :]
    rgb_c, sig_c, inbox_c = run_model(planes, osg, pts.reshape(-1, 3), opts)
    rgb_c, sig_c = rgb_c.reshape(M, S, 3), sig_c.reshape(M, S, 1)
    _, _, w_c = ray_march(rgb_c, sig_c, z_c[:, :, None], opts["white_back"])
    z_f, inds = sample_importance(z_c, w_c[:, :, 0], S_imp, noise_fine)
    pts_f = ray_o[:, None, :] + z_f[:, :, None] * ray_d[:, None, :]
    rgb_f, sig_f, inbox_f = run_model(planes, osg, pts_f.reshape(-1, 3), opts)
    rgb_f, sig_f = rgb_f.reshape(M, S_imp, 3), sig_f.reshape(M, S_imp, 1)
    z_all = torch.cat([z_c, z_f], 1)
    order = torch.sort(z_all, dim=1, stable=True)[1]
    z_all = torch.gather(z_all, 1, order)
    rgb_all = torch.gather(torch.cat([rgb_c, rgb_f], 1), 1, order[:, :, None].expand(-1, -1, 3))
    sig_all = torch.gather(torch.cat([sig_c, sig_f], 1), 1, order[:, :, None])
    rgb, depth, w = ray_march(rgb_all, sig_all, z_all[:, :, None], opts["white_back"])
    out = dict(rgb=rgb, depth=depth, weights=w.sum(1))
    if return_debug:
        out.update(valid=valid[:, 0], start=start[:, 0], end=end[:, 0], z_coarse=z_c, z_fine=z_f,
                   inbox_coarse=inbox_c.reshape(M, S), inbox_fine=inbox_f.reshape(M, S_imp),
                   inds=inds, order=order, sigma_coarse=sig_c[:, :, 0], w_coarse=w_c[:, :, 0])
    return out


def render_group(planes_per_view, osg, ray_o, ray_d, noise_coarse, noise_fine, opts):
    """One reference call of ImportanceRenderer.forward with batch N: view n samples planes_per_view[n], and
    the call's two global reductions are taken over all N*M rays -- the invalid-ray start/end fix-up
    (renderer.py:151-155) and the depth clamp range (ray_marcher.py:59-61).
    planes_per_view (N,3,C,H,W); ray_o/ray_d (N,M,3); noise_coarse (N,M,S); noise_fine (N,M,S_imp).
    Runs in the dtype of its inputs (float64 inputs: a float64 reference).
    Returns dict(rgb (N,M,3), depth (N,M,1), weights (N,M,1), valid (N,M))."""
    S, S_imp = opts["depth_resolution"], opts["depth_resolution_importance"]
    N, M, _ = ray_o.shape
    assert opts["ray_start"] == opts["ray_end"] == "auto"
    start, end = ray_limits_box(ray_o, ray_d, opts["box_warp"])  # (N,M,1)
    valid = end > start
    if bool(valid.any()):
        smin, smax = start[valid].min(), start[valid].max()
        start = torch.where(valid, start, smin.expand_as(start))
        end = torch.where(valid, end, smax.expand_as(end))
    steps = torch.arange(S, dtype=torch.float32).to(start.dtype) / (S - 1)
    z_all, rgb_all, sig_all = [], [], []
    for n in range(N):
        o, d, s, e = ray_o[n], ray_d[n], start[n], end[n]
        z_c = s + steps[None, :] * (e - s) + noise_coarse[n] * ((e - s) / (S - 1))
        pts = o[:, None, :] + z_c[:, :, None] * d[:, None, :]
        rgb_c, sig_c, _ = run_model(planes_per_view[n], osg, pts.reshape(-1, 3), opts)
        rgb_c, sig_c = rgb_c.reshape(M, S, 3), sig_c.reshape(M, S, 1)
        _, _, w_c = ray_march(rgb_c, sig_c, z_c[:, :, None], opts["white_back"])
        z_f, _ = sample_importance(z_c, w_c[:, :, 0], S_imp, noise_fine[n])
        pts_f = o[:, None, :] + z_f[:, :, None] * d[:, None, :]
        rgb_f, sig_f, _ = run_model(planes_per_view[n], osg, pts_f.reshape(-1, 3), opts)
        z = torch.cat([z_c, z_f], 1)
        order = torch.sort(z, dim=1, stable=True)[1]
        z_all.append(torch.gather(z, 1, order))
        rgb_all.append(torch.gather(torch.cat([rgb_c, rgb_f.reshape(M, S_imp, 3)], 1), 1,
                                    order[:, :, None].expand(-1, -1, 3)))
        sig_all.append(torch.gather(torch.cat([sig_c, sig_f.reshape(M, S_imp, 1)], 1), 1, order[:, :, None]))
    # one march over all N*M rays: its depth clamp takes min / max of every view's sorted depths
    rgb, depth, w = ray_march(torch.cat(rgb_all), torch.cat(sig_all), torch.cat(z_all)[:, :, None],
                              opts["white_back"])
    return dict(rgb=rgb.reshape(N, M, 3), depth=depth.reshape(N, M, 1), weights=w.sum(1).reshape(N, M, 1),
                valid=valid[..., 0])


def render_view(planes, osg, cam: torch.Tensor, res: int, opts, noise_coarse, noise_fine):
    """Triplane.forward for one camera row (25,): returns image_raw (3,res,res), image_depth
    (1,res,res), weights_samples (1,res,res), image_mask (1,res,res)."""
    c2w = cam[:16].reshape(1, 4, 4)
    K = cam[16:25].reshape(1, 3, 3)
    o, d = generate_rays(c2w, K, res)
    r = render_rays(planes, osg, o[0], d[0], opts, noise_coarse, noise_fine)
    img = r["rgb"].t().reshape(3, res, res)
    depth = r["depth"].t().reshape(1, res, res)
    wts = r["weights"].t().reshape(1, res, res)
    return dict(image_raw=img, image_depth=depth, weights_samples=wts,
                image_mask=wts * (1 + 2 * 0.001) - 0.001)
