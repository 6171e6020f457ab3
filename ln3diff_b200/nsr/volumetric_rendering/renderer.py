"""Mirror of reference nsr/volumetric_rendering/renderer.py:127-552 (ImportanceRenderer).

`ImportanceRenderer.forward(planes (N,3,C,H,W), decoder, ray_origins, ray_directions,
rendering_options, return_meta=False)` keeps the reference signature, return keys, RNG consumption
(one torch.rand_like of (N,M,S,1) then one torch.rand of (N*M,S) on the compute device,
renderer.py:464,530) and the per-call global reductions; the arithmetic is one call of the fused
ln3_render_views kernel.  The per-sample "details" tensors the reference also returns for its
training losses (coarse/fine coords and densities, all_coords, feature_volume, per-sample weights:
~100 MB per view) are not materialised: those dict entries are None."""
import torch

from ... import ops


def generate_planes():
    """reference renderer.py:26-36 (kept for API parity; the kernel hard-codes xy / yz / zx)."""
    return torch.tensor([[[1, 0, 0], [0, 1, 0], [0, 0, 1]], [[1, 0, 0], [0, 0, 1], [0, 1, 0]],
                         [[0, 0, 1], [1, 0, 0], [0, 1, 0]]], dtype=torch.float32)


class ImportanceRenderer(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.plane_axes = generate_planes()
        self._cl_cache = None   # (planes tensor (strong ref), its _version, channels-last copy)

    @staticmethod
    def _check_options(o):
        if not (o.get("ray_start") == o.get("ray_end") == "auto"):
            raise NotImplementedError("libln3b200 renders the Objaverse preset: ray_start = ray_end = 'auto'")
        S = o.get("depth_resolution")
        if S not in (64, 96) or o.get("depth_resolution_importance") != S:
            raise NotImplementedError("libln3b200 renders 64 + 64 or 96 + 96 coarse + importance samples per ray")
        if o.get("disparity_space_sampling", False) or o.get("clamp_mode", "softplus") != "softplus":
            raise NotImplementedError("unsupported sampling / clamp mode")
        if not o.get("filter_out_of_bbox", False):
            raise NotImplementedError("libln3b200 applies the Objaverse in-box filter")
        if o.get("density_noise", 0) > 0:
            raise NotImplementedError("density_noise is a training-time option")

    def _planes_cl(self, planes):
        """Channels-last copy of `planes`, reused while the caller keeps passing the same, unmodified tensor
        object (one object is rendered from many cameras, one `forward` per view,
        nsr/train_util_diffusion.py:292-302).  Identity + version, with the tensor kept alive: a different
        object's planes at a recycled address can never hit."""
        c = self._cl_cache
        if c is None or c[0] is not planes or c[1] != planes._version:
            c = self._cl_cache = (planes, planes._version, ops.planes_to_channels_last(planes.float().contiguous()))
        return c[2]

    @torch.no_grad()
    def forward(self, planes, decoder, ray_origins, ray_directions, rendering_options, return_meta=False):
        """rendering_options['osg_mlp_tf32'] (extension, default True): evaluate the 32->64->4 OSG MLP on the
        tensor cores with TF32 operands / fp32 accumulation (pixels within 1e-4 rel-L2 of the fp32 result,
        1.26x faster); False selects the exact fp32 SIMT path."""
        if not planes.is_cuda:
            raise RuntimeError("ln3diff_b200 ImportanceRenderer runs on CUDA only (no CPU fallback)")
        self._check_options(rendering_options)
        N, M, _ = ray_origins.shape
        S = rendering_options["depth_resolution"]
        # same draws, order, shapes and generator device as the reference
        noise_c = torch.rand_like(torch.empty((N, M, S, 1), device=ray_origins.device, dtype=torch.float32))
        noise_f = torch.rand(N * M, rendering_options["depth_resolution_importance"], device=ray_origins.device)
        w1, b1, w2, b2 = decoder.raw_parameters()
        out = ops.render_views(self._planes_cl(planes), ray_origins.float().contiguous(),
                               ray_directions.float().contiguous(), noise_c.reshape(N, M, S), noise_f, (w1, b1, w2, b2),
                               views_per_obj=1, group_size=N,
                               box_warp=rendering_options["box_warp"],
                               bbox_min=rendering_options["sampler_bbox_min"],
                               bbox_max=rendering_options["sampler_bbox_max"],
                               white_back=rendering_options.get("white_back", True),
                               mlp_tf32=rendering_options.get("osg_mlp_tf32", True), samples_per_ray=S)
        depth = out["depth"].permute(0, 2, 1)
        shape_synthesized = {"depth": depth}
        ret = {"feature_samples": out["rgb"].permute(0, 2, 1), "depth_samples": depth,
               "weights_samples": out["weights"].permute(0, 2, 1), "shape_synthesized": shape_synthesized,
               "visibility": None}
        if return_meta:
            ret.update({"all_coords": None, "feature_volume": None, "weights": None})
        return ret

    @torch.no_grad()
    def _run_model(self, planes, decoder, sample_coordinates, sample_directions, options):
        """Point queries (reference renderer.py:310-322): tri-plane gather + OSG decoder at
        `sample_coordinates` (N, P, 3); `sample_directions` is unused by OSGDecoder (nsr/triplane.py:356).
        `planes` is (N, 3, C, H, W) / (N, 3*C, H, W) NCHW, or (N, 3, H, W, C) channels-last when it comes
        from `decode_to_channels_last`.  Returns {'rgb': (N,P,3), 'sigma': (N,P,1)} with no in-box filter."""
        if not planes.is_cuda:
            raise RuntimeError("ln3diff_b200 ImportanceRenderer runs on CUDA only (no CPU fallback)")
        if options.get("density_noise", 0) > 0:
            raise NotImplementedError("density_noise is a training-time option")
        sigma, rgb = ops.query_points(self._as_channels_last(planes), decoder.raw_parameters(),
                                      points=sample_coordinates.float().contiguous(), box_warp=options["box_warp"],
                                      mlp_tf32=options.get("osg_mlp_tf32", True))
        return {"rgb": rgb, "sigma": sigma}

    def _as_channels_last(self, planes):
        if planes.dim() == 5 and planes.shape[-1] == 32 and planes.shape[2] != 32:
            return planes.contiguous()                      # already (N,3,H,W,32)
        if planes.dim() == 4:
            planes = planes.reshape(planes.shape[0], 3, -1, planes.shape[-2], planes.shape[-1])
        return self._planes_cl(planes)

