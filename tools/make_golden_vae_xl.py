"""TEST INFRASTRUCTURE.  Writes tests/golden/vae_xl.npz from the reference's OWN code (a reference checkout is needed;
its path is the first argument, default oracle/_stubs.REFERENCE_ROOT), on the CPU in fp32, for the DiT2-L/2 VAE of
the release (scripts/vae_xl_reconstruction.sh, dino_version 'mv-sd-dit-dynaInp-trilatent', num_frames 6):

  * MVEncoderGSDynamicInp (ldm/modules/diffusionmodules/model.py:604-623) as create_3DAE_model builds it with the
    release scripts' sd_E_ch=64, sd_E_num_res_blocks=1, loaded with the seeded weights of tests/vae_encoder_oracle.py
    (drawn over this encoder's own key table), on 2 objects x 6 views of the seeded 256^2 inputs of that file: the
    state_dict key -> shape table, the moments (2, 24, 32, 32) and object 0's mid-block SpatialTransformer3D output
    (every 8th pixel);
  * ImportanceRenderer.forward (nsr/volumetric_rendering/renderer.py:133-307) with the rendering options the
    reference's own rendering_options_defaults resolves for cfg 'objverse_tuneray_aug_resolution_96_96_auto'
    (96 + 96 samples per ray), on the planes, OSG weights and edge / missing rays of
    oracle.fixtures.render_group_inputs as one batch-3 call, with seeded (3, 36, 96) noise injected in place of the
    reference's torch.rand_like / torch.rand draws (stored, as are the rays).
Weights and encoder inputs are regenerated from their seeds, not stored.

Run:  python tools/make_golden_vae_xl.py [REFERENCE_ROOT]
"""
import contextlib
import io
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import _stubs  # noqa: E402

REF = sys.argv[1] if len(sys.argv) > 1 else _stubs.REFERENCE_ROOT

_stubs.install(REF)
_stubs.patch_dit_namespace()
import vae_encoder_oracle as vo  # noqa: E402
from oracle import fixtures as fx  # noqa: E402

NUM_FRAMES = 6
N_OBJ = 2
CFG = "objverse_tuneray_aug_resolution_96_96_auto"
NOISE_SEED = 61


def encoder_inputs():
    """2 objects x 6 views: the first 12 views of vae_encoder_oracle.enc_inputs (its generator draws 4 views per
    object, so 3 of its objects)."""
    return vo.enc_inputs(n_obj=N_OBJ * NUM_FRAMES // vo.VIEWS)


def _encoder():
    from ldm.modules.diffusionmodules.model import MVEncoderGSDynamicInp
    return MVEncoderGSDynamicInp(double_z=True, resolution=256, in_channels=vo.IN_CH, ch=vo.CH,
                                 ch_mult=list(vo.CH_MULT), num_res_blocks=vo.NUM_RES_BLOCKS, num_frames=NUM_FRAMES,
                                 dropout=0.0, attn_resolutions=[], out_ch=3, z_channels=vo.Z_CH,
                                 attn_kwargs={"n_heads": vo.HEADS, "d_head": vo.D_HEAD})


def rendering_options():
    """The reference's rendering_options_defaults for the 96_96 preset, with the triplane_decoder_defaults it reads."""
    from nsr.script_util import rendering_options_defaults
    opts = dict(cfg=CFG, density_reg=0.25, density_reg_p_dist=0.004, reg_type="l1", c_scale=1,
                patch_rendering_resolution=45)
    return rendering_options_defaults(type("Opts", (), opts)())


def _render(opts):
    from nsr.volumetric_rendering.renderer import ImportanceRenderer
    planes, osg, o, d, _, _ = fx.render_group_inputs()
    w1, b1, w2, b2 = osg
    S = opts["depth_resolution"]
    g = torch.Generator().manual_seed(NOISE_SEED)
    nc = torch.rand(o.shape[0], o.shape[1], S, generator=g)
    nf = torch.rand(o.shape[0], o.shape[1], opts["depth_resolution_importance"], generator=g)

    class Dec(torch.nn.Module):  # OSGDecoder arithmetic (nsr/triplane.py:356-375) on raw tensors
        decoder_output_dim = 3

        def forward(self, feats, dirs):
            v = feats.mean(1)
            N, M, C = v.shape
            v = v.view(N * M, C)
            h = torch.nn.functional.softplus(torch.addmm(b1.unsqueeze(0), v, (w1 * (1 / np.sqrt(32))).t()))
            yy = torch.addmm(b2.unsqueeze(0), h, (w2 * (1 / np.sqrt(64))).t()).view(N, M, -1)
            return {"rgb": torch.sigmoid(yy[..., 1:]) * (1 + 2 * 0.001) - 0.001, "sigma": yy[..., 0:1]}

    orl, orr = torch.rand_like, torch.rand
    torch.rand_like = lambda tt, *a, **k: nc.reshape(tt.shape)   # renderer.py:464, (N,M,S,1)
    torch.rand = lambda *s, **k: nf.reshape(*s)                  # renderer.py:530, (N*M,S_imp)
    try:
        r = ImportanceRenderer()(planes, Dec(), o.clone(), d.clone(), dict(opts))
    finally:
        torch.rand_like, torch.rand = orl, orr
    return dict(render_ray_o=o.numpy(), render_ray_d=d.numpy(), render_noise_coarse=nc.numpy(),
                render_noise_fine=nf.numpy(), render_rgb=r["feature_samples"].numpy(),
                render_depth=r["depth_samples"].numpy(), render_weights=r["weights_samples"].numpy())


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out = {}
    with contextlib.redirect_stdout(io.StringIO()):
        enc = _encoder()
    enc.eval()
    shapes = {k: list(v.shape) for k, v in enc.state_dict().items()}
    out["encoder_shapes"] = np.array(json.dumps(shapes))
    enc.load_state_dict(vo.enc_state_dict(shapes))
    mids = []
    hook = enc.mid.attn_1.register_forward_hook(lambda m, i, o: mids.append(o))
    with torch.no_grad():
        moments = enc(encoder_inputs())
    hook.remove()
    assert moments.shape == (N_OBJ, 24, 32, 32)
    out["moments"] = moments.numpy()
    out["mid_obj0_strided"] = mids[0][:NUM_FRAMES, :, ::vo.MID_STRIDE, ::vo.MID_STRIDE].contiguous().numpy()
    opts = rendering_options()
    assert opts["depth_resolution"] == opts["depth_resolution_importance"] == 96
    out["rendering_options"] = np.array(json.dumps(opts, sort_keys=True))
    out.update(_render(opts))
    path = os.path.join(ROOT, "tests", "golden", "vae_xl.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
