"""TEST INFRASTRUCTURE.  Writes tests/golden/vae_encoder.npz from the reference's OWN code (a reference checkout is
needed; its path is the first argument, default oracle/_stubs.REFERENCE_ROOT), on the CPU in fp32:

  * MVEncoder (ldm/modules/diffusionmodules/model.py:563-577) as create_3DAE_model builds it for 'mv-sd-dit' with the
    release scripts' sd_E_ch=64, sd_E_num_res_blocks=1, loaded with the seeded weights of tests/vae_encoder_oracle.py
    (every tensor random, including the zero-initialised proj_out), on 2 objects x 4 views of seeded 256^2 inputs:
    the moments (2, 24, 32, 32) and, for object 0, the output of the mid-block SpatialTransformer3D (every 8th pixel);
  * vae_reparameterization of the `_S` decoder (vit/vit_triplane.py:1786-1834) on those moments with seeded quant_conv
    weights, after torch.manual_seed(NOISE_SEED): mean / logvar / z of object 0 and the returned dict's keys;
  * the state_dict key -> shape tables of the reference MVEncoder and of the `_S` decoder with DiT2-B/2 and DiT2-L/2
    (constructed on the meta device).
Inputs and weights are regenerated from their seeds, not stored.

Run:  python tools/make_golden_vae_encoder.py [REFERENCE_ROOT]
"""
import contextlib
import io
import json
import os
import sys
import types

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


def _encoder():
    from ldm.modules.diffusionmodules.model import MVEncoder
    return MVEncoder(double_z=True, resolution=256, in_channels=vo.IN_CH, ch=vo.CH, ch_mult=list(vo.CH_MULT),
                     num_res_blocks=vo.NUM_RES_BLOCKS, num_frames=vo.VIEWS, dropout=0.0, attn_resolutions=[], out_ch=3,
                     z_channels=vo.Z_CH, attn_kwargs={"n_heads": vo.HEADS, "d_head": vo.D_HEAD})


def _decoder_shapes(arch):
    """Key -> shape of the reference `_S` decoder as create_3DAE_model assembles it (nsr/script_util.py:1355-1429)."""
    import vit.vit_triplane as vt
    from dit.dit_decoder import DiT2_models
    from nsr.triplane import Triplane
    from ln3diff_b200.utils import OBJAVERSE_RENDERING_KWARGS
    D = {"DiT2-B/2": 768, "DiT2-L/2": 1024}[arch]
    with torch.device("meta"):
        vd = DiT2_models[arch](input_size=16, num_classes=0, learn_sigma=False, in_channels=D, mixed_prediction=False,
                               context_dim=None, roll_out=True, plane_n=3, return_all_layers=False)
        tri = Triplane(25, 128, 3, rendering_kwargs=dict(OBJAVERSE_RENDERING_KWARGS), out_chans=96, triplane_size=224,
                       decoder_in_chans=32, decoder_output_dim=3)
        dec = vt.RodinSR_256_fusionv6_ConvQuant_liteSR_dinoInit3DAttn_SD_B_3L_C_withrollout_withSD_D_ditDecoder_S(
            vit_decoder=vd, triplane_decoder=tri, cls_token=False, sr_ratio=2, vae_p=2, ldm_z_channels=4,
            ldm_embed_dim=4)
    return {k: list(v.shape) for k, v in dec.state_dict().items()}


def _reparameterization(moments):
    """The `_S` class's own vae_reparameterization / vae_encode bound to a stand-in holding only what they read."""
    import vit.vit_triplane as vt
    cls = vt.RodinSR_256_fusionv6_ConvQuant_liteSR_dinoInit3DAttn_SD_B_3L_C_withrollout_withSD_D_ditDecoder_S
    me = torch.nn.Module()
    qc = torch.nn.Conv2d(24, 24, 1, groups=3)
    qw, qb = vo.quant_conv_params()
    qc.weight.data.copy_(qw)
    qc.bias.data.copy_(qb)
    me.superresolution = torch.nn.ModuleDict(dict(quant_conv=qc))
    me.plane_n, me.reparameterization_soft_clamp, me.vae_p, me.token_size, me.ldm_z_channels = 3, True, 2, 16, 4
    me.vae_encode = types.MethodType(cls.vae_encode, me)
    torch.manual_seed(vo.NOISE_SEED)
    with torch.no_grad():
        return cls.vae_reparameterization(me, moments, True)


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
    x = vo.enc_inputs()
    with torch.no_grad():
        moments = enc(x)
    hook.remove()
    assert moments.shape == (vo.N_OBJ, 24, 32, 32)
    out["moments"] = moments.numpy()
    out["mid_obj0_strided"] = mids[0][:vo.VIEWS, :, ::vo.MID_STRIDE, ::vo.MID_STRIDE].contiguous().numpy()
    ret = _reparameterization(moments)
    post = ret["posterior"]
    L = 32 * 32
    out["mean_obj0"] = post.mean[:1].reshape(1, 12, 32, 32).numpy()
    out["logvar_obj0"] = post.logvar[:1].reshape(1, 12, 32, 32).numpy()
    out["z_obj0"] = ret["latent_normalized_2Ddiffusion"][:1].numpy()
    out["log_q_obj0"] = ret["log_q_2Ddiffusion"][:1].numpy()
    out["ret_keys"] = np.array(json.dumps(sorted(ret.keys())))
    assert ret["latent_normalized"].shape == (vo.N_OBJ, 3 * L, 4)
    for arch in ("DiT2-B/2", "DiT2-L/2"):
        with contextlib.redirect_stdout(io.StringIO()):
            out["decoder_shapes_" + arch.split("-")[1][0]] = np.array(json.dumps(_decoder_shapes(arch)))
    path = os.path.join(ROOT, "tests", "golden", "vae_encoder.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
