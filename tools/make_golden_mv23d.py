"""TEST INFRASTRUCTURE.  Writes tests/golden/mv23d.npz from the reference's OWN code (a reference checkout is needed;
its path is the first argument, default oracle/_stubs.REFERENCE_ROOT):

  * DiT_I23D_PixelArt_MVCond_noClip (dit/dit_i23d.py:392-492), built directly at reduced size (depth 3, D 768,
    head_dim 64, context_dim 768) on the seeded weights / inputs of tests/mv23d_oracle.py: `forward` and
    `forward_with_cfg(..., 4.0)`, the unconditional row of `concat` all zero;
  * the key -> shape table of the full `DiT-PixArt-MV-L/2` the registry builds (constructed on the meta device);
  * FrozenDinov2ImageEmbedderMVPlucker.get_plucker_ray on tests/mv23d_oracle.ray_cameras() (every 7th pixel kept),
    and its aug_c loop (:1084-1088) over random_rotate_c on a (2, 6, 25) camera batch with `random` /
    `np.random` seeded: the rotated cameras and the next draws of both generators.
    sgm/modules/encoders/modules.py imports kiui / open_clip / kornia, so its three methods are extracted with `ast`
    and executed with `autocast` as the identity (the CPU path of the reference: fp32 arithmetic).

Run:  python tools/make_golden_mv23d.py [REFERENCE_ROOT]
"""
import ast
import contextlib
import io
import json
import math
import os
import random
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
import mv23d_oracle as mo  # noqa: E402


def _reference_methods(names):
    """The named methods of FrozenDinov2ImageEmbedderMVPlucker, compiled from the reference file's own source."""
    path = os.path.join(REF, "sgm", "modules", "encoders", "modules.py")
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "FrozenDinov2ImageEmbedderMVPlucker")
    fns = [f for f in cls.body if isinstance(f, ast.FunctionDef) and f.name in names]
    assert sorted(f.name for f in fns) == sorted(names)
    ns = dict(torch=torch, np=np, math=math, random=random, autocast=lambda f: f)
    exec(compile(ast.Module(body=fns, type_ignores=[]), path, "exec"), ns)

    class Embedder:
        reso_encoder = 224
    for n in names:
        setattr(Embedder, n, ns[n])
    return Embedder()


def main():
    import dit.dit_i23d as di
    out = {}
    # ---------------------------------------------------------------- denoiser
    with contextlib.redirect_stdout(io.StringIO()):
        ref = di.DiT_I23D_PixelArt_MVCond_noClip(input_size=32, patch_size=2, in_channels=4, hidden_size=mo.MV_HIDDEN,
                                                 depth=mo.MV_DEPTH, num_heads=mo.MV_HEADS, num_classes=0,
                                                 learn_sigma=False, context_dim=mo.MV_CONTEXT, pooling_ctx_dim=768,
                                                 roll_out=True)
    ref.eval()
    assert type(ref.blocks[0]).__name__ == "ImageCondDiTBlockPixelArtRMSNormNoClip"
    shapes = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    ref.load_state_dict(mo.mv_state_dict(shapes, ref.state_dict()["pos_embed"]))
    x, t, ctx = mo.mv_inputs()
    with torch.no_grad():
        out["out"] = ref(x, t, ctx).numpy()
        out["out_cfg"] = ref.forward_with_cfg(x, t, ctx, 4.0).numpy()
    with contextlib.redirect_stdout(io.StringIO()), torch.device("meta"):
        full = di.DiT_models["DiT-PixArt-MV-L/2"](input_size=32, num_classes=0, learn_sigma=False, in_channels=4,
                                                  context_dim=768, pooling_ctx_dim=768, roll_out=True)
    assert type(full).__name__ == "DiT_I23D_PixelArt_MVCond_noClip"
    out["mv_l2_shapes"] = np.array(json.dumps({k: list(v.shape) for k, v in full.state_dict().items()}))

    # ---------------------------------------------------------------- rays and camera augmentation
    emb = _reference_methods(["gen_rays", "get_plucker_ray", "random_rotate_c"])
    cams = mo.ray_cameras()
    with torch.no_grad():
        rays = emb.get_plucker_ray(cams)
    out["ray_cams"] = cams.numpy()
    out["rays_strided"] = rays[:, :, ::7, ::7].contiguous().numpy()

    from ln3diff_b200.utils import orbit_cameras
    c = orbit_cameras(12).reshape(2, 6, 25).clone()
    out["aug_in"] = c.numpy().copy()
    random.seed(1234)
    np.random.seed(4321)
    for idx_b in range(c.shape[0]):                 # the aug_c loop of forward (:1084-1088)
        for idx_v in range(c.shape[1]):
            if random.random() > 0.6:
                c[idx_b, idx_v] = emb.random_rotate_c(c[idx_b, idx_v])
    out["aug_out"] = c.numpy()
    out["aug_next_py"] = np.array([random.random() for _ in range(4)])
    out["aug_next_np"] = np.random.uniform(size=4)
    path = os.path.join(ROOT, "tests", "golden", "mv23d.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes;", "rotated", int((out["aug_in"] != out["aug_out"]).any(-1).sum()), "of 12")


if __name__ == "__main__":
    main()
