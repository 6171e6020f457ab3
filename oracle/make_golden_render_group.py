"""TEST INFRASTRUCTURE.  Golden vectors for a batched renderer call, produced by the reference's own code run in
the build container:

  render_group.npz   ImportanceRenderer.forward (nsr/volumetric_rendering/renderer.py:133-307, Objaverse preset)
                     on the batch of 3 objects / 3 views of oracle.fixtures.render_group_inputs with explicit noise.
                     One call: the invalid-ray start range (renderer.py:151-155) and the depth clamp range
                     (ray_marcher.py:59-61) are shared by the three views, and view 0 holds rays whose slab test
                     yields NaN (origin on a face, zero direction component), which the reference treats as
                     invalid.

Run:  python oracle/make_golden_render_group.py   (needs /root/reference; writes tests/golden/render_group.npz)
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import _stubs  # noqa: E402  (stubs for the reference's absent third-party imports)

_stubs.install()
sys.path.insert(0, "/root/reference")
from oracle import fixtures as fx  # noqa: E402
from oracle.render import OBJAVERSE_OPTS  # noqa: E402


def main():
    from nsr.volumetric_rendering.renderer import ImportanceRenderer
    planes, osg, o, d, nc, nf = fx.render_group_inputs()
    w1, b1, w2, b2 = osg

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
        r = ImportanceRenderer()(planes, Dec(), o.clone(), d.clone(), dict(OBJAVERSE_OPTS))
    finally:
        torch.rand_like, torch.rand = orl, orr
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "render_group.npz"),
                        ray_o=o.numpy(), ray_d=d.numpy(), rgb=r["feature_samples"].numpy(),
                        depth=r["depth_samples"].numpy(), weights=r["weights_samples"].numpy())
    print("render_group depth[:, :3]", r["depth_samples"][:, :3, 0].tolist())


if __name__ == "__main__":
    main()
