"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/dit_t23d_xl.npz by running the REFERENCE's own code.

Runs only in the build container (needs /root/reference, read-only; third-party gaps are filled by
oracle/_stubs.py).  Nothing is copied from the reference: the fixture holds the output the reference's
DiT_TriLatent produces at DiT-XL/2 width (hidden 1152, 16 heads of 72, TextCondDiTBlock, whose cross-attention
keeps 64-wide heads: inner width 1024) and depth 2 for the seeded inputs of oracle.fixtures.dit_inputs and the
key-seeded state_dict of oracle.dit.synth_state_dict, as oracle/make_golden.py does for dit_t23d.npz.
Re-run:  python -m oracle.make_golden_xl
"""
from __future__ import annotations

import contextlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import _stubs  # noqa: E402
from oracle import dit as odit  # noqa: E402
from oracle import fixtures as fx  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
XL_DEPTH = 2


def main():
    _stubs.install()
    os.makedirs(OUT, exist_ok=True)
    import dit.dit_models_xformers as dmx
    _stubs.patch_dit_namespace()
    import dit.dit_trilatent as dt

    with contextlib.redirect_stdout(io.StringIO()):
        ref = dt.DiT_TriLatent(depth=XL_DEPTH, hidden_size=1152, patch_size=2, num_heads=16, input_size=32,
                               num_classes=0, learn_sigma=False, in_channels=4, context_dim=768, roll_out=True,
                               vit_blk=dmx.TextCondDiTBlock)
    ref.eval()
    shapes = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    sd = odit.synth_state_dict(shapes, seed=7, keep={"pos_embed": ref.state_dict()["pos_embed"]})
    ref.load_state_dict(sd)
    x, t, ctx = fx.dit_inputs()
    with torch.no_grad():
        y = ref(x, t, {"crossattn": ctx})
    np.savez_compressed(os.path.join(OUT, "dit_t23d_xl.npz"), out=y.numpy(), t=t.numpy(),
                        pos_embed_checksum=np.float64(ref.state_dict()["pos_embed"].double().sum().item()))
    print("dit_t23d_xl", y.shape, float(y.abs().max()))


if __name__ == "__main__":
    main()
