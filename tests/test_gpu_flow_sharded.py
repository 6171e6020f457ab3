"""GPU: sharded image- and multi-view-to-3D (pipeline.images_to_3d_sharded / mvs_to_3d_sharded) against the
single-process pipelines.  One rank with one batch is images_to_3d / mvs_to_3d bit for bit (aug_c on); smaller
batches keep every condition's latents within the batched tolerance of its own image_to_3d call, and each batch's
frames are FrameSink.pack of the single-process renders for the same render noise.  A two-rank NCCL run needs two
GPUs and is skipped otherwise."""
import datetime
import os
import random

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

S, RES = 2, 32


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "-m gpu tests need a GPU"
    from ln3diff_b200 import _lib
    _lib.lib()
    return torch.device("cuda", 0)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


def _stub_image_embedder(dev):
    """A deterministic stand-in for the I23D image conditioner: (1, 3, H, W) -> tokens (1, 256, 2048) and a pooled
    (1, 768) embedding, both functions of the image."""
    from ln3diff_b200.sgm.modules.encoders.modules import AbstractEmbModel

    class Stub(AbstractEmbModel):
        def __init__(self):
            super().__init__()
            g = torch.Generator().manual_seed(4)
            self.wt = torch.randn(48, 256 * 8, generator=g).to(dev)
            self.wp = torch.randn(48, 768, generator=g).to(dev)

        def forward(self, img):
            feat = torch.nn.functional.adaptive_avg_pool2d(img.float(), 4).flatten(1)
            tok = torch.sin(feat @ self.wt).reshape(-1, 256, 8).repeat(1, 1, 256)
            return tok, torch.cos(feat @ self.wp)

    emb = Stub()
    emb._emb_config = {"input_key": "img", "ucg_rate": 0.0}
    return emb


def _i23d_parts(dev):
    from ln3diff_b200.sgm.modules.encoders.modules import GeneralConditioner
    from ln3diff_b200.utils import build_ae_decoder, build_i23d, orbit_cameras
    return (GeneralConditioner([_stub_image_embedder(dev)]), build_i23d("DiT-PixArt-B/2", device=dev),
            build_ae_decoder("DiT2-S/2", device=dev), orbit_cameras(30).to(dev))


def _images(P):
    return torch.rand(P, 3, 64, 64, generator=torch.Generator().manual_seed(13)) * 2 - 1


@pytest.fixture(scope="module")
def i23d(dev):
    return _i23d_parts(dev)


def _pack(dev, image_raw):
    from ln3diff_b200.frames import FrameSink
    return FrameSink(dev).pack(image_raw)


def test_one_rank_one_batch_is_images_to_3d_bit_for_bit(dev, i23d):
    from ln3diff_b200 import pipeline
    cond, m, dec, cams = i23d
    imgs = _images(3)
    lat, out, st = pipeline.images_to_3d(cond, m, dec, imgs, cams, num_samples=S, resolution=RES)
    sh = pipeline.images_to_3d_sharded(cond, m, dec, imgs, cams, num_samples=S, resolution=RES, batch=8)
    assert sh["shard"] == (0, 3) and sh["gather_bytes_per_rank"] == 0
    assert torch.equal(sh["latents"], lat)
    assert torch.equal(sh["frames_all"], _pack(dev, out["image_raw"])) and torch.equal(sh["frames"], sh["frames_all"])
    assert sh["frames_all"].shape == (3, S, 24, RES, RES, 3)
    for k in ("nfe", "accepted", "rejected"):
        assert sh["stats"][k] == st[k], k


def test_one_rank_one_batch_is_mvs_to_3d_bit_for_bit_with_aug_c(dev, i23d):
    """The release multi-view conditioner with aug_c=True, seeded: the same latents, frames and camera draws as
    mvs_to_3d, and both host generators end where mvs_to_3d leaves them."""
    from ln3diff_b200 import pipeline
    _, _, dec, cams = i23d
    P = 3
    cond, m, imgs, mv_cams = _mv_parts(dev, P)
    runs = []
    for sharded in (False, True):
        random.seed(5); np.random.seed(5)
        if sharded:
            sh = pipeline.mvs_to_3d_sharded(cond, m, dec, imgs, mv_cams, cams, num_samples=S, resolution=RES, batch=P)
            res = (sh["latents"], sh["frames_all"])
        else:
            lat, out, _ = pipeline.mvs_to_3d(cond, m, dec, imgs, mv_cams, cams, num_samples=S, resolution=RES)
            res = (lat, _pack(dev, out["image_raw"]))
        runs.append(res + ((random.random(), float(np.random.uniform())),))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert runs[0][2] == runs[1][2]


def _mv_parts(dev, P, V=3, W=256):
    from ln3diff_b200.sgm.modules.encoders.modules import FrozenDinov2ImageEmbedderMVPlucker, GeneralConditioner
    from ln3diff_b200.utils import build_mv23d, orbit_cameras
    emb = FrozenDinov2ImageEmbedderMVPlucker(arch="vitb", device=dev, n_cond_frames=V, enable_bf16=True, aug_c=True,
                                             random_init=True, width=W, depth=2, mlp_dim=4 * W, seed=3)
    emb._emb_config = {"input_key": "img-c", "ucg_rate": 0.0}
    m = build_mv23d(depth=2, hidden_size=384, num_heads=6, context_dim=W, device=dev)
    imgs = torch.rand(P, V, 3, 256, 256, generator=torch.Generator().manual_seed(12)) * 2 - 1
    mv_cams = torch.stack([orbit_cameras(V + i)[:V] for i in range(P)])
    return GeneralConditioner([emb]), m, imgs, mv_cams


def test_mvs_batches_smaller_than_the_shard_with_aug_c(dev, i23d):
    """P = 3 multi-view conditions with aug_c=True in batches of 2 + 1, seeded.  The camera draws of the second batch
    come after those of the first, so: each condition's latents are within the batched tolerance of mv_to_3d on that
    condition alone when the P calls run in order after the same seeds; each batch's latents and frames are those of
    mvs_to_3d over the batch's conditions, run in order after the same seeds, bit for bit; and both host generators
    end where those sequential calls leave them."""
    from ln3diff_b200 import pipeline
    _, _, dec, cams = i23d
    P = 3
    cond, m, imgs, mv_cams = _mv_parts(dev, P)
    kw = dict(num_samples=S, resolution=RES)
    seeded = lambda: (random.seed(5), np.random.seed(5))
    rng = lambda: (random.random(), float(np.random.uniform()))
    seeded()
    sh = pipeline.mvs_to_3d_sharded(cond, m, dec, imgs, mv_cams, cams, batch=2, **kw)
    rng_sh = rng()
    seeded()
    cam_d = [mv_cams[i:i + 1].clone().to(dev) for i in range(P)]          # mv_to_3d rotates these in place
    singles = [pipeline.mv_to_3d(cond, m, dec, imgs[i:i + 1], cam_d[i], cams, **kw)[0] for i in range(P)]
    assert rng() == rng_sh
    assert not torch.equal(torch.cat(cam_d).cpu(), mv_cams), "aug_c must have rotated some cameras"
    for i in range(P):
        rel = _rel(sh["latents"][i], singles[i])
        print(f"mv condition {i}: rel-L2 to mv_to_3d {rel:.3e}")
        assert rel <= 1e-2, i
    seeded()
    for i0, i1 in ((0, 2), (2, 3)):
        lat, out, _ = pipeline.mvs_to_3d(cond, m, dec, imgs[i0:i1], mv_cams[i0:i1], cams, **kw)
        assert torch.equal(sh["latents"][i0:i1], lat), i0
        assert torch.equal(sh["frames_all"][i0:i1], _pack(dev, out["image_raw"])), i0
    assert rng() == rng_sh


@pytest.mark.parametrize("method", ["dopri5", "rk4", "sde-euler"])
def test_batches_smaller_than_the_shard(dev, i23d, method):
    """P = 3 in batches of 2 + 1.  Each condition's latents are within the batched tolerance (rel-L2 1e-2, as between
    sample_flow_batched and sequential sample_flow calls) of image_to_3d on that image alone; each batch's latents and
    frames are those of images_to_3d over the batch's images, bit for bit (the same render noise: each batch's
    sample_flow_batched reseeds the generators)."""
    from ln3diff_b200 import pipeline
    cond, m, dec, cams = i23d
    kw = dict(num_samples=S, resolution=RES)
    if method == "rk4":
        kw.update(sampling_method="rk4", num_steps=6)
    elif method == "sde-euler":
        kw.update(sde={"sampling_method": "Euler"}, num_steps=6)
    P = 3
    imgs = _images(P)
    sh = pipeline.images_to_3d_sharded(cond, m, dec, imgs, cams, batch=2, **kw)
    assert sh["latents"].shape == (P, S, 12, 32, 32) and len(sh["stats"]["nfe"]) == P
    for i in range(P):
        lat, _ = pipeline.image_to_3d(cond, m, dec, imgs[i:i + 1], cams, **kw)
        rel = _rel(sh["latents"][i], lat)
        print(f"{method} condition {i}: rel-L2 to image_to_3d {rel:.3e}")
        assert rel <= 1e-2, (method, i)
    for i0, i1 in ((0, 2), (2, 3)):
        lat, out, st = pipeline.images_to_3d(cond, m, dec, imgs[i0:i1], cams, **kw)
        assert torch.equal(sh["latents"][i0:i1], lat), (method, i0)
        assert torch.equal(sh["frames_all"][i0:i1], _pack(dev, out["image_raw"])), (method, i0)
        assert sh["stats"]["nfe"][i0:i1] == st["nfe"]


# ------------------------------------------------------------------ two ranks over NCCL
def _nccl_worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300),
                            device_id=dev)
    from ln3diff_b200 import _lib, pipeline
    _lib.lib()
    cond, m, dec, cams = _i23d_parts(dev)
    sh = pipeline.images_to_3d_sharded(cond, m, dec, _images(3), cams, num_samples=S, resolution=RES, batch=1)
    ret[rank] = dict(latents=sh["latents"].cpu(), frames=sh["frames"].cpu(), frames_all=sh["frames_all"].cpu(),
                     shard=sh["shard"])
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="the two-rank NCCL run needs two GPUs")
def test_two_ranks_nccl_match_one_process(dev, i23d):
    """P = 3 on two ranks (2 + 1 images) in batches of 1: every rank holds every image's frames in image order, and
    each image's latents are within the batched tolerance of images_to_3d on one GPU."""
    from ln3diff_b200 import pipeline
    cond, m, dec, cams = i23d
    lat, _, _ = pipeline.images_to_3d(cond, m, dec, _images(3), cams, num_samples=S, resolution=RES)
    with mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_nccl_worker, args=(2, 35500 + os.getpid() % 2000, ret), nprocs=2, join=True)
        ret = dict(ret)
    assert ret[0]["shard"] == (0, 2) and ret[1]["shard"] == (2, 3)
    local = torch.cat([ret[0]["frames"], ret[1]["frames"]])
    for rank in (0, 1):
        assert torch.equal(ret[rank]["frames_all"], local), rank
        lo, hi = ret[rank]["shard"]
        for i in range(lo, hi):
            assert _rel(ret[rank]["latents"][i - lo], lat[i]) <= 1e-2, (rank, i)
