"""CPU, world size 2 (gloo): pipeline.images_to_3d_sharded and mvs_to_3d_sharded with CPU stand-ins for the
conditioner towers and the three CUDA stages (sample / decode + render / pack).  Every condition is conditioned
exactly once, on the rank that owns it and in order; frames_all on every rank equals a single-process run, for an
even split, a ragged split, batches smaller than the shard and a rank that holds no condition; with aug_c every rank
gives its conditions the camera rotations a single process gives them, and leaves `random` / `np.random` where a
single process leaves them."""
import datetime
import os
import random

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from ln3diff_b200.sgm.modules.encoders.modules import (AbstractEmbModel, FrozenDinov2ImageEmbedder,
                                                       FrozenDinov2ImageEmbedderMVPlucker, GeneralConditioner)

N, V_RENDER, RES = 2, 3, 8


class _ImageStub(AbstractEmbModel):
    """An I23D image conditioner on the CPU: tokens (B, 4, 3) and a pooled (B, 6), functions of the image.  Records
    the condition id held in pixel [0, 0, 0] of every image it sees."""

    def __init__(self):
        super().__init__()
        self.seen = []

    def forward(self, img):
        self.seen.append(int(img[0, 0, 0, 0]))
        f = img.float().mean(dim=(2, 3))
        return f[:, None, :] * torch.arange(1.0, 5.0)[None, :, None], f.sum(1, keepdim=True).repeat(1, 6)


class _TowerStub(FrozenDinov2ImageEmbedder):
    """Stands in for the DINOv2 tower that FrozenDinov2ImageEmbedderMVPlucker.forward calls (never constructed as a
    tower): records the condition id and the (augmented) cameras it is given, and returns tokens made of them."""

    def forward(self, image, no_dropout=False, cams=None):
        self.seen.append((int(image[0, 0, 0, 0, 0]), cams.clone()))
        return cams.float()[:, None, :].repeat(1, 2, 1) + image.float().mean()


class _MVStub(FrozenDinov2ImageEmbedderMVPlucker, _TowerStub):
    """The multi-view conditioner's own forward (aug_c included) over the CPU tower stub."""


def _mv_embedder(V):
    e = _MVStub.__new__(_MVStub)
    AbstractEmbModel.__init__(e)
    e.aug_c, e.n_cond_frames, e.seen = True, V, []
    e._emb_config = {"input_key": "img-c", "ucg_rate": 0.0}
    return e


def _image_embedder():
    e = _ImageStub()
    e._emb_config = {"input_key": "img", "ucg_rate": 0.0}
    return e


def _stages():
    """CPU stand-ins for sample_flow_batched, decode_and_render and FrameSink.pack: deterministic and independent per
    condition, like the real stages.  sample_fn records the size of every batch it runs."""
    sizes = []

    def sample_fn(c, uc):
        key = "concat" if "concat" in c else "crossattn"
        m = c[key].flatten(1).double().mean(1) - uc[key].flatten(1).double().sum(1)
        lat = (m[:, None] + torch.linspace(-1, 1, 12 * 32 * 32, dtype=torch.float64)[None]).float()
        n = m.shape[0] // N
        sizes.append(n)
        per_cond = [int(1e4 * abs(float(v))) % 97 for v in m[::N]]
        return lat.reshape(n, N, 12, 32, 32), dict(nfe=per_cond, accepted=[k // 2 for k in per_cond], batch_nfe=99)

    def render_fn(lat):
        base = lat[:, :3, :RES, :RES]
        img = torch.stack([torch.tanh(base * (v + 1)) for v in range(V_RENDER)], 1)
        return dict(image_raw=img, image_depth=img[:, :, :1] + 2.0)

    def pack_fn(r):
        return ((r["image_raw"].permute(0, 1, 3, 4, 2).double() * 127.5 + 127.5).clamp(0, 255)).to(torch.uint8)
    return sample_fn, render_fn, pack_fn, sizes


def _inputs(kind, P):
    g = torch.Generator().manual_seed(7)
    if kind == "img":
        x = torch.rand(P, 3, 8, 8, generator=g) * 0.5
        x[:, 0, 0, 0] = torch.arange(P, dtype=torch.float32)
        return (x,)
    x = torch.rand(P, 3, 3, 8, 8, generator=g) * 0.5
    x[:, 0, 0, 0, 0] = torch.arange(P, dtype=torch.float32)
    return x, torch.randn(P, 3, 25, generator=g)


def _run(kind, P, batch):
    """One sharded call in this process (world size from the process group, 1 without one) with freshly seeded host
    generators.  Returns its result and the conditioner's record."""
    from ln3diff_b200 import pipeline
    emb = _image_embedder() if kind == "img" else _mv_embedder(3)
    cond = GeneralConditioner([emb])
    s, r, p, sizes = _stages()
    fn = pipeline.images_to_3d_sharded if kind == "img" else pipeline.mvs_to_3d_sharded
    random.seed(11)
    np.random.seed(12)
    out = fn(cond, None, None, *_inputs(kind, P), torch.zeros(V_RENDER, 25), num_samples=N, resolution=RES,
             batch=batch, device="cpu", sample_fn=s, render_fn=r, pack_fn=p)
    rng_after = (random.random(), float(np.random.uniform()))
    return out, emb.seen, sizes, rng_after


def _worker(rank, world, port, kind, P, batch, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    out, seen, sizes, rng_after = _run(kind, P, batch)
    ret[rank] = dict(frames_all=out["frames_all"].clone(), frames=out["frames"].clone(), shard=out["shard"],
                     latents=out["latents"].clone(), stats=dict(out["stats"]), bytes=out["gather_bytes_per_rank"],
                     seen=seen, sizes=sizes, rng_after=rng_after)
    dist.barrier()
    dist.destroy_process_group()


def _two_ranks(kind, P, batch):
    with mp.Manager() as mgr:
        ret = mgr.dict()
        port = 33500 + (os.getpid() % 2000) + 7 * P + batch
        mp.spawn(_worker, args=(2, port, kind, P, batch, ret), nprocs=2, join=True)
        return dict(ret)


def _single_process_reference(kind, P):
    """What images_to_3d / mvs_to_3d compute with these stages: the conditioner once per condition in order over
    the whole list, one batched sample, one render, one pack."""
    from ln3diff_b200 import pipeline
    emb = _image_embedder() if kind == "img" else _mv_embedder(3)
    cond = GeneralConditioner([emb])
    s, r, p, _ = _stages()
    inp = _inputs(kind, P)
    prompts = [inp[0][i:i + 1].clone() if kind == "img" else
               {"img": inp[0][i:i + 1].clone(), "c": inp[1][i:i + 1].clone()} for i in range(P)]
    random.seed(11)
    np.random.seed(12)
    c, uc = pipeline._condition_list(cond, kind if kind == "img" else "img-c", prompts, N, "cpu")
    rng_after = (random.random(), float(np.random.uniform()))
    lat, st = s(c, uc)
    frames = p(r(lat.reshape(-1, *lat.shape[2:]))).reshape(P, N, V_RENDER, RES, RES, 3)
    return lat, st, frames, emb.seen, rng_after


def _check(kind, P, batch):
    ref_lat, ref_st, ref_frames, ref_seen, ref_rng = _single_process_reference(kind, P)
    one, one_seen, _, one_rng = _run(kind, P, batch)
    assert one["shard"] == (0, P) and torch.equal(one["frames_all"], ref_frames) and torch.equal(one["latents"], ref_lat)
    ret = _two_ranks(kind, P, batch)
    per = -(-P // 2)
    assert ret[0]["shard"] == (0, min(per, P)) and ret[1]["shard"] == (min(per, P), P)
    for rank in (0, 1):
        got = ret[rank]
        lo, hi = got["shard"]
        assert torch.equal(got["frames_all"], ref_frames), (kind, P, batch, rank)
        assert torch.equal(got["frames"], ref_frames[lo:hi]) and torch.equal(got["latents"], ref_lat[lo:hi])
        assert got["bytes"] == per * N * V_RENDER * RES * RES * 3
        for k in ("nfe", "accepted"):
            assert got["stats"].get(k, []) == ref_st[k][lo:hi], (k, rank)
        assert "batch_nfe" not in got["stats"]
        # the conditioner runs twice per condition (conditional and unconditional pass), only for this rank's ones
        ids = [s if kind == "img" else s[0] for s in got["seen"]]
        assert ids == [i for i in range(lo, hi) for _ in range(2)], (kind, P, batch, rank, ids)
        assert all(n <= batch for n in got["sizes"]) and sum(got["sizes"]) == hi - lo
        assert got["rng_after"] == ref_rng == one_rng
    return ret, ref_seen


def test_images_to_3d_sharded_two_ranks_equal_one_process():
    """Even split, ragged split (P = 5: 3 + 2), batches smaller than the shard (P = 5, batch 2), and P = 1 where
    rank 1 holds nothing but still joins the gather."""
    for P, batch in ((4, 8), (5, 8), (5, 2), (1, 8)):
        _check("img", P, batch)


def test_mvs_to_3d_sharded_applies_aug_c_draws_of_its_own_conditions():
    """aug_c: with the same seeds, every condition's cameras -- as its conditioner passes see them -- equal the ones a
    single process gives it, on rank 1 too, whose conditions come after rank 0's draws.  P = 5 in batches of 2."""
    ret, ref_seen = _check("mv", 5, 2)
    lo, hi = ret[1]["shard"]
    assert lo == 3
    ref_cams = {}
    for i, cams in ref_seen:
        ref_cams.setdefault(i, []).append(cams)
    rotated = 0
    for rank in (0, 1):
        mine = {}
        for i, cams in ret[rank]["seen"]:
            mine.setdefault(i, []).append(cams)
        for i, passes in mine.items():
            assert len(passes) == 2 and all(torch.equal(a, b) for a, b in zip(passes, ref_cams[i])), (rank, i)
    _, cams_in = _inputs("mv", 5)
    for i in range(lo, hi):
        rotated += int((ref_cams[i][0] != cams_in[i]).any(-1).sum())
    assert rotated > 0, "rank 1's conditions must include rotated cameras for the check to mean anything"


def test_mvs_to_3d_sharded_leaves_callers_cameras_and_skip_matches_conditioning():
    """skip_unconditional_conditioning advances `random` and `np.random` exactly as get_unconditional_conditioning
    does for the same condition, and a sharded call never rotates the caller's cameras."""
    emb = _mv_embedder(3)
    cond = GeneralConditioner([emb])
    imgs, cams = _inputs("mv", 3)
    batch_c = {"img-c": {"img": imgs[:1].clone(), "c": cams[:1].clone()}}
    random.seed(3); np.random.seed(4)
    cond.get_unconditional_conditioning(batch_c, force_uc_zero_embeddings=["img-c"])
    after_run = (random.getstate(), np.random.get_state()[1].tolist(), np.random.get_state()[2])
    random.seed(3); np.random.seed(4)
    cond.skip_unconditional_conditioning({"img-c": {"img": imgs[:1], "c": cams[:1]}})
    assert (random.getstate(), np.random.get_state()[1].tolist(), np.random.get_state()[2]) == after_run
    from ln3diff_b200 import pipeline
    s, r, p, _ = _stages()
    keep = cams.clone()
    pipeline.mvs_to_3d_sharded(cond, None, None, imgs, cams, torch.zeros(V_RENDER, 25), num_samples=N,
                               resolution=RES, device="cpu", sample_fn=s, render_fn=r, pack_fn=p)
    assert torch.equal(cams, keep)
