"""Mirror of the conditioner stack of reference sgm/modules/encoders/modules.py (SURVEY 8f-1):
`GeneralConditioner` (:80-190), `FrozenCLIPEmbedder` (:347-408, T23D), `FrozenOpenCLIPImageEmbedder` (:578-733),
`FrozenDinov2ImageEmbedder` (:735-868, I23D) and `FrozenDinov2ImageEmbedderMVPlucker` (:871-1104, MV23D) -- same class
names, constructor arguments, `input_key` / `ucg_rate` plumbing, output shapes and dictionary keys; the frozen towers
run on the libln3b200 kernels (`_tower.TransformerTower`) instead of transformers / open_clip / the dinov2 hub model.

Weights.  The reference constructors download pretrained weights (`CLIPTextModel.from_pretrained`,
`open_clip.create_model_and_transforms`, `torch.hub.load`).  There is no network here: every embedder takes
`state_dict=` with the keys the reference object would hold (`transformer.text_model.*` / `model.visual.*` /
`model.*` of the dinov2 hub module; bare sub-module keys are accepted too).  Without one the constructor does what
the reference does -- it calls the reference's own loader (`from_pretrained` / `open_clip` / `torch.hub`) -- and
RAISES when that cannot run (no network, package absent): random weights are never substituted silently;
`random_init=True` asks for them explicitly (benchmarks, tests).  CUDA only -- no CPU fallback.

Third-party arithmetic restated here (file:line = reference call site):
  * transformers CLIPTextModel (:367): token + position embedding, causal pre-LN blocks with QuickGELU, final
    LayerNorm, pooled = hidden state at the EOS position (argmax of the ids for the legacy eos_token_id 2).
  * open_clip VisionTransformer (:600-607,699-706): conv1 patchify (no bias), class token, positional embedding,
    ln_pre, pre-LN blocks (QuickGELU for the `openai` weights), ln_post, pooled = x[:, 0] @ proj, tokens = x[:, 1:].
  * dinov2 DinoVisionTransformer.forward_features (:774-781,831-836): patchify with bias, cls + interpolated
    position embedding, register tokens inserted after cls, pre-LN blocks with LayerScale and erf-GELU, final
    LayerNorm (eps 1e-6); `x_norm_patchtokens` = tokens after the registers.
  * kornia.geometry.resize(bicubic, align_corners=True, antialias=True) (:649-655,809-815): Gaussian blur with
    sigma = (factor - 1) / 2 when down-scaling, then torch bicubic interpolation -- PARITY UNPINNED (kornia is not
    in the image); it is image pre-processing, done with torch ops once per prompt.
"""
from __future__ import annotations

import math
import random
from contextlib import nullcontext
from typing import Dict, List, Optional, Union

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .... import ops
from ...._lib import ACT_GELU_ERF, ACT_QUICK_GELU
from ...util import instantiate_from_config
from ._tower import TransformerTower, _ln_pair


def expand_dims_like(x, y):
    while x.dim() != y.dim():
        x = x.unsqueeze(-1)
    return x


def disabled_train(self, mode=True):
    return self


class AbstractEmbModel(nn.Module):
    """reference :32-77 (attribute plumbing used by GeneralConditioner)."""

    def __init__(self):
        super().__init__()
        self._is_trainable = None
        self._ucg_rate = None
        self._input_key = None

    is_trainable = property(lambda s: s._is_trainable, lambda s, v: setattr(s, "_is_trainable", v))
    ucg_rate = property(lambda s: s._ucg_rate, lambda s, v: setattr(s, "_ucg_rate", v))
    input_key = property(lambda s: s._input_key, lambda s, v: setattr(s, "_input_key", v))


class GeneralConditioner(nn.Module):
    """reference :80-190: runs every embedder on its `input_key`, sorts the outputs into
    {'vector' (B,D), 'crossattn' (B,L,D), 'concat'} by rank and concatenates per key."""
    OUTPUT_DIM2KEYS = {2: "vector", 3: "crossattn", 4: "concat", 5: "concat"}
    KEY2CATDIM = {"vector": 1, "crossattn": 2, "concat": 1}

    def __init__(self, emb_models):
        super().__init__()
        embedders = []
        for n, embconfig in enumerate(emb_models):
            if isinstance(embconfig, nn.Module):     # already-built embedder (tests / programmatic use)
                embedder, embconfig = embconfig, getattr(embconfig, "_emb_config", {})
            else:
                embedder = instantiate_from_config(embconfig)
            assert isinstance(embedder, AbstractEmbModel), \
                f"embedder model {embedder.__class__.__name__} has to inherit from AbstractEmbModel"
            embedder.is_trainable = embconfig.get("is_trainable", False)
            embedder.ucg_rate = embconfig.get("ucg_rate", 0.0)
            if not embedder.is_trainable:
                embedder.train = disabled_train.__get__(embedder)
                for param in embedder.parameters():
                    param.requires_grad = False
                embedder.eval()
            if "input_key" in embconfig:
                embedder.input_key = embconfig["input_key"]
            elif "input_keys" in embconfig:
                embedder.input_keys = embconfig["input_keys"]
            else:
                raise KeyError(f"need either 'input_key' or 'input_keys' for embedder {embedder.__class__.__name__}")
            embedder.legacy_ucg_val = embconfig.get("legacy_ucg_value", None)
            if embedder.legacy_ucg_val is not None:
                embedder.ucg_prng = np.random.RandomState()
            embedders.append(embedder)
        self.embedders = nn.ModuleList(embedders)

    def possibly_get_ucg_val(self, embedder, batch: Dict) -> Dict:
        assert embedder.legacy_ucg_val is not None
        p = embedder.ucg_rate
        val = embedder.legacy_ucg_val
        for i in range(len(batch[embedder.input_key])):
            if embedder.ucg_prng.choice(2, p=[1 - p, p]):
                batch[embedder.input_key][i] = val
        return batch

    def forward(self, batch: Dict, force_zero_embeddings: Optional[List] = None) -> Dict:
        output = dict()
        if force_zero_embeddings is None:
            force_zero_embeddings = []
        for embedder in self.embedders:
            embedding_context = nullcontext if embedder.is_trainable else torch.no_grad
            with embedding_context():
                if hasattr(embedder, "input_key") and (embedder.input_key is not None):
                    if embedder.legacy_ucg_val is not None:
                        batch = self.possibly_get_ucg_val(embedder, batch)
                    emb_out = embedder(batch[embedder.input_key])
                elif hasattr(embedder, "input_keys"):
                    emb_out = embedder(*[batch[k] for k in embedder.input_keys])
            assert isinstance(emb_out, (torch.Tensor, list, tuple)), \
                f"encoder outputs must be tensors or a sequence, but got {type(emb_out)}"
            if not isinstance(emb_out, (list, tuple)):
                emb_out = [emb_out]
            for emb in emb_out:
                out_key = self.OUTPUT_DIM2KEYS[emb.dim()]
                if embedder.ucg_rate > 0.0 and embedder.legacy_ucg_val is None:
                    emb = (expand_dims_like(
                        torch.bernoulli((1.0 - embedder.ucg_rate) * torch.ones(emb.shape[0], device=emb.device)), emb) * emb)
                if hasattr(embedder, "input_key") and embedder.input_key in force_zero_embeddings:
                    emb = torch.zeros_like(emb)
                if out_key in output:
                    output[out_key] = torch.cat((output[out_key], emb), self.KEY2CATDIM[out_key])
                else:
                    output[out_key] = emb
        return output

    def get_unconditional_conditioning(self, batch_c: Dict, batch_uc: Optional[Dict] = None,
                                       force_uc_zero_embeddings: Optional[List[str]] = None,
                                       force_cond_zero_embeddings: Optional[List[str]] = None):
        if force_uc_zero_embeddings is None:
            force_uc_zero_embeddings = []
        ucg_rates = list()
        for embedder in self.embedders:
            ucg_rates.append(embedder.ucg_rate)
            embedder.ucg_rate = 0.0  # force no drop during inference
        c = self(batch_c, force_cond_zero_embeddings)
        uc = self(batch_c if batch_uc is None else batch_uc, force_uc_zero_embeddings)
        for embedder, rate in zip(self.embedders, ucg_rates):
            embedder.ucg_rate = rate
        return c, uc

    def skip_unconditional_conditioning(self, batch_c: Dict, batch_uc: Optional[Dict] = None) -> None:
        """Advances the global host generators (`random`, `np.random`) as get_unconditional_conditioning(batch_c,
        batch_uc) does, without running any embedder: every embedder with a `draw_augmentation` makes the draws of its
        conditional pass, then those of its unconditional pass.  A sharded run calls it for each condition another
        rank conditions, so that its own conditions get the draws a single process gives them."""
        for batch in (batch_c, batch_c if batch_uc is None else batch_uc):
            for embedder in self.embedders:
                draw = getattr(embedder, "draw_augmentation", None)
                if draw is not None and getattr(embedder, "input_key", None) is not None:
                    draw(batch[embedder.input_key])


# --------------------------------------------------------------------------------------------- helpers
def _strip(sd: dict, *prefixes: str) -> dict:
    """Keys with the first matching prefix removed (state dicts of the wrapper or of the bare sub-module)."""
    for p in prefixes:
        if any(k.startswith(p) for k in sd):
            return {k[len(p):]: v for k, v in sd.items() if k.startswith(p)}
    return dict(sd)


def _gaussian_kernel1d(ks: int, sigma: float, device) -> torch.Tensor:
    x = torch.arange(ks, device=device, dtype=torch.float32) - ks // 2
    if ks % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x.pow(2) / (2 * sigma * sigma))
    return g / g.sum()


def kornia_resize_bicubic(x: torch.Tensor, size=(224, 224), antialias: bool = True) -> torch.Tensor:
    """kornia.geometry.resize(x, size, interpolation='bicubic', align_corners=True, antialias=antialias)."""
    h, w = x.shape[-2:]
    fy, fx = h / size[0], w / size[1]
    if antialias and (fy > 1 or fx > 1):
        sig = (max((fy - 1.0) / 2.0, 0.001), max((fx - 1.0) / 2.0, 0.001))
        ks = [int(max(2.0 * 2 * sig[0], 3)), int(max(2.0 * 2 * sig[1], 3))]
        ks = [k + 1 if k % 2 == 0 else k for k in ks]
        C = x.shape[1]
        ky = _gaussian_kernel1d(ks[0], sig[0], x.device).view(1, 1, -1, 1).expand(C, 1, -1, 1)
        kx = _gaussian_kernel1d(ks[1], sig[1], x.device).view(1, 1, 1, -1).expand(C, 1, 1, -1)
        x = F.pad(x, (ks[1] // 2, ks[1] // 2, ks[0] // 2, ks[0] // 2), mode="reflect")
        x = F.conv2d(F.conv2d(x, ky, groups=C), kx, groups=C)
    return F.interpolate(x, size=size, mode="bicubic", align_corners=True)


def _patchify_gemm(img: torch.Tensor, w_packed: torch.Tensor, bias: Optional[torch.Tensor], patch: int) -> torch.Tensor:
    """Conv2d(3, D, kernel = stride = patch) as one wgmma GEMM: (B*n*n, 3*p*p padded to a multiple of 64) x W^T.
    Non-overlapping patches: the unfold is a pure permute."""
    B, C, Hh, Ww = img.shape
    n = Hh // patch
    cols = img.reshape(B, C, n, patch, n, patch).permute(0, 2, 4, 1, 3, 5).reshape(B * n * n, C * patch * patch)
    K = w_packed.shape[1]
    a = torch.zeros((cols.shape[0], K), device=img.device, dtype=torch.bfloat16)
    a[:, :cols.shape[1]] = cols
    return ops.gemm(a, w_packed, bias).float().view(B, n * n, -1)


def _pack_patch_weight(w: torch.Tensor, device) -> torch.Tensor:
    D = w.shape[0]
    k = w[0].numel()
    K = (k + 63) // 64 * 64
    out = torch.zeros((D, K), device=device, dtype=torch.bfloat16)
    out[:, :k] = w.detach().reshape(D, k).to(device=device, dtype=torch.bfloat16)
    return out


def _load_pretrained(what: str, loader):
    """Run the reference's weight loader; a failure is an error, never a silent random initialisation."""
    try:
        return loader()
    except Exception as e:  # noqa: BLE001 -- network / missing package / missing assets
        raise RuntimeError(f"{what}: the reference's pretrained loader failed ({type(e).__name__}: {e}); pass "
                           f"state_dict= (keys as the reference object holds them) or random_init=True") from e


def _randn(*shape, std=0.02, g=None):
    return torch.randn(*shape, generator=g) * std


# --------------------------------------------------------------------------------------------- CLIP text
class FrozenCLIPEmbedder(AbstractEmbModel):
    """Uses the CLIP transformer encoder for text (reference :347-408; transformers CLIPTextModel arithmetic)."""
    LAYERS = ["last", "pooled", "hidden"]

    def __init__(self, version="openai/clip-vit-large-patch14", device="cuda", max_length=77, freeze=True,
                 layer="last", layer_idx=None, always_return_pooled=False, *, state_dict: dict | None = None,
                 random_init: bool = False, tokenizer=None, vocab_size=49408, width=768, heads=12, depth=12,
                 mlp_dim=3072, eos_token_id=2, seed=0):
        super().__init__()
        assert layer in self.LAYERS
        self.device = device
        self.max_length = max_length
        self.layer = layer
        self.layer_idx = layer_idx
        self.return_pooled = always_return_pooled
        self.eos_token_id = eos_token_id
        if layer == "hidden":
            assert layer_idx is not None
            assert 0 <= abs(layer_idx) <= 12
        self.tokenizer = tokenizer
        if state_dict is None and not random_init:
            def _load():
                from transformers import CLIPTextModel, CLIPTokenizer   # the reference's own loader (:366-367)
                return CLIPTokenizer.from_pretrained(version), CLIPTextModel.from_pretrained(version).state_dict()
            self.tokenizer, state_dict = _load_pretrained("FrozenCLIPEmbedder", _load)
        if state_dict is None:
            g = torch.Generator().manual_seed(seed)
            sd = {"text_model.embeddings.token_embedding.weight": _randn(vocab_size, width, g=g),
                  "text_model.embeddings.position_embedding.weight": _randn(max_length, width, std=0.01, g=g),
                  "text_model.final_layer_norm.weight": torch.ones(width), "text_model.final_layer_norm.bias": torch.zeros(width)}
            for i in range(depth):
                p = f"text_model.encoder.layers.{i}."
                for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
                    sd[p + f"self_attn.{nm}.weight"] = _randn(width, width, g=g)
                    sd[p + f"self_attn.{nm}.bias"] = _randn(width, g=g)
                sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"] = _randn(mlp_dim, width, g=g), _randn(mlp_dim, g=g)
                sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"] = _randn(width, mlp_dim, g=g), _randn(width, g=g)
                for ln in ("layer_norm1", "layer_norm2"):
                    sd[p + ln + ".weight"], sd[p + ln + ".bias"] = torch.ones(width), torch.zeros(width)
            state_dict = sd
        sd = _strip(state_dict, "transformer.text_model.", "text_model.")
        dev = torch.device(device)
        self.register_buffer("token_embedding", sd["embeddings.token_embedding.weight"].detach().float().to(dev), persistent=False)
        self.register_buffer("position_embedding", sd["embeddings.position_embedding.weight"].detach().float().to(dev), persistent=False)
        width = self.token_embedding.shape[1]
        n_layers = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("encoder.layers."))
        heads = width // 64
        self.tower = TransformerTower(width, heads, ACT_QUICK_GELU, 1e-5, True, dev)
        for i in range(n_layers):
            p = f"encoder.layers.{i}."
            self.tower.add_layer(
                ln1=(sd[p + "layer_norm1.weight"], sd[p + "layer_norm1.bias"]),
                qkv_w=torch.cat([sd[p + f"self_attn.{n}.weight"] for n in ("q_proj", "k_proj", "v_proj")], 0),
                qkv_b=torch.cat([sd[p + f"self_attn.{n}.bias"] for n in ("q_proj", "k_proj", "v_proj")], 0),
                proj_w=sd[p + "self_attn.out_proj.weight"], proj_b=sd[p + "self_attn.out_proj.bias"],
                ln2=(sd[p + "layer_norm2.weight"], sd[p + "layer_norm2.bias"]),
                fc1_w=sd[p + "mlp.fc1.weight"], fc1_b=sd[p + "mlp.fc1.bias"],
                fc2_w=sd[p + "mlp.fc2.weight"], fc2_b=sd[p + "mlp.fc2.bias"])
        self._final_ln = _ln_pair(sd["final_layer_norm.weight"], sd["final_layer_norm.bias"], dev)
        if freeze:
            self.freeze()

    def freeze(self):
        for param in self.parameters():
            param.requires_grad = False

    def tokenize(self, text) -> torch.Tensor:
        if self.tokenizer is None:
            raise RuntimeError("FrozenCLIPEmbedder: no tokenizer assets in this environment; pass `tokenizer=` "
                               "(a transformers CLIPTokenizer) or call encode_tokens(input_ids)")
        enc = self.tokenizer(text, truncation=True, max_length=self.max_length, return_length=True,
                             return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
        return enc["input_ids"]

    @torch.no_grad()
    def encode_tokens(self, tokens: torch.Tensor):
        """transformers CLIPTextTransformer.forward on token ids (B, L)."""
        tokens = tokens.to(self.token_embedding.device)
        B, L = tokens.shape
        x = (self.token_embedding[tokens] + self.position_embedding[:L]).contiguous()
        hidden = [] if self.layer == "hidden" else None
        self.tower.run(x, hidden_states=hidden)
        last = self.tower.layer_norm(x, self._final_ln)
        if self.eos_token_id == 2:     # legacy configs (openai/clip-vit-large-patch14): EOS is the largest id
            eos = tokens.to(torch.int).argmax(dim=-1)
        else:
            eos = (tokens.to(torch.int) == self.eos_token_id).int().argmax(dim=-1)
        pooled = last[torch.arange(B, device=last.device), eos]
        if self.layer == "last":
            z = last
        elif self.layer == "pooled":
            z = pooled[:, None, :]
        else:
            z = hidden[self.layer_idx]
        if self.return_pooled:
            return z, pooled
        return z

    def forward(self, text):
        if isinstance(text, torch.Tensor):
            return self.encode_tokens(text)
        return self.encode_tokens(self.tokenize(text))

    def encode(self, text):
        return self(text)


# --------------------------------------------------------------------------------------------- image towers
class _ImageEmbedderBase(AbstractEmbModel):
    MEAN, STD = (0.0, 0.0, 0.0), (1.0, 1.0, 1.0)

    def _init_common(self, device, max_length, antialias, ucg_rate, unsqueeze_dim, repeat_to_max_len, num_image_crops,
                     output_tokens):
        self.max_crops = num_image_crops
        self.pad_to_max_len = self.max_crops > 0
        self.repeat_to_max_len = repeat_to_max_len and (not self.pad_to_max_len)
        self.device = device
        self.max_length = max_length
        self.antialias = antialias
        self.register_buffer("mean", torch.Tensor(self.MEAN), persistent=False)
        self.register_buffer("std", torch.Tensor(self.STD), persistent=False)
        self.ucg_rate = ucg_rate
        self.unsqueeze_dim = unsqueeze_dim
        self.stored_batch = None
        self.output_tokens = output_tokens

    def preprocess(self, x):
        """reference :647-659 / :807-819: resize to 224 (bicubic, antialias), [-1,1] -> [0,1], normalise."""
        x = kornia_resize_bicubic(x.float(), (224, 224), antialias=self.antialias)
        x = (x + 1.0) / 2.0
        return (x - self.mean.to(x.device)[None, :, None, None]) / self.std.to(x.device)[None, :, None, None]

    def freeze(self):
        for param in self.parameters():
            param.requires_grad = False

    def encode(self, text):
        return self(text)


class FrozenOpenCLIPImageEmbedder(_ImageEmbedderBase):
    """Uses the OpenCLIP vision transformer encoder for images (reference :578-733)."""
    MEAN, STD = (0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)

    def __init__(self, arch="ViT-L-14", version="openai", device="cuda", max_length=77, freeze=True, antialias=True,
                 ucg_rate=0.0, unsqueeze_dim=False, repeat_to_max_len=False, num_image_crops=0, output_tokens=False,
                 init_device=None, *, state_dict: dict | None = None, random_init: bool = False, width=1024, heads=16,
                 depth=24, mlp_dim=4096, embed_dim=768, patch=14, image_size=224, seed=0):
        super().__init__()
        self._init_common(device, max_length, antialias, ucg_rate, unsqueeze_dim, repeat_to_max_len, num_image_crops,
                          output_tokens)
        if state_dict is None and not random_init:
            def _load():
                import open_clip   # the reference's own loader (:600-604); not in this image
                model, _, _ = open_clip.create_model_and_transforms(arch, device=torch.device("cpu"), pretrained=version)
                return {"model." + k: v for k, v in model.state_dict().items()}
            state_dict = _load_pretrained("FrozenOpenCLIPImageEmbedder", _load)
        if state_dict is None:
            g = torch.Generator().manual_seed(seed)
            n = (image_size // patch) ** 2 + 1
            sd = {"conv1.weight": _randn(width, 3, patch, patch, g=g), "class_embedding": _randn(width, g=g),
                  "positional_embedding": _randn(n, width, std=0.01, g=g), "proj": _randn(width, embed_dim, std=width ** -0.5, g=g)}
            for ln in ("ln_pre", "ln_post"):
                sd[ln + ".weight"], sd[ln + ".bias"] = torch.ones(width), torch.zeros(width)
            for i in range(depth):
                p = f"transformer.resblocks.{i}."
                sd[p + "attn.in_proj_weight"], sd[p + "attn.in_proj_bias"] = _randn(3 * width, width, g=g), _randn(3 * width, g=g)
                sd[p + "attn.out_proj.weight"], sd[p + "attn.out_proj.bias"] = _randn(width, width, g=g), _randn(width, g=g)
                sd[p + "mlp.c_fc.weight"], sd[p + "mlp.c_fc.bias"] = _randn(mlp_dim, width, g=g), _randn(mlp_dim, g=g)
                sd[p + "mlp.c_proj.weight"], sd[p + "mlp.c_proj.bias"] = _randn(width, mlp_dim, g=g), _randn(width, g=g)
                for ln in ("ln_1", "ln_2"):
                    sd[p + ln + ".weight"], sd[p + ln + ".bias"] = torch.ones(width), torch.zeros(width)
            state_dict = sd
        sd = _strip(state_dict, "model.visual.", "visual.")
        dev = torch.device(device)
        self.patch = sd["conv1.weight"].shape[-1]
        width = sd["conv1.weight"].shape[0]
        self._conv_w = _pack_patch_weight(sd["conv1.weight"], dev)
        self.register_buffer("class_embedding", sd["class_embedding"].detach().float().to(dev), persistent=False)
        self.register_buffer("positional_embedding", sd["positional_embedding"].detach().float().to(dev), persistent=False)
        n_layers = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("transformer.resblocks."))
        # open_clip builds QuickGELU blocks for the `openai` pretrained tag, nn.GELU otherwise
        act = ACT_QUICK_GELU if version == "openai" else ACT_GELU_ERF
        self.tower = TransformerTower(width, width // 64, act, 1e-5, False, dev)
        for i in range(n_layers):
            p = f"transformer.resblocks.{i}."
            self.tower.add_layer(ln1=(sd[p + "ln_1.weight"], sd[p + "ln_1.bias"]),
                                 qkv_w=sd[p + "attn.in_proj_weight"], qkv_b=sd[p + "attn.in_proj_bias"],
                                 proj_w=sd[p + "attn.out_proj.weight"], proj_b=sd[p + "attn.out_proj.bias"],
                                 ln2=(sd[p + "ln_2.weight"], sd[p + "ln_2.bias"]),
                                 fc1_w=sd[p + "mlp.c_fc.weight"], fc1_b=sd[p + "mlp.c_fc.bias"],
                                 fc2_w=sd[p + "mlp.c_proj.weight"], fc2_b=sd[p + "mlp.c_proj.bias"])
        self._ln_pre = _ln_pair(sd["ln_pre.weight"], sd["ln_pre.bias"], dev)
        self._ln_post = _ln_pair(sd["ln_post.weight"], sd["ln_post.bias"], dev)
        pw = sd["proj"].detach().t().contiguous()                       # (embed, width): nn.Linear layout
        self._embed_dim = pw.shape[0]
        n_pad = (pw.shape[0] + 127) // 128 * 128
        self._proj_w = torch.zeros((n_pad, width), device=dev, dtype=torch.bfloat16)
        self._proj_w[:pw.shape[0]] = pw.to(device=dev, dtype=torch.bfloat16)
        if freeze:
            self.freeze()

    @torch.no_grad()
    def visual(self, img: torch.Tensor):
        """open_clip VisionTransformer.forward on a pre-processed image batch (B,3,224,224) -> (pooled, tokens)."""
        B = img.shape[0]
        x = _patchify_gemm(img, self._conv_w, None, self.patch)
        x = torch.cat([self.class_embedding.expand(B, 1, -1), x], dim=1) + self.positional_embedding
        x = self.tower.layer_norm(x.contiguous(), self._ln_pre).contiguous()
        self.tower.run(x)
        x = self.tower.layer_norm(x, self._ln_post)
        pooled = ops.gemm(x[:, 0].to(torch.bfloat16).contiguous(), self._proj_w).float()[:, :self._embed_dim]
        return pooled, x[:, 1:]

    def encode_with_vision_transformer(self, img):
        if img.dim() == 5:
            assert self.max_crops == img.shape[1]
            img = img.reshape(-1, *img.shape[2:])
        img = self.preprocess(img.to(self.class_embedding.device))
        x, tokens = self.visual(img)
        if not self.output_tokens:
            tokens = None
        if self.max_crops > 0:
            x = x.reshape(-1, self.max_crops, x.shape[-1])
            x = torch.bernoulli((1.0 - self.ucg_rate) * torch.ones(x.shape[0], x.shape[1], 1, device=x.device)) * x
            if tokens is not None:
                tokens = tokens.reshape(-1, self.max_crops, *tokens.shape[1:]).permute(0, 2, 1, 3).flatten(2)
        if self.output_tokens:
            return x, tokens
        return x

    def forward(self, image, no_dropout=False):
        z = self.encode_with_vision_transformer(image)
        tokens = None
        if self.output_tokens:
            z, tokens = z[0], z[1]
        z = z.to(image.dtype)
        if self.ucg_rate > 0.0 and not no_dropout and not (self.max_crops > 0):
            z = torch.bernoulli((1.0 - self.ucg_rate) * torch.ones(z.shape[0], device=z.device))[:, None] * z
            if tokens is not None:
                tokens = expand_dims_like(torch.bernoulli((1.0 - self.ucg_rate) * torch.ones(tokens.shape[0], device=tokens.device)),
                                          tokens) * tokens
        if self.unsqueeze_dim:
            z = z[:, None, :]
        if self.output_tokens:
            assert not self.repeat_to_max_len
            assert not self.pad_to_max_len
            return tokens, z
        if self.repeat_to_max_len:
            z_ = z[:, None, :] if z.dim() == 2 else z
            return z_.expand(-1, self.max_length, -1).contiguous(), z
        elif self.pad_to_max_len:
            assert z.dim() == 3
            z_pad = torch.cat((z, torch.zeros(z.shape[0], self.max_length - z.shape[1], z.shape[2], device=z.device)), 1)
            return z_pad, z_pad[:, 0, ...]
        return z


class FrozenDinov2ImageEmbedder(_ImageEmbedderBase):
    """Uses the Dino-v2 (ViT-L/14 with 4 registers) for low-level image embedding (reference :735-868): returns the
    normalised patch tokens (B, 256, 1024) (`x_norm_patchtokens`), optionally with the cls token."""
    MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)

    def __init__(self, arch="vitl", version="dinov2", device="cuda", max_length=77, freeze=True, antialias=True,
                 ucg_rate=0.0, unsqueeze_dim=False, repeat_to_max_len=False, num_image_crops=0, output_tokens=False,
                 output_cls=False, init_device=None, *, state_dict: dict | None = None, random_init: bool = False,
                 width=1024, depth=24, mlp_dim=4096, patch=14, num_register_tokens=4, pos_grid=37,
                 interpolate_antialias=True, interpolate_offset=0.0, seed=0):
        super().__init__()
        self._init_common(device, max_length, antialias, ucg_rate, unsqueeze_dim, repeat_to_max_len, num_image_crops,
                          output_tokens)
        self.output_cls = output_cls
        self.interpolate_antialias, self.interpolate_offset = interpolate_antialias, interpolate_offset
        if state_dict is None and not random_init:
            def _load():
                model = torch.hub.load(f"facebookresearch/{version}", f"{version}_{arch}14_reg", pretrained=True)  # :760-765
                return {"model." + k: v for k, v in model.state_dict().items()}
            state_dict = _load_pretrained("FrozenDinov2ImageEmbedder", _load)
        if state_dict is None:
            state_dict = self._random_state_dict(width, depth, mlp_dim, patch, num_register_tokens, pos_grid, seed)
        sd = _strip(state_dict, "model.")
        dev = torch.device(device)
        width = sd["cls_token"].shape[-1]
        self.patch = sd["patch_embed.proj.weight"].shape[-1]
        self._conv_w = _pack_patch_weight(sd["patch_embed.proj.weight"], dev)
        self._conv_b = sd["patch_embed.proj.bias"].detach().float().to(dev).contiguous()
        self.register_buffer("cls_token", sd["cls_token"].detach().float().to(dev), persistent=False)
        self.register_buffer("register_tokens", sd["register_tokens"].detach().float().to(dev), persistent=False)
        self.register_buffer("pos_embed", sd["pos_embed"].detach().float().to(dev), persistent=False)
        self._pos_cache: dict = {}
        n_layers = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))
        self.tower = TransformerTower(width, width // 64, ACT_GELU_ERF, 1e-6, False, dev)
        for i in range(n_layers):
            p = f"blocks.{i}."
            self.tower.add_layer(ln1=(sd[p + "norm1.weight"], sd[p + "norm1.bias"]),
                                 qkv_w=sd[p + "attn.qkv.weight"], qkv_b=sd[p + "attn.qkv.bias"],
                                 proj_w=sd[p + "attn.proj.weight"], proj_b=sd[p + "attn.proj.bias"], ls1=sd[p + "ls1.gamma"],
                                 ln2=(sd[p + "norm2.weight"], sd[p + "norm2.bias"]),
                                 fc1_w=sd[p + "mlp.fc1.weight"], fc1_b=sd[p + "mlp.fc1.bias"],
                                 fc2_w=sd[p + "mlp.fc2.weight"], fc2_b=sd[p + "mlp.fc2.bias"], ls2=sd[p + "ls2.gamma"])
        self._norm = _ln_pair(sd["norm.weight"], sd["norm.bias"], dev)
        if freeze:
            self.freeze()

    @staticmethod
    def _random_state_dict(width, depth, mlp_dim, patch, num_register_tokens, pos_grid, seed, in_chans=3) -> dict:
        """random_init=True: a seeded DINOv2-with-registers state dict (hub key layout, no `model.` prefix)."""
        g = torch.Generator().manual_seed(seed)
        sd = {"cls_token": _randn(1, 1, width, g=g), "register_tokens": _randn(1, num_register_tokens, width, g=g),
              "pos_embed": _randn(1, 1 + pos_grid * pos_grid, width, g=g),
              "patch_embed.proj.weight": _randn(width, in_chans, patch, patch, g=g), "patch_embed.proj.bias": _randn(width, g=g),
              "norm.weight": torch.ones(width), "norm.bias": torch.zeros(width)}
        for i in range(depth):
            p = f"blocks.{i}."
            sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"] = _randn(3 * width, width, g=g), _randn(3 * width, g=g)
            sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"] = _randn(width, width, g=g), _randn(width, g=g)
            sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"] = _randn(mlp_dim, width, g=g), _randn(mlp_dim, g=g)
            sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"] = _randn(width, mlp_dim, g=g), _randn(width, g=g)
            sd[p + "ls1.gamma"], sd[p + "ls2.gamma"] = torch.full((width,), 0.5), torch.full((width,), 0.5)
            for ln in ("norm1", "norm2"):
                sd[p + ln + ".weight"], sd[p + ln + ".bias"] = torch.ones(width), torch.zeros(width)
        return sd

    def interpolate_pos_encoding(self, n_side: int) -> torch.Tensor:
        """dinov2 DinoVisionTransformer.interpolate_pos_encoding for an n_side x n_side patch grid."""
        if n_side in self._pos_cache:
            return self._pos_cache[n_side]
        pe = self.pos_embed
        N = pe.shape[1] - 1
        M = int(math.sqrt(N))
        assert M * M == N
        if M == n_side:
            out = pe
        else:
            cls_pe, patch_pe = pe[:, :1], pe[:, 1:]
            kw = {}
            if self.interpolate_offset:
                s = float(n_side + self.interpolate_offset) / M
                kw["scale_factor"] = (s, s)
            else:
                kw["size"] = (n_side, n_side)
            patch_pe = F.interpolate(patch_pe.reshape(1, M, M, -1).permute(0, 3, 1, 2), mode="bicubic",
                                     antialias=self.interpolate_antialias, **kw)
            assert patch_pe.shape[-2:] == (n_side, n_side)
            out = torch.cat([cls_pe, patch_pe.permute(0, 2, 3, 1).reshape(1, n_side * n_side, -1)], dim=1)
        self._pos_cache[n_side] = out
        return out

    @torch.no_grad()
    def forward_features(self, img: torch.Tensor, patch_tokens: Optional[torch.Tensor] = None) -> dict:
        """dinov2 forward_features on a pre-processed batch (B,3,H,W), H = W = 14 n.  `patch_tokens` (B, n*n, D):
        the patch embedding already computed by the caller (the 9-channel input of the multi-view embedder)."""
        B = img.shape[0]
        n = img.shape[-1] // self.patch
        x = _patchify_gemm(img, self._conv_w, self._conv_b, self.patch) if patch_tokens is None else patch_tokens
        x = torch.cat([self.cls_token.expand(B, -1, -1), x], dim=1) + self.interpolate_pos_encoding(n)
        R = self.register_tokens.shape[1]
        x = torch.cat([x[:, :1], self.register_tokens.expand(B, -1, -1), x[:, 1:]], dim=1).contiguous()
        self.tower.run(x)
        xn = self.tower.layer_norm(x, self._norm)
        return {"x_norm_clstoken": xn[:, 0], "x_norm_regtokens": xn[:, 1:R + 1], "x_norm_patchtokens": xn[:, R + 1:],
                "x_prenorm": x}

    def encode_with_vision_transformer(self, img, **kwargs):
        if img.dim() == 5:
            img = img.reshape(-1, *img.shape[2:])
        img = self.preprocess(img.to(self.cls_token.device))
        ret = self.forward_features(img)
        if not self.output_cls:
            return ret["x_norm_patchtokens"]
        return ret["x_norm_clstoken"], ret["x_norm_patchtokens"]

    def forward(self, image, no_dropout=False, **kwargs):
        tokens = self.encode_with_vision_transformer(image, **kwargs)
        z = None
        if self.output_cls:
            z, tokens = tokens[0], tokens[1]     # (the reference indexes an unset `z` here, :844-846)
            z = z.to(image.dtype)
        tokens = tokens.to(image.dtype)
        if self.ucg_rate > 0.0 and not no_dropout and not (self.max_crops > 0):
            if z is not None:
                z = torch.bernoulli((1.0 - self.ucg_rate) * torch.ones(z.shape[0], device=z.device))[:, None] * z
            tokens = expand_dims_like(torch.bernoulli((1.0 - self.ucg_rate) * torch.ones(tokens.shape[0], device=tokens.device)),
                                      tokens) * tokens
        if self.output_cls:
            return tokens, z
        return tokens


# --------------------------------------------------------------------------------------------- multi-view DINOv2
def _nine_channel_patch_embed(state_dict: dict) -> dict:
    """The reference constructor's patch-embedding surgery (:922-938): a 3-channel `patch_embed.proj.weight` becomes a
    zero-initialised 9-channel one whose first three input channels are the pretrained weights (the bias is kept).
    A state dict that already holds the 9-channel weight (a trained MV23D checkpoint) is returned unchanged."""
    sd = dict(state_dict)
    for k in ("model.patch_embed.proj.weight", "patch_embed.proj.weight"):
        w = sd.get(k)
        if w is not None and w.shape[1] == 3:
            w9 = torch.zeros(w.shape[0], 9, *w.shape[2:], dtype=w.dtype)
            w9[:, :3] = w.detach().cpu()
            sd[k] = w9
    return sd


class FrozenDinov2ImageEmbedderMVPlucker(FrozenDinov2ImageEmbedder):
    """The multi-view conditioner of the MV23D release (reference :871-1104; config
    sgm/configs/mv23d-plucker-clipl-compat-fm-lognorm-noclip.yaml: arch='vitb', enable_bf16=True, n_cond_frames=6,
    modLN=False, aug_c=True, input_key 'img-c'): DINOv2 ViT-B/14 with 4 registers whose patch embedding takes 9
    channels, RGB plus the Plücker ray [o x d, d] of every pixel of the 224 x 224 view.  forward({'img': (B,V,3,H,W),
    'c': (B,V,25)}) -> normalised patch tokens (B, n_cond_frames, 256, width), which GeneralConditioner files under
    'concat'.

    The 9-channel patch operand comes from one kernel (ops.plucker_patchify: rays, cat, bf16 cast and im2col) and the
    patch embedding from one GEMM; the tower is FrozenDinov2ImageEmbedder's.  The operand is bf16 whatever
    `enable_bf16` says: under the engine's bf16 autocast the reference's patch-embedding conv rounds it to bf16 too.
    `modLN` is accepted and ignored, as in the reference.

    aug_c=True rotates each conditioning camera with probability 0.4 before the rays are built -- at inference too,
    as the reference does (:1079-1088): `random.random()` per (b, v) and, on a hit, `np.random.uniform` for the angle
    and `random.random()` for the axis, rotating the caller's camera tensor in place, in its dtype."""

    def __init__(self, arch="vitl", version="dinov2", device="cuda", max_length=77, freeze=True, antialias=True,
                 ucg_rate=0.0, unsqueeze_dim=False, repeat_to_max_len=False, num_image_crops=0, output_tokens=False,
                 output_cls=False, init_device=None, n_cond_frames=4, enable_bf16=False, modLN=False, aug_c=False, *,
                 state_dict: dict | None = None, random_init: bool = False, width=768, depth=12, mlp_dim=3072, patch=14,
                 num_register_tokens=4, pos_grid=37, interpolate_antialias=True, interpolate_offset=0.0, seed=0):
        if output_cls:
            raise NotImplementedError("FrozenDinov2ImageEmbedderMVPlucker: output_cls (the reference cannot run it either)")
        if state_dict is None and not random_init:
            def _load():
                model = torch.hub.load(f"facebookresearch/{version}", f"{version}_{arch}14_reg", pretrained=True)  # :760-765
                return {"model." + k: v for k, v in model.state_dict().items()}
            state_dict = _load_pretrained("FrozenDinov2ImageEmbedderMVPlucker", _load)
        if state_dict is None:
            state_dict = FrozenDinov2ImageEmbedder._random_state_dict(width, depth, mlp_dim, patch, num_register_tokens,
                                                                      pos_grid, seed, in_chans=9)
        super().__init__(arch, version, device, max_length, freeze, antialias, ucg_rate, unsqueeze_dim, repeat_to_max_len,
                         num_image_crops, output_tokens, output_cls, init_device,
                         state_dict=_nine_channel_patch_embed(state_dict), interpolate_antialias=interpolate_antialias,
                         interpolate_offset=interpolate_offset)
        if self.patch != 14 or self._conv_w.shape[1] != 1792:
            raise NotImplementedError("FrozenDinov2ImageEmbedderMVPlucker: a 9-channel 14x14 patch embedding is required")
        self.n_cond_frames = n_cond_frames
        self.enable_bf16 = enable_bf16
        self.dtype = torch.bfloat16 if enable_bf16 else torch.float32
        self.aug_c = aug_c
        self.reso_encoder = 224

    def preprocess(self, x):
        """reference :1015-1047.  Its ucg_rate > 0 branch (scale jitter and Gaussian noise) runs only outside
        get_unconditional_conditioning, i.e. in training."""
        if self.ucg_rate > 0.0:
            raise NotImplementedError("FrozenDinov2ImageEmbedderMVPlucker with ucg_rate > 0: the reference's "
                                      "training-time augmentation is not implemented (inference runs through "
                                      "GeneralConditioner.get_unconditional_conditioning, which sets ucg_rate = 0)")
        return super().preprocess(x)

    @staticmethod
    def draw_rotation() -> tuple:
        """The draws of random_rotate_c: (angle, about_z) from np.random.uniform(0, 2 pi), then random.random() > 0.5."""
        degree = np.random.uniform(0, math.pi * 2)
        return degree, random.random() > 0.5

    @staticmethod
    def rotate_c(c: torch.Tensor, degree, about_z: bool) -> torch.Tensor:
        """The rotation of random_rotate_c for given draws: about z or y by `degree`, applied to the cam2world of one
        (25,) camera row on its device, in its dtype."""
        intrinsics, c2ws = c[16:], c[:16].reshape(4, 4)
        cs, sn = np.cos(degree), np.sin(degree)
        if about_z:
            rot = [[cs, -sn, 0, 0], [sn, cs, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]]
        else:
            rot = [[cs, 0, sn, 0], [0, 1, 0, 0], [-sn, 0, cs, 0], [0, 0, 0, 1]]
        rot = torch.tensor(rot).to(c2ws)
        return torch.cat([torch.matmul(rot, c2ws).reshape(-1), intrinsics])

    @classmethod
    def random_rotate_c(cls, c: torch.Tensor) -> torch.Tensor:
        """reference :1049-1076: a random rotation about z or y (InstantMesh's camera augmentation) applied to the
        cam2world of one (25,) camera row, in the row's dtype.  RNG: np.random.uniform, then random.random()."""
        return cls.rotate_c(c, *cls.draw_rotation())

    @classmethod
    def draw_camera_augmentation(cls, B: int, V: int) -> list:
        """The host RNG draws of augment_cameras on a (B, V, 25) batch, in its order: per (b, v) random.random() > 0.6
        decides, and a hit draws the rotation (draw_rotation).  Returns B lists of V entries, (degree, about_z) or
        None.  Nothing is applied, so a caller can advance `random` and `np.random` exactly as augment_cameras would."""
        return [[cls.draw_rotation() if random.random() > 0.6 else None for _ in range(V)] for _ in range(B)]

    @classmethod
    def apply_camera_augmentation(cls, c: torch.Tensor, draws: list) -> torch.Tensor:
        """Rotates the cameras of c (B, V, 25) in place by draws of draw_camera_augmentation(B, V), on c's device, in
        its dtype.  Draws no random numbers."""
        for b, row in enumerate(draws):
            for v, d in enumerate(row):
                if d is not None:
                    c[b, v] = cls.rotate_c(c[b, v], *d)
        return c

    @classmethod
    def augment_cameras(cls, c: torch.Tensor) -> torch.Tensor:
        """aug_c (reference :1084-1088): every camera of c (B, V, 25) is rotated, in place, with probability 0.4."""
        return cls.apply_camera_augmentation(c, cls.draw_camera_augmentation(c.shape[0], c.shape[1]))

    def draw_augmentation(self, img_c) -> list | None:
        """The host RNG draws forward(img_c) makes (its aug_c camera draws, or none), made without running it."""
        return self.draw_camera_augmentation(*img_c["c"].shape[:2]) if self.aug_c else None

    def encode_with_vision_transformer(self, img, cams=None, **kwargs):
        """(B*V, 3, H, W) views + (B*V, 25) cameras -> patch tokens (B*V, 256, width)."""
        if img.dim() == 5:
            img = img.reshape(-1, *img.shape[2:])
        dev = self.cls_token.device
        img = self.preprocess(img.to(dev)).contiguous()
        a = ops.plucker_patchify(img, cams.to(device=dev, dtype=torch.float32).contiguous(), ldo=self._conv_w.shape[1])
        patches = ops.gemm(a, self._conv_w, self._conv_b).float().view(img.shape[0], -1, self._conv_w.shape[0])
        return self.forward_features(img, patch_tokens=patches)["x_norm_patchtokens"]

    def forward(self, img_c, no_dropout=False):
        mv_image, c = img_c["img"], img_c["c"]
        if self.aug_c:
            self.augment_cameras(c)
        B, V = mv_image.shape[0], self.n_cond_frames
        cams = c[:, :V].reshape(-1, c.shape[-1])
        tokens = super().forward(mv_image[:, :V], no_dropout=no_dropout, cams=cams)
        return tokens.reshape(B, -1, *tokens.shape[1:])
