"""Mirror of reference ldm/modules/diffusionmodules/model.py: the SD conv `Decoder` (:625-731) and
its blocks (ResnetBlock :94-153, Upsample :54-69, MemoryEfficientAttnBlock :209-272) as parameter
containers with the reference's state_dict keys.  The arithmetic runs in
ln3diff_b200.vit.vit_triplane on the NHWC fp32 conv kernels of libln3b200.

The stage-1 VAE encoders `MVEncoder` (:459-577, Downsample :72-91, mid-block SpatialTransformer3D of
ldm/modules/attention.py:390-463) and `MVEncoderGSDynamicInp` (:604-623, the DiT2-L/2 VAE's encoder) are built here
with their own NHWC forward: one shared trunk, then a conv fusion or a mean over the views.  Convolutions on ln3_conv_nhwc /
ln3_downsample_nhwc (TF32 by default, `conv_tf32 = False` for exact fp32), the multi-view transformer on the bf16
wgmma GEMM and attention kernels with fp32 accumulation and an fp32 residual stream."""
import torch
import torch.nn as nn

from .... import ops
from ...._lib import NORM_LAYER


def Normalize(in_channels, num_groups=32):
    return nn.GroupNorm(num_groups=num_groups, num_channels=in_channels, eps=1e-6, affine=True)


class Upsample(nn.Module):
    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if with_conv:
            self.conv = nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)


class ResnetBlock(nn.Module):
    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout, temb_channels=512):
        super().__init__()
        out_channels = in_channels if out_channels is None else out_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        assert temb_channels == 0 and not conv_shortcut
        self.norm1 = Normalize(in_channels)
        self.conv1 = nn.Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.norm2 = Normalize(out_channels)
        self.conv2 = nn.Conv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if in_channels != out_channels:
            self.nin_shortcut = nn.Conv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)


class MemoryEfficientAttnBlock(nn.Module):
    def __init__(self, in_channels):
        super().__init__()
        self.in_channels = in_channels
        self.norm = Normalize(in_channels)
        self.q = nn.Conv2d(in_channels, in_channels, kernel_size=1)
        self.k = nn.Conv2d(in_channels, in_channels, kernel_size=1)
        self.v = nn.Conv2d(in_channels, in_channels, kernel_size=1)
        self.proj_out = nn.Conv2d(in_channels, in_channels, kernel_size=1)


class Decoder(nn.Module):
    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, give_pre_end=False, tanh_out=False,
                 use_linear_attn=False, attn_type="vanilla", **ignorekwargs):
        super().__init__()
        if attn_resolutions or give_pre_end or tanh_out or use_linear_attn:
            raise NotImplementedError("only the conv_sr configuration of the release decoder is built")
        self.ch, self.num_resolutions, self.num_res_blocks = ch, len(ch_mult), num_res_blocks
        self.resolution, self.in_channels = resolution, in_channels
        block_in = ch * ch_mult[self.num_resolutions - 1]
        self.conv_in = nn.Conv2d(z_channels, block_in, kernel_size=3, stride=1, padding=1)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=0, dropout=dropout)
        self.mid.attn_1 = MemoryEfficientAttnBlock(block_in)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=0, dropout=dropout)
        self.up = nn.ModuleList()
        for i_level in reversed(range(self.num_resolutions)):
            block = nn.ModuleList()
            block_out = ch * ch_mult[i_level]
            for _ in range(num_res_blocks + 1):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=0, dropout=dropout))
                block_in = block_out
            up = nn.Module()
            up.block = block
            up.attn = nn.ModuleList()
            if i_level != 0:
                up.upsample = Upsample(block_in, resamp_with_conv)
            self.up.insert(0, up)
        self.norm_out = Normalize(block_in)
        self.conv_out = nn.Conv2d(block_in, out_ch, kernel_size=3, stride=1, padding=1)


# ---------------------------------------------------------------------------------------------- encoder
class Downsample(nn.Module):
    """model.py:72-91 parameters: Conv2d(C, C, 3, stride 2, padding 0) after F.pad(x, (0,1,0,1))."""

    def __init__(self, in_channels, with_conv):
        super().__init__()
        if not with_conv:
            raise NotImplementedError("Downsample(with_conv=False) (avg_pool2d) is not used by the release encoder")
        self.with_conv = with_conv
        self.conv = nn.Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)


class CrossAttention(nn.Module):
    """Parameters of the self-attention of BasicTransformerBlock (ldm/modules/attention.py:245-307): to_q/k/v without
    bias, to_out = Sequential(Linear, Dropout).  q_norm / k_norm are identities in the encoder (qk_norm=False)."""

    def __init__(self, query_dim, heads=8, dim_head=64):
        super().__init__()
        inner = heads * dim_head
        self.heads, self.dim_head = heads, dim_head
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(query_dim, inner, bias=False)
        self.to_v = nn.Linear(query_dim, inner, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, query_dim), nn.Dropout(0.0))


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(nn.Module):
    """FeedForward(dim, glu=True) (attention.py:54-81): net = [GEGLU(dim, 4 dim), Dropout, Linear(4 dim, dim)]."""

    def __init__(self, dim, mult=4):
        super().__init__()
        inner = int(dim * mult)
        self.net = nn.Sequential(GEGLU(dim, inner), nn.Dropout(0.0), nn.Linear(inner, dim))


class BasicTransformerBlock3D(nn.Module):
    """attention.py:310-340, 390-402: attn1 over the tokens of all views of an object, attn2 per view, GEGLU FF, each
    behind an affine LayerNorm (eps 1e-5) and a residual."""

    def __init__(self, dim, n_heads, d_head):
        super().__init__()
        self.attn1 = CrossAttention(dim, n_heads, d_head)
        self.ff = FeedForward(dim)
        self.attn2 = CrossAttention(dim, n_heads, d_head)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(dim), nn.LayerNorm(dim), nn.LayerNorm(dim)


class SpatialTransformer3D(nn.Module):
    """attention.py:405-463 with depth 1, no context, use_linear=False: GroupNorm -> proj_in (1x1) -> tokens ->
    BasicTransformerBlock3D -> proj_out (1x1, zero-initialised in the reference) + x_in."""

    def __init__(self, in_channels, n_heads, d_head, depth=1, dropout=0.0, context_dim=None, disable_self_attn=False,
                 use_linear=False, use_checkpoint=True):
        super().__init__()
        if depth != 1 or context_dim is not None or disable_self_attn or use_linear or dropout:
            raise NotImplementedError("only the encoder's SpatialTransformer3D (depth 1, self-attention, 1x1 convs) is built")
        inner = n_heads * d_head
        self.in_channels, self.n_heads, self.d_head = in_channels, n_heads, d_head
        self.norm = Normalize(in_channels)
        self.proj_in = nn.Conv2d(in_channels, inner, kernel_size=1, stride=1, padding=0)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock3D(inner, n_heads, d_head)])
        self.proj_out = nn.Conv2d(inner, in_channels, kernel_size=1, stride=1, padding=0)
        nn.init.zeros_(self.proj_out.weight)
        nn.init.zeros_(self.proj_out.bias)
        self.use_linear = False


class _MVEncoderTrunk(nn.Module):
    """The SD `Encoder` (model.py:459-560) with the 'mv-vanilla' mid-block attention, as the multi-view encoders build
    it: parameters as the reference's, forward on the NHWC kernels.  The reference's single-view `Encoder` (ShapeNet /
    FFHQ configurations, outside the release inference paths) is not mirrored and keeps resolving to the reference's
    own class under the overlay."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, double_z=True, use_linear_attn=False,
                 attn_type="mv-vanilla", attn_kwargs={}, add_fusion_layer=False, **ignore_kwargs):
        super().__init__()
        if attn_type != "mv-vanilla" or attn_resolutions or use_linear_attn or dropout:
            raise NotImplementedError("attn_type other than 'mv-vanilla', attn_resolutions, linear attention and dropout "
                                      "are not used by the release encoder")
        self.ch, self.temb_ch = ch, 0
        self.num_resolutions, self.num_res_blocks = len(ch_mult), num_res_blocks
        self.resolution, self.in_channels = resolution, in_channels
        self.conv_in = nn.Conv2d(in_channels, ch, kernel_size=3, stride=1, padding=1)
        in_ch_mult = (1,) + tuple(ch_mult)
        self.in_ch_mult = in_ch_mult
        self.down = nn.ModuleList()
        block_in = ch
        for i_level in range(self.num_resolutions):
            block = nn.ModuleList()
            block_in, block_out = ch * in_ch_mult[i_level], ch * ch_mult[i_level]
            for _ in range(num_res_blocks):
                block.append(ResnetBlock(in_channels=block_in, out_channels=block_out, temb_channels=0, dropout=dropout))
                block_in = block_out
            down = nn.Module()
            down.block = block
            down.attn = nn.ModuleList()
            if i_level != self.num_resolutions - 1:
                down.downsample = Downsample(block_in, resamp_with_conv)
            self.down.append(down)
        self.mid = nn.Module()
        self.mid.block_1 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=0, dropout=dropout)
        self.mid.attn_1 = SpatialTransformer3D(block_in, **attn_kwargs)
        self.mid.block_2 = ResnetBlock(in_channels=block_in, out_channels=block_in, temb_channels=0, dropout=dropout)
        self.norm_out = Normalize(block_in)
        zc = 2 * z_channels if double_z else z_channels
        self.conv_out = nn.Conv2d(block_in, zc, kernel_size=3, stride=1, padding=1)
        if add_fusion_layer:
            self.fusion_layer = nn.Conv2d(zc * 4, zc, kernel_size=3, stride=1, padding=1)
        self._prep = None

    # ------------------------------------------------------------------ weight repack
    def _apply(self, fn, *a, **kw):
        self._prep = None
        return super()._apply(fn, *a, **kw)

    def load_state_dict(self, *a, **kw):
        self._prep = None
        return super().load_state_dict(*a, **kw)

    @torch.no_grad()
    def prepare(self):
        dev = self.conv_in.weight.device
        if dev.type != "cuda":
            raise RuntimeError("ln3diff_b200 encoder runs on CUDA only (no CPU fallback)")
        bf = lambda w: w.detach().to(dev, torch.bfloat16).contiguous()
        f32 = lambda w: w.detach().to(dev, torch.float32).contiguous()
        pk = lambda conv: (f32(conv.weight.permute(2, 3, 1, 0).reshape(-1, conv.weight.shape[1], conv.weight.shape[0])),
                           f32(conv.bias))
        ln = lambda n: (f32(n.bias).reshape(1, -1), (f32(n.weight) - 1.0).reshape(1, -1).contiguous())

        def res(rb):
            d = dict(n1=(f32(rb.norm1.weight), f32(rb.norm1.bias)), c1=pk(rb.conv1),
                     n2=(f32(rb.norm2.weight), f32(rb.norm2.bias)), c2=pk(rb.conv2))
            if hasattr(rb, "nin_shortcut"):
                d["nin"] = pk(rb.nin_shortcut)
            return d

        st = self.mid.attn_1
        tb = st.transformer_blocks[0]
        inner = st.n_heads * st.d_head
        att = lambda a: dict(qkv=bf(torch.cat([a.to_q.weight, a.to_k.weight, a.to_v.weight], 0)),
                             o=(bf(a.to_out[0].weight), f32(a.to_out[0].bias)))
        g = tb.ff.net[0].proj
        self._prep = dict(
            conv_in=pk(self.conv_in),
            down=[dict(blocks=[res(b) for b in d.block], down=pk(d.downsample.conv) if hasattr(d, "downsample") else None)
                  for d in self.down],
            mid1=res(self.mid.block_1), mid2=res(self.mid.block_2),
            st=dict(n=(f32(st.norm.weight), f32(st.norm.bias)), proj_in=pk(st.proj_in), proj_out=pk(st.proj_out),
                    ln1=ln(tb.norm1), ln2=ln(tb.norm2), ln3=ln(tb.norm3), attn1=att(tb.attn1), attn2=att(tb.attn2),
                    # GEGLU: proj(x).chunk(2, -1) = (value, gate) -> value rows [0, inner*4), gate rows after them
                    ff_v=(bf(g.weight[:4 * inner]), f32(g.bias[:4 * inner])),
                    ff_g=(bf(g.weight[4 * inner:]), f32(g.bias[4 * inner:])),
                    ff_o=(bf(tb.ff.net[2].weight), f32(tb.ff.net[2].bias))),
            norm_out=(f32(self.norm_out.weight), f32(self.norm_out.bias)), conv_out=pk(self.conv_out))
        if hasattr(self, "fusion_layer"):
            self._prep["fusion"] = pk(self.fusion_layer)
        return self._prep

    # ------------------------------------------------------------------ forward (NHWC)
    # 3x3 convolutions (and the stride-2 Downsample convs) on the tensor cores: TF32 operands, fp32 accumulate.
    # False: exact fp32 SIMT convolutions.  The mid-block transformer always runs bf16 GEMM operands with fp32
    # accumulation and an fp32 residual stream.
    conv_tf32 = True

    def _res(self, x, W):
        tf = self.conv_tf32
        h = ops.conv_nhwc(x, *W["c1"], ksize=3, gn=ops.groupnorm_stats(x, *W["n1"]), swish=True, tf32=tf)
        sc = ops.conv_nhwc(x, *W["nin"], ksize=1) if "nin" in W else x
        return ops.conv_nhwc(h, *W["c2"], ksize=3, gn=ops.groupnorm_stats(h, *W["n2"]), swish=True, residual=sc, tf32=tf)

    def _attn(self, a, A, xs, groups: int, heads: int, inner: int):
        """x += to_out(softmax attention of to_q/k/v(a)) with the tokens split into `groups` sequences."""
        rows = a.shape[0]
        qkv = ops.gemm(a, A["qkv"])
        q3 = qkv.view(groups, rows // groups, 3 * inner)
        att = ops.fmha(q3[:, :, :inner], q3[:, :, inner:2 * inner], q3[:, :, 2 * inner:], heads)
        ops.gemm(att.view(rows, inner), A["o"][0], A["o"][1], out_kind=ops.OUT_RESID_F32, out=xs)

    def _spatial_transformer(self, h, P, num_frames: int):
        """SpatialTransformer3D.forward (attention.py:442-463) on NHWC h (N, H, W, C) -> (N, H, W, C)."""
        st = self.mid.attn_1
        N, H, W_, _ = h.shape
        heads, inner = st.n_heads, st.n_heads * st.d_head
        rows = N * H * W_
        t = ops.conv_nhwc(h, *P["proj_in"], ksize=1, gn=ops.groupnorm_stats(h, *P["n"]))   # (N, H, W, inner) fp32
        xs = t.view(rows, inner)                                                           # the residual stream
        ln = lambda pair: ops.norm_modulate(xs, norm=NORM_LAYER, shift=pair[0], scale=pair[1], mod_rows=rows, eps=1e-5)
        # attn1: '(b f) l c -> b (f l) c' -- in NHWC the views of an object are already consecutive rows
        self._attn(ln(P["ln1"]), P["attn1"], xs, N // num_frames, heads, inner)
        self._attn(ln(P["ln2"]), P["attn2"], xs, N, heads, inner)
        ops.gemm(self._geglu(ln(P["ln3"]), P)[1], *P["ff_o"], out_kind=ops.OUT_RESID_F32, out=xs)
        return ops.conv_nhwc(t, *P["proj_out"], ksize=1, residual=h)

    @staticmethod
    def _geglu(a, P):
        """GEGLU (attention.py:54-61) of the bf16 rows `a`: value * gelu_erf(gate) in fp32 and its bf16 copy (the
        operand of ff.net.2).  The gate GEMM applies erf-GELU in its epilogue; the value GEMM's gated-residual epilogue
        adds gate * value onto zeros, i.e. writes the product, and stores the bf16 copy."""
        gate = ops.gemm(a, *P["ff_g"], act=ops.ACT_GELU_ERF, out_kind=ops.OUT_F32)
        prod = torch.zeros_like(gate)
        prod_bf = torch.empty(gate.shape, device=gate.device, dtype=torch.bfloat16)
        ops.gemm(a, *P["ff_v"], out_kind=ops.OUT_RESID_F32, out=prod, gate=gate, gate_rows=1, out2=prod_bf)
        return prod, prod_bf

    def _trunk_nhwc(self, x, num_frames: int):
        """Encoder.forward (model.py:526-560) with the mid-block attention over groups of `num_frames` views:
        x (B*F, in_channels, R, R) fp32 CUDA -> per-view moments (B*F, R/8, R/8, 2*z_channels) NHWC fp32."""
        if not x.is_cuda:
            raise RuntimeError("ln3diff_b200 encoder runs on CUDA only (no CPU fallback)")
        if self._prep is None:
            self.prepare()
        P = self._prep
        F_ = num_frames
        assert x.dim() == 4 and x.shape[0] % F_ == 0 and x.shape[1] == self.in_channels, "x must be (B*views, C, H, W)"
        tf = self.conv_tf32
        h = x.float().permute(0, 2, 3, 1).contiguous()                         # NCHW -> NHWC (plumbing copy)
        h = ops.conv_nhwc(h, *P["conv_in"], ksize=3, tf32=tf)
        for lvl in P["down"]:
            for W in lvl["blocks"]:
                h = self._res(h, W)
            if lvl["down"] is not None:
                h = ops.downsample_nhwc(h, *lvl["down"], tf32=tf)
        h = self._res(h, P["mid1"])
        h = self._spatial_transformer(h, P["st"], F_)
        h = self._res(h, P["mid2"])
        return ops.conv_nhwc(h, *P["conv_out"], ksize=3, gn=ops.groupnorm_stats(h, *P["norm_out"]), swish=True, tf32=tf)


class MVEncoder(_MVEncoderTrunk):
    """model.py:563-577: the trunk plus a conv fusion of the 4 views of each object (pixel-nerf style)."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, double_z=True, use_linear_attn=False,
                 attn_type="mv-vanilla", attn_kwargs={}, **ignore_kwargs):
        super().__init__(ch=ch, out_ch=out_ch, ch_mult=ch_mult, num_res_blocks=num_res_blocks,
                         attn_resolutions=attn_resolutions, dropout=dropout, resamp_with_conv=resamp_with_conv,
                         in_channels=in_channels, resolution=resolution, z_channels=z_channels, double_z=double_z,
                         use_linear_attn=use_linear_attn, attn_type=attn_type, attn_kwargs=attn_kwargs,
                         add_fusion_layer=True)
        self.num_frames = 4

    @torch.no_grad()
    def forward_nhwc(self, x):
        """x (B*4, in_channels, R, R) fp32 CUDA -> fused moments (B, R/8, R/8, 2*z_channels) NHWC fp32."""
        F_ = self.num_frames
        h = self._trunk_nhwc(x, F_)
        N, S, _, Z = h.shape
        # fusion_layer(cat(feat.chunk(F), dim=1)): input channel v*Z + c is channel c of view v
        fused = h.view(N // F_, F_, S, S, Z).permute(0, 2, 3, 1, 4).reshape(N // F_, S, S, F_ * Z)
        return ops.conv_nhwc(fused, *self._prep["fusion"], ksize=3, tf32=self.conv_tf32)

    def forward(self, x):
        """(B*4, in_channels, 256, 256) fp32 -> moments (B, 2*z_channels, 32, 32) fp32, returned as an NCHW view of the
        NHWC kernel output (torch.channels_last memory format)."""
        return self.forward_nhwc(x).permute(0, 3, 1, 2)


class MVEncoderGS(nn.Module):
    def __init__(self, *a, **kw):
        raise NotImplementedError("MVEncoderGS (pixel-aligned Gaussian-splatting encoder) is not part of the release "
                                  "VAE; only MVEncoder is built")


class MissingArgumentError(NotImplementedError, TypeError):
    """A required constructor argument is missing.  A TypeError as Python raises for the reference's signature, and a
    NotImplementedError like the other encoder configurations this package does not build."""


_REQUIRED = object()


class MVEncoderGSDynamicInp(_MVEncoderTrunk):
    """model.py:604-623, the encoder of the DiT2-L/2 VAE (dino_version 'mv-sd-dit-dynaInp-trilatent', num_frames 6 in
    the release scripts): the trunk without a fusion layer, then the mean of the per-view moments over each object's
    views (ln3_view_mean_nhwc)."""

    def __init__(self, *, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions, dropout=0,
                 resamp_with_conv=True, in_channels, resolution, z_channels, double_z=True, use_linear_attn=False,
                 attn_type="mv-vanilla", num_frames=_REQUIRED, **ignore_kwargs):
        if num_frames is _REQUIRED:
            raise MissingArgumentError("MVEncoderGSDynamicInp.__init__() missing 1 required keyword-only argument: "
                                       "'num_frames'")
        super().__init__(ch=ch, out_ch=out_ch, ch_mult=ch_mult, num_res_blocks=num_res_blocks,
                         attn_resolutions=attn_resolutions, dropout=dropout, resamp_with_conv=resamp_with_conv,
                         in_channels=in_channels, resolution=resolution, z_channels=z_channels, double_z=double_z,
                         use_linear_attn=use_linear_attn, attn_type=attn_type, add_fusion_layer=False, **ignore_kwargs)
        self.num_frames = num_frames

    @torch.no_grad()
    def forward_nhwc(self, x, num_frames=None):
        """x (B*F, in_channels, R, R) fp32 CUDA -> pooled moments (B, R/8, R/8, 2*z_channels) NHWC fp32.  As the
        reference, the mid-block attention groups the views by self.num_frames whatever `num_frames` is; `num_frames`
        (default self.num_frames) only sets the pooling: h.chunk(N // num_frames), then the mean of each chunk."""
        h = self._trunk_nhwc(x, self.num_frames)
        if num_frames is None:
            num_frames = self.num_frames
        assert num_frames > 4
        N = h.shape[0]
        if N // num_frames <= 0:
            raise RuntimeError(f"chunk expects `chunks` to be greater than 0, got: {N // num_frames}")
        size = -(-N // (N // num_frames))  # torch.chunk: equal chunks of ceil(N / chunks), a shorter last one
        full = N // size
        out = ops.view_mean_nhwc(h[:full * size], size)
        if full * size < N:
            out = torch.cat([out, ops.view_mean_nhwc(h[full * size:], N - full * size)], 0)
        return out

    def forward(self, x, num_frames=None):
        """(B*F, in_channels, 256, 256) fp32 -> moments (B, 2*z_channels, 32, 32) fp32, returned as an NCHW view of the
        NHWC kernel output (torch.channels_last memory format)."""
        return self.forward_nhwc(x, num_frames).permute(0, 3, 1, 2)
