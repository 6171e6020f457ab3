// Convolutional tail of the tri-plane VAE decoder (fp32 SIMT, NHWC).
//
// Replaces the cuDNN / aten launches of the reference's `superresolution['conv_sr']` =
// ldm Decoder(z_channels=1024, ch=32, ch_mult=[1,2,2,4], num_res_blocks=1, out_ch=32)
// (ldm/modules/diffusionmodules/model.py:625-731: ResnetBlock :94-153, Upsample :54-69,
// MemoryEfficientAttnBlock :209-272, GroupNorm(32, eps 1e-6) + swish :46-52) and of
// PatchEmbedTriplane (vit/vit_triplane.py:58-108).
//
// Layout: activations are NHWC fp32.  The DiT2 decoder's token stream (3B, 16*16, 1024) already IS
// NHWC, and the last conv writes (3B, 128, 128, 32) = exactly the channels-last tri-plane the ray
// marcher gathers from, so the reference's '(b n) c h w' / 'b (n c) h w' permute copies disappear.
//   conv_nhwc       3x3 (pad 1) or 1x1 conv + bias, optional fused GroupNorm-apply + swish on the
//                   input (per (image, channel) scale/shift from groupnorm_stats), optional fused
//                   nearest-2x upsample of the input, optional residual add
//   groupnorm_stats per (image, group) mean / rstd -> per (image, channel) scale / shift
//   attn_single_head  softmax(q k^T / sqrt(C)) v for the 256-token mid block (C = 128)
//   patch_embed_triplane  grouped 2x2/s2 conv + the reference's channel interleave -> tokens
// The decode is < 1 % of the pipeline's FLOPs (20 GFLOP / latent vs 307 TFLOP of sampling), so these
// kernels favour exact fp32 parity with the reference over tensor-core throughput.
#include "common.cuh"
#include "ln3_internal.h"

namespace ln3 {

// ------------------------------------------------------------------ conv (NHWC, direct)
// Block: 8x8 output pixels x COT output channels; 256 threads = 64 pixels x 4 channel groups, each
// thread accumulates COT/4 channels.  Input channels are consumed in chunks of 16 staged in smem as
// [cin][10x10 halo tile] (pixel fastest -> conflict-free reads), weights as [tap][cin][COT].
//
// DOWN = the encoder's Downsample (ldm/modules/diffusionmodules/model.py:72-91): F.pad(x, (0,1,0,1)) then a 3x3
// conv with stride 2 and no padding.  a.H, a.W are then the (even) INPUT dims; the 8x8 output tile reads input rows
// and columns [2*t0, 2*t0 + 17), a 17x17 tile whose last row / column is the zero pad at the image edge.  Each
// staged row is stored de-interleaved -- even columns at positions 0..8, odd columns at 9..16 -- so that the eight
// output columns of one tap read eight consecutive words.
static constexpr int kCT = 8;        // tile edge (pixels)
static constexpr int kCinChunk = 16;
static constexpr int kDownTW = 2 * kCT + 1;   // staged tile edge of the stride-2 conv

// staged position of tile column c (0..16) in a de-interleaved stride-2 row, and its inverse
__device__ __forceinline__ int down_pos(int c) { return (c & 1) ? 9 + (c >> 1) : (c >> 1); }
__device__ __forceinline__ int down_col(int p) { return p < 9 ? 2 * p : 2 * (p - 9) + 1; }

template <int COT, int KS, bool DOWN>
__global__ void __launch_bounds__(256)
conv_nhwc_kernel(const ln3_conv_args a) {
  static_assert(!DOWN || KS == 3, "the stride-2 conv is 3x3");
  constexpr int HALO = (KS == 3 && !DOWN) ? 1 : 0;
  constexpr int TW = DOWN ? kDownTW : kCT + 2 * HALO;   // staged tile edge
  constexpr int NACC = COT / 4;
  __shared__ float s_in[kCinChunk][TW * TW + 1];
  __shared__ __align__(16) float s_w[KS * KS][kCinChunk][COT];

  const int n = blockIdx.z;
  const int Ho = DOWN ? a.H / 2 : a.H, Wo = DOWN ? a.W / 2 : a.W;
  const int tiles_x = (Wo + kCT - 1) / kCT;
  const int ty0 = (blockIdx.x / tiles_x) * kCT, tx0 = (blockIdx.x % tiles_x) * kCT;
  const int co0 = blockIdx.y * COT;
  const int pix = threadIdx.x & 63, q = threadIdx.x >> 6;
  const int py = pix >> 3, px = pix & 7;
  const int Hin = a.upsample ? a.H / 2 : a.H, Win = a.upsample ? a.W / 2 : a.W;

  float acc[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0.f;

  for (int c0 = 0; c0 < a.Cin; c0 += kCinChunk) {
    // stage input tile (GroupNorm-apply + swish + nearest upsample fused into the load)
    for (int i = threadIdx.x; i < TW * TW * kCinChunk; i += 256) {
      const int ci = i % kCinChunk, t = i / kCinChunk;   // channel fastest in gmem (NHWC)
      const int yy = DOWN ? 2 * ty0 + t / TW : ty0 + t / TW - HALO;
      const int xx = DOWN ? 2 * tx0 + down_col(t % TW) : tx0 + t % TW - HALO;
      float v = 0.f;
      if (yy >= 0 && yy < a.H && xx >= 0 && xx < a.W && c0 + ci < a.Cin) {
        const int ys = a.upsample ? (yy >> 1) : yy, xs = a.upsample ? (xx >> 1) : xx;
        v = a.x[((static_cast<long long>(n) * Hin + ys) * Win + xs) * a.Cin + c0 + ci];
        if (a.in_scale != nullptr) {
          v = fmaf(v, a.in_scale[n * a.Cin + c0 + ci], a.in_shift[n * a.Cin + c0 + ci]);
          if (a.in_swish) v = v / (1.f + __expf(-v));
        }
      }
      s_in[ci][t] = v;
    }
    // stage weights [tap][cin][COT] from the repacked [KS*KS][Cin][Cout] tensor
    for (int i = threadIdx.x; i < KS * KS * kCinChunk * COT; i += 256) {
      const int co = i % COT, r = i / COT, ci = r % kCinChunk, tap = r / kCinChunk;
      float w = 0.f;
      if (c0 + ci < a.Cin && co0 + co < a.Cout)
        w = a.w[(static_cast<long long>(tap) * a.Cin + c0 + ci) * a.Cout + co0 + co];
      s_w[tap][ci][co] = w;
    }
    __syncthreads();
#pragma unroll
    for (int tap = 0; tap < KS * KS; ++tap) {
      const int t = DOWN ? (2 * py + tap / 3) * TW + down_pos(2 * px + tap % 3) : (py + tap / KS) * TW + (px + tap % KS);
#pragma unroll 4
      for (int ci = 0; ci < kCinChunk; ++ci) {
        const float xv = s_in[ci][t];
        const float4* wp = reinterpret_cast<const float4*>(&s_w[tap][ci][q * NACC]);
#pragma unroll
        for (int i = 0; i < NACC / 4; ++i) {
          const float4 w = wp[i];
          acc[4 * i + 0] = fmaf(xv, w.x, acc[4 * i + 0]);
          acc[4 * i + 1] = fmaf(xv, w.y, acc[4 * i + 1]);
          acc[4 * i + 2] = fmaf(xv, w.z, acc[4 * i + 2]);
          acc[4 * i + 3] = fmaf(xv, w.w, acc[4 * i + 3]);
        }
      }
    }
    __syncthreads();
  }
  const int oy = ty0 + py, ox = tx0 + px;
  if (oy < Ho && ox < Wo) {
    const long long o = ((static_cast<long long>(n) * Ho + oy) * Wo + ox) * a.Cout + co0 + q * NACC;
#pragma unroll
    for (int i = 0; i < NACC; ++i) {
      const int co = co0 + q * NACC + i;
      if (co < a.Cout) {
        float v = acc[i] + (a.bias ? a.bias[co] : 0.f);
        if (a.residual) v += a.residual[o + i];
        a.out[o + i] = v;
      }
    }
  }
}

// ------------------------------------------------------------------ 3x3 conv on the tensor cores (TF32)
// Same tiling and the same fused prologue as conv_nhwc_kernel<COT, 3>; the inner product becomes an implicit
// GEMM per block -- M = 64 output pixels, N = COT channels, K = 16 input channels x 9 taps per staged chunk --
// issued as mma.sync.m16n8k8 TF32 (fp32 accumulate): 72 MMAs + 216 LDS per warp and chunk instead of
// 2304 FFMA + 720 LDS per thread.  Warp w: pixel rows 2*(w&3), 2*(w&3)+1 of the 8x8 tile (one m-tile),
// channel half w>>2.  smem rows are padded to strides = 8 (mod 32) words so that the (g, t) fragment
// pattern of a warp touches 32 distinct banks.  DOWN: the stride-2 Downsample conv on the 17x17 de-interleaved tile of
// conv_nhwc_kernel (a.H, a.W = input dims); the eight A rows g of one tap are then eight consecutive staged words.
template <int COT, bool DOWN>
__global__ void __launch_bounds__(256)
conv3x3_tf32_kernel(const ln3_conv_args a) {
  constexpr int TW = DOWN ? kDownTW : kCT + 2;   // staged tile edge
  constexpr int SIN = DOWN ? 296 : 104;          // >= TW*TW, = 8 (mod 32)
  constexpr int SW = COT + 8;            // = 8 (mod 32)
  constexpr int NT = COT / 16;           // n-tiles (of 8 channels) per warp
  __shared__ uint32_t s_in[kCinChunk][SIN];
  __shared__ uint32_t s_w[9][kCinChunk][SW];

  const int n = blockIdx.z;
  const int Ho = DOWN ? a.H / 2 : a.H, Wo = DOWN ? a.W / 2 : a.W;
  const int tiles_x = (Wo + kCT - 1) / kCT;
  const int ty0 = (blockIdx.x / tiles_x) * kCT, tx0 = (blockIdx.x % tiles_x) * kCT;
  const int co0 = blockIdx.y * COT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int mt = warp & 3, nh = warp >> 2;
  const int Hin = a.upsample ? a.H / 2 : a.H, Win = a.upsample ? a.W / 2 : a.W;

  float acc[NT][4];
#pragma unroll
  for (int i = 0; i < NT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;

  for (int c0 = 0; c0 < a.Cin; c0 += kCinChunk) {
    for (int i = threadIdx.x; i < TW * TW * kCinChunk; i += 256) {
      const int ci = i % kCinChunk, tt = i / kCinChunk;   // channel fastest in gmem (NHWC)
      const int yy = DOWN ? 2 * ty0 + tt / TW : ty0 + tt / TW - 1;
      const int xx = DOWN ? 2 * tx0 + down_col(tt % TW) : tx0 + tt % TW - 1;
      float v = 0.f;
      if (yy >= 0 && yy < a.H && xx >= 0 && xx < a.W && c0 + ci < a.Cin) {
        const int ys = a.upsample ? (yy >> 1) : yy, xs = a.upsample ? (xx >> 1) : xx;
        v = a.x[((static_cast<long long>(n) * Hin + ys) * Win + xs) * a.Cin + c0 + ci];
        if (a.in_scale != nullptr) {
          v = fmaf(v, a.in_scale[n * a.Cin + c0 + ci], a.in_shift[n * a.Cin + c0 + ci]);
          if (a.in_swish) v = v / (1.f + __expf(-v));
        }
      }
      s_in[ci][tt] = to_tf32(v);
    }
    for (int i = threadIdx.x; i < 9 * kCinChunk * COT; i += 256) {
      const int co = i % COT, r = i / COT, ci = r % kCinChunk, tap = r / kCinChunk;
      float w = 0.f;
      if (c0 + ci < a.Cin && co0 + co < a.Cout)
        w = a.w[(static_cast<long long>(tap) * a.Cin + c0 + ci) * a.Cout + co0 + co];
      s_w[tap][ci][co] = to_tf32(w);
    }
    __syncthreads();
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      // A rows: g -> pixel (2*mt, g), g + 8 -> pixel (2*mt + 1, g); shifted by the tap inside the halo tile
      const int p0 = DOWN ? (4 * mt + tap / 3) * TW + down_pos(2 * g + tap % 3) : (2 * mt + tap / 3) * TW + g + tap % 3;
      constexpr int DR = DOWN ? 2 * TW : TW;   // staged distance between the two output rows
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        const uint32_t af[4] = {s_in[8 * ks + t][p0], s_in[8 * ks + t][p0 + DR], s_in[8 * ks + t + 4][p0],
                                s_in[8 * ks + t + 4][p0 + DR]};
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
          const int cb = nh * (COT / 2) + nt * 8 + g;
          mma_tf32(acc[nt], af, s_w[tap][8 * ks + t][cb], s_w[tap][8 * ks + t + 4][cb]);
        }
      }
    }
    __syncthreads();
  }
  // D fragment: rows g / g + 8 = pixels (2*mt, g) / (2*mt + 1, g); columns 2t, 2t + 1 of each n-tile
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int oy = ty0 + 2 * mt + half, ox = tx0 + g;
    if (oy < Ho && ox < Wo) {
      const long long o = ((static_cast<long long>(n) * Ho + oy) * Wo + ox) * a.Cout;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const int co = co0 + nh * (COT / 2) + nt * 8 + 2 * t;
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (co + e < a.Cout) {
            float v = acc[nt][2 * half + e] + (a.bias ? a.bias[co + e] : 0.f);
            if (a.residual) v += a.residual[o + co + e];
            a.out[o + co + e] = v;
          }
      }
    }
  }
}

// 64 output channels per CTA, or 32 when the 64-channel grid would leave the GPU under two CTAs per SM (the 16 x 16
// and 32 x 32 levels of the VAE decoder: 192 CTAs; the kernel is bound by the latency of its staging loads -- ncu
// long_scoreboard 8.5 cycles per issue, 16 % warps active -- so more, smaller CTAs hide more of it).
int conv_cout_tile(int N, int H, int W, int Cout) {
  if (Cout < 64) return 32;
  const long long tiles = static_cast<long long>((H + kCT - 1) / kCT) * ((W + kCT - 1) / kCT);
  if (tiles * ((Cout + 63) / 64) * N < 2LL * device_sm_count()) return 32;
  return 64;
}

int conv_nhwc(const ln3_conv_args* a, cudaStream_t stream) {
  if (a->ksize != 1 && a->ksize != 3) return set_error(LN3_EUNSUPPORTED, "conv: ksize must be 1 or 3");
  if (a->precision != LN3_MLP_FP32 && a->precision != LN3_MLP_TF32)
    return set_error(LN3_EINVAL, "conv: precision must be LN3_MLP_FP32 or LN3_MLP_TF32");
  if (a->N < 0 || a->H <= 0 || a->W <= 0 || a->Cin <= 0 || a->Cout <= 0)
    return set_error(LN3_EINVAL, "conv: need N >= 0 and positive H, W, Cin, Cout");
  if (a->upsample && ((a->H | a->W) & 1)) return set_error(LN3_EINVAL, "conv: upsample needs even H, W");
  if ((a->in_scale == nullptr) != (a->in_shift == nullptr))
    return set_error(LN3_EINVAL, "conv: in_scale / in_shift must be given together");
  if (!a->x || !a->w || !a->out) return set_error(LN3_EINVAL, "conv: null pointer");
  if (a->N == 0) return LN3_OK;
  const int tiles = ((a->H + kCT - 1) / kCT) * ((a->W + kCT - 1) / kCT);
  const int cot = conv_cout_tile(a->N, a->H, a->W, a->Cout);
  dim3 grid(tiles, (a->Cout + cot - 1) / cot, a->N);
  if (a->ksize == 3 && a->precision == LN3_MLP_TF32) {
    if (cot == 64) conv3x3_tf32_kernel<64, false><<<grid, 256, 0, stream>>>(*a);
    else conv3x3_tf32_kernel<32, false><<<grid, 256, 0, stream>>>(*a);
  } else if (a->ksize == 3) {
    if (cot == 64) conv_nhwc_kernel<64, 3, false><<<grid, 256, 0, stream>>>(*a);
    else conv_nhwc_kernel<32, 3, false><<<grid, 256, 0, stream>>>(*a);
  } else {
    if (cot == 64) conv_nhwc_kernel<64, 1, false><<<grid, 256, 0, stream>>>(*a);
    else conv_nhwc_kernel<32, 1, false><<<grid, 256, 0, stream>>>(*a);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "conv launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// 32 output channels per CTA: the 17x17 staged tile with 64 channels of weights would exceed 48 KB of static smem
// (TF32: 18.9 KB input + 41.5 KB weights).  The encoder's three Downsample convs have 64..256 channels, so the grid
// is tiles x Cout/32 x views: 2048 / 1024 / 512 CTAs per 4 views.
int downsample_nhwc(const ln3_conv_args* a, cudaStream_t stream) {
  if (a->ksize != 3) return set_error(LN3_EINVAL, "downsample: ksize must be 3");
  if (a->upsample) return set_error(LN3_EINVAL, "downsample: upsample is not supported");
  if (a->in_scale != nullptr || a->in_shift != nullptr)
    return set_error(LN3_EINVAL, "downsample: in_scale / in_shift (fused GroupNorm) are not supported");
  if (a->residual != nullptr) return set_error(LN3_EINVAL, "downsample: residual is not supported");
  if (a->precision != LN3_MLP_FP32 && a->precision != LN3_MLP_TF32)
    return set_error(LN3_EINVAL, "downsample: precision must be LN3_MLP_FP32 or LN3_MLP_TF32");
  if (a->N < 0 || a->H <= 0 || a->W <= 0 || a->Cin <= 0 || a->Cout <= 0)
    return set_error(LN3_EINVAL, "downsample: need N >= 0 and positive H, W, Cin, Cout");
  if ((a->H | a->W) & 1) return set_error(LN3_EINVAL, "downsample: H, W (input dims) must be even");
  if (!a->x || !a->w || !a->out) return set_error(LN3_EINVAL, "downsample: null pointer");
  if (a->N == 0) return LN3_OK;
  const int tiles = ((a->H / 2 + kCT - 1) / kCT) * ((a->W / 2 + kCT - 1) / kCT);
  dim3 grid(tiles, (a->Cout + 31) / 32, a->N);
  if (a->precision == LN3_MLP_TF32) conv3x3_tf32_kernel<32, true><<<grid, 256, 0, stream>>>(*a);
  else conv_nhwc_kernel<32, 3, true><<<grid, 256, 0, stream>>>(*a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "downsample launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ VAE posterior (quant_conv + DiagonalGaussian)
// One thread per (object, pixel): the 24 fused moments of the pixel (NHWC) -> grouped 1x1 quant_conv (out channel o
// reads in channels [8*(o/8), 8*(o/8) + 8)) -> mean = channels 0..11, logvar = channels 12..23 (the reference's
// reshape (B, 8, 3, H, W) + chunk(2, dim=1): latent channel j = c*3 + n is conv channel j, its logvar conv channel
// 12 + j) -> soft clamp 20*tanh(lv/20) -> std = exp(0.5*lv) -> z = mean + std*noise.  The three outputs are written in
// the (B, 12, S, S) layout, consecutive threads on consecutive pixels.
__global__ void __launch_bounds__(256)
vae_posterior_kernel(const ln3_vae_posterior_args a) {
  __shared__ float s_w[24 * 8 + 24];
  for (int i = threadIdx.x; i < 24 * 8; i += blockDim.x) s_w[i] = a.w[i];
  if (threadIdx.x < 24) s_w[24 * 8 + threadIdx.x] = a.bias[threadIdx.x];
  __syncthreads();
  const int L = a.S * a.S;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(a.B) * L) return;
  const int b = static_cast<int>(idx / L), l = static_cast<int>(idx % L);
  float h[24];
  const float* hp = a.moments + idx * 24;
#pragma unroll
  for (int c = 0; c < 24; ++c) h[c] = __ldg(hp + c);
  const long long obase = static_cast<long long>(b) * 12 * L + l;
#pragma unroll
  for (int j = 0; j < 12; ++j) {
    float m = 0.f, lv = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      m = fmaf(s_w[j * 8 + k], h[(j / 8) * 8 + k], m);
      lv = fmaf(s_w[(12 + j) * 8 + k], h[((12 + j) / 8) * 8 + k], lv);
    }
    m = __fadd_rn(m, s_w[192 + j]);
    lv = __fadd_rn(lv, s_w[192 + 12 + j]);
    // torch: logvar.div(20.).tanh().mul(20.); std = exp(0.5 * logvar); mean + std * randn -- one rounding per op
    lv = __fmul_rn(tanhf(__fdiv_rn(lv, 20.f)), 20.f);
    const long long o = obase + static_cast<long long>(j) * L;
    a.mean[o] = m;
    a.logvar[o] = lv;
    a.z[o] = a.noise ? __fadd_rn(m, __fmul_rn(expf(__fmul_rn(0.5f, lv)), a.noise[o])) : m;
  }
}

int vae_posterior(const ln3_vae_posterior_args* a, cudaStream_t stream) {
  if (a->B < 0 || a->S <= 0) return set_error(LN3_EINVAL, "vae_posterior: need B >= 0 and S > 0");
  if (!a->moments || !a->w || !a->bias || !a->mean || !a->logvar || !a->z)
    return set_error(LN3_EINVAL, "vae_posterior: null pointer (only noise may be NULL)");
  if (a->B == 0) return LN3_OK;
  const long long n = static_cast<long long>(a->B) * a->S * a->S;
  if ((n + 255) / 256 > 0x7fffffffLL) return set_error(LN3_EINVAL, "vae_posterior: B*S*S too large");
  vae_posterior_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(*a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "vae_posterior launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ view mean (MVEncoderGSDynamicInp pooling)
// feat.mean(keepdim=True, dim=0) over the F consecutive views of each object: one thread per output element,
// consecutive threads on consecutive channels (coalesced reads of every view).  The sum runs over the views in
// order in fp32 and is divided by F once (IEEE division).
__global__ void __launch_bounds__(256)
view_mean_kernel(const float* __restrict__ x, float* __restrict__ out, long long n_out, long long per_view, int F) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  const long long b = i / per_view, r = i - b * per_view;
  const float* src = x + b * F * per_view + r;
  float s = __ldg(src);
  for (int f = 1; f < F; ++f) s = __fadd_rn(s, __ldg(src + f * per_view));
  out[i] = __fdiv_rn(s, static_cast<float>(F));
}

int view_mean_nhwc(const float* x, float* out, int B, int F, int S, int C, cudaStream_t stream) {
  if (F <= 0 || B < 0 || S <= 0 || C <= 0) return set_error(LN3_EINVAL, "view_mean_nhwc: need F > 0, B >= 0, S > 0, C > 0");
  if (!x || !out) return set_error(LN3_EINVAL, "view_mean_nhwc: null pointer");
  if (B == 0) return LN3_OK;
  const long long per_view = static_cast<long long>(S) * S * C, n = per_view * B;
  if ((n + 255) / 256 > 0x7fffffffLL) return set_error(LN3_EINVAL, "view_mean_nhwc: B*S*S*C too large");
  view_mean_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, stream>>>(x, out, n, per_view, F);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "view_mean_nhwc launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ GroupNorm statistics
// One block per (image, group): mean / biased variance over H*W*(C/G) elements (two-pass, fp32 with
// a shifted second pass for accuracy) -> per-channel scale = gamma*rstd, shift = beta - mean*scale.
__global__ void __launch_bounds__(256)
groupnorm_stats_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                       const float* __restrict__ beta, int HW, int C, int G, float eps,
                       float* __restrict__ scale, float* __restrict__ shift) {
  __shared__ float red[32];
  __shared__ float s_mean, s_rstd;
  const int n = blockIdx.y, g = blockIdx.x;
  const int cpg = C / G;
  const float* xb = x + static_cast<long long>(n) * HW * C + g * cpg;
  const long long cnt = static_cast<long long>(HW) * cpg;
  auto block_sum = [&](float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
    if (threadIdx.x < 32) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    __syncthreads();
    return t;  // valid in thread 0
  };
  float s = 0.f;
  for (long long i = threadIdx.x; i < cnt; i += blockDim.x) s += xb[(i / cpg) * C + (i % cpg)];
  s = block_sum(s);
  if (threadIdx.x == 0) s_mean = s / static_cast<float>(cnt);
  __syncthreads();
  const float mean = s_mean;
  float q = 0.f;
  for (long long i = threadIdx.x; i < cnt; i += blockDim.x) {
    const float d = xb[(i / cpg) * C + (i % cpg)] - mean;
    q = fmaf(d, d, q);
  }
  q = block_sum(q);
  if (threadIdx.x == 0) s_rstd = rsqrtf(q / static_cast<float>(cnt) + eps);
  __syncthreads();
  if (threadIdx.x < cpg) {
    const int c = g * cpg + threadIdx.x;
    const float sc = gamma[c] * s_rstd;
    scale[n * C + c] = sc;
    shift[n * C + c] = beta[c] - mean * sc;
  }
}

int groupnorm_stats(const float* x, const float* gamma, const float* beta, int N, int HW, int C, int G,
                    float eps, float* scale, float* shift, cudaStream_t stream) {
  if (N <= 0) return LN3_OK;
  if (G <= 0 || C <= 0 || HW <= 0) return set_error(LN3_EINVAL, "groupnorm: need positive G, C, HW");
  if (C % G != 0 || C / G > 256) return set_error(LN3_EINVAL, "groupnorm: bad C / G");
  groupnorm_stats_kernel<<<dim3(G, N), 256, 0, stream>>>(x, gamma, beta, HW, C, G, eps, scale, shift);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "groupnorm launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ single-head attention (mid block)
// q, k, v, out: (N, L, C) fp32 NHWC tokens (ldm AttnBlock, ldm/modules/diffusionmodules/model.py:156-207; 256 tokens x
// 128 channels per plane in the release decoder).  A CTA takes 8 query rows of one image (one warp each) and walks the
// keys in blocks of 32 staged in shared memory (K padded to a 33-float pitch per channel so that "lane = key" reads are
// conflict free): lane j scores key j with a 128-term dot product, the block's max / sum are two warp reductions, and
// the output accumulates p_j V_j with lane = channel (p broadcast through shared memory).  The first version streamed one
// key at a time per warp with five shuffles and two exponentials in a dependent chain: 540 us per launch.
template <int C>
__global__ void __launch_bounds__(256)
attn_single_head_kernel(const float* __restrict__ q, const float* __restrict__ k,
                        const float* __restrict__ v, float* __restrict__ out, int L, float scale) {
  constexpr int PER = C / 32;
  __shared__ float sk[C][33];       // K block, transposed: sk[c][j]
  __shared__ float sv[32][C];       // V block
  __shared__ float sq[8][C];        // the CTA's query rows (pre-scaled)
  __shared__ float sp[8][32];       // probabilities of the current block, per warp
  const int n = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  const bool live = row < L;
  const float* kb = k + static_cast<long long>(n) * L * C;
  const float* vb = v + static_cast<long long>(n) * L * C;
  if (live) {
    const float* qb = q + (static_cast<long long>(n) * L + row) * C;
#pragma unroll
    for (int i = 0; i < PER; ++i) sq[warp][lane + 32 * i] = qb[lane + 32 * i] * scale;
  }
  float o[PER];
#pragma unroll
  for (int i = 0; i < PER; ++i) o[i] = 0.f;
  float m = -INFINITY, l = 0.f;
  for (int j0 = 0; j0 < L; j0 += 32) {
    __syncthreads();   // previous block fully consumed (also orders the sq writes before the first use)
    for (int i = threadIdx.x; i < 32 * C; i += 256) {
      const int jj = i / C, c = i - jj * C;
      const bool ok = j0 + jj < L;
      const float kv = ok ? kb[static_cast<long long>(j0 + jj) * C + c] : 0.f;
      sk[c][jj] = kv;
      sv[jj][c] = ok ? vb[static_cast<long long>(j0 + jj) * C + c] : 0.f;
    }
    __syncthreads();
    if (live) {
      float sc = 0.f;
#pragma unroll 8
      for (int c = 0; c < C; ++c) sc = fmaf(sq[warp][c], sk[c][lane], sc);
      if (j0 + lane >= L) sc = -INFINITY;
      float bm = sc;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, off));
      const float mn = fmaxf(m, bm);
      const float alpha = __expf(m - mn), pj = __expf(sc - mn);
      float bs = pj;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) bs += __shfl_xor_sync(0xffffffffu, bs, off);
      l = l * alpha + bs;
      m = mn;
      sp[warp][lane] = pj;
      __syncwarp();
#pragma unroll
      for (int i = 0; i < PER; ++i) o[i] *= alpha;
#pragma unroll 8
      for (int jj = 0; jj < 32; ++jj) {
        const float pp = sp[warp][jj];
#pragma unroll
        for (int i = 0; i < PER; ++i) o[i] = fmaf(pp, sv[jj][lane + 32 * i], o[i]);
      }
      __syncwarp();
    }
  }
  if (live) {
    float* ob = out + (static_cast<long long>(n) * L + row) * C;
    const float inv = 1.f / l;
#pragma unroll
    for (int i = 0; i < PER; ++i) ob[lane + 32 * i] = o[i] * inv;
  }
}

int attn_single_head(const float* q, const float* k, const float* v, float* out, int N, int L, int C,
                     cudaStream_t stream) {
  if (N <= 0) return LN3_OK;
  if (L <= 0) return set_error(LN3_EINVAL, "attn_single_head: need L > 0");
  const dim3 grid((L + 7) / 8, N);
  const float scale = 1.0f / sqrtf(static_cast<float>(C));
  switch (C) {
    case 32: attn_single_head_kernel<32><<<grid, 256, 0, stream>>>(q, k, v, out, L, scale); break;
    case 64: attn_single_head_kernel<64><<<grid, 256, 0, stream>>>(q, k, v, out, L, scale); break;
    case 128: attn_single_head_kernel<128><<<grid, 256, 0, stream>>>(q, k, v, out, L, scale); break;
    default: return set_error(LN3_EUNSUPPORTED, "attn_single_head: C must be 32, 64 or 128");
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "attn_single_head launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ PatchEmbedTriplane
// Conv2d(3*Cz -> 3*E, k = s = 2, groups = 3) followed by reshape (B, 3E, h, w) -> (B, E, 3, h, w) ->
// tokens (B, 3*h*w, E): tokens[b, n*hw + l, e] = conv_out[b, e*3 + n, l]   (vit_triplane.py:100-106),
// where output channel o = e*3 + n belongs to conv group o / E and reads input channels
// [ (o/E)*Cz, (o/E+1)*Cz ).  Optional SiLU'd bf16 copy (the DiT2 adaLN operand).
__global__ void __launch_bounds__(256)
patch_embed_triplane_kernel(const float* __restrict__ x, const float* __restrict__ w,
                            const float* __restrict__ bias, int B, int Cz, int S, int E,
                            float in_mul, float* __restrict__ tokens, __nv_bfloat16* __restrict__ silu_bf16) {
  __shared__ float xin[3][16][4];  // [group][cz][2x2]
  const int P = S / 2, L = P * P;
  const int tok = blockIdx.x;  // b * 3L + n * L + l
  const int b = tok / (3 * L);
  const int nl = tok - b * 3 * L;
  const int n = nl / L, l = nl - n * L;
  const int pi = l / P, pj = l - pi * P;
  if (threadIdx.x < 3 * Cz * 4) {
    const int g = threadIdx.x / (Cz * 4), r = threadIdx.x % (Cz * 4), c = r >> 2, p = (r >> 1) & 1, qq = r & 1;
    xin[g][c][r & 3] = in_mul * x[((static_cast<long long>(b) * (3 * Cz) + g * Cz + c) * S + 2 * pi + p) * S + 2 * pj + qq];
  }
  __syncthreads();
  const int K = Cz * 4;
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    const int o = e * 3 + n;
    const int g = o / E;
    float acc = bias ? bias[o] : 0.f;
    const float* wr = w + static_cast<long long>(o) * K;
    for (int kk = 0; kk < K; ++kk) acc = fmaf(wr[kk], xin[g][kk >> 2][kk & 3], acc);
    tokens[static_cast<long long>(tok) * E + e] = acc;
    if (silu_bf16) silu_bf16[static_cast<long long>(tok) * E + e] = __float2bfloat16(silu(acc));
  }
}

int patch_embed_triplane(const float* x, const float* w, const float* bias, int B, int Cz, int S, int E,
                         float in_mul, float* tokens, void* silu_bf16, cudaStream_t stream) {
  if (B <= 0) return LN3_OK;
  if (Cz <= 0 || Cz > 16 || (S & 1)) return set_error(LN3_EINVAL, "patch_embed_triplane: need 1 <= Cz <= 16, even S");
  if (S <= 0 || E <= 0) return set_error(LN3_EINVAL, "patch_embed_triplane: need positive S, E");
  const int L = (S / 2) * (S / 2);
  patch_embed_triplane_kernel<<<B * 3 * L, 256, 0, stream>>>(x, w, bias, B, Cz, S, E, in_mul, tokens,
                                                             reinterpret_cast<__nv_bfloat16*>(silu_bf16));
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "patch_embed_triplane launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

}  // namespace ln3
