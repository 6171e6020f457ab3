// Fused tri-plane volumetric renderer for sm_90a (fp32 SIMT, one warp per ray).
//
// Replaces, for the Objaverse rendering preset (nsr/script_util.py:761-797), the whole of
//   nsr/volumetric_rendering/renderer.py:133-307  ImportanceRenderer.forward
//   (get_ray_limits_box, sample_stratified, run_model/_forward_pass, sample_from_planes +
//    F.grid_sample, OSGDecoder, MipRayMarcher2 x2, sample_importance/sample_pdf, unify_samples)
// which in the reference materialises (V,3,M*S,32) sampled features twice per view (~3 GB of HBM
// traffic per 128x128 view).  Here a ray never leaves its warp:
//   phase A (lane = sample): depths, world points, in-box test, 12 bilinear taps (offset+weight)
//   phase B (lane = channel): each tap is one coalesced 128-byte read of the channels-last plane
//            (L1/L2 resident), blended feature rows staged in shared memory
//   phase C (lane = sample): 32->64 softplus ->4 MLP from smem-resident weights, sigmoid / sigma
//   then transmittance scan, importance resampling (cdf scan + binary search), second
//   evaluation, rank-sort merge of the S+S samples and the final compositing scan.
// S = S_importance is 64 (objaverse_tuneray_aug_resolution_64_64_auto) or 96 (..._96_96_auto, the DiT2-L/2
// VAE's preset): a lane holds one sample of each of the S/32 blocks.
// Global reductions of the reference (min/max of valid ray starts, renderer.py:151-155; depth clamp
// range, ray_marcher.py:59-61) are per "group" of consecutive views (= one reference call) and
// handled by a tiny pre-pass and finalize kernel.  Noise is an explicit input (the reference
// draws torch.rand_like / torch.rand: renderer.py:464,530).
#include <float.h>
#include <limits.h>

#include "common.cuh"
#include "ln3_internal.h"

namespace ln3 {

static constexpr int kC = 32;          // plane feature channels
static constexpr int kHid = 64;        // OSG hidden width
static constexpr int kWarpsPerBlock = 16;  // one 512-thread CTA per SM: a 4x4 pixel tile of rays marches in lock-step

__device__ __forceinline__ int float_key(float f) {  // monotone float -> int map
  int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7FFFFFFF;
}
__device__ __forceinline__ float key_float(int k) {
  return __int_as_float(k >= 0 ? k : k ^ 0x7FFFFFFF);
}

// workspace layout: int keys[G][4] = {start_min, start_max, depth_min, depth_max}; then
// float limits[V*M][2]
__global__ void render_init_kernel(int* keys, int G) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g < G) {
    keys[g * 4 + 0] = INT_MAX;
    keys[g * 4 + 1] = INT_MIN;
    keys[g * 4 + 2] = INT_MAX;
    keys[g * 4 + 3] = INT_MIN;
  }
}

// torch.max / torch.min of two tensors propagate a NaN operand; fmaxf / fminf would drop it.  A ray with an
// exactly-zero direction component whose origin lies on that slab's face gets t = 0 * inf = NaN: the reference
// then finds end > start false and treats the ray as invalid (it inherits the group's start range).
__device__ __forceinline__ float max_nan(float a, float b) { return (a != a) ? a : (b != b) ? b : fmaxf(a, b); }
__device__ __forceinline__ float min_nan(float a, float b) { return (a != a) ? a : (b != b) ? b : fminf(a, b); }

// math_utils.get_ray_limits_box (math_utils.py:124-190), IEEE op for op.
__global__ void __launch_bounds__(256)
ray_limits_kernel(const float* __restrict__ ray_o, const float* __restrict__ ray_d, int V, int M,
                  int group_size, float hi, float lo, int* keys, float* limits) {
  const long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= static_cast<long long>(V) * M) return;
  float tmin, tmax;
  bool valid = true;
  {
    const float o0 = ray_o[r * 3 + 0], o1 = ray_o[r * 3 + 1], o2 = ray_o[r * 3 + 2];
    const float i0 = __fdiv_rn(1.f, ray_d[r * 3 + 0]), i1 = __fdiv_rn(1.f, ray_d[r * 3 + 1]),
                i2 = __fdiv_rn(1.f, ray_d[r * 3 + 2]);
    const bool n0 = i0 < 0, n1 = i1 < 0, n2 = i2 < 0;
    tmin = __fmul_rn(__fsub_rn(n0 ? hi : lo, o0), i0);
    tmax = __fmul_rn(__fsub_rn(n0 ? lo : hi, o0), i0);
    const float tymin = __fmul_rn(__fsub_rn(n1 ? hi : lo, o1), i1);
    const float tymax = __fmul_rn(__fsub_rn(n1 ? lo : hi, o1), i1);
    if (tmin > tymax || tymin > tmax) valid = false;
    tmin = max_nan(tmin, tymin);
    tmax = min_nan(tmax, tymax);
    const float tzmin = __fmul_rn(__fsub_rn(n2 ? hi : lo, o2), i2);
    const float tzmax = __fmul_rn(__fsub_rn(n2 ? lo : hi, o2), i2);
    if (tmin > tzmax || tzmin > tmax) valid = false;
    tmin = max_nan(tmin, tzmin);
    tmax = min_nan(tmax, tzmax);
  }
  if (!valid) {
    tmin = -1.f;
    tmax = -2.f;
  }
  limits[r * 2 + 0] = tmin;
  limits[r * 2 + 1] = tmax;
  if (tmax > tmin) {  // is_ray_valid = ray_end > ray_start (renderer.py:149)
    const int g = static_cast<int>(r / M) / group_size;
    const int k = float_key(tmin);
    atomicMin(&keys[g * 4 + 0], k);
    atomicMax(&keys[g * 4 + 1], k);
  }
}

struct RenderParams {
  const float* planes;  // [n_obj][3][H][W][C] channels-last
  const int* view_obj;  // [V] or null (view v -> object v / views_per_obj)
  const float* ray_o;
  const float* ray_d;
  const float* noise_c;
  const float* noise_f;
  const float* w1;
  const float* b1;
  const float* w2;
  const float* b2;
  float* rgb;
  float* depth;
  float* wsum;
  int* keys;
  const float* limits;
  int V, M, H, W, group_size, views_per_obj;
  int image_w;        // > 0: ray m of a view is pixel (m % image_w, m / image_w) -> 4x4 pixel-tile schedule
  float coord_scale;  // 2 / box_warp (rounded to fp32 like the reference's scalar multiply)
  float bbox_min, bbox_max;
  int white_back;
  int mlp_tf32;   // 1: OSG MLP on the tensor cores (TF32 operands, fp32 accumulate); 0: exact fp32 SIMT
  int no_filter;  // 1: raw decoder output for every point (ImportanceRenderer._run_model), no in-box filter
  // optional debug outputs (tests): in-box masks / importance indices / sort permutation, S samples per pass
  unsigned char* dbg_inbox;  // [V*M][2S]
  int* dbg_inds;             // [V*M][S]
  int* dbg_order;            // [V*M][2S]
  float* dbg_zfine;          // [V*M][S]
};

// Per-warp buffers of one 32-sample model evaluation (eval_batch).
struct GatherSmem {
  int tap_off[32][12];
  float tap_w[32][12];
  float feat[32][36];   // stride 36: A-fragment reads (row g, col t) hit 32 distinct banks; rows 16-B aligned
};

template <int S>
struct WarpSmem {
  GatherSmem g;
  float cdf[S];
  float bins[S];
  float sz[2 * S];   // merged samples: depth, sigma, r, g, b
  float ss[2 * S];
  float sr[2 * S];
  float sg[2 * S];
  float sb[2 * S];
};
static_assert(2 * 96 <= 32 * 36, "the unify stage stages 2S depths in GatherSmem::feat");

struct OsgSmem {
  float w1[kHid][kC];  // pre-scaled by 1/sqrt(32)
  float b1[kHid];
  float w2[4][kHid];   // pre-scaled by 1/8
  float b2[4];
  // TF32 tensor-core path: the same weights as mma.m16n8k8 B fragments (tf32-rounded), one float2 per lane
  float2 w1f[8][4][32];  // [n-tile of 8 hidden units][k-step of 8 features][lane] = (b0, b1)
  float2 w2f[8][32];     // [k-step = layer-1 n-tile][lane]; hidden units in layer-1 accumulator order
};

// 191,760 B at S = 64 and 216,336 B at S = 96: both fit the 232,448 B opt-in limit with 16 warps per CTA.
template <int S>
struct BlockSmem {
  OsgSmem osg;
  WarpSmem<S> warp[kWarpsPerBlock];
};
static_assert(sizeof(BlockSmem<96>) <= 232448, "S = 96 must fit one 16-warp CTA per SM");

// Fill the weight copies of a block (fp32 rows for the SIMT path, tf32 B fragments for the mma path).
__device__ __forceinline__ void load_osg_weights(OsgSmem& bs, const float* w1, const float* b1, const float* w2,
                                                 const float* b2) {
  for (int i = threadIdx.x; i < kHid * kC; i += blockDim.x)
    (&bs.w1[0][0])[i] = __fmul_rn(w1[i], 0.17677669529663687f);  // weight_gain = 1/sqrt(32)
  for (int i = threadIdx.x; i < 4 * kHid; i += blockDim.x) (&bs.w2[0][0])[i] = __fmul_rn(w2[i], 0.125f);
  if (threadIdx.x < kHid) bs.b1[threadIdx.x] = b1[threadIdx.x];
  if (threadIdx.x < 4) bs.b2[threadIdx.x] = b2[threadIdx.x];
  for (int i = threadIdx.x; i < 8 * 4 * 32; i += blockDim.x) {
    const int ln = i & 31, ks = (i >> 5) & 3, nt = i >> 7, g = ln >> 2, t = ln & 3;
    const float* row = w1 + (8 * nt + g) * kC + 8 * ks;  // B[k][n] = W1[n][k]
    bs.w1f[nt][ks][ln] = make_float2(__uint_as_float(to_tf32(__fmul_rn(row[t], 0.17677669529663687f))),
                                     __uint_as_float(to_tf32(__fmul_rn(row[t + 4], 0.17677669529663687f))));
  }
  for (int i = threadIdx.x; i < 8 * 32; i += blockDim.x) {
    const int ln = i & 31, nt = i >> 5, g = ln >> 2, t = ln & 3;
    // layer-2 k index t <-> hidden unit 8nt + 2t, k index t+4 <-> hidden unit 8nt + 2t + 1 (the order in
    // which a lane holds the layer-1 accumulators), outputs n = g < 4 (sigma, r, g, b), zero padding above
    const float v0 = g < 4 ? __fmul_rn(w2[g * kHid + 8 * nt + 2 * t], 0.125f) : 0.f;
    const float v1 = g < 4 ? __fmul_rn(w2[g * kHid + 8 * nt + 2 * t + 1], 0.125f) : 0.f;
    bs.w2f[nt][ln] = make_float2(__uint_as_float(to_tf32(v0)), __uint_as_float(to_tf32(v1)));
  }
}

__device__ __forceinline__ float softplus_t(float x) {  // torch.nn.Softplus(beta=1, threshold=20)
  return x > 20.f ? x : log1pf(expf(x));
}
// softplus(x) = max(x, 0) + ln(1 + e^-|x|) with MUFU ex2 / lg2 (abs error ~1e-7: 1 + e^-|x| is in
// [1, 2] where lg2.approx is accurate to 2^-22); used for the 64 hidden units of every sample.
__device__ __forceinline__ float softplus_fast(float x) {
  const float e = fast_exp2(-fabsf(x) * 1.4426950408889634f);
  float l;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(l) : "f"(1.f + e));
  return fmaf(l, 0.6931471805599453f, fmaxf(x, 0.f));
}

__device__ __forceinline__ float warp_incl_prod(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v *= t;
  }
  return v;
}
__device__ __forceinline__ float warp_incl_sum(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// grid_sample(bilinear, zeros, align_corners=False) taps of one plane for coordinate (gx -> W, gy -> H)
__device__ __forceinline__ void plane_taps(float gx, float gy, int H, int W, int plane_base,
                                           int* off, float* w) {
  const float ix = ((gx + 1.f) * W - 1.f) / 2.f;
  const float iy = ((gy + 1.f) * H - 1.f) / 2.f;
  const float x0f = floorf(ix), y0f = floorf(iy);
  const float x1f = x0f + 1.f, y1f = y0f + 1.f;
  const float wx1 = ix - x0f, wx0 = x1f - ix, wy1 = iy - y0f, wy0 = y1f - iy;
  // floorf of NaN / huge values: clamp before the int conversion
  const int x0 = static_cast<int>(fminf(fmaxf(x0f, -2.f), static_cast<float>(W + 1)));
  const int y0 = static_cast<int>(fminf(fmaxf(y0f, -2.f), static_cast<float>(H + 1)));
  const int x1 = x0 + 1, y1 = y0 + 1;
  const bool vx0 = x0 >= 0 && x0 < W, vx1 = x1 >= 0 && x1 < W;
  const bool vy0 = y0 >= 0 && y0 < H, vy1 = y1 >= 0 && y1 < H;
  const bool fin = (ix == ix) && (iy == iy);
  off[0] = (vx0 && vy0) ? plane_base + (y0 * W + x0) * kC : plane_base;
  off[1] = (vx1 && vy0) ? plane_base + (y0 * W + x1) * kC : plane_base;
  off[2] = (vx0 && vy1) ? plane_base + (y1 * W + x0) * kC : plane_base;
  off[3] = (vx1 && vy1) ? plane_base + (y1 * W + x1) * kC : plane_base;
  w[0] = (fin && vx0 && vy0) ? wx0 * wy0 : 0.f;
  w[1] = (fin && vx1 && vy0) ? wx1 * wy0 : 0.f;
  w[2] = (fin && vx0 && vy1) ? wx0 * wy1 : 0.f;
  w[3] = (fin && vx1 && vy1) ? wx1 * wy1 : 0.f;
}

// Evaluate the implicit model on 32 samples (one per lane): returns sigma / rgb for this lane's
// sample with the reference's out-of-box filter applied.
// Not inlined: four copies of this body put the kernel at 164 KB of SASS and "no instruction" (i-cache
// miss) became the top stall once the MLP moved to the tensor cores; the precision is a template
// parameter so that only one MLP body is in the instruction stream.
template <bool TF32>
__device__ __noinline__ void eval_batch(const RenderParams& p, const OsgSmem& bs, GatherSmem& ws,
                                           const float* __restrict__ planes_obj, int lane,
                                           float px, float py, float pz, bool& inbox, float& sigma,
                                           float& cr, float& cg, float& cb) {
  inbox = (px >= p.bbox_min && px <= p.bbox_max) && (py >= p.bbox_min && py <= p.bbox_max) &&
          (pz >= p.bbox_min && pz <= p.bbox_max);
  // The out-of-box filter (renderer.py:391-405) overwrites the network output of every sample outside the box, so
  // a batch with no sample inside needs neither the gather nor the MLP: rays that miss the volume (their samples
  // are spread over the group's global [min start, max end] range, all outside) cost only the bookkeeping.
  if (!p.no_filter && !__any_sync(0xffffffffu, inbox)) {
    sigma = -FLT_MAX / 3.f;
    cr = cg = cb = 0.f;
    return;
  }
  // phase A: taps for this lane's sample
  {
    const float sx = p.coord_scale * px, sy = p.coord_scale * py, sz = p.coord_scale * pz;
    const int HWC = p.H * p.W * kC;
    plane_taps(sx, sy, p.H, p.W, 0, &ws.tap_off[lane][0], &ws.tap_w[lane][0]);        // (x, y)
    plane_taps(sy, sz, p.H, p.W, HWC, &ws.tap_off[lane][4], &ws.tap_w[lane][4]);      // (y, z)
    plane_taps(sz, sx, p.H, p.W, 2 * HWC, &ws.tap_off[lane][8], &ws.tap_w[lane][8]);  // (z, x)
  }
  __syncwarp();
  // phase B: 8 lanes x float4 cover one 128-byte texel; the 4 lane groups work on 4 samples at once,
  // so one LDG.128 warp instruction fetches one tap for 4 samples (4 coalesced lines).
  {
    const int grp = lane >> 3, c4 = (lane & 7) * 4;
    const float* pl_base = planes_obj + c4;
#pragma unroll 2
    for (int s0 = 0; s0 < 32; s0 += 4) {
      const int sidx = s0 + grp;
      float4 f[3];
#pragma unroll
      for (int pl = 0; pl < 3; ++pl) {
        const int4 o = *reinterpret_cast<const int4*>(&ws.tap_off[sidx][pl * 4]);
        const float4 w = *reinterpret_cast<const float4*>(&ws.tap_w[sidx][pl * 4]);
        const float4 v0 = __ldg(reinterpret_cast<const float4*>(pl_base + o.x));
        const float4 v1 = __ldg(reinterpret_cast<const float4*>(pl_base + o.y));
        const float4 v2 = __ldg(reinterpret_cast<const float4*>(pl_base + o.z));
        const float4 v3 = __ldg(reinterpret_cast<const float4*>(pl_base + o.w));
        f[pl].x = ((v0.x * w.x + v1.x * w.y) + v2.x * w.z) + v3.x * w.w;
        f[pl].y = ((v0.y * w.x + v1.y * w.y) + v2.y * w.z) + v3.y * w.w;
        f[pl].z = ((v0.z * w.x + v1.z * w.y) + v2.z * w.z) + v3.z * w.w;
        f[pl].w = ((v0.w * w.x + v1.w * w.y) + v2.w * w.z) + v3.w * w.w;
      }
      // sampled_features.mean(1).  Exact path: IEEE division by 3 as torch's CPU mean (the oracle / goldens).
      // TF32 path: sum * (1/3) as torch's CUDA mean kernel computes it (MeanOps multiplies by the fp32 factor
      // 1/N) -- a last-ulp difference that the TF32 rounding of the MLP operand swallows; four IEEE divisions per
      // lane here were ~10 % of the kernel's stall samples.
      if constexpr (TF32) {
        constexpr float kThird = 1.0f / 3.0f;
        ws.feat[sidx][c4 + 0] = ((f[0].x + f[1].x) + f[2].x) * kThird;
        ws.feat[sidx][c4 + 1] = ((f[0].y + f[1].y) + f[2].y) * kThird;
        ws.feat[sidx][c4 + 2] = ((f[0].z + f[1].z) + f[2].z) * kThird;
        ws.feat[sidx][c4 + 3] = ((f[0].w + f[1].w) + f[2].w) * kThird;
      } else {
        ws.feat[sidx][c4 + 0] = ((f[0].x + f[1].x) + f[2].x) / 3.f;
        ws.feat[sidx][c4 + 1] = ((f[0].y + f[1].y) + f[2].y) / 3.f;
        ws.feat[sidx][c4 + 2] = ((f[0].z + f[1].z) + f[2].z) / 3.f;
        ws.feat[sidx][c4 + 3] = ((f[0].w + f[1].w) + f[2].w) / 3.f;
      }
    }
  }
  __syncwarp();
  float y0, y1, y2, y3;
  if constexpr (TF32) {
    // phase C on the tensor cores: [32 samples x 32] x [32 x 64] -> softplus -> [32 x 64] x [64 x 8(4 used)]
    // as mma.m16n8k8 TF32 (fp32 accumulate): 64 + 16 MMAs instead of 2304 FFMA + 768 LDS per lane.
    const int g = lane >> 2, t = lane & 3;
    uint32_t a[2][4][4];  // [m-tile][k-step][fragment]
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        a[mt][ks][0] = to_tf32(ws.feat[16 * mt + g][8 * ks + t]);
        a[mt][ks][1] = to_tf32(ws.feat[16 * mt + g + 8][8 * ks + t]);
        a[mt][ks][2] = to_tf32(ws.feat[16 * mt + g][8 * ks + t + 4]);
        a[mt][ks][3] = to_tf32(ws.feat[16 * mt + g + 8][8 * ks + t + 4]);
      }
    float o[2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      o[mt][0] = o[mt][2] = t < 2 ? bs.b2[2 * t] : 0.f;
      o[mt][1] = o[mt][3] = t < 2 ? bs.b2[2 * t + 1] : 0.f;
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      float h[2][4];
      const float bb0 = bs.b1[8 * nt + 2 * t], bb1 = bs.b1[8 * nt + 2 * t + 1];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) h[mt][0] = h[mt][2] = bb0, h[mt][1] = h[mt][3] = bb1;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const float2 b = bs.w1f[nt][ks][lane];
        mma_tf32(h[0], a[0][ks], __float_as_uint(b.x), __float_as_uint(b.y));
        mma_tf32(h[1], a[1][ks], __float_as_uint(b.x), __float_as_uint(b.y));
      }
      // the layer-1 accumulator fragment IS the layer-2 A fragment for k-step nt (hidden units permuted
      // consistently in w2f): a0 = d0, a1 = d2, a2 = d1, a3 = d3
      const float2 b2f = bs.w2f[nt][lane];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const uint32_t a2[4] = {to_tf32(softplus_fast(h[mt][0])), to_tf32(softplus_fast(h[mt][2])),
                                to_tf32(softplus_fast(h[mt][1])), to_tf32(softplus_fast(h[mt][3]))};
        mma_tf32(o[mt], a2, __float_as_uint(b2f.x), __float_as_uint(b2f.y));
      }
    }
    // back to lane = sample through the (now idle) feature buffer: y[sample][4]
    __syncwarp();
    float* ybuf = &ws.feat[0][0];
    if (t < 2) {
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        *reinterpret_cast<float2*>(ybuf + (16 * mt + g) * 4 + 2 * t) = make_float2(o[mt][0], o[mt][1]);
        *reinterpret_cast<float2*>(ybuf + (16 * mt + g + 8) * 4 + 2 * t) = make_float2(o[mt][2], o[mt][3]);
      }
    }
    __syncwarp();
    const float4 yv = *reinterpret_cast<const float4*>(ybuf + lane * 4);
    y0 = yv.x, y1 = yv.y, y2 = yv.z, y3 = yv.w;
  } else {
  // phase C (exact fp32 SIMT): lane = sample; 32 -> 64 (softplus) -> 4
  float x[kC];
#pragma unroll
  for (int c = 0; c < kC; c += 4) {
    const float4 v = *reinterpret_cast<const float4*>(&ws.feat[lane][c]);
    x[c] = v.x, x[c + 1] = v.y, x[c + 2] = v.z, x[c + 3] = v.w;
  }
  y0 = bs.b2[0], y1 = bs.b2[1], y2 = bs.b2[2], y3 = bs.b2[3];
#pragma unroll 4
  for (int j = 0; j < kHid; ++j) {
    float acc = bs.b1[j];
#pragma unroll
    for (int c = 0; c < kC; c += 4) {
      const float4 w = *reinterpret_cast<const float4*>(&bs.w1[j][c]);
      acc = fmaf(x[c], w.x, acc);
      acc = fmaf(x[c + 1], w.y, acc);
      acc = fmaf(x[c + 2], w.z, acc);
      acc = fmaf(x[c + 3], w.w, acc);
    }
    const float h = softplus_fast(acc);
    y0 = fmaf(h, bs.w2[0][j], y0);
    y1 = fmaf(h, bs.w2[1][j], y1);
    y2 = fmaf(h, bs.w2[2][j], y2);
    y3 = fmaf(h, bs.w2[3][j], y3);
  }
  }
  __syncwarp();
  if (inbox || p.no_filter) {
    sigma = y0;
    cr = 1.f / (1.f + expf(-y1)) * 1.002f - 0.001f;
    cg = 1.f / (1.f + expf(-y2)) * 1.002f - 0.001f;
    cb = 1.f / (1.f + expf(-y3)) * 1.002f - 0.001f;
  } else {  // renderer.py:391-405: rgb 0, sigma = nan_to_num(-inf) / 3
    sigma = -FLT_MAX / 3.f;
    cr = cg = cb = 0.f;
  }
}

// Schedule: one CTA (16 warps = 16 rays) per SM walks work items; an item is a 4x4 PIXEL TILE of one view when the
// rays of a view form an image (image_w > 0), else 16 consecutive rays.  Neighbouring pixels' rays pass through
// neighbouring texels at every depth index, and the 16 warps of a tile start together, so a texel line fetched by
// one warp is usually an L1 hit for its neighbours (ncu: L1 hit rate 34 % -> 61.5 %, L2->L1 traffic -40 %): the
// 64 KB of L1 left beside the shared-memory carve-out only helps rays that are co-resident in space AND time.
// There is no barrier per item: rays that miss the volume skip the gather and the MLP (eval_batch) and their
// warps simply move on to the next tile.
template <bool TF32, int NB>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, 1)
render_rays_kernel(const RenderParams p) {
  constexpr int S = 32 * NB;  // coarse == importance sample count
  extern __shared__ uint8_t smem_raw[];
  BlockSmem<S>& bs = *reinterpret_cast<BlockSmem<S>*>(smem_raw);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  load_osg_weights(bs.osg, p.w1, p.b1, p.w2, p.b2);
  __syncthreads();
  WarpSmem<S>& ws = bs.warp[warp];

  const long long total = static_cast<long long>(p.V) * p.M;
  const int tiles_x = p.image_w > 0 ? p.image_w / 4 : 0;
  const long long n_items = (total + kWarpsPerBlock - 1) / kWarpsPerBlock;   // tiles cover a view exactly (host check)
  const int items_per_view = p.M / kWarpsPerBlock;
  for (long long item = blockIdx.x; item < n_items; item += gridDim.x) {
    long long ray;
    if (tiles_x > 0) {
      const int v = static_cast<int>(item / items_per_view);
      const int tt = static_cast<int>(item - static_cast<long long>(v) * items_per_view);
      const int ty = tt / tiles_x, tx = tt - ty * tiles_x;
      ray = static_cast<long long>(v) * p.M + (ty * 4 + (warp >> 2)) * p.image_w + tx * 4 + (warp & 3);
    } else {
      ray = item * kWarpsPerBlock + warp;
    }
    if (ray >= total) continue;   // linear schedule, last item only
    const int view = static_cast<int>(ray / p.M);
    const int grp = view / p.group_size;
    const int obj = p.view_obj ? p.view_obj[view] : view / p.views_per_obj;
    const float* planes_obj = p.planes + static_cast<long long>(obj) * 3 * p.H * p.W * kC;
    const float ox = p.ray_o[ray * 3], oy = p.ray_o[ray * 3 + 1], oz = p.ray_o[ray * 3 + 2];
    const float dx = p.ray_d[ray * 3], dy = p.ray_d[ray * 3 + 1], dz = p.ray_d[ray * 3 + 2];
    float start = p.limits[ray * 2], end = p.limits[ray * 2 + 1];
    if (!(end > start)) {  // invalid ray: global min / max of the valid starts (renderer.py:151-155)
      const int kmin = p.keys[grp * 4 + 0];
      if (kmin != INT_MAX) {
        start = key_float(kmin);
        end = key_float(p.keys[grp * 4 + 1]);
      }
    }
    // ---- stratified coarse depths (renderer.py:455-466, math_utils.linspace)
    const float span = __fsub_rn(end, start);
    const float delta = __fdiv_rn(span, static_cast<float>(S - 1));
    float zc[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const int j = b * 32 + lane;
      const float step = __fdiv_rn(static_cast<float>(j), static_cast<float>(S - 1));
      const float base = __fadd_rn(start, __fmul_rn(step, span));
      zc[b] = __fadd_rn(base, __fmul_rn(p.noise_c[ray * S + j], delta));
    }
    float sc[NB], rc[NB], gc[NB], bc[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const float px = __fadd_rn(ox, __fmul_rn(zc[b], dx));
      const float py = __fadd_rn(oy, __fmul_rn(zc[b], dy));
      const float pz = __fadd_rn(oz, __fmul_rn(zc[b], dz));
      bool inbox;
      eval_batch<TF32>(p, bs.osg, ws.g, planes_obj, lane, px, py, pz, inbox, sc[b], rc[b], gc[b], bc[b]);
      if (p.dbg_inbox) p.dbg_inbox[ray * (2 * S) + b * 32 + lane] = inbox;
    }
    // ---- coarse ray march -> weights (ray_marcher.py:26-47); interval i = samples (i, i+1)
    float wgt[NB];  // weight of interval b*32+lane (interval S-1 does not exist)
    {
      float alpha[NB], om[NB];
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        float zn = __shfl_down_sync(0xffffffffu, zc[b], 1);
        float sn = __shfl_down_sync(0xffffffffu, sc[b], 1);
        if (b < NB - 1) {
          const float z32 = __shfl_sync(0xffffffffu, zc[b + 1], 0), s32 = __shfl_sync(0xffffffffu, sc[b + 1], 0);
          if (lane == 31) { zn = z32; sn = s32; }
        }
        const bool has = (b < NB - 1) || (lane < 31);
        const float dlt = zn - zc[b];
        const float smid = softplus_t((sc[b] + sn) / 2.f - 1.f);
        alpha[b] = has ? 1.f - expf(-(smid * dlt)) : 0.f;
        om[b] = has ? (1.f - alpha[b]) + 1e-10f : 1.f;
      }
      // transmittance: inclusive product per block, chained across blocks by the previous blocks' total
      float inc[NB], tot[NB];
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        inc[b] = warp_incl_prod(om[b], lane);
        if (b > 0) inc[b] *= tot[b - 1];
        if (b < NB - 1) tot[b] = __shfl_sync(0xffffffffu, inc[b], 31);
      }
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        float ex = __shfl_up_sync(0xffffffffu, inc[b], 1);
        if (lane == 0) ex = b > 0 ? tot[b - 1] : 1.f;
        wgt[b] = alpha[b] * ex;
      }
    }
    // ---- importance sampling (renderer.py:479-552)
    float zf[NB];
    {
      // smoothed[i] = (max(w[i-1], w[i]) + max(w[i], w[i+1])) / 2 + 0.01 for i = 0..S-2 (w[-1] = w[S-1] = -inf)
      float sm[NB];
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        float prev = __shfl_up_sync(0xffffffffu, wgt[b], 1);
        float next = __shfl_down_sync(0xffffffffu, wgt[b], 1);
        if (b < NB - 1) {
          const float w32 = __shfl_sync(0xffffffffu, wgt[b + 1], 0);
          if (lane == 31) next = w32;
        }
        if (b == 0) {
          if (lane == 0) prev = -INFINITY;
        } else {
          const float w31 = __shfl_sync(0xffffffffu, wgt[b - 1], 31);
          if (lane == 0) prev = w31;
        }
        if (b == NB - 1 && lane >= 30) next = -INFINITY;  // interval S-2's right neighbour is the pad
        sm[b] = (fmaxf(prev, wgt[b]) + fmaxf(wgt[b], next)) / 2.f + 0.01f;
      }
      // pdf over smoothed[1..S-3] (S-3 weights), bins = mid-points of the S coarse depths (S-1)
      float wv[NB];
#pragma unroll
      for (int b = 0; b < NB; ++b) {  // index b*32+lane in 1..S-3
        const bool in = (b > 0 || lane >= 1) && (b < NB - 1 || lane <= 29);
        wv[b] = in ? sm[b] + 1e-5f : 0.f;
      }
      float tot = warp_sum_f(wv[0]);
#pragma unroll
      for (int b = 1; b < NB; ++b) tot += warp_sum_f(wv[b]);
      float pdf[NB];
#pragma unroll
      for (int b = 0; b < NB; ++b) pdf[b] = wv[b] / tot;
      float c[NB];
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        c[b] = warp_incl_sum(pdf[b], lane);
        if (b > 0) c[b] += __shfl_sync(0xffffffffu, c[b - 1], 31);
      }
      // cdf[0] = 0, cdf[k] = sum of pdf over smoothed[1..k], k = 1..S-3  (S-2 entries)
      ws.cdf[lane] = (lane == 0) ? 0.f : c[0];
#pragma unroll
      for (int b = 1; b < NB; ++b)
        if (b < NB - 1 || lane <= 29) ws.cdf[b * 32 + lane] = c[b];
      // bins (z_mid) 0..S-2
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        float zn = __shfl_down_sync(0xffffffffu, zc[b], 1);
        if (b < NB - 1) {
          const float z32 = __shfl_sync(0xffffffffu, zc[b + 1], 0);
          if (lane == 31) zn = z32;
        }
        if (b < NB - 1 || lane < 31) ws.bins[b * 32 + lane] = 0.5f * (zc[b] + zn);
      }
      __syncwarp();
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        const float u = p.noise_f[ray * S + b * 32 + lane];
        // searchsorted(cdf[0..S-3], u, right=True): first index with cdf > u
        int lo = 0, hi = S - 2;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (ws.cdf[mid] <= u) lo = mid + 1; else hi = mid;
        }
        const int below = max(lo - 1, 0), above = min(lo, S - 3);
        const float cb0 = ws.cdf[below], cb1 = ws.cdf[above];
        const float bb0 = ws.bins[below], bb1 = ws.bins[above];
        float den = cb1 - cb0;
        if (den < 1e-5f) den = 1.f;
        zf[b] = bb0 + (u - cb0) / den * (bb1 - bb0);
        if (p.dbg_inds) p.dbg_inds[ray * S + b * 32 + lane] = lo;
        if (p.dbg_zfine) p.dbg_zfine[ray * S + b * 32 + lane] = zf[b];
      }
      __syncwarp();
    }
    // ---- fine pass
    float sf[NB], rf[NB], gf[NB], bf[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) {
      const float px = __fadd_rn(ox, __fmul_rn(zf[b], dx));
      const float py = __fadd_rn(oy, __fmul_rn(zf[b], dy));
      const float pz = __fadd_rn(oz, __fmul_rn(zf[b], dz));
      bool inbox;
      eval_batch<TF32>(p, bs.osg, ws.g, planes_obj, lane, px, py, pz, inbox, sf[b], rf[b], gf[b], bf[b]);
      if (p.dbg_inbox) p.dbg_inbox[ray * (2 * S) + S + b * 32 + lane] = inbox;
    }
    // ---- unify: stable rank sort of the 2S (coarse ++ fine) depths (renderer.py:422-435)
    constexpr int Q = 2 * NB;  // 32-sample blocks of the merged ray
    {
      float* stage = &ws.g.feat[0][0];  // 2S unsorted depths
#pragma unroll
      for (int b = 0; b < NB; ++b) {
        stage[b * 32 + lane] = zc[b];
        stage[S + b * 32 + lane] = zf[b];
      }
      __syncwarp();
      int rank[Q];
      float mine[Q];
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        rank[q] = 0;
        mine[q] = q < NB ? zc[q % NB] : zf[q % NB];
      }
      // rank = #(z_k < mine) + #(z_k == mine with k < my index).  My index is q*32 + lane, so against a
      // whole 32-block kb the tie-break is a compile-time choice (kb < q: "<=", kb > q: "<") and only the
      // own block needs the lane-dependent form; candidates come four per LDS.128.
#pragma unroll
      for (int kb = 0; kb < Q; ++kb) {
#pragma unroll 2
        for (int kk = 0; kk < 32; kk += 4) {
          const float4 z4 = *reinterpret_cast<const float4*>(stage + kb * 32 + kk);
          const float zs[4] = {z4.x, z4.y, z4.z, z4.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float zk = zs[e];
#pragma unroll
            for (int q = 0; q < Q; ++q) {
              if (kb < q) rank[q] += zk <= mine[q];
              else if (kb > q) rank[q] += zk < mine[q];
              else rank[q] += (zk < mine[q]) || (zk == mine[q] && kk + e < lane);
            }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        const int b = q % NB;
        ws.sz[rank[q]] = mine[q];
        ws.ss[rank[q]] = q < NB ? sc[b] : sf[b];
        ws.sr[rank[q]] = q < NB ? rc[b] : rf[b];
        ws.sg[rank[q]] = q < NB ? gc[b] : gf[b];
        ws.sb[rank[q]] = q < NB ? bc[b] : bf[b];
        if (p.dbg_order) p.dbg_order[ray * (2 * S) + rank[q]] = q * 32 + lane;
      }
      __syncwarp();
    }
    // ---- final march over 2S-1 intervals (ray_marcher.py:26-68)
    float acc_r = 0.f, acc_g = 0.f, acc_b = 0.f, acc_d = 0.f, acc_w = 0.f;
    {
      float carry = 1.f;
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        const int i = q * 32 + lane;
        const bool has = i < 2 * S - 1;
        const int i1 = has ? i + 1 : i;
        const float z0 = ws.sz[i], z1 = ws.sz[i1];
        const float smid = softplus_t((ws.ss[i] + ws.ss[i1]) / 2.f - 1.f);
        const float alpha = has ? 1.f - expf(-(smid * (z1 - z0))) : 0.f;
        const float om = has ? (1.f - alpha) + 1e-10f : 1.f;
        const float inc = warp_incl_prod(om, lane) * carry;
        float ex = __shfl_up_sync(0xffffffffu, inc, 1);
        if (lane == 0) ex = carry;
        carry = __shfl_sync(0xffffffffu, inc, 31);
        const float w = alpha * ex;
        acc_w += w;
        acc_r += w * ((ws.sr[i] + ws.sr[i1]) / 2.f);
        acc_g += w * ((ws.sg[i] + ws.sg[i1]) / 2.f);
        acc_b += w * ((ws.sb[i] + ws.sb[i1]) / 2.f);
        acc_d += w * ((z0 + z1) / 2.f);
      }
    }
    acc_w = warp_sum_f(acc_w);
    acc_r = warp_sum_f(acc_r);
    acc_g = warp_sum_f(acc_g);
    acc_b = warp_sum_f(acc_b);
    acc_d = warp_sum_f(acc_d);
    if (lane == 0) {
      const int m = static_cast<int>(ray - static_cast<long long>(view) * p.M);
      float r = acc_r, g = acc_g, b = acc_b;
      if (p.white_back) {
        r = r + 1.f - acc_w;
        g = g + 1.f - acc_w;
        b = b + 1.f - acc_w;
      }
      float* o = p.rgb + static_cast<long long>(view) * 3 * p.M;
      o[m] = r * 2.f - 1.f;
      o[p.M + m] = g * 2.f - 1.f;
      o[2 * p.M + m] = b * 2.f - 1.f;
      p.depth[ray] = acc_d;  // clamped by render_finalize_kernel
      p.wsum[ray] = acc_w;
      atomicMin(&p.keys[grp * 4 + 2], float_key(ws.sz[0]));
      atomicMax(&p.keys[grp * 4 + 3], float_key(ws.sz[2 * S - 1]));
    }
    __syncwarp();
  }
}

// composite_depth = clamp(nan_to_num(depth, inf), min(depths), max(depths))  (ray_marcher.py:58-61)
__global__ void render_finalize_kernel(float* depth, const int* keys, int V, int M, int group_size) {
  const long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= static_cast<long long>(V) * M) return;
  const int g = static_cast<int>(r / M) / group_size;
  const float lo = key_float(keys[g * 4 + 2]), hi = key_float(keys[g * 4 + 3]);
  float d = depth[r];
  if (d != d) d = INFINITY;
  if (isinf(d)) d = d > 0 ? FLT_MAX : -FLT_MAX;
  depth[r] = fminf(fmaxf(d, lo), hi);
}

// 2-D tile schedule when a view is an image whose width and height are multiples of 4, else 0 (linear order)
int render_tile_width(int M, int image_w) {
  return (image_w > 0 && image_w % 4 == 0 && M % image_w == 0 && (M / image_w) % 4 == 0) ? image_w : 0;
}

size_t render_workspace_bytes(int V, int M, int group_size) {
  const int G = (V + group_size - 1) / group_size;
  return static_cast<size_t>(G) * 4 * sizeof(int) + static_cast<size_t>(V) * M * 2 * sizeof(float) + 256;
}

// One instantiation per (MLP precision, samples per ray): the dynamic shared memory is opted in per kernel.
template <int NB>
static int launch_render_rays(const RenderParams& p, long long blocks, cudaStream_t stream) {
  constexpr size_t smem = sizeof(BlockSmem<32 * NB>);
  static DeviceOnce once;
  if (int rc = once.run([] {
        cudaError_t e = cudaFuncSetAttribute(render_rays_kernel<false, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             static_cast<int>(smem));
        if (e == cudaSuccess)
          e = cudaFuncSetAttribute(render_rays_kernel<true, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(smem));
        return e == cudaSuccess ? LN3_OK : set_error(LN3_ECUDA, "render: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      }))
    return rc;
  if (p.mlp_tf32)
    render_rays_kernel<true, NB><<<static_cast<unsigned>(blocks), kWarpsPerBlock * 32, smem, stream>>>(p);
  else
    render_rays_kernel<false, NB><<<static_cast<unsigned>(blocks), kWarpsPerBlock * 32, smem, stream>>>(p);
  return LN3_OK;
}

int render_views(const ln3_render_args* a, cudaStream_t stream) {
  if (a->V <= 0 || a->M <= 0) return LN3_OK;
  if (a->C != kC || a->S != a->S_importance || (a->S != 64 && a->S != 96))
    return set_error(LN3_EUNSUPPORTED, "render: needs 32 plane channels and 64+64 or 96+96 samples per ray");
  if (a->decoder_output_dim != 3 || a->hidden_dim != kHid)
    return set_error(LN3_EUNSUPPORTED, "render: OSG decoder must be 32 -> 64 -> 1+3");
  if (a->group_size <= 0) return set_error(LN3_EINVAL, "render: group_size must be > 0");
  if (!a->planes_cl || !a->ray_o || !a->ray_d || !a->noise_coarse || !a->noise_fine || !a->rgb ||
      !a->depth || !a->weights || !a->workspace)
    return set_error(LN3_EINVAL, "render: null pointer");
  if (a->workspace_bytes < render_workspace_bytes(a->V, a->M, a->group_size))
    return set_error(LN3_EINVAL, "render: workspace too small");
  if (a->view_obj == nullptr && a->views_per_obj <= 0)
    return set_error(LN3_EINVAL, "render: need view_obj or views_per_obj");
  const int G = (a->V + a->group_size - 1) / a->group_size;
  int* keys = reinterpret_cast<int*>(a->workspace);
  float* limits = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(a->workspace) +
                                           ((static_cast<size_t>(G) * 16 + 255) / 256) * 256);
  const long long rays = static_cast<long long>(a->V) * a->M;
  render_init_kernel<<<(G + 127) / 128, 128, 0, stream>>>(keys, G);
  ray_limits_kernel<<<static_cast<unsigned>((rays + 255) / 256), 256, 0, stream>>>(
      a->ray_o, a->ray_d, a->V, a->M, a->group_size, static_cast<float>(a->box_warp / 2),
      static_cast<float>(-1 * (a->box_warp / 2)), keys, limits);

  RenderParams p;
  p.planes = a->planes_cl;
  p.view_obj = a->view_obj;
  p.ray_o = a->ray_o;
  p.ray_d = a->ray_d;
  p.noise_c = a->noise_coarse;
  p.noise_f = a->noise_fine;
  p.w1 = a->w1; p.b1 = a->b1; p.w2 = a->w2; p.b2 = a->b2;
  p.rgb = a->rgb; p.depth = a->depth; p.wsum = a->weights;
  p.keys = keys;
  p.limits = limits;
  p.V = a->V; p.M = a->M; p.H = a->H; p.W = a->W;
  p.image_w = render_tile_width(a->M, a->image_w);
  p.group_size = a->group_size;
  p.views_per_obj = a->views_per_obj > 0 ? a->views_per_obj : 1;
  p.coord_scale = static_cast<float>(2.0 / a->box_warp);
  p.bbox_min = static_cast<float>(a->bbox_min); p.bbox_max = static_cast<float>(a->bbox_max);
  p.white_back = a->white_back;
  p.no_filter = 0;
  p.mlp_tf32 = a->mlp_precision == LN3_MLP_TF32;
  p.dbg_inbox = a->dbg_inbox; p.dbg_inds = a->dbg_inds; p.dbg_order = a->dbg_order;
  p.dbg_zfine = a->dbg_zfine;

  const int sms = device_sm_count();
  long long blocks = (rays + kWarpsPerBlock - 1) / kWarpsPerBlock;
  if (blocks > sms) blocks = sms;  // persistent: one 16-warp CTA per SM, grid-stride over 16-ray items
  if (int rc = a->S == 64 ? launch_render_rays<2>(p, blocks, stream) : launch_render_rays<3>(p, blocks, stream))
    return rc;
  render_finalize_kernel<<<static_cast<unsigned>((rays + 255) / 256), 256, 0, stream>>>(
      a->depth, keys, a->V, a->M, a->group_size);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "render launch: %s", cudaGetErrorString(e));
  count_launch(4);
  return LN3_OK;
}

// ------------------------------------------------------------------ point queries (mesh extraction)
// ImportanceRenderer._run_model (renderer.py:310-322) as called by forward_points /
// triplane_decode_grid (vit/vit_triplane.py:2009-2120): tri-plane gather + OSG decoder at arbitrary
// points, no in-box filter, no compositing.  Points come from memory or are generated in the kernel as
// the reference's grid: torch.linspace per axis (fp32: start + i*step below the midpoint, end - (n-1-i)*step
// above it), meshgrid 'ij', flattened (i*G + j)*G + k.
struct QueryParams {
  const float* points;  // [n_obj][P][3] or null -> grid mode
  float* sigma;         // [n_obj][P]
  float* rgb;           // [n_obj][P][3]
  long long P;
  int n_obj, grid;
  float lo[3], hi[3], step[3];
};

__device__ __forceinline__ float linspace_at(float lo, float hi, float step, int n, int i) {
  return i < n / 2 ? __fadd_rn(lo, __fmul_rn(step, static_cast<float>(i)))
                   : __fsub_rn(hi, __fmul_rn(step, static_cast<float>(n - i - 1)));
}

template <bool TF32>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, 1)
query_points_kernel(const RenderParams p, const QueryParams q) {
  extern __shared__ uint8_t smem_raw[];
  BlockSmem<64>& bs = *reinterpret_cast<BlockSmem<64>*>(smem_raw);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  load_osg_weights(bs.osg, p.w1, p.b1, p.w2, p.b2);
  __syncthreads();
  WarpSmem<64>& ws = bs.warp[warp];
  const long long chunks_per_obj = (q.P + 31) / 32;
  const long long total = chunks_per_obj * q.n_obj;
  const long long stride = static_cast<long long>(gridDim.x) * kWarpsPerBlock;
  for (long long ch = static_cast<long long>(blockIdx.x) * kWarpsPerBlock + warp; ch < total; ch += stride) {
    const int obj = static_cast<int>(ch / chunks_per_obj);
    const long long i = (ch - obj * chunks_per_obj) * 32 + lane;
    const bool live = i < q.P;
    const long long ii = live ? i : q.P - 1;
    float px, py, pz;
    if (q.points != nullptr) {
      const float* pt = q.points + (static_cast<long long>(obj) * q.P + ii) * 3;
      px = pt[0], py = pt[1], pz = pt[2];
    } else {
      const int G = q.grid;
      const int iz = static_cast<int>(ii % G), iy = static_cast<int>((ii / G) % G), ix = static_cast<int>(ii / (static_cast<long long>(G) * G));
      px = linspace_at(q.lo[0], q.hi[0], q.step[0], G, ix);
      py = linspace_at(q.lo[1], q.hi[1], q.step[1], G, iy);
      pz = linspace_at(q.lo[2], q.hi[2], q.step[2], G, iz);
    }
    const float* planes_obj = p.planes + static_cast<long long>(obj) * 3 * p.H * p.W * kC;
    bool inbox;
    float sg, cr, cg, cb;
    eval_batch<TF32>(p, bs.osg, ws.g, planes_obj, lane, px, py, pz, inbox, sg, cr, cg, cb);
    if (live) {
      const long long o = static_cast<long long>(obj) * q.P + i;
      q.sigma[o] = sg;
      q.rgb[o * 3 + 0] = cr;
      q.rgb[o * 3 + 1] = cg;
      q.rgb[o * 3 + 2] = cb;
    }
  }
}

int query_points(const ln3_query_points_args* a, cudaStream_t stream) {
  if (a->n_obj <= 0) return LN3_OK;
  if (a->C != kC || a->hidden_dim != kHid || a->decoder_output_dim != 3)
    return set_error(LN3_EUNSUPPORTED, "query_points: needs 32 plane channels and a 32 -> 64 -> 1+3 OSG decoder");
  if (!a->planes_cl || !a->sigma || !a->rgb || !a->w1 || !a->b1 || !a->w2 || !a->b2)
    return set_error(LN3_EINVAL, "query_points: null pointer");
  QueryParams q;
  q.points = a->points;
  q.sigma = a->sigma;
  q.rgb = a->rgb;
  q.n_obj = a->n_obj;
  q.grid = a->grid_size;
  if (a->points == nullptr) {
    if (a->grid_size < 2 || a->grid_size > 2048) return set_error(LN3_EINVAL, "query_points: grid_size must be in [2, 2048]");
    q.P = static_cast<long long>(a->grid_size) * a->grid_size * a->grid_size;
    const float lo[3] = {a->aabb_min_x, a->aabb_min_y, a->aabb_min_z};
    const float hi[3] = {a->aabb_max_x, a->aabb_max_y, a->aabb_max_z};
    for (int d = 0; d < 3; ++d) {
      q.lo[d] = lo[d];
      q.hi[d] = hi[d];
      q.step[d] = (hi[d] - lo[d]) / static_cast<float>(a->grid_size - 1);  // torch.linspace, fp32
    }
  } else {
    if (a->P <= 0) return LN3_OK;
    q.P = a->P;
    for (int d = 0; d < 3; ++d) q.lo[d] = q.hi[d] = q.step[d] = 0.f;
  }
  RenderParams p = {};
  p.planes = a->planes_cl;
  p.w1 = a->w1; p.b1 = a->b1; p.w2 = a->w2; p.b2 = a->b2;
  p.H = a->H; p.W = a->W;
  p.coord_scale = static_cast<float>(2.0 / a->box_warp);
  p.bbox_min = 0.f; p.bbox_max = 0.f;
  p.no_filter = 1;
  p.image_w = 0;
  p.mlp_tf32 = a->mlp_precision == LN3_MLP_TF32;
  static DeviceOnce once;
  if (int rc = once.run([] {
        cudaError_t e = cudaFuncSetAttribute(query_points_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             static_cast<int>(sizeof(BlockSmem<64>)));
        if (e == cudaSuccess)
          e = cudaFuncSetAttribute(query_points_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(sizeof(BlockSmem<64>)));
        return e == cudaSuccess ? LN3_OK : set_error(LN3_ECUDA, "query_points: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      }))
    return rc;
  const long long chunks = ((q.P + 31) / 32) * q.n_obj;
  long long blocks = (chunks + kWarpsPerBlock - 1) / kWarpsPerBlock;
  const int sms = device_sm_count();
  if (blocks > sms) blocks = sms;  // one 16-warp CTA per SM
  if (p.mlp_tf32)
    query_points_kernel<true><<<static_cast<unsigned>(blocks), kWarpsPerBlock * 32, sizeof(BlockSmem<64>), stream>>>(p, q);
  else
    query_points_kernel<false><<<static_cast<unsigned>(blocks), kWarpsPerBlock * 32, sizeof(BlockSmem<64>), stream>>>(p, q);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "query_points launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ ray generation (R1)
// RaySampler.forward (ray_sampler.py:197-257): pixel centres (i+0.5)/res, x fastest.
__global__ void generate_rays_kernel(const float* __restrict__ cams, int V, int res,
                                     float* __restrict__ ray_o, float* __restrict__ ray_d) {
  const long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int M = res * res;
  if (r >= static_cast<long long>(V) * M) return;
  const int v = static_cast<int>(r / M), m = static_cast<int>(r - static_cast<long long>(v) * M);
  const float* c = cams + v * 25;
  const float fx = c[16], sk = c[17], cx = c[18], fy = c[20], cy = c[21];
  const int i = m / res, j = m - i * res;
  const float inv = 1.f / res, half = 0.5f / res;
  const float xc = __fadd_rn(__fmul_rn(static_cast<float>(j), inv), half);
  const float yc = __fadd_rn(__fmul_rn(static_cast<float>(i), inv), half);
  // x_lift = (x - cx + cy*sk/fy - sk*y/fy) / fx ; y_lift = (y - cy) / fy
  const float xl = __fdiv_rn(__fsub_rn(__fadd_rn(__fsub_rn(xc, cx), __fdiv_rn(__fmul_rn(cy, sk), fy)),
                                       __fdiv_rn(__fmul_rn(sk, yc), fy)), fx);
  const float yl = __fdiv_rn(__fsub_rn(yc, cy), fy);
  float w[3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    w[k] = ((c[k * 4 + 0] * xl + c[k * 4 + 1] * yl) + c[k * 4 + 2]) + c[k * 4 + 3];
  const float lx = c[3], ly = c[7], lz = c[11];
  const float dx = w[0] - lx, dy = w[1] - ly, dz = w[2] - lz;
  const float n = fmaxf(sqrtf((dx * dx + dy * dy) + dz * dz), 1e-12f);
  ray_o[r * 3 + 0] = lx; ray_o[r * 3 + 1] = ly; ray_o[r * 3 + 2] = lz;
  ray_d[r * 3 + 0] = dx / n; ray_d[r * 3 + 1] = dy / n; ray_d[r * 3 + 2] = dz / n;
}

int generate_rays(const float* cams, int V, int res, float* ray_o, float* ray_d, cudaStream_t stream) {
  if (V <= 0 || res <= 0) return LN3_OK;
  const long long rays = static_cast<long long>(V) * res * res;
  generate_rays_kernel<<<static_cast<unsigned>((rays + 255) / 256), 256, 0, stream>>>(cams, V, res, ray_o, ray_d);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "generate_rays launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ planes NCHW -> channels-last
// (n_obj, 3*C, H, W) [channel = plane*C + c] -> (n_obj, 3, H, W, C); tiled smem transpose.
__global__ void planes_to_cl_kernel(const float* __restrict__ in, float* __restrict__ out, int HW) {
  __shared__ float tile[32][33];
  const int np = blockIdx.z;  // obj*3 + plane
  const int p0 = blockIdx.x * 32;
  const float* src = in + static_cast<long long>(np) * kC * HW;
  float* dst = out + static_cast<long long>(np) * HW * kC;
  for (int c = threadIdx.y; c < kC; c += blockDim.y) {
    const int pix = p0 + threadIdx.x;
    tile[c][threadIdx.x] = pix < HW ? src[static_cast<long long>(c) * HW + pix] : 0.f;
  }
  __syncthreads();
  for (int q = threadIdx.y; q < 32; q += blockDim.y) {
    const int pix = p0 + q;
    if (pix < HW) dst[static_cast<long long>(pix) * kC + threadIdx.x] = tile[threadIdx.x][q];
  }
}

int planes_to_channels_last(const float* planes, int n_obj, int C, int H, int W, float* out,
                            cudaStream_t stream) {
  if (n_obj <= 0) return LN3_OK;
  if (C != kC) return set_error(LN3_EUNSUPPORTED, "planes_to_channels_last: C must be 32");
  const int HW = H * W;
  dim3 grid((HW + 31) / 32, 1, n_obj * 3), block(32, 8);
  planes_to_cl_kernel<<<grid, block, 0, stream>>>(planes, out, HW);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "planes_to_channels_last launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

}  // namespace ln3
