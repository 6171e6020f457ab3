// 9-channel patch operand of the multi-view DINOv2 conditioner (FrozenDinov2ImageEmbedderMVPlucker):
// RGB + Plücker camera rays, im2col'd for the 14x14 patch-embedding GEMM in one pass.
// Reference call sites and the rounding order are documented in include/ln3b200.h.
#include "common.cuh"
#include "ln3_internal.h"

namespace ln3 {

namespace {

constexpr int kRes = 224;                  // FrozenDinov2ImageEmbedderMVPlucker.reso_encoder
constexpr int kPatch = 14;
constexpr int kGrid = kRes / kPatch;       // 16 x 16 patches
constexpr int kPix = kPatch * kPatch;      // 196 columns per channel
constexpr int kCols = 9 * kPix;            // 1764 = Conv2d(9, D, 14, 14).weight.reshape(D, -1) width
constexpr int kPairs = kPix / 2;           // each thread owns two horizontally adjacent pixels

__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

struct Ray {
  float m0, m1, m2, d0, d1, d2;  // o x d, d
};

// gen_rays + get_plucker_ray for one pixel (x, y) of the 224 x 224 grid.  Every operation is explicitly
// rounded (no FMA contraction) so that the order is the reference's op order, see the header.
__device__ __forceinline__ Ray plucker_ray(const float* __restrict__ c, int x, int y) {
  const float u = __fdiv_rn(__fadd_rn(static_cast<float>(x), 0.5f), static_cast<float>(kRes));
  const float v = __fdiv_rn(__fadd_rn(static_cast<float>(y), 0.5f), static_cast<float>(kRes));
  const float a = __fdiv_rn(__fsub_rn(u, c[18]), c[16]);          // (xx - cx) / fx
  const float b = __fdiv_rn(__fsub_rn(v, c[21]), c[20]);          // (yy - cy) / fy
  const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)), 1.0f));
  // dirs /= norm (fp32), then the bf16 matmul c2w[:3, :3] @ dirs: bf16 operands, fp32 sum, bf16 result
  const float e0 = bf16_round(__fdiv_rn(a, nrm)), e1 = bf16_round(__fdiv_rn(b, nrm)),
              e2 = bf16_round(__fdiv_rn(1.0f, nrm));
  float d[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float r0 = bf16_round(c[4 * i]), r1 = bf16_round(c[4 * i + 1]), r2 = bf16_round(c[4 * i + 2]);
    d[i] = bf16_round(__fadd_rn(__fadd_rn(__fmul_rn(r0, e0), __fmul_rn(r1, e1)), __fmul_rn(r2, e2)));
  }
  // torch.cross(o fp32, d bf16) is promoted to fp32; o = c2w[:3, 3]
  const float o0 = c[3], o1 = c[7], o2 = c[11];
  Ray r;
  r.m0 = __fsub_rn(__fmul_rn(o1, d[2]), __fmul_rn(o2, d[1]));
  r.m1 = __fsub_rn(__fmul_rn(o2, d[0]), __fmul_rn(o0, d[2]));
  r.m2 = __fsub_rn(__fmul_rn(o0, d[1]), __fmul_rn(o1, d[0]));
  r.d0 = d[0];
  r.d1 = d[1];
  r.d2 = d[2];
  return r;
}

// One CTA per output row (= one 14 x 14 patch of one view).  Thread t < 98 owns the pixel pair (ky, 2j), (ky, 2j+1)
// of the patch and writes both of them in every channel with one 32-bit store; all threads then zero the padding.
__global__ void __launch_bounds__(128)
plucker_patchify_kernel(const float* __restrict__ image, const float* __restrict__ cams,
                        __nv_bfloat16* __restrict__ out, long long ldo) {
  const int row = blockIdx.x;                                     // n * 256 + py * 16 + px
  const int n = row / (kGrid * kGrid), py = (row / kGrid) % kGrid, px = row % kGrid;
  __nv_bfloat16* o = out + static_cast<long long>(row) * ldo;
  const int t = threadIdx.x;
  if (t < kPairs) {
    const int ky = t / (kPatch / 2), kx = (t % (kPatch / 2)) * 2;
    const int y = py * kPatch + ky, x = px * kPatch + kx;
    const int col = ky * kPatch + kx;
    const float* c = cams + static_cast<long long>(n) * 25;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float2 p = *reinterpret_cast<const float2*>(
          image + ((static_cast<long long>(n) * 3 + ch) * kRes + y) * kRes + x);
      *reinterpret_cast<uint32_t*>(o + ch * kPix + col) = pack_bf16x2(p.x, p.y);
    }
    const Ray r0 = plucker_ray(c, x, y), r1 = plucker_ray(c, x + 1, y);
    *reinterpret_cast<uint32_t*>(o + 3 * kPix + col) = pack_bf16x2(r0.m0, r1.m0);
    *reinterpret_cast<uint32_t*>(o + 4 * kPix + col) = pack_bf16x2(r0.m1, r1.m1);
    *reinterpret_cast<uint32_t*>(o + 5 * kPix + col) = pack_bf16x2(r0.m2, r1.m2);
    *reinterpret_cast<uint32_t*>(o + 6 * kPix + col) = pack_bf16x2(r0.d0, r1.d0);
    *reinterpret_cast<uint32_t*>(o + 7 * kPix + col) = pack_bf16x2(r0.d1, r1.d1);
    *reinterpret_cast<uint32_t*>(o + 8 * kPix + col) = pack_bf16x2(r0.d2, r1.d2);
  }
  for (long long j = kCols + 2 * t; j < ldo; j += 2 * blockDim.x) *reinterpret_cast<uint32_t*>(o + j) = 0u;
}

bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

}  // namespace

int plucker_patchify(const ln3_plucker_patchify_args* a, cudaStream_t stream) {
  if (a->N < 0) return set_error(LN3_EINVAL, "plucker_patchify: N < 0");
  if (a->ldo < kCols || a->ldo % 8)
    return set_error(LN3_EINVAL, "plucker_patchify: ldo must be >= 1764 and a multiple of 8 (got %lld)", a->ldo);
  if (!a->image || !a->cams || !a->out) return set_error(LN3_EINVAL, "plucker_patchify: null pointer");
  if (misaligned16(a->image) || misaligned16(a->cams) || misaligned16(a->out))
    return set_error(LN3_EINVAL, "plucker_patchify: image, cams and out must be 16-byte aligned");
  if (a->N == 0) return LN3_OK;
  if (static_cast<long long>(a->N) * kGrid * kGrid > 0x7fffffffLL)
    return set_error(LN3_EINVAL, "plucker_patchify: N too large");
  plucker_patchify_kernel<<<a->N * kGrid * kGrid, 128, 0, stream>>>(
      a->image, a->cams, static_cast<__nv_bfloat16*>(a->out), a->ldo);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "plucker_patchify launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

}  // namespace ln3
