// Persistent warp-specialised FP8 (e4m3) GEMM for sm_90a with 1 x 128 activation block scales and per-channel
// weight scales (format in include/ln3b200.h):
//   out = epilogue(w_scale[n] * sum_kb a_scale[m, kb] * (A[m, kb-block] . W[n, kb-block]))
// The opt-in precision of the DiT blocks' qkv / fc1 / fc2 GEMMs (dit/_denoiser.py).
//
// Three warpgroups per CTA, one CTA per SM, 128 x 128 output tiles, BK = 128 (128 e4m3 = one 128B-swizzle row):
//   warpgroups 0, 1 : consumers.  Warpgroup w computes rows [64 w, 64 w + 64) of the tile: four wgmma.m64n128k32
//                     e4m3 per k-block into a 64-register partial accumulator, which is then promoted --
//                     acc = fmaf(a_scale[m, kb], partial, acc) -- into a second, fp32 accumulator.  The promotion
//                     per 128-deep block bounds the error of the tensor core's narrower fp8 accumulation to one
//                     block.  2 x 64 accumulator registers fit the 168 registers a thread of a 384-thread CTA gets;
//                     a 128 x 128 tile per warpgroup (the bf16 kernel's) would not leave room for the second one.
//                     A warpgroup's promotion runs while the other warpgroup's MMAs keep the tensor core busy.
//   warpgroup 2     : TMA producer (40 registers; one lane issues cp.async.bulk.tensor into a kStages-deep ring).
// The epilogue stores straight from the accumulator layout (bf16 pairs, or e4m3 pairs plus one block scale per
// row and 128-column tile: the tile's row absmax is a max over the 4 lanes of a quad).
// Each CTA walks tiles blockIdx.x, +gridDim.x, ...; every output element sees the same instructions in the same
// k order whatever the grid, so results do not depend on the schedule.
#include "common.cuh"
#include "ln3_internal.h"

namespace ln3 {
namespace {

constexpr int BM = 128;
constexpr int BN = 128;
// Head width of the head-RMSNorm epilogue: whole heads per BN tile, weights [nsec][kHnHead].  The denoisers
// with q/k norms all have 64-wide heads; DiT-XL/2's 72-wide heads carry none (TextCondDiTBlock), and the
// host (ops.gemm / ops.gemm_fp8) refuses any other head_norm weight width.
constexpr int kHnHead = 64;
static_assert(BN % kHnHead == 0, "head-norm heads must tile BN");
constexpr int BK = 128;  // 128 e4m3 = 128 bytes = one 128B-swizzle row
constexpr int kStages = 6;
constexpr int kABytes = BM * BK;  // 16 KB
constexpr int kBBytes = BN * BK;  // 16 KB
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kThreads = 3 * 128;
constexpr int kConsumerRegs = 232;
constexpr int kProducerRegs = 40;
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/;
static_assert(kSmemBytes <= 227 * 1024, "shared memory per block on sm_90");

struct Fp8Params {
  int M, N, K;
  const float* a_scale;
  long long a_scale_ld;
  const float* w_scale;
  const float* bias;
  void* out;
  long long ldo;
  float* out_scale;
  long long out_scale_ld;
  const float* hn_w;
  int hn_nsec, hn_sec_cols;
  float hn_eps;
};

enum { kEpiBf16 = 0, kEpiBf16HeadNorm = 1, kEpiFp8 = 2, kEpiFp8Gelu = 3 };

// Epilogue of one warpgroup's 64 x 128 accumulator.  wgmma layout: lane 4g + q of warp w holds rows
// 16 w + g (acc[4 i], acc[4 i + 1]) and 16 w + g + 8 (acc[4 i + 2], acc[4 i + 3]), columns 8 i + 2 q, +1.
template <int EPI>
__device__ __forceinline__ void epilogue(const Fp8Params& p, float* acc, int m_base, int n_base, int lane, int tn) {
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int i = 0; i < BN / 8; ++i) {
    const float2 ws = __ldg(reinterpret_cast<const float2*>(p.w_scale + n_base + 8 * i + 2 * q));
    float2 b = make_float2(0.f, 0.f);
    if (p.bias != nullptr) b = __ldg(reinterpret_cast<const float2*>(p.bias + n_base + 8 * i + 2 * q));
    acc[4 * i] = fmaf(acc[4 * i], ws.x, b.x);
    acc[4 * i + 1] = fmaf(acc[4 * i + 1], ws.y, b.y);
    acc[4 * i + 2] = fmaf(acc[4 * i + 2], ws.x, b.x);
    acc[4 * i + 3] = fmaf(acc[4 * i + 3], ws.y, b.y);
  }
  if constexpr (EPI == kEpiBf16HeadNorm) {
    // a 64-column head of one row lives in the 4 lanes of a quad (16 values each); same arithmetic as the bf16 GEMM
#pragma unroll
    for (int h = 0; h < BN / kHnHead; ++h) {
      const int sec = (n_base + kHnHead * h) / p.hn_sec_cols;
      if (sec >= p.hn_nsec) continue;
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int i = 8 * h; i < 8 * h + 8; ++i) {
        s0 = fmaf(acc[4 * i], acc[4 * i], fmaf(acc[4 * i + 1], acc[4 * i + 1], s0));
        s1 = fmaf(acc[4 * i + 2], acc[4 * i + 2], fmaf(acc[4 * i + 3], acc[4 * i + 3], s1));
      }
      s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
      s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
      const float r0 = rsqrtf(s0 * (1.0f / kHnHead) + p.hn_eps), r1 = rsqrtf(s1 * (1.0f / kHnHead) + p.hn_eps);
      const float* w = p.hn_w + sec * kHnHead;
#pragma unroll
      for (int i = 8 * h; i < 8 * h + 8; ++i) {
        const float2 ww = __ldg(reinterpret_cast<const float2*>(w + 8 * (i - 8 * h) + 2 * q));
        acc[4 * i] *= r0 * ww.x; acc[4 * i + 1] *= r0 * ww.y;
        acc[4 * i + 2] *= r1 * ww.x; acc[4 * i + 3] *= r1 * ww.y;
      }
    }
  }
  if constexpr (EPI == kEpiFp8Gelu) {
#pragma unroll
    for (int i = 0; i < BN / 4; ++i) gelu_erf_poly2(acc[2 * i], acc[2 * i + 1]);
  }
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int m = m_base + g + 8 * half;
    if constexpr (EPI == kEpiFp8 || EPI == kEpiFp8Gelu) {
      float amax = 0.f;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i)
        amax = fmaxf(amax, fmaxf(fabsf(acc[4 * i + 2 * half]), fabsf(acc[4 * i + 2 * half + 1])));
      amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
      amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
      const float s = fp8_block_scale(amax);
      if (m >= p.M) continue;
      uint8_t* o = reinterpret_cast<uint8_t*>(p.out) + m * p.ldo + n_base + 2 * q;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i)
        *reinterpret_cast<uint16_t*>(o + 8 * i) = fp8_code2(acc[4 * i + 2 * half], acc[4 * i + 2 * half + 1], s);
      if (q == 0) p.out_scale[m * p.out_scale_ld + tn] = s;
    } else {
      if (m >= p.M) continue;
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + m * p.ldo + n_base + 2 * q;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i)
        *reinterpret_cast<uint32_t*>(o + 8 * i) = pack_bf16x2(acc[4 * i + 2 * half], acc[4 * i + 2 * half + 1]);
    }
  }
}

template <int EPI>
__global__ void __launch_bounds__(kThreads, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                const Fp8Params p) {
  if (threadIdx.x >= 256) {
    setmaxnreg_dec<kProducerRegs>();
  } else {
    setmaxnreg_inc<kConsumerRegs>();
  }
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kABytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);  // [kStages]
  uint64_t* empty_bar = full_bar + kStages;                                         // [kStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_m = (p.M + BM - 1) / BM, tiles_n = p.N / BN;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = p.K / BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);  // both consumer warpgroups read every stage
    }
    fence_barrier_init();
  }
  __syncthreads();

  // M first inside an N panel: concurrently resident tiles share W panels in the L2 while A panels stream
  if (warp >= 8) {
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        const int tm = t % tiles_m, tn = t / tiles_m;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait_silent(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], kStageBytes);
          tma_load_2d(smem_a + stage * kABytes, &tmap_a, &full_bar[stage], kb * BK, tm * BM);
          tma_load_2d(smem_b + stage * kBBytes, &tmap_b, &full_bar[stage], kb * BK, tn * BN);
          if (++stage == kStages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const uint64_t a_desc0 = make_smem_desc_sw128(smem_u32(smem_a + wg * 64 * BK), 16, 1024);
  const uint64_t b_desc0 = make_smem_desc_sw128(smem_u32(smem_b), 16, 1024);
  const bool leader = (threadIdx.x & 127) == 0;
  const int g = lane >> 2;
  uint32_t slot = 0;  // ring position of the tile's first k-block
  float acc[BN / 2], part[BN / 2];
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const int tm = t % tiles_m, tn = t / tiles_m;
    const int m_base = tm * BM + wg * 64 + (warp & 3) * 16;
    // a_scale rows of this thread's two accumulator rows; rows >= M read as scale 0 (their A rows are TMA zero fill)
    const int m0 = m_base + g, m1 = m0 + 8;
    const float* sa0 = m0 < p.M ? p.a_scale + m0 * p.a_scale_ld : nullptr;
    const float* sa1 = m1 < p.M ? p.a_scale + m1 * p.a_scale_ld : nullptr;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    auto issue = [&](float* part, int kb, float& s0, float& s1) {
      const uint32_t pos = slot + kb, stage = pos % kStages;
      s0 = sa0 != nullptr ? __ldg(sa0 + kb) : 0.f;
      s1 = sa1 != nullptr ? __ldg(sa1 + kb) : 0.f;
      mbar_wait_silent(&full_bar[stage], (pos / kStages) & 1);
      const uint64_t da = a_desc0 + stage * (kABytes >> 4);
      const uint64_t db = b_desc0 + stage * (kBBytes >> 4);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 32; ++k) wgmma_m64n128k32_e4m3_ss(part, da + 2 * k, db + 2 * k, k != 0 ? 1u : 0u);
      wgmma_commit();
    };
    auto promote = [&](float* part, int kb, float s0, float s1) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) reg_fence(part[i]);
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        acc[4 * i] = fmaf(s0, part[4 * i], acc[4 * i]);
        acc[4 * i + 1] = fmaf(s0, part[4 * i + 1], acc[4 * i + 1]);
        acc[4 * i + 2] = fmaf(s1, part[4 * i + 2], acc[4 * i + 2]);
        acc[4 * i + 3] = fmaf(s1, part[4 * i + 3], acc[4 * i + 3]);
      }
      if (leader) mbar_arrive(&empty_bar[(slot + kb) % kStages]);
    };
    for (int kb = 0; kb < num_kb; ++kb) {
      float s0, s1;
      issue(part, kb, s0, s1);
      wgmma_wait<0>();
      promote(part, kb, s0, s1);
    }
    slot += num_kb;
    epilogue<EPI>(p, acc, m_base, tn * BN, lane, tn);
  }
}

template <int EPI>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const Fp8Params& p, cudaStream_t stream) {
  static DeviceOnce once;
  if (int rc = once.run([] {
        cudaError_t e = cudaFuncSetAttribute(gemm_fp8_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             kSmemBytes);
        return e == cudaSuccess ? LN3_OK : set_error(LN3_ECUDA, "gemm_fp8: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      }))
    return rc;
  const int tiles = ((p.M + BM - 1) / BM) * (p.N / BN);
  const int sms = device_sm_count();
  const int grid = tiles < sms ? tiles : sms;
  gemm_fp8_kernel<EPI><<<grid, kThreads, kSmemBytes, stream>>>(ta, tb, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "gemm_fp8 launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

}  // namespace

size_t gemm_fp8_workspace_bytes() { return 0; }

int gemm_fp8(const ln3_gemm_fp8_args* a, cudaStream_t stream) {
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return set_error(LN3_EINVAL, "gemm_fp8: empty problem");
  if (a->K % BK != 0) return set_error(LN3_EINVAL, "gemm_fp8: K=%d must be a multiple of %d", a->K, BK);
  if (a->N % BN != 0) return set_error(LN3_EINVAL, "gemm_fp8: N=%d must be a multiple of %d", a->N, BN);
  if (a->A == nullptr || a->W == nullptr || a->out == nullptr || a->a_scale == nullptr || a->w_scale == nullptr)
    return set_error(LN3_EINVAL, "gemm_fp8: A, W, out, a_scale and w_scale must be given");
  if (a->lda < a->K || a->ldw < a->K || a->lda % 16 != 0 || a->ldw % 16 != 0)
    return set_error(LN3_EINVAL, "gemm_fp8: lda/ldw must be >= K and multiples of 16 bytes");
  if (misaligned16(a->A) || misaligned16(a->W) || misaligned16(a->out) || misaligned16(a->bias) ||
      misaligned16(a->w_scale) || misaligned16(a->head_norm_w))
    return set_error(LN3_EINVAL, "gemm_fp8: A, W, out, bias, w_scale and head_norm_w must be 16-byte aligned");
  if (a->a_scale_ld < a->K / BK) return set_error(LN3_EINVAL, "gemm_fp8: a_scale_ld must be >= K/128");
  const bool fp8_out = a->out_kind == LN3_OUT_FP8;
  const long long row_bytes = a->ldo * (fp8_out ? 1 : 2);
  if (a->ldo < a->N || row_bytes % 16 != 0)
    return set_error(LN3_EINVAL, "gemm_fp8: ldo must be >= N with a row pitch that is a multiple of 16 bytes");
  if (fp8_out && (a->out_scale == nullptr || a->out_scale_ld < a->N / BN))
    return set_error(LN3_EINVAL, "gemm_fp8: LN3_OUT_FP8 needs out_scale with out_scale_ld >= N/128");
  int epi;
  if (a->out_kind == LN3_OUT_BF16 && a->act == LN3_ACT_NONE) {
    epi = a->head_norm_w != nullptr ? kEpiBf16HeadNorm : kEpiBf16;
  } else if (fp8_out && (a->act == LN3_ACT_NONE || a->act == LN3_ACT_GELU_ERF)) {
    if (a->head_norm_w != nullptr) return set_error(LN3_EUNSUPPORTED, "gemm_fp8: head_norm needs LN3_OUT_BF16");
    epi = a->act == LN3_ACT_GELU_ERF ? kEpiFp8Gelu : kEpiFp8;
  } else {
    return set_error(LN3_EUNSUPPORTED, "gemm_fp8: output kind %d with activation %d is not implemented", a->out_kind,
                     a->act);
  }
  if (epi == kEpiBf16HeadNorm &&
      (a->head_norm_nsec <= 0 || a->head_norm_sec_cols <= 0 || a->head_norm_sec_cols % kHnHead != 0))
    return set_error(LN3_EINVAL, "gemm_fp8: head_norm sections must be positive multiples of %d columns (the head width)", kHnHead);

  CUtensorMap ta, tb;
  int rc = make_tmap_2d_u8(&ta, a->A, a->M, a->K, a->lda, BM, BK);
  if (rc) return rc;
  rc = make_tmap_2d_u8(&tb, a->W, a->N, a->K, a->ldw, BN, BK);
  if (rc) return rc;
  Fp8Params p;
  p.M = a->M;
  p.N = a->N;
  p.K = a->K;
  p.a_scale = a->a_scale;
  p.a_scale_ld = a->a_scale_ld;
  p.w_scale = a->w_scale;
  p.bias = a->bias;
  p.out = a->out;
  p.ldo = a->ldo;
  p.out_scale = a->out_scale;
  p.out_scale_ld = a->out_scale_ld;
  p.hn_w = a->head_norm_w;
  p.hn_nsec = a->head_norm_nsec;
  p.hn_sec_cols = a->head_norm_sec_cols;
  p.hn_eps = a->head_norm_eps;
  switch (epi) {
    case kEpiBf16: return launch<kEpiBf16>(ta, tb, p, stream);
    case kEpiBf16HeadNorm: return launch<kEpiBf16HeadNorm>(ta, tb, p, stream);
    case kEpiFp8: return launch<kEpiFp8>(ta, tb, p, stream);
    default: return launch<kEpiFp8Gelu>(ta, tb, p, stream);
  }
}

}  // namespace ln3
