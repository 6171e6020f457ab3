// Fused multi-head attention forward for sm_90a (head_dim 64, bf16 in, fp32 softmax / accumulate).
//
// Replaces xformers.ops.memory_efficient_attention at its three call sites on the path:
//   vit/vision_transformer.py:114-118 (DiT self-attention, (B, N, 3, H, 64) packed qkv),
//   ldm/modules/attention.py:279-307  (cross-attention; the reference's three permute+contiguous
//                                       copies disappear: heads are addressed through the TMA map),
//   dit/dit_decoder.py                (in-plane / global attention of the DiT2 VAE decoder).
// Semantics: out = softmax(q k^T * scale) v, optionally causal (key j visible to query i when j <= i), with an
// optional second K/V source appended after the first along the sequence.
//
// One CTA = 128 query rows of one (batch, head):
//   warpgroups 0, 1 : softmax / MMA warpgroups; warpgroup w owns query rows [64 w, 64 w + 64).
//                     S = Q K^T with wgmma.m64n128k16 (Q and K from 128B-swizzled smem), online softmax in
//                     registers (a row lives in the 4 lanes of a quad), P converted in registers to the A
//                     fragments of O += P V (wgmma.m64n64k16, A from registers, V transposed from smem).
//   warp 8 lane 0   : TMA producer (Q once, K / V ring of kStages 128-key blocks)
#include <cstdlib>

#include "common.cuh"
#include "ln3_internal.h"

namespace ln3 {

static constexpr int kQT = 128;   // query rows per CTA
static constexpr int kKT = 128;   // keys per block
static constexpr int kHD = 64;    // head dim
static constexpr int kTileBytes = 128 * kHD * 2;  // 16 KB
static constexpr int kStages = 4;
static constexpr int kThreads = 2 * 128 + 32;
// Q | K[kStages] | V[kStages] | barriers
static constexpr int kFmhaSmem = 1024 + kTileBytes * (1 + 2 * kStages) + 256;

struct FmhaParams {
  int Lq, Lkv, Lkv2;   // Lkv2: rows of the second K/V source (0 = none)
  int nb1, nb2;        // 128-key blocks of each source
  float scale_log2;    // softmax scale * log2(e)
  int causal;
  __nv_bfloat16* out;
  long long o_ld, o_bs;
};

__global__ void __launch_bounds__(kThreads, 1)
fmha_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_k2,
                const __grid_constant__ CUtensorMap tmap_v2, const FmhaParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kTileBytes;               // [kStages]
  uint8_t* sV = sK + kStages * kTileBytes;     // [kStages]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kStages * kTileBytes);
  uint64_t* q_full = bars;                     // [1]
  uint64_t* kv_full = bars + 1;                // [kStages]
  uint64_t* kv_empty = bars + 1 + kStages;     // [kStages], one arrival per warpgroup

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kQT;
  const int h = blockIdx.y, b = blockIdx.z;
  // causal: blocks past the last query row of this CTA are fully masked (first K/V source only)
  const int nb1 = p.causal ? min(p.nb1, (min(q0 + kQT, p.Lq) - 1) / kKT + 1) : p.nb1;
  const int nblocks = nb1 + p.nb2;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp == 8) {
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, kTileBytes);
      tma_load_3d(sQ, &tmap_q, q_full, h * kHD, q0, b);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < nblocks; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1);
        mbar_arrive_expect_tx(&kv_full[stage], 2 * kTileBytes);
        const bool second = j >= nb1;
        const int row = (second ? j - nb1 : j) * kKT;
        tma_load_3d(sK + stage * kTileBytes, second ? &tmap_k2 : &tmap_k, &kv_full[stage], h * kHD, row, b);
        tma_load_3d(sV + stage * kTileBytes, second ? &tmap_v2 : &tmap_v, &kv_full[stage], h * kHD, row, b);
        if (++stage == kStages) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  const int g = lane >> 2, q = lane & 3;
  // query rows of this thread: r0 (accumulator slots 4i, 4i+1) and r0 + 8 (slots 4i+2, 4i+3)
  const int r0 = q0 + wg * 64 + (warp & 3) * 16 + g;
  const uint64_t q_desc = make_smem_desc_sw128(smem_u32(sQ + wg * (64 * 128)), 16, 1024);
  const uint64_t k_desc0 = make_smem_desc_sw128(smem_u32(sK), 16, 1024);
  const uint64_t v_desc0 = make_smem_desc_sw128(smem_u32(sV), 16, 1024);

  float o[kHD / 2];
#pragma unroll
  for (int i = 0; i < kHD / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait(q_full, 0);

  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0; j < nblocks; ++j) {
    const bool second = j >= nb1;
    const int kbase = (second ? j - nb1 : j) * kKT;
    const int klen = second ? p.Lkv2 : p.Lkv;
    mbar_wait(&kv_full[stage], phase);
    float s[kKT / 2];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kHD / 16; ++k)
      wgmma_m64n128k16_ss(s, q_desc + 2 * k, k_desc0 + static_cast<uint32_t>(stage) * (kTileBytes >> 4) + 2 * k,
                          k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < kKT / 2; ++i) reg_fence(s[i]);

    // scale to log2 units, mask keys past the source's end (TMA zero-filled them) and, causally, keys > row
    const bool need_mask = kbase + kKT > klen || (p.causal && !second && kbase + kKT - 1 > r0);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < kKT / 8; ++i) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v = s[4 * i + e] * p.scale_log2;
        if (need_mask) {
          const int key = kbase + 8 * i + 2 * q + (e & 1);
          const int row = r0 + 8 * (e >> 1);
          if (key >= klen || (p.causal && !second && key > row)) v = -INFINITY;
        }
        s[4 * i + e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    }
    float alpha[2], m_use[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m_run[r], mx[r]);
      m_use[r] = m_new == -INFINITY ? 0.f : m_new;   // a row with no visible key yet
      alpha[r] = fast_exp2(m_run[r] - m_use[r]);
      m_run[r] = m_new;
      l_run[r] *= alpha[r];
    }
    // P = 2^(s - m) as the bf16 A fragments of P V: k-step kk covers keys [16 kk, 16 kk + 16)
    uint32_t pa[kKT / 16][4];
#pragma unroll
    for (int kk = 0; kk < kKT / 16; ++kk) {
      float e[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        e[t] = fast_exp2(s[8 * kk + t] - m_use[(t >> 1) & 1]);
        l_run[(t >> 1) & 1] += e[t];
      }
      pa[kk][0] = pack_bf16x2(e[0], e[1]);
      pa[kk][1] = pack_bf16x2(e[2], e[3]);
      pa[kk][2] = pack_bf16x2(e[4], e[5]);
      pa[kk][3] = pack_bf16x2(e[6], e[7]);
    }
#pragma unroll
    for (int i = 0; i < kHD / 8; ++i) {
      o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kKT / 16; ++kk)
      wgmma_m64n64k16_rs_tb(o, pa[kk], v_desc0 + static_cast<uint32_t>(stage) * (kTileBytes >> 4) + kk * 128, 1u);
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < kHD / 2; ++i) reg_fence(o[i]);
    if ((threadIdx.x & 127) == 0) mbar_arrive(&kv_empty[stage]);
    if (++stage == kStages) {
      stage = 0;
      phase ^= 1;
    }
  }

  // final normalisation; the row sum is spread over the 4 lanes of the quad
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const float inv[2] = {l_run[0] > 0.f ? 1.f / l_run[0] : 0.f, l_run[1] > 0.f ? 1.f / l_run[1] : 0.f};
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = r0 + 8 * r;
    if (row >= p.Lq) continue;
    __nv_bfloat16* dst = p.out + b * p.o_bs + row * p.o_ld + h * kHD + 2 * q;
#pragma unroll
    for (int i = 0; i < kHD / 8; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16x2(o[4 * i + 2 * r] * inv[r], o[4 * i + 2 * r + 1] * inv[r]);
  }
}

int fmha_fwd(const ln3_fmha_args* a, cudaStream_t stream) {
  if (a->head_dim != kHD) return set_error(LN3_EUNSUPPORTED, "fmha: head_dim must be 64");
  if (a->B <= 0 || a->H <= 0 || a->Lq <= 0 || a->Lkv <= 0)
    return set_error(LN3_EINVAL, "fmha: empty problem");
  if ((a->q_ld | a->k_ld | a->v_ld | a->o_ld | a->q_bs | a->k_bs | a->v_bs | a->o_bs) % 8)
    return set_error(LN3_EINVAL, "fmha: strides must be multiples of 8 elements");
  if ((reinterpret_cast<uintptr_t>(a->q) | reinterpret_cast<uintptr_t>(a->k) |
       reinterpret_cast<uintptr_t>(a->v) | reinterpret_cast<uintptr_t>(a->out)) & 15)
    return set_error(LN3_EINVAL, "fmha: pointers must be 16-byte aligned");
  if (a->causal && (a->k2 != nullptr || a->v2 != nullptr))
    return set_error(LN3_EINVAL, "fmha: causal attention takes a single K/V source");
  const bool two = a->k2 != nullptr || a->v2 != nullptr;
  if (two) {
    if (!a->k2 || !a->v2 || a->Lkv2 <= 0) return set_error(LN3_EINVAL, "fmha: k2/v2/Lkv2 must be given together");
    if ((a->k2_ld | a->v2_ld | a->k2_bs | a->v2_bs) % 8 ||
        ((reinterpret_cast<uintptr_t>(a->k2) | reinterpret_cast<uintptr_t>(a->v2)) & 15))
      return set_error(LN3_EINVAL, "fmha: k2/v2 alignment");
  }
  if (a->B > 65535 || a->H > 65535) return set_error(LN3_EUNSUPPORTED, "fmha: batch or head count above 65535");
  static DeviceOnce once;   // the shared-memory opt-in is per device
  if (int rc = once.run([] {
        cudaError_t e = cudaFuncSetAttribute(fmha_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFmhaSmem);
        return e == cudaSuccess ? LN3_OK : set_error(LN3_ECUDA, "fmha: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      }))
    return rc;
  CUtensorMap tq, tk, tv, tk2, tv2;
  int rc;
  const long long cols = static_cast<long long>(a->H) * kHD;
  if ((rc = make_tmap_3d_bf16(&tq, a->q, cols, a->Lq, a->B, a->q_ld, a->q_bs, kHD, kQT))) return rc;
  if ((rc = make_tmap_3d_bf16(&tk, a->k, cols, a->Lkv, a->B, a->k_ld, a->k_bs, kHD, kKT))) return rc;
  if ((rc = make_tmap_3d_bf16(&tv, a->v, cols, a->Lkv, a->B, a->v_ld, a->v_bs, kHD, kKT))) return rc;
  if (two) {
    if ((rc = make_tmap_3d_bf16(&tk2, a->k2, cols, a->Lkv2, a->B, a->k2_ld, a->k2_bs, kHD, kKT))) return rc;
    if ((rc = make_tmap_3d_bf16(&tv2, a->v2, cols, a->Lkv2, a->B, a->v2_ld, a->v2_bs, kHD, kKT))) return rc;
  } else {
    tk2 = tk;
    tv2 = tv;
  }
  FmhaParams p;
  p.Lq = a->Lq;
  p.Lkv = a->Lkv;
  p.Lkv2 = two ? a->Lkv2 : 0;
  p.nb1 = (a->Lkv + kKT - 1) / kKT;
  p.nb2 = two ? (a->Lkv2 + kKT - 1) / kKT : 0;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.causal = a->causal ? 1 : 0;
  p.out = reinterpret_cast<__nv_bfloat16*>(a->out);
  p.o_ld = a->o_ld;
  p.o_bs = a->o_bs;
  const dim3 grid((a->Lq + kQT - 1) / kQT, a->H, a->B);
  cudaError_t e = launch_pdl(fmha_fwd_kernel, grid, dim3(kThreads), kFmhaSmem, stream, tq, tk, tv, tk2, tv2, p);
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "fmha launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

}  // namespace ln3
