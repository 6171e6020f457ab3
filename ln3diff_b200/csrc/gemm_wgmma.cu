// Persistent warp-specialised bf16 GEMM for sm_90a:  D[M,N] = epilogue(A[M,K] . W[N,K]^T)
//
// Replaces the cuBLAS/cuBLASLt launches behind every nn.Linear of the reference DiT blocks
// (dit/dit_models_xformers.py:231-323 DiTBlock/TextCondDiTBlock, vit/vision_transformer.py:106-124
// qkv/proj, ldm/modules/attention.py:245-307 to_q/to_k/to_v/to_out, xformers FusedMLP) and fuses
// the elementwise tail that follows each of them in the reference (bias, GELU / SiLU, the
// adaLN-Zero `x + gate * f(.)` residual update, the per-head q/k RMSNorm) into the register epilogue.
//
// Ping-pong schedule, three warpgroups per CTA, one CTA per SM:
//   warpgroups 0, 1 : consumers (232 registers via setmaxnreg).  Each owns a whole 128 x 128 tile: two
//                     wgmma.m64n128k16 per 16-deep k step into 128 fp32 accumulators per thread, with one MMA
//                     group kept in flight across k-blocks.  The two take alternate tiles of the CTA's sequence
//                     and a named-barrier hand-over makes their mainloops alternate, so the epilogue of one
//                     runs while the other's MMAs keep the tensor core busy.
//   warpgroup 2     : TMA producer (40 registers; one lane issues cp.async.bulk.tensor, 128B swizzle, into a
//                     kStages-deep ring shared by both consumers in tile order).
// bf16 outputs are written through a per-consumer 32 KB staging tile in shared memory (128B-swizzled, bank
// conflict free) and stored with TMA tensor stores that clip rows >= M; an output pitch that rules out a tensor
// map, and the fp32 / residual outputs, store straight from the accumulator layout.
// Each CTA walks tiles blockIdx.x, +gridDim.x, ...; every output element sees the same wgmma instructions in the
// same k order as with one 64-row warpgroup per tile half, so results do not depend on the schedule.
#include "common.cuh"
#include "ln3_internal.h"

namespace ln3 {

static constexpr int BM = 128;
static constexpr int BN = 128;
static constexpr int BK = 64;  // 64 bf16 = 128 bytes = one 128B-swizzle row
// Head width of the head-RMSNorm epilogue: whole heads per BN tile, weights [nsec][kHnHead].  The denoisers
// with q/k norms all have 64-wide heads; DiT-XL/2's 72-wide heads carry none (TextCondDiTBlock), and the
// host (ops.gemm / ops.gemm_fp8) refuses any other head_norm weight width.
static constexpr int kHnHead = 64;
static_assert(BN % kHnHead == 0, "head-norm heads must tile BN");
static constexpr int kStages = 5;
static constexpr int kABytes = BM * BK * 2;  // 16 KB
static constexpr int kBBytes = BN * BK * 2;  // 16 KB
static constexpr int kStageBytes = kABytes + kBBytes;
static constexpr int kGemmThreads = 3 * 128;  // two consumer warpgroups + one producer warpgroup
// setmaxnreg budget: 2 x 128 x 232 + 128 x 40 = 64512 <= the 65536 registers of an SM (one CTA per SM)
static constexpr int kConsumerRegs = 232;
static constexpr int kProducerRegs = 40;
static constexpr int kOrderBar = 1;  // named barriers 1, 2: "consumer warpgroup 0 / 1 may issue its mainloop"
static constexpr int kStoreBar = 3;  // named barriers 3, 4: the 128 threads of consumer warpgroup 0 / 1
static constexpr int kOutStageBytes = BM * BN * 2;  // 32 KB bf16 staging tile per consumer warpgroup
static constexpr int kSmemBytes = kStages * kStageBytes + 2 * kOutStageBytes + 1024 /*align*/ + 256 /*barriers*/;
static_assert(kSmemBytes <= 227 * 1024, "shared memory per block on sm_90");
// internal activation ids (not in the ABI): erf-GELU by the packed polynomial of common.cuh, and the
// activation read from GemmParams::act at run time (fp32 / residual outputs with an activation: rare)
static constexpr int kActGeluErfPoly = 100;
static constexpr int kActRuntime = 101;

struct GemmParams {
  int M, N, K;
  int act;                 // LN3_ACT_* (kActRuntime kernels only)
  const float* bias;       // [N] or null
  void* out;               // bf16 [M,ldo] or f32 [M,ldo] (for RESID: f32 residual, updated in place)
  long long ldo;           // leading dim of out, elements
  __nv_bfloat16* out2;     // optional bf16 copy of the updated residual (RESID only), ld = ldo2
  long long ldo2;
  const float* gate;       // RESID: gate[(m / gate_rows) * gate_ld + n]; null -> 1
  int gate_rows;
  long long gate_ld;
  const float* hn_w;       // per-head RMSNorm weights [nsec][64] (HN kernels only)
  int hn_nsec, hn_sec_cols;
  float hn_eps;
  int tma_store;           // bf16 output through the staging tile and tensor map (ldo % 8 == 0), else direct stores
  int n_first;             // tile walk: N first across the whole width, else M first inside each N panel
};

template <int ACT>
__device__ __forceinline__ void activate(float& a, float& b, int act) {
  if constexpr (ACT == kActRuntime) {
    switch (act) {
      case LN3_ACT_GELU_ERF: activate<LN3_ACT_GELU_ERF>(a, b, act); break;
      case LN3_ACT_GELU_TANH: activate<LN3_ACT_GELU_TANH>(a, b, act); break;
      case LN3_ACT_SILU: activate<LN3_ACT_SILU>(a, b, act); break;
      case LN3_ACT_QUICK_GELU: activate<LN3_ACT_QUICK_GELU>(a, b, act); break;
      default: break;
    }
  } else if constexpr (ACT == LN3_ACT_GELU_ERF) {
    a = gelu_erf_fast(a); b = gelu_erf_fast(b);
  } else if constexpr (ACT == kActGeluErfPoly) {
    gelu_erf_poly2(a, b);
  } else if constexpr (ACT == LN3_ACT_GELU_TANH) {
    a = gelu_tanh(a); b = gelu_tanh(b);
  } else if constexpr (ACT == LN3_ACT_SILU) {
    a = silu(a); b = silu(b);
  } else if constexpr (ACT == LN3_ACT_QUICK_GELU) {
    a = quick_gelu(a); b = quick_gelu(b);
  }
}

// Epilogue of one warpgroup's 64 x 128 accumulator.  wgmma layout: lane 4g + q of warp w holds rows
// 16 w + g (acc[4 i], acc[4 i + 1]) and 16 w + g + 8 (acc[4 i + 2], acc[4 i + 3]), columns 8 i + 2 q, +1.
// bf16 output goes to `stage_out` (row r_base + g of the tile) when it is set, else straight to global memory.
template <int ACT, int OUT, bool HN>
__device__ __forceinline__ void epilogue(const GemmParams& p, float* acc, int m_base, int n_base, int lane,
                                         uint8_t* stage_out, int r_base) {
  const int g = lane >> 2, q = lane & 3;
  if (p.bias != nullptr) {
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n_base + 8 * i + 2 * q));
      acc[4 * i] += b.x; acc[4 * i + 1] += b.y; acc[4 * i + 2] += b.x; acc[4 * i + 3] += b.y;
    }
  }
  if constexpr (HN) {
    // a 64-column head of one row lives in the 4 lanes of a quad (16 values each)
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
#pragma unroll
  for (int i = 0; i < BN / 4; ++i) activate<ACT>(acc[2 * i], acc[2 * i + 1], p.act);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int m = m_base + g + 8 * half;
    if (m >= p.M) continue;
    if constexpr (OUT == LN3_OUT_BF16) {
      if (stage_out != nullptr) {
        // staging tile: two 64-column halves of BM rows x 128 B in the 128B-swizzle layout of the output tensor
        // map (16-byte chunk c of row r at chunk c ^ (r & 7)); the 8 rows x 4 lanes of one store hit 32 banks
        const int r = r_base + g + 8 * half;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i)
          *reinterpret_cast<uint32_t*>(stage_out + (i >> 3) * (BM * 128) + r * 128 + (((i & 7) ^ (r & 7)) << 4) +
                                       4 * q) = pack_bf16x2(acc[4 * i + 2 * half], acc[4 * i + 2 * half + 1]);
        continue;
      }
      __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + m * p.ldo + n_base + 2 * q;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i)
        *reinterpret_cast<uint32_t*>(o + 8 * i) = pack_bf16x2(acc[4 * i + 2 * half], acc[4 * i + 2 * half + 1]);
    } else if constexpr (OUT == LN3_OUT_F32) {
      float* o = reinterpret_cast<float*>(p.out) + m * p.ldo + n_base + 2 * q;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i)
        *reinterpret_cast<float2*>(o + 8 * i) = make_float2(acc[4 * i + 2 * half], acc[4 * i + 2 * half + 1]);
    } else {  // LN3_OUT_RESID_F32: x[m,n] += gate * val  (+ bf16 copy of the new x)
      float* o = reinterpret_cast<float*>(p.out) + m * p.ldo + n_base + 2 * q;
      const float* gate_row =
          p.gate ? p.gate + static_cast<long long>(m / p.gate_rows) * p.gate_ld + n_base + 2 * q : nullptr;
      __nv_bfloat16* o2 = p.out2 ? p.out2 + m * p.ldo2 + n_base + 2 * q : nullptr;
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        float2 x = *reinterpret_cast<const float2*>(o + 8 * i);
        float2 gt = make_float2(1.f, 1.f);
        if (gate_row != nullptr) gt = __ldg(reinterpret_cast<const float2*>(gate_row + 8 * i));
        x.x = fmaf(gt.x, acc[4 * i + 2 * half], x.x);
        x.y = fmaf(gt.y, acc[4 * i + 2 * half + 1], x.y);
        *reinterpret_cast<float2*>(o + 8 * i) = x;
        if (o2 != nullptr) *reinterpret_cast<uint32_t*>(o2 + 8 * i) = pack_bf16x2(x.x, x.y);
      }
    }
  }
}

template <int ACT, int OUT, bool HN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                 const __grid_constant__ CUtensorMap tmap_o, const GemmParams p) {
  // Registers move to the consumers before any value is live: ptxas spills what is held across setmaxnreg.
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
  uint8_t* smem_out = smem + kStages * kStageBytes;                                // [2][kOutStageBytes]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem_out + 2 * kOutStageBytes);  // [kStages]
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
      mbar_init(&empty_bar[i], 1);  // released by the one consumer warpgroup that owns the tile
    }
    fence_barrier_init();
  }
  __syncthreads();

  // Tile order: consecutive CTAs walk M first inside an N panel, so the concurrently resident tiles share
  // W panels (L2 reuse) while A panels stream.  With p.n_first they walk N first across the whole width instead:
  // when A does not fit in the L2, each A panel is then read from memory once rather than once per N panel.
  auto tile_of = [&](int t, int& tm, int& tn) {
    if (p.n_first) {
      tm = t / tiles_n;
      tn = t % tiles_n;
    } else {
      tm = t % tiles_m;
      tn = t / tiles_m;
    }
  };
  if (warp >= 8) {
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
        int tm, tn;
        tile_of(t, tm, tn);
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

  // Ping-pong: warpgroup wg owns the CTA's tiles number wg, wg + 2, ... of its sequence, whole.  The ring holds
  // the k-blocks of consecutive tiles back to back, so each warpgroup steps over the other's num_kb slots.
  // Named barrier kOrderBar + wg hands the tensor core over: a warpgroup issues its mainloop only after the
  // other one has issued all of its own, so one warpgroup's epilogue runs under the other's MMAs.  The hand-over
  // also keeps the parity waits exact: a warpgroup starts at slot s only once every slot < s has completed, so
  // the full barrier of slot s is at most one phase behind and its parity cannot alias an older phase.
  const int wg = warp >> 2;
  const int grid = static_cast<int>(gridDim.x);
  const uint64_t a_desc0 = make_smem_desc_sw128(smem_u32(smem_a), 16, 1024);
  const uint64_t b_desc0 = make_smem_desc_sw128(smem_u32(smem_b), 16, 1024);
  uint32_t slot = wg * num_kb;  // ring position of this warpgroup's next k-block
  // bf16 output through this warpgroup's staging tile and TMA stores, when the output allows a tensor map
  const bool staged = OUT == LN3_OUT_BF16 && p.tma_store;
  const bool leader = (threadIdx.x & 127) == 0;
  uint8_t* stage_out = staged ? smem_out + wg * kOutStageBytes : nullptr;
  float acc0[BN / 2], acc1[BN / 2];  // rows [0, 64) and [64, 128) of the tile
  for (int t = blockIdx.x + wg * grid; t < num_tiles; t += 2 * grid) {
    int tm, tn;
    tile_of(t, tm, tn);
    if (t >= 2 * grid || wg == 1) named_bar_sync(kOrderBar + wg, 256);
    uint32_t stage = slot % kStages, phase = (slot / kStages) & 1;
    uint32_t prev_stage = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait_silent(&full_bar[stage], phase);
      const uint64_t da = a_desc0 + stage * (kABytes >> 4);
      const uint64_t db = b_desc0 + stage * (kBBytes >> 4);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint32_t acc_in = (kb | k) != 0 ? 1u : 0u;
        wgmma_m64n128k16_ss(acc0, da + 2 * k, db + 2 * k, acc_in);
        wgmma_m64n128k16_ss(acc1, da + ((64 * 128) >> 4) + 2 * k, db + 2 * k, acc_in);
      }
      wgmma_commit();
      // one MMA group stays in flight: the previous k-block's group is done, so its stage goes back to the producer
      wgmma_wait<1>();
      if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
    }
    if (t + grid < num_tiles) named_bar_arrive(kOrderBar + (wg ^ 1), 256);  // the other warpgroup's turn
    wgmma_wait<0>();
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty_bar[prev_stage]);
    slot += 2 * num_kb;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) {
      reg_fence(acc0[i]);
      reg_fence(acc1[i]);
    }
    const int m_base = tm * BM + (warp & 3) * 16;
    if (staged) {  // the previous tile's store has finished reading the staging buffer
      if (leader) tma_store_wait_read();
      named_bar_sync(kStoreBar + wg, 128);
    }
    epilogue<ACT, OUT, HN>(p, acc0, m_base, tn * BN, lane, stage_out, (warp & 3) * 16);
    epilogue<ACT, OUT, HN>(p, acc1, m_base + 64, tn * BN, lane, stage_out, 64 + (warp & 3) * 16);
    if (staged) {
      fence_proxy_async_smem();  // the generic-proxy writes become visible to the TMA engine
      named_bar_sync(kStoreBar + wg, 128);
      if (leader) {
        tma_store_2d(stage_out, &tmap_o, tn * BN, tm * BM);
        tma_store_2d(stage_out + BM * 128, &tmap_o, tn * BN + 64, tm * BM);
        tma_store_commit();
      }
    }
  }
  if (staged && leader) tma_store_wait_all();
}

// ---------------------------------------------------------------------------------- host
template <int ACT, int OUT, bool HN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const GemmParams& p,
                       cudaStream_t stream) {
  static DeviceOnce once;
  if (int rc = once.run([] {
        cudaError_t e = cudaFuncSetAttribute(gemm_bf16_kernel<ACT, OUT, HN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             kSmemBytes);
        return e == cudaSuccess ? LN3_OK : set_error(LN3_ECUDA, "gemm: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      }))
    return rc;
  const int tiles = ((p.M + BM - 1) / BM) * (p.N / BN);
  const int sms = device_sm_count();
  const int grid = tiles < sms ? tiles : sms;
  gemm_bf16_kernel<ACT, OUT, HN><<<grid, kGemmThreads, kSmemBytes, stream>>>(ta, tb, to, p);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "gemm launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

size_t gemm_workspace_bytes() { return 0; }

int gemm_bf16(const ln3_gemm_args* a, cudaStream_t stream) {
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return set_error(LN3_EINVAL, "gemm: empty problem");
  if (a->K % BK != 0) return set_error(LN3_EINVAL, "gemm: K=%d must be a multiple of %d", a->K, BK);
  if (a->N % BN != 0) return set_error(LN3_EINVAL, "gemm: N=%d must be a multiple of %d", a->N, BN);
  if (a->lda % 8 != 0 || a->ldw % 8 != 0)
    return set_error(LN3_EINVAL, "gemm: lda/ldw must be multiples of 8 elements (16 bytes)");
  if ((reinterpret_cast<uintptr_t>(a->A) | reinterpret_cast<uintptr_t>(a->W) |
       reinterpret_cast<uintptr_t>(a->out)) & 15)
    return set_error(LN3_EINVAL, "gemm: pointers must be 16-byte aligned");
  if (a->out_kind == LN3_OUT_RESID_F32 && a->gate != nullptr && a->gate_rows <= 0)
    return set_error(LN3_EINVAL, "gemm: gate_rows must be > 0");
  // the epilogue stores column pairs: 8-byte aligned rows for fp32, 4-byte for bf16
  {
    const size_t esz = (a->out_kind == LN3_OUT_BF16) ? 2 : 4;
    bool ok = (a->ldo % 2) == 0 && (reinterpret_cast<uintptr_t>(a->out) % (2 * esz)) == 0;
    if (a->out2 != nullptr) ok = ok && (a->ldo2 % 2) == 0 && (reinterpret_cast<uintptr_t>(a->out2) % 4) == 0;
    if (a->gate != nullptr) ok = ok && (a->gate_ld % 2) == 0 && (reinterpret_cast<uintptr_t>(a->gate) % 8) == 0;
    if (a->bias != nullptr) ok = ok && (reinterpret_cast<uintptr_t>(a->bias) % 8) == 0;
    if (!ok) return set_error(LN3_EINVAL, "gemm: out/out2/gate/bias rows must hold aligned column pairs");
  }
  CUtensorMap ta, tb;
  int rc = make_tmap_2d_bf16(&ta, a->A, a->M, a->K, a->lda, BM, BK);
  if (rc) return rc;
  rc = make_tmap_2d_bf16(&tb, a->W, a->N, a->K, a->ldw, BN, BK);
  if (rc) return rc;
  // bf16 output rows 16-byte aligned (out is, by the check above): TMA stores of 128-row x 64-column boxes that
  // clip rows >= M; any other pitch keeps the direct stores.  `to` is not read by the other kernels.
  CUtensorMap to = tb;
  const bool tma_store = a->out_kind == LN3_OUT_BF16 && a->ldo % 8 == 0;
  if (tma_store) {
    rc = make_tmap_2d_bf16(&to, a->out, a->M, a->N, a->ldo, BM, 64);
    if (rc) return rc;
  }

  GemmParams p;
  p.M = a->M;
  p.N = a->N;
  p.K = a->K;
  p.act = a->act;
  p.bias = a->bias;
  p.out = a->out;
  p.ldo = a->ldo;
  p.out2 = reinterpret_cast<__nv_bfloat16*>(a->out2);
  p.ldo2 = a->ldo2;
  p.gate = a->gate;
  p.gate_rows = a->gate_rows > 0 ? a->gate_rows : 1;
  p.gate_ld = a->gate_ld;
  p.hn_w = a->head_norm_w;
  p.hn_nsec = a->head_norm_nsec;
  p.hn_sec_cols = a->head_norm_sec_cols;
  p.hn_eps = a->head_norm_eps;
  p.tma_store = tma_store ? 1 : 0;
  // N-first walk when A does not fit in the L2 but W fits in half of it (the MLP's fc2: a 100 MB A, an 8 MB W)
  const long long l2 = device_l2_bytes();
  p.n_first = 2LL * a->M * a->K > l2 && 2LL * a->N * a->K <= l2 / 2;
  if (a->head_norm_w != nullptr) {
    if (a->out_kind != LN3_OUT_BF16 || a->act != LN3_ACT_NONE)
      return set_error(LN3_EINVAL, "gemm: head_norm needs LN3_OUT_BF16 and no activation");
    if (a->head_norm_nsec <= 0 || a->head_norm_sec_cols <= 0 || a->head_norm_sec_cols % kHnHead != 0)
      return set_error(LN3_EINVAL, "gemm: head_norm sections must be positive multiples of %d columns (the head width)", kHnHead);
    return launch_gemm<LN3_ACT_NONE, LN3_OUT_BF16, true>(ta, tb, to, p, stream);
  }
  if (a->act < LN3_ACT_NONE || a->act > LN3_ACT_QUICK_GELU) return set_error(LN3_EINVAL, "gemm: unknown activation %d", a->act);
  if (a->out_kind == LN3_OUT_RESID_F32) {
    if (a->act != LN3_ACT_NONE) return launch_gemm<kActRuntime, LN3_OUT_RESID_F32, false>(ta, tb, to, p, stream);
    return launch_gemm<LN3_ACT_NONE, LN3_OUT_RESID_F32, false>(ta, tb, to, p, stream);
  }
  if (a->out_kind == LN3_OUT_F32) {
    if (a->act != LN3_ACT_NONE) return launch_gemm<kActRuntime, LN3_OUT_F32, false>(ta, tb, to, p, stream);
    return launch_gemm<LN3_ACT_NONE, LN3_OUT_F32, false>(ta, tb, to, p, stream);
  }
  if (a->out_kind != LN3_OUT_BF16) return set_error(LN3_EINVAL, "gemm: unknown output kind %d", a->out_kind);
  switch (a->act) {
    case LN3_ACT_NONE: return launch_gemm<LN3_ACT_NONE, LN3_OUT_BF16, false>(ta, tb, to, p, stream);
    case LN3_ACT_GELU_ERF: return launch_gemm<kActGeluErfPoly, LN3_OUT_BF16, false>(ta, tb, to, p, stream);
    case LN3_ACT_GELU_TANH: return launch_gemm<LN3_ACT_GELU_TANH, LN3_OUT_BF16, false>(ta, tb, to, p, stream);
    case LN3_ACT_SILU: return launch_gemm<LN3_ACT_SILU, LN3_OUT_BF16, false>(ta, tb, to, p, stream);
    case LN3_ACT_QUICK_GELU: return launch_gemm<LN3_ACT_QUICK_GELU, LN3_OUT_BF16, false>(ta, tb, to, p, stream);
    default: return set_error(LN3_EINVAL, "gemm: unknown activation %d", a->act);
  }
}

}  // namespace ln3
