// Fused multi-head attention forward for sm_90a (head_dim 64 or 72, bf16 in, fp32 softmax / accumulate).
//
// Replaces xformers.ops.memory_efficient_attention at its three call sites on the path:
//   vit/vision_transformer.py:114-118 (DiT self-attention, (B, N, 3, H, 64) packed qkv),
//   ldm/modules/attention.py:279-307  (cross-attention; the reference's three permute+contiguous
//                                       copies disappear: heads are addressed through the TMA map),
//   dit/dit_decoder.py                (in-plane / global attention of the DiT2 VAE decoder).
// Semantics: out = softmax(q k^T * scale) v, optionally causal (key j visible to query i when j <= i), with an
// optional second K/V source appended after the first along the sequence.
//
// Persistent CTAs, one per SM, walk the 128-query-row tiles blockIdx.x, +gridDim.x, ... in (query tile, head,
// batch) order, so the CTAs that run at the same time share their (batch, head) K / V in L2.  The order is static
// (no tile counter), so a launch leaves no state behind and replays from a CUDA graph.
//   warpgroups 0, 1 : softmax / MMA warpgroups; warpgroup w owns query rows [64 w, 64 w + 64) of the tile.
//                     S = Q K^T with wgmma.m64n128k16 (Q and K from 128B-swizzled smem), online softmax in
//                     registers (a row lives in the 4 lanes of a quad), P converted in registers to the A
//                     fragments of O += P V (wgmma.m64n64k16, A from registers, V transposed from smem).
//   warp 8 lane 0   : TMA producer: each tile's Q, then its K / V blocks into a ring of kStages 128-key stages.  The
//                     ring runs on across tiles, and the next tile's Q loads as soon as both warpgroups have their
//                     last S of the current tile, so the next tile's loads hide under the last block and the stores.
// Pipeline of one warpgroup, per 128-key block j (live per thread: S, P_j and O):
//   issue S_{j+1} = Q K_{j+1}^T and O += P_j V_j as two commit groups; wait for S_{j+1} alone and run its softmax
//   while P_j V_j is on the tensor core; then wait for P_j V_j, release stage j, rescale O by alpha_{j+1} and
//   convert S_{j+1} to P_{j+1}.
// Ping-pong: named barriers 1 and 2 make the two warpgroups issue their MMA batches in strict alternation, so one
// warpgroup's softmax runs while the other's MMAs occupy the tensor core.
// Shared memory (148.7 KB, one CTA per SM): Q (16 KB) | K[kStages] (16 KB each) | V[kStages] | mbarriers.
// Head dim 72 (DiT-XL/2: 1152 / 16 heads) is the same kernel with an 8-column tail per operand, in unswizzled smem
// tiles of 16-byte rows beside the 64-column swizzled ones:
//   S: one more k16 step over head columns 64..79 of Q and K.  The TMA loads columns 64..71 (a box of exactly 8
//      columns, so it never reads the next head); columns 72..79 are a zero half written once per CTA and never
//      loaded, so they add exactly 0 to S.
//   P V: wgmma.m64n64k16 on V's first 64 columns as for head dim 64, plus wgmma.m64n8k16 on its 8-column tail
//      (2 KB per stage).  One m64n72k16 would need V's 72 columns in one MN-major operand, i.e. a second 16 KB
//      swizzle atom per stage holding 8 useful columns; n64 + n8 keeps the 64-column path as it is.
//   Shared memory: the tails add 4 KB (Q) + 4 stages x 6 KB (K 4 KB incl. its zero half, V 2 KB) = 28 KB, for
//   177.4 KB (177,408 B) in all.
// The head-dim-64 instantiation is compiled from the same source with the tail code removed at compile time.
// Every output element goes through the same instructions in the same order as in a sequential schedule (128-key
// blocks in order, the same wgmma shapes and k order, the same fp32 softmax sequence), so the result does not
// depend on the schedule.  The waits are the printf-free mbar_wait_silent: a function call in the kernel would
// make ptxas serialise every wgmma (C7510).
#include <cstdlib>

#include "common.cuh"
#include "ln3_internal.h"

namespace ln3 {

static constexpr int kQT = 128;   // query rows per tile
static constexpr int kKT = 128;   // keys per block
static constexpr int kSW = 64;    // head columns of the swizzled tiles (one 128-byte row)
static constexpr int kTileBytes = 128 * kSW * 2;  // 16 KB
static constexpr int kStages = 4;
static constexpr int kThreads = 2 * 128 + 32;
static constexpr int kOrderBar = 1;   // named barriers 1, 2: "warpgroup 0 / 1 may issue its next MMA batch"
// head dim 72: 8 tail columns per row, 16-byte rows, 128 rows per tile
static constexpr int kTail = 8;
static constexpr int kTailBytes = 128 * kTail * 2;   // 2 KB; Q and K tails are followed by a 2 KB zero half
static constexpr int kTailSmem = 2 * kTailBytes + kStages * 3 * kTailBytes;
// Q | K[kStages] | V[kStages] | (head dim 72: Qt | Kt[kStages] | Vt[kStages]) | barriers
template <int HD>
static constexpr int kFmhaSmem = 1024 + kTileBytes * (1 + 2 * kStages) + (HD > kSW ? kTailSmem : 0) + 256;

// The tails' tensor maps (head dim 72 only): 8-column boxes at head column 64, no swizzle.
template <int HD>
struct FmhaTailMaps {
  CUtensorMap q, k, v;
};
template <>
struct FmhaTailMaps<64> {};

struct FmhaParams {
  int Lq, Lkv, Lkv2;   // Lkv2: rows of the second K/V source (0 = none)
  int nb1, nb2;        // 128-key blocks of each source
  int H, n_qt;         // heads, query tiles per (batch, head)
  long long n_tiles;   // n_qt * H * B
  float scale_log2;    // softmax scale * log2(e)
  int causal;
  __nv_bfloat16* out;
  long long o_ld, o_bs;
};

struct Tile {
  int q0, h, b, nb1, nblocks;
};

__device__ __forceinline__ Tile decode_tile(const FmhaParams& p, long long t) {
  Tile d;
  const long long bh = t / p.n_qt;
  d.q0 = static_cast<int>(t - bh * p.n_qt) * kQT;
  d.h = static_cast<int>(bh % p.H);
  d.b = static_cast<int>(bh / p.H);
  // causal: blocks past the last query row of this tile are fully masked (first K/V source only)
  d.nb1 = p.causal ? min(p.nb1, (min(d.q0 + kQT, p.Lq) - 1) / kKT + 1) : p.nb1;
  d.nblocks = d.nb1 + p.nb2;
  return d;
}

// Online softmax of block j, in place on the raw scores s (s becomes 2^(s c - m)).  Per element: s c, the row max,
// ex2(v - m_use); l is scaled by alpha before the row's adds and summed per lane in key order, the first add of
// each row fused with the rescale (alpha l + e, as a sequential loop compiles it).  The intrinsics pin each
// rounding so that no reorganisation of the loop can contract a different pair.
__device__ __forceinline__ void softmax_block(const FmhaParams& p, float* s, float* m_run, float* l_run,
                                              float* alpha, int j, int nb1, int r0, int q) {
  const bool second = j >= nb1;
  const int kbase = (second ? j - nb1 : j) * kKT;
  const int klen = second ? p.Lkv2 : p.Lkv;
  // scale to log2 units, mask keys past the source's end (TMA zero-filled them) and, causally, keys > row
  const bool need_mask = kbase + kKT > klen || (p.causal && !second && kbase + kKT - 1 > r0);
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < kKT / 8; ++i) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float v = __fmul_rn(s[4 * i + e], p.scale_log2);
      if (need_mask) {
        const int key = kbase + 8 * i + 2 * q + (e & 1);
        const int row = r0 + 8 * (e >> 1);
        if (key >= klen || (p.causal && !second && key > row)) v = -INFINITY;
      }
      s[4 * i + e] = v;
      mx[e >> 1] = fmaxf(mx[e >> 1], v);
    }
  }
  float m_use[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    const float m_new = fmaxf(m_run[r], mx[r]);
    m_use[r] = m_new == -INFINITY ? 0.f : m_new;   // a row with no visible key yet
    alpha[r] = fast_exp2(__fsub_rn(m_run[r], m_use[r]));
    m_run[r] = m_new;
  }
  // slots 8 kk .. 8 kk + 7 are keys [16 kk, 16 kk + 16): slots 0, 1, 4, 5 row r0, slots 2, 3, 6, 7 row r0 + 8
#pragma unroll
  for (int kk = 0; kk < kKT / 16; ++kk) {
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int r = (t >> 1) & 1;
      const float e = fast_exp2(__fsub_rn(s[8 * kk + t], m_use[r]));
      s[8 * kk + t] = e;
      l_run[r] = (kk == 0 && (t == 0 || t == 2)) ? __fmaf_rn(alpha[r], l_run[r], e) : __fadd_rn(l_run[r], e);
    }
  }
}

// P = bf16(2^(s - m)) as the A fragments of P V: k-step kk covers keys [16 kk, 16 kk + 16)
__device__ __forceinline__ void pack_p(const float* s, uint32_t (*pa)[4]) {
#pragma unroll
  for (int kk = 0; kk < kKT / 16; ++kk) {
    pa[kk][0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
    pa[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
    pa[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
    pa[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
  }
}

// qt_desc / kt_desc: the head-dim-72 tail step (columns 64..79), unused for head dim 64
template <int HD>
__device__ __forceinline__ void issue_s(float* s, uint64_t q_desc, uint64_t k_desc, uint64_t qt_desc, uint64_t kt_desc) {
#pragma unroll
  for (int k = 0; k < kSW / 16; ++k) wgmma_m64n128k16_ss(s, q_desc + 2 * k, k_desc + 2 * k, k != 0 ? 1u : 0u);
  if constexpr (HD > kSW) wgmma_m64n128k16_ss(s, qt_desc, kt_desc, 1u);
  wgmma_commit();
}

// ot / vt_desc: the head-dim-72 tail columns 64..71 of O and V, unused for head dim 64
template <int HD>
__device__ __forceinline__ void issue_pv(float* o, float* ot, const uint32_t (*pa)[4], uint64_t v_desc,
                                         uint64_t vt_desc) {
#pragma unroll
  for (int kk = 0; kk < kKT / 16; ++kk) {
    wgmma_m64n64k16_rs_tb(o, pa[kk], v_desc + kk * 128, 1u);
    if constexpr (HD > kSW) wgmma_m64n8k16_rs_tb(ot, pa[kk], vt_desc + kk * ((16 * kTail * 2) >> 4), 1u);
  }
  wgmma_commit();
}

template <int HD>
__global__ void __launch_bounds__(kThreads, 1)
fmha_fwd_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                const __grid_constant__ CUtensorMap tmap_v, const __grid_constant__ CUtensorMap tmap_k2,
                const __grid_constant__ CUtensorMap tmap_v2, const FmhaParams p,
                const __grid_constant__ FmhaTailMaps<HD> tails) {
  constexpr bool kHasTail = HD > kSW;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kTileBytes;               // [kStages]
  uint8_t* sV = sK + kStages * kTileBytes;     // [kStages]
  uint8_t* sQt = sV + kStages * kTileBytes;       // head dim 72: [tail | zeros]
  uint8_t* sKt = sQt + 2 * kTailBytes;           // [kStages] x [tail | zeros]
  uint8_t* sVt = sKt + kStages * 2 * kTailBytes;  // [kStages]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + kStages * kTileBytes + (kHasTail ? kTailSmem : 0));
  uint64_t* q_full = bars;                     // [1]
  uint64_t* q_empty = bars + 1;                // [1], one arrival per warpgroup
  uint64_t* kv_full = bars + 2;                // [kStages]
  uint64_t* kv_empty = bars + 2 + kStages;     // [kStages], one arrival per warpgroup

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 2);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 2);
    }
    fence_barrier_init();
  }
  if constexpr (kHasTail) {
    // the zero halves (head columns 72..79) of the Q tail and of every K tail stage; the wgmma reads them through
    // the async proxy
    for (int i = threadIdx.x; i < (1 + kStages) * (kTailBytes / 16); i += kThreads) {
      const int tile = i / (kTailBytes / 16), off = (i % (kTailBytes / 16)) * 16;
      *reinterpret_cast<uint4*>(sQt + tile * 2 * kTailBytes + kTailBytes + off) = make_uint4(0, 0, 0, 0);
    }
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0, tcount = 0;
      for (long long t = blockIdx.x; t < p.n_tiles; t += gridDim.x, ++tcount) {
        const Tile d = decode_tile(p, t);
        mbar_wait_silent(q_empty, (tcount & 1) ^ 1);
        mbar_arrive_expect_tx(q_full, kTileBytes + (kHasTail ? kTailBytes : 0));
        tma_load_3d(sQ, &tmap_q, q_full, d.h * HD, d.q0, d.b);
        if constexpr (kHasTail) tma_load_3d(sQt, &tails.q, q_full, d.h * HD + kSW, d.q0, d.b);
        for (int j = 0; j < d.nblocks; ++j) {
          mbar_wait_silent(&kv_empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&kv_full[stage], 2 * kTileBytes + (kHasTail ? 2 * kTailBytes : 0));
          const bool second = j >= d.nb1;
          const int row = (second ? j - d.nb1 : j) * kKT;
          tma_load_3d(sK + stage * kTileBytes, second ? &tmap_k2 : &tmap_k, &kv_full[stage], d.h * HD, row, d.b);
          tma_load_3d(sV + stage * kTileBytes, second ? &tmap_v2 : &tmap_v, &kv_full[stage], d.h * HD, row, d.b);
          if constexpr (kHasTail) {   // head dim 72 has a single K/V source (host-checked)
            tma_load_3d(sKt + stage * 2 * kTailBytes, &tails.k, &kv_full[stage], d.h * HD + kSW, row, d.b);
            tma_load_3d(sVt + stage * kTailBytes, &tails.v, &kv_full[stage], d.h * HD + kSW, row, d.b);
          }
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
  const int g = lane >> 2, q = lane & 3;
  const bool leader = (threadIdx.x & 127) == 0;
  const uint64_t q_desc = make_smem_desc_sw128(smem_u32(sQ + wg * (64 * 128)), 16, 1024);
  const uint64_t k_desc0 = make_smem_desc_sw128(smem_u32(sK), 16, 1024);
  const uint64_t v_desc0 = make_smem_desc_sw128(smem_u32(sV), 16, 1024);
  // tails: K-major Q / K with the zero half one lbo (kTailBytes) past the loaded columns, 8-row groups 128 B apart;
  // MN-major V, 8 columns wide: 8-key groups 128 B apart (lbo = sbo, so either reading of the two fields holds)
  const uint64_t qt_desc = make_smem_desc_plain(smem_u32(sQt + wg * 64 * (kTail * 2)), kTailBytes, 128);
  const uint64_t kt_desc0 = make_smem_desc_plain(smem_u32(sKt), kTailBytes, 128);
  const uint64_t vt_desc0 = make_smem_desc_plain(smem_u32(sVt), 128, 128);

  // Ping-pong hand-over: a warpgroup issues an MMA batch once the other one has issued its previous batch.  Both
  // warpgroups issue nblocks + 1 batches per tile, so the alternation holds across tiles; warpgroup 0 skips the
  // wait before its first batch, and warpgroup 1 the hand-over after its last batch, which nobody waits for.
  bool first_batch = true;
  auto batch_begin = [&]() {
    if (wg == 1 || !first_batch) named_bar_sync(kOrderBar + wg, 256);
    first_batch = false;
  };
  auto batch_end = [&](bool last) {
    if (wg == 0 || !last) named_bar_arrive(kOrderBar + (wg ^ 1), 256);
  };

  int stage = 0;
  uint32_t phase = 0, tcount = 0;
  for (long long t = blockIdx.x; t < p.n_tiles; t += gridDim.x, ++tcount) {
    const Tile d = decode_tile(p, t);
    const bool last_tile = t + gridDim.x >= p.n_tiles;
    // query rows of this thread: r0 (accumulator slots 4i, 4i+1) and r0 + 8 (slots 4i+2, 4i+3)
    const int r0 = d.q0 + wg * 64 + (warp & 3) * 16 + g;
    float o[kSW / 2], ot[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < kSW / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, alpha[2];
    float s[kKT / 2];
    uint32_t pa[kKT / 16][4];

    // block 0: S_0 alone (O is still zero, so it needs no rescale)
    mbar_wait_silent(q_full, tcount & 1);
    mbar_wait_silent(&kv_full[stage], phase);
    batch_begin();
    wgmma_fence();
    issue_s<HD>(s, q_desc, k_desc0 + static_cast<uint32_t>(stage) * (kTileBytes >> 4), qt_desc,
                kt_desc0 + static_cast<uint32_t>(stage) * ((2 * kTailBytes) >> 4));
    batch_end(false);
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < kKT / 2; ++i) reg_fence(s[i]);
    if (d.nblocks == 1 && leader) mbar_arrive(q_empty);   // the tile's last S has read Q
    softmax_block(p, s, m_run, l_run, alpha, 0, d.nb1, r0, q);
    pack_p(s, pa);

    for (int j = 0; j + 1 < d.nblocks; ++j) {
      const int cur = stage;
      if (++stage == kStages) {
        stage = 0;
        phase ^= 1;
      }
      mbar_wait_silent(&kv_full[stage], phase);
      batch_begin();
      wgmma_fence();
      issue_s<HD>(s, q_desc, k_desc0 + static_cast<uint32_t>(stage) * (kTileBytes >> 4), qt_desc,
                  kt_desc0 + static_cast<uint32_t>(stage) * ((2 * kTailBytes) >> 4));
      issue_pv<HD>(o, ot, pa, v_desc0 + static_cast<uint32_t>(cur) * (kTileBytes >> 4),
                   vt_desc0 + static_cast<uint32_t>(cur) * (kTailBytes >> 4));
      batch_end(false);
      wgmma_wait<1>();   // S_{j+1} has landed; P_j V_j may still run
#pragma unroll
      for (int i = 0; i < kKT / 2; ++i) reg_fence(s[i]);
      if (j + 2 == d.nblocks && leader) mbar_arrive(q_empty);
      softmax_block(p, s, m_run, l_run, alpha, j + 1, d.nb1, r0, q);
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < kSW / 2; ++i) reg_fence(o[i]);
      if constexpr (kHasTail) {
#pragma unroll
        for (int i = 0; i < 4; ++i) reg_fence(ot[i]);
      }
      if (leader) mbar_arrive(&kv_empty[cur]);
#pragma unroll
      for (int i = 0; i < kSW / 8; ++i) {
        o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
        o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
      }
      if constexpr (kHasTail) {
        ot[0] *= alpha[0]; ot[1] *= alpha[0];
        ot[2] *= alpha[1]; ot[3] *= alpha[1];
      }
      pack_p(s, pa);
    }

    // last block: P V alone
    batch_begin();
    wgmma_fence();
    issue_pv<HD>(o, ot, pa, v_desc0 + static_cast<uint32_t>(stage) * (kTileBytes >> 4),
                 vt_desc0 + static_cast<uint32_t>(stage) * (kTailBytes >> 4));
    batch_end(last_tile);
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < kSW / 2; ++i) reg_fence(o[i]);
    if constexpr (kHasTail) {
#pragma unroll
      for (int i = 0; i < 4; ++i) reg_fence(ot[i]);
    }
    if (leader) mbar_arrive(&kv_empty[stage]);
    if (++stage == kStages) {
      stage = 0;
      phase ^= 1;
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
      __nv_bfloat16* dst = p.out + d.b * p.o_bs + row * p.o_ld + d.h * HD + 2 * q;
#pragma unroll
      for (int i = 0; i < kSW / 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + 8 * i) =
            pack_bf16x2(o[4 * i + 2 * r] * inv[r], o[4 * i + 2 * r + 1] * inv[r]);
      if constexpr (kHasTail)
        *reinterpret_cast<uint32_t*>(dst + kSW) = pack_bf16x2(ot[2 * r] * inv[r], ot[2 * r + 1] * inv[r]);
    }
  }
}

template <int HD>
static int fmha_launch(const ln3_fmha_args* a, bool two, cudaStream_t stream) {
  static DeviceOnce once;   // the shared-memory opt-in is per device
  if (int rc = once.run([] {
        cudaError_t e = cudaFuncSetAttribute(fmha_fwd_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             kFmhaSmem<HD>);
        return e == cudaSuccess ? LN3_OK : set_error(LN3_ECUDA, "fmha: cudaFuncSetAttribute: %s", cudaGetErrorString(e));
      }))
    return rc;
  CUtensorMap tq, tk, tv, tk2, tv2;
  FmhaTailMaps<HD> tails;
  int rc;
  const long long cols = static_cast<long long>(a->H) * HD;
  if ((rc = make_tmap_3d_bf16(&tq, a->q, cols, a->Lq, a->B, a->q_ld, a->q_bs, kSW, kQT))) return rc;
  if ((rc = make_tmap_3d_bf16(&tk, a->k, cols, a->Lkv, a->B, a->k_ld, a->k_bs, kSW, kKT))) return rc;
  if ((rc = make_tmap_3d_bf16(&tv, a->v, cols, a->Lkv, a->B, a->v_ld, a->v_bs, kSW, kKT))) return rc;
  if constexpr (HD > kSW) {
    if ((rc = make_tmap_3d_bf16(&tails.q, a->q, cols, a->Lq, a->B, a->q_ld, a->q_bs, kTail, kQT))) return rc;
    if ((rc = make_tmap_3d_bf16(&tails.k, a->k, cols, a->Lkv, a->B, a->k_ld, a->k_bs, kTail, kKT))) return rc;
    if ((rc = make_tmap_3d_bf16(&tails.v, a->v, cols, a->Lkv, a->B, a->v_ld, a->v_bs, kTail, kKT))) return rc;
  }
  if (two) {
    if ((rc = make_tmap_3d_bf16(&tk2, a->k2, cols, a->Lkv2, a->B, a->k2_ld, a->k2_bs, kSW, kKT))) return rc;
    if ((rc = make_tmap_3d_bf16(&tv2, a->v2, cols, a->Lkv2, a->B, a->v2_ld, a->v2_bs, kSW, kKT))) return rc;
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
  p.H = a->H;
  p.n_qt = (a->Lq + kQT - 1) / kQT;
  p.n_tiles = static_cast<long long>(p.n_qt) * a->H * a->B;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.causal = a->causal ? 1 : 0;
  p.out = reinterpret_cast<__nv_bfloat16*>(a->out);
  p.o_ld = a->o_ld;
  p.o_bs = a->o_bs;
  const int sms = device_sm_count();
  const int grid = p.n_tiles < sms ? static_cast<int>(p.n_tiles) : sms;
  fmha_fwd_kernel<HD><<<grid, kThreads, kFmhaSmem<HD>, stream>>>(tq, tk, tv, tk2, tv2, p, tails);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "fmha launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

int fmha_fwd(const ln3_fmha_args* a, cudaStream_t stream) {
  if (a->head_dim != 64 && a->head_dim != 72) return set_error(LN3_EUNSUPPORTED, "fmha: head_dim must be 64 or 72");
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
    if (a->head_dim != 64) return set_error(LN3_EUNSUPPORTED, "fmha: a second K/V source needs head_dim 64");
    if (!a->k2 || !a->v2 || a->Lkv2 <= 0) return set_error(LN3_EINVAL, "fmha: k2/v2/Lkv2 must be given together");
    if ((a->k2_ld | a->v2_ld | a->k2_bs | a->v2_bs) % 8 ||
        ((reinterpret_cast<uintptr_t>(a->k2) | reinterpret_cast<uintptr_t>(a->v2)) & 15))
      return set_error(LN3_EINVAL, "fmha: k2/v2 alignment");
  }
  if (a->B > 65535 || a->H > 65535) return set_error(LN3_EUNSUPPORTED, "fmha: batch or head count above 65535");
  return a->head_dim == 64 ? fmha_launch<64>(a, two, stream) : fmha_launch<72>(a, two, stream);
}

}  // namespace ln3
