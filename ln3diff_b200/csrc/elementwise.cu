// HBM-bound glue kernels of the DiT / sampler path (fp32 SIMT, vectorised, coalesced):
//   norm_modulate      LayerNorm/RMSNorm + adaLN modulate -> bf16 GEMM operand (or e4m3 + block scales: _fp8)
//   quantize_fp8_rows  fp32 / bf16 rows -> e4m3 codes + 1 x 128 block scales
//   timestep_embedding sinusoidal features of the timestep
//   patch_embed        roll-out rearrange + 2x2 patch conv + pos_embed -> fp32 token stream
//   final_layer        LN + modulate + Linear(D -> 4*Cout) + unpatchify -> fp32 latent layout
//   sampler_update     x' = a x + w0 m0 + w1 m1 + s noise (all sampler engines, one launch/step)
// Reference call sites are cited per kernel in include/ln3b200.h.
#include <cstdlib>

#include "common.cuh"
#include "ln3_internal.h"

namespace ln3 {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == LN3_ACT_SILU) return silu(v);
  if (act == LN3_ACT_GELU_ERF) return gelu_erf(v);
  if (act == LN3_ACT_GELU_TANH) return gelu_tanh(v);
  return v;
}

// ------------------------------------------------------------------ norm + modulate
// One warp per row; the row lives in registers (NV float4 per lane, D = 128 * NV).
template <int NV>
__global__ void __launch_bounds__(256)
norm_modulate_kernel(const ln3_norm_modulate_args a) {
  const int lane = threadIdx.x & 31;
  // grid-stride over rows: the host sizes the grid to one resident wave, so there is no partial last wave
  for (int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < a.rows;
       row += gridDim.x * (blockDim.x >> 5)) {
  const float* x = a.x + static_cast<long long>(row) * a.ldx;
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = *reinterpret_cast<const float4*>(x + (i * 32 + lane) * 4);
  if (a.resid != nullptr) {
    // fused residual update: x += gate * resid (bf16), written back in place
    const __nv_bfloat16* rr = reinterpret_cast<const __nv_bfloat16*>(a.resid) + static_cast<long long>(row) * a.resid_ld;
    const __nv_bfloat16* r2 = nullptr;   // outside rows with resid_out_gate: own resid row first, then the bcast row
    const float* g2 = nullptr;
    if (a.resid_bcast != nullptr && (row < a.resid_row_begin || row >= a.resid_row_end)) {
      if (a.resid_out_gate != nullptr) {
        r2 = rr;
        g2 = a.resid_out_gate + static_cast<long long>(row / a.resid_out_gate_rows) * a.resid_out_gate_ld;
      }
      rr = reinterpret_cast<const __nv_bfloat16*>(a.resid_bcast) + static_cast<long long>(row / a.resid_bcast_rows) * a.resid_bcast_ld;
    }
    const float* gg = a.resid_gate ? a.resid_gate + static_cast<long long>(row / a.resid_gate_rows) * a.resid_gate_ld : nullptr;
    float* xw = const_cast<float*>(x);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 32 + lane) * 4;
      if (r2 != nullptr) {
        const uint2 qb = *reinterpret_cast<const uint2*>(r2 + c);
        const __nv_bfloat162 q01 = *reinterpret_cast<const __nv_bfloat162*>(&qb.x);
        const __nv_bfloat162 q23 = *reinterpret_cast<const __nv_bfloat162*>(&qb.y);
        const float4 h = __ldg(reinterpret_cast<const float4*>(g2 + c));
        v[i].x = fmaf(h.x, __low2float(q01), v[i].x);
        v[i].y = fmaf(h.y, __high2float(q01), v[i].y);
        v[i].z = fmaf(h.z, __low2float(q23), v[i].z);
        v[i].w = fmaf(h.w, __high2float(q23), v[i].w);
      }
      const uint2 rb = *reinterpret_cast<const uint2*>(rr + c);
      const __nv_bfloat162 r01 = *reinterpret_cast<const __nv_bfloat162*>(&rb.x);
      const __nv_bfloat162 r23 = *reinterpret_cast<const __nv_bfloat162*>(&rb.y);
      float4 g = make_float4(1.f, 1.f, 1.f, 1.f);
      if (gg != nullptr && r2 == nullptr) g = __ldg(reinterpret_cast<const float4*>(gg + c));
      v[i].x = fmaf(g.x, __low2float(r01), v[i].x);
      v[i].y = fmaf(g.y, __high2float(r01), v[i].y);
      v[i].z = fmaf(g.z, __low2float(r23), v[i].z);
      v[i].w = fmaf(g.w, __high2float(r23), v[i].w);
      *reinterpret_cast<float4*>(xw + c) = v[i];
    }
    if (a.out == nullptr) continue;
  }

  float mean = 0.f, rstd = 1.f;
  if (a.norm == LN3_NORM_LAYER) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    mean = warp_sum(s) / static_cast<float>(a.D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
      q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
    rstd = rsqrtf(warp_sum(q) / static_cast<float>(a.D) + a.eps);
  } else if (a.norm == LN3_NORM_RMS) {
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      q += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
    rstd = rsqrtf(warp_sum(q) / static_cast<float>(a.D) + a.eps);
  }
  const float* sh = nullptr;
  const float* sc = nullptr;
  if (a.shift != nullptr) {
    const long long g = row / a.mod_rows;
    sh = a.shift + g * a.mod_ld;
    sc = a.scale + g * a.mod_ld;
  }
  __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(a.out) + static_cast<long long>(row) * a.ldo;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    float4 y = make_float4((v[i].x - mean) * rstd, (v[i].y - mean) * rstd, (v[i].z - mean) * rstd,
                           (v[i].w - mean) * rstd);
    if (a.weight != nullptr) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(a.weight + c));
      y.x *= w.x; y.y *= w.y; y.z *= w.z; y.w *= w.w;
    }
    if (sh != nullptr) {
      float4 s1 = __ldg(reinterpret_cast<const float4*>(sc + c));
      float4 s0 = __ldg(reinterpret_cast<const float4*>(sh + c));
      if (a.scale_tab != nullptr) {
        const float4 t1 = __ldg(reinterpret_cast<const float4*>(a.scale_tab + c));
        const float4 t0 = __ldg(reinterpret_cast<const float4*>(a.shift_tab + c));
        s1.x += t1.x; s1.y += t1.y; s1.z += t1.z; s1.w += t1.w;
        s0.x += t0.x; s0.y += t0.y; s0.z += t0.z; s0.w += t0.w;
      }
      y.x = fmaf(y.x, 1.f + s1.x, s0.x);
      y.y = fmaf(y.y, 1.f + s1.y, s0.y);
      y.z = fmaf(y.z, 1.f + s1.z, s0.z);
      y.w = fmaf(y.w, 1.f + s1.w, s0.w);
    }
    if (a.act != LN3_ACT_NONE) {
      y.x = apply_act(y.x, a.act); y.y = apply_act(y.y, a.act);
      y.z = apply_act(y.z, a.act); y.w = apply_act(y.w, a.act);
    }
    uint2 pk;
    pk.x = pack_bf16x2(y.x, y.y);
    pk.y = pack_bf16x2(y.z, y.w);
    *reinterpret_cast<uint2*>(o + c) = pk;
  }
  }  // row loop
}

// ---- 256-bit kernels (D % 256 == 0, 32-byte aligned rows: every DiT / DiT2 call) -------------------------
// A lane owns NV8 chunks of 8 consecutive columns: the fp32 row moves as 256-bit accesses and the bf16 rows as
// 128-bit accesses.  nm_row_body is the arithmetic of one row; same operations in the same order per element as
// the float4 kernel above.
//   v      the row of x (registers)
//   rown   this row's own residual row resid[row] (bf16, one uint4 per chunk), meaningful iff nm_needs_own_row()
__device__ __forceinline__ bool nm_outside(const ln3_norm_modulate_args& a, int row) {
  return a.resid_bcast != nullptr && (row < a.resid_row_begin || row >= a.resid_row_end);
}
__device__ __forceinline__ bool nm_needs_own_row(const ln3_norm_modulate_args& a, int row) {
  return a.resid != nullptr && (!nm_outside(a, row) || a.resid_out_gate != nullptr);
}

// LN3_RESID_L2=1: residual-stream accesses carry the L2 evict_last priority (set once per process).  The branches
// on it also shape ptxas's register allocation: without them the D = 1024 kernel spills at its 80-register cap.
__constant__ int c_nm_l2_hint;

// Outputs of the row body: `enabled()` is false for a residual-only pass; `store(row, lane, c, y)` writes the 8
// normalised values of columns [c, c + 8), called by all 32 lanes for the same chunk index.
struct NmOutBf16 {
  void* out;
  long long ldo;
  __device__ __forceinline__ bool enabled() const { return out != nullptr; }
  __device__ __forceinline__ void store(int row, int, int c, const float (&y)[8]) const {
    uint4 pk;
    pk.x = pack_bf16x2(y[0], y[1]);
    pk.y = pack_bf16x2(y[2], y[3]);
    pk.z = pack_bf16x2(y[4], y[5]);
    pk.w = pack_bf16x2(y[6], y[7]);
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(out) + static_cast<long long>(row) * ldo + c) = pk;
  }
};
// e4m3 codes + 1 x 128 block scales (include/ln3b200.h): a 128-column block is chunk i of 16 consecutive lanes
struct NmOutFp8 {
  void* out;
  float* out_scale;
  long long ldo, out_scale_ld;
  __device__ __forceinline__ bool enabled() const { return true; }
  __device__ __forceinline__ void store(int row, int lane, int c, const float (&y)[8]) const {
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) amax = fmaxf(amax, fabsf(y[j]));
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float s = fp8_block_scale(amax);
    uint2 pk;
    pk.x = fp8_code2(y[0], y[1], s) | (static_cast<uint32_t>(fp8_code2(y[2], y[3], s)) << 16);
    pk.y = fp8_code2(y[4], y[5], s) | (static_cast<uint32_t>(fp8_code2(y[6], y[7], s)) << 16);
    *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(out) + static_cast<long long>(row) * ldo + c) = pk;
    if ((lane & 15) == 0) out_scale[static_cast<long long>(row) * out_scale_ld + c / 128] = s;
  }
};

template <int NV8, class Out>
__device__ __forceinline__ void nm_row_body(const ln3_norm_modulate_args& a, int row, int lane, float (&v)[NV8][8],
                                            const uint4 (&rown)[NV8], const Out& out) {
  float* x = const_cast<float*>(a.x) + static_cast<long long>(row) * a.ldx;
  auto ld8 = [&](const float* p8, float* d8) {
    const float4 p0 = __ldg(reinterpret_cast<const float4*>(p8));
    const float4 p1 = __ldg(reinterpret_cast<const float4*>(p8 + 4));
    d8[0] = p0.x, d8[1] = p0.y, d8[2] = p0.z, d8[3] = p0.w, d8[4] = p1.x, d8[5] = p1.y, d8[6] = p1.z, d8[7] = p1.w;
  };
  auto axpy8 = [&](float* acc, const float* g8, const uint4& rb) {
    const uint32_t rw[4] = {rb.x, rb.y, rb.z, rb.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const __nv_bfloat162 r2 = *reinterpret_cast<const __nv_bfloat162*>(&rw[j]);
      acc[2 * j] = fmaf(g8[2 * j], __low2float(r2), acc[2 * j]);
      acc[2 * j + 1] = fmaf(g8[2 * j + 1], __high2float(r2), acc[2 * j + 1]);
    }
  };
  if (a.resid != nullptr) {
    const bool outside = nm_outside(a, row);
    const bool own = !outside || a.resid_out_gate != nullptr;
    // gate of the own row: resid_gate inside, resid_out_gate outside
    const float* g_own = nullptr;
    if (!outside) {
      if (a.resid_gate) g_own = a.resid_gate + static_cast<long long>(row / a.resid_gate_rows) * a.resid_gate_ld;
    } else if (a.resid_out_gate) {
      g_own = a.resid_out_gate + static_cast<long long>(row / a.resid_out_gate_rows) * a.resid_out_gate_ld;
    }
    // outside rows: the per-group broadcast row, gated by resid_gate unless the own row took a gate of its own
    const __nv_bfloat16* rb = nullptr;
    const float* g_b = nullptr;
    if (outside) {
      rb = reinterpret_cast<const __nv_bfloat16*>(a.resid_bcast) + static_cast<long long>(row / a.resid_bcast_rows) * a.resid_bcast_ld;
      if (a.resid_out_gate == nullptr && a.resid_gate)
        g_b = a.resid_gate + static_cast<long long>(row / a.resid_gate_rows) * a.resid_gate_ld;
    }
#pragma unroll
    for (int i = 0; i < NV8; ++i) {
      const int c = (i * 32 + lane) * 8;
      float g[8] = {1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f};
      if (own) {
        if (g_own != nullptr) ld8(g_own + c, g);
        axpy8(v[i], g, rown[i]);
      }
      if (rb != nullptr) {
        float gb[8] = {1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f};
        if (g_b != nullptr) ld8(g_b + c, gb);
        axpy8(v[i], gb, *reinterpret_cast<const uint4*>(rb + c));
      }
      if (c_nm_l2_hint) stg256_f32_el(x + c, v[i]);
      else stg256_f32(x + c, v[i]);
    }
    if (!out.enabled()) return;
  }
  float mean = 0.f, rstd = 1.f;
  if (a.norm == LN3_NORM_LAYER) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV8; ++i)  // same pairing as the float4 kernel: ((a+b)+(c+d)) per 4 columns
      s += ((v[i][0] + v[i][1]) + (v[i][2] + v[i][3])) + ((v[i][4] + v[i][5]) + (v[i][6] + v[i][7]));
    mean = warp_sum(s) / static_cast<float>(a.D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float dlt = v[i][j] - mean;
        q = fmaf(dlt, dlt, q);
      }
    rstd = rsqrtf(warp_sum(q) / static_cast<float>(a.D) + a.eps);
  } else if (a.norm == LN3_NORM_RMS) {
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) q = fmaf(v[i][j], v[i][j], q);
    rstd = rsqrtf(warp_sum(q) / static_cast<float>(a.D) + a.eps);
  }
  const float* sh = nullptr;
  const float* sc = nullptr;
  if (a.shift != nullptr) {
    const long long g = row / a.mod_rows;
    sh = a.shift + g * a.mod_ld;
    sc = a.scale + g * a.mod_ld;
  }
#pragma unroll
  for (int i = 0; i < NV8; ++i) {
    const int c = (i * 32 + lane) * 8;
    float y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = (v[i][j] - mean) * rstd;
    if (a.weight != nullptr) {
      float w[8];
      ld8(a.weight + c, w);
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] *= w[j];
    }
    if (sh != nullptr) {
      float s1[8], s0[8];
      ld8(sc + c, s1);
      ld8(sh + c, s0);
      if (a.scale_tab != nullptr) {
        float t1[8], t0[8];
        ld8(a.scale_tab + c, t1);
        ld8(a.shift_tab + c, t0);
#pragma unroll
        for (int j = 0; j < 8; ++j) s1[j] += t1[j], s0[j] += t0[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = fmaf(y[j], 1.f + s1[j], s0[j]);
    }
    if (a.act != LN3_ACT_NONE) {
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = apply_act(y[j], a.act);
    }
    out.store(row, lane, c, y);
  }
}

// Warp per row straight from global memory.  (A software-pipelined variant -- next row's loads issued before the
// current row's arithmetic, 2 CTAs/SM at 128 registers -- measured slower: 36.9 vs 32.8 us; so did a shared-memory
// staged kernel fed by bulk copies, 48 vs 36 us.  Occupancy at <= 80 registers beats explicit prefetch here.)
template <int NV8>
__device__ __forceinline__ void nm_load_row(const ln3_norm_modulate_args& a, int row, int lane, float (&v)[NV8][8],
                                            uint4 (&rown)[NV8]) {
  const float* x = a.x + static_cast<long long>(row) * a.ldx;
  if (c_nm_l2_hint) {
#pragma unroll
    for (int i = 0; i < NV8; ++i) ldg256_na_el(x + (i * 32 + lane) * 8, v[i]);
  } else {
#pragma unroll
    for (int i = 0; i < NV8; ++i) ldg256_na(x + (i * 32 + lane) * 8, v[i]);
  }
  if (nm_needs_own_row(a, row)) {
    const __nv_bfloat16* rr = reinterpret_cast<const __nv_bfloat16*>(a.resid) + static_cast<long long>(row) * a.resid_ld;
#pragma unroll
    for (int i = 0; i < NV8; ++i) rown[i] = *reinterpret_cast<const uint4*>(rr + (i * 32 + lane) * 8);
  } else {
#pragma unroll
    for (int i = 0; i < NV8; ++i) rown[i] = make_uint4(0, 0, 0, 0);
  }
}

template <int NV8, class Out>
__global__ void __launch_bounds__(256, 3)
norm_modulate_wide_kernel(const ln3_norm_modulate_args a, const Out out) {
  const int lane = threadIdx.x & 31;
  // A CTA owns a contiguous run of rows (not a grid-stride comb): consecutive token rows share their sample's
  // shift / scale / gate vectors, which then stay in L1 instead of every SM cycling through all samples' vectors
  // (LN + residual pass 36-38 -> 32.8 us at DiT-L/2 B'=16).
  const int per_cta = (a.rows + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const int row_begin = static_cast<int>(blockIdx.x) * per_cta;
  const int row_end = min(a.rows, row_begin + per_cta);
  for (int row = row_begin + (threadIdx.x >> 5); row < row_end; row += (blockDim.x >> 5)) {
    float v[NV8][8];
    uint4 rown[NV8];
    nm_load_row<NV8>(a, row, lane, v, rown);
    nm_row_body<NV8>(a, row, lane, v, rown, out);
  }
}

// Every pointer the glue kernels read or write with 128-bit (or 64-bit) accesses must be 16-byte aligned: a
// column-offset view such as mod[:, 1:1+D] would otherwise pass the shape checks and issue misaligned loads.
static bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

// Argument checks of the norm_modulate entry points; `out` / `ldo` are the output this call writes.
static int nm_check(const ln3_norm_modulate_args* a, const void* out, long long ldo) {
  if (a->D % 128 != 0 || a->D > 2048 || a->D <= 0)
    return set_error(LN3_EINVAL, "norm_modulate: D=%d must be a multiple of 128, <= 2048", a->D);
  if ((a->shift == nullptr) != (a->scale == nullptr))
    return set_error(LN3_EINVAL, "norm_modulate: shift and scale must be given together");
  if ((a->shift_tab == nullptr) != (a->scale_tab == nullptr))
    return set_error(LN3_EINVAL, "norm_modulate: shift_tab and scale_tab must be given together");
  if (a->shift != nullptr && a->mod_rows <= 0)
    return set_error(LN3_EINVAL, "norm_modulate: mod_rows must be > 0");
  if (a->ldx % 4 || ldo % 4 || (a->shift && a->mod_ld % 4))
    return set_error(LN3_EINVAL, "norm_modulate: leading dimensions must be multiples of 4");
  if (out == nullptr && a->resid == nullptr) return set_error(LN3_EINVAL, "norm_modulate: out is NULL");
  // out and resid need only 8 bytes in the float4 kernel and 16 in the 256-bit one: one rule, the stricter
  if (misaligned16(a->x) || misaligned16(out) || misaligned16(a->shift) || misaligned16(a->scale) ||
      misaligned16(a->shift_tab) || misaligned16(a->scale_tab) || misaligned16(a->weight) || misaligned16(a->resid) ||
      misaligned16(a->resid_gate) || misaligned16(a->resid_bcast) || misaligned16(a->resid_out_gate))
    return set_error(LN3_EINVAL, "norm_modulate: x, out, shift, scale, tables, weight, resid, resid_bcast and gates must be 16-byte aligned");
  if (a->resid != nullptr) {
    if (a->resid_ld % 4) return set_error(LN3_EINVAL, "norm_modulate: resid_ld must be a multiple of 4");
    if (a->resid_gate != nullptr && (a->resid_gate_rows <= 0 || a->resid_gate_ld % 4))
      return set_error(LN3_EINVAL, "norm_modulate: bad resid_gate_rows / resid_gate_ld");
    if (a->resid_bcast != nullptr &&
        (a->resid_bcast_rows <= 0 || a->resid_bcast_ld % 8 ||
         a->resid_row_begin < 0 || a->resid_row_end < a->resid_row_begin || a->resid_row_end > a->rows))
      return set_error(LN3_EINVAL, "norm_modulate: bad resid_bcast arguments");
    if (a->resid_out_gate != nullptr &&
        (a->resid_bcast == nullptr || a->resid_out_gate_rows <= 0 || a->resid_out_gate_ld % 4))
      return set_error(LN3_EINVAL, "norm_modulate: resid_out_gate needs resid_bcast, rows > 0 and ld %% 4 == 0");
  } else if (a->resid_bcast != nullptr) {
    return set_error(LN3_EINVAL, "norm_modulate: resid_bcast needs resid");
  }
  return LN3_OK;
}

// x, ldx and resid as the 256-bit kernels need them (D itself is checked by the caller)
static bool nm_wide_input(const ln3_norm_modulate_args* a) {
  return a->ldx % 8 == 0 && (reinterpret_cast<uintptr_t>(a->x) & 31) == 0 &&
         (a->resid == nullptr || (a->resid_ld % 8 == 0 && (reinterpret_cast<uintptr_t>(a->resid) & 15) == 0));
}

static int nm_l2_hint_once() {  // LN3_RESID_L2=1: evict_last hints on the residual stream (uploaded once per device)
  static DeviceOnce l2_once;
  return l2_once.run([] {
    const int v = (getenv("LN3_RESID_L2") && atoi(getenv("LN3_RESID_L2")) != 0) ? 1 : 0;
    cudaError_t e = cudaMemcpyToSymbol(c_nm_l2_hint, &v, sizeof(v));
    return e == cudaSuccess ? LN3_OK : set_error(LN3_ECUDA, "norm_modulate: constant upload: %s", cudaGetErrorString(e));
  });
}

static constexpr int kNmWarps = 8;

template <class Out>
static int nm_launch_wide(const ln3_norm_modulate_args* a, const Out& out, cudaStream_t stream) {
  const int blocks_needed = (a->rows + kNmWarps - 1) / kNmWarps;
  const int wave3 = device_sm_count() * 3;  // 3 resident blocks per SM at <= 80 registers
  const dim3 grid(blocks_needed < wave3 ? blocks_needed : wave3), block(kNmWarps * 32);
  switch (a->D / 256) {
    case 1: norm_modulate_wide_kernel<1, Out><<<grid, block, 0, stream>>>(*a, out); break;
    case 2: norm_modulate_wide_kernel<2, Out><<<grid, block, 0, stream>>>(*a, out); break;
    case 3: norm_modulate_wide_kernel<3, Out><<<grid, block, 0, stream>>>(*a, out); break;
    case 4: norm_modulate_wide_kernel<4, Out><<<grid, block, 0, stream>>>(*a, out); break;
    case 5: norm_modulate_wide_kernel<5, Out><<<grid, block, 0, stream>>>(*a, out); break;
    default: norm_modulate_wide_kernel<6, Out><<<grid, block, 0, stream>>>(*a, out); break;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "norm_modulate launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

int norm_modulate(const ln3_norm_modulate_args* a, cudaStream_t stream) {
  if (a->rows <= 0) return LN3_OK;
  if (int rc = nm_check(a, a->out, a->ldo)) return rc;
  const int blocks_needed = (a->rows + kNmWarps - 1) / kNmWarps;
  const int wave = device_sm_count() * 4;  // 4 x 256-thread blocks resident per SM (<= 64 regs/thread)
  dim3 grid(blocks_needed < wave ? blocks_needed : wave), block(kNmWarps * 32);
  const bool wide = a->D % 256 == 0 && a->D <= 1536 && a->ldo % 8 == 0 && nm_wide_input(a) &&
                    (a->out == nullptr || (reinterpret_cast<uintptr_t>(a->out) & 15) == 0);
  if (int rc = nm_l2_hint_once()) return rc;
  if (wide) return nm_launch_wide(a, NmOutBf16{a->out, a->ldo}, stream);
  switch (a->D / 128) {
#define LN3_NM_CASE(n) \
  case n: norm_modulate_kernel<n><<<grid, block, 0, stream>>>(*a); break;
    LN3_NM_CASE(1) LN3_NM_CASE(2) LN3_NM_CASE(3) LN3_NM_CASE(4) LN3_NM_CASE(5) LN3_NM_CASE(6)
    LN3_NM_CASE(7) LN3_NM_CASE(8) LN3_NM_CASE(9) LN3_NM_CASE(10) LN3_NM_CASE(11) LN3_NM_CASE(12)
    LN3_NM_CASE(13) LN3_NM_CASE(14) LN3_NM_CASE(15) LN3_NM_CASE(16)
#undef LN3_NM_CASE
    default: return set_error(LN3_EINVAL, "norm_modulate: unsupported D");
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "norm_modulate launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// The fp8 output exists for the 256-bit kernels only (every DiT-L/2 and DiT-B/2 width); other shapes are refused.
int norm_modulate_fp8(const ln3_norm_modulate_fp8_args* f, cudaStream_t stream) {
  const ln3_norm_modulate_args* a = &f->base;
  if (a->out != nullptr) return set_error(LN3_EINVAL, "norm_modulate_fp8: base.out must be NULL (the output is out)");
  if (f->out == nullptr || f->out_scale == nullptr)
    return set_error(LN3_EINVAL, "norm_modulate_fp8: out and out_scale must be given");
  if (a->rows <= 0) return LN3_OK;
  if (int rc = nm_check(a, f->out, f->ldo)) return rc;
  if (f->ldo < a->D || f->ldo % 16 != 0 || f->out_scale_ld < a->D / 128)
    return set_error(LN3_EINVAL, "norm_modulate_fp8: ldo must be >= D and a multiple of 16, out_scale_ld >= D/128");
  if (a->D % 256 != 0 || a->D > 1536 || !nm_wide_input(a))
    return set_error(LN3_EUNSUPPORTED,
                     "norm_modulate_fp8: needs D %% 256 == 0, D <= 1536, ldx %% 8 == 0, x 32-byte aligned and "
                     "resid_ld %% 8 == 0 (D=%d)", a->D);
  if (int rc = nm_l2_hint_once()) return rc;
  return nm_launch_wide(a, NmOutFp8{f->out, f->out_scale, f->ldo, f->out_scale_ld}, stream);
}

// ------------------------------------------------------------------ fp8 block quantisation
// One warp per 128-column block of a row: 4 consecutive values per lane, the absmax over the warp.
template <typename T>
__global__ void __launch_bounds__(256)
quantize_fp8_kernel(const T* __restrict__ x, long long ldx, int rows, int nblk, uint8_t* __restrict__ out,
                    long long ldo, float* __restrict__ out_scale, long long out_scale_ld) {
  const long long w = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= static_cast<long long>(rows) * nblk) return;
  const int lane = threadIdx.x & 31;
  const int row = static_cast<int>(w / nblk), c = static_cast<int>(w % nblk) * 128 + lane * 4;
  float v[4];
  if constexpr (sizeof(T) == 4) {
    const float4 t = *reinterpret_cast<const float4*>(x + row * ldx + c);
    v[0] = t.x, v[1] = t.y, v[2] = t.z, v[3] = t.w;
  } else {
    const uint2 t = *reinterpret_cast<const uint2*>(x + row * ldx + c);
    const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162*>(&t.x);
    const __nv_bfloat162 hi = *reinterpret_cast<const __nv_bfloat162*>(&t.y);
    v[0] = __low2float(lo), v[1] = __high2float(lo), v[2] = __low2float(hi), v[3] = __high2float(hi);
  }
  float amax = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const float s = fp8_block_scale(amax);
  *reinterpret_cast<uint32_t*>(out + row * ldo + c) =
      fp8_code2(v[0], v[1], s) | (static_cast<uint32_t>(fp8_code2(v[2], v[3], s)) << 16);
  if (lane == 0) out_scale[row * out_scale_ld + c / 128] = s;
}

int quantize_fp8_rows(const void* x, int x_bf16, long long ldx, int rows, int D, void* out, long long ldo,
                      float* out_scale, long long out_scale_ld, cudaStream_t stream) {
  if (rows <= 0) return LN3_OK;
  if (x == nullptr || out == nullptr || out_scale == nullptr)
    return set_error(LN3_EINVAL, "quantize_fp8_rows: null pointer");
  if (D <= 0 || D % 128 != 0) return set_error(LN3_EINVAL, "quantize_fp8_rows: D=%d must be a positive multiple of 128", D);
  if (ldx < D || ldo < D || out_scale_ld < D / 128)
    return set_error(LN3_EINVAL, "quantize_fp8_rows: ldx and ldo must be >= D, out_scale_ld >= D/128");
  if (ldx % (x_bf16 ? 8 : 4) != 0 || ldo % 16 != 0 || misaligned16(x) || misaligned16(out))
    return set_error(LN3_EINVAL, "quantize_fp8_rows: x and out must be 16-byte aligned with 16-byte row pitches");
  const long long warps = static_cast<long long>(rows) * (D / 128);
  const dim3 grid(static_cast<unsigned>((warps + 7) / 8)), block(256);
  if (x_bf16)
    quantize_fp8_kernel<<<grid, block, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), ldx, rows, D / 128,
                                                   static_cast<uint8_t*>(out), ldo, out_scale, out_scale_ld);
  else
    quantize_fp8_kernel<<<grid, block, 0, stream>>>(static_cast<const float*>(x), ldx, rows, D / 128,
                                                   static_cast<uint8_t*>(out), ldo, out_scale, out_scale_ld);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "quantize_fp8_rows launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ timestep embedding
__global__ void timestep_embedding_kernel(const float* __restrict__ t, int B,
                                          __nv_bfloat16* __restrict__ out) {
  const int b = blockIdx.x;
  const int i = threadIdx.x;  // 0..127
  if (b >= B) return;
  // freqs = exp(-ln(10000) * i / 128) in fp32, as torch.exp(fp32 tensor) computes it
  const float f = expf(-9.210340371976184f * static_cast<float>(i) / 128.0f);
  const float arg = t[b] * f;
  out[b * 256 + i] = __float2bfloat16(cosf(arg));
  out[b * 256 + 128 + i] = __float2bfloat16(sinf(arg));
}

int timestep_embedding(const float* t, int B, void* out_bf16, cudaStream_t stream) {
  if (B <= 0) return LN3_OK;
  timestep_embedding_kernel<<<B, 128, 0, stream>>>(t, B, reinterpret_cast<__nv_bfloat16*>(out_bf16));
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "timestep_embedding launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ patch embed
// Block = one token (b, n, l); threads stride over D.  K = Cin*4 (<= 64) inputs staged in smem.
__global__ void __launch_bounds__(256)
patch_embed_kernel(const ln3_patch_embed_args a) {
  __shared__ float xin[64];
  const int P = a.S / 2, L = P * P;
  const int tok = blockIdx.x;  // b * 3L + n * L + l
  const int b = tok / (3 * L);
  const int nl = tok - b * 3 * L;
  const int n = nl / L, l = nl - n * L;
  const int pi = l / P, pj = l - pi * P;
  const int K = a.Cin * 4;
  if (threadIdx.x < K) {
    const int c = threadIdx.x >> 2, p = (threadIdx.x >> 1) & 1, q = threadIdx.x & 1;
    const float s = a.in_scale ? a.in_scale[b] : 1.f;
    xin[threadIdx.x] =
        s * a.x[((static_cast<long long>(b) * (3 * a.Cin) + c * 3 + n) * a.S + 2 * pi + p) * a.S +
                2 * pj + q];
  }
  __syncthreads();
  float* o = a.tokens + static_cast<long long>(tok) * a.D;
  const float* pe = a.pos_embed ? a.pos_embed + static_cast<long long>(nl) * a.D : nullptr;
  for (int d = threadIdx.x; d < a.D; d += blockDim.x) {
    float acc = a.bias ? a.bias[d] : 0.f;
    const float* w = a.weight + static_cast<long long>(d) * K;
    for (int k = 0; k < K; ++k) acc = fmaf(w[k], xin[k], acc);
    if (pe) acc += pe[d];
    o[d] = acc;
  }
}

// Cin == 4 fast path (the tri-latent: K = 16).  Block = 16 consecutive tokens; each thread keeps the
// 16 weights of its output channel in registers and walks the tokens, so the weight matrix is read once
// per block instead of once per token and every store is a coalesced 1 KB row segment.
constexpr int kPeTok = 16;
__global__ void __launch_bounds__(256)
patch_embed_k16_kernel(const ln3_patch_embed_args a) {
  __shared__ float xin[kPeTok][16];
  const int P = a.S / 2, L = P * P;
  const int ntok = a.B * 3 * L;
  const int tok0 = blockIdx.x * kPeTok;
  {
    const int t = threadIdx.x >> 4, k = threadIdx.x & 15;
    const int tok = tok0 + t;
    if (tok < ntok) {
      const int b = tok / (3 * L);
      const int nl = tok - b * 3 * L;
      const int n = nl / L, l = nl - n * L;
      const int pi = l / P, pj = l - pi * P;
      const int c = k >> 2, p = (k >> 1) & 1, q = k & 1;
      const float s = a.in_scale ? a.in_scale[b] : 1.f;
      xin[t][k] = s * a.x[((static_cast<long long>(b) * 12 + c * 3 + n) * a.S + 2 * pi + p) * a.S + 2 * pj + q];
    }
  }
  __syncthreads();
  // a thread owns four consecutive output channels: 64 weights in registers, 128-bit pos_embed loads and
  // token stores (the 4-byte version ran at 0.8 TB/s)
  for (int d = threadIdx.x * 4; d < a.D; d += 1024) {
    float w[4][16];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float4* wp = reinterpret_cast<const float4*>(a.weight + static_cast<long long>(d + j) * 16);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float4 v = __ldg(wp + i);
        w[j][4 * i] = v.x, w[j][4 * i + 1] = v.y, w[j][4 * i + 2] = v.z, w[j][4 * i + 3] = v.w;
      }
    }
    float4 bias = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.bias) bias = __ldg(reinterpret_cast<const float4*>(a.bias + d));
    const int nl0 = tok0 % (3 * L);
#pragma unroll 4
    for (int t = 0; t < kPeTok; ++t) {
      const int tok = tok0 + t;
      float acc[4] = {bias.x, bias.y, bias.z, bias.w};
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const float xv = xin[t][k];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] = fmaf(w[j][k], xv, acc[j]);
      }
      if (tok < ntok) {
        if (a.pos_embed) {
          const float4 pe = __ldg(reinterpret_cast<const float4*>(a.pos_embed + static_cast<long long>((nl0 + t) % (3 * L)) * a.D + d));
          acc[0] += pe.x, acc[1] += pe.y, acc[2] += pe.z, acc[3] += pe.w;
        }
        *reinterpret_cast<float4*>(a.tokens + static_cast<long long>(tok) * a.D + d) = make_float4(acc[0], acc[1], acc[2], acc[3]);
      }
    }
  }
}

int patch_embed(const ln3_patch_embed_args* a, cudaStream_t stream) {
  if (a->B <= 0) return LN3_OK;
  if (a->S % 2 || a->Cin <= 0 || a->Cin > 16 || a->D <= 0)
    return set_error(LN3_EINVAL, "patch_embed: need even S, 1 <= Cin <= 16");
  const int L = (a->S / 2) * (a->S / 2);
  // the k16 kernel moves weight, bias, pos_embed and tokens as float4; the generic kernel uses scalar accesses
  if (a->Cin == 4 && a->D % 4 == 0 && !misaligned16(a->weight) && !misaligned16(a->bias) &&
      !misaligned16(a->pos_embed) && !misaligned16(a->tokens))
    patch_embed_k16_kernel<<<(a->B * 3 * L + kPeTok - 1) / kPeTok, 256, 0, stream>>>(*a);
  else
    patch_embed_kernel<<<a->B * 3 * L, 256, 0, stream>>>(*a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "patch_embed launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ final layer
// One warp per token: LN + modulate in registers, then 4*Cout dot products (warp reductions),
// scattered into the unpatchified '(b, c*3+n, 2i+p, 2j+q)' layout.
// Two tokens per warp: the 4*Cout weight rows are read once for both, and the 2 x 16 dot-product partials
// are reduced with one 31-shuffle reduce-scatter (lane tk*16 + o ends up with output o of token tk) instead
// of 32 five-step warp sums.  Requires 4*Cout == 16 (every release config: Cout = 4); other sizes take
// the one-token kernel below.
template <int NV>
__global__ void __launch_bounds__(128)
final_layer2_kernel(const ln3_final_layer_args a) {
  const int P = a.S / 2, L = P * P;
  const int ntok = a.B * 3 * L;
  const int tok0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 2;
  if (tok0 >= ntok) return;
  const int lane = threadIdx.x & 31;
  float4 v[2][NV];
#pragma unroll
  for (int tk = 0; tk < 2; ++tk) {
    const int tok = tok0 + tk < ntok ? tok0 + tk : ntok - 1;
    const int b = tok / (3 * L);
    const float* x = a.x + static_cast<long long>(tok) * a.D;
#pragma unroll
    for (int i = 0; i < NV; ++i) v[tk][i] = *reinterpret_cast<const float4*>(x + (i * 32 + lane) * 4);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) s += (v[tk][i].x + v[tk][i].y) + (v[tk][i].z + v[tk][i].w);
    const float mean = warp_sum(s) / static_cast<float>(a.D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float dx = v[tk][i].x - mean, dy = v[tk][i].y - mean, dz = v[tk][i].z - mean, dw = v[tk][i].w - mean;
      q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
    const float rstd = rsqrtf(warp_sum(q) / static_cast<float>(a.D) + 1e-6f);
    const float* sh = a.shift + static_cast<long long>(b) * a.mod_ld;
    const float* sc = a.scale + static_cast<long long>(b) * a.mod_ld;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = (i * 32 + lane) * 4;
      float4 s1 = __ldg(reinterpret_cast<const float4*>(sc + c));
      float4 s0 = __ldg(reinterpret_cast<const float4*>(sh + c));
      if (a.scale_tab != nullptr) {
        const float4 t1 = __ldg(reinterpret_cast<const float4*>(a.scale_tab + c));
        const float4 t0 = __ldg(reinterpret_cast<const float4*>(a.shift_tab + c));
        s1.x += t1.x; s1.y += t1.y; s1.z += t1.z; s1.w += t1.w;
        s0.x += t0.x; s0.y += t0.y; s0.z += t0.z; s0.w += t0.w;
      }
      v[tk][i].x = fmaf((v[tk][i].x - mean) * rstd, 1.f + s1.x, s0.x);
      v[tk][i].y = fmaf((v[tk][i].y - mean) * rstd, 1.f + s1.y, s0.y);
      v[tk][i].z = fmaf((v[tk][i].z - mean) * rstd, 1.f + s1.z, s0.z);
      v[tk][i].w = fmaf((v[tk][i].w - mean) * rstd, 1.f + s1.w, s0.w);
    }
  }
  float acc[32];  // [tk * 16 + o]
#pragma unroll
  for (int o = 0; o < 16; ++o) {
    const float* w = a.weight + static_cast<long long>(o) * a.D;
    float a0 = 0.f, a1 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 ww = __ldg(reinterpret_cast<const float4*>(w + (i * 32 + lane) * 4));
      a0 = fmaf(v[0][i].x, ww.x, a0); a0 = fmaf(v[0][i].y, ww.y, a0);
      a0 = fmaf(v[0][i].z, ww.z, a0); a0 = fmaf(v[0][i].w, ww.w, a0);
      a1 = fmaf(v[1][i].x, ww.x, a1); a1 = fmaf(v[1][i].y, ww.y, a1);
      a1 = fmaf(v[1][i].z, ww.z, a1); a1 = fmaf(v[1][i].w, ww.w, a1);
    }
    acc[o] = a0;
    acc[16 + o] = a1;
  }
  // reduce-scatter over the warp: after the stage with offset h, acc[0 .. h) holds partial sums of the
  // values whose index has bit h equal to the lane's bit h
#pragma unroll
  for (int h = 16; h >= 1; h >>= 1) {
    const bool up = (lane & h) != 0;
#pragma unroll
    for (int i = 0; i < h; ++i) {
      const float send = up ? acc[i] : acc[i + h];
      const float keep = up ? acc[i + h] : acc[i];
      acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, h);
    }
  }
  const int tk = lane >> 4, oidx = lane & 15;
  const int tok = tok0 + tk;
  if (tok < ntok) {
    const int b = tok / (3 * L);
    const int nl = tok - b * 3 * L;
    const int n = nl / L, l = nl - n * L;
    const int pi = l / P, pj = l - pi * P;
    // unpatchify: feature index = (p * 2 + q) * Cout + c   ('nhwpqc->nchpwq')
    const int c = oidx % a.Cout, pq = oidx / a.Cout, pp = pq >> 1, qq = pq & 1;
    a.out[((static_cast<long long>(b) * (3 * a.Cout) + c * 3 + n) * a.S + 2 * pi + pp) * a.S + 2 * pj + qq] =
        acc[0] + (a.bias ? a.bias[oidx] : 0.f);
  }
}

template <int NV>
__global__ void __launch_bounds__(128)
final_layer_kernel(const ln3_final_layer_args a) {
  const int P = a.S / 2, L = P * P;
  const int tok = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (tok >= a.B * 3 * L) return;
  const int lane = threadIdx.x & 31;
  const int b = tok / (3 * L);
  const int nl = tok - b * 3 * L;
  const int n = nl / L, l = nl - n * L;
  const int pi = l / P, pj = l - pi * P;
  const float* x = a.x + static_cast<long long>(tok) * a.D;
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = *reinterpret_cast<const float4*>(x + (i * 32 + lane) * 4);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) / static_cast<float>(a.D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
    q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
  }
  const float rstd = rsqrtf(warp_sum(q) / static_cast<float>(a.D) + 1e-6f);
  const float* sh = a.shift + static_cast<long long>(b) * a.mod_ld;
  const float* sc = a.scale + static_cast<long long>(b) * a.mod_ld;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    float4 s1 = __ldg(reinterpret_cast<const float4*>(sc + c));
    float4 s0 = __ldg(reinterpret_cast<const float4*>(sh + c));
    if (a.scale_tab != nullptr) {
      const float4 t1 = __ldg(reinterpret_cast<const float4*>(a.scale_tab + c));
      const float4 t0 = __ldg(reinterpret_cast<const float4*>(a.shift_tab + c));
      s1.x += t1.x; s1.y += t1.y; s1.z += t1.z; s1.w += t1.w;
      s0.x += t0.x; s0.y += t0.y; s0.z += t0.z; s0.w += t0.w;
    }
    v[i].x = fmaf((v[i].x - mean) * rstd, 1.f + s1.x, s0.x);
    v[i].y = fmaf((v[i].y - mean) * rstd, 1.f + s1.y, s0.y);
    v[i].z = fmaf((v[i].z - mean) * rstd, 1.f + s1.z, s0.z);
    v[i].w = fmaf((v[i].w - mean) * rstd, 1.f + s1.w, s0.w);
  }
  const int nout = 4 * a.Cout;
  for (int oidx = 0; oidx < nout; ++oidx) {
    const float* w = a.weight + static_cast<long long>(oidx) * a.D;
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 ww = __ldg(reinterpret_cast<const float4*>(w + (i * 32 + lane) * 4));
      acc = fmaf(v[i].x, ww.x, acc);
      acc = fmaf(v[i].y, ww.y, acc);
      acc = fmaf(v[i].z, ww.z, acc);
      acc = fmaf(v[i].w, ww.w, acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) {
      // unpatchify: feature index = (p * 2 + q) * Cout + c   ('nhwpqc->nchpwq')
      const int c = oidx % a.Cout, pq = oidx / a.Cout, p = pq >> 1, qq = pq & 1;
      a.out[((static_cast<long long>(b) * (3 * a.Cout) + c * 3 + n) * a.S + 2 * pi + p) * a.S +
            2 * pj + qq] = acc + (a.bias ? a.bias[oidx] : 0.f);
    }
  }
}

int final_layer(const ln3_final_layer_args* a, cudaStream_t stream) {
  if (a->B <= 0) return LN3_OK;
  if (a->D % 128 != 0 || a->D > 2048) return set_error(LN3_EINVAL, "final_layer: bad D=%d", a->D);
  if (a->shift == nullptr || a->scale == nullptr)
    return set_error(LN3_EINVAL, "final_layer: shift/scale required");
  // odd S would leave the last output row and column unwritten (tokens cover 2x2 patches)
  if (a->S <= 0 || a->S % 2 || a->Cout <= 0)
    return set_error(LN3_EINVAL, "final_layer: need even S > 0 and Cout > 0 (S=%d, Cout=%d)", a->S, a->Cout);
  if (a->mod_ld % 4) return set_error(LN3_EINVAL, "final_layer: mod_ld must be a multiple of 4");
  if ((a->shift_tab == nullptr) != (a->scale_tab == nullptr))
    return set_error(LN3_EINVAL, "final_layer: shift_tab and scale_tab must be given together");
  if (misaligned16(a->x) || misaligned16(a->shift) || misaligned16(a->scale) || misaligned16(a->shift_tab) ||
      misaligned16(a->scale_tab) || misaligned16(a->weight))
    return set_error(LN3_EINVAL, "final_layer: x, shift, scale, tables and weight must be 16-byte aligned");
  const int L = (a->S / 2) * (a->S / 2);
  const int toks = a->B * 3 * L;
  dim3 grid((toks + 3) / 4), block(128);
  if (4 * a->Cout == 16 && (a->D == 768 || a->D == 1024)) {
    dim3 grid2((toks + 7) / 8);
    if (a->D == 1024) final_layer2_kernel<8><<<grid2, block, 0, stream>>>(*a);
    else final_layer2_kernel<6><<<grid2, block, 0, stream>>>(*a);
    cudaError_t e2 = cudaGetLastError();
    if (e2 != cudaSuccess) return set_error(LN3_ECUDA, "final_layer launch: %s", cudaGetErrorString(e2));
    count_launch();
    return LN3_OK;
  }
  switch (a->D / 128) {
#define LN3_FL_CASE(n) \
  case n: final_layer_kernel<n><<<grid, block, 0, stream>>>(*a); break;
    LN3_FL_CASE(1) LN3_FL_CASE(2) LN3_FL_CASE(3) LN3_FL_CASE(4) LN3_FL_CASE(5) LN3_FL_CASE(6)
    LN3_FL_CASE(7) LN3_FL_CASE(8) LN3_FL_CASE(9) LN3_FL_CASE(10) LN3_FL_CASE(11) LN3_FL_CASE(12)
    LN3_FL_CASE(13) LN3_FL_CASE(14) LN3_FL_CASE(15) LN3_FL_CASE(16)
#undef LN3_FL_CASE
    default: return set_error(LN3_EINVAL, "final_layer: unsupported D");
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "final_layer launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

// ------------------------------------------------------------------ sampler update
__global__ void __launch_bounds__(256)
sampler_update_kernel(const ln3_sampler_update_args a) {
  const int b = blockIdx.y;
  const float4 cf = *reinterpret_cast<const float4*>(a.coef + b * 4);
  const long long base = static_cast<long long>(b) * a.n_per_sample;
  const long long n4 = a.n_per_sample >> 2;
  for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long off = base + i * 4;
    const float4 x = *reinterpret_cast<const float4*>(a.x + off);
    const float4 m0 = *reinterpret_cast<const float4*>(a.m0 + off);
    float4 r = make_float4(cf.x * x.x, cf.x * x.y, cf.x * x.z, cf.x * x.w);
    r.x = fmaf(cf.y, m0.x, r.x); r.y = fmaf(cf.y, m0.y, r.y);
    r.z = fmaf(cf.y, m0.z, r.z); r.w = fmaf(cf.y, m0.w, r.w);
    if (a.m1 != nullptr) {
      const float4 m1 = *reinterpret_cast<const float4*>(a.m1 + off);
      r.x = fmaf(cf.z, m1.x, r.x); r.y = fmaf(cf.z, m1.y, r.y);
      r.z = fmaf(cf.z, m1.z, r.z); r.w = fmaf(cf.z, m1.w, r.w);
    }
    if (a.noise != nullptr) {
      const float4 nz = *reinterpret_cast<const float4*>(a.noise + off);
      r.x = fmaf(cf.w, nz.x, r.x); r.y = fmaf(cf.w, nz.y, r.y);
      r.z = fmaf(cf.w, nz.z, r.z); r.w = fmaf(cf.w, nz.w, r.w);
    }
    *reinterpret_cast<float4*>(a.x_out + off) = r;
  }
}

int sampler_affine_update(const ln3_sampler_update_args* a, cudaStream_t stream) {
  if (a->B <= 0 || a->n_per_sample <= 0) return LN3_OK;
  if (a->n_per_sample % 4) return set_error(LN3_EINVAL, "sampler_update: n_per_sample % 4 != 0");
  if (!a->x || !a->m0 || !a->coef || !a->x_out) return set_error(LN3_EINVAL, "sampler_update: null pointer");
  if (misaligned16(a->x) || misaligned16(a->m0) || misaligned16(a->m1) || misaligned16(a->noise) ||
      misaligned16(a->x_out) || misaligned16(a->coef))
    return set_error(LN3_EINVAL, "sampler_update: x, m0, m1, noise, x_out and coef must be 16-byte aligned");
  const long long n4 = a->n_per_sample / 4;
  int gx = static_cast<int>((n4 + 255) / 256);
  if (gx > 1024) gx = 1024;
  dim3 grid(gx, a->B);
  sampler_update_kernel<<<grid, 256, 0, stream>>>(*a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "sampler_update launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

}  // namespace ln3
