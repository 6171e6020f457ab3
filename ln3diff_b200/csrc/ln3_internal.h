// Internal declarations shared by the translation units of libln3b200.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <atomic>
#include <mutex>

#include "../../include/ln3b200.h"

namespace ln3 {

// Records a thread-local error message and returns `code` (so `return set_error(...)` works).
int set_error(int code, const char* fmt, ...);
void count_launch(int n = 1);
int device_sm_count();
// Per-device one-shot guard.  cudaFuncSetAttribute(MaxDynamicSharedMemorySize) and the SM count belong to
// the device that is current at the call; one process may drive several GPUs and two host threads may race
// the first call, so "done" is tracked per device ordinal (bit d of a mask) under a mutex.
struct DeviceOnce {
  std::atomic<unsigned long long> done{0};
  std::mutex mu;
  template <class F>
  int run(F&& init) {   // init() -> LN3_OK or a negative LN3_E* code (after set_error)
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
    const unsigned long long bit = 1ull << (dev & 63);
    if (done.load(std::memory_order_acquire) & bit) return LN3_OK;
    std::lock_guard<std::mutex> lk(mu);
    if (done.load(std::memory_order_relaxed) & bit) return LN3_OK;
    const int rc = init();
    if (rc == LN3_OK) done.fetch_or(bit, std::memory_order_release);
    return rc;
  }
};

// Programmatic dependent launch (opt-in with LN3_PDL=1; 12.05 vs 12.04 ms per forward, i.e. no gain): kernels that call pdl_wait() before their first
// dependent memory access may be launched with this; their CTAs are scheduled while the previous
// kernel of the stream drains, hiding launch latency and the per-CTA prologue.
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// 2-D bf16 tensor map: tensor [rows, cols] with row pitch `ld` elements, box [box_rows, box_cols],
// 128-byte swizzle (box_cols must be 64), zero fill out of bounds.
int make_tmap_2d_bf16(CUtensorMap* out, const void* ptr, long long rows, long long cols,
                      long long ld, int box_rows, int box_cols);
// 3-D bf16 tensor map: tensor [d2, d1, d0] (d0 contiguous) with element strides (s2, s1, 1),
// box [1, box1, box0], 128-byte swizzle.
int make_tmap_3d_bf16(CUtensorMap* out, const void* ptr, long long d0, long long d1, long long d2,
                      long long s1, long long s2, int box0, int box1);

int gemm_bf16(const ln3_gemm_args* a, cudaStream_t stream);
size_t gemm_workspace_bytes();
int fmha_fwd(const ln3_fmha_args* a, cudaStream_t stream);
int norm_modulate(const ln3_norm_modulate_args* a, cudaStream_t stream);
int timestep_embedding(const float* t, int B, void* out_bf16, cudaStream_t stream);
int patch_embed(const ln3_patch_embed_args* a, cudaStream_t stream);
int plucker_patchify(const ln3_plucker_patchify_args* a, cudaStream_t stream);
int final_layer(const ln3_final_layer_args* a, cudaStream_t stream);
int sampler_affine_update(const ln3_sampler_update_args* a, cudaStream_t stream);
size_t render_workspace_bytes(int V, int M, int group_size);
int render_views(const ln3_render_args* a, cudaStream_t stream);
int query_points(const ln3_query_points_args* a, cudaStream_t stream);
int generate_rays(const float* cams, int V, int res, float* ray_o, float* ray_d, cudaStream_t stream);
int planes_to_channels_last(const float* planes, int n_obj, int C, int H, int W, float* out,
                            cudaStream_t stream);

int pack_frames(const ln3_pack_frames_args* a, cudaStream_t stream);
size_t marching_cubes_workspace_bytes(int nx, int ny, int nz);
int marching_cubes_count(const ln3_marching_cubes_args* a, cudaStream_t stream);
int marching_cubes_emit(const ln3_marching_cubes_args* a, cudaStream_t stream);

int conv_nhwc(const ln3_conv_args* a, cudaStream_t stream);
int groupnorm_stats(const float* x, const float* gamma, const float* beta, int N, int HW, int C, int G,
                    float eps, float* scale, float* shift, cudaStream_t stream);
int attn_single_head(const float* q, const float* k, const float* v, float* out, int N, int L, int C,
                     cudaStream_t stream);
int patch_embed_triplane(const float* x, const float* w, const float* bias, int B, int Cz, int S, int E,
                         float in_mul, float* tokens, void* silu_bf16, cudaStream_t stream);

}  // namespace ln3
