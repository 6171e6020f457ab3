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
int device_l2_bytes();
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

// 2-D bf16 tensor map: tensor [rows, cols] with row pitch `ld` elements, box [box_rows, box_cols],
// 128-byte swizzle (box_cols must be 64), zero fill out of bounds.
int make_tmap_2d_bf16(CUtensorMap* out, const void* ptr, long long rows, long long cols,
                      long long ld, int box_rows, int box_cols);
// 3-D bf16 tensor map: tensor [d2, d1, d0] (d0 contiguous) with element strides (s2, s1, 1),
// box [1, box1, box0], 128-byte swizzle for box0 = 64, none for box0 = 8 (rows of 16 bytes, packed).
int make_tmap_3d_bf16(CUtensorMap* out, const void* ptr, long long d0, long long d1, long long d2,
                      long long s1, long long s2, int box0, int box1);

// 2-D byte (e4m3) tensor map: [rows, cols] with row pitch `ld` bytes, box [box_rows, 128], 128-byte swizzle.
int make_tmap_2d_u8(CUtensorMap* out, const void* ptr, long long rows, long long cols, long long ld, int box_rows,
                    int box_cols);

int gemm_bf16(const ln3_gemm_args* a, cudaStream_t stream);
size_t gemm_fp8_workspace_bytes();
int gemm_fp8(const ln3_gemm_fp8_args* a, cudaStream_t stream);
int norm_modulate_fp8(const ln3_norm_modulate_fp8_args* a, cudaStream_t stream);
int quantize_fp8_rows(const void* x, int x_bf16, long long ldx, int rows, int D, void* out, long long ldo,
                      float* out_scale, long long out_scale_ld, cudaStream_t stream);
size_t gemm_workspace_bytes();
int fmha_fwd(const ln3_fmha_args* a, cudaStream_t stream);
int norm_modulate(const ln3_norm_modulate_args* a, cudaStream_t stream);
int timestep_embedding(const float* t, int B, void* out_bf16, cudaStream_t stream);
int patch_embed(const ln3_patch_embed_args* a, cudaStream_t stream);
int plucker_patchify(const ln3_plucker_patchify_args* a, cudaStream_t stream);
int final_layer(const ln3_final_layer_args* a, cudaStream_t stream);
int sampler_affine_update(const ln3_sampler_update_args* a, cudaStream_t stream);
int sampler_step(const ln3_sampler_step_args* a, cudaStream_t stream);   // arguments validated by the caller
int flow_sde_step(const ln3_flow_sde_step_args* a, cudaStream_t stream);   // arguments validated by the caller
size_t render_workspace_bytes(int V, int M, int group_size);
int render_tile_width(int M, int image_w);
int render_views(const ln3_render_args* a, cudaStream_t stream);
int query_points(const ln3_query_points_args* a, cudaStream_t stream);
int generate_rays(const float* cams, int V, int res, float* ray_o, float* ray_d, cudaStream_t stream);
int planes_to_channels_last(const float* planes, int n_obj, int C, int H, int W, float* out,
                            cudaStream_t stream);

int pack_frames(const ln3_pack_frames_args* a, cudaStream_t stream);
size_t marching_cubes_workspace_bytes(int nx, int ny, int nz);
int marching_cubes_count(const ln3_marching_cubes_args* a, cudaStream_t stream);
int marching_cubes_emit(const ln3_marching_cubes_args* a, cudaStream_t stream);

int conv_cout_tile(int N, int H, int W, int Cout);
int conv_nhwc(const ln3_conv_args* a, cudaStream_t stream);
int groupnorm_stats(const float* x, const float* gamma, const float* beta, int N, int HW, int C, int G,
                    float eps, float* scale, float* shift, cudaStream_t stream);
int attn_single_head(const float* q, const float* k, const float* v, float* out, int N, int L, int C,
                     cudaStream_t stream);
int patch_embed_triplane(const float* x, const float* w, const float* bias, int B, int Cz, int S, int E,
                         float in_mul, float* tokens, void* silu_bf16, cudaStream_t stream);
int downsample_nhwc(const ln3_conv_args* a, cudaStream_t stream);
int vae_posterior(const ln3_vae_posterior_args* a, cudaStream_t stream);
int view_mean_nhwc(const float* x, float* out, int B, int F, int S, int C, cudaStream_t stream);
int ode_stages(int method);   // stage forwards per attempt, LN3_EUNSUPPORTED for an unknown method
size_t ode_workspace_bytes(int B, long long n_per_sample);
int ode_stage(const ln3_ode_args* a, int method, int stage, cudaStream_t stream);
int ode_initial_step(const ln3_ode_args* a, int method, int phase, cudaStream_t stream);
int ode_step(const ln3_ode_args* a, int method, cudaStream_t stream);

}  // namespace ln3
