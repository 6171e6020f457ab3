// extern "C" surface of libln3b200 + shared host utilities (error text, tensor-map encoding).
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include <cstdlib>

#include "ln3_internal.h"

namespace ln3 {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void count_launch(int n) { g_launches.fetch_add(static_cast<unsigned long long>(n)); }

bool pdl_enabled() {
  static const bool on = getenv("LN3_PDL") && atoi(getenv("LN3_PDL")) != 0;  // opt-in: measured no gain inside CUDA graphs
  return on;
}

int device_sm_count() {
  static std::atomic<int> sms[64];   // per device ordinal; 0 = not queried yet
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 1;
  std::atomic<int>& slot = sms[dev & 63];
  int n = slot.load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 1;
    slot.store(n, std::memory_order_relaxed);
  }
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || p == nullptr) {
      set_error(LN3_ECUDA, "cuTensorMapEncodeTiled entry point unavailable: %s",
                cudaGetErrorString(e));
      return nullptr;
    }
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* ptr, long long rows, long long cols,
                      long long ld, int box_rows, int box_cols) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return LN3_ECUDA;
  if (box_cols != 64) return set_error(LN3_EINVAL, "tmap: box_cols must be 64 (128B swizzle)");
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(LN3_ECUDA, "cuTensorMapEncodeTiled(2d rows=%lld cols=%lld ld=%lld) -> %d", rows,
                     cols, ld, static_cast<int>(r));
  return LN3_OK;
}

int make_tmap_3d_bf16(CUtensorMap* out, const void* ptr, long long d0, long long d1, long long d2,
                      long long s1, long long s2, int box0, int box1) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return LN3_ECUDA;
  if (box0 != 64) return set_error(LN3_EINVAL, "tmap: box0 must be 64 (128B swizzle)");
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(d0), static_cast<cuuint64_t>(d1),
                        static_cast<cuuint64_t>(d2)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(s1) * 2, static_cast<cuuint64_t>(s2) * 2};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(box0), static_cast<cuuint32_t>(box1), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(LN3_ECUDA, "cuTensorMapEncodeTiled(3d %lldx%lldx%lld) -> %d", d2, d1, d0,
                     static_cast<int>(r));
  return LN3_OK;
}

}  // namespace ln3

using namespace ln3;

extern "C" {

int ln3_abi_version(void) { return LN3_ABI_VERSION; }
const char* ln3_last_error(void) { return g_err; }
unsigned long long ln3_launch_count(void) { return g_launches.load(); }
void ln3_add_launch_count(unsigned long long n) { g_launches.fetch_add(n); }

int ln3_gemm_bf16(const ln3_gemm_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "gemm: null args");
  return gemm_bf16(args, static_cast<cudaStream_t>(stream));
}

size_t ln3_gemm_workspace_bytes(void) { return gemm_workspace_bytes(); }
int ln3_fmha_fwd(const ln3_fmha_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "fmha: null args");
  return fmha_fwd(args, static_cast<cudaStream_t>(stream));
}
int ln3_norm_modulate(const ln3_norm_modulate_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "norm_modulate: null args");
  return norm_modulate(args, static_cast<cudaStream_t>(stream));
}
int ln3_timestep_embedding(const float* t, int B, void* out_bf16, void* stream) {
  if (!t || !out_bf16) return set_error(LN3_EINVAL, "timestep_embedding: null pointer");
  return timestep_embedding(t, B, out_bf16, static_cast<cudaStream_t>(stream));
}
int ln3_patch_embed(const ln3_patch_embed_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "patch_embed: null args");
  return patch_embed(args, static_cast<cudaStream_t>(stream));
}
int ln3_plucker_patchify(const ln3_plucker_patchify_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "plucker_patchify: null args");
  return plucker_patchify(args, static_cast<cudaStream_t>(stream));
}
int ln3_final_layer(const ln3_final_layer_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "final_layer: null args");
  return final_layer(args, static_cast<cudaStream_t>(stream));
}
int ln3_sampler_affine_update(const ln3_sampler_update_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "sampler_update: null args");
  return sampler_affine_update(args, static_cast<cudaStream_t>(stream));
}

size_t ln3_render_workspace_bytes(int V, int M, int group_size) {
  if (V <= 0 || M <= 0 || group_size <= 0) return 0;
  return render_workspace_bytes(V, M, group_size);
}
int ln3_render_views(const ln3_render_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "render: null args");
  return render_views(args, static_cast<cudaStream_t>(stream));
}
int ln3_query_points(const ln3_query_points_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "query_points: null args");
  return query_points(args, static_cast<cudaStream_t>(stream));
}
int ln3_generate_rays(const float* cams, int V, int res, float* ray_o, float* ray_d, void* stream) {
  if (!cams || !ray_o || !ray_d) return set_error(LN3_EINVAL, "generate_rays: null pointer");
  return generate_rays(cams, V, res, ray_o, ray_d, static_cast<cudaStream_t>(stream));
}
int ln3_planes_to_channels_last(const float* planes, int n_obj, int C, int H, int W, float* out,
                                void* stream) {
  if (!planes || !out) return set_error(LN3_EINVAL, "planes_to_channels_last: null pointer");
  return planes_to_channels_last(planes, n_obj, C, H, W, out, static_cast<cudaStream_t>(stream));
}

size_t ln3_marching_cubes_workspace_bytes(int nx, int ny, int nz) { return marching_cubes_workspace_bytes(nx, ny, nz); }
int ln3_marching_cubes_count(const ln3_marching_cubes_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "marching_cubes_count: null args");
  return marching_cubes_count(args, static_cast<cudaStream_t>(stream));
}
int ln3_marching_cubes_emit(const ln3_marching_cubes_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "marching_cubes_emit: null args");
  return marching_cubes_emit(args, static_cast<cudaStream_t>(stream));
}
int ln3_pack_frames(const ln3_pack_frames_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "pack_frames: null args");
  return pack_frames(args, static_cast<cudaStream_t>(stream));
}

int ln3_conv_nhwc(const ln3_conv_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "conv: null args");
  return conv_nhwc(args, static_cast<cudaStream_t>(stream));
}
int ln3_groupnorm_stats(const float* x, const float* gamma, const float* beta, int N, int HW, int C,
                        int G, float eps, float* scale, float* shift, void* stream) {
  if (!x || !gamma || !beta || !scale || !shift) return set_error(LN3_EINVAL, "groupnorm: null pointer");
  return groupnorm_stats(x, gamma, beta, N, HW, C, G, eps, scale, shift, static_cast<cudaStream_t>(stream));
}
int ln3_attn_single_head(const float* q, const float* k, const float* v, float* out, int N, int L,
                         int C, void* stream) {
  if (!q || !k || !v || !out) return set_error(LN3_EINVAL, "attn_single_head: null pointer");
  return attn_single_head(q, k, v, out, N, L, C, static_cast<cudaStream_t>(stream));
}
int ln3_patch_embed_triplane(const float* x, const float* w, const float* bias, int B, int Cz, int S,
                             int E, float in_mul, float* tokens, void* silu_bf16, void* stream) {
  if (!x || !w || !tokens) return set_error(LN3_EINVAL, "patch_embed_triplane: null pointer");
  return patch_embed_triplane(x, w, bias, B, Cz, S, E, in_mul, tokens, silu_bf16,
                              static_cast<cudaStream_t>(stream));
}

}  // extern "C"
