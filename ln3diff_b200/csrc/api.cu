// extern "C" surface of libln3b200 + shared host utilities (error text, tensor-map encoding).
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <vector>

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

int device_l2_bytes() {
  static std::atomic<int> l2[64];   // per device ordinal; 0 = not queried yet
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  std::atomic<int>& slot = l2[dev & 63];
  int n = slot.load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrL2CacheSize, dev) != cudaSuccess || n <= 0) n = 0;
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

int make_tmap_2d_u8(CUtensorMap* out, const void* ptr, long long rows, long long cols, long long ld, int box_rows,
                    int box_cols) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return LN3_ECUDA;
  if (box_cols != 128) return set_error(LN3_EINVAL, "tmap: box_cols must be 128 (128B swizzle)");
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(LN3_ECUDA, "cuTensorMapEncodeTiled(2d u8 rows=%lld cols=%lld ld=%lld) -> %d", rows, cols, ld,
                     static_cast<int>(r));
  return LN3_OK;
}

int make_tmap_3d_bf16(CUtensorMap* out, const void* ptr, long long d0, long long d1, long long d2,
                      long long s1, long long s2, int box0, int box1) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return LN3_ECUDA;
  if (box0 != 64 && box0 != 8) return set_error(LN3_EINVAL, "tmap: box0 must be 64 (128B swizzle) or 8 (no swizzle)");
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(d0), static_cast<cuuint64_t>(d1),
                        static_cast<cuuint64_t>(d2)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(s1) * 2, static_cast<cuuint64_t>(s2) * 2};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(box0), static_cast<cuuint32_t>(box1), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(ptr), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  box0 == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(LN3_ECUDA, "cuTensorMapEncodeTiled(3d %lldx%lldx%lld) -> %d", d2, d1, d0,
                     static_cast<int>(r));
  return LN3_OK;
}

// Checks shared by the ln3_ode_* entry points (see include/ln3b200.h); `need` selects the buffers the call reads.
enum { ODE_NEED_STAGE = 1, ODE_NEED_K = 2, ODE_NEED_K0 = 4, ODE_NEED_OUT = 8, ODE_NEED_WS = 16 };

static bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

// `stages`: the stage derivatives k[0 .. stages-1] that ODE_NEED_K requires.
static int ode_validate(const ln3_ode_args* a, int need, const char* what, int stages = 6) {
  if (!a) return set_error(LN3_EINVAL, "%s: null args", what);
  if (a->B <= 0 || a->G <= 0) return set_error(LN3_EINVAL, "%s: B and G must be positive", what);
  if (a->n_per_sample <= 0 || a->n_per_sample % 4)
    return set_error(LN3_EINVAL, "%s: n_per_sample must be a positive multiple of 4", what);
  if (a->max_num_steps < 0) return set_error(LN3_EINVAL, "%s: max_num_steps < 0", what);
  if (!a->y || !a->f0 || !a->state || !a->row_group || !a->row_group_host)
    return set_error(LN3_EINVAL, "%s: null y, f0, state or row map", what);
  if (misaligned16(a->y) || misaligned16(a->f0))
    return set_error(LN3_EINVAL, "%s: y and f0 must be 16-byte aligned", what);
  if ((need & ODE_NEED_STAGE) && (!a->y_stage || !a->t_rows || misaligned16(a->y_stage)))
    return set_error(LN3_EINVAL, "%s: y_stage (16-byte aligned) and t_rows are required", what);
  const int nk = (need & ODE_NEED_K) ? stages : (need & ODE_NEED_K0) ? 1 : 0;
  for (int j = 0; j < nk; ++j)
    if (!a->k[j] || misaligned16(a->k[j]))
      return set_error(LN3_EINVAL, "%s: k[%d] is null or not 16-byte aligned", what, j);
  if ((need & ODE_NEED_OUT) && (!a->out || misaligned16(a->out)))
    return set_error(LN3_EINVAL, "%s: out is null or not 16-byte aligned", what);
  if ((need & ODE_NEED_WS) && (!a->workspace || a->workspace_bytes < ode_workspace_bytes(a->B, a->n_per_sample)))
    return set_error(LN3_EINVAL, "%s: workspace smaller than ln3_ode_workspace_bytes(B, n_per_sample)", what);
  std::vector<int> rows(static_cast<size_t>(a->G), 0);
  for (int r = 0; r < a->B; ++r) {
    const int g = a->row_group_host[r];
    if (g < 0 || g >= a->G) return set_error(LN3_EINVAL, "%s: row_group[%d] = %d is outside [0, %d)", what, r, g, a->G);
    ++rows[g];
  }
  for (int g = 0; g < a->G; ++g)
    if (rows[g] == 0) return set_error(LN3_EINVAL, "%s: group %d has no rows", what, g);
  return LN3_OK;
}

// The rules of ln3_sampler_step (include/ln3b200.h): shapes, NULLs, alignment, and no output range overlapping
// another output or an input except the two in-place aliases x_out == x and eval_out == x_eval.
static int sampler_step_validate(const ln3_sampler_step_args* a) {
  if (!a) return set_error(LN3_EINVAL, "sampler_step: null args");
  if (a->B < 0 || a->n_per_sample < 0) return set_error(LN3_EINVAL, "sampler_step: negative B or n_per_sample");
  if (a->n_per_sample % 4) return set_error(LN3_EINVAL, "sampler_step: n_per_sample % 4 != 0");
  if (a->B > 0 && a->n_per_sample > (1ll << 50) / (8ll * a->B))
    return set_error(LN3_EINVAL, "sampler_step: B * n_per_sample too large");
  if (!a->x || !a->x_eval || !a->net_u || !a->coef)
    return set_error(LN3_EINVAL, "sampler_step: null x, x_eval, net_u or coef");
  if (!a->x_out && !a->eval_out && !a->hist_out) return set_error(LN3_EINVAL, "sampler_step: no output");
  struct Range { const char* name; const void* p; unsigned long long bytes; };
  const unsigned long long row = 4ull * static_cast<unsigned long long>(a->B) * a->n_per_sample;
  const Range in[] = {{"x", a->x, row}, {"x_eval", a->x_eval, row}, {"net_u", a->net_u, row},
                      {"net_c", a->net_c, row}, {"hist[0]", a->hist[0], row}, {"hist[1]", a->hist[1], row},
                      {"hist[2]", a->hist[2], row}, {"noise", a->noise, row},
                      {"coef", a->coef, 48ull * static_cast<unsigned long long>(a->B)}};
  const Range out[] = {{"x_out", a->x_out, row}, {"eval_out", a->eval_out, 2 * row}, {"hist_out", a->hist_out, row}};
  for (const Range& r : in)
    if (misaligned16(r.p)) return set_error(LN3_EINVAL, "sampler_step: %s must be 16-byte aligned", r.name);
  for (const Range& r : out)
    if (misaligned16(r.p)) return set_error(LN3_EINVAL, "sampler_step: %s must be 16-byte aligned", r.name);
  auto overlap = [](const Range& u, const Range& v) {
    if (!u.p || !v.p || u.bytes == 0 || v.bytes == 0) return false;
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(u.p), b0 = reinterpret_cast<uintptr_t>(v.p);
    return a0 < b0 + v.bytes && b0 < a0 + u.bytes;
  };
  for (int i = 0; i < 3; ++i) {
    for (int j = i + 1; j < 3; ++j)
      if (overlap(out[i], out[j]))
        return set_error(LN3_EINVAL, "sampler_step: outputs %s and %s overlap", out[i].name, out[j].name);
    for (int j = 0; j < 9; ++j) {
      const bool alias = out[i].p == in[j].p && ((i == 0 && j == 0) || (i == 1 && j == 1));
      if (!alias && overlap(out[i], in[j]))
        return set_error(LN3_EINVAL, "sampler_step: output %s overlaps input %s", out[i].name, in[j].name);
    }
  }
  return LN3_OK;
}

// The rules of ln3_flow_sde_step (include/ln3b200.h): sizes, mode, NULLs, the noise row mapping, alignment, and no
// output range overlapping another output or an input except the in-place updates x_out == x and y_out == y.
static int flow_sde_step_validate(const ln3_flow_sde_step_args* a) {
  if (!a) return set_error(LN3_EINVAL, "flow_sde_step: null args");
  if (a->R < 0 || a->n < 0) return set_error(LN3_EINVAL, "flow_sde_step: negative R or n");
  if (a->R > 32767) return set_error(LN3_EINVAL, "flow_sde_step: R > 32767 (2R rows are one grid dimension)");
  if (a->n % 4) return set_error(LN3_EINVAL, "flow_sde_step: n % 4 != 0");
  if (a->R > 0 && a->n > (1ll << 50) / (8ll * a->R)) return set_error(LN3_EINVAL, "flow_sde_step: R * n too large");
  if (a->mode != LN3_SDE_DRIFT && a->mode != LN3_SDE_VELOCITY && a->mode != LN3_SDE_SCORE)
    return set_error(LN3_EINVAL, "flow_sde_step: unknown mode %d", a->mode);
  if (!a->y || !a->f) return set_error(LN3_EINVAL, "flow_sde_step: null y or f");
  if (!a->x_out && !a->y_out && !a->hist_out) return set_error(LN3_EINVAL, "flow_sde_step: no output");
  if (a->noise && (a->N <= 0 || a->N > a->R || a->R % a->N))
    return set_error(LN3_EINVAL, "flow_sde_step: noise rows need 0 < N <= R and R %% N == 0 (N = %d, R = %d)", a->N,
                     a->R);
  struct Range { const char* name; const void* p; unsigned long long bytes; };
  const unsigned long long rows = 8ull * static_cast<unsigned long long>(a->R) * a->n;   // 2R rows of fp32
  const unsigned long long nrows = a->noise ? 8ull * static_cast<unsigned long long>(a->N) * a->n : 0;
  const Range in[] = {{"x", a->x, rows}, {"y", a->y, rows}, {"f", a->f, rows}, {"hist", a->hist, rows},
                      {"noise", a->noise, nrows}};
  const Range out[] = {{"x_out", a->x_out, rows}, {"y_out", a->y_out, rows}, {"hist_out", a->hist_out, rows}};
  for (const Range& r : in)
    if (misaligned16(r.p)) return set_error(LN3_EINVAL, "flow_sde_step: %s must be 16-byte aligned", r.name);
  for (const Range& r : out)
    if (misaligned16(r.p)) return set_error(LN3_EINVAL, "flow_sde_step: %s must be 16-byte aligned", r.name);
  auto overlap = [](const Range& u, const Range& v) {
    if (!u.p || !v.p || u.bytes == 0 || v.bytes == 0) return false;
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(u.p), b0 = reinterpret_cast<uintptr_t>(v.p);
    return a0 < b0 + v.bytes && b0 < a0 + u.bytes;
  };
  for (int i = 0; i < 3; ++i) {
    for (int j = i + 1; j < 3; ++j)
      if (overlap(out[i], out[j]))
        return set_error(LN3_EINVAL, "flow_sde_step: outputs %s and %s overlap", out[i].name, out[j].name);
    for (int j = 0; j < 5; ++j) {
      const bool alias = out[i].p == in[j].p && ((i == 0 && j == 0) || (i == 1 && j == 1));
      if (!alias && overlap(out[i], in[j]))
        return set_error(LN3_EINVAL, "flow_sde_step: output %s overlaps input %s", out[i].name, in[j].name);
    }
  }
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
int ln3_sampler_step(const ln3_sampler_step_args* args, void* stream) {
  const int rc = sampler_step_validate(args);
  if (rc != LN3_OK) return rc;
  return sampler_step(args, static_cast<cudaStream_t>(stream));
}
int ln3_flow_sde_step(const ln3_flow_sde_step_args* args, void* stream) {
  const int rc = flow_sde_step_validate(args);
  if (rc != LN3_OK) return rc;
  return flow_sde_step(args, static_cast<cudaStream_t>(stream));
}

size_t ln3_render_workspace_bytes(int V, int M, int group_size) {
  if (V <= 0 || M <= 0 || group_size <= 0) return 0;
  return render_workspace_bytes(V, M, group_size);
}
int ln3_render_tile_width(int M, int image_w) {
  if (M <= 0) return 0;
  return render_tile_width(M, image_w);
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

int ln3_conv_cout_tile(int N, int H, int W, int Cout) {
  if (N <= 0 || H <= 0 || W <= 0 || Cout <= 0) return 0;
  return conv_cout_tile(N, H, W, Cout);
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

int ln3_downsample_nhwc(const ln3_conv_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "downsample: null args");
  return downsample_nhwc(args, static_cast<cudaStream_t>(stream));
}
int ln3_vae_posterior(const ln3_vae_posterior_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "vae_posterior: null args");
  return vae_posterior(args, static_cast<cudaStream_t>(stream));
}
int ln3_view_mean_nhwc(const float* x, float* out, int B, int F, int S, int C, void* stream) {
  return view_mean_nhwc(x, out, B, F, S, C, static_cast<cudaStream_t>(stream));
}

size_t ln3_ode_workspace_bytes(int B, long long n_per_sample) {
  if (B <= 0 || n_per_sample <= 0) return 0;
  return ode_workspace_bytes(B, n_per_sample);
}
int ln3_ode_stages(int method) { return ode_stages(method); }
int ln3_ode_rk_stage(const ln3_ode_args* args, int method, int stage, void* stream) {
  const int S = ode_stages(method);
  if (S < 0) return S;
  if (stage < 0 || stage > S) return set_error(LN3_EINVAL, "ode_stage: stage %d is outside 0..%d", stage, S);
  int rc = ode_validate(args, ODE_NEED_STAGE, "ode_stage");
  if (rc != LN3_OK) return rc;
  for (int j = 0; j + 1 < stage; ++j)   // stage i reads k[0 .. i-2]
    if (!args->k[j] || misaligned16(args->k[j]))
      return set_error(LN3_EINVAL, "ode_stage: k[%d] is null or not 16-byte aligned", j);
  return ode_stage(args, method, stage, static_cast<cudaStream_t>(stream));
}
int ln3_ode_rk_initial_step(const ln3_ode_args* args, int method, int phase, void* stream) {
  const int S = ode_stages(method);
  if (S < 0) return S;
  if (phase != 0 && phase != 1) return set_error(LN3_EINVAL, "ode_initial_step: phase must be 0 or 1");
  int rc = ode_validate(args, ODE_NEED_WS | (phase == 1 ? ODE_NEED_K0 : 0), "ode_initial_step");
  if (rc != LN3_OK) return rc;
  return ode_initial_step(args, method, phase, static_cast<cudaStream_t>(stream));
}
int ln3_ode_rk_step(const ln3_ode_args* args, int method, void* stream) {
  const int S = ode_stages(method);
  if (S < 0) return S;
  int rc = ode_validate(args, ODE_NEED_STAGE | ODE_NEED_K | ODE_NEED_OUT | ODE_NEED_WS, "ode_step", S);
  if (rc != LN3_OK) return rc;
  return ode_step(args, method, static_cast<cudaStream_t>(stream));
}
int ln3_ode_stage(const ln3_ode_args* args, int stage, void* stream) {
  return ln3_ode_rk_stage(args, LN3_ODE_DOPRI5, stage, stream);
}
int ln3_ode_initial_step(const ln3_ode_args* args, int phase, void* stream) {
  return ln3_ode_rk_initial_step(args, LN3_ODE_DOPRI5, phase, stream);
}
int ln3_ode_step(const ln3_ode_args* args, void* stream) { return ln3_ode_rk_step(args, LN3_ODE_DOPRI5, stream); }


size_t ln3_gemm_fp8_workspace_bytes(void) { return gemm_fp8_workspace_bytes(); }
int ln3_gemm_fp8(const ln3_gemm_fp8_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "gemm_fp8: null args");
  return gemm_fp8(args, static_cast<cudaStream_t>(stream));
}
int ln3_norm_modulate_fp8(const ln3_norm_modulate_fp8_args* args, void* stream) {
  if (!args) return set_error(LN3_EINVAL, "norm_modulate_fp8: null args");
  return norm_modulate_fp8(args, static_cast<cudaStream_t>(stream));
}
int ln3_quantize_fp8_rows(const void* x, int x_bf16, long long ldx, int rows, int D, void* out, long long ldo,
                          float* out_scale, long long out_scale_ld, void* stream) {
  return quantize_fp8_rows(x, x_bf16, ldx, rows, D, out, ldo, out_scale, out_scale_ld,
                           static_cast<cudaStream_t>(stream));
}

}  // extern "C"
