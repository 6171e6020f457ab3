// Flow-matching SDE step: the elementwise tail of one drift evaluation of the transport's Euler-Maruyama and Heun
// samplers around a CFG denoiser, specified in include/ln3b200.h (ln3_flow_sde_step_args).  One launch reads the
// forward output's two CFG halves, the evaluated input and optionally the state, a history buffer and the step's
// noise draw, and writes any of the next state, the next forward's input and the drift.  The arguments are
// validated in api.cu before this is called.
#include "ln3_internal.h"

namespace ln3 {

namespace {

__device__ __forceinline__ float4 ld4(const float* p, long long off) {
  return *reinterpret_cast<const float4*>(p + off);
}

__device__ __forceinline__ float lane(const float4& v, int k) {
  return k == 0 ? v.x : k == 1 ? v.y : k == 2 ? v.z : v.w;
}

__device__ __forceinline__ void set_lane(float4& v, int k, float s) {
  if (k == 0) v.x = s; else if (k == 1) v.y = s; else if (k == 2) v.z = s; else v.w = s;
}

__global__ void __launch_bounds__(256)
flow_sde_step_kernel(const ln3_flow_sde_step_args a) {
  const int r = blockIdx.y;
  const int j = r < a.R ? r : r - a.R;
  const long long row = static_cast<long long>(r) * a.n;
  const long long cond = static_cast<long long>(j) * a.n;
  const long long unc = static_cast<long long>(a.R + j) * a.n;
  const long long nrow = a.noise ? static_cast<long long>((r < a.R ? 0 : a.N) + j % a.N) * a.n : 0;
  const long long n4 = a.n >> 2;
  for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long off = i * 4;
    const float4 fc = ld4(a.f, cond + off), fu = ld4(a.f, unc + off), y = ld4(a.y, row + off);
    const float4 x = a.x ? ld4(a.x, row + off) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 h = a.hist ? ld4(a.hist, row + off) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 w = a.noise ? ld4(a.noise, nrow + off) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 d, ox, oy;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float u = lane(fu, k), yk = lane(y, k);
      const float v = __fadd_rn(u, __fmul_rn(a.cfg_scale, __fsub_rn(lane(fc, k), u)));
      const float sc = __fdiv_rn(__fsub_rn(__fmul_rn(a.t, v), yk), a.var);
      const float dk = a.mode == LN3_SDE_DRIFT ? __fadd_rn(v, __fmul_rn(a.diffusion, sc))
                       : a.mode == LN3_SDE_VELOCITY ? v : sc;
      set_lane(d, k, dk);
      const float terms[5] = {lane(x, k), yk, dk, lane(h, k), lane(w, k)};
      float vx = __fmul_rn(a.cx[0], terms[0]), vy = __fmul_rn(a.cy[0], terms[0]);
#pragma unroll
      for (int q = 1; q < 5; ++q) {
        vx = fmaf(a.cx[q], terms[q], vx);
        vy = fmaf(a.cy[q], terms[q], vy);
      }
      set_lane(ox, k, vx);
      set_lane(oy, k, vy);
    }
    if (a.x_out != nullptr) *reinterpret_cast<float4*>(a.x_out + row + off) = ox;
    if (a.y_out != nullptr) *reinterpret_cast<float4*>(a.y_out + row + off) = oy;
    if (a.hist_out != nullptr) *reinterpret_cast<float4*>(a.hist_out + row + off) = d;
  }
}

}  // namespace

int flow_sde_step(const ln3_flow_sde_step_args* a, cudaStream_t stream) {
  if (a->R == 0 || a->n == 0) return LN3_OK;
  const long long n4 = a->n / 4;
  int gx = static_cast<int>((n4 + 255) / 256);
  if (gx > 1024) gx = 1024;
  dim3 grid(gx, 2 * a->R);
  flow_sde_step_kernel<<<grid, 256, 0, stream>>>(*a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "flow_sde_step launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

}  // namespace ln3
