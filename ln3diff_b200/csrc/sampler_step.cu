// Fused sampler step: the elementwise tail of one denoiser evaluation of every sgm EDM-family sampler
// (Euler-ancestral, Heun, DPM++ 2S-a, DPM++ 2M, LMS), specified in include/ln3b200.h (ln3_sampler_step_args).
// One launch per evaluation reads the state, the evaluation input, the two CFG halves of the network output and up
// to three history buffers, and writes the next state, both halves of the next forward's input and the new history
// entry.  The arguments are validated in api.cu before this is called.
#include "ln3_internal.h"

namespace ln3 {

namespace {

__device__ __forceinline__ float4 ld4(const float* p, long long off) {
  return *reinterpret_cast<const float4*>(p + off);
}

// acc += w * v, per lane
__device__ __forceinline__ void fma4(float4& acc, float w, const float4 v) {
  acc.x = fmaf(w, v.x, acc.x); acc.y = fmaf(w, v.y, acc.y);
  acc.z = fmaf(w, v.z, acc.z); acc.w = fmaf(w, v.w, acc.w);
}

__global__ void __launch_bounds__(256)
sampler_step_kernel(const ln3_sampler_step_args a) {
  const int b = blockIdx.y;
  const float4* cf = reinterpret_cast<const float4*>(a.coef + b * 12);
  const float4 c0 = cf[0];   // k0 k1 k2 a
  const float4 c1 = cf[1];   // b  c  h0 h1
  const float4 c2 = cf[2];   // h2 s  -  -
  const long long base = static_cast<long long>(b) * a.n_per_sample;
  const long long second = static_cast<long long>(a.B) * a.n_per_sample;   // eval_out's conditional half
  const long long n4 = a.n_per_sample >> 2;
  for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long off = base + i * 4;
    const float4 xe = ld4(a.x_eval, off);
    const float4 nu = ld4(a.net_u, off);
    float4 e = make_float4(c0.x * xe.x, c0.x * xe.y, c0.x * xe.z, c0.x * xe.w);
    fma4(e, c0.y, nu);
    if (a.net_c != nullptr) fma4(e, c0.z, ld4(a.net_c, off));
    const float4 x = ld4(a.x, off);
    float4 v = make_float4(c0.w * x.x, c0.w * x.y, c0.w * x.z, c0.w * x.w);
    fma4(v, c1.x, xe);
    fma4(v, c1.y, e);
    if (a.hist[0] != nullptr) fma4(v, c1.z, ld4(a.hist[0], off));
    if (a.hist[1] != nullptr) fma4(v, c1.w, ld4(a.hist[1], off));
    if (a.hist[2] != nullptr) fma4(v, c2.x, ld4(a.hist[2], off));
    if (a.noise != nullptr) fma4(v, c2.y, ld4(a.noise, off));
    if (a.x_out != nullptr) *reinterpret_cast<float4*>(a.x_out + off) = v;
    if (a.eval_out != nullptr) {
      *reinterpret_cast<float4*>(a.eval_out + off) = v;
      *reinterpret_cast<float4*>(a.eval_out + second + off) = v;
    }
    if (a.hist_out != nullptr) *reinterpret_cast<float4*>(a.hist_out + off) = e;
  }
}

}  // namespace

int sampler_step(const ln3_sampler_step_args* a, cudaStream_t stream) {
  if (a->B == 0 || a->n_per_sample == 0) return LN3_OK;
  const long long n4 = a->n_per_sample / 4;
  int gx = static_cast<int>((n4 + 255) / 256);
  if (gx > 1024) gx = 1024;
  dim3 grid(gx, a->B);
  sampler_step_kernel<<<grid, 256, 0, stream>>>(*a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "sampler_step launch: %s", cudaGetErrorString(e));
  count_launch();
  return LN3_OK;
}

}  // namespace ln3
