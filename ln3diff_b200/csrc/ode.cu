// Grouped adaptive explicit Runge-Kutta: the per-attempt arithmetic of transport/rk.py:odeint_rk_adaptive (dopri5,
// bosh3, fehlberg2, adaptive_heun) for G independent groups of rows in one batch, with the accept / reject control on
// the device.  Each kernel takes the method and reads its Butcher tableau from c_tab.
//   ode_stage    y_stage = y + dt_g sum_j beta_ij k_j and the per-row fp32 forward time (one launch per stage); for
//                a tableau that is not FSAL, the solution y1 = y + dt_g sum_j c_sol_j k_j after the last stage
//   ode_norm     fixed-partition float64 partial sums of squared scaled quantities, per (row, 1024-element chunk)
//   ode_control  one CTA per group: its rows' partials in row, chunk order -> ratio / step controller / counters
//   ode_commit   y <- y1, f0 <- f1 = k[last] on accept, the dense output at t_end when the group finishes
// Every fp32 operation that the host solver performs on tensors is individually rounded here in the same order (no
// FMA contraction), and every float64 scalar operation likewise, so the only intended difference from the host
// solver is the order of the error-norm reduction.  Reference call sites are cited in include/ln3b200.h.
#include <cmath>
#include <cstdint>

#include "ln3_internal.h"

namespace ln3 {

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = kThreads * 4;   // elements per partial sum: one float4 per thread
constexpr int kMethods = 4;            // LN3_ODE_DOPRI5 .. LN3_ODE_ADAPTIVE_HEUN

// transport/rk.py TABLEAUS (the same double expressions).  beta rows, c_sol, c_err and c_mid are zero-padded to
// 7 terms (k_0 = f0 .. k_6); a zero coefficient is skipped, as _lincomb skips it.
struct Tableau {
  int stages;        // stage forwards per attempt (beta rows)
  int fsal;          // c_sol is the last beta row with a trailing 0: y1 is the last stage's input
  double expo;       // 1 / order: the step controller's and the initial step's exponent
  double alpha[6];
  double beta[6][7];
  double c_sol[7];
  double c_err[7];
  double c_mid[7];
};

constexpr Tableau kTab[kMethods] = {
    {6, 1, 1.0 / 5,   // dopri5
     {1.0 / 5, 3.0 / 10, 4.0 / 5, 8.0 / 9, 1.0, 1.0},
     {{1.0 / 5},
      {3.0 / 40, 9.0 / 40},
      {44.0 / 45, -56.0 / 15, 32.0 / 9},
      {19372.0 / 6561, -25360.0 / 2187, 64448.0 / 6561, -212.0 / 729},
      {9017.0 / 3168, -355.0 / 33, 46732.0 / 5247, 49.0 / 176, -5103.0 / 18656},
      {35.0 / 384, 0.0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84}},
     {35.0 / 384, 0.0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84, 0.0},
     {35.0 / 384 - 1951.0 / 21600, 0.0, 500.0 / 1113 - 22642.0 / 50085, 125.0 / 192 - 451.0 / 720,
      -2187.0 / 6784 - -12231.0 / 42400, 11.0 / 84 - 649.0 / 6300, -1.0 / 60.0},
     {6025192743.0 / 30085553152.0 / 2, 0.0, 51252292925.0 / 65400821598.0 / 2,
      -2691868925.0 / 45128329728.0 / 2, 187940372067.0 / 1594534317056.0 / 2,
      -1776094331.0 / 19743644256.0 / 2, 11237099.0 / 235043384.0 / 2}},
    {3, 1, 1.0 / 3,   // bosh3 (Bogacki-Shampine 3(2))
     {1.0 / 2, 3.0 / 4, 1.0},
     {{1.0 / 2}, {0.0, 3.0 / 4}, {2.0 / 9, 1.0 / 3, 4.0 / 9}},
     {2.0 / 9, 1.0 / 3, 4.0 / 9, 0.0},
     {2.0 / 9 - 7.0 / 24, 1.0 / 3 - 1.0 / 4, 4.0 / 9 - 1.0 / 3, -1.0 / 8},
     {0.0, 0.5, 0.0, 0.0}},
    {2, 0, 1.0 / 2,   // fehlberg2 (Runge-Kutta-Fehlberg 2(1))
     {1.0 / 2, 1.0},
     {{1.0 / 2}, {1.0 / 256, 255.0 / 256}},
     {1.0 / 512, 255.0 / 256, 1.0 / 512},
     {-1.0 / 512, 0.0, 1.0 / 512},
     {0.0, 0.5, 0.0}},
    {1, 0, 1.0 / 2,   // adaptive_heun (Heun-Euler 2(1))
     {1.0},
     {{1.0}},
     {0.5, 0.5},
     {0.5, -0.5},
     {0.5, 0.0}},
};
__constant__ Tableau c_tab[kMethods] = {kTab[0], kTab[1], kTab[2], kTab[3]};

enum { MODE_ERR = 0, MODE_INIT0 = 1, MODE_INIT1 = 2 };

__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
// Python's builtins: max(a, b) keeps a unless b > a, min(a, b) keeps a unless b < a (NaN handling included)
__device__ __forceinline__ double py_max(double a, double b) { return b > a ? b : a; }
__device__ __forceinline__ double py_min(double a, double b) { return b < a ? b : a; }

__device__ __forceinline__ void ld4(const float* p, long long off, float v[4]) {
  const float4 q = *reinterpret_cast<const float4*>(p + off);
  v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
}
__device__ __forceinline__ void st4(float* p, long long off, const float v[4]) {
  *reinterpret_cast<float4*>(p + off) = make_float4(v[0], v[1], v[2], v[3]);
}

// k_j of the current attempt: k_0 = f0, k_j = a.k[j-1]
__device__ __forceinline__ const float* kptr(const ln3_ode_args& a, int j) { return j == 0 ? a.f0 : a.k[j - 1]; }

// ------------------------------------------------------------------ stage combination
// stage 1..stages: the stage inputs; stage == stages + 1 (tableaus that are not FSAL): y1 = y + dt sum_j c_sol_j k_j
// into y_stage, no forward time.
__global__ void __launch_bounds__(kThreads) ode_stage_kernel(const ln3_ode_args a, int method, int stage) {
  const int r = blockIdx.y;
  const ln3_ode_group* s = a.state + a.row_group[r];
  if (s->status != LN3_ODE_RUNNING) return;
  const double t = s->t, dt = s->dt;
  const long long base = static_cast<long long>(r) * a.n_per_sample;
  const long long n4 = a.n_per_sample >> 2;
  if (stage == 0) {   // initial-step probe: y0 + h0 * f0 at t0 + h0
    if (blockIdx.x == 0 && threadIdx.x == 0) a.t_rows[r] = static_cast<float>(__dadd_rn(t, dt));
    const float h = static_cast<float>(dt);
    for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += static_cast<long long>(gridDim.x) * blockDim.x) {
      float y[4], f[4];
      ld4(a.y, base + i * 4, y);
      ld4(a.f0, base + i * 4, f);
#pragma unroll
      for (int e = 0; e < 4; ++e) y[e] = add(y[e], mul(h, f[e]));
      st4(a.y_stage, base + i * 4, y);
    }
    return;
  }
  const Tableau& tb = c_tab[method];
  const int row = stage - 1;
  const bool sol = row == tb.stages;
  const double* coef = sol ? tb.c_sol : tb.beta[row];
  if (!sol && blockIdx.x == 0 && threadIdx.x == 0)
    a.t_rows[r] = static_cast<float>(__dadd_rn(t, __dmul_rn(tb.alpha[row], dt)));
  float cf[7];
#pragma unroll
  for (int j = 0; j < 7; ++j) cf[j] = static_cast<float>(__dmul_rn(coef[j], dt));
  for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float acc[4], k[4];
    ld4(a.y, base + i * 4, acc);
    for (int j = 0; j < stage; ++j) {
      if (coef[j] == 0.0) continue;   // _lincomb skips zero coefficients
      ld4(kptr(a, j), base + i * 4, k);
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[e] = add(acc[e], mul(k[e], cf[j]));
    }
    st4(a.y_stage, base + i * 4, acc);
  }
}

// ------------------------------------------------------------------ deterministic partial sums
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sum of v over the CTA in a fixed order (xor tree per warp, warps in index order); valid in thread 0.
__device__ __forceinline__ double block_sum_d(double v, double* sh) {
  v = warp_sum_d(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; ++w) s += sh[w];
  return s;
}

// grid (nchunk, B): partial[(r * nchunk + c) * 2 + q] = sum over chunk c of row r of q-th squared quantity
__global__ void __launch_bounds__(kThreads) ode_norm_kernel(const ln3_ode_args a, int method, int mode) {
  __shared__ double sh[kThreads / 32];
  const int r = blockIdx.y, c = blockIdx.x;
  if (a.state[a.row_group[r]].status != LN3_ODE_RUNNING) return;
  const long long base = static_cast<long long>(r) * a.n_per_sample;
  const long long i4 = static_cast<long long>(c) * kThreads + threadIdx.x;
  const float atol = static_cast<float>(a.atol), rtol = static_cast<float>(a.rtol);
  double s0 = 0.0, s1 = 0.0;
  if (i4 < (a.n_per_sample >> 2)) {
    const long long off = base + i4 * 4;
    float y[4], f[4];
    ld4(a.y, off, y);
    if (mode == MODE_ERR) {
      const double dt = a.state[a.row_group[r]].dt;
      float err[4] = {0.f, 0.f, 0.f, 0.f}, k[4], y1[4];
      const double* c_err = c_tab[method].c_err;
      for (int j = 0; j < 7; ++j) {
        if (c_err[j] == 0.0) continue;
        const float cj = static_cast<float>(__dmul_rn(c_err[j], dt));
        ld4(kptr(a, j), off, k);
#pragma unroll
        for (int e = 0; e < 4; ++e) err[e] = add(err[e], mul(k[e], cj));
      }
      ld4(a.y_stage, off, y1);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float tol = add(atol, mul(rtol, fmaxf(fabsf(y[e]), fabsf(y1[e]))));
        const float q = __fdiv_rn(err[e], tol);
        s0 += static_cast<double>(mul(q, q));
      }
    } else {
      ld4(a.f0, off, f);
      float k[4];
      if (mode == MODE_INIT1) ld4(a.k[0], off, k);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float scale = add(atol, mul(fabsf(y[e]), rtol));
        if (mode == MODE_INIT0) {
          const float q0 = __fdiv_rn(y[e], scale), q1 = __fdiv_rn(f[e], scale);
          s0 += static_cast<double>(mul(q0, q0));
          s1 += static_cast<double>(mul(q1, q1));
        } else {
          const float q = __fdiv_rn(sub(k[e], f[e]), scale);
          s0 += static_cast<double>(mul(q, q));
        }
      }
    }
  }
  s0 = block_sum_d(s0, sh);
  s1 = block_sum_d(s1, sh);
  if (threadIdx.x == 0) {
    double* p = static_cast<double*>(a.workspace) + (static_cast<long long>(r) * gridDim.x + c) * 2;
    p[0] = s0;
    p[1] = s1;
  }
}

// The checks odeint_dopri5 makes before every attempt.
__device__ __forceinline__ void check_next_attempt(ln3_ode_group& s, int max_num_steps) {
  if (s.accepted + s.rejected >= max_num_steps) s.status = LN3_ODE_EMAXSTEPS;
  else if (!(__dadd_rn(s.t, s.dt) > s.t)) s.status = LN3_ODE_EUNDERFLOW;
}

// grid G: group g's sums over its rows (ascending) and their chunks (ascending), then the scalar control logic.
__global__ void __launch_bounds__(kThreads) ode_control_kernel(const ln3_ode_args a, int method, int mode, int nchunk) {
  __shared__ double sh[kThreads / 32];
  const int g = blockIdx.x;
  ln3_ode_group* sp = a.state + g;
  if (sp->status != LN3_ODE_RUNNING) {
    if (threadIdx.x == 0) sp->event = 0;
    return;
  }
  const double* part = static_cast<const double*>(a.workspace);
  double s0 = 0.0, s1 = 0.0;
  int rows = 0;
  for (int r = 0; r < a.B; ++r) {
    if (a.row_group[r] != g) continue;
    ++rows;
    for (int c = threadIdx.x; c < nchunk; c += kThreads) {
      s0 += part[(static_cast<long long>(r) * nchunk + c) * 2];
      s1 += part[(static_cast<long long>(r) * nchunk + c) * 2 + 1];
    }
  }
  s0 = block_sum_d(s0, sh);
  s1 = block_sum_d(s1, sh);
  if (threadIdx.x != 0) return;
  ln3_ode_group s = *sp;
  const double count = static_cast<double>(rows) * static_cast<double>(a.n_per_sample);
  if (mode == MODE_INIT0) {   // _initial_step: d0, d1 -> h0 (the probe's step)
    const double d0 = sqrt(s0 / count), d1 = sqrt(s1 / count);
    s.dt = (d0 < 1e-5 || d1 < 1e-5) ? 1e-6 : 0.01 * d0 / d1;
    s.aux = d1;
    s.event = 0;
  } else if (mode == MODE_INIT1) {   // d2 from the probe's forward, h1, dt = min(100 h0, h1)
    const double h0 = s.dt, d1 = s.aux;
    const double d2 = sqrt(s0 / count) / h0;
    double h1;
    if (d1 <= 1e-15 && d2 <= 1e-15) h1 = py_max(1e-6, h0 * 1e-3);
    else h1 = pow(0.01 / py_max(d1, d2), c_tab[method].expo);
    s.dt = py_min(100 * h0, h1);
    s.nfe = 2;
    s.event = 0;
    check_next_attempt(s, a.max_num_steps);
  } else {
    const double ratio = sqrt(s0 / count), dt = s.dt;
    s.ratio = ratio;
    s.dt_step = dt;
    s.nfe += c_tab[method].stages;
    if (ratio <= 1.0) {
      s.t_prev = s.t;
      s.t = __dadd_rn(s.t, dt);
      s.accepted += 1;
      s.event = s.t >= a.t_end ? 2 : 1;
      if (s.event == 2) s.status = LN3_ODE_DONE;
    } else {
      s.rejected += 1;
      s.event = 0;
    }
    if (ratio == 0.0) {
      s.dt = dt * a.ifactor;
    } else {
      const double df = ratio < 1.0 ? 1.0 : a.dfactor;
      s.dt = dt * py_min(a.ifactor, py_max(a.safety / pow(ratio, c_tab[method].expo), df));
    }
    if (s.status == LN3_ODE_RUNNING) check_next_attempt(s, a.max_num_steps);
  }
  *sp = s;
}

// ------------------------------------------------------------------ commit + dense output
__global__ void __launch_bounds__(kThreads) ode_commit_kernel(const ln3_ode_args a, int method) {
  const int r = blockIdx.y;
  const ln3_ode_group* sp = a.state + a.row_group[r];
  const int ev = sp->event;
  if (ev == 0) return;
  const double dt = sp->dt_step;
  const long long base = static_cast<long long>(r) * a.n_per_sample;
  const long long n4 = a.n_per_sample >> 2;
  const Tableau& tb = c_tab[method];
  const float* f1p = a.k[tb.stages - 1];   // f1 = k[last], also when y1 was recomputed from c_sol
  float cm[7];
  float fdt = 0.f, f2dt = 0.f, x1 = 0.f, x2 = 0.f, x3 = 0.f, x4 = 0.f;
  if (ev == 2) {
#pragma unroll
    for (int j = 0; j < 7; ++j) cm[j] = static_cast<float>(__dmul_rn(tb.c_mid[j], dt));
    fdt = static_cast<float>(dt);
    f2dt = static_cast<float>(2 * dt);
    const double x = (a.t_end - sp->t_prev) / (sp->t - sp->t_prev);   // _interp_eval
    const double xp2 = x * x, xp3 = xp2 * x, xp4 = xp3 * x;
    x1 = static_cast<float>(x); x2 = static_cast<float>(xp2); x3 = static_cast<float>(xp3); x4 = static_cast<float>(xp4);
  }
  for (long long i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long off = base + i * 4;
    float y[4], f0[4], y1[4], f1[4];
    ld4(a.y, off, y);
    ld4(a.y_stage, off, y1);
    ld4(f1p, off, f1);
    if (ev == 2) {
      ld4(a.f0, off, f0);
      float ym[4], k[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) ym[e] = y[e];
      for (int j = 0; j < 7; ++j) {
        if (tb.c_mid[j] == 0.0) continue;
        ld4(kptr(a, j), off, k);
#pragma unroll
        for (int e = 0; e < 4; ++e) ym[e] = add(ym[e], mul(k[e], cm[j]));
      }
      float o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        // a = 2 dt (f1 - f0) - 8 (y1 + y) + 16 y_mid;  b = dt (5 f0 - 3 f1) + 18 y + 14 y1 - 32 y_mid;
        // c = dt (f1 - 4 f0) - 11 y - 5 y1 + 16 y_mid;  interp = [y, dt f0, c, b, a]
        const float qa = add(sub(mul(f2dt, sub(f1[e], f0[e])), mul(8.f, add(y1[e], y[e]))), mul(16.f, ym[e]));
        const float qb = sub(add(add(mul(fdt, sub(mul(5.f, f0[e]), mul(3.f, f1[e]))), mul(18.f, y[e])),
                                 mul(14.f, y1[e])), mul(32.f, ym[e]));
        const float qc = add(sub(sub(mul(fdt, sub(f1[e], mul(4.f, f0[e]))), mul(11.f, y[e])), mul(5.f, y1[e])),
                             mul(16.f, ym[e]));
        float tot = add(y[e], mul(x1, mul(fdt, f0[e])));
        tot = add(tot, mul(x2, qc));
        tot = add(tot, mul(x3, qb));
        tot = add(tot, mul(x4, qa));
        o[e] = tot;
      }
      st4(a.out, off, o);
    }
    st4(a.y, off, y1);
    st4(a.f0, off, f1);
  }
}

long long nchunks(long long n) { return (n + kChunk - 1) / kChunk; }

int launched(const char* what, int n) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "%s launch: %s", what, cudaGetErrorString(e));
  count_launch(n);
  return LN3_OK;
}

dim3 row_grid(const ln3_ode_args* a) {
  long long gx = (a->n_per_sample / 4 + kThreads - 1) / kThreads;
  if (gx > 1024) gx = 1024;
  return dim3(static_cast<unsigned>(gx), a->B);
}

int launch_norm_control(const ln3_ode_args* a, int method, int mode, cudaStream_t stream) {
  const long long nc = nchunks(a->n_per_sample);
  if (nc > 0x7fffffffLL) return set_error(LN3_EUNSUPPORTED, "ode: n_per_sample too large");
  ode_norm_kernel<<<dim3(static_cast<unsigned>(nc), a->B), kThreads, 0, stream>>>(*a, method, mode);
  ode_control_kernel<<<a->G, kThreads, 0, stream>>>(*a, method, mode, static_cast<int>(nc));
  return launched("ode_norm/control", 2);
}

}  // namespace

// Arguments are validated by the ln3_ode_* entry points (api.cu), the method by ode_stages.
int ode_stages(int method) {
  if (method < 0 || method >= kMethods) return set_error(LN3_EUNSUPPORTED, "ode: unknown method %d", method);
  return kTab[method].stages;
}

size_t ode_workspace_bytes(int B, long long n_per_sample) {
  return static_cast<size_t>(B) * static_cast<size_t>(nchunks(n_per_sample)) * 2 * sizeof(double);
}

int ode_stage(const ln3_ode_args* a, int method, int stage, cudaStream_t stream) {
  ode_stage_kernel<<<row_grid(a), kThreads, 0, stream>>>(*a, method, stage);
  return launched("ode_stage", 1);
}

int ode_initial_step(const ln3_ode_args* a, int method, int phase, cudaStream_t stream) {
  return launch_norm_control(a, method, phase == 0 ? MODE_INIT0 : MODE_INIT1, stream);
}

int ode_step(const ln3_ode_args* a, int method, cudaStream_t stream) {
  if (!kTab[method].fsal) {   // y_stage <- y1 = y + dt c_sol . k; f1 stays k[last] (torchdiffeq's _runge_kutta_step)
    const int rc = ode_stage(a, method, kTab[method].stages + 1, stream);
    if (rc != LN3_OK) return rc;
  }
  const int rc = launch_norm_control(a, method, MODE_ERR, stream);
  if (rc != LN3_OK) return rc;
  ode_commit_kernel<<<row_grid(a), kThreads, 0, stream>>>(*a, method);
  return launched("ode_commit", 1);
}

}  // namespace ln3
