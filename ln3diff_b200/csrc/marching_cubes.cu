// Marching cubes on the device: replaces the CPU `mcubes.marching_cubes(sigma_grid, mesh_thres)` call of the
// reference's mesh export (nsr/train_util_diffusion.py:221-223) that follows the 192^3 point query
// (vit/vit_triplane.py:2051-2120 -> ln3_query_points).  Integer / index work, HBM- and L2-bound.
//
// Mesh layout (indexed, vertices shared between cells like PyMCubes):
//   * a vertex lives on a lattice edge whose end points straddle the iso value (`v <= iso` on exactly one side);
//     the edge is OWNED by its lower lattice point p = (i, j, k) and numbered by (linear index of p, axis);
//     position = p + t e_axis, t = (iso - f(p)) / (f(p + e_axis) - f(p))   (PyMCubes' linear interpolation)
//   * a cell's triangles come from the generated case tables (mc_tables.h; corner / edge numbering and winding of
//     the classic table, face-consistent ambiguity rule), ordered by the cell's linear index.
// Passes (grid = blocks of 1024 consecutive lattice points, z fastest):
//   count   : per block, number of owned crossed edges and of triangles        -> block_counts
//   scan    : one CTA, exclusive scan of the block counts                        -> block_offsets, totals
//   vertices: recount + intra-block scan; packs (first vertex index << 3 | crossed-axis mask) per lattice
//             point and writes the vertex positions
//   faces   : recount + intra-block scan; resolves the three cube edges of every triangle through the packed
//             per-point word of the owning lattice point
// The volume (28 MB at 192^3) stays in the 50 MB L2 between the passes; nothing else is materialised.
#include "common.cuh"
#include "ln3_internal.h"
#include "mc_tables.h"

namespace ln3 {

namespace {

constexpr int kMcThreads = 256;
constexpr int kMcPerThread = 4;
constexpr int kMcBlockPts = kMcThreads * kMcPerThread;

__constant__ uint8_t c_num_tris[256];
__constant__ uint8_t c_tri_table[256][3 * LN3_MC_MAX_TRIS];
__constant__ uint8_t c_edge_owner[12][4];

struct McDims {
  int nx, ny, nz;
  int n;       // lattice points (< 2^28: all index arithmetic is 32-bit)
  int sy, sx;  // strides of j and i (sz = 1)
  float iso;
};

struct McIjk { int i, j, k; };
// (i, j, k) of linear index p: two 32-bit divisions, once per thread; the thread's further points advance k with carry
__device__ __forceinline__ McIjk mc_ijk(const McDims& d, int p) {
  McIjk c;
  const int t = p / d.nz;
  c.k = p - t * d.nz;
  c.i = t / d.ny;
  c.j = t - c.i * d.ny;
  return c;
}
__device__ __forceinline__ void mc_next(const McDims& d, McIjk& c) {
  if (++c.k == d.nz) {
    c.k = 0;
    if (++c.j == d.ny) c.j = 0, ++c.i;
  }
}

struct McPoint {
  uint32_t mask;  // bit a: owned edge along axis a (0 = x / i, 1 = y / j, 2 = z / k) is crossed
  uint32_t cube;  // case index of the cell whose lower corner this point is (0 when the cell is outside)
  float f0, f1[3];
};

__device__ __forceinline__ McPoint classify(const float* __restrict__ g, const McDims& d, int p, const McIjk& c3) {
  McPoint r;
  r.mask = 0;
  r.cube = 0;
  const bool hx = c3.i + 1 < d.nx, hy = c3.j + 1 < d.ny, hz = c3.k + 1 < d.nz;
  r.f0 = __ldg(g + p);
  const bool in0 = r.f0 <= d.iso;
  r.f1[0] = hx ? __ldg(g + p + d.sx) : r.f0;
  r.f1[1] = hy ? __ldg(g + p + d.sy) : r.f0;
  r.f1[2] = hz ? __ldg(g + p + 1) : r.f0;
  const bool inx = r.f1[0] <= d.iso, iny = r.f1[1] <= d.iso, inz = r.f1[2] <= d.iso;
  if (hx && inx != in0) r.mask |= 1;
  if (hy && iny != in0) r.mask |= 2;
  if (hz && inz != in0) r.mask |= 4;
  if (hx && hy && hz) {
    uint32_t c = (in0 ? 1u : 0u) | (inx ? 2u : 0u) | (iny ? 8u : 0u) | (inz ? 16u : 0u);
    if (__ldg(g + p + d.sx + d.sy) <= d.iso) c |= 4u;          // corner 2 (1,1,0)
    if (__ldg(g + p + d.sx + 1) <= d.iso) c |= 32u;            // corner 5 (1,0,1)
    if (__ldg(g + p + d.sx + d.sy + 1) <= d.iso) c |= 64u;     // corner 6 (1,1,1)
    if (__ldg(g + p + d.sy + 1) <= d.iso) c |= 128u;           // corner 7 (0,1,1)
    r.cube = c;
  }
  return r;
}

// exclusive scan of one value per thread over the CTA (256 threads); returns the exclusive prefix, total in `total`
__device__ __forceinline__ int block_exclusive_scan(int v, int* smem8, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int n = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += n;
  }
  if (lane == 31) smem8[warp] = inc;
  __syncthreads();
  int wbase = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kMcThreads / 32; ++w) {
    const int s = smem8[w];
    if (w < warp) wbase += s;
    tot += s;
  }
  __syncthreads();
  total = tot;
  return wbase + inc - v;
}

__global__ void __launch_bounds__(kMcThreads) mc_count_kernel(const float* __restrict__ g, McDims d, int2* __restrict__ block_counts) {
  __shared__ int sm[2][kMcThreads / 32];
  const int base = blockIdx.x * kMcBlockPts + threadIdx.x * kMcPerThread;
  int nv = 0, nt = 0;
  McIjk c3 = mc_ijk(d, base < d.n ? base : 0);
#pragma unroll
  for (int u = 0; u < kMcPerThread; ++u) {
    const int p = base + u;
    if (p < d.n) {
      const McPoint r = classify(g, d, p, c3);
      nv += __popc(r.mask);
      nt += c_num_tris[r.cube];
    }
    mc_next(d, c3);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    nv += __shfl_xor_sync(0xffffffffu, nv, o);
    nt += __shfl_xor_sync(0xffffffffu, nt, o);
  }
  if ((threadIdx.x & 31) == 0) { sm[0][threadIdx.x >> 5] = nv; sm[1][threadIdx.x >> 5] = nt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0, b = 0;
    for (int w = 0; w < kMcThreads / 32; ++w) { a += sm[0][w]; b += sm[1][w]; }
    block_counts[blockIdx.x] = make_int2(a, b);
  }
}

// one CTA of 1024 threads: exclusive scan of (nv, nt) over the blocks; totals[0..1] = sums
__global__ void __launch_bounds__(1024) mc_scan_kernel(const int2* __restrict__ counts, int nblocks, int2* __restrict__ offsets,
                                                       int* __restrict__ totals) {
  __shared__ int2 wsum[32];
  __shared__ int2 carry_s;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry_s = make_int2(0, 0);
  __syncthreads();
  for (int b0 = 0; b0 < nblocks; b0 += 1024) {
    const int b = b0 + threadIdx.x;
    const int2 v = b < nblocks ? counts[b] : make_int2(0, 0);
    int2 inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int nx = __shfl_up_sync(0xffffffffu, inc.x, o), ny = __shfl_up_sync(0xffffffffu, inc.y, o);
      if (lane >= o) { inc.x += nx; inc.y += ny; }
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    int2 wb = make_int2(0, 0), tot = make_int2(0, 0);
    for (int w = 0; w < 32; ++w) {
      const int2 s = wsum[w];
      if (w < warp) { wb.x += s.x; wb.y += s.y; }
      tot.x += s.x; tot.y += s.y;
    }
    const int2 carry = carry_s;
    if (b < nblocks) offsets[b] = make_int2(carry.x + wb.x + inc.x - v.x, carry.y + wb.y + inc.y - v.y);
    __syncthreads();
    if (threadIdx.x == 0) carry_s = make_int2(carry.x + tot.x, carry.y + tot.y);
    __syncthreads();
  }
  if (threadIdx.x == 0) { totals[0] = carry_s.x; totals[1] = carry_s.y; }
}

struct McAffine { float s[3], o[3]; };

__global__ void __launch_bounds__(kMcThreads) mc_vertices_kernel(const float* __restrict__ g, McDims d, const int2* __restrict__ block_offsets,
                                                                 uint32_t* __restrict__ vert_index, float* __restrict__ vertices,
                                                                 int max_vertices, McAffine aff) {
  __shared__ int sm[kMcThreads / 32];
  const int base = blockIdx.x * kMcBlockPts + threadIdx.x * kMcPerThread;
  McPoint r[kMcPerThread];
  int nv = 0;
  const McIjk c0 = mc_ijk(d, base < d.n ? base : 0);
  McIjk c3 = c0;
#pragma unroll
  for (int u = 0; u < kMcPerThread; ++u) {
    const int p = base + u;
    if (p < d.n) r[u] = classify(g, d, p, c3);
    else { r[u].mask = 0; r[u].cube = 0; }
    nv += __popc(r[u].mask);
    mc_next(d, c3);
  }
  c3 = c0;
  int total;
  int first = block_offsets[blockIdx.x].x + block_exclusive_scan(nv, sm, total);
#pragma unroll
  for (int u = 0; u < kMcPerThread; ++u, mc_next(d, c3)) {
    const int p = base + u;
    if (p >= d.n) break;
    vert_index[p] = (static_cast<uint32_t>(first) << 3) | r[u].mask;
    if (r[u].mask) {
      const float c[3] = {static_cast<float>(c3.i), static_cast<float>(c3.j), static_cast<float>(c3.k)};
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (r[u].mask >> a & 1) {
          if (first < max_vertices) {
            const float tt = __fdiv_rn(d.iso - r[u].f0, r[u].f1[a] - r[u].f0);
            float* v = vertices + static_cast<long long>(first) * 3;
#pragma unroll
            for (int q = 0; q < 3; ++q) v[q] = fmaf(c[q] + (q == a ? tt : 0.f), aff.s[q], aff.o[q]);
          }
          ++first;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(kMcThreads) mc_faces_kernel(const float* __restrict__ g, McDims d, const int2* __restrict__ block_offsets,
                                                              const uint32_t* __restrict__ vert_index, int* __restrict__ faces,
                                                              int max_faces) {
  __shared__ int sm[kMcThreads / 32];
  const int base = blockIdx.x * kMcBlockPts + threadIdx.x * kMcPerThread;
  uint32_t cube[kMcPerThread];
  int nt = 0;
  McIjk c3 = mc_ijk(d, base < d.n ? base : 0);
#pragma unroll
  for (int u = 0; u < kMcPerThread; ++u) {
    const int p = base + u;
    cube[u] = p < d.n ? classify(g, d, p, c3).cube : 0u;
    nt += c_num_tris[cube[u]];
    mc_next(d, c3);
  }
  int total;
  int first = block_offsets[blockIdx.x].y + block_exclusive_scan(nt, sm, total);
  if (total == 0) return;
#pragma unroll
  for (int u = 0; u < kMcPerThread; ++u) {
    const int n = c_num_tris[cube[u]];
    if (n == 0) continue;
    const int p = base + u;
    for (int r = 0; r < n; ++r, ++first) {
      if (first >= max_faces) continue;
      int idx[3];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int e = c_tri_table[cube[u]][3 * r + q];
        const int owner = p + c_edge_owner[e][0] * d.sx + c_edge_owner[e][1] * d.sy + c_edge_owner[e][2];
        const uint32_t w = __ldg(vert_index + owner);
        const int axis = c_edge_owner[e][3];
        idx[q] = static_cast<int>(w >> 3) + __popc(w & 7u & ((1u << axis) - 1u));
      }
      int* f = faces + static_cast<long long>(first) * 3;
      f[0] = idx[0]; f[1] = idx[1]; f[2] = idx[2];
    }
  }
}

int upload_tables() {
  static DeviceOnce once;
  return once.run([] {
    cudaError_t e = cudaMemcpyToSymbol(c_num_tris, kMcNumTris, sizeof(kMcNumTris));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_tri_table, kMcTriTable, sizeof(kMcTriTable));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_edge_owner, kMcEdgeOwner, sizeof(kMcEdgeOwner));
    return e == cudaSuccess ? LN3_OK : set_error(LN3_ECUDA, "marching_cubes: table upload: %s", cudaGetErrorString(e));
  });
}

struct McLayout {
  int nblocks;
  size_t off_counts, off_offsets, off_index, total;
};

McLayout mc_layout(long long n) {
  McLayout l;
  l.nblocks = static_cast<int>((n + kMcBlockPts - 1) / kMcBlockPts);
  auto up = [](size_t v) { return (v + 255) & ~static_cast<size_t>(255); };
  l.off_counts = 0;
  l.off_offsets = up(sizeof(int2) * l.nblocks);
  l.off_index = l.off_offsets + up(sizeof(int2) * l.nblocks);
  l.total = l.off_index + up(sizeof(uint32_t) * static_cast<size_t>(n));
  return l;
}

int mc_check(const ln3_marching_cubes_args* a, McDims& d, McLayout& l) {
  if (!a->grid || !a->workspace || !a->totals) return set_error(LN3_EINVAL, "marching_cubes: null grid / workspace / totals");
  if (a->nx < 2 || a->ny < 2 || a->nz < 2) return set_error(LN3_EINVAL, "marching_cubes: every dimension must be >= 2");
  d.nx = a->nx; d.ny = a->ny; d.nz = a->nz;
  const long long n64 = static_cast<long long>(a->nx) * a->ny * a->nz;
  if (n64 >= (1ll << 28)) return set_error(LN3_EUNSUPPORTED, "marching_cubes: more than 2^28 lattice points");
  d.n = static_cast<int>(n64);
  d.sy = a->nz;
  d.sx = a->ny * a->nz;
  d.iso = a->iso;
  l = mc_layout(d.n);
  if (a->workspace_bytes < l.total) return set_error(LN3_EINVAL, "marching_cubes: workspace too small (%zu < %zu)", a->workspace_bytes, l.total);
  if (reinterpret_cast<uintptr_t>(a->workspace) & 255) return set_error(LN3_EINVAL, "marching_cubes: workspace must be 256-byte aligned");
  return LN3_OK;
}

}  // namespace

size_t marching_cubes_workspace_bytes(int nx, int ny, int nz) {
  if (nx < 2 || ny < 2 || nz < 2) return 0;
  return mc_layout(static_cast<long long>(nx) * ny * nz).total;
}

int marching_cubes_count(const ln3_marching_cubes_args* a, cudaStream_t stream) {
  McDims d;
  McLayout l;
  if (int rc = mc_check(a, d, l)) return rc;
  if (int rc = upload_tables()) return rc;
  uint8_t* ws = static_cast<uint8_t*>(a->workspace);
  int2* counts = reinterpret_cast<int2*>(ws + l.off_counts);
  int2* offsets = reinterpret_cast<int2*>(ws + l.off_offsets);
  mc_count_kernel<<<l.nblocks, kMcThreads, 0, stream>>>(a->grid, d, counts);
  mc_scan_kernel<<<1, 1024, 0, stream>>>(counts, l.nblocks, offsets, a->totals);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "marching_cubes_count launch: %s", cudaGetErrorString(e));
  count_launch(2);
  return LN3_OK;
}

int marching_cubes_emit(const ln3_marching_cubes_args* a, cudaStream_t stream) {
  McDims d;
  McLayout l;
  if (int rc = mc_check(a, d, l)) return rc;
  if (!a->vertices || !a->faces || a->max_vertices < 0 || a->max_faces < 0)
    return set_error(LN3_EINVAL, "marching_cubes_emit: null outputs");
  if (int rc = upload_tables()) return rc;
  uint8_t* ws = static_cast<uint8_t*>(a->workspace);
  const int2* offsets = reinterpret_cast<const int2*>(ws + l.off_offsets);
  uint32_t* index = reinterpret_cast<uint32_t*>(ws + l.off_index);
  McAffine aff;
  for (int q = 0; q < 3; ++q) { aff.s[q] = a->scale[q]; aff.o[q] = a->offset[q]; }
  mc_vertices_kernel<<<l.nblocks, kMcThreads, 0, stream>>>(a->grid, d, offsets, index, a->vertices, a->max_vertices, aff);
  mc_faces_kernel<<<l.nblocks, kMcThreads, 0, stream>>>(a->grid, d, offsets, index, a->faces, a->max_faces);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(LN3_ECUDA, "marching_cubes_emit launch: %s", cudaGetErrorString(e));
  count_launch(2);
  return LN3_OK;
}

}  // namespace ln3
