// Coarse-to-fine evaluation of the SDF grid (DESIGN.md §4.9): the network runs only at the grid points of blocks that can
// hold the iso-surface, every other point is filled by trilinear interpolation, and the result is a complete dense
// [R,R,R] grid for the unchanged marching cubes.  Definitions, shared with the numpy twin oracle/adaptive_oracle.py:
//   * s0 = the largest power of two <= 16 that divides res (s0 = 1: the dense grid); the stride-s0 lattice is evaluated
//     first, then levels s = s0, s0/2, ..., 2;
//   * level s classifies the blocks of size s (closed cubes of lattice points, origin a multiple of s): every block at the
//     first level, later only the children of active parents.  A block is active when its 8 corners are not all on one
//     side of iso under marching cubes' predicate v < iso, or when some corner has |v - iso| <= tau_s (float32),
//     tau_s = float32(band * (s/2) * sqrt(hx^2 + hy^2 + hz^2)) computed in float64;
//   * the stride-s/2 points of active blocks that are not yet evaluated form the level's list, in ascending linear index
//     (mark byte -> per-chunk counts -> the library's exclusive scan -> in-order write);
//   * fill: a point never evaluated takes the trilinear interpolation (x, then y, then z; (1-t)*a + t*b rounded per
//     operation, no FMA) of the corners of the finest classified inactive block containing it; among several blocks of
//     that level the first in (z, y, x) order, each axis trying the block starting at or below the point first.
// Byte-per-point passes over the grid (1 B mark, states per block); the network evaluation is the cost.
#include <algorithm>
#include <cmath>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "adaptive_common.cuh"
#include "common.cuh"

namespace disn {
namespace {

constexpr int AD_THREADS = 256;
constexpr int AD_ITEMS = 8;
constexpr int AD_CHUNK = AD_THREADS * AD_ITEMS;   // mark bytes per compaction block

inline unsigned blocks_of(int64_t n) { return (unsigned)((n + AD_THREADS - 1) / AD_THREADS); }

struct Levels {
  int n;                          // number of refinement levels (log2 s0)
  int s[AD_MAX_LEVELS];           // block size of level l (s0 >> l)
  int nb[AD_MAX_LEVELS];          // blocks per axis (res / s)
  int64_t off[AD_MAX_LEVELS];     // offset of level l's states in the state buffer
};

// the stride-s lattice in ascending linear index; its points are marked evaluated
__global__ void __launch_bounds__(AD_THREADS) lattice_kernel(int R, int s, int M, int32_t* __restrict__ list,
                                                             uint8_t* __restrict__ mark) {
  const int64_t j = (int64_t)blockIdx.x * AD_THREADS + threadIdx.x;
  if (j >= (int64_t)M * M * M) return;
  const int xi = (int)(j % M), yi = (int)((j / M) % M), zi = (int)(j / ((int64_t)M * M));
  const int32_t i = (int32_t)(((int64_t)zi * s * R + (int64_t)yi * s) * R + (int64_t)xi * s);
  list[j] = i;
  mark[i] = 1;
}

// grid[list[j]] = src[j] (network values) or field[list[j]] (given field)
__global__ void __launch_bounds__(AD_THREADS) scatter_kernel(const int32_t* __restrict__ list, int64_t n,
                                                             const float* __restrict__ vals, const float* __restrict__ field,
                                                             float* __restrict__ grid) {
  const int64_t j = (int64_t)blockIdx.x * AD_THREADS + threadIdx.x;
  if (j >= n) return;
  const int32_t i = list[j];
  grid[i] = field ? field[i] : vals[j];
}

// one thread per block of size s: state 0 = not classified (parent inactive), 1 = inactive, 2 = active; an active block
// marks its not yet evaluated stride-s/2 points with 2 (concurrent writers store the same value)
__global__ void __launch_bounds__(AD_THREADS) classify_kernel(const float* __restrict__ grid, int R, int s, int nb,
                                                              const uint8_t* __restrict__ parent, uint8_t* __restrict__ st,
                                                              uint8_t* __restrict__ mark, float iso, float tau) {
  const int64_t b = (int64_t)blockIdx.x * AD_THREADS + threadIdx.x;
  if (b >= (int64_t)nb * nb * nb) return;
  const int bx = (int)(b % nb), by = (int)((b / nb) % nb), bz = (int)(b / ((int64_t)nb * nb));
  if (parent) {
    const int pn = nb >> 1;
    if (parent[((int64_t)(bz >> 1) * pn + (by >> 1)) * pn + (bx >> 1)] != 2) { st[b] = 0; return; }
  }
  const int64_t o = ((int64_t)bz * s * R + (int64_t)by * s) * R + (int64_t)bx * s;
  const int64_t dx = s, dy = (int64_t)s * R, dz = (int64_t)s * R * R;
  float v[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = grid[o + ((k & 1) ? dx : 0) + ((k & 2) ? dy : 0) + ((k & 4) ? dz : 0)];
  const bool active = block_active(v, iso, tau);
  st[b] = active ? 2 : 1;
  if (!active) return;
  const int h = s >> 1;
  for (int kz = 0; kz < 3; ++kz)
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) {
        const int64_t p = o + ((int64_t)kz * h * R + (int64_t)ky * h) * R + (int64_t)kx * h;
        if (mark[p] == 0) mark[p] = 2;
      }
}

// per chunk of AD_CHUNK mark bytes: the number of 2s
__global__ void __launch_bounds__(AD_THREADS) count_kernel(const uint8_t* __restrict__ mark, int64_t n,
                                                           uint32_t* __restrict__ chunk) {
  using Reduce = cub::BlockReduce<uint32_t, AD_THREADS>;
  __shared__ typename Reduce::TempStorage tmp;
  const int64_t base = (int64_t)blockIdx.x * AD_CHUNK + (int64_t)threadIdx.x * AD_ITEMS;
  uint32_t cnt = 0;
#pragma unroll
  for (int k = 0; k < AD_ITEMS; ++k)
    if (base + k < n) cnt += (mark[base + k] == 2) ? 1u : 0u;
  const uint32_t tot = Reduce(tmp).Sum(cnt);
  if (threadIdx.x == 0) chunk[blockIdx.x] = tot;
}

// after the exclusive scan of the chunk counts: the marked points in ascending order, then marked evaluated
__global__ void __launch_bounds__(AD_THREADS) compact_kernel(uint8_t* __restrict__ mark, int64_t n,
                                                             const uint32_t* __restrict__ chunk, int32_t* __restrict__ list) {
  using Scan = cub::BlockScan<uint32_t, AD_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  const int64_t base = (int64_t)blockIdx.x * AD_CHUNK + (int64_t)threadIdx.x * AD_ITEMS;
  uint32_t flags = 0, cnt = 0;
#pragma unroll
  for (int k = 0; k < AD_ITEMS; ++k)
    if (base + k < n && mark[base + k] == 2) { flags |= 1u << k; ++cnt; }
  uint32_t pos;
  Scan(tmp).ExclusiveSum(cnt, pos);
  if (!flags) return;
  pos += chunk[blockIdx.x];
#pragma unroll
  for (int k = 0; k < AD_ITEMS; ++k)
    if (flags & (1u << k)) {
      list[pos++] = (int32_t)(base + k);
      mark[base + k] = 1;
    }
}

__global__ void __launch_bounds__(AD_THREADS) fill_kernel(float* __restrict__ grid, const uint8_t* __restrict__ mark,
                                                          const uint8_t* __restrict__ st, int R, Levels lv) {
  const int64_t i = (int64_t)blockIdx.x * AD_THREADS + threadIdx.x;
  if (i >= (int64_t)R * R * R || mark[i]) return;
  const int x = (int)(i % R), y = (int)((i / R) % R), z = (int)(i / ((int64_t)R * R));
  for (int l = lv.n - 1; l >= 0; --l) {          // finest level first
    const int s = lv.s[l], nb = lv.nb[l];
    int qx[2], qy[2], qz[2];
    const int nx = block_candidates(x, s, nb, qx), ny = block_candidates(y, s, nb, qy), nz = block_candidates(z, s, nb, qz);
    for (int a = 0; a < nz; ++a)
      for (int b = 0; b < ny; ++b)
        for (int d = 0; d < nx; ++d) {
          if (st[lv.off[l] + ((int64_t)qz[a] * nb + qy[b]) * nb + qx[d]] != 1) continue;
          const int ox = qx[d] * s, oy = qy[b] * s, oz = qz[a] * s;
          const float inv = 1.f / (float)s;      // s is a power of two: the products below are exact
          const float tx = (float)(x - ox) * inv, ty = (float)(y - oy) * inv, tz = (float)(z - oz) * inv;
          const int64_t o = ((int64_t)oz * R + oy) * R + ox;
          const int64_t sy = (int64_t)s * R, sz = (int64_t)s * R * R;
          float v[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) v[k] = grid[o + ((k & 1) ? s : 0) + ((k & 2) ? sy : 0) + ((k & 4) ? sz : 0)];
          grid[i] = trilinear(v, tx, ty, tz);
          return;
        }
  }
}

// the list's values into the grid: the network at the listed points, or the given field
int evaluate_list(disn_ctx* c, const float* field, int image, const float* d_tm, int R, const int32_t* list, int64_t n,
                  float* grid) {
  if (n == 0) return 0;
  const float* vals = nullptr;
  if (!field) {
    if (c->ad_vals.ensure((size_t)n * sizeof(float))) return -1;
    if (eval_grid_points(c, image, R, d_tm, list, n, c->ad_vals.as<float>())) return -1;
    vals = c->ad_vals.as<float>();
  }
  scatter_kernel<<<blocks_of(n), AD_THREADS, 0, c->stream>>>(list, n, vals, field, grid);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace

int adaptive_run(disn_ctx* c, const float* field, int image, const float* d_tm, int32_t res, const double* sdf_params,
                 float iso, double band, int64_t* level_counts, int32_t* n_levels) {
  const int R = res + 1;
  const int64_t n = (int64_t)R * R * R;
  const int s0 = coarse_stride(res);
  Levels lv{};
  int64_t states = 0;
  for (int s = s0; s >= 2; s >>= 1, ++lv.n) {
    lv.s[lv.n] = s;
    lv.nb[lv.n] = res / s;
    lv.off[lv.n] = states;
    states += (int64_t)lv.nb[lv.n] * lv.nb[lv.n] * lv.nb[lv.n];
  }
  const int64_t nchunks = (n + AD_CHUNK - 1) / AD_CHUNK;
  const int64_t M = res / s0 + 1;
  c->ad_R = 0;
  if (c->ad_grid.ensure((size_t)n * sizeof(float)) || c->ad_mark.ensure((size_t)n) ||
      c->ad_state.ensure((size_t)std::max<int64_t>(states, 1)) || c->ad_chunk.ensure((size_t)nchunks * sizeof(uint32_t)) ||
      c->ad_sums.ensure((size_t)(scan_scratch_elems(nchunks) + 1) * sizeof(uint32_t)) ||
      c->ad_host.ensure(sizeof(uint32_t)) || c->ad_list.ensure((size_t)M * M * M * sizeof(int32_t)))
    return -1;
  for (cudaEvent_t& e : c->ad_ev)
    if (!e) DISN_CUDA_OK(cudaEventCreate(&e));
  cudaStream_t st = c->stream;
  float* grid = c->ad_grid.as<float>();
  uint8_t* mark = c->ad_mark.as<uint8_t>();
  uint8_t* state = c->ad_state.as<uint8_t>();
  uint32_t* chunk = c->ad_chunk.as<uint32_t>();
  uint32_t* total = c->ad_sums.as<uint32_t>();          // first word: the level total; the scan scratch follows
  uint32_t* sums = total + 1;
  DISN_CUDA_OK(cudaEventRecord(c->ad_ev[0], st));

  if (s0 == 1) {            // no power of two divides res: the dense grid
    if (field) DISN_CUDA_OK(cudaMemcpyAsync(grid, field, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    else if (eval_grid_points<int32_t>(c, image, R, d_tm, nullptr, n, grid)) return -1;
    DISN_CUDA_OK(cudaMemsetAsync(mark, 1, (size_t)n, st));
    DISN_CUDA_OK(cudaEventRecord(c->ad_ev[1], st));
    level_counts[0] = n;
    *n_levels = 1;
    c->ad_R = R;
    c->ad_levels = 0;
    return 0;
  }

  // coarse lattice
  DISN_CUDA_OK(cudaMemsetAsync(mark, 0, (size_t)n, st));
  int32_t* list = c->ad_list.as<int32_t>();
  lattice_kernel<<<blocks_of(M * M * M), AD_THREADS, 0, st>>>(R, s0, (int)M, list, mark);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  if (evaluate_list(c, field, image, d_tm, R, list, M * M * M, grid)) return -1;
  level_counts[0] = M * M * M;
  DISN_CUDA_OK(cudaEventRecord(c->ad_ev[1], st));

  uint32_t* h_total = c->ad_host.as<uint32_t>();
  for (int l = 0; l < lv.n; ++l) {
    const int s = lv.s[l], nb = lv.nb[l];
    const float tau = level_tau(band, s, sdf_params, res);
    const int64_t nblk = (int64_t)nb * nb * nb;
    classify_kernel<<<blocks_of(nblk), AD_THREADS, 0, st>>>(grid, R, s, nb, l ? state + lv.off[l - 1] : nullptr,
                                                            state + lv.off[l], mark, iso, tau);
    count_kernel<<<(unsigned)nchunks, AD_THREADS, 0, st>>>(mark, n, chunk);
    c->launches += 2;
    DISN_CUDA_OK(cudaGetLastError());
    if (exclusive_scan(c, chunk, nchunks, total, sums)) return -1;
    DISN_CUDA_OK(cudaMemcpyAsync(h_total, total, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    DISN_CUDA_OK(cudaStreamSynchronize(st));             // the level's count sizes its list
    const int64_t cnt = *h_total;
    level_counts[l + 1] = cnt;
    if (c->ad_list.ensure((size_t)std::max<int64_t>(cnt, 1) * sizeof(int32_t))) return -1;
    list = c->ad_list.as<int32_t>();
    compact_kernel<<<(unsigned)nchunks, AD_THREADS, 0, st>>>(mark, n, chunk, list);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
    if (evaluate_list(c, field, image, d_tm, R, list, cnt, grid)) return -1;
    DISN_CUDA_OK(cudaEventRecord(c->ad_ev[2 + l], st));
  }
  fill_kernel<<<blocks_of(n), AD_THREADS, 0, st>>>(grid, mark, state, R, lv);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaEventRecord(c->ad_ev[2 + lv.n], st));
  *n_levels = lv.n + 1;
  c->ad_R = R;
  c->ad_levels = lv.n;
  return 0;
}

}  // namespace disn
