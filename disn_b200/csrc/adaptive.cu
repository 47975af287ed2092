// Coarse-to-fine evaluation of the SDF grid (DESIGN.md §4.9): the network runs only at the grid points of blocks that can
// hold the iso-surface, every other point is filled by trilinear interpolation.  Definitions, shared with the numpy twin
// oracle/adaptive_oracle.py:
//   * s0 = the largest power of two <= 16 that divides res (s0 = 1: the dense grid); the stride-s0 lattice is evaluated
//     first, then levels s = s0, s0/2, ..., 2;
//   * level s classifies the blocks of size s (closed cubes of lattice points, origin a multiple of s): every block at the
//     first level, later only the children of active parents.  A block is active when its 8 corners are not all on one
//     side of iso under marching cubes' predicate v < iso, or when some corner has |v - iso| <= tau_s (float32),
//     tau_s = float32(band * (s/2) * sqrt(hx^2 + hy^2 + hz^2)) computed in float64;
//   * the level's list: the stride-s/2 points of active blocks that are not yet evaluated, in ascending linear index;
//   * fill: a point never evaluated takes the trilinear interpolation (x, then y, then z; (1-t)*a + t*b rounded per
//     operation, no FMA) of the corners of the finest classified inactive block containing it; among several blocks of
//     that level the first in (z, y, x) order, each axis trying the block starting at or below the point first.
// adaptive_refine is the one refinement of both coarse-to-fine paths.  Each level classifies the children of the previous
// level's active blocks; its new points are the non-corner stride-s/2 points of its active blocks, each emitted once by
// its owner (the active block with the smallest index among those that contain it), then radix-sorted into the list.  The
// network evaluates the lattice and each list through eval_grid_points (api.cu), one host synchronisation per level.  The
// values go into a sink: the dense grid and its marks (adaptive_run here), or per-level hash tables (adaptive_mesh.cu).
// adaptive_run then fills every unmarked point, giving a complete [R,R,R] grid for the unchanged marching cubes.
#include <algorithm>
#include <cmath>

#include <cub/device/device_radix_sort.cuh>

#include "adaptive_common.cuh"
#include "common.cuh"

namespace disn {
namespace {

constexpr int AD_THREADS = 256;
constexpr int64_t AD_CHUNK = (int64_t)1 << 24;     // points per network call (4 B of values each)

inline unsigned blocks_of(int64_t n) { return (unsigned)((n + AD_THREADS - 1) / AD_THREADS); }

// the stride-s0 lattice: read from a given field into coarse (field non-null), and written into the dense grid, marked
// evaluated (grid non-null)
__global__ void __launch_bounds__(AD_THREADS) lattice_kernel(const float* __restrict__ field, int R, int s0, int M,
                                                             float* __restrict__ coarse, float* __restrict__ grid,
                                                             uint8_t* __restrict__ mark) {
  const int64_t j = (int64_t)blockIdx.x * AD_THREADS + threadIdx.x;
  if (j >= (int64_t)M * M * M) return;
  const int64_t x = (j % M) * s0, y = ((j / M) % M) * s0, z = (j / ((int64_t)M * M)) * s0;
  const int64_t i = (z * R + y) * R + x;
  const float v = field ? field[i] : coarse[j];
  if (field) coarse[j] = v;
  if (grid) {
    grid[i] = v;
    mark[i] = 1;
  }
}

// classify the level's blocks; active ones are appended to `active` (counter[0])
__global__ void __launch_bounds__(AD_THREADS) classify_kernel(Field f, int l, const uint32_t* __restrict__ parents, int64_t n,
                                                              float tau, uint8_t* __restrict__ st,
                                                              uint32_t* __restrict__ active,
                                                              unsigned long long* __restrict__ counter) {
  const int64_t j = (int64_t)blockIdx.x * AD_THREADS + threadIdx.x;
  const int s = f.s[l], nb = f.nb[l];
  bool act = false;
  uint32_t b = 0;
  if (j < n) {
    int bx, by, bz;
    classified_block(j, parents, nb, bx, by, bz);
    float v[8];
    if (f.grid) block_corners<true>(f, s, bx, by, bz, v);
    else block_corners<false>(f, s, bx, by, bz, v);
    act = block_active(v, f.iso, tau);
    b = (uint32_t)(((int64_t)bz * nb + by) * nb + bx);
    st[b] = act ? 2 : 1;
  }
  const unsigned long long pos = warp_append(act ? 1u : 0u, counter);
  if (act) active[pos] = b;
}

// The level's new points owned by active block (bx, by, bz): its 19 non-corner stride-s/2 points, each unless an active
// block with a smaller index also contains it.  kEmit: write their linear indices from out[pos] on; returns the count.
template <bool kEmit>
__device__ __forceinline__ uint32_t owned_points(const Field& f, int l, int bx, int by, int bz, unsigned long long* out,
                                                 unsigned long long pos) {
  const int s = f.s[l], nb = f.nb[l], h = s >> 1, R = f.R;
  const uint8_t* st = f.st[l];
  const int64_t self = ((int64_t)bz * nb + by) * nb + bx;
  uint32_t cnt = 0;
  for (int kz = 0; kz < 3; ++kz)
    for (int ky = 0; ky < 3; ++ky)
      for (int kx = 0; kx < 3; ++kx) {
        if (kx != 1 && ky != 1 && kz != 1) continue;        // a corner: evaluated by an earlier level
        // the other blocks containing the point: along an axis with k = 0 the block below, with k = 2 the block above
        const int ex = kx == 1 ? 0 : kx - 1, ey = ky == 1 ? 0 : ky - 1, ez = kz == 1 ? 0 : kz - 1;
        bool owner = true;
        for (int oz = 0; oz <= (ez != 0); ++oz)
          for (int oy = 0; oy <= (ey != 0); ++oy)
            for (int ox = 0; ox <= (ex != 0); ++ox) {
              if (!(ox | oy | oz)) continue;
              const int nx = bx + ox * ex, ny = by + oy * ey, nz = bz + oz * ez;
              if (block_is_active(st, nb, nx, ny, nz) && ((int64_t)nz * nb + ny) * nb + nx < self) owner = false;
            }
        if (!owner) continue;
        if (kEmit)
          out[pos + cnt] = ((unsigned long long)(bz * s + kz * h) * R + (by * s + ky * h)) * R + (bx * s + kx * h);
        ++cnt;
      }
  return cnt;
}

// kEmit = false: the number of new points of the level -> counter[1]; true: their linear indices (unsorted) -> out
template <bool kEmit>
__global__ void __launch_bounds__(AD_THREADS) level_points_kernel(Field f, int l, const uint32_t* __restrict__ parents,
                                                                  int64_t n, unsigned long long* __restrict__ counter,
                                                                  unsigned long long* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * AD_THREADS + threadIdx.x;
  const int nb = f.nb[l];
  int bx = 0, by = 0, bz = 0;
  bool act = false;
  if (j < n) {
    classified_block(j, parents, nb, bx, by, bz);
    act = f.st[l][((int64_t)bz * nb + by) * nb + bx] == 2;
  }
  const uint32_t cnt = act ? owned_points<false>(f, l, bx, by, bz, nullptr, 0) : 0u;
  const unsigned long long pos = warp_append(cnt, counter);
  if (kEmit && cnt) owned_points<true>(f, l, bx, by, bz, out, pos);
}

// values at sorted keys (the network's vals[j], or the given field) into the dense grid, marked evaluated (grid
// non-null), or into the level's hash table
__global__ void __launch_bounds__(AD_THREADS) store_kernel(const unsigned long long* __restrict__ keys, int64_t n,
                                                           const float* __restrict__ vals, const float* __restrict__ field,
                                                           float* __restrict__ grid, uint8_t* __restrict__ mark,
                                                           unsigned long long* __restrict__ tkeys,
                                                           float* __restrict__ tvals, unsigned long long cap) {
  const int64_t j = (int64_t)blockIdx.x * AD_THREADS + threadIdx.x;
  if (j >= n) return;
  const unsigned long long key = keys[j];
  const float v = field ? field[key] : vals[j];
  if (grid) {
    grid[key] = v;
    mark[key] = 1;
    return;
  }
  unsigned long long i = slot_of(key, cap);
  while (atomicCAS(&tkeys[i], AM_EMPTY, key) != AM_EMPTY)
    if (++i == cap) i = 0;
  tvals[i] = v;
}

// every point the refinement did not evaluate takes the fill; in place, since it reads only marked points.  (At the
// default minimum of one block per SM ptxas keeps it in 32 registers and spills; 4 lets it use 40.)
__global__ void __launch_bounds__(AD_THREADS, 4) fill_kernel(Field f, const uint8_t* __restrict__ mark, float* grid) {
  const int R = f.R;
  const int64_t i = (int64_t)blockIdx.x * AD_THREADS + threadIdx.x;
  if (i >= (int64_t)R * R * R || mark[i]) return;
  grid[i] = value_at<true>(f, (int)(i % R), (int)((i / R) % R), (int)(i / ((int64_t)R * R)));
}

// the level's n sorted keys and their values (the given field, or the network one chunk at a time through ad_vals) into
// the dense grid or the level's table
int store_level(disn_ctx* c, const float* field, int image, const float* d_tm, int R, const unsigned long long* keys,
                int64_t n, float* grid, uint8_t* mark, unsigned long long* tkeys, float* tvals, unsigned long long cap) {
  const int64_t chunk = field ? n : std::min<int64_t>(n, AD_CHUNK);
  if (!field && c->ad_vals.ensure((size_t)chunk * sizeof(float))) return -1;
  for (int64_t j0 = 0; j0 < n; j0 += chunk) {
    const int64_t m = std::min<int64_t>(chunk, n - j0);
    if (!field && eval_grid_points(c, image, R, d_tm, keys + j0, m, c->ad_vals.as<float>())) return -1;
    store_kernel<<<blocks_of(m), AD_THREADS, 0, c->stream>>>(keys + j0, m, c->ad_vals.as<float>(), field, grid, mark,
                                                             tkeys, tvals, cap);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
  }
  return 0;
}

}  // namespace

int sort_keys(disn_ctx* c, DevBuffer (&keys)[2], int64_t n, int bits, unsigned long long** sorted) {
  DISN_REQUIRE(n < ((int64_t)1 << 31), "coarse-to-fine: a list of 2^31 or more keys");
  cub::DoubleBuffer<unsigned long long> db(keys[0].as<unsigned long long>(), keys[1].as<unsigned long long>());
  size_t tmp = 0;
  DISN_CUDA_OK(cub::DeviceRadixSort::SortKeys(nullptr, tmp, db, (int)n, 0, bits, c->stream));
  if (c->ad_sort_tmp.ensure(std::max<size_t>(tmp, 1))) return -1;
  DISN_CUDA_OK(cub::DeviceRadixSort::SortKeys(c->ad_sort_tmp.as<void>(), tmp, db, (int)n, 0, bits, c->stream));
  *sorted = db.Current();
  return 0;
}

int adaptive_refine(disn_ctx* c, const float* field, int image, const float* d_tm, int32_t res, const double* sdf_params,
                    float iso, double band, float* grid, uint8_t* mark, cudaEvent_t* ev, Refinement& r,
                    int64_t* level_counts, int32_t* n_levels) {
  cudaStream_t st = c->stream;
  const int R = res + 1;
  r = Refinement{};
  Field& f = r.f;
  f.R = R;
  f.s0 = coarse_stride(res);
  f.iso = iso;
  f.grid = grid;
  while ((1 << f.lg0) < f.s0) ++f.lg0;
  f.M = res / f.s0 + 1;
  int64_t state_off[AD_MAX_LEVELS] = {}, states = 0;
  for (int s = f.s0; s >= 2; s >>= 1, ++f.n) {
    f.s[f.n] = s;
    f.nb[f.n] = res / s;
    state_off[f.n] = states;
    states += (int64_t)f.nb[f.n] * f.nb[f.n] * f.nb[f.n];
  }
  const int64_t nM = (int64_t)f.M * f.M * f.M;
  if (c->ad_state.ensure((size_t)std::max<int64_t>(states, 1)) || c->ad_coarse.ensure((size_t)nM * sizeof(float)) ||
      c->ad_cnt.ensure(4 * sizeof(unsigned long long)) || c->ad_host.ensure(4 * sizeof(unsigned long long)))
    return -1;
  unsigned long long* cnt = c->ad_cnt.as<unsigned long long>();
  unsigned long long* hcnt = c->ad_host.as<unsigned long long>();
  for (int l = 0; l < f.n; ++l) f.st[l] = c->ad_state.as<uint8_t>() + state_off[l];

  // coarse lattice
  float* coarse = c->ad_coarse.as<float>();
  f.coarse = coarse;
  if (!field && eval_grid_points<unsigned long long>(c, image, R, d_tm, nullptr, nM, coarse, f.s0)) return -1;
  if (field || grid) {
    lattice_kernel<<<blocks_of(nM), AD_THREADS, 0, st>>>(field, R, f.s0, f.M, coarse, grid, mark);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
  }
  level_counts[0] = nM;
  if (ev) DISN_CUDA_OK(cudaEventRecord(ev[0], st));

  // levels: classify the children of the previous level's active blocks, emit the owned new points, sort, evaluate
  r.nclass[0] = states > 0 ? (int64_t)f.nb[0] * f.nb[0] * f.nb[0] : 0;
  for (int l = 0; l < f.n; ++l) {
    const int64_t n = r.nclass[l];
    DISN_CUDA_OK(cudaMemsetAsync(const_cast<uint8_t*>(f.st[l]), 0, (size_t)f.nb[l] * f.nb[l] * f.nb[l], st));
    DISN_CUDA_OK(cudaMemsetAsync(cnt, 0, 2 * sizeof(unsigned long long), st));
    if (c->ad_active[l].ensure((size_t)std::max<int64_t>(n, 1) * sizeof(uint32_t))) return -1;
    if (n) {
      classify_kernel<<<blocks_of(n), AD_THREADS, 0, st>>>(f, l, r.parents[l], n, level_tau(band, f.s[l], sdf_params, res),
                                                           const_cast<uint8_t*>(f.st[l]), c->ad_active[l].as<uint32_t>(), cnt);
      level_points_kernel<false><<<blocks_of(n), AD_THREADS, 0, st>>>(f, l, r.parents[l], n, cnt + 1, nullptr);
      c->launches += 2;
      DISN_CUDA_OK(cudaGetLastError());
    }
    DISN_CUDA_OK(cudaMemcpyAsync(hcnt, cnt, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    DISN_CUDA_OK(cudaStreamSynchronize(st));               // the level's counts size its list and the next level
    const int64_t n_active = (int64_t)hcnt[0], n_new = (int64_t)hcnt[1];
    level_counts[l + 1] = n_new;
    if (l + 1 < f.n) {
      r.nclass[l + 1] = 8 * n_active;
      r.parents[l + 1] = c->ad_active[l].as<uint32_t>();
    }
    if (n_new) {
      const unsigned long long cap = grid ? 0 : (unsigned long long)(n_new + n_new / 2 + 1);
      if (c->ad_keys[0].ensure((size_t)n_new * 8) || c->ad_keys[1].ensure((size_t)n_new * 8) ||
          (!grid && c->am_table[l].ensure((size_t)cap * 12)))
        return -1;
      DISN_CUDA_OK(cudaMemsetAsync(cnt + 1, 0, sizeof(unsigned long long), st));
      level_points_kernel<true><<<blocks_of(n), AD_THREADS, 0, st>>>(f, l, r.parents[l], n, cnt + 1,
                                                                      c->ad_keys[0].as<unsigned long long>());
      c->launches++;
      DISN_CUDA_OK(cudaGetLastError());
      unsigned long long* keys = nullptr;
      if (sort_keys(c, c->ad_keys, n_new, key_bits((unsigned long long)R * R * R), &keys)) return -1;
      unsigned long long* tkeys = grid ? nullptr : c->am_table[l].as<unsigned long long>();
      float* tvals = grid ? nullptr : reinterpret_cast<float*>(tkeys + cap);
      if (!grid) DISN_CUDA_OK(cudaMemsetAsync(tkeys, 0xff, (size_t)cap * 8, st));
      if (store_level(c, field, image, d_tm, R, keys, n_new, grid, mark, tkeys, tvals, cap)) return -1;
      if (!grid) f.t[l] = Table{tkeys, tvals, cap};
    }
    if (ev) DISN_CUDA_OK(cudaEventRecord(ev[1 + l], st));
  }
  *n_levels = f.n + 1;
  return 0;
}

int adaptive_run(disn_ctx* c, const float* field, int image, const float* d_tm, int32_t res, const double* sdf_params,
                 float iso, double band, int64_t* level_counts, int32_t* n_levels) {
  const int R = res + 1;
  const int64_t n = (int64_t)R * R * R;
  c->ad_R = 0;
  if (c->ad_grid.ensure((size_t)n * sizeof(float)) || c->ad_mark.ensure((size_t)n)) return -1;
  for (cudaEvent_t& e : c->ad_ev)
    if (!e) DISN_CUDA_OK(cudaEventCreate(&e));
  cudaStream_t st = c->stream;
  float* grid = c->ad_grid.as<float>();
  uint8_t* mark = c->ad_mark.as<uint8_t>();
  DISN_CUDA_OK(cudaEventRecord(c->ad_ev[0], st));

  if (coarse_stride(res) == 1) {            // no power of two divides res: the dense grid
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

  // the refinement's values go into the grid, marked; then every unmarked point takes the fill
  DISN_CUDA_OK(cudaMemsetAsync(mark, 0, (size_t)n, st));
  Refinement r;
  if (adaptive_refine(c, field, image, d_tm, res, sdf_params, iso, band, grid, mark, c->ad_ev + 1, r, level_counts,
                      n_levels))
    return -1;
  fill_kernel<<<blocks_of(n), AD_THREADS, 0, st>>>(r.f, mark, grid);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaEventRecord(c->ad_ev[2 + r.f.n], st));
  c->ad_R = R;
  c->ad_levels = r.f.n;
  return 0;
}

}  // namespace disn
