// Coarse-to-fine meshing without a dense grid (DESIGN.md §4.10).  The refinement is adaptive.cu's adaptive_refine, the
// one the dense grid runs; only where its values go differs:
//   * values: the stride-s0 lattice densely ([M,M,M]), every level's list in its own open-addressing hash table (int64
//     key, float value, load <= 2/3).  A point's level follows from its coordinates, so a lookup probes one table; a miss
//     means the point was never evaluated and takes the fill rule (value_at, adaptive_common.cuh);
//   * marching cubes visits only the candidate cells K (§4.10) and numbers vertices by the rank of their edge id among
//     the sorted crossing edges, faces by cell then table order: mc.cu's mesh of the dense adaptive grid, bit for bit.
// One host synchronisation per level in the refinement and two for the mesh.
#include <algorithm>
#include <cmath>

#include "adaptive_common.cuh"
#include "common.cuh"
#include "mc_table.h"

namespace disn {
namespace {

constexpr int AM_THREADS = 256;

inline unsigned blocks_of(int64_t n) { return (unsigned)((n + AM_THREADS - 1) / AM_THREADS); }

__device__ __forceinline__ int cell_case_at(const Field& f, int cx, int cy, int cz) {
  float v[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = value_at<false>(f, cx + (k & 1), cy + ((k >> 1) & 1), cz + ((k >> 2) & 1));
  return cell_case_of(v, f.iso);
}

// ---- candidate cells and the mesh -------------------------------------------------------------------------------------

// An inactive block is near iso when some corner lies within 8 ulp of its largest corner magnitude (plus the smallest
// normal, for underflow) of iso: only then can the 7 roundings of the fill put an interpolated value on the other side
// than its corners (their error is below 6.01 ulp of that magnitude).
__device__ __forceinline__ bool near_iso(const float (&v)[8], float iso) {
  double amax = 0.0;
#pragma unroll
  for (int k = 0; k < 8; ++k) amax = fmax(amax, fabs((double)v[k]));
  const double margin = __dadd_rn(__dmul_rn(amax, 0x1p-21), 0x1p-126);
  bool near = false;
#pragma unroll
  for (int k = 0; k < 8; ++k) near |= fabs(__dsub_rn((double)v[k], (double)iso)) <= margin;
  return near;
}

// Crossing cells among the candidates of the level's classified blocks: every cell of an active block of the last
// level; the cells of an inactive block with a corner in an active block of the same level (its boundary layer toward
// active neighbours, across faces, edges and corners); every cell of an inactive block near iso.  kEmit = false: their
// number -> counter; true: their cell ids (origin linear index) -> out.
template <bool kEmit>
__global__ void __launch_bounds__(AM_THREADS) cells_kernel(Field f, int l, const uint32_t* __restrict__ parents, int64_t n,
                                                           unsigned long long* __restrict__ counter,
                                                           unsigned long long* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * AM_THREADS + threadIdx.x;
  const int s = f.s[l], nb = f.nb[l], R = f.R;
  const uint8_t* st = f.st[l];
  int bx = 0, by = 0, bz = 0;
  uint32_t nbr = 0;            // bit (dz+1)*9 + (dy+1)*3 + (dx+1): that neighbour is active
  bool all = false;
  if (j < n) {
    classified_block(j, parents, nb, bx, by, bz);
    const uint8_t state = st[((int64_t)bz * nb + by) * nb + bx];
    if (state == 2) {
      all = l == f.n - 1;
    } else {
      float v[8];
      block_corners<false>(f, s, bx, by, bz, v);
      all = near_iso(v, f.iso);
      if (!all)
        for (int d = 0; d < 27; ++d)
          if (d != 13 && block_is_active(st, nb, bx + d % 3 - 1, by + (d / 3) % 3 - 1, bz + d / 9 - 1)) nbr |= 1u << d;
    }
  }
  uint32_t cnt = 0;
  if (all || nbr) {
    for (int i = 0; i < s * s * s; ++i) {
      const int ix = i % s, iy = (i / s) % s, iz = i / (s * s);
      if (!all) {
        // neighbour offsets a corner of this cell reaches per axis: 0, and -1 / +1 on the block's low / high layer
        const int lox = ix == 0 ? -1 : 0, hix = ix == s - 1 ? 1 : 0;
        const int loy = iy == 0 ? -1 : 0, hiy = iy == s - 1 ? 1 : 0;
        const int loz = iz == 0 ? -1 : 0, hiz = iz == s - 1 ? 1 : 0;
        if (!(lox | hix | loy | hiy | loz | hiz)) continue;
        bool cand = false;
        for (int dz = loz; dz <= hiz; ++dz)
          for (int dy = loy; dy <= hiy; ++dy)
            for (int dx = lox; dx <= hix; ++dx) cand |= (nbr >> ((dz + 1) * 9 + (dy + 1) * 3 + dx + 1)) & 1u;
        if (!cand) continue;
      }
      const int cx = bx * s + ix, cy = by * s + iy, cz = bz * s + iz;
      const int cs = cell_case_at(f, cx, cy, cz);
      if (cs == 0 || cs == 255) continue;
      if (kEmit) out[atomicAdd(counter, 1ull)] = ((unsigned long long)cz * R + cy) * R + cx;
      ++cnt;
    }
  }
  if (!kEmit) warp_append(cnt, counter);
}

// The crossing edges a cell owns: edge (point q, axis a) belongs to the cell of lowest coordinates that contains it, so
// along each other axis b the cell owns it when the edge lies on its upper side (offset 1) or the cell is at 0.
__device__ __forceinline__ uint32_t owned_edges(int cs, int cx, int cy, int cz, int R, unsigned long long* out) {
  uint32_t cnt = 0;
  const int c[3] = {cx, cy, cz};
  for (int e = 0; e < 12; ++e) {
    const int a = kMcEdge[e][0];
    const int o[3] = {kMcEdge[e][1], kMcEdge[e][2], kMcEdge[e][3]};
    const int k0 = o[0] + 2 * o[1] + 4 * o[2], k1 = k0 + (1 << a);
    if (!(((cs >> k0) ^ (cs >> k1)) & 1)) continue;
    bool own = true;
    for (int b = 0; b < 3; ++b)
      if (b != a && o[b] == 0 && c[b] != 0) own = false;
    if (!own) continue;
    if (out) out[cnt] = (((unsigned long long)(cz + o[2]) * R + (cy + o[1])) * R + (cx + o[0])) * 3 + a;
    ++cnt;
  }
  return cnt;
}

// per crossing cell (ascending): its case, its triangle count (for the scan) and its owned edges -> counter
__global__ void __launch_bounds__(AM_THREADS) cell_case_kernel(Field f, const unsigned long long* __restrict__ cells,
                                                               int64_t n, uint8_t* __restrict__ cases,
                                                               uint32_t* __restrict__ ntri,
                                                               unsigned long long* __restrict__ counter) {
  const int64_t j = (int64_t)blockIdx.x * AM_THREADS + threadIdx.x;
  const int R = f.R;
  uint32_t cnt = 0;
  if (j < n) {
    const unsigned long long i = cells[j];
    const int cx = (int)(i % R), cy = (int)((i / R) % R), cz = (int)(i / ((unsigned long long)R * R));
    const int cs = cell_case_at(f, cx, cy, cz);
    cases[j] = (uint8_t)cs;
    ntri[j] = (uint32_t)kMcNumTris[cs];
    cnt = owned_edges(cs, cx, cy, cz, R, nullptr);
  }
  warp_append(cnt, counter);
}

__global__ void __launch_bounds__(AM_THREADS) edges_kernel(const unsigned long long* __restrict__ cells, int64_t n, int R,
                                                           const uint8_t* __restrict__ cases,
                                                           unsigned long long* __restrict__ counter,
                                                           unsigned long long* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * AM_THREADS + threadIdx.x;
  int cx = 0, cy = 0, cz = 0, cs = 0;
  uint32_t cnt = 0;
  if (j < n) {
    const unsigned long long i = cells[j];
    cx = (int)(i % R); cy = (int)((i / R) % R); cz = (int)(i / ((unsigned long long)R * R));
    cs = cases[j];
    cnt = owned_edges(cs, cx, cy, cz, R, nullptr);
  }
  const unsigned long long pos = warp_append(cnt, counter);
  if (cnt) owned_edges(cs, cx, cy, cz, R, out + pos);
}

struct Geom {
  double lo[3], h[3];
};

// vertex v = the crossing edge of rank v
__global__ void __launch_bounds__(AM_THREADS) vertices_kernel(Field f, Geom g, const unsigned long long* __restrict__ edges,
                                                              int64_t n, float* __restrict__ verts) {
  const int64_t j = (int64_t)blockIdx.x * AM_THREADS + threadIdx.x;
  if (j >= n) return;
  const int R = f.R;
  const unsigned long long e = edges[j], q = e / 3;
  const int a = (int)(e % 3);
  const int idx[3] = {(int)(q % R), (int)((q / R) % R), (int)(q / ((unsigned long long)R * R))};
  const float v0 = value_at<false>(f, idx[0], idx[1], idx[2]);
  const float v1 = value_at<false>(f, idx[0] + (a == 0), idx[1] + (a == 1), idx[2] + (a == 2));
  edge_vertex(g.lo, g.h, idx, a, v0, v1, f.iso, verts + j * 3);
}

__device__ __forceinline__ int32_t rank_of(const unsigned long long* __restrict__ edges, int64_t n, unsigned long long e) {
  int64_t lo = 0, hi = n;                          // the edge is present: lower bound
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (edges[mid] < e) lo = mid + 1; else hi = mid;
  }
  return (int32_t)lo;
}

// faces cell by cell (ascending), triangles in table order; foff = exclusive scan of the triangle counts
__global__ void __launch_bounds__(AM_THREADS) faces_kernel(const unsigned long long* __restrict__ cells, int64_t n, int R,
                                                           const uint8_t* __restrict__ cases,
                                                           const uint32_t* __restrict__ foff,
                                                           const unsigned long long* __restrict__ edges, int64_t ne,
                                                           int32_t* __restrict__ faces) {
  const int64_t j = (int64_t)blockIdx.x * AM_THREADS + threadIdx.x;
  if (j >= n) return;
  const unsigned long long i = cells[j];
  const int cx = (int)(i % R), cy = (int)((i / R) % R), cz = (int)(i / ((unsigned long long)R * R));
  const int cs = cases[j];
  const int nt = kMcNumTris[cs];
  const int64_t f0 = foff[j];
  for (int t = 0; t < nt; ++t)
    for (int k = 0; k < 3; ++k) {
      const int e = kMcTris[cs][3 * t + k];
      const unsigned long long id =
          (((unsigned long long)(cz + kMcEdge[e][3]) * R + (cy + kMcEdge[e][2])) * R + (cx + kMcEdge[e][1])) * 3 +
          kMcEdge[e][0];
      faces[(f0 + t) * 3 + k] = rank_of(edges, ne, id);
    }
}

}  // namespace

// the network's coordinate rows (c->d_rows) and the refinement's buffers are held for this call, so they count here
size_t adaptive_mesh_bytes(const disn_ctx* c) {
  size_t b = c->ad_state.bytes() + c->ad_coarse.bytes() + c->d_rows.bytes() + c->ad_vals.bytes() + c->ad_sort_tmp.bytes() +
             c->am_case.bytes() + c->am_tri.bytes() + c->am_sums.bytes() + c->ad_cnt.bytes();
  for (int k = 0; k < 2; ++k) b += c->ad_keys[k].bytes() + c->am_edges[k].bytes();
  for (int l = 0; l < AD_MAX_LEVELS; ++l) b += c->am_table[l].bytes() + c->ad_active[l].bytes();
  return b;
}

int adaptive_mesh_run(disn_ctx* c, const float* field, int image, const float* d_tm, int32_t res, const double* sdf_params,
                      float iso, double band, int64_t* level_counts, int32_t* n_levels) {
  cudaStream_t st = c->stream;
  const int R = res + 1;
  c->am_nv = -1;
  c->am_edges_sorted = nullptr;
  for (cudaEvent_t& e : c->am_ev)
    if (!e) DISN_CUDA_OK(cudaEventCreate(&e));
  DISN_CUDA_OK(cudaEventRecord(c->am_ev[0], st));
  Refinement r;
  if (adaptive_refine(c, field, image, d_tm, res, sdf_params, iso, band, nullptr, nullptr, nullptr, r, level_counts,
                      n_levels))
    return -1;
  const Field& f = r.f;
  const int64_t* nclass = r.nclass;
  const uint32_t* const* parents = r.parents;
  unsigned long long* cnt = c->ad_cnt.as<unsigned long long>();
  unsigned long long* hcnt = c->ad_host.as<unsigned long long>();
  DISN_CUDA_OK(cudaEventRecord(c->am_ev[1], st));

  // crossing cells among the candidates, ascending
  DISN_CUDA_OK(cudaMemsetAsync(cnt, 0, sizeof(unsigned long long), st));
  for (int l = 0; l < f.n; ++l)
    if (nclass[l]) {
      cells_kernel<false><<<blocks_of(nclass[l]), AM_THREADS, 0, st>>>(f, l, parents[l], nclass[l], cnt, nullptr);
      c->launches++;
    }
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaMemcpyAsync(hcnt, cnt, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  DISN_CUDA_OK(cudaStreamSynchronize(st));
  const int64_t n_cells = (int64_t)hcnt[0];
  int64_t nv = 0, nf = 0;
  unsigned long long* cells = nullptr;
  if (n_cells) {
    if (c->ad_keys[0].ensure((size_t)n_cells * 8) || c->ad_keys[1].ensure((size_t)n_cells * 8)) return -1;
    DISN_CUDA_OK(cudaMemsetAsync(cnt, 0, sizeof(unsigned long long), st));
    for (int l = 0; l < f.n; ++l)
      if (nclass[l]) {
        cells_kernel<true><<<blocks_of(nclass[l]), AM_THREADS, 0, st>>>(f, l, parents[l], nclass[l], cnt,
                                                                         c->ad_keys[0].as<unsigned long long>());
        c->launches++;
      }
    DISN_CUDA_OK(cudaGetLastError());
    if (sort_keys(c, c->ad_keys, n_cells, key_bits((unsigned long long)R * R * R), &cells)) return -1;
  }
  DISN_CUDA_OK(cudaEventRecord(c->am_ev[2], st));

  if (n_cells) {
    // cases, triangle offsets and the owned crossing edges
    if (c->am_case.ensure((size_t)n_cells) || c->am_tri.ensure((size_t)n_cells * sizeof(uint32_t)) ||
        c->am_sums.ensure((size_t)(scan_scratch_elems(n_cells) + 1) * sizeof(uint32_t)))
      return -1;
    uint8_t* cases = c->am_case.as<uint8_t>();
    uint32_t* foff = c->am_tri.as<uint32_t>();
    uint32_t* ftotal = c->am_sums.as<uint32_t>();
    DISN_CUDA_OK(cudaMemsetAsync(cnt, 0, sizeof(unsigned long long), st));
    cell_case_kernel<<<blocks_of(n_cells), AM_THREADS, 0, st>>>(f, cells, n_cells, cases, foff, cnt);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
    if (exclusive_scan(c, foff, n_cells, ftotal, ftotal + 1)) return -1;
    DISN_CUDA_OK(cudaMemcpyAsync(hcnt, cnt, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    uint32_t* hf = reinterpret_cast<uint32_t*>(hcnt + 1);
    DISN_CUDA_OK(cudaMemcpyAsync(hf, ftotal, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    DISN_CUDA_OK(cudaStreamSynchronize(st));
    nv = (int64_t)hcnt[0];
    nf = (int64_t)*hf;
    // up to 5 triangles per cell: with fewer than 2^32 / 5 cells the 32-bit offsets cannot wrap
    if (nv >= ((int64_t)1 << 31) || n_cells * 5 >= ((int64_t)1 << 32) || nf >= ((int64_t)1 << 31)) {
      set_error("mesh_grid_adaptive: the mesh has 2^31 or more vertices or faces (int32 face indices)");
      return -2;
    }
    if (c->am_edges[0].ensure((size_t)nv * 8) || c->am_edges[1].ensure((size_t)nv * 8)) return -1;
    DISN_CUDA_OK(cudaMemsetAsync(cnt, 0, sizeof(unsigned long long), st));
    edges_kernel<<<blocks_of(n_cells), AM_THREADS, 0, st>>>(cells, n_cells, R, cases, cnt,
                                                            c->am_edges[0].as<unsigned long long>());
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
    unsigned long long* edges = nullptr;
    if (sort_keys(c, c->am_edges, nv, key_bits((unsigned long long)R * R * R * 3), &edges)) return -1;
    c->am_edges_sorted = edges;
    if (c->mesh.replace(nv, nf)) return -1;
    Geom g;
    for (int k = 0; k < 3; ++k) { g.lo[k] = sdf_params[k]; g.h[k] = (sdf_params[3 + k] - sdf_params[k]) / (double)(R - 1); }
    vertices_kernel<<<blocks_of(nv), AM_THREADS, 0, st>>>(f, g, edges, nv, c->mesh.verts());
    faces_kernel<<<blocks_of(n_cells), AM_THREADS, 0, st>>>(cells, n_cells, R, cases, foff, edges, nv, c->mesh.faces());
    c->launches += 2;
    DISN_CUDA_OK(cudaGetLastError());
  } else if (c->mesh.replace(0, 0)) {
    return -1;
  }
  DISN_CUDA_OK(cudaEventRecord(c->am_ev[3], st));
  DISN_CUDA_OK(cudaStreamSynchronize(st));
  c->mesh.commit(nv, nf);
  c->am_nv = nv;
  return 0;
}

}  // namespace disn
