// Coarse-to-fine meshing without a dense grid (DESIGN.md §4.10).  The levels, the activity predicate, tau_s and the fill
// rule are §4.9's (adaptive_common.cuh); only the storage differs:
//   * block states: one byte per block per level, as in adaptive.cu; a level classifies the 8 children of the previous
//     level's active blocks (a list, not a pass over all blocks);
//   * the new points of level s are the non-corner stride-s/2 points of its active blocks, each emitted once by its owner
//     (the active block with the smallest index among those that contain it), then radix-sorted into ascending linear
//     index: the dense path's list;
//   * values: the stride-s0 lattice densely ([M,M,M]), every level's list in its own open-addressing hash table (int64
//     key, float value, load <= 2/3).  A point's level follows from its coordinates, so a lookup probes one table; a miss
//     means the point was never evaluated and takes the fill rule;
//   * marching cubes visits only the candidate cells K (§4.10) and numbers vertices by the rank of their edge id among
//     the sorted crossing edges, faces by cell then table order: mc.cu's mesh of the dense adaptive grid, bit for bit.
// The network evaluates each list in chunks of explicit points built from the float32 axis tables (point_of then reads
// the floats grid mode reads), one host synchronisation per level and two for the mesh.
#include <algorithm>
#include <cmath>

#include <cub/device/device_radix_sort.cuh>

#include "adaptive_common.cuh"
#include "common.cuh"
#include "mc_table.h"

namespace disn {
namespace {

constexpr int AM_THREADS = 256;
constexpr int64_t AM_CHUNK = (int64_t)1 << 24;     // points per network call (12 B of coordinates each)
constexpr unsigned long long AM_EMPTY = ~0ull;     // free hash slot

inline unsigned blocks_of(int64_t n) { return (unsigned)((n + AM_THREADS - 1) / AM_THREADS); }

struct Table {
  const unsigned long long* keys;
  const float* vals;
  unsigned long long cap;                          // 0: no table (an empty or not yet evaluated level)
};

// what the device kernels read: the lattice values, the states and the hash table of every level
struct Field {
  int R, s0, lg0, n;                               // points per axis, coarse stride, log2(s0), number of levels
  int M;                                           // coarse lattice points per axis
  const float* coarse;                             // [M,M,M]
  int s[AD_MAX_LEVELS], nb[AD_MAX_LEVELS];
  const uint8_t* st[AD_MAX_LEVELS];                // 0 = not classified, 1 = inactive, 2 = active
  Table t[AD_MAX_LEVELS];
  float iso;
};

__device__ __forceinline__ unsigned long long slot_of(unsigned long long key, unsigned long long cap) {
  unsigned long long h = key;                      // splitmix64 finaliser, then [0, cap) by a 64x64 high product
  h ^= h >> 30; h *= 0xbf58476d1ce4e5b9ull;
  h ^= h >> 27; h *= 0x94d049bb133111ebull;
  h ^= h >> 31;
  return __umul64hi(h, cap);
}

__device__ __forceinline__ bool lookup(const Table& t, unsigned long long key, float& v) {
  if (t.cap == 0) return false;
  unsigned long long i = slot_of(key, t.cap);
  while (true) {
    const unsigned long long k = t.keys[i];
    if (k == key) { v = t.vals[i]; return true; }
    if (k == AM_EMPTY) return false;
    if (++i == t.cap) i = 0;
  }
}

// the stored value of point (x, y, z) if it was evaluated: the coarse lattice, or the table of the only level that can
// have evaluated it (lowest set bit b of x|y|z below log2(s0): level s = 2^(b+1))
__device__ __forceinline__ bool stored(const Field& f, int x, int y, int z, float& v) {
  const int g = x | y | z;
  if ((g & (f.s0 - 1)) == 0) {
    v = f.coarse[((int64_t)(z / f.s0) * f.M + y / f.s0) * f.M + x / f.s0];
    return true;
  }
  const int l = f.lg0 - __ffs(g);
  return lookup(f.t[l], ((unsigned long long)z * f.R + y) * f.R + x, v);
}

// the 8 corner values of block (bx, by, bz) of size s (all evaluated: the stride-s points of an active parent)
__device__ __forceinline__ void block_corners(const Field& f, int s, int bx, int by, int bz, float (&v)[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k)
    stored(f, (bx + (k & 1)) * s, (by + ((k >> 1) & 1)) * s, (bz + ((k >> 2) & 1)) * s, v[k]);
}

// the dense adaptive grid's value at (x, y, z): stored, else the fill of the finest classified inactive block
__device__ float value_at(const Field& f, int x, int y, int z) {
  float v;
  if (stored(f, x, y, z, v)) return v;
  for (int l = f.n - 1; l >= 0; --l) {             // finest level first
    const int s = f.s[l], nb = f.nb[l];
    int qx[2], qy[2], qz[2];
    const int nx = block_candidates(x, s, nb, qx), ny = block_candidates(y, s, nb, qy), nz = block_candidates(z, s, nb, qz);
    for (int a = 0; a < nz; ++a)
      for (int b = 0; b < ny; ++b)
        for (int d = 0; d < nx; ++d) {
          if (f.st[l][((int64_t)qz[a] * nb + qy[b]) * nb + qx[d]] != 1) continue;
          float cv[8];
          block_corners(f, s, qx[d], qy[b], qz[a], cv);
          const float inv = 1.f / (float)s;        // s is a power of two: the products below are exact
          const float tx = (float)(x - qx[d] * s) * inv, ty = (float)(y - qy[b] * s) * inv,
                      tz = (float)(z - qz[a] * s) * inv;
          return trilinear(cv, tx, ty, tz);
        }
  }
  return __int_as_float(0x7fc00000);               // unreachable: every point lies in a classified inactive block
}

__device__ __forceinline__ int cell_case_at(const Field& f, int cx, int cy, int cz) {
  float v[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = value_at(f, cx + (k & 1), cy + ((k >> 1) & 1), cz + ((k >> 2) & 1));
  return cell_case_of(v, f.iso);
}

// Every lane of the warp calls this with its count; returns the lane's first slot of a range reserved from *counter.
__device__ __forceinline__ unsigned long long warp_append(uint32_t cnt, unsigned long long* counter) {
  const int lane = threadIdx.x & 31;
  uint32_t incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += n;
  }
  const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
  unsigned long long base = 0;
  if (lane == 31 && total) base = atomicAdd(counter, (unsigned long long)total);
  base = __shfl_sync(0xffffffffu, base, 31);
  return base + incl - cnt;
}

// block j of a level's classified set: every block at the first level, else child j & 7 of active parent j >> 3
__device__ __forceinline__ void classified_block(int64_t j, const uint32_t* parents, int nb, int& bx, int& by, int& bz) {
  if (!parents) {
    bx = (int)(j % nb); by = (int)((j / nb) % nb); bz = (int)(j / ((int64_t)nb * nb));
    return;
  }
  const int pn = nb >> 1;
  const uint32_t p = parents[j >> 3];
  const int c = (int)(j & 7);
  bx = 2 * (int)(p % pn) + (c & 1);
  by = 2 * (int)((p / pn) % pn) + ((c >> 1) & 1);
  bz = 2 * (int)(p / ((uint32_t)pn * pn)) + ((c >> 2) & 1);
}

__device__ __forceinline__ bool block_is_active(const uint8_t* st, int nb, int bx, int by, int bz) {
  return bx >= 0 && by >= 0 && bz >= 0 && bx < nb && by < nb && bz < nb &&
         st[((int64_t)bz * nb + by) * nb + bx] == 2;
}

// ---- coarse lattice and level lists ---------------------------------------------------------------------------------

// xyz rows of points [j0, j0 + n): keys[j] (linear indices), or the stride-s0 lattice point j in lattice order
__global__ void __launch_bounds__(AM_THREADS) xyz_kernel(const unsigned long long* __restrict__ keys, int64_t j0, int64_t n,
                                                         int R, int s0, int M, const float* __restrict__ axes,
                                                         float* __restrict__ xyz) {
  const int64_t j = (int64_t)blockIdx.x * AM_THREADS + threadIdx.x;
  if (j >= n) return;
  int x, y, z;
  if (keys) {
    const unsigned long long i = keys[j0 + j];
    x = (int)(i % R); y = (int)((i / R) % R); z = (int)(i / ((unsigned long long)R * R));
  } else {
    const int64_t i = j0 + j;
    x = (int)(i % M) * s0; y = (int)((i / M) % M) * s0; z = (int)(i / ((int64_t)M * M)) * s0;
  }
  xyz[j * 3 + 0] = axes[x]; xyz[j * 3 + 1] = axes[R + y]; xyz[j * 3 + 2] = axes[2 * R + z];
}

// the lattice values read from a given dense field
__global__ void __launch_bounds__(AM_THREADS) lattice_from_field_kernel(const float* __restrict__ field, int R, int s0, int M,
                                                                        float* __restrict__ coarse) {
  const int64_t j = (int64_t)blockIdx.x * AM_THREADS + threadIdx.x;
  if (j >= (int64_t)M * M * M) return;
  const int64_t x = (j % M) * s0, y = ((j / M) % M) * s0, z = (j / ((int64_t)M * M)) * s0;
  coarse[j] = field[(z * R + y) * R + x];
}

// classify the level's blocks; active ones are appended to `active` (counter[0])
__global__ void __launch_bounds__(AM_THREADS) classify_kernel(Field f, int l, const uint32_t* __restrict__ parents, int64_t n,
                                                              float tau, uint8_t* __restrict__ st,
                                                              uint32_t* __restrict__ active,
                                                              unsigned long long* __restrict__ counter) {
  const int64_t j = (int64_t)blockIdx.x * AM_THREADS + threadIdx.x;
  const int s = f.s[l], nb = f.nb[l];
  bool act = false;
  uint32_t b = 0;
  if (j < n) {
    int bx, by, bz;
    classified_block(j, parents, nb, bx, by, bz);
    float v[8];
    block_corners(f, s, bx, by, bz, v);
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
__global__ void __launch_bounds__(AM_THREADS) level_points_kernel(Field f, int l, const uint32_t* __restrict__ parents,
                                                                  int64_t n, unsigned long long* __restrict__ counter,
                                                                  unsigned long long* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * AM_THREADS + threadIdx.x;
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

__global__ void __launch_bounds__(AM_THREADS) table_insert_kernel(const unsigned long long* __restrict__ keys, int64_t n,
                                                                  const float* __restrict__ vals,
                                                                  const float* __restrict__ field,
                                                                  unsigned long long* __restrict__ tkeys,
                                                                  float* __restrict__ tvals, unsigned long long cap) {
  const int64_t j = (int64_t)blockIdx.x * AM_THREADS + threadIdx.x;
  if (j >= n) return;
  const unsigned long long key = keys[j];
  const float v = field ? field[key] : vals[j];
  unsigned long long i = slot_of(key, cap);
  while (atomicCAS(&tkeys[i], AM_EMPTY, key) != AM_EMPTY)
    if (++i == cap) i = 0;
  tvals[i] = v;
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
      block_corners(f, s, bx, by, bz, v);
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
  const float v0 = value_at(f, idx[0], idx[1], idx[2]);
  const float v1 = value_at(f, idx[0] + (a == 0), idx[1] + (a == 1), idx[2] + (a == 2));
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

int key_bits(unsigned long long max_key) {
  int b = 1;
  while (b < 64 && (max_key >> b)) ++b;
  return b;
}

// sorts n keys of keys[0] (keys[1] is the alternate buffer); returns the buffer that holds the result
int sort_keys(disn_ctx* c, DevBuffer (&keys)[2], int64_t n, int bits, unsigned long long** sorted) {
  DISN_REQUIRE(n < ((int64_t)1 << 31), "mesh_grid_adaptive: a list of 2^31 or more keys");
  cub::DoubleBuffer<unsigned long long> db(keys[0].as<unsigned long long>(), keys[1].as<unsigned long long>());
  size_t tmp = 0;
  DISN_CUDA_OK(cub::DeviceRadixSort::SortKeys(nullptr, tmp, db, (int)n, 0, bits, c->stream));
  if (c->am_sort_tmp.ensure(std::max<size_t>(tmp, 1))) return -1;
  DISN_CUDA_OK(cub::DeviceRadixSort::SortKeys(c->am_sort_tmp.as<void>(), tmp, db, (int)n, 0, bits, c->stream));
  *sorted = db.Current();
  return 0;
}

// the network at n explicit points xyz of one image -> out (pred / sdf_weight), as eval_indexed does in grid mode
int evaluate_points(disn_ctx* c, int image, const float* d_tm, const float* xyz, int64_t n, float* out) {
  PointJob job{};
  job.B = 1; job.N = n; job.pts = xyz; job.pts_rot = nullptr;
  job.gbias = c->gbias.as<float>() + (int64_t)image * kHidden;
  job.pmap = c->pmap.as<float>() + (int64_t)image * c->cfg.img_h * c->cfg.img_w * kHidden;
  job.trans_mat = d_tm;
  job.out_pred = out;
  job.out_div = c->cfg.sdf_weight;
  return run_point_job(c, job);
}

// values of n points (keys, or the coarse lattice with keys == nullptr) in chunks: xyz rows, then the network into
// out[j] (lattice) or the chunk buffer and from there into the level's table
int evaluate_chunks(disn_ctx* c, int image, const float* d_tm, const Field& f, const unsigned long long* keys, int64_t n,
                    float* out, unsigned long long* tkeys, float* tvals, unsigned long long cap) {
  const int64_t chunk = std::min<int64_t>(n, AM_CHUNK);
  if (c->am_xyz.ensure((size_t)chunk * 3 * sizeof(float)) || (keys && c->am_vals.ensure((size_t)chunk * sizeof(float))))
    return -1;
  for (int64_t j0 = 0; j0 < n; j0 += chunk) {
    const int64_t m = std::min<int64_t>(chunk, n - j0);
    xyz_kernel<<<blocks_of(m), AM_THREADS, 0, c->stream>>>(keys, j0, m, f.R, f.s0, f.M, c->d_axes.as<float>(),
                                                           c->am_xyz.as<float>());
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
    float* dst = keys ? c->am_vals.as<float>() : out + j0;
    if (evaluate_points(c, image, d_tm, c->am_xyz.as<float>(), m, dst)) return -1;
    if (keys) {
      table_insert_kernel<<<blocks_of(m), AM_THREADS, 0, c->stream>>>(keys + j0, m, dst, nullptr, tkeys, tvals, cap);
      c->launches++;
      DISN_CUDA_OK(cudaGetLastError());
    }
  }
  return 0;
}

}  // namespace

size_t adaptive_mesh_bytes(const disn_ctx* c) {
  size_t b = c->am_state.bytes() + c->am_coarse.bytes() + c->am_xyz.bytes() + c->am_vals.bytes() + c->am_sort_tmp.bytes() +
             c->am_case.bytes() + c->am_tri.bytes() + c->am_sums.bytes() + c->am_cnt.bytes();
  for (int k = 0; k < 2; ++k) b += c->am_keys[k].bytes() + c->am_edges[k].bytes();
  for (int l = 0; l < AD_MAX_LEVELS; ++l) b += c->am_table[l].bytes() + c->am_active[l].bytes();
  return b;
}

int adaptive_mesh_run(disn_ctx* c, const float* field, int image, const float* d_tm, int32_t res, const double* sdf_params,
                      float iso, double band, int64_t* level_counts, int32_t* n_levels, int64_t* n_verts,
                      int64_t* n_faces) {
  cudaStream_t st = c->stream;
  const int R = res + 1;
  c->am_nv = -1;
  c->am_edges_sorted = nullptr;
  Field f{};
  f.R = R;
  f.s0 = coarse_stride(res);
  f.iso = iso;
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
  if (c->am_state.ensure((size_t)std::max<int64_t>(states, 1)) || c->am_coarse.ensure((size_t)nM * sizeof(float)) ||
      c->am_cnt.ensure(4 * sizeof(unsigned long long)) || c->am_host.ensure(4 * sizeof(unsigned long long)))
    return -1;
  for (cudaEvent_t& e : c->am_ev)
    if (!e) DISN_CUDA_OK(cudaEventCreate(&e));
  unsigned long long* cnt = c->am_cnt.as<unsigned long long>();
  unsigned long long* hcnt = c->am_host.as<unsigned long long>();
  for (int l = 0; l < f.n; ++l) f.st[l] = c->am_state.as<uint8_t>() + state_off[l];
  DISN_CUDA_OK(cudaEventRecord(c->am_ev[0], st));

  // coarse lattice
  float* coarse = c->am_coarse.as<float>();
  f.coarse = coarse;
  if (field) {
    lattice_from_field_kernel<<<blocks_of(nM), AM_THREADS, 0, st>>>(field, R, f.s0, f.M, coarse);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
  } else if (evaluate_chunks(c, image, d_tm, f, nullptr, nM, coarse, nullptr, nullptr, 0)) {
    return -1;
  }
  level_counts[0] = nM;

  // levels: classify the children of the previous level's active blocks, emit the owned new points, sort, evaluate
  int64_t nclass[AD_MAX_LEVELS] = {};
  const uint32_t* parents[AD_MAX_LEVELS] = {};
  nclass[0] = states > 0 ? (int64_t)f.nb[0] * f.nb[0] * f.nb[0] : 0;
  for (int l = 0; l < f.n; ++l) {
    const int64_t n = nclass[l];
    DISN_CUDA_OK(cudaMemsetAsync(const_cast<uint8_t*>(f.st[l]), 0, (size_t)f.nb[l] * f.nb[l] * f.nb[l], st));
    DISN_CUDA_OK(cudaMemsetAsync(cnt, 0, 2 * sizeof(unsigned long long), st));
    if (c->am_active[l].ensure((size_t)std::max<int64_t>(n, 1) * sizeof(uint32_t))) return -1;
    if (n) {
      classify_kernel<<<blocks_of(n), AM_THREADS, 0, st>>>(f, l, parents[l], n, level_tau(band, f.s[l], sdf_params, res),
                                                           const_cast<uint8_t*>(f.st[l]), c->am_active[l].as<uint32_t>(), cnt);
      level_points_kernel<false><<<blocks_of(n), AM_THREADS, 0, st>>>(f, l, parents[l], n, cnt + 1, nullptr);
      c->launches += 2;
      DISN_CUDA_OK(cudaGetLastError());
    }
    DISN_CUDA_OK(cudaMemcpyAsync(hcnt, cnt, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    DISN_CUDA_OK(cudaStreamSynchronize(st));               // the level's counts size its list and the next level
    const int64_t n_active = (int64_t)hcnt[0], n_new = (int64_t)hcnt[1];
    level_counts[l + 1] = n_new;
    if (l + 1 < f.n) {
      nclass[l + 1] = 8 * n_active;
      parents[l + 1] = c->am_active[l].as<uint32_t>();
    }
    if (n_new == 0) continue;
    const unsigned long long cap = (unsigned long long)(n_new + n_new / 2 + 1);
    if (c->am_keys[0].ensure((size_t)n_new * 8) || c->am_keys[1].ensure((size_t)n_new * 8) ||
        c->am_table[l].ensure((size_t)cap * 12))
      return -1;
    DISN_CUDA_OK(cudaMemsetAsync(cnt + 1, 0, sizeof(unsigned long long), st));
    level_points_kernel<true><<<blocks_of(n), AM_THREADS, 0, st>>>(f, l, parents[l], n, cnt + 1,
                                                                    c->am_keys[0].as<unsigned long long>());
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
    unsigned long long* keys = nullptr;
    if (sort_keys(c, c->am_keys, n_new, key_bits((unsigned long long)R * R * R), &keys)) return -1;
    unsigned long long* tkeys = c->am_table[l].as<unsigned long long>();
    float* tvals = reinterpret_cast<float*>(tkeys + cap);
    DISN_CUDA_OK(cudaMemsetAsync(tkeys, 0xff, (size_t)cap * 8, st));
    if (field) {
      table_insert_kernel<<<blocks_of(n_new), AM_THREADS, 0, st>>>(keys, n_new, nullptr, field, tkeys, tvals, cap);
      c->launches++;
      DISN_CUDA_OK(cudaGetLastError());
    } else if (evaluate_chunks(c, image, d_tm, f, keys, n_new, nullptr, tkeys, tvals, cap)) {
      return -1;
    }
    f.t[l] = Table{tkeys, tvals, cap};
  }
  *n_levels = f.n + 1;
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
    if (c->am_keys[0].ensure((size_t)n_cells * 8) || c->am_keys[1].ensure((size_t)n_cells * 8)) return -1;
    DISN_CUDA_OK(cudaMemsetAsync(cnt, 0, sizeof(unsigned long long), st));
    for (int l = 0; l < f.n; ++l)
      if (nclass[l]) {
        cells_kernel<true><<<blocks_of(nclass[l]), AM_THREADS, 0, st>>>(f, l, parents[l], nclass[l], cnt,
                                                                         c->am_keys[0].as<unsigned long long>());
        c->launches++;
      }
    DISN_CUDA_OK(cudaGetLastError());
    if (sort_keys(c, c->am_keys, n_cells, key_bits((unsigned long long)R * R * R), &cells)) return -1;
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
    c->mc_nv = c->mc_nf = 0;                               // the resident mesh is replaced from here on
    if (ensure_mesh(c->mc_verts, c->mc_faces, nv, nf)) return -1;
    Geom g;
    for (int k = 0; k < 3; ++k) { g.lo[k] = sdf_params[k]; g.h[k] = (sdf_params[3 + k] - sdf_params[k]) / (double)(R - 1); }
    vertices_kernel<<<blocks_of(nv), AM_THREADS, 0, st>>>(f, g, edges, nv, c->mc_verts.as<float>());
    faces_kernel<<<blocks_of(n_cells), AM_THREADS, 0, st>>>(cells, n_cells, R, cases, foff, edges, nv,
                                                            c->mc_faces.as<int32_t>());
    c->launches += 2;
    DISN_CUDA_OK(cudaGetLastError());
  } else {
    c->mc_nv = c->mc_nf = 0;
    if (ensure_mesh(c->mc_verts, c->mc_faces, 0, 0)) return -1;
  }
  DISN_CUDA_OK(cudaEventRecord(c->am_ev[3], st));
  DISN_CUDA_OK(cudaStreamSynchronize(st));
  c->mc_nv = nv; c->mc_nf = nf;
  c->am_nv = nv;
  if (n_verts) *n_verts = nv;
  if (n_faces) *n_faces = nf;
  return 0;
}

}  // namespace disn
