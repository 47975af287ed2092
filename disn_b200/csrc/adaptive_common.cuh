// Definitions shared by the coarse-to-fine grid (adaptive.cu), the dense marching cubes (mc.cu) and the surface-only
// mesher (adaptive_mesh.cu): DESIGN.md §4.9 / §4.10.  Both paths call these, so they compute the same bits.  The
// refinement itself (adaptive_refine, adaptive.cu) is one for both paths; they differ only in where the values go.
#pragma once
#include <stdint.h>

#include <cmath>

#include "common.cuh"

namespace disn {

constexpr int AD_MAX_LEVELS = 4;                   // s0 <= 16: levels 16, 8, 4, 2

// s0: the largest power of two <= 16 that divides res (1: no refinement, the dense grid)
inline int coarse_stride(int res) {
  int s0 = 16;
  while (s0 > 1 && res % s0) s0 >>= 1;
  return s0;
}

// tau_s = float32(band * (s/2) * sqrt(hx^2 + hy^2 + hz^2)) in float64, h = (max - min) / res per axis
inline float level_tau(double band, int s, const double* sdf_params, int res) {
  const double hx = (sdf_params[3] - sdf_params[0]) / res, hy = (sdf_params[4] - sdf_params[1]) / res,
               hz = (sdf_params[5] - sdf_params[2]) / res;
  return (float)(band * (s / 2) * std::sqrt(hx * hx + hy * hy + hz * hz));
}

// Block activity from its 8 corner values (corner k at (k & 1, k >> 1 & 1, k >> 2 & 1)): the corners are not all on one
// side of iso under marching cubes' v < iso, or one lies within tau of it (float32)
__device__ __forceinline__ bool block_active(const float (&v)[8], float iso, float tau) {
  int below = 0;
  bool near = false;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    below += (v[k] < iso) ? 1 : 0;
    near |= fabsf(__fsub_rn(v[k], iso)) <= tau;
  }
  return (below != 0 && below != 8) || near;
}

__device__ __forceinline__ float lerp_rn(float t, float a, float b) {
  return __fadd_rn(__fmul_rn(__fsub_rn(1.f, t), a), __fmul_rn(t, b));
}

// Fill value at (tx, ty, tz) in [0,1]^3 of a block with corner values v (order as above): x, then y, then z, each step
// rounded per operation
__device__ __forceinline__ float trilinear(const float (&v)[8], float tx, float ty, float tz) {
  float cz[2];
#pragma unroll
  for (int kz = 0; kz < 2; ++kz) {
    const float c0 = lerp_rn(tx, v[4 * kz + 0], v[4 * kz + 1]);
    const float c1 = lerp_rn(tx, v[4 * kz + 2], v[4 * kz + 3]);
    cz[kz] = lerp_rn(ty, c0, c1);
  }
  return lerp_rn(tz, cz[0], cz[1]);
}

// candidate block origins (in blocks) of coordinate c at block size s: the block starting at or below c, then the block
// ending at c; returns how many are valid
__device__ __forceinline__ int block_candidates(int c, int s, int nb, int (&q)[2]) {
  int k = 0;
  const int q0 = c / s;
  if (q0 < nb) q[k++] = q0;
  if (c % s == 0 && q0 >= 1) q[k++] = q0 - 1;
  return k;
}

// marching-cubes case of a cell from its corner values (bit k set: corner k is inside, v < iso)
__device__ __forceinline__ int cell_case_of(const float (&v)[8], float iso) {
  int cs = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) cs |= (v[k] < iso) ? (1 << k) : 0;
  return cs;
}

// Vertex on the lattice edge from point idx along axis a, values v0f at idx and v1f at its neighbour: float64 with one
// rounding per operation (as the oracle computes it), then float32
__device__ __forceinline__ void edge_vertex(const double (&lo)[3], const double (&h)[3], const int (&idx)[3], int a,
                                            float v0f, float v1f, float iso, float* out) {
  double p[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) p[k] = __dadd_rn(lo[k], __dmul_rn((double)idx[k], h[k]));
  const double t = __ddiv_rn(__dsub_rn((double)iso, (double)v0f), __dsub_rn((double)v1f, (double)v0f));
  p[a] = __dadd_rn(p[a], __dmul_rn(t, h[a]));
  out[0] = (float)p[0]; out[1] = (float)p[1]; out[2] = (float)p[2];
}

// ---- the refinement's values and block states ------------------------------------------------------------------------

constexpr unsigned long long AM_EMPTY = ~0ull;     // free hash slot

struct Table {
  const unsigned long long* keys;
  const float* vals;
  unsigned long long cap;                          // 0: no table (an empty or not yet evaluated level)
};

// what the device kernels read: the lattice values, the states of every level, and the evaluated values of the levels:
// the dense grid (dense path) or one hash table per level (mesher)
struct Field {
  int R, s0, lg0, n;                               // points per axis, coarse stride, log2(s0), number of levels
  int M;                                           // coarse lattice points per axis
  const float* coarse;                             // [M,M,M]
  const float* grid;                               // [R,R,R] (nullptr: the tables)
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

// the stored value of point (x, y, z) if it was evaluated, without a grid: the coarse lattice, or the table of the only
// level that can have evaluated it (lowest set bit b of x|y|z below log2(s0): level s = 2^(b+1))
__device__ __forceinline__ bool stored(const Field& f, int x, int y, int z, float& v) {
  const int g = x | y | z;
  if ((g & (f.s0 - 1)) == 0) {
    v = f.coarse[((int64_t)(z / f.s0) * f.M + y / f.s0) * f.M + x / f.s0];
    return true;
  }
  const int l = f.lg0 - __ffs(g);
  return lookup(f.t[l], ((unsigned long long)z * f.R + y) * f.R + x, v);
}

// the 8 corner values of block (bx, by, bz) of size s (all evaluated: the stride-s points of an active parent), from the
// dense grid (kGrid) or the lattice and tables.  A compile-time choice: a run-time branch here slows the mesher's kernels.
template <bool kGrid>
__device__ __forceinline__ void block_corners(const Field& f, int s, int bx, int by, int bz, float (&v)[8]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int x = (bx + (k & 1)) * s, y = (by + ((k >> 1) & 1)) * s, z = (bz + ((k >> 2) & 1)) * s;
    if (kGrid) v[k] = f.grid[((int64_t)z * f.R + y) * f.R + x];
    else stored(f, x, y, z, v[k]);
  }
}

// the dense adaptive grid's value at (x, y, z): stored, else the fill of the finest classified inactive block.  kGrid: the
// dense grid's fill of a point the refinement did not evaluate
template <bool kGrid>
static __device__ float value_at(const Field& f, int x, int y, int z) {
  float v;
  if (!kGrid && stored(f, x, y, z, v)) return v;
  for (int l = f.n - 1; l >= 0; --l) {             // finest level first
    const int s = f.s[l], nb = f.nb[l];
    int qx[2], qy[2], qz[2];
    const int nx = block_candidates(x, s, nb, qx), ny = block_candidates(y, s, nb, qy), nz = block_candidates(z, s, nb, qz);
    for (int a = 0; a < nz; ++a)
      for (int b = 0; b < ny; ++b)
        for (int d = 0; d < nx; ++d) {
          if (f.st[l][((int64_t)qz[a] * nb + qy[b]) * nb + qx[d]] != 1) continue;
          float cv[8];
          block_corners<kGrid>(f, s, qx[d], qy[b], qz[a], cv);
          const float inv = 1.f / (float)s;        // s is a power of two: the products below are exact
          const float tx = (float)(x - qx[d] * s) * inv, ty = (float)(y - qy[b] * s) * inv,
                      tz = (float)(z - qz[a] * s) * inv;
          return trilinear(cv, tx, ty, tz);
        }
  }
  return __int_as_float(0x7fc00000);               // unreachable: every point lies in a classified inactive block
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

// ---- the refinement (adaptive.cu) ------------------------------------------------------------------------------------

// what a refinement leaves for the caller's passes over the classified blocks
struct Refinement {
  Field f;
  int64_t nclass[AD_MAX_LEVELS];                   // classified blocks of each level
  const uint32_t* parents[AD_MAX_LEVELS];          // the level's parents: the previous level's active blocks (nullptr at
                                                   // the first level, which classifies every block)
};

// The lattice and levels of §4.9 for res with s0 >= 2, values from `field` (device [R,R,R]) when it is non-null, else
// from the network (eval_grid_points).  The values go into `grid`, with `mark` set to 1 at every evaluated point, when
// grid is non-null (mark must be zero on entry); else into one hash table per level (c->am_table).  ev, when non-null,
// gets one event after the lattice and one after each level.  Level counts: [lattice, level s0, ..., level 2].
int adaptive_refine(disn_ctx* c, const float* field, int image, const float* d_tm, int32_t res, const double* sdf_params,
                    float iso, double band, float* grid, uint8_t* mark, cudaEvent_t* ev, Refinement& r,
                    int64_t* level_counts, int32_t* n_levels);

inline int key_bits(unsigned long long max_key) {
  int b = 1;
  while (b < 64 && (max_key >> b)) ++b;
  return b;
}

// radix-sorts n keys of keys[0] (keys[1] is the alternate buffer) on c->stream; *sorted = the buffer holding the result
int sort_keys(disn_ctx* c, DevBuffer (&keys)[2], int64_t n, int bits, unsigned long long** sorted);

}  // namespace disn
