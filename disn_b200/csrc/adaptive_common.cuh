// Definitions shared by the coarse-to-fine grid (adaptive.cu), the dense marching cubes (mc.cu) and the surface-only
// mesher (adaptive_mesh.cu): DESIGN.md §4.9 / §4.10.  Both paths call these, so they compute the same bits.
#pragma once
#include <stdint.h>

#include <cmath>

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

}  // namespace disn
