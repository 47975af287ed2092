// Signed distance field of the resident mesh on an R^3 grid: the reference's closed computeDistanceField -s step
// (preprocessing/create_point_sdf_grid.py:200-210).  Definitions are shared with the CPU twin oracle/mesh_sdf_oracle.py,
// which this file reproduces bit for bit (DESIGN.md §4.7):
//   * grid point (i,j,k) = (X[i], Y[j], Z[k]), the float64-linspace -> float32 tables of disn_eval_grid; layout [z][y][x];
//   * d(p) = float32(sqrt(min over faces of d2(p, face))), d2 = |p - q|^2 with q from Ericson's region-based closest point
//     on a triangle (Real-Time Collision Detection §5.1.5) in float64 on the widened float32 coordinates; a face whose
//     float64 cross product is exactly zero counts as its three edge segments;
//   * the grid edge between 6-neighbours is blocked when the closed segment crosses a closed face (per-axis line
//     rasterisation: closed 2D edge-function test with canonically ordered edges, crossing coordinate from the plane
//     equation, a crossing exactly on a grid point blocks both incident edges);
//   * wall point: d <= sigma; exterior: non-wall and connected to a non-wall boundary point through open edges between
//     non-wall points; output +d on exterior points, -d elsewhere.
// fp64, integer and tree-walk work: nothing for the tensor cores.  Built with --fmad=false.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>

#include "common.cuh"

namespace disn {
namespace {

constexpr int SD_THREADS = 256;
constexpr int LEAF = 4;                  // faces per BVH leaf
constexpr int STACK = 32;                // > tree depth: leaves < 2^31 / 3 / LEAF < 2^28
constexpr double PRUNE_REL = 0x1p-20;    // relative and absolute (x max |coordinate|) slack of the BVH pruning test
constexpr double PRUNE_ABS = 0x1p-24;

// mesh statistics: ordered-int encodings of the vertex AABB, a non-finite flag, and the 64-bit raster work total
enum { S_LO = 0, S_HI = 3, S_BAD = 6, S_WORK = 8, S_COUNT = 10 };

inline unsigned grid_of(int64_t n) { return (unsigned)((n + SD_THREADS - 1) / SD_THREADS); }

__device__ __forceinline__ uint32_t ord(float f) {          // monotone float -> uint32 map
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
inline float unord(uint32_t u) {
  u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
  float f;
  std::memcpy(&f, &u, sizeof f);
  return f;
}

__global__ void __launch_bounds__(SD_THREADS) sdf_stats_kernel(const float* __restrict__ verts, int64_t nv,
                                                               uint32_t* stats) {
  const int64_t v = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x;
  if (v >= nv) return;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float x = verts[3 * v + a];
    if (!isfinite(x)) { atomicOr(&stats[S_BAD], 1u); return; }
    atomicMin(&stats[S_LO + a], ord(x));
    atomicMax(&stats[S_HI + a], ord(x));
  }
}

__device__ __forceinline__ uint32_t spread10(uint32_t x) {    // 10 bits -> every third bit
  x &= 0x3ffu;
  x = (x | (x << 16)) & 0x030000ffu;
  x = (x | (x << 8)) & 0x0300f00fu;
  x = (x | (x << 4)) & 0x030c30c3u;
  x = (x | (x << 2)) & 0x09249249u;
  return x;
}

// 30-bit Morton code of each face centroid in the mesh AABB (keys) and the face index (values)
__global__ void __launch_bounds__(SD_THREADS) sdf_morton_kernel(const float* __restrict__ verts,
                                                                const int32_t* __restrict__ faces, int64_t nf,
                                                                float3 lo, float3 scale, uint32_t* __restrict__ key,
                                                                int32_t* __restrict__ val) {
  const int64_t f = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x;
  if (f >= nf) return;
  float c[3];
  const float l[3] = {lo.x, lo.y, lo.z}, s[3] = {scale.x, scale.y, scale.z};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float m = (verts[3 * faces[3 * f] + a] + verts[3 * faces[3 * f + 1] + a] + verts[3 * faces[3 * f + 2] + a]) / 3.f;
    c[a] = fminf(fmaxf((m - l[a]) * s[a], 0.f), 1023.f);
  }
  key[f] = spread10((uint32_t)c[0]) | (spread10((uint32_t)c[1]) << 1) | (spread10((uint32_t)c[2]) << 2);
  val[f] = (int32_t)f;
}

// triangles in Morton order (9 floats each) and the leaf boxes; leaves past the last face get empty boxes
__global__ void __launch_bounds__(SD_THREADS) sdf_leaves_kernel(const float* __restrict__ verts,
                                                                const int32_t* __restrict__ faces,
                                                                const int32_t* __restrict__ order, int64_t nf,
                                                                int64_t nleaf_slots, float* __restrict__ tri,
                                                                float4* __restrict__ blo, float4* __restrict__ bhi) {
  const int64_t l = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x;
  if (l >= nleaf_slots) return;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int64_t t = l * LEAF; t < min((l + 1) * LEAF, nf); ++t) {
    const int64_t f = order[t];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const float x = verts[3 * (int64_t)faces[3 * f + k] + a];
        tri[9 * t + 3 * k + a] = x;
        lo[a] = fminf(lo[a], x);
        hi[a] = fmaxf(hi[a], x);
      }
  }
  const int64_t node = nleaf_slots - 1 + l;
  blo[node] = make_float4(lo[0], lo[1], lo[2], 0.f);
  bhi[node] = make_float4(hi[0], hi[1], hi[2], 0.f);
}

// one level of the implicit (heap-ordered) tree: node n = union of children 2n+1, 2n+2
__global__ void __launch_bounds__(SD_THREADS) sdf_refit_kernel(int64_t first, int64_t count, float4* blo, float4* bhi) {
  const int64_t i = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x;
  if (i >= count) return;
  const int64_t n = first + i;
  const float4 a = blo[2 * n + 1], b = blo[2 * n + 2], c = bhi[2 * n + 1], d = bhi[2 * n + 2];
  blo[n] = make_float4(fminf(a.x, b.x), fminf(a.y, b.y), fminf(a.z, b.z), 0.f);
  bhi[n] = make_float4(fmaxf(c.x, d.x), fmaxf(c.y, d.y), fmaxf(c.z, d.z), 0.f);
}

// ---- exact point-triangle distance (the oracle's tri_dist2, operation for operation) ----------------------------------
struct D3 { double x, y, z; };
__device__ __forceinline__ D3 sub(D3 a, D3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ double dot(D3 a, D3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
__device__ __forceinline__ double dist2(D3 p, D3 q) { return dot(sub(p, q), sub(p, q)); }
__device__ __forceinline__ D3 cross(D3 a, D3 b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}

__device__ __forceinline__ double seg_dist2(D3 p, D3 a, D3 b) {
  const D3 e = sub(b, a);
  const double ee = dot(e, e);
  if (ee == 0.0) return dist2(p, a);
  double t = dot(sub(p, a), e) / ee;
  t = t < 0.0 ? 0.0 : (t > 1.0 ? 1.0 : t);
  return dist2(p, {a.x + t * e.x, a.y + t * e.y, a.z + t * e.z});
}

__device__ double tri_dist2(D3 p, D3 a, D3 b, D3 c) {
  const D3 ab = sub(b, a), ac = sub(c, a);
  const D3 n = cross(ab, ac);
  if (n.x == 0.0 && n.y == 0.0 && n.z == 0.0) {
    double d = seg_dist2(p, a, b);
    const double d1 = seg_dist2(p, b, c), d2 = seg_dist2(p, c, a);
    if (d1 < d) d = d1;
    if (d2 < d) d = d2;
    return d;
  }
  const D3 ap = sub(p, a);
  const double d1 = dot(ab, ap), d2 = dot(ac, ap);
  if (d1 <= 0.0 && d2 <= 0.0) return dist2(p, a);
  const D3 bp = sub(p, b);
  const double d3 = dot(ab, bp), d4 = dot(ac, bp);
  if (d3 >= 0.0 && d4 <= d3) return dist2(p, b);
  const double vc = d1 * d4 - d3 * d2;
  if (vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0) {
    const double v = d1 / (d1 - d3);
    return dist2(p, {a.x + v * ab.x, a.y + v * ab.y, a.z + v * ab.z});
  }
  const D3 cp = sub(p, c);
  const double d5 = dot(ab, cp), d6 = dot(ac, cp);
  if (d6 >= 0.0 && d5 <= d6) return dist2(p, c);
  const double vb = d5 * d2 - d1 * d6;
  if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) {
    const double w = d2 / (d2 - d6);
    return dist2(p, {a.x + w * ac.x, a.y + w * ac.y, a.z + w * ac.z});
  }
  const double va = d3 * d6 - d5 * d4;
  if (va <= 0.0 && (d4 - d3) >= 0.0 && (d5 - d6) >= 0.0) {
    const double w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
    const D3 bc = sub(c, b);
    return dist2(p, {b.x + w * bc.x, b.y + w * bc.y, b.z + w * bc.z});
  }
  const double denom = 1.0 / ((va + vb) + vc);
  const double v = vb * denom, w = vc * denom;
  return dist2(p, {(a.x + ab.x * v) + ac.x * w, (a.y + ab.y * v) + ac.y * w, (a.z + ab.z * v) + ac.z * w});
}

__device__ __forceinline__ double box_lb(D3 p, const float4* blo, const float4* bhi, int64_t n) {
  const float4 lo = blo[n], hi = bhi[n];
  const double dx = fmax(fmax((double)lo.x - p.x, p.x - (double)hi.x), 0.0);
  const double dy = fmax(fmax((double)lo.y - p.y, p.y - (double)hi.y), 0.0);
  const double dz = fmax(fmax((double)lo.z - p.z, p.z - (double)hi.z), 0.0);
  return (dx * dx + dy * dy) + dz * dz;
}

// A node is skipped only when its box is farther than the best distance so far plus a slack far above the rounding of
// any face's computed distance, so the minimum equals the brute-force minimum over all faces.
__device__ __forceinline__ double prune_threshold(double best, double slack) {
  const double r = sqrt(best) * (1.0 + PRUNE_REL) + slack;
  return r * r;
}

// One thread per grid point; a warp covers a 4x4x2 brick (a block 8x4x4) so its threads walk the same nodes.  Nearest
// child first, an explicit stack; d = float32(sqrt(min d2)) into dist.
__global__ void __launch_bounds__(128) sdf_distance_kernel(const float* __restrict__ axes, int R,
                                                           const float* __restrict__ tri, int64_t nf,
                                                           const float4* __restrict__ blo, const float4* __restrict__ bhi,
                                                           int64_t nleaf_slots, double slack, float* __restrict__ dist) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x = blockIdx.x * 8 + (warp & 1) * 4 + (lane & 3);
  const int y = blockIdx.y * 4 + ((lane >> 2) & 3);
  const int z = blockIdx.z * 4 + (warp >> 1) * 2 + (lane >> 4);
  if (x >= R || y >= R || z >= R) return;
  const D3 p = {(double)axes[x], (double)axes[R + y], (double)axes[2 * R + z]};
  const int64_t first_leaf = nleaf_slots - 1;
  double best = INFINITY, thr = INFINITY;
  int32_t stack[STACK];
  int sp = 0;
  int64_t node = 0;
  while (true) {
    if (node >= first_leaf) {
      const int64_t t0 = (node - first_leaf) * LEAF, t1 = min(t0 + LEAF, nf);
      for (int64_t t = t0; t < t1; ++t) {
        const float* v = tri + 9 * t;
        const double d2 = tri_dist2(p, {(double)v[0], (double)v[1], (double)v[2]}, {(double)v[3], (double)v[4], (double)v[5]},
                                    {(double)v[6], (double)v[7], (double)v[8]});
        if (d2 < best) { best = d2; thr = prune_threshold(best, slack); }
      }
    } else {
      const int64_t l = 2 * node + 1, r = l + 1;
      const double ll = box_lb(p, blo, bhi, l), lr = box_lb(p, blo, bhi, r);
      const bool tl = !(ll > thr), tr = !(lr > thr);
      if (tl && tr) {
        const bool left_first = ll <= lr;
        stack[sp++] = (int32_t)(left_first ? r : l);
        node = left_first ? l : r;
        continue;
      }
      if (tl || tr) { node = tl ? l : r; continue; }
    }
    node = -1;
    while (sp > 0) {
      const int64_t n = stack[--sp];
      if (!(box_lb(p, blo, bhi, n) > thr)) { node = n; break; }
    }
    if (node < 0) break;
  }
  dist[((int64_t)z * R + y) * R + x] = (float)sqrt(best);
}

// ---- blocked grid edges ------------------------------------------------------------------------------------------------
// first index i with G[i] >= t (lower) / G[i] > t (upper) in the increasing float32 table G[0..n)
__device__ __forceinline__ int lower_idx(const float* G, int n, double t) {
  int lo = 0, hi = n;
  while (lo < hi) { const int m = (lo + hi) >> 1; if ((double)G[m] < t) lo = m + 1; else hi = m; }
  return lo;
}
__device__ __forceinline__ int upper_idx(const float* G, int n, double t) {
  int lo = 0, hi = n;
  while (lo < hi) { const int m = (lo + hi) >> 1; if ((double)G[m] <= t) lo = m + 1; else hi = m; }
  return lo;
}

struct Face {
  float v[3][3];
  __device__ void load(const float* verts, const int32_t* faces, int64_t f) {
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int a = 0; a < 3; ++a) v[k][a] = verts[3 * (int64_t)faces[3 * f + k] + a];
  }
};

// lines of axis a the face's projected bounding box covers: j in [j0, j0+nj) on axis (a+1)%3, k in [k0, k0+nk) on
// (a+2)%3; none when the face's normal has a zero a-component (the face is parallel to the lines)
__device__ __forceinline__ int64_t face_lines(const Face& F, const double n[3], int a, const float* G, int R, int& j0,
                                              int& nj, int& k0) {
  if (n[a] == 0.0) return 0;
  const int b = (a + 1) % 3, c = (a + 2) % 3;
  const float bmin = fminf(fminf(F.v[0][b], F.v[1][b]), F.v[2][b]), bmax = fmaxf(fmaxf(F.v[0][b], F.v[1][b]), F.v[2][b]);
  const float cmin = fminf(fminf(F.v[0][c], F.v[1][c]), F.v[2][c]), cmax = fmaxf(fmaxf(F.v[0][c], F.v[1][c]), F.v[2][c]);
  j0 = lower_idx(G + b * R, R, bmin);
  nj = max(upper_idx(G + b * R, R, bmax) - j0, 0);
  k0 = lower_idx(G + c * R, R, cmin);
  const int nk = max(upper_idx(G + c * R, R, cmax) - k0, 0);
  return (int64_t)nj * nk;
}

__device__ __forceinline__ void face_normal(const Face& F, double n[3]) {
  const D3 A = {F.v[0][0], F.v[0][1], F.v[0][2]}, B = {F.v[1][0], F.v[1][1], F.v[1][2]}, C = {F.v[2][0], F.v[2][1], F.v[2][2]};
  const D3 m = cross(sub(B, A), sub(C, A));
  n[0] = m.x; n[1] = m.y; n[2] = m.z;
}

__device__ __forceinline__ void load_axes(const float* axes, int R, float* G) {
  for (int i = threadIdx.x; i < 3 * R; i += blockDim.x) G[i] = axes[i];
  __syncthreads();
}

// per face: number of (axis, line) work items; cnt[nf] = 0 so the exclusive scan ends in the total
__global__ void __launch_bounds__(SD_THREADS) sdf_line_count_kernel(const float* __restrict__ verts,
                                                                    const int32_t* __restrict__ faces, int64_t nf,
                                                                    const float* __restrict__ axes, int R,
                                                                    uint32_t* __restrict__ cnt,
                                                                    unsigned long long* total) {
  extern __shared__ float G[];
  load_axes(axes, R, G);
  const int64_t f = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x;
  if (f == 0) cnt[nf] = 0;
  if (f >= nf) return;
  Face F;
  F.load(verts, faces, f);
  double n[3];
  face_normal(F, n);
  int64_t s = 0;
  int j0, nj, k0;
#pragma unroll
  for (int a = 0; a < 3; ++a) s += face_lines(F, n, a, G, R, j0, nj, k0);
  cnt[f] = (uint32_t)s;
  atomicAdd(total, (unsigned long long)s);
}

// edge function of the projected edge P->Q at s, evaluated with the endpoints in lexicographic (x,y,z) order and negated
// when reversed: faces sharing an edge classify a line through it identically
__device__ __forceinline__ bool lex_less(const float* p, const float* q) {
  return p[0] < q[0] || (p[0] == q[0] && (p[1] < q[1] || (p[1] == q[1] && p[2] < q[2])));
}
__device__ __forceinline__ double edge_fn(const float* P, const float* Q, int b, int c, double sb, double sc) {
  const bool rev = lex_less(Q, P);
  const float* u = rev ? Q : P;
  const float* v = rev ? P : Q;
  const double e = ((double)v[b] - (double)u[b]) * (sc - (double)u[c]) - ((double)v[c] - (double)u[c]) * (sb - (double)u[b]);
  return rev ? -e : e;
}

__device__ __forceinline__ void set_bit(uint32_t* bits, int64_t idx, uint32_t bit) {
  atomicOr(&bits[idx >> 2], bit << (8 * (idx & 3)));
}

// Grid-stride over the (face, axis, line) items: face = last f with offs[f] <= w; a closed 2D point-in-triangle test on
// the line, then the crossing coordinate from the plane equation blocks the grid edge(s) whose closed segment holds it.
__global__ void __launch_bounds__(SD_THREADS) sdf_raster_kernel(const float* __restrict__ verts,
                                                                const int32_t* __restrict__ faces, int64_t nf,
                                                                const float* __restrict__ axes, int R,
                                                                const uint32_t* __restrict__ offs,
                                                                const uint32_t* __restrict__ d_total,
                                                                uint32_t* bits) {
  extern __shared__ float G[];
  load_axes(axes, R, G);
  const uint32_t total = *d_total;
  for (int64_t w = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x; w < total; w += (int64_t)gridDim.x * SD_THREADS) {
    int64_t lo = 0, hi = nf;                       // largest f in [0, nf) with offs[f] <= w
    while (hi - lo > 1) { const int64_t m = (lo + hi) >> 1; if (offs[m] <= w) lo = m; else hi = m; }
    const int64_t f = lo;
    int64_t local = w - (int64_t)offs[f];
    if (local < 0) continue;
    Face F;
    F.load(verts, faces, f);
    double n[3];
    face_normal(F, n);
    for (int a = 0; a < 3; ++a) {
      int j0, nj, k0;
      const int64_t m = face_lines(F, n, a, G, R, j0, nj, k0);
      if (local >= m) { local -= m; continue; }
      const int b = (a + 1) % 3, c = (a + 2) % 3;
      const int j = j0 + (int)(local % nj), k = k0 + (int)(local / nj);
      const double sb = G[b * R + j], sc = G[c * R + k];
      const double e0 = edge_fn(F.v[1], F.v[2], b, c, sb, sc);
      const double e1 = edge_fn(F.v[2], F.v[0], b, c, sb, sc);
      const double e2 = edge_fn(F.v[0], F.v[1], b, c, sb, sc);
      if ((e0 >= 0.0 && e1 >= 0.0 && e2 >= 0.0) || (e0 <= 0.0 && e1 <= 0.0 && e2 <= 0.0)) {
        const double A[3] = {F.v[0][0], F.v[0][1], F.v[0][2]};
        const double t = A[a] - (n[b] * (sb - A[b]) + n[c] * (sc - A[c])) / n[a];
        const int i0 = max(lower_idx(G + a * R, R, t) - 1, 0), i1 = min(upper_idx(G + a * R, R, t) - 1, R - 2);
        int q[3];
        q[b] = j; q[c] = k;
        for (int i = i0; i <= i1; ++i) {
          q[a] = i;
          set_bit(bits, ((int64_t)q[2] * R + q[1]) * R + q[0], 1u << a);
        }
      }
      break;
    }
  }
}

// ---- exterior flood fill -----------------------------------------------------------------------------------------------
constexpr uint8_t EXTERIOR_ROOT = 8;        // bit of a root's edge byte: reached by a non-wall boundary point

__global__ void __launch_bounds__(SD_THREADS) sdf_init_kernel(int32_t* __restrict__ parent, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x;
  if (i < n) parent[i] = (int32_t)i;
}

// hook each non-wall point to its +x, +y, +z neighbours over open edges between non-wall points
__global__ void __launch_bounds__(SD_THREADS) sdf_union_kernel(const float* __restrict__ dist, double sigma,
                                                               int R, const uint8_t* __restrict__ bits, int32_t* parent) {
  const int64_t n = (int64_t)R * R * R;
  const int64_t i = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x;
  if (i >= n || (double)dist[i] <= sigma) return;
  const int x = (int)(i % R), y = (int)((i / R) % R), z = (int)(i / ((int64_t)R * R));
  const int co[3] = {x, y, z};
  const int64_t stride[3] = {1, R, (int64_t)R * R};
  const uint8_t e = bits[i];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    if (co[a] < R - 1 && !(e & (1u << a)) && !((double)dist[i + stride[a]] <= sigma))
      uf_union(parent, (int32_t)i, (int32_t)(i + stride[a]));
}

__global__ void __launch_bounds__(SD_THREADS) sdf_flatten_kernel(int32_t* parent, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x;
  if (i < n) parent[i] = uf_root(parent, (int32_t)i);
}

__global__ void __launch_bounds__(SD_THREADS) sdf_boundary_kernel(const float* __restrict__ dist, double sigma, int R,
                                                                  const int32_t* __restrict__ parent, uint32_t* bits) {
  const int64_t n = (int64_t)R * R * R;
  const int64_t i = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x;
  if (i >= n) return;
  const int x = (int)(i % R), y = (int)((i / R) % R), z = (int)(i / ((int64_t)R * R));
  const bool boundary = x == 0 || y == 0 || z == 0 || x == R - 1 || y == R - 1 || z == R - 1;
  if (boundary && !((double)dist[i] <= sigma)) set_bit(bits, parent[i], EXTERIOR_ROOT);
}

__global__ void __launch_bounds__(SD_THREADS) sdf_sign_kernel(float* dist, double sigma, int64_t n,
                                                              const int32_t* __restrict__ parent,
                                                              const uint8_t* __restrict__ bits) {
  const int64_t i = (int64_t)blockIdx.x * SD_THREADS + threadIdx.x;
  if (i >= n) return;
  const float d = dist[i];
  const bool exterior = !((double)d <= sigma) && (bits[parent[i]] & EXTERIOR_ROOT);
  dist[i] = exterior ? d : -d;
}

struct SdfBufs {
  uint32_t *key, *key_alt, *cnt, *scan, *total32;
  int32_t *val, *val_alt, *parent;
  unsigned long long* work;
  float *tri, *dist;
  float4 *blo, *bhi;
  float* axes;
  uint32_t* bits;
  void* cub_tmp;
};

size_t carve(char* base, int64_t nf, int64_t nleaf_slots, int R, bool own_dist, size_t cub_bytes, SdfBufs& b) {
  const int64_t npts = (int64_t)R * R * R;
  Arena a{base};
  b.key = a.take<uint32_t>(nf);
  b.key_alt = a.take<uint32_t>(nf);
  b.val = a.take<int32_t>(nf);
  b.val_alt = a.take<int32_t>(nf);
  b.cub_tmp = a.take<char>(cub_bytes);
  b.tri = a.take<float>(9 * nf);
  b.blo = a.take<float4>(2 * nleaf_slots);
  b.bhi = a.take<float4>(2 * nleaf_slots);
  b.axes = a.take<float>(3 * R);
  b.cnt = a.take<uint32_t>(nf + 1);
  b.scan = a.take<uint32_t>(scan_scratch_elems(nf + 1));
  b.total32 = a.take<uint32_t>(1);
  b.work = a.take<unsigned long long>(1);
  b.bits = a.take<uint32_t>((npts + 3) / 4);
  b.parent = a.take<int32_t>(npts);
  b.dist = own_dist ? a.take<float>(npts) : nullptr;
  return a.off;
}

}  // namespace

// Stream-ordered: statistics (one host synchronisation: the AABB for the automatic box and the non-finite guard) ->
// Morton sort -> leaves -> per-level refit -> distance -> line counts -> scan -> rasterise -> union-find -> flatten ->
// boundary flags -> sign; a second synchronisation at the end (output copy, the raster work total).
int mesh_sdf(disn_ctx* c, int32_t res, const double* bbox, double expand_rate, double sigma, float* out,
             double* bbox_out, bool device_out) {
  const int64_t nv = c->mesh.nv(), nf = c->mesh.nf();
  DISN_REQUIRE(nf > 0, "mesh_sdf: no resident mesh with faces (disn_mesh_load / disn_mc_run first)");
  DISN_REQUIRE(nv < ((int64_t)1 << 31) && 3 * nf < ((int64_t)1 << 31), "mesh too large for 32-bit indices");
  const int R = res + 1;
  const int64_t npts = (int64_t)R * R * R;
  cudaStream_t s = c->stream;
  for (cudaEvent_t& e : c->sdf_ev)
    if (!e) DISN_CUDA_OK(cudaEventCreate(&e));

  // host staging: stats words, then 3R float axis tables
  if (c->sdf_host.ensure(S_COUNT * sizeof(uint32_t) + 3 * (size_t)R * sizeof(float))) return -1;
  uint32_t* hs = c->sdf_host.as<uint32_t>();
  float* haxes = reinterpret_cast<float*>(hs + S_COUNT);

  const int64_t nleaves = (nf + LEAF - 1) / LEAF;
  int64_t nleaf_slots = 1;
  while (nleaf_slots < nleaves) nleaf_slots <<= 1;
  size_t cub_bytes = 0;
  {
    cub::DoubleBuffer<uint32_t> k0(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> v0(nullptr, nullptr);
    DISN_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, k0, v0, (int)nf, 0, 30, s));
  }
  SdfBufs b;
  const size_t bytes = carve(nullptr, nf, nleaf_slots, R, !device_out, cub_bytes, b);
  if (c->sdf_arena.ensure(bytes, bytes / 4)) return -1;
  carve(c->sdf_arena.as<char>(), nf, nleaf_slots, R, !device_out, cub_bytes, b);
  float* dist = device_out ? out : b.dist;
  const float* verts = c->mesh.verts();
  const int32_t* faces = c->mesh.faces();

  // statistics: AABB (ordered ints, min words start at all-ones) and the non-finite flag
  DISN_CUDA_OK(cudaEventRecord(c->sdf_ev[0], s));
  DISN_CUDA_OK(cudaMemsetAsync(b.bits, 0xff, 3 * sizeof(uint32_t), s));     // S_LO words live in the edge bits for now
  DISN_CUDA_OK(cudaMemsetAsync(b.bits + 3, 0, 5 * sizeof(uint32_t), s));
  sdf_stats_kernel<<<grid_of(nv), SD_THREADS, 0, s>>>(verts, nv, b.bits);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaMemcpyAsync(hs, b.bits, 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  DISN_REQUIRE(hs[S_BAD] == 0, "mesh_sdf: the resident mesh has non-finite vertex coordinates");
  float lo[3], hi[3];
  for (int a = 0; a < 3; ++a) { lo[a] = unord(hs[S_LO + a]); hi[a] = unord(hs[S_HI + a]); }
  double box[6];
  if (bbox) {
    std::memcpy(box, bbox, sizeof box);
  } else {
    double ext = 0.0;
    for (int a = 0; a < 3; ++a) ext = std::max(ext, (double)hi[a] - (double)lo[a]);
    const double half = ext * expand_rate / 2.0;
    for (int a = 0; a < 3; ++a) {
      const double centre = ((double)lo[a] + (double)hi[a]) / 2.0;
      box[a] = centre - half;
      box[3 + a] = centre + half;
    }
  }
  for (int a = 0; a < 3; ++a)
    DISN_REQUIRE(std::isfinite(box[a]) && std::isfinite(box[3 + a]) && box[a] < box[3 + a],
                 "mesh_sdf: box min must be below max on every axis (a flat mesh has no automatic box)");
  if (bbox_out) std::memcpy(bbox_out, box, sizeof box);
  double maxabs = 0.0;
  for (int a = 0; a < 3; ++a) {
    axis_table(box[a], box[3 + a], R, haxes + a * R);
    maxabs = std::max({maxabs, std::fabs((double)lo[a]), std::fabs((double)hi[a]), std::fabs(box[a]), std::fabs(box[3 + a])});
  }
  DISN_CUDA_OK(cudaMemcpyAsync(b.axes, haxes, 3 * (size_t)R * sizeof(float), cudaMemcpyHostToDevice, s));

  // BVH: Morton sort (stable LSD radix sort: ties keep face order), triangles and leaves in that order, refit level by level
  float3 flo = make_float3(lo[0], lo[1], lo[2]), scale;
  float* sc = &scale.x;
  for (int a = 0; a < 3; ++a) sc[a] = hi[a] > lo[a] ? 1024.f / (hi[a] - lo[a]) : 0.f;
  sdf_morton_kernel<<<grid_of(nf), SD_THREADS, 0, s>>>(verts, faces, nf, flo, scale, b.key, b.val);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  cub::DoubleBuffer<uint32_t> keys(b.key, b.key_alt);
  cub::DoubleBuffer<int32_t> vals(b.val, b.val_alt);
  DISN_CUDA_OK(cub::DeviceRadixSort::SortPairs(b.cub_tmp, cub_bytes, keys, vals, (int)nf, 0, 30, s));
  c->launches++;      // CUB's sort counted as one launch
  sdf_leaves_kernel<<<grid_of(nleaf_slots), SD_THREADS, 0, s>>>(verts, faces, vals.Current(), nf, nleaf_slots, b.tri,
                                                                b.blo, b.bhi);
  c->launches++;
  for (int64_t level = nleaf_slots / 2; level >= 1; level /= 2) {
    sdf_refit_kernel<<<grid_of(level), SD_THREADS, 0, s>>>(level - 1, level, b.blo, b.bhi);
    c->launches++;
  }
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaEventRecord(c->sdf_ev[1], s));

  // unsigned distance
  const dim3 dgrid((R + 7) / 8, (R + 3) / 4, (R + 3) / 4);
  sdf_distance_kernel<<<dgrid, 128, 0, s>>>(b.axes, R, b.tri, nf, b.blo, b.bhi, nleaf_slots, PRUNE_ABS * maxabs, dist);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaEventRecord(c->sdf_ev[2], s));

  // blocked edges
  const size_t smem = 3 * (size_t)R * sizeof(float);
  DISN_CUDA_OK(cudaMemsetAsync(b.bits, 0, (size_t)((npts + 3) / 4) * sizeof(uint32_t), s));
  DISN_CUDA_OK(cudaMemsetAsync(b.work, 0, sizeof(unsigned long long), s));
  sdf_line_count_kernel<<<grid_of(nf), SD_THREADS, smem, s>>>(verts, faces, nf, b.axes, R, b.cnt, b.work);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  if (exclusive_scan(c, b.cnt, nf + 1, b.total32, b.scan)) return -1;
  sdf_raster_kernel<<<(unsigned)c->num_sms * 8, SD_THREADS, smem, s>>>(verts, faces, nf, b.axes, R, b.cnt, b.total32,
                                                                       b.bits);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaEventRecord(c->sdf_ev[3], s));

  // exterior flood fill and sign
  const uint8_t* bytes8 = reinterpret_cast<const uint8_t*>(b.bits);
  sdf_init_kernel<<<grid_of(npts), SD_THREADS, 0, s>>>(b.parent, npts);
  sdf_union_kernel<<<grid_of(npts), SD_THREADS, 0, s>>>(dist, sigma, R, bytes8, b.parent);
  sdf_flatten_kernel<<<grid_of(npts), SD_THREADS, 0, s>>>(b.parent, npts);
  sdf_boundary_kernel<<<grid_of(npts), SD_THREADS, 0, s>>>(dist, sigma, R, b.parent, b.bits);
  sdf_sign_kernel<<<grid_of(npts), SD_THREADS, 0, s>>>(dist, sigma, npts, b.parent, bytes8);
  c->launches += 5;
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaEventRecord(c->sdf_ev[4], s));

  if (!device_out) DISN_CUDA_OK(cudaMemcpyAsync(out, dist, (size_t)npts * sizeof(float), cudaMemcpyDeviceToHost, s));
  unsigned long long* hwork = reinterpret_cast<unsigned long long*>(hs + S_WORK);
  DISN_CUDA_OK(cudaMemcpyAsync(hwork, b.work, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  for (int i = 0; i < 4; ++i) DISN_CUDA_OK(cudaEventElapsedTime(&c->sdf_phase_ms[i], c->sdf_ev[i], c->sdf_ev[i + 1]));
  DISN_REQUIRE(*hwork <= 0xffffffffull, "mesh_sdf: " + std::to_string(*hwork) +
                                            " (face, grid line) pairs exceed the 32-bit rasterisation index");
  return 0;
}

}  // namespace disn
