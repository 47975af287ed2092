// Surface-sample normalisation of the resident mesh: the reference's get_normalize_mesh
// (preprocessing/create_point_sdf_grid.py:169-198: trimesh.sample.sample_surface per part, centroid and max distance of
// the samples, (v - c) / m).  Definitions are shared with the CPU twin oracle/mesh_norm_oracle.py, which this file
// reproduces bit for bit (DESIGN.md §4.8):
//   * a_f = 0.5 * sqrt((cx*cx + cy*cy) + cz*cz), c = (v1 - v0) x (v2 - v0) in float64 on the widened float32 vertices;
//   * Q_f = rint(a_f * 2^s) in int64, s = 62 - e with a_max * n_faces = m * 2^e, m in [0.5, 1) (s = 0 when a_max = 0):
//     no part total reaches 2^63; faces are scanned in part order (stable), part totals Q_p are exact integer sums;
//   * sample j of part p with draws (u, r1, r2): k = floor(u * 2^53), t = floor(k * Q_p / 2^53) (128-bit product), the face
//     of p with cum_excl <= t < cum_incl (a zero-area face is never picked); if r1 + r2 > 1 both drop by 1, then |.|;
//     point = (e1 * r1 + e2 * r2) + v0 per coordinate, e1 = v1 - v0, e2 = v2 - v0, float64;
//   * centroid = ((double)S / N) * 2^-32, S = int64 sum of rint(p * 2^32) (order-free integer atomics);
//     m = max sqrt((dx*dx + dy*dy) + dz*dz), d = p - centroid (integer atomicMax on the bits of a non-negative double);
//   * vertices become float32(((double)v - c) / m); faces do not change.
// Integer / fp64 work on a few MB: nothing for the tensor cores.  Built with --fmad=false.
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"

namespace disn {
namespace {

constexpr int NM_THREADS = 256;
constexpr double TWO53 = 9007199254740992.0;

// statistics words (unsigned long long): non-finite flag, max face area bits, fixed-point sums x3, max |p| bits, m bits
enum { W_BAD = 0, W_AMAX, W_SUM, W_MAXABS = W_SUM + 3, W_M, W_COUNT };

inline unsigned grid_of(int64_t n) { return (unsigned)((n + NM_THREADS - 1) / NM_THREADS); }

__device__ __forceinline__ double face_area(const float* __restrict__ verts, const int32_t* __restrict__ faces, int64_t f) {
  double v[3][3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int a = 0; a < 3; ++a) v[k][a] = (double)verts[3 * (int64_t)faces[3 * f + k] + a];
  const double e1[3] = {v[1][0] - v[0][0], v[1][1] - v[0][1], v[1][2] - v[0][2]};
  const double e2[3] = {v[2][0] - v[0][0], v[2][1] - v[0][1], v[2][2] - v[0][2]};
  const double cx = e1[1] * e2[2] - e1[2] * e2[1];
  const double cy = e1[2] * e2[0] - e1[0] * e2[2];
  const double cz = e1[0] * e2[1] - e1[1] * e2[0];
  return 0.5 * sqrt((cx * cx + cy * cy) + cz * cz);
}

__device__ __forceinline__ void max_bits(unsigned long long* w, double x) {   // x >= 0: bits order like values
  atomicMax(w, (unsigned long long)__double_as_longlong(x));
}

__global__ void __launch_bounds__(NM_THREADS) nm_check_kernel(const float* __restrict__ verts, int64_t nv,
                                                              unsigned long long* stats) {
  const int64_t i = (int64_t)blockIdx.x * NM_THREADS + threadIdx.x;
  if (i < 3 * nv && !isfinite(verts[i])) atomicOr(&stats[W_BAD], 1ull);
}

__global__ void __launch_bounds__(NM_THREADS) nm_area_max_kernel(const float* __restrict__ verts,
                                                                 const int32_t* __restrict__ faces, int64_t nf,
                                                                 unsigned long long* stats) {
  const int64_t f = (int64_t)blockIdx.x * NM_THREADS + threadIdx.x;
  if (f < nf) max_bits(&stats[W_AMAX], face_area(verts, faces, f));
}

// q[i] = rint(a * 2^s) of the i-th face in part order (order = nullptr: face order)
__global__ void __launch_bounds__(NM_THREADS) nm_quant_kernel(const float* __restrict__ verts,
                                                              const int32_t* __restrict__ faces,
                                                              const int32_t* __restrict__ order, int64_t nf, int s,
                                                              long long* __restrict__ q) {
  const int64_t i = (int64_t)blockIdx.x * NM_THREADS + threadIdx.x;
  if (i >= nf) return;
  q[i] = __double2ll_rn(ldexp(face_area(verts, faces, order ? order[i] : i), s));
}

__device__ __forceinline__ long long part_base(const long long* incl, int32_t start) {
  return start > 0 ? incl[start - 1] : 0ll;
}

__global__ void nm_part_total_kernel(const long long* __restrict__ incl, const int32_t* __restrict__ part_start, int P,
                                     long long* __restrict__ part_q) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int32_t b = part_start[p], e = part_start[p + 1];
  part_q[p] = e > b ? incl[e - 1] - part_base(incl, b) : 0ll;
}

// one thread per sample: part by binary search over the sample offsets, face by binary search over the part's scan
__global__ void __launch_bounds__(NM_THREADS) nm_sample_kernel(const float* __restrict__ verts,
                                                               const int32_t* __restrict__ faces,
                                                               const int32_t* __restrict__ order,
                                                               const long long* __restrict__ incl,
                                                               const int32_t* __restrict__ part_start,
                                                               const long long* __restrict__ sample_start,
                                                               const long long* __restrict__ part_q, int P,
                                                               const double* __restrict__ draws, int64_t N,
                                                               double* __restrict__ samples, unsigned long long* stats) {
  const int64_t j = (int64_t)blockIdx.x * NM_THREADS + threadIdx.x;
  if (j >= N) return;
  int lo = 0, hi = P - 1;                         // last part with sample_start[p] <= j
  while (lo < hi) { const int m = (lo + hi + 1) >> 1; if (sample_start[m] <= j) lo = m; else hi = m - 1; }
  const int p = lo;
  const unsigned long long k = (unsigned long long)(draws[3 * j] * TWO53);
  const unsigned long long Q = (unsigned long long)part_q[p];
  const unsigned long long t = (__umul64hi(k, Q) << 11) | ((k * Q) >> 53);
  const int32_t b = part_start[p];
  const long long T = part_base(incl, b) + (long long)t;
  int64_t l = b, h = part_start[p + 1] - 1;       // first i with incl[i] > T
  while (l < h) { const int64_t m = (l + h) >> 1; if (incl[m] > T) h = m; else l = m + 1; }
  const int64_t f = order ? order[l] : l;
  double v[3][3];
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int a = 0; a < 3; ++a) v[c][a] = (double)verts[3 * (int64_t)faces[3 * f + c] + a];
  double r1 = draws[3 * j + 1], r2 = draws[3 * j + 2];
  if (r1 + r2 > 1.0) { r1 -= 1.0; r2 -= 1.0; }
  r1 = fabs(r1);
  r2 = fabs(r2);
  double amax = 0.0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double x = ((v[1][a] - v[0][a]) * r1 + (v[2][a] - v[0][a]) * r2) + v[0][a];
    samples[3 * j + a] = x;
    amax = fmax(amax, fabs(x));
    atomicAdd(&stats[W_SUM + a], (unsigned long long)__double2ll_rn(x * 4294967296.0));
  }
  max_bits(&stats[W_MAXABS], amax);
}

__device__ __forceinline__ double centroid_of(long long S, int64_t N) { return ((double)S / (double)N) * 0x1p-32; }

__global__ void __launch_bounds__(NM_THREADS) nm_radius_kernel(const double* __restrict__ samples, int64_t N,
                                                               unsigned long long* stats) {
  const int64_t j = (int64_t)blockIdx.x * NM_THREADS + threadIdx.x;
  if (j >= N) return;
  double d[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) d[a] = samples[3 * j + a] - centroid_of((long long)stats[W_SUM + a], N);
  max_bits(&stats[W_M], sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]));
}

__global__ void __launch_bounds__(NM_THREADS) nm_transform_kernel(float* verts, int64_t nv, double cx, double cy,
                                                                  double cz, double m) {
  const int64_t i = (int64_t)blockIdx.x * NM_THREADS + threadIdx.x;
  if (i >= 3 * nv) return;
  const int a = (int)(i % 3);
  const double c = a == 0 ? cx : (a == 1 ? cy : cz);
  verts[i] = (float)(((double)verts[i] - c) / m);
}

struct NormBufs {
  int32_t *order, *part_start;
  long long *q, *incl, *part_q, *sample_start;
  double *draws, *samples;
  unsigned long long* stats;
  void* cub_tmp;
};

size_t carve(char* base, int64_t nf, int P, int64_t N, size_t cub_bytes, NormBufs& b) {
  Arena a{base};
  b.stats = a.take<unsigned long long>(W_COUNT);
  b.order = a.take<int32_t>(nf);
  b.part_start = a.take<int32_t>(P + 1);
  b.q = a.take<long long>(nf);
  b.incl = a.take<long long>(nf);
  b.part_q = a.take<long long>(P);
  b.sample_start = a.take<long long>(P + 1);
  b.draws = a.take<double>(3 * N);
  b.samples = a.take<double>(3 * N);
  b.cub_tmp = a.take<char>(cub_bytes);
  return a.off;
}

// Shared by both entry points: checks, the area scan in part order and the part totals (on the device in b.part_q).
// Host outputs: the statistics words after the first synchronisation and the shift s.
int part_scan(disn_ctx* c, const int32_t* part_ids, int32_t P, int64_t N, NormBufs& b, int* shift) {
  const int64_t nv = c->mesh.nv(), nf = c->mesh.nf();
  DISN_REQUIRE(nf > 0, "mesh_normalize: no resident mesh with faces (disn_mesh_load / disn_mc_run first)");
  DISN_REQUIRE(nv < ((int64_t)1 << 31) && 3 * nf < ((int64_t)1 << 31), "mesh too large for 32-bit indices");
  DISN_REQUIRE(P >= 1 && P <= nf && (part_ids || P == 1),
               "mesh_normalize: 1 <= n_parts <= n_faces (part_ids may be NULL only for one part)");
  // stable counting sort of the faces by part (host: the ids come from the host)
  std::vector<int32_t> start(P + 1, 0), order;
  if (part_ids) {
    for (int64_t f = 0; f < nf; ++f) {
      const int32_t p = part_ids[f];
      DISN_REQUIRE(p >= 0 && p < P, "mesh_normalize: face " + std::to_string(f) + " has part id " + std::to_string(p) +
                                        " outside [0, " + std::to_string(P) + ")");
      start[p + 1]++;
    }
    for (int p = 0; p < P; ++p) start[p + 1] += start[p];
    order.resize(nf);
    std::vector<int32_t> cur(start.begin(), start.end() - 1);
    for (int64_t f = 0; f < nf; ++f) order[cur[part_ids[f]]++] = (int32_t)f;
  } else {
    start[1] = (int32_t)nf;
  }
  size_t cub_bytes = 0;
  DISN_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, cub_bytes, (long long*)nullptr, (long long*)nullptr, (int)nf,
                                             c->stream));
  const size_t bytes = carve(nullptr, nf, P, N, cub_bytes, b);
  if (c->nm_arena.ensure(bytes, bytes / 4) || c->nm_host.ensure(W_COUNT * sizeof(unsigned long long))) return -1;
  carve(c->nm_arena.as<char>(), nf, P, N, cub_bytes, b);
  cudaStream_t s = c->stream;
  const float* verts = c->mesh.verts();
  const int32_t* faces = c->mesh.faces();
  const int32_t* d_order = part_ids ? b.order : nullptr;
  if (part_ids)
    DISN_CUDA_OK(cudaMemcpyAsync(b.order, order.data(), (size_t)nf * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  DISN_CUDA_OK(cudaMemcpyAsync(b.part_start, start.data(), (size_t)(P + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  DISN_CUDA_OK(cudaMemsetAsync(b.stats, 0, W_COUNT * sizeof(unsigned long long), s));
  nm_check_kernel<<<grid_of(3 * nv), NM_THREADS, 0, s>>>(verts, nv, b.stats);
  nm_area_max_kernel<<<grid_of(nf), NM_THREADS, 0, s>>>(verts, faces, nf, b.stats);
  c->launches += 2;
  DISN_CUDA_OK(cudaGetLastError());
  unsigned long long* hs = c->nm_host.as<unsigned long long>();
  DISN_CUDA_OK(cudaMemcpyAsync(hs, b.stats, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  DISN_REQUIRE(hs[W_BAD] == 0, "mesh_normalize: the resident mesh has non-finite vertex coordinates");
  double amax;
  std::memcpy(&amax, &hs[W_AMAX], sizeof amax);
  int e = 0;
  if (amax > 0.0) std::frexp(amax * (double)nf, &e);
  *shift = amax > 0.0 ? 62 - e : 0;
  nm_quant_kernel<<<grid_of(nf), NM_THREADS, 0, s>>>(verts, faces, d_order, nf, *shift, b.q);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cub::DeviceScan::InclusiveSum(b.cub_tmp, cub_bytes, b.q, b.incl, (int)nf, s));
  c->launches++;      // CUB's scan counted as one launch
  nm_part_total_kernel<<<(P + 127) / 128, 128, 0, s>>>(b.incl, b.part_start, P, b.part_q);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace

int mesh_part_areas(disn_ctx* c, const int32_t* part_ids, int32_t n_parts, int64_t* part_q, int32_t* shift) {
  NormBufs b;
  int s = 0;
  if (int rc = part_scan(c, part_ids, n_parts, 0, b, &s)) return rc;
  if (part_q)
    DISN_CUDA_OK(cudaMemcpyAsync(part_q, b.part_q, (size_t)n_parts * sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  if (shift) *shift = s;
  return 0;
}

int mesh_normalize(disn_ctx* c, const int32_t* part_ids, int32_t n_parts, const int64_t* amounts, const double* draws,
                   int64_t n_draws, const double* given, double* centroid_out, double* m_out, double* samples_out) {
  cudaStream_t s = c->stream;
  const int64_t nv = c->mesh.nv();
  double cen[3], m;
  if (given) {
    DISN_REQUIRE(c->mesh.nf() > 0, "mesh_normalize: no resident mesh with faces (disn_mesh_load / disn_mc_run first)");
    for (int a = 0; a < 3; ++a) cen[a] = given[a];
    m = given[3];
    DISN_REQUIRE(std::isfinite(cen[0]) && std::isfinite(cen[1]) && std::isfinite(cen[2]) && std::isfinite(m) && m > 0.0,
                 "mesh_normalize: the given centroid must be finite and m finite and > 0");
    if (c->nm_arena.ensure(W_COUNT * sizeof(unsigned long long)) || c->nm_host.ensure(sizeof(unsigned long long))) return -1;
    unsigned long long* st = c->nm_arena.as<unsigned long long>();
    DISN_CUDA_OK(cudaMemsetAsync(st, 0, sizeof(unsigned long long), s));
    nm_check_kernel<<<grid_of(3 * nv), NM_THREADS, 0, s>>>(c->mesh.verts(), nv, st);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
    unsigned long long* hs = c->nm_host.as<unsigned long long>();
    DISN_CUDA_OK(cudaMemcpyAsync(hs, st, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    DISN_CUDA_OK(cudaStreamSynchronize(s));
    DISN_REQUIRE(hs[W_BAD] == 0, "mesh_normalize: the resident mesh has non-finite vertex coordinates");
  } else {
    DISN_REQUIRE(amounts && (draws || n_draws == 0) && n_draws >= 0, "mesh_normalize: amounts and draws are required");
    // host-only checks of the caller's arrays first: nothing is sized from them before they agree
    DISN_REQUIRE(c->mesh.nf() > 0, "mesh_normalize: no resident mesh with faces (disn_mesh_load / disn_mc_run first)");
    DISN_REQUIRE(n_parts >= 1 && n_parts <= c->mesh.nf() && (part_ids || n_parts == 1),
                 "mesh_normalize: 1 <= n_parts <= n_faces (part_ids may be NULL only for one part)");
    std::vector<long long> pq(n_parts), sstart(n_parts + 1, 0);
    for (int p = 0; p < n_parts; ++p) {
      DISN_REQUIRE(amounts[p] >= 0, "mesh_normalize: amount of part " + std::to_string(p) + " is negative");
      DISN_REQUIRE(amounts[p] <= INT32_MAX, "mesh_normalize: amount of part " + std::to_string(p) + " exceeds 2^31 - 1");
      sstart[p + 1] = sstart[p] + amounts[p];
    }
    const int64_t N = sstart[n_parts];
    DISN_REQUIRE(N == n_draws, "mesh_normalize: " + std::to_string(n_draws) + " draws for " + std::to_string(N) +
                                   " samples (the sum of the amounts)");
    DISN_REQUIRE(N > 0, "mesh_normalize: no samples (zero total area or all amounts zero)");
    for (int64_t i = 0; i < 3 * N; ++i)
      DISN_REQUIRE(draws[i] >= 0.0 && draws[i] < 1.0, "mesh_normalize: draws must lie in [0, 1)");
    NormBufs b;
    int shift = 0;
    if (int rc = part_scan(c, part_ids, n_parts, N, b, &shift)) return rc;
    DISN_CUDA_OK(cudaMemcpyAsync(pq.data(), b.part_q, (size_t)n_parts * sizeof(long long), cudaMemcpyDeviceToHost, s));
    DISN_CUDA_OK(cudaStreamSynchronize(s));
    for (int p = 0; p < n_parts; ++p)
      DISN_REQUIRE(amounts[p] == 0 || pq[p] > 0,
                   "mesh_normalize: part " + std::to_string(p) + " has zero area and cannot be sampled");
    DISN_CUDA_OK(cudaMemcpyAsync(b.sample_start, sstart.data(), (size_t)(n_parts + 1) * sizeof(long long),
                                 cudaMemcpyHostToDevice, s));
    DISN_CUDA_OK(cudaMemcpyAsync(b.draws, draws, (size_t)N * 3 * sizeof(double), cudaMemcpyHostToDevice, s));
    nm_sample_kernel<<<grid_of(N), NM_THREADS, 0, s>>>(c->mesh.verts(), c->mesh.faces(),
                                                       part_ids ? b.order : nullptr, b.incl, b.part_start,
                                                       b.sample_start, b.part_q, n_parts, b.draws, N, b.samples,
                                                       b.stats);
    nm_radius_kernel<<<grid_of(N), NM_THREADS, 0, s>>>(b.samples, N, b.stats);
    c->launches += 2;
    DISN_CUDA_OK(cudaGetLastError());
    unsigned long long* hs = c->nm_host.as<unsigned long long>();
    DISN_CUDA_OK(cudaMemcpyAsync(hs, b.stats, W_COUNT * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    if (samples_out)
      DISN_CUDA_OK(cudaMemcpyAsync(samples_out, b.samples, (size_t)N * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
    DISN_CUDA_OK(cudaStreamSynchronize(s));
    double maxabs;
    std::memcpy(&maxabs, &hs[W_MAXABS], sizeof maxabs);
    std::memcpy(&m, &hs[W_M], sizeof m);
    DISN_REQUIRE(maxabs * (double)N < 1073741824.0,
                 "mesh_normalize: max |sample coordinate| * N = " + std::to_string(maxabs * (double)N) +
                     " must stay below 2^30 (int64 fixed-point centroid sums)");
    for (int a = 0; a < 3; ++a) cen[a] = ((double)(long long)hs[W_SUM + a] / (double)N) * 0x1p-32;
    DISN_REQUIRE(m > 0.0 && std::isfinite(m), "mesh_normalize: every sample lies on the centroid (m = 0)");
  }
  nm_transform_kernel<<<grid_of(3 * nv), NM_THREADS, 0, s>>>(c->mesh.verts(), nv, cen[0], cen[1], cen[2], m);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  if (centroid_out) std::memcpy(centroid_out, cen, sizeof cen);
  if (m_out) *m_out = m;
  return 0;
}

}  // namespace disn
