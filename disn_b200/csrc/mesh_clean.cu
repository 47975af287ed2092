// Small-part removal on the resident mesh: the reference's postprocessing/clean_smallparts.py:38-54
// (pymesh.separate_mesh + keep rule + pymesh.merge_meshes) on the mesh marching cubes leaves in HBM, or one uploaded with
// mesh_load.  Definitions are shared with the CPU twin oracle/mesh_clean_oracle.py, which this file reproduces bit for bit:
//   * two faces are connected when they share an undirected edge {a,b}, a != b (PyMesh's "face" connectivity);
//     components are numbered in order of their smallest face index;
//   * n_c = number of distinct vertices referenced by the faces of c;
//   * centroid = ((double)S / n_c) * 2^-32 with S the int64 sum of q = rint(v * 2^32) over those vertices (integer atomics
//     are associative, so the sums do not depend on the order the atomics land in); norm = sqrt((x*x + y*y) + z*z);
//   * keep c iff (double)n_c > (double)max n_c * num_thresh and norm < dist_thresh;
//   * the kept faces and the vertices they reference, both in their original order, faces renumbered.
// Integer and atomic work bound by HBM / L2 latency; no tensor-core work.  Built with --fmad=false.
#include <algorithm>
#include <cstring>

#include "common.cuh"

namespace disn {
namespace {

constexpr int CL_THREADS = 256;
constexpr unsigned FULL = 0xffffffffu;

// device totals: the three scan totals, the component count, max n_c, kept components, max |coordinate| bits
enum { T_NNZ = 0, T_NCOMP, T_NV_OUT, T_NF_OUT, T_MAXC, T_NKEPT, T_MAXABS, T_COUNT = 8 };

inline unsigned grid_of(int64_t n) { return (unsigned)((n + CL_THREADS - 1) / CL_THREADS); }

// corner histogram (vertex degrees) and union-find initialisation
__global__ void __launch_bounds__(CL_THREADS) clean_degree_kernel(const int32_t* __restrict__ faces, int64_t nf,
                                                                  uint32_t* __restrict__ deg, int32_t* __restrict__ parent) {
  const int64_t f = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  if (f >= nf) return;
#pragma unroll
  for (int k = 0; k < 3; ++k) atomicAdd(&deg[faces[3 * f + k]], 1u);
  parent[f] = (int32_t)f;
}

// vertex -> incident-face CSR: inc[offs[v] .. offs[v+1]) = faces with a corner at v (a face appears once per such corner)
__global__ void __launch_bounds__(CL_THREADS) clean_scatter_kernel(const int32_t* __restrict__ faces, int64_t nf,
                                                                   uint32_t* __restrict__ cursor, int32_t* __restrict__ inc) {
  const int64_t f = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  if (f >= nf) return;
#pragma unroll
  for (int k = 0; k < 3; ++k) inc[atomicAdd(&cursor[faces[3 * f + k]], 1u)] = (int32_t)f;
}

// For each non-degenerate edge (a,b) of face f: every face g > f among a's incident faces that also has a corner at b
// shares the edge {a,b} with f (any two distinct corners of a triangle are joined by one of its edges).
__global__ void __launch_bounds__(CL_THREADS) clean_union_kernel(const int32_t* __restrict__ faces, int64_t nf,
                                                                 const uint32_t* __restrict__ offs,
                                                                 const int32_t* __restrict__ inc, int32_t* parent) {
  const int64_t f = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  if (f >= nf) return;
  const int32_t v[3] = {faces[3 * f], faces[3 * f + 1], faces[3 * f + 2]};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int32_t a = v[k], b = v[(k + 1) % 3];
    if (a == b) continue;
    const uint32_t e = offs[a + 1];
    for (uint32_t i = offs[a]; i < e; ++i) {
      const int32_t g = inc[i];
      if (g <= f) continue;
      if (faces[3 * (int64_t)g] == b || faces[3 * (int64_t)g + 1] == b || faces[3 * (int64_t)g + 2] == b)
        uf_union(parent, (int32_t)f, g);
    }
  }
}

// Full path compression and root flags (rflag[nf] = 0 so the scan's total is the component count).  The walk to the root
// only reads: a pointer-jumping store from another thread could otherwise overwrite the root this thread stored.
__global__ void __launch_bounds__(CL_THREADS) clean_flatten_kernel(int32_t* parent, int64_t nf, uint32_t* __restrict__ rflag) {
  const int64_t f = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  if (f == 0) rflag[nf] = 0;
  if (f >= nf) return;
  volatile const int32_t* p = parent;
  int32_t r = (int32_t)f, n;
  while ((n = p[r]) != r) r = n;
  parent[f] = r;
  rflag[f] = (r == (int32_t)f) ? 1u : 0u;
}

// dense component number of each face (in place: parent -> label); rflag holds the exclusive scan of the root flags
__global__ void __launch_bounds__(CL_THREADS) clean_label_kernel(int32_t* __restrict__ parent, int64_t nf,
                                                                 const uint32_t* __restrict__ rflag) {
  const int64_t f = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  if (f >= nf) return;
  parent[f] = (int32_t)rflag[parent[f]];
}

__device__ __forceinline__ void add_vertex(uint32_t* cnt, unsigned long long* sums, int32_t c, uint32_t n,
                                           const long long q[3]) {
  atomicAdd(&cnt[c], n);
#pragma unroll
  for (int a = 0; a < 3; ++a) atomicAdd(&sums[3 * (int64_t)c + a], (unsigned long long)q[a]);
}

// Per vertex: +1 count and +q sums for every distinct component among its incident faces, and max |coordinate| over all
// vertices (the int64 range guard).  Nearly every vertex lies in one component and neighbouring vertices share it, so
// the contribution of each vertex's first component is summed over the warp when all its lanes agree: one atomic per
// warp instead of one per vertex on the few addresses of the large components.  Further components of a vertex (a
// vertex where parts touch) are found by a scan of its earlier incident faces.  Every lane reaches the warp collectives.
__global__ void __launch_bounds__(CL_THREADS) clean_vertex_kernel(const float* __restrict__ verts, int64_t nv,
                                                                  const uint32_t* __restrict__ offs,
                                                                  const int32_t* __restrict__ inc,
                                                                  const int32_t* __restrict__ label, uint32_t* cnt,
                                                                  unsigned long long* sums, uint32_t* totals) {
  const int64_t v = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  const int lane = threadIdx.x & 31;
  uint32_t b = 0, e = 0, abits = 0;
  long long q[3] = {0, 0, 0};
  if (v < nv) {
    b = offs[v];
    e = offs[v + 1];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float x = verts[3 * v + a];
      abits = max(abits, __float_as_uint(x) & 0x7fffffffu);     // NaN sorts above +inf and fails the guard
      q[a] = __double2ll_rn(__dmul_rn((double)x, 4294967296.0));  // exact: 24-bit significand times 2^32
    }
  }
  const uint32_t wmax = __reduce_max_sync(FULL, abits);
  if (lane == 0 && wmax) atomicMax(&totals[T_MAXABS], wmax);

  const bool valid = e > b;
  const int32_t c0 = valid ? label[inc[b]] : -1;
  const unsigned vmask = __ballot_sync(FULL, valid);
  const unsigned grp = __match_any_sync(FULL, c0);
  if (__any_sync(FULL, valid && grp == vmask)) {      // every valid lane has the same first component
    long long s[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      s[a] = valid ? q[a] : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s[a] += __shfl_xor_sync(FULL, s[a], o);
    }
    if (lane == __ffs(vmask) - 1) add_vertex(cnt, sums, c0, (uint32_t)__popc(vmask), s);
  } else if (valid) {
    add_vertex(cnt, sums, c0, 1u, q);
  }
  if (!valid) return;
  for (uint32_t i = b + 1; i < e; ++i) {
    const int32_t ci = label[inc[i]];
    if (ci == c0) continue;
    bool seen = false;
    for (uint32_t j = b + 1; j < i && !seen; ++j) seen = label[inc[j]] == ci;
    if (!seen) add_vertex(cnt, sums, ci, 1u, q);
  }
}

__global__ void __launch_bounds__(CL_THREADS) clean_maxcount_kernel(const uint32_t* __restrict__ cnt, int64_t cap,
                                                                    uint32_t* totals) {
  const int64_t c = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  const uint32_t m = (c < cap && c < (int64_t)totals[T_NCOMP]) ? cnt[c] : 0u;
  const uint32_t w = __reduce_max_sync(FULL, m);
  if ((threadIdx.x & 31) == 0 && w) atomicMax(&totals[T_MAXC], w);
}

// keep rule, float64 with one rounding per operation (the oracle's numpy arithmetic)
__global__ void __launch_bounds__(CL_THREADS) clean_keep_kernel(const uint32_t* __restrict__ cnt,
                                                                const unsigned long long* __restrict__ sums, int64_t cap,
                                                                double dist_thresh, double num_thresh,
                                                                uint8_t* __restrict__ keep, uint32_t* totals) {
  const int64_t c = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  bool k = false;
  if (c < cap && c < (int64_t)totals[T_NCOMP]) {
    const double n = (double)cnt[c];
    double sq = 0.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double x = __dmul_rn(__ddiv_rn(__ll2double_rn((long long)sums[3 * c + a]), n), 0x1p-32);
      sq = __dadd_rn(sq, __dmul_rn(x, x));
    }
    k = n > __dmul_rn((double)totals[T_MAXC], num_thresh) && __dsqrt_rn(sq) < dist_thresh;
    keep[c] = k ? 1 : 0;
  }
  const unsigned kb = __ballot_sync(FULL, k);
  if ((threadIdx.x & 31) == 0 && kb) atomicAdd(&totals[T_NKEPT], (uint32_t)__popc(kb));
}

// face keep flags and vertex keep flags (vflag was zeroed; concurrent stores of 1 are benign)
__global__ void __launch_bounds__(CL_THREADS) clean_flags_kernel(const int32_t* __restrict__ faces, int64_t nf,
                                                                 const int32_t* __restrict__ label,
                                                                 const uint8_t* __restrict__ keep,
                                                                 uint32_t* __restrict__ fflag, uint32_t* vflag) {
  const int64_t f = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  if (f == 0) fflag[nf] = 0;
  if (f >= nf) return;
  const uint32_t k = keep[label[f]];
  fflag[f] = k;
  if (k) {
#pragma unroll
    for (int j = 0; j < 3; ++j) vflag[faces[3 * f + j]] = 1u;
  }
}

// stable compaction: vmap / fmap are the exclusive scans of the keep flags (n + 1 entries, flag = next - this)
__global__ void __launch_bounds__(CL_THREADS) clean_compact_verts_kernel(const float* __restrict__ verts, int64_t nv,
                                                                         const uint32_t* __restrict__ vmap,
                                                                         float* __restrict__ out) {
  const int64_t v = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  if (v >= nv) return;
  const uint32_t o = vmap[v];
  if (vmap[v + 1] == o) return;
#pragma unroll
  for (int a = 0; a < 3; ++a) out[3 * (int64_t)o + a] = verts[3 * v + a];
}

__global__ void __launch_bounds__(CL_THREADS) clean_compact_faces_kernel(const int32_t* __restrict__ faces, int64_t nf,
                                                                         const uint32_t* __restrict__ fmap,
                                                                         const uint32_t* __restrict__ vmap,
                                                                         int32_t* __restrict__ out) {
  const int64_t f = (int64_t)blockIdx.x * CL_THREADS + threadIdx.x;
  if (f >= nf) return;
  const uint32_t o = fmap[f];
  if (fmap[f + 1] == o) return;
#pragma unroll
  for (int j = 0; j < 3; ++j) out[3 * (int64_t)o + j] = (int32_t)vmap[faces[3 * f + j]];
}

struct CleanBufs {
  uint32_t *offs, *cursor, *vflag, *rflag, *fflag, *cnt, *scan, *totals;
  int32_t *inc, *label;
  unsigned long long* sums;
  uint8_t* keep;
};

size_t carve(char* base, int64_t nv, int64_t nf, CleanBufs& b) {
  Arena a{base};
  b.offs = a.take<uint32_t>(nv + 1);
  b.cursor = a.take<uint32_t>(nv);
  b.vflag = a.take<uint32_t>(nv + 1);
  b.inc = a.take<int32_t>(3 * nf);
  b.label = a.take<int32_t>(nf);
  b.rflag = a.take<uint32_t>(nf + 1);
  b.fflag = a.take<uint32_t>(nf + 1);
  b.cnt = a.take<uint32_t>(nf);
  b.sums = a.take<unsigned long long>(3 * nf);
  b.keep = a.take<uint8_t>(nf);
  b.scan = a.take<uint32_t>(scan_scratch_elems(std::max(nv, nf) + 1));
  b.totals = a.take<uint32_t>(T_COUNT);
  return a.off;
}

}  // namespace

// Upload a host mesh into the resident mesh (verts [nv,3] float32, faces [nf,3] int32 0-based).
int mesh_load(disn_ctx* c, const float* verts, int64_t nv, const int32_t* faces, int64_t nf) {
  if (c->mesh.replace(nv, nf)) return -1;
  if (nv)
    DISN_CUDA_OK(cudaMemcpyAsync(c->mesh.verts(), verts, (size_t)nv * 3 * sizeof(float), cudaMemcpyHostToDevice,
                                 c->stream));
  if (nf)
    DISN_CUDA_OK(cudaMemcpyAsync(c->mesh.faces(), faces, (size_t)nf * 3 * sizeof(int32_t), cudaMemcpyHostToDevice,
                                 c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  c->mesh.commit(nv, nf);
  return 0;
}

// Clean the resident mesh in place.  Degree histogram -> scan -> CSR scatter -> union-find -> flatten -> scan of the root
// flags -> labels -> per-vertex reductions -> max count -> keep flags -> face / vertex flags -> two scans -> compaction into
// the spare buffers, which then become the resident mesh.  Stream-ordered with one host synchronisation at the end (the
// totals); component arrays are sized by the face count, an upper bound on the component count.  A mesh failing the
// int64 range guard is refused after that synchronisation and stays resident unchanged.
int mesh_clean(disn_ctx* c, double dist_thresh, double num_thresh, int32_t* face_component, int64_t* n_components,
               int64_t* n_kept, int64_t* n_verts, int64_t* n_faces) {
  const int64_t nv = c->mesh.nv(), nf = c->mesh.nf();
  DISN_REQUIRE(nv < ((int64_t)1 << 31) && 3 * nf < ((int64_t)1 << 31), "mesh too large for 32-bit indices");
  auto out = [&](int64_t comps, int64_t kept) {
    if (n_components) *n_components = comps;
    if (n_kept) *n_kept = kept;
    if (n_verts) *n_verts = c->mesh.nv();
    if (n_faces) *n_faces = c->mesh.nf();
  };
  if (nf == 0) {          // no faces: nothing references a vertex, the cleaned mesh is empty
    c->mesh.clear();
    out(0, 0);
    return 0;
  }
  CleanBufs b;
  const size_t bytes = carve(nullptr, nv, nf, b);
  if (c->cl_arena.ensure(bytes, bytes / 4) || c->cl_totals_host.ensure(T_COUNT * sizeof(uint32_t)) ||
      c->mesh.reserve_spare(nv, nf))
    return -1;
  carve(c->cl_arena.as<char>(), nv, nf, b);

  cudaStream_t s = c->stream;
  const float* verts = c->mesh.verts();
  const int32_t* faces = c->mesh.faces();
  uint32_t* T = b.totals;
  DISN_CUDA_OK(cudaMemsetAsync(b.offs, 0, (size_t)(nv + 1) * sizeof(uint32_t), s));
  DISN_CUDA_OK(cudaMemsetAsync(b.vflag, 0, (size_t)(nv + 1) * sizeof(uint32_t), s));
  DISN_CUDA_OK(cudaMemsetAsync(b.cnt, 0, (size_t)nf * sizeof(uint32_t), s));
  DISN_CUDA_OK(cudaMemsetAsync(b.sums, 0, (size_t)nf * 3 * sizeof(unsigned long long), s));
  DISN_CUDA_OK(cudaMemsetAsync(T, 0, T_COUNT * sizeof(uint32_t), s));

  clean_degree_kernel<<<grid_of(nf), CL_THREADS, 0, s>>>(faces, nf, b.offs, b.label);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  if (exclusive_scan(c, b.offs, nv + 1, T + T_NNZ, b.scan)) return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(b.cursor, b.offs, (size_t)nv * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  clean_scatter_kernel<<<grid_of(nf), CL_THREADS, 0, s>>>(faces, nf, b.cursor, b.inc);
  clean_union_kernel<<<grid_of(nf), CL_THREADS, 0, s>>>(faces, nf, b.offs, b.inc, b.label);
  clean_flatten_kernel<<<grid_of(nf), CL_THREADS, 0, s>>>(b.label, nf, b.rflag);
  c->launches += 3;
  DISN_CUDA_OK(cudaGetLastError());
  if (exclusive_scan(c, b.rflag, nf + 1, T + T_NCOMP, b.scan)) return -1;
  clean_label_kernel<<<grid_of(nf), CL_THREADS, 0, s>>>(b.label, nf, b.rflag);
  clean_vertex_kernel<<<grid_of(nv), CL_THREADS, 0, s>>>(verts, nv, b.offs, b.inc, b.label, b.cnt, b.sums, T);
  clean_maxcount_kernel<<<grid_of(nf), CL_THREADS, 0, s>>>(b.cnt, nf, T);
  clean_keep_kernel<<<grid_of(nf), CL_THREADS, 0, s>>>(b.cnt, b.sums, nf, dist_thresh, num_thresh, b.keep, T);
  clean_flags_kernel<<<grid_of(nf), CL_THREADS, 0, s>>>(faces, nf, b.label, b.keep, b.fflag, b.vflag);
  c->launches += 5;
  DISN_CUDA_OK(cudaGetLastError());
  if (exclusive_scan(c, b.fflag, nf + 1, T + T_NF_OUT, b.scan)) return -1;
  if (exclusive_scan(c, b.vflag, nv + 1, T + T_NV_OUT, b.scan)) return -1;
  clean_compact_verts_kernel<<<grid_of(nv), CL_THREADS, 0, s>>>(verts, nv, b.vflag, c->mesh.spare_verts());
  clean_compact_faces_kernel<<<grid_of(nf), CL_THREADS, 0, s>>>(faces, nf, b.fflag, b.vflag, c->mesh.spare_faces());
  c->launches += 2;
  DISN_CUDA_OK(cudaGetLastError());
  if (face_component)
    DISN_CUDA_OK(cudaMemcpyAsync(face_component, b.label, (size_t)nf * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  uint32_t* h = c->cl_totals_host.as<uint32_t>();
  DISN_CUDA_OK(cudaMemcpyAsync(h, T, T_COUNT * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  DISN_CUDA_OK(cudaStreamSynchronize(s));

  float maxabs_f;
  std::memcpy(&maxabs_f, &h[T_MAXABS], sizeof(float));
  const double maxabs = (double)maxabs_f;
  DISN_REQUIRE(maxabs * (double)nv < 1073741824.0,
               "mesh_clean: max |coordinate| * n_verts = " + std::to_string(maxabs * (double)nv) +
                   " must stay below 2^30 (int64 fixed-point centroid sums)");
  c->mesh.swap_spare(h[T_NV_OUT], h[T_NF_OUT]);
  out(h[T_NCOMP], h[T_NKEPT]);
  return 0;
}

}  // namespace disn
