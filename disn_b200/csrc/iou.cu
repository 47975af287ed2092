// IoU evaluator of the reference (test/test_iou.py:208-233, `iou_pymesh`): both meshes are voxelised with
// pymesh.VoxelGrid(2/dim), the VERTICES of the resulting voxel meshes are binned with ((v + 1.1) / 2.4 * dim).astype(int)
// into dim^3 occupancy grids, IoU = |A and B| / |A or B|.
//
// PyMesh is an un-vendored third-party dependency of the reference (no version pinned; README asks for a source build) and
// cannot be loaded here, so its voxeliser is RESTATED (parity unpinned against PyMesh itself):
//   * cells are indexed by integer triples k; cell k is the cube centred at k * cell with half-size cell / 2
//     (PyMesh's HashGrid keys are round(x / cell_size));
//   * a cell is occupied iff it overlaps at least one triangle (closed separating-axis test, 13 axes);
//   * the voxel mesh's vertices are the 8 corners (k +- 1/2) * cell of every occupied cell.
// The binning is the reference's expression; bins outside [0, dim) are dropped (numpy would wrap negatives and raise on
// >= dim; ShapeNet meshes are normalised into the unit sphere so neither happens).
// Voxel window: a corner p lands in a bin iff (p + 1.1) / 2.4 * dim is in (-1, dim), i.e. p in (-1.1 - 2.4/dim, 1.3), so
// cell k can contribute only if k * cell is in (-1.1 - 2.4/dim - cell/2, 1.3 + cell/2) = (-(0.55 dim + 1.7), 0.65 dim + 0.5)
// cells.  The hashed cells are k in [-voff, vhi) with voff = floor(11 dim / 20) + 4 and vhi = floor(13 dim / 20) + 4, which
// covers that range with more than one cell to spare on each side (621^3 bits = 30 MB at dim 512); cells outside it
// are skipped, which drops nothing.  The CPU twin oracle/metrics_oracle.py:iou_voxel derives the same window
// (voxel_window) and does the same float64 operations in the same order; this file is compiled with
// --fmad=false so that the classification is identical (tests assert equal occupancy grids).
// One voxeliser serves both entry points: disn_iou_views voxelises one reference mesh and V views (test_iou.py's views of
// one object) with one launch per mesh set, face f finding its mesh by a search of the face offsets; disn_iou is V = 1.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"

namespace disn {
namespace {

// voxel index range [-voff, vhi) per axis (see the window rule above)
struct VoxWindow {
  int voff, vhi, vg;
};

VoxWindow voxel_window(int dim) {
  VoxWindow w;
  w.voff = 11 * dim / 20 + 4;
  w.vhi = 13 * dim / 20 + 4;
  w.vg = w.voff + w.vhi;
  return w;
}

__device__ __forceinline__ bool axis_sep(double ax, double ay, double az, const double v[3][3], double half) {
  const double p0 = ax * v[0][0] + ay * v[0][1] + az * v[0][2];
  const double p1 = ax * v[1][0] + ay * v[1][1] + az * v[1][2];
  const double p2 = ax * v[2][0] + ay * v[2][1] + az * v[2][2];
  const double r = half * (fabs(ax) + fabs(ay) + fabs(az));
  return fmin(p0, fmin(p1, p2)) > r || fmax(p0, fmax(p1, p2)) < -r;
}

// closed triangle / axis-aligned cube overlap (separating axes: 3 cube normals, triangle normal, 9 edge cross products)
__device__ bool tri_cube_overlap(const double c[3], double half, const double t[3][3]) {
  double v[3][3];
  for (int k = 0; k < 3; ++k)
    for (int a = 0; a < 3; ++a) v[k][a] = t[k][a] - c[a];
  for (int a = 0; a < 3; ++a) {
    if (fmin(v[0][a], fmin(v[1][a], v[2][a])) > half || fmax(v[0][a], fmax(v[1][a], v[2][a])) < -half) return false;
  }
  double e[3][3];
  for (int a = 0; a < 3; ++a) { e[0][a] = v[1][a] - v[0][a]; e[1][a] = v[2][a] - v[1][a]; e[2][a] = v[0][a] - v[2][a]; }
  const double nx = e[0][1] * e[1][2] - e[0][2] * e[1][1];
  const double ny = e[0][2] * e[1][0] - e[0][0] * e[1][2];
  const double nz = e[0][0] * e[1][1] - e[0][1] * e[1][0];
  {
    const double d = nx * v[0][0] + ny * v[0][1] + nz * v[0][2];
    const double r = half * (fabs(nx) + fabs(ny) + fabs(nz));
    if (fabs(d) > r) return false;
  }
  for (int i = 0; i < 3; ++i) {
    if (axis_sep(0.0, -e[i][2], e[i][1], v, half)) return false;     // x cross e
    if (axis_sep(e[i][2], 0.0, -e[i][0], v, half)) return false;     // y cross e
    if (axis_sep(-e[i][1], e[i][0], 0.0, v, half)) return false;     // z cross e
  }
  return true;
}

// mesh of face f in a batch whose faces are [foff[m], foff[m+1]) (largest m with foff[m] <= f)
__device__ __forceinline__ int mesh_of(const int64_t* __restrict__ foff, int M, int64_t f) {
  int lo = 0, hi = M;     // foff[lo] <= f < foff[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (foff[mid] <= f) lo = mid; else hi = mid;
  }
  return lo;
}

// M meshes in one launch: mesh m has vertices [voff[m], voff[m+1]) of verts and faces [foff[m], foff[m+1]) of faces (its
// own vertex ids); its cells go to the bitmap vox + m * vox_words
__global__ void voxelize_kernel(const float* __restrict__ verts, const int64_t* __restrict__ voff,
                                const int32_t* __restrict__ faces, const int64_t* __restrict__ foff, int M, double cell,
                                VoxWindow win, int64_t vox_words, uint32_t* __restrict__ vox) {
  const int64_t vg = win.vg, nf = foff[M];
  for (int64_t f = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; f < nf; f += (int64_t)gridDim.x * blockDim.x) {
    const int m = mesh_of(foff, M, f);
    const float* mv = verts + voff[m] * 3;
    uint32_t* mvox = vox + m * vox_words;
    double t[3][3];
    double lo[3], hi[3];
    for (int k = 0; k < 3; ++k) {
      const float* p = mv + (int64_t)faces[f * 3 + k] * 3;
      for (int a = 0; a < 3; ++a) t[k][a] = (double)p[a];
    }
    int k0[3], k1[3];
    for (int a = 0; a < 3; ++a) {
      lo[a] = fmin(t[0][a], fmin(t[1][a], t[2][a]));
      hi[a] = fmax(t[0][a], fmax(t[1][a], t[2][a]));
      // clamped to the window in double before the cast, so that far-out coordinates cannot overflow it; a triangle
      // entirely outside the window gets k1 < k0 on some axis and no cells
      k0[a] = (int)fmin(fmax(floor(lo[a] / cell - 0.5), (double)-win.voff), (double)win.vhi);
      k1[a] = (int)fmax(fmin(ceil(hi[a] / cell + 0.5), (double)(win.vhi - 1)), (double)(-win.voff - 1));
    }
    for (int kz = k0[2]; kz <= k1[2]; ++kz)
      for (int ky = k0[1]; ky <= k1[1]; ++ky)
        for (int kx = k0[0]; kx <= k1[0]; ++kx) {
          const double c[3] = {(double)kx * cell, (double)ky * cell, (double)kz * cell};
          if (!tri_cube_overlap(c, cell * 0.5, t)) continue;
          const int64_t id = ((int64_t)(kz + win.voff) * vg + (ky + win.voff)) * vg + (kx + win.voff);
          atomicOr(&mvox[id >> 5], 1u << (id & 31));
        }
  }
}

// corners of occupied cells -> ((c + 1.1) / 2.4 * dim) truncated -> occupancy bits; M bitmaps of vox_words words each
// into M grids of occ_words words each
__global__ void corners_kernel(const uint32_t* __restrict__ vox, int M, int64_t vox_words, double cell, int dim,
                               VoxWindow win, int64_t occ_words, uint32_t* __restrict__ occ) {
  const int64_t vg = win.vg, nwords = (int64_t)M * vox_words;
  for (int64_t gw = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; gw < nwords; gw += (int64_t)gridDim.x * blockDim.x) {
    uint32_t bits = vox[gw];
    if (!bits) continue;
    const int64_t m = gw / vox_words, w = gw - m * vox_words;
    uint32_t* mocc = occ + m * occ_words;
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      const int64_t id = w * 32 + b;
      const int kx = (int)(id % vg) - win.voff, ky = (int)((id / vg) % vg) - win.voff, kz = (int)(id / (vg * vg)) - win.voff;
      for (int cz = 0; cz < 2; ++cz)
        for (int cy = 0; cy < 2; ++cy)
          for (int cx = 0; cx < 2; ++cx) {
            const double p[3] = {((double)kx + (cx ? 0.5 : -0.5)) * cell, ((double)ky + (cy ? 0.5 : -0.5)) * cell,
                                 ((double)kz + (cz ? 0.5 : -0.5)) * cell};
            int ind[3];
            bool ok = true;
            for (int a = 0; a < 3; ++a) {
              const double q = (p[a] + 1.1) / 2.4 * (double)dim;
              ind[a] = (int)q;                       // astype(int): truncation toward zero
              ok = ok && ind[a] >= 0 && ind[a] < dim;   // q in (-1, 0) truncates to bin 0, exactly like numpy
            }
            if (!ok) continue;
            const int64_t o = ((int64_t)ind[0] * dim + ind[1]) * dim + ind[2];     // v[ind[:,0], ind[:,1], ind[:,2]]
            atomicOr(&mocc[o >> 5], 1u << (o & 31));
          }
    }
  }
}

// counts of ref AND / OR view v for every view: grid (x, y) = (blocks per view, views), out[2v] / out[2v+1]
__global__ void iou_count_kernel(const uint32_t* __restrict__ ref, const uint32_t* __restrict__ views, int V,
                                 int64_t nwords, unsigned long long* __restrict__ out) {
  for (int v = blockIdx.y; v < V; v += gridDim.y) {
    const uint32_t* b = views + (int64_t)v * nwords;
    unsigned long long inter = 0, uni = 0;
    for (int64_t w = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; w < nwords; w += (int64_t)gridDim.x * blockDim.x) {
      inter += __popc(ref[w] & b[w]);
      uni += __popc(ref[w] | b[w]);
    }
    for (int o = 16; o > 0; o >>= 1) {
      inter += __shfl_xor_sync(0xffffffffu, inter, o);
      uni += __shfl_xor_sync(0xffffffffu, uni, o);
    }
    if ((threadIdx.x & 31) == 0) { atomicAdd(&out[2 * v], inter); atomicAdd(&out[2 * v + 1], uni); }
  }
}

__global__ void unpack_bits_kernel(const uint32_t* __restrict__ bits, int64_t n, uint8_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (bits[i >> 5] >> (i & 31)) & 1u;
}

// The reference mesh against V views (disn_iou is V = 1).  Arguments are validated by the callers.  Scratch is per call:
// V + 1 voxel bitmaps and occupancy grids, the meshes, their offsets and the counts; the grid unpacking buffer only when a
// grid is asked for (occ_outs[m], m = 0 the reference, 1..V the views, each may be null).
int iou_views(disn_ctx* c, const float* ref_verts, int64_t ref_nv, const int32_t* ref_faces, int64_t ref_nf, int32_t V,
              const float* verts, const int64_t* vert_offsets, const int32_t* faces, const int64_t* face_offsets,
              int32_t dim, int64_t* intersection, int64_t* uni, uint8_t* const* occ_outs) {
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const VoxWindow win = voxel_window(dim);
  const int64_t vox_words = ((int64_t)win.vg * win.vg * win.vg + 31) / 32, n_occ = (int64_t)dim * dim * dim,
                occ_words = (n_occ + 31) / 32;
  const int64_t nv = vert_offsets[V], nf = face_offsets[V];
  bool want_grid = false;
  for (int m = 0; m <= V; ++m) want_grid = want_grid || occ_outs[m];
  // host image of the offsets: reference {0, nv} {0, nf}, then the views' vert_offsets and face_offsets
  std::vector<int64_t> offs(4 + 2 * ((size_t)V + 1));
  offs[0] = 0; offs[1] = ref_nv; offs[2] = 0; offs[3] = ref_nf;
  std::copy(vert_offsets, vert_offsets + V + 1, offs.begin() + 4);
  std::copy(face_offsets, face_offsets + V + 1, offs.begin() + 5 + V);
  uint32_t *vox, *occ;
  unsigned long long* cnt;
  uint8_t* unp;
  int64_t* doffs;
  float *drv, *dv;
  int32_t *drf, *df;
  auto carve = [&](char* base) {
    Arena a{base};
    vox = a.take<uint32_t>((size_t)(V + 1) * vox_words);
    occ = a.take<uint32_t>((size_t)(V + 1) * occ_words);
    cnt = a.take<unsigned long long>(2 * (size_t)V);
    unp = want_grid ? a.take<uint8_t>(n_occ) : nullptr;
    doffs = a.take<int64_t>(offs.size());
    drv = a.take<float>(3 * ref_nv);
    drf = a.take<int32_t>(3 * ref_nf);
    dv = a.take<float>(3 * nv);
    df = a.take<int32_t>(3 * nf);
    return a.off;
  };
  DevBuffer buf;     // per call, freed on every exit path
  if (buf.ensure(carve(nullptr))) return -1;
  carve(buf.as<char>());
  const double cell = 2.0 / (double)dim;                 // pymesh.VoxelGrid(2./dim)
  const int grid = c->num_sms * 8;
  cudaStream_t s = c->stream;
  DISN_CUDA_OK(cudaMemsetAsync(vox, 0, (size_t)(V + 1) * vox_words * 4, s));
  DISN_CUDA_OK(cudaMemsetAsync(occ, 0, (size_t)(V + 1) * occ_words * 4, s));
  DISN_CUDA_OK(cudaMemsetAsync(cnt, 0, 16 * (size_t)V, s));
  DISN_CUDA_OK(cudaMemcpyAsync(doffs, offs.data(), offs.size() * 8, cudaMemcpyHostToDevice, s));
  DISN_CUDA_OK(cudaMemcpyAsync(drv, ref_verts, (size_t)ref_nv * 12, cudaMemcpyHostToDevice, s));
  DISN_CUDA_OK(cudaMemcpyAsync(drf, ref_faces, (size_t)ref_nf * 12, cudaMemcpyHostToDevice, s));
  DISN_CUDA_OK(cudaMemcpyAsync(dv, verts, (size_t)nv * 12, cudaMemcpyHostToDevice, s));
  DISN_CUDA_OK(cudaMemcpyAsync(df, faces, (size_t)nf * 12, cudaMemcpyHostToDevice, s));
  // the reference mesh into slot 0, the V views into slots 1..V
  voxelize_kernel<<<grid, 128, 0, s>>>(drv, doffs, drf, doffs + 2, 1, cell, win, vox_words, vox);
  corners_kernel<<<grid, 256, 0, s>>>(vox, 1, vox_words, cell, dim, win, occ_words, occ);
  voxelize_kernel<<<grid, 128, 0, s>>>(dv, doffs + 4, df, doffs + 5 + V, V, cell, win, vox_words, vox + vox_words);
  corners_kernel<<<grid, 256, 0, s>>>(vox + vox_words, V, vox_words, cell, dim, win, occ_words, occ + occ_words);
  const dim3 cgrid((unsigned)std::max(1, grid / V), (unsigned)std::min(V, 65535));
  iou_count_kernel<<<cgrid, 256, 0, s>>>(occ, occ + occ_words, V, occ_words, cnt);
  c->launches += 5;
  DISN_CUDA_OK(cudaGetLastError());
  std::vector<unsigned long long> h(2 * (size_t)V);
  DISN_CUDA_OK(cudaMemcpyAsync(h.data(), cnt, 16 * (size_t)V, cudaMemcpyDeviceToHost, s));
  for (int m = 0; m <= V; ++m) {
    if (!occ_outs[m]) continue;
    unpack_bits_kernel<<<grid, 256, 0, s>>>(occ + m * occ_words, n_occ, unp);   // stream order keeps unp's reuse safe
    DISN_CUDA_OK(cudaMemcpyAsync(occ_outs[m], unp, (size_t)n_occ, cudaMemcpyDeviceToHost, s));
  }
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  for (int v = 0; v < V; ++v) {
    intersection[v] = (int64_t)h[2 * v];
    uni[v] = (int64_t)h[2 * v + 1];
  }
  return 0;
}

}  // namespace
}  // namespace disn

using namespace disn;

extern "C" int disn_iou(disn_ctx* c, const float* verts1, int64_t nv1, const int32_t* faces1, int64_t nf1,
                        const float* verts2, int64_t nv2, const int32_t* faces2, int64_t nf2, int32_t dim,
                        int64_t* intersection, int64_t* uni, uint8_t* occ1_out, uint8_t* occ2_out) {
  DISN_REQUIRE(c && verts1 && faces1 && verts2 && faces2 && intersection && uni, "null argument");
  DISN_REQUIRE(dim >= 2 && dim <= 512 && nv1 > 0 && nf1 > 0 && nv2 > 0 && nf2 > 0, "dim in [2,512], non-empty meshes");
  for (int m = 0; m < 2; ++m) {       // reject out-of-range vertex ids up front (device reads are unchecked)
    const int32_t* f = m ? faces2 : faces1;
    const int64_t nf = m ? nf2 : nf1, nv = m ? nv2 : nv1;
    for (int64_t i = 0; i < nf * 3; ++i) DISN_REQUIRE(f[i] >= 0 && f[i] < nv, "face index out of range");
  }
  const int64_t vo[2] = {0, nv2}, fo[2] = {0, nf2};
  uint8_t* const outs[2] = {occ1_out, occ2_out};
  return iou_views(c, verts1, nv1, faces1, nf1, 1, verts2, vo, faces2, fo, dim, intersection, uni, outs);
}

extern "C" int disn_iou_views(disn_ctx* c, const float* ref_verts, int64_t ref_nv, const int32_t* ref_faces, int64_t ref_nf,
                              int32_t V, const float* verts, const int64_t* vert_offsets, const int32_t* faces,
                              const int64_t* face_offsets, int32_t dim, int64_t* intersection, int64_t* uni,
                              uint8_t* occ_out) {
  DISN_REQUIRE(c && ref_verts && ref_faces && verts && vert_offsets && faces && face_offsets && intersection && uni,
               "null argument");
  DISN_REQUIRE(dim >= 2 && dim <= 512, "dim in [2,512]");
  DISN_REQUIRE(V >= 1, "V >= 1");
  DISN_REQUIRE(ref_nf > 0, "the reference mesh has no faces");
  for (int64_t i = 0; i < ref_nf * 3; ++i) DISN_REQUIRE(ref_faces[i] >= 0 && ref_faces[i] < ref_nv,
                                                        "reference mesh: face index out of range");
  DISN_REQUIRE(vert_offsets[0] == 0 && face_offsets[0] == 0, "vert_offsets[0] and face_offsets[0] must be 0");
  for (int32_t v = 0; v < V; ++v) {
    const std::string view = "view " + std::to_string(v) + ": ";
    DISN_REQUIRE(vert_offsets[v + 1] >= vert_offsets[v], view + "vert_offsets decrease");
    DISN_REQUIRE(face_offsets[v + 1] >= face_offsets[v], view + "face_offsets decrease");
    DISN_REQUIRE(face_offsets[v + 1] > face_offsets[v], view + "no faces");
    const int64_t nv = vert_offsets[v + 1] - vert_offsets[v];
    for (int64_t i = face_offsets[v] * 3; i < face_offsets[v + 1] * 3; ++i)
      DISN_REQUIRE(faces[i] >= 0 && faces[i] < nv, view + "face index out of range");
  }
  const int64_t n_occ = (int64_t)dim * dim * dim;
  std::vector<uint8_t*> outs((size_t)V + 1, nullptr);
  if (occ_out)
    for (int32_t m = 0; m <= V; ++m) outs[m] = occ_out + m * n_occ;
  return iou_views(c, ref_verts, ref_nv, ref_faces, ref_nf, V, verts, vert_offsets, faces, face_offsets, dim, intersection,
                   uni, outs.data());
}
