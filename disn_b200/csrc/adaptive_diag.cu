// Diagnostics of the coarse-to-fine grid (adaptive.cu) and mesh (adaptive_mesh.cu), exported by libdisn_b200_test.so
// only: the evaluated-point mask of the last grid, the refinement and the mesh with values read from a given dense field
// instead of the network, the phase times, the mesher's buffer bytes and the edge ids of its vertices.
#include <cmath>

#include "../../include/disn_b200_test.h"
#include "adaptive_common.cuh"
#include "common.cuh"

using namespace disn;

extern "C" {

int disn_adaptive_mask(disn_ctx* c, int64_t first, int64_t n, uint8_t* out) {
  DISN_REQUIRE(c && (out || n == 0), "null argument");
  DISN_REQUIRE(c->ad_R > 0, "adaptive_mask: no coarse-to-fine grid has been computed");
  DISN_REQUIRE(first >= 0 && n >= 0 && first + n <= (int64_t)c->ad_R * c->ad_R * c->ad_R,
               "adaptive_mask: [first, first + n) must lie inside the last call's (sdf_res+1)^3 points");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  if (n == 0) return 0;
  DISN_CUDA_OK(cudaMemcpyAsync(out, c->ad_mark.as<uint8_t>() + first, (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

int disn_adaptive_from_field(disn_ctx* c, const float* field, int32_t sdf_res, const double* sdf_params, float iso,
                             double band, uint32_t flags, float** grid_dev, int64_t* level_counts, int32_t* n_levels) {
  DISN_REQUIRE(c && field && sdf_params && grid_dev && level_counts && n_levels, "null argument");
  DISN_REQUIRE(sdf_res >= 1 && (int64_t)(sdf_res + 1) * (sdf_res + 1) * (sdf_res + 1) <= INT32_MAX,
               "adaptive_from_field: 1 <= sdf_res and (sdf_res+1)^3 < 2^31");
  DISN_REQUIRE(std::isfinite(iso), "adaptive_from_field: iso must be finite");
  DISN_REQUIRE(!std::isnan(band) && band >= 0.0, "adaptive_from_field: band must be >= 0");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const int64_t n = (int64_t)(sdf_res + 1) * (sdf_res + 1) * (sdf_res + 1);
  const float* d = field;
  if (!(flags & DISN_DEVICE_PTR)) {
    if (c->ad_field.ensure((size_t)n * sizeof(float))) return -1;
    DISN_CUDA_OK(cudaMemcpyAsync(c->ad_field.as<float>(), field, (size_t)n * sizeof(float), cudaMemcpyHostToDevice,
                                 c->stream));
    d = c->ad_field.as<float>();
  }
  if (adaptive_run(c, d, 0, nullptr, sdf_res, sdf_params, iso, band, level_counts, n_levels)) return -1;
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  *grid_dev = c->ad_grid.as<float>();
  return 0;
}

int disn_adaptive_phase_ms(disn_ctx* c, float* ms, int32_t* n) {
  DISN_REQUIRE(c && ms && n, "null argument");
  DISN_REQUIRE(c->ad_R > 0, "adaptive_phase_ms: no coarse-to-fine grid has been computed");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const int k = c->ad_levels == 0 ? 1 : c->ad_levels + 2;    // coarse (or dense), each level, fill
  for (int i = 0; i < k; ++i) DISN_CUDA_OK(cudaEventElapsedTime(&ms[i], c->ad_ev[i], c->ad_ev[i + 1]));
  *n = k;
  return 0;
}

int disn_mesh_adaptive_from_field(disn_ctx* c, const float* field, int32_t sdf_res, const double* sdf_params, float iso,
                                  double band, uint32_t flags, int64_t* level_counts, int32_t* n_levels, int64_t* n_verts,
                                  int64_t* n_faces) {
  DISN_REQUIRE(c && field && sdf_params && level_counts && n_levels, "null argument");
  DISN_REQUIRE(sdf_res >= 1 && (int64_t)(sdf_res + 1) * (sdf_res + 1) * (sdf_res + 1) <= INT32_MAX,
               "mesh_adaptive_from_field: 1 <= sdf_res and (sdf_res+1)^3 < 2^31");
  DISN_REQUIRE(coarse_stride(sdf_res) > 1, "mesh_adaptive_from_field: sdf_res must be even (s0 >= 2)");
  DISN_REQUIRE(std::isfinite(iso), "mesh_adaptive_from_field: iso must be finite");
  DISN_REQUIRE(!std::isnan(band) && band >= 0.0, "mesh_adaptive_from_field: band must be >= 0");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const int64_t n = (int64_t)(sdf_res + 1) * (sdf_res + 1) * (sdf_res + 1);
  const float* d = field;
  if (!(flags & DISN_DEVICE_PTR)) {
    if (c->ad_field.ensure((size_t)n * sizeof(float))) return -1;
    DISN_CUDA_OK(cudaMemcpyAsync(c->ad_field.as<float>(), field, (size_t)n * sizeof(float), cudaMemcpyHostToDevice,
                                 c->stream));
    d = c->ad_field.as<float>();
  }
  const int rc = adaptive_mesh_run(c, d, 0, nullptr, sdf_res, sdf_params, iso, band, level_counts, n_levels, nullptr,
                                   nullptr);
  return finish_mesh_call(c, rc, n_verts, n_faces);
}

int disn_mesh_adaptive_phase_ms(disn_ctx* c, float* ms) {
  DISN_REQUIRE(c && ms, "null argument");
  DISN_REQUIRE(c->am_nv >= 0, "mesh_adaptive_phase_ms: no coarse-to-fine mesh has been computed");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  for (int i = 0; i < 3; ++i) DISN_CUDA_OK(cudaEventElapsedTime(&ms[i], c->am_ev[i], c->am_ev[i + 1]));
  return 0;
}

int disn_mesh_adaptive_bytes(disn_ctx* c, int64_t* bytes) {
  DISN_REQUIRE(c && bytes, "null argument");
  *bytes = (int64_t)adaptive_mesh_bytes(c);
  return 0;
}

int disn_mesh_adaptive_edges(disn_ctx* c, int64_t first, int64_t n, int64_t* out) {
  DISN_REQUIRE(c && (out || n == 0), "null argument");
  DISN_REQUIRE(c->am_nv >= 0, "mesh_adaptive_edges: no coarse-to-fine mesh has been computed");
  DISN_REQUIRE(first >= 0 && n >= 0 && first + n <= c->am_nv,
               "mesh_adaptive_edges: [first, first + n) must lie inside the last mesh's vertices");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  if (n == 0) return 0;
  DISN_CUDA_OK(cudaMemcpyAsync(out, c->am_edges_sorted + first, (size_t)n * sizeof(int64_t), cudaMemcpyDeviceToHost,
                               c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

}  // extern "C"
