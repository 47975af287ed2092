// Point samples of a signed distance field in HBM: the reference's sample_sdf (preprocessing/create_point_sdf_grid.py:
// 74-113) and the strided sample_sdf of create_point_sdf_fullgrid.py:70-96.  Definitions (DESIGN.md §4.8), shared with the
// numpy twins in oracle/mesh_norm_oracle.py and equal to the host sample_sdf bit for bit:
//   * dis = float32(sdf - iso) (iso as float32); band b holds the flat indices with lo_b <= dis < hi_b, the edges as float32
//     (numpy 2 casts the Python-float thresholds to float32 before comparing);
//   * each band's indices are compacted stably in ascending order (np.argwhere's order) with the library's uint32 scan;
//   * the host draws the choices with np.random.randint; row j of the gather is (X[i % R], Y[i / R % R], Z[i / R^2],
//     sdf[i]) for i = band_b[choice_j], with the float32 axis tables the host function builds;
//   * strided: out[zi][yi][xi] = sdf[zi*reduce][yi*reduce][xi*reduce], (R-1)/reduce + 1 points per axis.
// Bandwidth-bound streaming passes over the field; no tensor-core work.
#include <algorithm>
#include <string>

#include "common.cuh"

namespace disn {
namespace {

constexpr int SS_THREADS = 256;

inline unsigned grid_of(int64_t n) { return (unsigned)((n + SS_THREADS - 1) / SS_THREADS); }

// flag[i] = lo <= float32(sdf[i] - iso) < hi; flag[n] = 0 so the exclusive scan ends in the band's count
__global__ void __launch_bounds__(SS_THREADS) band_flag_kernel(const float* __restrict__ sdf, int64_t n, float iso,
                                                               float lo, float hi, uint32_t* __restrict__ flag) {
  const int64_t i = (int64_t)blockIdx.x * SS_THREADS + threadIdx.x;
  if (i == n) flag[n] = 0;
  if (i >= n) return;
  const float d = __fsub_rn(sdf[i], iso);
  flag[i] = (d >= lo && d < hi) ? 1u : 0u;
}

// band b's list starts after the lists of bands 0..b-1 (their counts are on the device)
__global__ void __launch_bounds__(SS_THREADS) band_scatter_kernel(const uint32_t* __restrict__ scan, int64_t n,
                                                                  const uint32_t* __restrict__ counts, int b,
                                                                  uint32_t* __restrict__ list) {
  const int64_t i = (int64_t)blockIdx.x * SS_THREADS + threadIdx.x;
  if (i >= n) return;
  const uint32_t o = scan[i];
  if (scan[i + 1] == o) return;
  uint64_t base = 0;
  for (int k = 0; k < b; ++k) base += counts[k];
  if (base + o < (uint64_t)n) list[base + o] = (uint32_t)i;     // disjoint bands (checked on the host) always fit
}

struct BandGather {
  int64_t kstart[5];      // row offsets of the four bands' choices
  uint32_t lstart[4];     // list offsets of the four bands
};

__global__ void __launch_bounds__(SS_THREADS) band_gather_kernel(const float* __restrict__ sdf, int R,
                                                                 const float* __restrict__ axes,
                                                                 const uint32_t* __restrict__ list,
                                                                 const int64_t* __restrict__ choice, BandGather g,
                                                                 float* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * SS_THREADS + threadIdx.x;
  if (j >= g.kstart[4]) return;
  uint32_t l0 = g.lstart[0];           // list offset of j's band (unrolled: no local-memory indexing of the parameter)
#pragma unroll
  for (int b = 1; b < 4; ++b)
    if (j >= g.kstart[b]) l0 = g.lstart[b];
  const uint32_t i = list[l0 + (uint32_t)choice[j]];
  const uint32_t x = i % (uint32_t)R, y = (i / (uint32_t)R) % (uint32_t)R, z = i / ((uint32_t)R * (uint32_t)R);
  out[4 * j] = axes[x];
  out[4 * j + 1] = axes[R + y];
  out[4 * j + 2] = axes[2 * R + z];
  out[4 * j + 3] = sdf[i];
}

__global__ void __launch_bounds__(SS_THREADS) strided_kernel(const float* __restrict__ sdf, int R, int reduce, int M,
                                                             float* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * SS_THREADS + threadIdx.x;
  if (j >= (int64_t)M * M * M) return;
  const int64_t xi = j % M, yi = (j / M) % M, zi = j / ((int64_t)M * M);
  out[j] = sdf[((zi * reduce) * R + yi * reduce) * R + xi * reduce];
}

const float* field_input(disn_ctx* c, const float* sdf, int64_t n, bool device_ptr) {
  if (device_ptr) return sdf;
  if (c->smp_in.ensure((size_t)n * sizeof(float))) return nullptr;
  if (cudaMemcpyAsync(c->smp_in.as<float>(), sdf, (size_t)n * sizeof(float), cudaMemcpyHostToDevice, c->stream) !=
      cudaSuccess) {
    set_error("sdf_sample: upload of the host field failed");
    return nullptr;
  }
  return c->smp_in.as<float>();
}

}  // namespace

// Four flag -> scan -> scatter passes, one host synchronisation (the counts).  The lists, the field address and R stay in
// the context for band_gather.
int band_count(disn_ctx* c, const float* sdf, int32_t R, float iso, const float* edges, bool device_ptr, int64_t* counts) {
  const int64_t n = (int64_t)R * R * R;
  c->smp_R = 0;
  const float* d = field_input(c, sdf, n, device_ptr);
  if (!d) return -1;
  if (c->smp_flag.ensure((size_t)(n + 1) * sizeof(uint32_t)) ||
      c->smp_scan.ensure((size_t)scan_scratch_elems(n + 1) * sizeof(uint32_t)) ||
      c->smp_list.ensure((size_t)n * sizeof(uint32_t)) || c->smp_counts.ensure(4 * sizeof(uint32_t)) ||
      c->smp_host.ensure(4 * sizeof(uint32_t)))
    return -1;
  cudaStream_t s = c->stream;
  uint32_t* flag = c->smp_flag.as<uint32_t>();
  uint32_t* cnt = c->smp_counts.as<uint32_t>();
  for (int b = 0; b < 4; ++b) {
    band_flag_kernel<<<grid_of(n + 1), SS_THREADS, 0, s>>>(d, n, iso, edges[2 * b], edges[2 * b + 1], flag);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
    if (exclusive_scan(c, flag, n + 1, cnt + b, c->smp_scan.as<uint32_t>())) return -1;
    band_scatter_kernel<<<grid_of(n), SS_THREADS, 0, s>>>(flag, n, cnt, b, c->smp_list.as<uint32_t>());
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
  }
  uint32_t* h = c->smp_host.as<uint32_t>();
  DISN_CUDA_OK(cudaMemcpyAsync(h, cnt, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  for (int b = 0; b < 4; ++b) counts[b] = c->smp_n[b] = h[b];
  c->smp_src = d;
  c->smp_R = R;
  return 0;
}

int band_gather(disn_ctx* c, const float* axes, const int64_t* choices, const int64_t* k, float* out) {
  DISN_REQUIRE(c->smp_R > 0, "sdf_band_gather: no band lists (disn_sdf_band_count first)");
  const int R = c->smp_R;
  BandGather g;
  g.kstart[0] = 0;
  uint32_t l = 0;
  for (int b = 0; b < 4; ++b) {
    DISN_REQUIRE(k[b] >= 0, "sdf_band_gather: negative sample count");
    g.kstart[b + 1] = g.kstart[b] + k[b];
    g.lstart[b] = l;
    l += (uint32_t)c->smp_n[b];
  }
  const int64_t K = g.kstart[4];
  for (int b = 0; b < 4; ++b)
    for (int64_t j = g.kstart[b]; j < g.kstart[b + 1]; ++j)
      DISN_REQUIRE(choices[j] >= 0 && choices[j] < c->smp_n[b],
                   "sdf_band_gather: choice " + std::to_string(choices[j]) + " outside band " + std::to_string(b) +
                       " of " + std::to_string(c->smp_n[b]) + " points");
  if (K == 0) return 0;
  const size_t axes_bytes = ((3 * (size_t)R * sizeof(float)) + 255) & ~(size_t)255;
  if (c->smp_gather.ensure(axes_bytes + (size_t)K * sizeof(int64_t) + (size_t)K * 4 * sizeof(float))) return -1;
  char* base = c->smp_gather.as<char>();
  float* d_axes = reinterpret_cast<float*>(base);
  int64_t* d_choice = reinterpret_cast<int64_t*>(base + axes_bytes);
  float* d_out = reinterpret_cast<float*>(d_choice + K);
  cudaStream_t s = c->stream;
  DISN_CUDA_OK(cudaMemcpyAsync(d_axes, axes, 3 * (size_t)R * sizeof(float), cudaMemcpyHostToDevice, s));
  DISN_CUDA_OK(cudaMemcpyAsync(d_choice, choices, (size_t)K * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  band_gather_kernel<<<grid_of(K), SS_THREADS, 0, s>>>(c->smp_src, R, d_axes, c->smp_list.as<uint32_t>(), d_choice, g,
                                                       d_out);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaMemcpyAsync(out, d_out, (size_t)K * 4 * sizeof(float), cudaMemcpyDeviceToHost, s));
  DISN_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

int sdf_strided(disn_ctx* c, const float* sdf, int32_t R, int32_t reduce, bool device_ptr, float* out) {
  const int64_t n = (int64_t)R * R * R;
  const int M = (R - 1) / reduce + 1;
  const int64_t m = (int64_t)M * M * M;
  if (!device_ptr) c->smp_R = 0;       // the staging buffer the band lists may point at is about to change
  const float* d = field_input(c, sdf, n, device_ptr);
  if (!d) return -1;
  if (c->smp_gather.ensure((size_t)m * sizeof(float))) return -1;
  strided_kernel<<<grid_of(m), SS_THREADS, 0, c->stream>>>(d, R, reduce, M, c->smp_gather.as<float>());
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaMemcpyAsync(out, c->smp_gather.as<float>(), (size_t)m * sizeof(float), cudaMemcpyDeviceToHost,
                               c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

}  // namespace disn
