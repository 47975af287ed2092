// Checkpoint score at ground-truth SDF samples -- the metrics the reference's test/test_sdf_acc.py prints
// (models/model_normalization.py:279-299, non-binary branch): the point kernel evaluates pred_sdf at the samples, then one
// reduction kernel forms, per image, the sign-agreement count and the float64 sums of the weighted L1 and of the
// real-valued L1.  Every term is formed in float32 in TF's order; the sums have a fixed order, so repeated calls are
// bitwise equal.
#include <cmath>

#include "common.cuh"

namespace disn {
namespace {

constexpr int ACC_THREADS = 512;

// One CTA per image: thread t takes samples t, t + 512, ... in order, then a fixed shared-memory tree adds the partials.
__global__ void __launch_bounds__(ACC_THREADS) sdf_acc_kernel(const float* __restrict__ pred, const float* __restrict__ val,
                                                              int64_t N, float iso, float sw, float mw,
                                                              long long* __restrict__ count, double* __restrict__ wsum,
                                                              double* __restrict__ rsum) {
  __shared__ long long s_cnt[ACC_THREADS];
  __shared__ double s_w[ACC_THREADS], s_r[ACC_THREADS];
  const int b = blockIdx.x, t = threadIdx.x;
  const float* p = pred + (int64_t)b * N;
  const float* v = val + (int64_t)b * N;
  long long cnt = 0;
  double ws = 0.0, rs = 0.0;
  for (int64_t n = t; n < N; n += ACC_THREADS) {
    const float gt = __fsub_rn(v[n], iso);                      // sdf_val - 0.003 in float32
    const float pr = p[n];
    cnt += (gt > 0.f) == (pr > 0.f);                            // tf.equal(tf.greater(gt, 0), tf.greater(pred, 0))
    // to_float(gt <= 0.01) * mask_weight + to_float(gt > 0.01)
    const float w = __fadd_rn(__fmul_rn(gt <= 0.01f ? 1.f : 0.f, mw), gt > 0.01f ? 1.f : 0.f);
    ws += (double)__fmul_rn(fabsf(__fsub_rn(__fmul_rn(gt, sw), pr)), w);   // |gt * sdf_weight - pred| * weight_mask
    rs += (double)fabsf(__fsub_rn(gt, __fdiv_rn(pr, sw)));                  // |gt - pred / sdf_weight|
  }
  s_cnt[t] = cnt; s_w[t] = ws; s_r[t] = rs;
  __syncthreads();
  for (int s = ACC_THREADS / 2; s > 0; s >>= 1) {
    if (t < s) {
      s_cnt[t] += s_cnt[t + s];
      s_w[t] += s_w[t + s];
      s_r[t] += s_r[t + s];
    }
    __syncthreads();
  }
  if (t == 0) {
    count[b] = s_cnt[0];
    wsum[b] = s_w[0];
    rsum[b] = s_r[0];
  }
}

}  // namespace
}  // namespace disn

using namespace disn;

extern "C" int disn_sdf_metrics(disn_ctx* c, const float* pts, const float* trans_mat, const float* gt, int32_t B, int64_t N,
                                float iso_offset, float sdf_weight, float mask_weight, uint32_t flags, float* pred,
                                int64_t* count, double* wsum, double* rsum) {
  DISN_REQUIRE(c && pts && trans_mat && gt && count && wsum && rsum, "null argument");
  DISN_REQUIRE(c->enc_B > 0, not_encoded(c));
  DISN_REQUIRE(B == c->enc_B, "batch differs from the encoded batch");
  DISN_REQUIRE(N >= 1, "sdf_metrics: N >= 1 samples per image");
  DISN_REQUIRE(std::isfinite(iso_offset) && std::isfinite(mask_weight) && std::isfinite(sdf_weight) && sdf_weight != 0.f,
               "sdf_metrics: iso_offset, mask_weight and a non-zero sdf_weight must be finite");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const bool dev = (flags & DISN_DEVICE_PTR) != 0;
  const size_t n = (size_t)B * N;
  PointJob job{};
  job.B = B; job.N = N; job.out_div = 1.0f;      // disn_eval_points's job: pred_sdf, not divided by sdf_weight
  const float* d_gt = gt;
  long long* d_cnt = reinterpret_cast<long long*>(count);
  double *d_w = wsum, *d_r = rsum;
  if (dev) {
    job.pts = pts; job.trans_mat = trans_mat;
    if (!pred && c->d_out.ensure(n * sizeof(float))) return -1;
    job.out_pred = pred ? pred : c->d_out.as<float>();
  } else {
    if (ensure_point_scratch(c, (int64_t)n) || c->d_gt.ensure(n * sizeof(float)) ||
        c->d_acc.ensure((size_t)B * (sizeof(long long) + 2 * sizeof(double))))
      return -1;
    DISN_CUDA_OK(cudaMemcpyAsync(c->d_pts.as<float>(), pts, n * 3 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    DISN_CUDA_OK(cudaMemcpyAsync(c->d_tm.as<float>(), trans_mat, (size_t)B * 12 * sizeof(float), cudaMemcpyHostToDevice,
                                 c->stream));
    DISN_CUDA_OK(cudaMemcpyAsync(c->d_gt.as<float>(), gt, n * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    job.pts = c->d_pts.as<float>(); job.trans_mat = c->d_tm.as<float>();
    job.out_pred = c->d_out.as<float>();
    d_gt = c->d_gt.as<float>();
    d_cnt = c->d_acc.as<long long>();
    d_w = reinterpret_cast<double*>(d_cnt + B);
    d_r = d_w + B;
  }
  if (run_point_job(c, job)) return -1;
  sdf_acc_kernel<<<B, ACC_THREADS, 0, c->stream>>>(job.out_pred, d_gt, N, iso_offset, sdf_weight, mask_weight, d_cnt, d_w,
                                                   d_r);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  if (dev) return 0;     // asynchronous: the f16f8 overflow status is reported by the next synchronising call
  DISN_CUDA_OK(cudaMemcpyAsync(count, d_cnt, (size_t)B * sizeof(long long), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(wsum, d_w, (size_t)B * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(rsum, d_r, (size_t)B * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  if (pred) DISN_CUDA_OK(cudaMemcpyAsync(pred, job.out_pred, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return check_status(c);
}
