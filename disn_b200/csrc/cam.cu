// Camera-pose heads of the reference's estimated-camera path (the step that produces `trans_mat` when the drivers
// run with --cam_est: demo/demo.py:195-258, cam_est/model_cam.py:47-109, models/posenet.py:22-36,91-124).
// Input: the 1024-d VGG-16 embedding of the image (same encoder kernels as the SDF path, camera checkpoint's
// weights).  One CTA per image evaluates the three tiny fully-connected heads (utils/tf_util.py:328-362:
// y = relu(x.W + b), last layer linear), builds the rotation from the 6-D ortho representation, applies the
// predicted isotropic scale, appends the translation row and right-multiplies by K^T:
//     pred_RT[4,3] = [ (s*I).R ; t ],   pred_trans_mat[4,3] = pred_RT . K^T.
// The pose geometry rounds every product, sum, square root and quotient to float32 on its own, like TF's separate ops:
// this file is built with --fmad=false.  A contracted cross product x*y' - x'*y keeps the rounding error of one product,
// so for y_raw parallel to x_raw it yields a residual of ~3e-8 instead of TF's exact zero, which the normalisation (clamp
// 1e-8) then blows up into a unit z column pointing anywhere.  The heads' dot products use explicit fmaf (unaffected).
#include "common.cuh"

namespace disn {
namespace {

struct CamHeadWeights {
  const float *s1w, *s1b, *s2w, *s2b, *s3w, *s3b;      // scale: 1024-64-32-1
  const float *r1w, *r1b, *r2w, *r2b, *r3w, *r3b;      // ortho6d: 1024-512-256-6
  const float *t1w, *t1b, *t2w, *t2b, *t3w, *t3b;      // translation: 1024-128-64-3
};

// out[n] = act(b[n] + sum_k in[k] * W[k][n]); threads over n (coalesced rows of W)
__device__ void fc_layer(const float* in, int K, const float* __restrict__ W, const float* __restrict__ b, float* out,
                         int N, bool relu) {
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < K; ++k) acc = fmaf(in[k], W[(size_t)k * N + n], acc);
    acc += b[n];
    out[n] = relu ? fmaxf(acc, 0.f) : acc;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256) cam_heads_kernel(const float* __restrict__ emb, int emb_dim, CamHeadWeights w,
                                                        const float* __restrict__ Kmat /*[3,3]*/,
                                                        float* __restrict__ out_rt, float* __restrict__ out_tm) {
  __shared__ float x[1024], h1[512], h2[256], o_scale[1], o_rot[6], o_tr[3];
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < emb_dim; i += blockDim.x) x[i] = emb[(size_t)b * emb_dim + i];
  __syncthreads();
  fc_layer(x, emb_dim, w.s1w, w.s1b, h1, 64, true);
  fc_layer(h1, 64, w.s2w, w.s2b, h2, 32, true);
  fc_layer(h2, 32, w.s3w, w.s3b, o_scale, 1, false);
  fc_layer(x, emb_dim, w.r1w, w.r1b, h1, 512, true);
  fc_layer(h1, 512, w.r2w, w.r2b, h2, 256, true);
  fc_layer(h2, 256, w.r3w, w.r3b, o_rot, 6, false);
  fc_layer(x, emb_dim, w.t1w, w.t1b, h1, 128, true);
  fc_layer(h1, 128, w.t2w, w.t2b, h2, 64, true);
  fc_layer(h2, 64, w.t3w, w.t3b, o_tr, 3, false);
  if (threadIdx.x == 0) {
    // models/posenet.py:22-36 compute_rotation_matrix_from_ortho6d
    float xr[3] = {o_rot[0], o_rot[1], o_rot[2]}, yr[3] = {o_rot[3], o_rot[4], o_rot[5]};
    float n = fmaxf(sqrtf(xr[0] * xr[0] + xr[1] * xr[1] + xr[2] * xr[2]), 1e-8f);
    float xv[3] = {xr[0] / n, xr[1] / n, xr[2] / n};
    float z[3] = {xv[1] * yr[2] - xv[2] * yr[1], xv[2] * yr[0] - xv[0] * yr[2], xv[0] * yr[1] - xv[1] * yr[0]};
    n = fmaxf(sqrtf(z[0] * z[0] + z[1] * z[1] + z[2] * z[2]), 1e-8f);
    z[0] /= n; z[1] /= n; z[2] /= n;
    float yv[3] = {z[1] * xv[2] - z[2] * xv[1], z[2] * xv[0] - z[0] * xv[2], z[0] * xv[1] - z[1] * xv[0]};
    const float s = o_scale[0];
    float rt[4][3];
    for (int i = 0; i < 3; ++i) { rt[i][0] = s * xv[i]; rt[i][1] = s * yv[i]; rt[i][2] = s * z[i]; }   // columns x,y,z
    // models/posenet.py:118 translation offset constant
    rt[3][0] = o_tr[0] + (-0.00193892f); rt[3][1] = o_tr[1] + 0.00169222f; rt[3][2] = o_tr[2] + 1.3949631f;
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 3; ++j) {
        if (out_rt) out_rt[(size_t)b * 12 + i * 3 + j] = rt[i][j];
        float a = 0.f;                                       // (RT . K^T)[i][j] = sum_k RT[i][k] * K[j][k]
        for (int k = 0; k < 3; ++k) a = fmaf(rt[i][k], Kmat[j * 3 + k], a);
        out_tm[(size_t)b * 12 + i * 3 + j] = a;
      }
  }
}

}  // namespace

int launch_cam_heads(disn_ctx* c, int B, const float* d_emb, const float* d_K, float* d_rt, float* d_tm) {
  DISN_REQUIRE(c->cfg.num_classes <= 1024, "camera heads expect an embedding of at most 1024");
  CamHeadWeights w;
  // each variable must hold exactly the elements the kernel reads: [in, out] weights and [out] biases
  auto get = [&](const char* n, int64_t numel, const float*& p) -> int {
    const std::string name = std::string("cameraprediction/") + n;
    auto it = c->weights.find(name);
    DISN_REQUIRE(it != c->weights.end(), "missing variable " + name);
    DISN_REQUIRE(it->second.numel == numel, "mis-shaped variable " + name);
    p = it->second.ptr();
    return 0;
  };
  const int64_t e = c->cfg.num_classes;
  if (get("scale/fc1/weights", e * 64, w.s1w) || get("scale/fc1/biases", 64, w.s1b) ||
      get("scale/fc2/weights", 64 * 32, w.s2w) || get("scale/fc2/biases", 32, w.s2b) ||
      get("scale/fc3/weights", 32, w.s3w) || get("scale/fc3/biases", 1, w.s3b) ||
      get("ortho6d/fc1/weights", e * 512, w.r1w) || get("ortho6d/fc1/biases", 512, w.r1b) ||
      get("ortho6d/fc2/weights", 512 * 256, w.r2w) || get("ortho6d/fc2/biases", 256, w.r2b) ||
      get("ortho6d/fc3/weights", 256 * 6, w.r3w) || get("ortho6d/fc3/biases", 6, w.r3b) ||
      get("translation/fc1/weights", e * 128, w.t1w) || get("translation/fc1/biases", 128, w.t1b) ||
      get("translation/fc2/weights", 128 * 64, w.t2w) || get("translation/fc2/biases", 64, w.t2b) ||
      get("translation/fc3/weights", 64 * 3, w.t3w) || get("translation/fc3/biases", 3, w.t3b))
    return -2;
  cam_heads_kernel<<<B, 256, 0, c->stream>>>(d_emb, c->cfg.num_classes, w, d_K, d_rt, d_tm);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  return 0;
}

int cam_predict(disn_ctx* c, const float* imgs, int B, int H, int W, int C, const float* K, float* d_K, float* d_rt,
                float* d_tm) {
  if (encoder_run(c, imgs, B, H, W, C, false, /*embedding_only=*/true)) return -1;
  static const float kDefaultK[9] = {149.84375f, 0.f, 68.5f, 0.f, 149.84375f, 68.5f, 0.f, 0.f, 1.f};
  DISN_CUDA_OK(cudaMemcpyAsync(d_K, K ? K : kDefaultK, 9 * 4, cudaMemcpyHostToDevice, c->stream));
  return launch_cam_heads(c, B, c->emb.as<float>(), d_K, d_rt, d_tm);
}

namespace {

// Camera checkpoint score -- the losses of cam_est/model_cam.py:125-239 that eval_one_epoch (cam_est/
// train_sdf_cam.py:459-565) fetches, per image.  Per point p, with h = [p, 1] and every matrix product summed in k order:
//   sub = h.pred_RT - h.RT                                     -> sums[0] += |sub|^2 (element by element), sums[2] += sqrt(|sub|^2)
//   xy = (h.tm)[:2] / (h.tm)[2] for tm and pred_tm (get_img_points) -> sums[1] += |xy_pr - xy_gt|^2 (element by element),
//        sums[3] += sqrt(|clamp(xy_gt) - clamp(xy_pr)|^2) with the reference's hard-coded [0, 136] clamp
// and sums[4] = sum over the 12 entries of (pred_tm - tm)^2.  The terms are float32, one rounding per op (this file is
// built with --fmad=false); the sums are float64 in a fixed order (thread-strided loop, then a fixed tree), so repeated
// calls are bitwise equal.
constexpr int CAM_ACC_THREADS = 256;

__device__ __forceinline__ void homo_mul(const float* p, const float* M, float* out) {   // [p, 1] . M[4,3]
  for (int j = 0; j < 3; ++j) out[j] = ((p[0] * M[j] + p[1] * M[3 + j]) + p[2] * M[6 + j]) + M[9 + j];
}

__device__ __forceinline__ float clamp136(float x) { return fminf(136.f, fmaxf(0.f, x)); }

__global__ void __launch_bounds__(CAM_ACC_THREADS) cam_acc_kernel(const float* __restrict__ pts, int64_t N,
                                                                  const float* __restrict__ tm, const float* __restrict__ rt,
                                                                  const float* __restrict__ pred_tm,
                                                                  const float* __restrict__ pred_rt,
                                                                  double* __restrict__ sums) {
  __shared__ float m[4][12];      // tm, RT, pred_tm, pred_RT of this image
  __shared__ double s[4][CAM_ACC_THREADS];
  const int b = blockIdx.x, t = threadIdx.x;
  if (t < 48) {
    const float* src = t < 12 ? tm : t < 24 ? rt : t < 36 ? pred_tm : pred_rt;
    m[t / 12][t % 12] = src[(size_t)b * 12 + t % 12];
  }
  __syncthreads();
  const float* P = pts + (size_t)b * N * 3;
  double rotpc = 0.0, rot2d = 0.0, rot3d = 0.0, dist2d = 0.0;
  for (int64_t n = t; n < N; n += CAM_ACC_THREADS) {
    const float p[3] = {P[3 * n], P[3 * n + 1], P[3 * n + 2]};
    float a[3], g[3], u[3], v[3];
    homo_mul(p, m[3], a);
    homo_mul(p, m[1], g);
    const float s0 = a[0] - g[0], s1 = a[1] - g[1], s2 = a[2] - g[2];
    const float q0 = s0 * s0, q1 = s1 * s1, q2 = s2 * s2;
    rotpc = ((rotpc + (double)q0) + (double)q1) + (double)q2;
    rot3d += (double)sqrtf((q0 + q1) + q2);
    homo_mul(p, m[0], u);
    homo_mul(p, m[2], v);
    const float xg = u[0] / u[2], yg = u[1] / u[2], xp = v[0] / v[2], yp = v[1] / v[2];
    const float dx = xp - xg, dy = yp - yg;
    rot2d = (rot2d + (double)(dx * dx)) + (double)(dy * dy);
    const float cx = clamp136(xg) - clamp136(xp), cy = clamp136(yg) - clamp136(yp);
    dist2d += (double)sqrtf(cx * cx + cy * cy);
  }
  s[0][t] = rotpc; s[1][t] = rot2d; s[2][t] = rot3d; s[3][t] = dist2d;
  __syncthreads();
  for (int h = CAM_ACC_THREADS / 2; h > 0; h >>= 1) {
    if (t < h)
      for (int k = 0; k < 4; ++k) s[k][t] += s[k][t + h];
    __syncthreads();
  }
  if (t == 0) {
    double mat = 0.0;
    for (int i = 0; i < 12; ++i) {
      const float d = m[2][i] - m[0][i];
      mat += (double)(d * d);
    }
    for (int k = 0; k < 4; ++k) sums[(size_t)b * 5 + k] = s[k][0];
    sums[(size_t)b * 5 + 4] = mat;
  }
}

}  // namespace
}  // namespace disn

using namespace disn;

extern "C" int disn_cam_metrics(disn_ctx* c, const float* imgs, int32_t B, int32_t H, int32_t W, int32_t C, const float* K,
                                const float* pts, int64_t N, const float* trans_mat, const float* RT, float* out_rt,
                                float* out_trans_mat, double* sums) {
  DISN_REQUIRE(c && imgs && pts && trans_mat && RT && sums, "null argument");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  DISN_REQUIRE(B >= 1 && B <= c->cfg.max_batch, "cam_metrics: batch outside [1, max_batch of the context]");
  DISN_REQUIRE(N >= 1, "cam_metrics: N >= 1 points per image");
  float *dK, *dRT, *dTM, *dPts, *dGtTM, *dGtRT;
  double* dSums;
  auto carve = [&](char* base) {
    Arena a{base};
    dK = a.take<float>(9);
    dRT = a.take<float>((size_t)B * 12);
    dTM = a.take<float>((size_t)B * 12);
    dGtRT = a.take<float>((size_t)B * 12);
    dGtTM = a.take<float>((size_t)B * 12);
    dSums = a.take<double>((size_t)B * 5);
    dPts = a.take<float>((size_t)B * N * 3);
    return a.off;
  };
  if (c->nn_scratch.ensure(carve(nullptr))) return -1;
  carve(c->nn_scratch.as<char>());
  if (cam_predict(c, imgs, B, H, W, C, K, dK, dRT, dTM)) return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(dPts, pts, (size_t)B * N * 3 * 4, cudaMemcpyHostToDevice, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(dGtTM, trans_mat, (size_t)B * 12 * 4, cudaMemcpyHostToDevice, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(dGtRT, RT, (size_t)B * 12 * 4, cudaMemcpyHostToDevice, c->stream));
  cam_acc_kernel<<<B, CAM_ACC_THREADS, 0, c->stream>>>(dPts, N, dGtTM, dGtRT, dTM, dRT, dSums);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  if (out_rt) DISN_CUDA_OK(cudaMemcpyAsync(out_rt, dRT, (size_t)B * 12 * 4, cudaMemcpyDeviceToHost, c->stream));
  if (out_trans_mat) DISN_CUDA_OK(cudaMemcpyAsync(out_trans_mat, dTM, (size_t)B * 12 * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(sums, dSums, (size_t)B * 5 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}
