// Diagnostic of the camera-pose heads (libdisn_b200_test.so): the heads of disn_cam_estimate on a caller's embedding.
#include "../../include/disn_b200_test.h"
#include "common.cuh"

using namespace disn;

extern "C" int disn_debug_cam_heads(disn_ctx* c, const float* emb, int32_t B, const float* K, float* out_rt,
                                    float* out_trans_mat) {
  DISN_REQUIRE(c && emb && out_rt && out_trans_mat, "null argument");
  DISN_REQUIRE(B >= 1, "batch must be positive");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  static const float kDefaultK[9] = {149.84375f, 0.f, 68.5f, 0.f, 149.84375f, 68.5f, 0.f, 0.f, 1.f};
  const size_t ne = (size_t)B * c->cfg.num_classes;
  DevBuffer d_emb, d_K, d_rt, d_tm;     // own buffers: the context's encoder products stay as they are
  if (d_emb.ensure(ne * 4) || d_K.ensure(9 * 4) || d_rt.ensure((size_t)B * 12 * 4) || d_tm.ensure((size_t)B * 12 * 4))
    return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(d_emb.as<float>(), emb, ne * 4, cudaMemcpyHostToDevice, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(d_K.as<float>(), K ? K : kDefaultK, 9 * 4, cudaMemcpyHostToDevice, c->stream));
  if (launch_cam_heads(c, B, d_emb.as<float>(), d_K.as<float>(), d_rt.as<float>(), d_tm.as<float>())) {
    cudaStreamSynchronize(c->stream);     // the copies above read the caller's buffers
    return -1;
  }
  DISN_CUDA_OK(cudaMemcpyAsync(out_rt, d_rt.as<float>(), (size_t)B * 12 * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(out_trans_mat, d_tm.as<float>(), (size_t)B * 12 * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}
