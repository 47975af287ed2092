// Diagnostics of the tensor-core point kernel (point_tc.cu), exported by libdisn_b200_test.so only: the packed weight
// half-stage images of one operand mode and the e5m2 activation scales, as tc_pack_weights left them in the context.
#include <cstring>

#include "../../include/disn_b200_test.h"
#include "common.cuh"

using namespace disn;

namespace {
// HS_PER_TILE (2 streams x 2 halves x 33 stages) half-stages of 32 KB each, the layout documented at tc_pack_weights
constexpr int64_t kPackedBytes = (int64_t)2 * 2 * 33 * 32768;
}  // namespace

extern "C" {

int disn_debug_tc_weights(disn_ctx* c, int32_t precision, int64_t nbytes, uint8_t* image, float* act_scale) {
  DISN_REQUIRE(c && image && act_scale, "null argument");
  DISN_REQUIRE(precision == DISN_PREC_BF16X3 || precision == DISN_PREC_F16F8,
               "debug_tc_weights: precision must be DISN_PREC_BF16X3 or DISN_PREC_F16F8");
  DISN_REQUIRE(nbytes == kPackedBytes, "debug_tc_weights: the packed image holds " + std::to_string(kPackedBytes) + " bytes");
  const DevBuffer& w = precision == DISN_PREC_F16F8 ? c->tc_weights_f8 : c->tc_weights;
  DISN_REQUIRE(w.as<void>() != nullptr && (int64_t)w.bytes() >= kPackedBytes,
               "debug_tc_weights: tensor-core weights not packed (call disn_finalize_weights)");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  DISN_CUDA_OK(cudaMemcpyAsync(image, w.as<void>(), (size_t)kPackedBytes, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  memcpy(act_scale, c->tc_act_scale, sizeof(c->tc_act_scale));
  return 0;
}

}  // extern "C"
