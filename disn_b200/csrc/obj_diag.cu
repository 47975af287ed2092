// Diagnostic of the OBJ reader (libdisn_b200_test.so): its host coordinate converter on a batch of tokens.
#include <string>

#include "../../include/disn_b200_test.h"
#include "common.cuh"

using namespace disn;

extern "C" int disn_debug_obj_tokens(const char* text, const int64_t* offsets, const int32_t* lengths, int64_t n,
                                     float* out) {
  DISN_REQUIRE(text && offsets && lengths && out && n >= 0, "null argument");
  for (int64_t i = 0; i < n; ++i) {
    bool overflow = false;
    if (obj_token_to_float(text + offsets[i], lengths[i], &out[i], &overflow))
      DISN_REQUIRE(false, "token " + std::to_string(i) + " (" + std::string(text + offsets[i], lengths[i]) +
                              ") is outside the OBJ reader's grammar");
  }
  return 0;
}
