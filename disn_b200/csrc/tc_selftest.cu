// Self-test of the warpgroup-MMA building blocks used by the tensor-core kernels: one warpgroup computes
// D[128 x 256] = A[128 x 64] * B[256 x 64]^T (bf16 in, fp32 accumulate) as four m64n128 blocks, `passes` times
// accumulated, exercising SW128 K-major descriptors of tiles written by threads (A) and by the bulk-copy engine from a
// host-swizzled image (B), and the register layout of the accumulator fragment.
#include <vector>

#include "common.cuh"
#include "tc_common.cuh"

namespace disn {
namespace {

struct SelfSmem {
  alignas(1024) uint8_t a_tile[64 * 128];     // 64 rows x 64 bf16, SW128
  alignas(1024) uint8_t b_tile[128 * 128];    // 128 rows x 64 bf16, SW128
  alignas(8) uint64_t b_full;
};

// D block (c, h) -> D_out[c][64 h + row][col], the layout the test-suite reassembles
__device__ __forceinline__ void store_block(float* D, int c, int h, const float (&acc)[64]) {
  const int tid = threadIdx.x, lane = tid & 31;
  const int r0 = (tid >> 5) * 16 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int row = r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + (lane & 3) * 2 + (i & 1);
    D[((size_t)c * 128 + h * 64 + row) * 128 + col] = acc[i];
  }
}

__global__ void __launch_bounds__(128, 1)
tc_selftest_kernel(const __nv_bfloat16* __restrict__ A,       // [128][64] row-major
                   const uint8_t* __restrict__ Bimg,          // 2 x 16 KB pre-swizzled halves
                   float* __restrict__ D,                     // [2][128][128]
                   int passes) {
  extern __shared__ uint8_t smem_raw[];
  // dynamic smem is only 16-B aligned by contract: round the shared-window address up to 1024 B
  SelfSmem& s = *reinterpret_cast<SelfSmem*>(smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u));
  const int tid = threadIdx.x;
  if (tid == 0) {
    tc::mbar_init(&s.b_full, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  uint32_t phase = 0;
  for (int c = 0; c < 2; ++c)
    for (int h = 0; h < 2; ++h) {
      // A rows of block c written by threads exactly like the epilogues do (thread = row, 8 x 16 B chunks)
      if (tid < 64) {
        const uint4* src = reinterpret_cast<const uint4*>(A + (size_t)(c * 64 + tid) * 64);
#pragma unroll
        for (int k = 0; k < 8; ++k) *reinterpret_cast<uint4*>(s.a_tile + tc::sw128_offset(tid, k)) = src[k];
      }
      tc::fence_proxy_async_smem();
      __syncthreads();
      if (tid == 0) {
        tc::mbar_arrive_expect_tx(&s.b_full, 128 * 128);
        tc::bulk_g2s(s.b_tile, Bimg + (size_t)h * 128 * 128, 128 * 128, &s.b_full);
      }
      tc::mbar_wait(&s.b_full, phase);
      phase ^= 1u;
      float acc[64];
      tc::acc_fence(acc);
      tc::wgmma_fence();
      const uint32_t a0 = tc::smem_u32(s.a_tile), b0 = tc::smem_u32(s.b_tile);
      for (int p = 0; p < passes; ++p)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          tc::wgmma_m64n128<tc::KIND_BF16>(acc, tc::desc_sw128(a0 + 32u * k), tc::desc_sw128(b0 + 32u * k), (p | k) ? 1u : 0u);
      tc::wgmma_commit();
      tc::wgmma_wait<0>();
      tc::acc_fence(acc);
      store_block(D, c, h, acc);
      __syncthreads();                        // the tiles are rewritten for the next block
    }
}

}  // namespace
}  // namespace disn

// Returns 0 and max |D - ref| in *max_err. Host pointers: A [128*64] fp32 values (rounded to bf16 inside),
// B [256*64] fp32.  Exposed through the C ABI for the GPU test-suite.
extern "C" int disn_tc_selftest(int device, const float* A, const float* B, int passes, float* D_out /*[2*128*128]*/) {
  using namespace disn;
  DISN_CUDA_OK(cudaSetDevice(device));
  std::vector<__nv_bfloat16> a(128 * 64);
  for (int i = 0; i < 128 * 64; ++i) a[i] = __float2bfloat16(A[i]);
  std::vector<uint8_t> bimg(2 * 128 * 128);
  for (int n = 0; n < 256; ++n)
    for (int k = 0; k < 64; ++k) {
      __nv_bfloat16 v = __float2bfloat16(B[n * 64 + k]);
      int half = n / 128, row = n % 128;
      uint32_t off = tc::sw128_offset(row, k / 8) + (k % 8) * 2;
      memcpy(&bimg[(size_t)half * 128 * 128 + off], &v, 2);
    }
  __nv_bfloat16* dA = nullptr; uint8_t* dB = nullptr; float* dD = nullptr;
  DISN_CUDA_OK(cudaMalloc(&dA, a.size() * 2));
  DISN_CUDA_OK(cudaMalloc(&dB, bimg.size()));
  DISN_CUDA_OK(cudaMalloc(&dD, 2 * 128 * 128 * sizeof(float)));
  DISN_CUDA_OK(cudaMemcpy(dA, a.data(), a.size() * 2, cudaMemcpyHostToDevice));
  DISN_CUDA_OK(cudaMemcpy(dB, bimg.data(), bimg.size(), cudaMemcpyHostToDevice));
  DISN_CUDA_OK(cudaMemset(dD, 0xff, 2 * 128 * 128 * sizeof(float)));
  DISN_CUDA_OK(cudaFuncSetAttribute(tc_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)sizeof(SelfSmem) + 1024));
  tc_selftest_kernel<<<1, 128, sizeof(SelfSmem) + 1024>>>(dA, dB, dD, passes);
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaDeviceSynchronize());
  DISN_CUDA_OK(cudaMemcpy(D_out, dD, 2 * 128 * 128 * sizeof(float), cudaMemcpyDeviceToHost));
  cudaFree(dA); cudaFree(dB); cudaFree(dD);
  return 0;
}

// ---------------------------------------------------------------------------------------------------------
// Mixed-kind self-test (building block of DISN_PREC_F16F8):
//   D = fp16(A16) * fp16(B16)^T   (SW128 tiles, 4 x K=16, main accumulator)
//     + e5m2(A8) * e5m2(B8)^T     (SW64 tiles of bytes, 2 x K=32, zero-initialised second accumulator added in fp32,
//                                  as the point kernel does)
// mode bit 0 enables the f16 part, bit 1 the f8 part.
// ---------------------------------------------------------------------------------------------------------
#include <cuda_fp16.h>
#include <cuda_fp8.h>

namespace disn {
namespace {

struct MixSmem {
  alignas(1024) uint8_t a16[64 * 128];
  alignas(1024) uint8_t b16[128 * 128];
  alignas(1024) uint8_t a8[64 * 64];
  alignas(1024) uint8_t b8[128 * 64];
  alignas(8) uint64_t b_full;
};

__global__ void __launch_bounds__(128, 1)
tc_selftest_mixed_kernel(const __half* __restrict__ A16, const uint8_t* __restrict__ A8,      // [128][64] row-major
                         const uint8_t* __restrict__ Bimg,   // per 128-row half: 16 KB SW128 fp16 + 8 KB SW64 e5m2
                         float* __restrict__ D, int mode) {
  extern __shared__ uint8_t smem_raw[];
  MixSmem& s = *reinterpret_cast<MixSmem*>(smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u));
  const int tid = threadIdx.x;
  if (tid == 0) {
    tc::mbar_init(&s.b_full, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  uint32_t phase = 0;
  for (int c = 0; c < 2; ++c)
    for (int h = 0; h < 2; ++h) {
      if (tid < 64) {
        const uint4* src = reinterpret_cast<const uint4*>(A16 + (size_t)(c * 64 + tid) * 64);
#pragma unroll
        for (int k = 0; k < 8; ++k) *reinterpret_cast<uint4*>(s.a16 + tc::sw128_offset(tid, k)) = src[k];
        const uint4* src8 = reinterpret_cast<const uint4*>(A8 + (size_t)(c * 64 + tid) * 64);
#pragma unroll
        for (int k = 0; k < 4; ++k) *reinterpret_cast<uint4*>(s.a8 + tc::sw64_offset(tid, k)) = src8[k];
      }
      tc::fence_proxy_async_smem();
      __syncthreads();
      if (tid == 0) {
        tc::mbar_arrive_expect_tx(&s.b_full, 128 * 128 + 128 * 64);
        tc::bulk_g2s(s.b16, Bimg + (size_t)h * (128 * 192), 128 * 128, &s.b_full);
        tc::bulk_g2s(s.b8, Bimg + (size_t)h * (128 * 192) + 128 * 128, 128 * 64, &s.b_full);
      }
      tc::mbar_wait(&s.b_full, phase);
      phase ^= 1u;
      float acc[64], cor[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = cor[i] = 0.f;
      tc::acc_fence(acc);
      tc::acc_fence(cor);
      tc::wgmma_fence();
      if (mode & 1)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          tc::wgmma_m64n128<tc::KIND_F16>(acc, tc::desc_sw128(tc::smem_u32(s.a16) + 32u * k),
                                          tc::desc_sw128(tc::smem_u32(s.b16) + 32u * k), k ? 1u : 0u);
      if (mode & 2)
#pragma unroll
        for (int k = 0; k < 2; ++k)
          tc::wgmma_m64n128<tc::KIND_E5M2>(cor, tc::desc_sw64(tc::smem_u32(s.a8) + 32u * k),
                                           tc::desc_sw64(tc::smem_u32(s.b8) + 32u * k), k ? 1u : 0u);
      tc::wgmma_commit();
      tc::wgmma_wait<0>();
      tc::acc_fence(acc);
      tc::acc_fence(cor);
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] += cor[i];
      store_block(D, c, h, acc);
      __syncthreads();
    }
}

}  // namespace
}  // namespace disn

// Host fp32 inputs A16,A8 [128*64], B16,B8 [256*64]; the e5m2 roundings actually used are returned in A8q/B8q so the
// caller can form the exact reference.  D_out [2*128*128]: D_out[c][64 h + r][j] = D[64 c + r][128 h + j].
extern "C" int disn_tc_selftest_mixed(int device, const float* A16, const float* B16, const float* A8, const float* B8,
                                      int mode, float* A8q, float* B8q, float* D_out) {
  using namespace disn;
  DISN_CUDA_OK(cudaSetDevice(device));
  std::vector<__half> a16(128 * 64);
  std::vector<uint8_t> a8(128 * 64), bimg(2 * 128 * 192);
  for (int i = 0; i < 128 * 64; ++i) {
    a16[i] = __float2half_rn(A16[i]);
    a8[i] = (uint8_t)__nv_cvt_float_to_fp8(A8[i], __NV_SATFINITE, __NV_E5M2);
    A8q[i] = __half2float(__half(__nv_cvt_fp8_to_halfraw(a8[i], __NV_E5M2)));
  }
  for (int n = 0; n < 256; ++n)
    for (int k = 0; k < 64; ++k) {
      const int half = n / 128, row = n % 128;
      __half v = __float2half_rn(B16[n * 64 + k]);
      memcpy(&bimg[(size_t)half * 128 * 192 + tc::sw128_offset(row, k / 8) + (k % 8) * 2], &v, 2);
      const uint8_t q = (uint8_t)__nv_cvt_float_to_fp8(B8[n * 64 + k], __NV_SATFINITE, __NV_E5M2);
      bimg[(size_t)half * 128 * 192 + 128 * 128 + tc::sw64_offset(row, k / 16) + (k % 16)] = q;
      B8q[n * 64 + k] = __half2float(__half(__nv_cvt_fp8_to_halfraw(q, __NV_E5M2)));
    }
  __half* dA = nullptr; uint8_t *dA8 = nullptr, *dB = nullptr; float* dD = nullptr;
  DISN_CUDA_OK(cudaMalloc(&dA, a16.size() * 2));
  DISN_CUDA_OK(cudaMalloc(&dA8, a8.size()));
  DISN_CUDA_OK(cudaMalloc(&dB, bimg.size()));
  DISN_CUDA_OK(cudaMalloc(&dD, 2 * 128 * 128 * sizeof(float)));
  DISN_CUDA_OK(cudaMemcpy(dA, a16.data(), a16.size() * 2, cudaMemcpyHostToDevice));
  DISN_CUDA_OK(cudaMemcpy(dA8, a8.data(), a8.size(), cudaMemcpyHostToDevice));
  DISN_CUDA_OK(cudaMemcpy(dB, bimg.data(), bimg.size(), cudaMemcpyHostToDevice));
  DISN_CUDA_OK(cudaMemset(dD, 0xff, 2 * 128 * 128 * sizeof(float)));
  DISN_CUDA_OK(cudaDeviceSynchronize());
  DISN_CUDA_OK(cudaFuncSetAttribute(tc_selftest_mixed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)sizeof(MixSmem) + 1024));
  tc_selftest_mixed_kernel<<<1, 128, sizeof(MixSmem) + 1024>>>(dA, dA8, dB, dD, mode);
  DISN_CUDA_OK(cudaGetLastError());
  DISN_CUDA_OK(cudaDeviceSynchronize());
  DISN_CUDA_OK(cudaMemcpy(D_out, dD, 2 * 128 * 128 * sizeof(float), cudaMemcpyDeviceToHost));
  cudaFree(dA); cudaFree(dA8); cudaFree(dB); cudaFree(dD);
  return 0;
}
