// Implicit-GEMM convolution / GEMM on Hopper tensor cores (warpgroup MMA) for the image encoder (sm_90a).
//
//   C[M, N] = act( A[M, K] * W[K, N] + bias ),  A = NHWC activations viewed through a 3x3 SAME im2col
//   (K = 9*Cin, k = tap*Cin + ci -- the row order of TF's HWIO weights) or a plain row-major matrix.
//
// Same precision scheme as the point kernel: every fp32 operand is split into bf16 hi + lo and each product is
// three MMAs (hi*hi + lo*hi + hi*lo) with fp32 accumulation, so the encoder keeps fp32-level accuracy
// (the reference runs VGG in fp32; models/CNN/vgg.py:187-196, models/model_normalization.py:76).
//
// One CTA = 128 pixels x 128 output channels, two warpgroups (wgmma m64n128k16, 64 rows each), 64-wide K slices
// double-buffered in shared memory: while the tensor cores work on slice t, every thread gathers its part of slice t+1
// of A (a half-warp reads the 64 channels of one filter tap of one pixel row, 256 contiguous bytes; zeros outside the
// image), splits it to bf16 hi / lo into the K-major 128B-swizzled tile, and thread 0 has the bulk-copy engine fetch
// the host-packed [W_hi | W_lo] 32 KB image of slice t+1.
// Jobs = (m-tile, n-block, k-split); a persistent grid walks them.  Under-filled layers are split along K and
// reduced by splitk_reduce_kernel.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "tc_common.cuh"

namespace disn {
namespace {

constexpr int CT_THREADS = 256;
constexpr int CT_A_HALF = 16384;    // 128 rows x 64 k x bf16
constexpr int CT_B_TILE = 16384;    // 128 rows x 64 k x bf16
constexpr int CT_B_STAGE = 2 * CT_B_TILE;

struct ConvTcSmem {
  alignas(1024) uint8_t a[2][2][CT_A_HALF];    // [slot][hi|lo]   64 KB
  alignas(1024) uint8_t b[2][CT_B_STAGE];      // [slot][hi|lo]   64 KB
  alignas(8) uint64_t bfull[2];
};

struct ConvTcJob {
  const float* A;          // NHWC activations [B,H,W,Cin] or row-major [M,K]
  const uint8_t* wpk;      // packed weights: [n-block][k-slice][hi|lo][128 x 64 SW128]
  const float* bias;       // [N] or nullptr
  float* C;                // [M,N] fp32
  float* ws;               // split-K workspace [splits][M][N] or nullptr
  int M, N, K;             // K multiple of 64
  int H, W, Cin;           // im2col geometry (Cin multiple of 64); H == 0 -> plain matrix
  int relu;
  int m_tiles, n_blocks, splits, slices_per_split;
};

__global__ void __launch_bounds__(CT_THREADS, 1) conv_tc_kernel(ConvTcJob job) {
  extern __shared__ uint8_t smem_raw[];
  ConvTcSmem& s = *reinterpret_cast<ConvTcSmem*>(smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int total_jobs = job.m_tiles * job.n_blocks * job.splits;
  const int my_jobs = ((int)blockIdx.x < total_jobs) ? (total_jobs - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
  const int nsl = job.slices_per_split;
  const int total = my_jobs * nsl;          // this CTA's K slices, all jobs

  if (tid == 0) {
    tc::mbar_init(&s.bfull[0], 1);
    tc::mbar_init(&s.bfull[1], 1);
    tc::fence_barrier_init();
  }
  __syncthreads();

  // job index -> (m-tile, n-block, split): n-block fastest so neighbouring CTAs share the A rows in L2
  auto decode = [&](int j, int& mt, int& nb, int& sp) {
    nb = j % job.n_blocks;
    const int r = j / job.n_blocks;
    mt = r % job.m_tiles;
    sp = r / job.m_tiles;
  };
  auto load_b = [&](int q) {      // thread 0: B image of slice q into slot q & 1
    int mt, nb, sp;
    decode((int)blockIdx.x + (q / nsl) * (int)gridDim.x, mt, nb, sp);
    const uint8_t* src = job.wpk + ((size_t)nb * (job.K / 64) + (size_t)sp * nsl + (size_t)(q % nsl)) * CT_B_STAGE;
    tc::mbar_arrive_expect_tx(&s.bfull[q & 1], CT_B_STAGE);
    tc::bulk_g2s(s.b[q & 1], src, CT_B_STAGE, &s.bfull[q & 1]);
  };
  // A slice q -> registers: thread owns float4 f4 (of 16) of rows row0 + 16 i, i < 8
  const int f4 = tid & 15, row0 = tid >> 4;
  auto load_a = [&](int q, float4 (&v)[8]) {
    int mt, nb, sp;
    decode((int)blockIdx.x + (q / nsl) * (int)gridDim.x, mt, nb, sp);
    const int k0 = (sp * nsl + q % nsl) * 64;
    int tap = 0, dy = 0, dx = 0, c0 = k0;
    if (job.H > 0) {
      tap = k0 / job.Cin;
      dy = tap / 3 - 1; dx = tap % 3 - 1;
      c0 = k0 % job.Cin;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int m = mt * 128 + row0 + 16 * i;
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m >= job.M) continue;
      if (job.H > 0) {
        const int r = m % (job.H * job.W);
        const int y = r / job.W + dy, x = r % job.W + dx;
        if (y < 0 || y >= job.H || x < 0 || x >= job.W) continue;
        const int64_t pix = (int64_t)m + (int64_t)dy * job.W + dx;
        v[i] = __ldg(reinterpret_cast<const float4*>(job.A + pix * job.Cin + c0) + f4);
      } else {
        v[i] = __ldg(reinterpret_cast<const float4*>(job.A + (int64_t)m * job.K + k0) + f4);
      }
    }
  };
  auto store_a = [&](const float4 (&v)[8], int slot) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      uint32_t h0, h1, l0, l1;
      tc::split_bf16x2(v[i].x, v[i].y, h0, l0);
      tc::split_bf16x2(v[i].z, v[i].w, h1, l1);
      const uint32_t off = tc::sw128_offset((uint32_t)(row0 + 16 * i), (uint32_t)(f4 >> 1)) + (uint32_t)(f4 & 1) * 8u;
      *reinterpret_cast<uint2*>(s.a[slot][0] + off) = make_uint2(h0, h1);
      *reinterpret_cast<uint2*>(s.a[slot][1] + off) = make_uint2(l0, l1);
    }
  };

  const int wg = warp >> 2;                     // rows [64 wg, 64 wg + 64) of the tile
  const uint32_t a_base = tc::smem_u32(s.a[0][0]) + (uint32_t)wg * 8192u, b_base = tc::smem_u32(s.b[0]);
  float acc[64];
  float4 v[8];
  if (total > 0) {
    if (tid == 0) load_b(0);
    load_a(0, v);
    store_a(v, 0);
  }
  for (int q = 0; q < total; ++q) {
    const int slot = q & 1, t = q % nsl;
    tc::fence_proxy_async_smem();
    __syncthreads();                            // A(q) stored; every MMA of slice q-1 has completed
    if (tid == 0 && q + 1 < total) load_b(q + 1);
    tc::mbar_wait(&s.bfull[slot], (uint32_t)(q >> 1) & 1u);
    const uint32_t a_hi = a_base + (uint32_t)slot * (2 * CT_A_HALF), a_lo = a_hi + CT_A_HALF;
    const uint32_t b_hi = b_base + (uint32_t)slot * CT_B_STAGE, b_lo = b_hi + CT_B_TILE;
    tc::acc_fence(acc);
    tc::wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      tc::wgmma_m64n128<tc::KIND_BF16>(acc, tc::desc_sw128(a_hi + 32u * k), tc::desc_sw128(b_hi + 32u * k), (t | k) ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      tc::wgmma_m64n128<tc::KIND_BF16>(acc, tc::desc_sw128(a_lo + 32u * k), tc::desc_sw128(b_hi + 32u * k), 1u);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      tc::wgmma_m64n128<tc::KIND_BF16>(acc, tc::desc_sw128(a_hi + 32u * k), tc::desc_sw128(b_lo + 32u * k), 1u);
    tc::wgmma_commit();
    if (q + 1 < total) {                        // next slice's A while the tensor cores run
      load_a(q + 1, v);
      store_a(v, slot ^ 1);
    }
    tc::wgmma_wait<0>();
    tc::acc_fence(acc);
    if (t == nsl - 1) {
      // ===================== epilogue: +bias, ReLU -> fp32 store (or raw split-K partials to the workspace) =========
      int mt, nb, sp;
      decode((int)blockIdx.x + (q / nsl) * (int)gridDim.x, mt, nb, sp);
      const bool fin = !job.ws;                 // final values (bias, ReLU) or raw split-K partials
      const float lo = (fin && job.relu) ? 0.f : -INFINITY;
      const int rbase = mt * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = nb * 128 + 8 * j + (lane & 3) * 2;
        if (col >= job.N) continue;             // N is a multiple of 32; the padded columns are never stored
        const float2 b2 = (fin && job.bias) ? __ldg(reinterpret_cast<const float2*>(job.bias + col)) : make_float2(0.f, 0.f);
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
          const int m = rbase + 8 * e2;
          if (m >= job.M) continue;
          float* dst = job.ws ? job.ws + ((size_t)sp * job.M + m) * job.N : job.C + (size_t)m * job.N;
          *reinterpret_cast<float2*>(dst + col) =
              make_float2(fmaxf(acc[4 * j + 2 * e2] + b2.x, lo), fmaxf(acc[4 * j + 2 * e2 + 1] + b2.y, lo));
        }
      }
    }
  }
}

}  // namespace

// [K, N] fp32 row-major (device) -> packed B stage images [N/128][K/64][hi|lo][128 x 64 SW128 bf16] (device)
int conv_tc_pack(disn_ctx* c, const float* d_w, int K, int N, DevBuffer& out) {
  std::vector<float> w((size_t)K * N);
  DISN_CUDA_OK(cudaMemcpyAsync(w.data(), d_w, w.size() * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  const int ns = K / 64, nbk = (N + 127) / 128;
  std::vector<uint8_t> img((size_t)nbk * ns * CT_B_STAGE, 0);   // rows beyond N stay zero
  for (int nb = 0; nb < nbk; ++nb)
    for (int t = 0; t < ns; ++t)
      for (int part = 0; part < 2; ++part) {
        uint8_t* dst = img.data() + ((size_t)nb * ns + t) * CT_B_STAGE + (size_t)part * CT_B_TILE;
        for (int nl = 0; nl < 128 && nb * 128 + nl < N; ++nl)
          for (int k = 0; k < 64; ++k) {
            const float v = w[(size_t)(t * 64 + k) * N + nb * 128 + nl];
            const __nv_bfloat16 hi = __float2bfloat16(v);
            const __nv_bfloat16 o = part == 0 ? hi : __float2bfloat16(v - __bfloat162float(hi));
            memcpy(dst + tc::sw128_offset(nl, k / 8) + (k % 8) * 2, &o, 2);
          }
      }
  // copy on the context's (non-blocking) stream and wait: a plain cudaMemcpy from pageable memory may return before
  // the DMA has landed and is not ordered against kernels on a non-blocking stream
  if (out.ensure(img.size())) return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(out.as<uint8_t>(), img.data(), img.size(), cudaMemcpyHostToDevice, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

// returns the number of K splits used (>= 1); when > 1 the caller reduces `ws` (splits x M x N) afterwards
int launch_conv_tc(disn_ctx* c, const float* A, const uint8_t* wpk, const float* bias, float* C, float* ws,
                   int64_t ws_elems, int M, int N, int K, int H, int W, int Cin, int relu, int* splits_out) {
  DISN_REQUIRE(K % 64 == 0 && N % 32 == 0 && (H == 0 || Cin % 64 == 0), "conv_tc: K%64, N%32, Cin%64");
  const int smem = (int)sizeof(ConvTcSmem) + 1024;
  if (!c->attr_conv_tc) {    // per context (= per device): the attribute is a property of the function ON a device
    DISN_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    c->attr_conv_tc = true;
  }
  const int sms = c->num_sms;
  ConvTcJob job{};
  job.A = A; job.wpk = wpk; job.bias = bias; job.C = C; job.M = M; job.N = N; job.K = K;
  job.H = H; job.W = W; job.Cin = Cin; job.relu = relu;
  job.m_tiles = (M + 127) / 128;
  job.n_blocks = (N + 127) / 128;
  const int slices = K / 64;
  int splits = 1;
  const int tiles = job.m_tiles * job.n_blocks;
  if (tiles < sms) {                     // under-filled: split K so that ~2 waves of jobs exist
    int want = (2 * sms + tiles - 1) / tiles;
    for (int d = std::min(want, slices); d >= 1; --d)
      if (slices % d == 0 && (int64_t)d * M * N <= ws_elems) { splits = d; break; }
  }
  job.splits = splits;
  job.slices_per_split = slices / splits;
  job.ws = splits > 1 ? ws : nullptr;
  const int total = tiles * splits;
  const int grid = std::min(total, sms);
  conv_tc_kernel<<<grid, CT_THREADS, smem, c->stream>>>(job);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  *splits_out = splits;
  return 0;
}

}  // namespace disn
