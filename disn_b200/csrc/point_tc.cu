// Fused per-point SDF kernel on Hopper tensor cores (warpgroup MMA; DISN_PREC_BF16X3 / DISN_PREC_F16F8), sm_90a.
//
// Same math as point_fp32.cu (projection -> gather of the folded feature map -> two point-MLP streams
// -> sum; models/model_normalization.py:241-251,169-206, models/sdfnet.py:69-92,171-190), but the four
// wide layers of each stream run on the tensor cores.  To hold the reference's 1e-4 bar the fp32 operands
// are split (template parameter kMode, DESIGN.md section 3):
//   MODE_BF16X3  x = hi + lo (two bf16), each product = 3 bf16 MMAs (hi*hi + lo*hi + hi*lo), error ~2^-17;
//   MODE_F16F8   fp16 main product + e5m2 first-order correction products (K = 32 per instruction, twice the fp16
//                rate).  Hopper's e5m2 MMAs keep only ~14 bits when they add into a large accumulator, so the
//                corrections of each K slice go to a zero-initialised second accumulator that is added to the main
//                one in fp32 on the CUDA cores.
//
// Organisation (one CTA per SM, persistent over tiles of 64 query points):
//   * two consumer warpgroups; warpgroup h computes output features [128h, 128h + 128) of every 256-wide N block of a
//     layer as wgmma m64n128 (M = the tile's 64 points), fp32 accumulators in registers (two N blocks for the
//     512-wide layers);
//   * activations never leave the SM: a layer's input (64 points x up to 512 features) sits in shared memory as
//     K-major 128-byte-swizzled operand tiles (bf16 hi | lo, or fp16 | e5m2 residual | e5m2 copy); when both warpgroups
//     are done with a layer the epilogue (bias / folded image features, ReLU, operand split) overwrites it in place
//     with the next layer's input;  fold1/conv1 (3 -> 64) and fold2/conv5 (256 -> 1) run on the CUDA cores;
//   * weights are pre-split and pre-swizzled on the host into the exact shared-memory images of the B operand
//     (32 KB per 128 output features x 64 k), packed in consumption order and streamed by the bulk-copy engine
//     (cp.async.bulk) through a 3-slot mbarrier ring.  Half-stages alternate between the two warpgroups, so each
//     (slot, warpgroup) has its own "landed" and "empty" barrier and every barrier phase has one waiter.  A consumer
//     warpgroup issues all MMAs of a half-stage as one commit group and waits for it once; each of its warps then
//     arrives on the slot's empty barrier.  A third, producer warpgroup refills the ring: one of its threads waits for
//     each slot's release and issues the next half-stage's bulk copy, in half-stage order, so the refill is off the
//     consumers' path from one MMA group to the next.  The register file is split with setmaxnreg: the producer
//     warpgroup gives back all but 24 registers per thread and the consumers rise to 240 (launched at 168);
//   * the small per-stream parameters (biases, fold1/conv1, fold2/conv5) are read from global memory through the
//     read-only cache: the lanes of a warp read different features, and the constant bank would serialise them.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "common.cuh"
#include "point_tc_layout.cuh"
#include "tc_common.cuh"

namespace disn {
namespace {

constexpr int PTS = 64;               // points per tile (the wgmma M)
constexpr int NCONS = 256;            // two consumer warpgroups: threads [0, 256)
constexpr int NTHREADS = NCONS + 128; // and the producer warpgroup: threads [256, 384)
// registers per thread after the roles split (setmaxnreg); launched at 65536 / 384 rounded down to 8, i.e. 168
constexpr int REG_PRODUCER = 24;
constexpr int REG_CONSUMER = 240;
static_assert(128 * REG_PRODUCER + NCONS * REG_CONSUMER <= 65536, "register split exceeds the register file");
constexpr int NSLOT = 3;              // weight ring slots
constexpr int W_TILE = 16384;         // 128 rows x 64 k x 2 B (SW128)
constexpr int W8_TILE = 8192;         // 128 rows x 64 k x 1 B (SW64)
constexpr int HS_BYTES = 2 * W_TILE;  // half-stage: [W_hi | W_lo] or [fp16 W | e5m2 W | e5m2 residual of W]
using ptc::X_TILE;                     // 64 rows x 64 k x 2 B (SW128)
using ptc::X8_TILE;                    // 64 rows x 64 k x 1 B (SW64)
using ptc::X_SLICE;                    // one 64-wide K slice: [hi | lo] or [fp16 | e5m2 residual | e5m2 copy]
constexpr int STAGES_PER_STREAM = 33; // 1 + 8 + 16 + 8 (K slice, 256-wide N block) stages
constexpr int HS_PER_TILE = 2 * 2 * STAGES_PER_STREAM;
// correction products DISN_PREC_F16F8 keeps in each tensor layer l = 0..3 (fold1/conv2, fold1/conv3, fold2/conv1,
// fold2/conv2): bit 2l (a - h(a)).w ("first"), bit 2l+1 a.(w - h(w)) ("second").  Every correction except the second
// product of fold2/conv1 (DESIGN.md section 3).
constexpr int CORR_DEFAULT = 0xDF;
__host__ __device__ constexpr int layer_k(int l) { return l == 0 ? 64 : (l == 1 ? 256 : 512); }
__host__ __device__ constexpr int layer_n(int l) { return (l == 1 || l == 2) ? 512 : 256; }
constexpr int kLayerPos[4] = {0, 1, 9, 25};   // first stage of each tensor layer within a stream

// operand-format modes of the kernel
constexpr int MODE_BF16X3 = 0;   // x = hi + lo (bf16): hi*hi + lo*hi + hi*lo, 12 MMAs per 64-wide K slice
constexpr int MODE_F16F8 = 1;    // fp16 main product + two e5m2 correction products:
                                 //   a.w ~= h(a).h(w) + e((a-h(a)).2^s1).e(w.2^-s1) + e(a.2^-s2).e((w-h(w)).2^s2), 4 + 2 + 2 MMAs

struct TcSmem {
  alignas(1024) uint8_t w[NSLOT][HS_BYTES];     // weight ring                                  96 KB
  alignas(1024) uint8_t x[8][X_SLICE];          // activations of the current layer's input   128 KB
};

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// bilinear taps of point n into the projected feature map (element offsets, -1 = outside; weights 0 there)
__device__ __forceinline__ void taps_of(const PointJob& job, int b, int64_t n, int (&off)[4], float (&wg)[4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) { off[k] = -1; wg[k] = 0.f; }
  if (n >= job.N) return;
  if (job.pfeat) {        // explicit per-point features: one "tap" of weight 1 at this point's row of pfeat
    off[0] = (int)(((int64_t)b * job.N + n) * kHidden);
    wg[0] = 1.f;
    return;
  }
  float x, y, z, xr, yr, zr, u, v;
  point_of(job, b, n, x, y, z, xr, yr, zr);
  project(job.trans_mat + b * 12, job.clamp_max, x, y, z, u, v);
  const int Wm = job.img_w, Hm = job.img_h;
  if (u > -1.f && v > -1.f && u < (float)Wm && v < (float)Hm) {
    const int fx = (int)floorf(u), fy = (int)floorf(v);
    const int cx = fx + 1, cy = fy + 1;
    const float dx = (float)cx - u, dy = (float)cy - v;
    const int tx[4] = {fx, cx, fx, cx}, ty[4] = {fy, cy, cy, fy};
    const float ww[4] = {dx * dy, (1.f - dx) * (1.f - dy), dx * (1.f - dy), (1.f - dx) * dy};
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (tx[k] >= 0 && tx[k] < Wm && ty[k] >= 0 && ty[k] < Hm) {
        off[k] = (ty[k] * Wm + tx[k]) * kHidden;
        wg[k] = ww[k];
      }
  }
}

static_assert(ptc::store_offset_mismatches() == 0, "epilogue / prologue store offsets disagree with the swizzled layout");

// write activations (a, b) of two adjacent features of one point into the activation buffer `x` in the operand format
// of kMode: the 2-byte pair at byte offset o16 (ptc::epi_off16 / pro_off16), MODE_F16F8's e5m2 pairs at o8
// (ptc::epi_off8 / pro_off8).  MODE_F16F8 also folds the fp16 values into `amax` (all values are post-ReLU, i.e. >= 0):
// an activation above fp16's 65504 becomes +inf there, which the kernel reports through PointJob::status instead of
// producing a silent inf.  `copy`: MODE_F16F8 also stores the e5m2 copy, which only the consuming layer's second
// correction product reads (a compile-time constant after inlining).
template <int kMode>
__device__ __forceinline__ void store_pair(uint8_t* x, uint32_t o16, uint32_t o8, float a, float b, float sc_lo,
                                           float sc_hi, __half2& amax, bool copy) {
  if constexpr (kMode == MODE_BF16X3) {
    uint32_t hi, lo;
    tc::split_bf16x2(a, b, hi, lo);
    *reinterpret_cast<uint32_t*>(x + o16) = hi;
    *reinterpret_cast<uint32_t*>(x + o16 + X_TILE) = lo;
  } else {
    const __half2 hh = __floats2half2_rn(a, b);
    amax = __hmax2(amax, hh);
    *reinterpret_cast<__half2*>(x + o16) = hh;
    const float ra = a - __low2float(hh), rb = b - __high2float(hh);      // fp16 rounding residual (first correction)
    const __nv_fp8x2_storage_t l = __nv_cvt_float2_to_fp8x2(make_float2(ra * sc_lo, rb * sc_lo), __NV_SATFINITE, __NV_E5M2);
    *reinterpret_cast<__nv_fp8x2_storage_t*>(x + o8) = l;
    if (copy) {
      const __half2 hs = __hmul2(hh, __float2half2_rn(sc_hi));   // power-of-two scale: exact up to fp16 underflow
      const __nv_fp8x2_storage_t g =
          __nv_cvt_halfraw2_to_fp8x2(*reinterpret_cast<const __half2_raw*>(&hs), __NV_SATFINITE, __NV_E5M2);
      *reinterpret_cast<__nv_fp8x2_storage_t*>(x + o8 + X8_TILE) = g;
    }
  }
}

// the consumers hold two 64-register accumulators (plus the 64-register correction accumulator of MODE_F16F8)
template <int kMode>
__global__ void __launch_bounds__(NTHREADS, 1)
point_tc_kernel(PointJob job, const uint8_t* __restrict__ wpk,
                 int64_t tiles_per_img) {
  extern __shared__ uint8_t smem_raw[];
  TcSmem& s = *reinterpret_cast<TcSmem*>(smem_raw + ((1024u - (tc::smem_u32(smem_raw) & 1023u)) & 1023u));
  __shared__ float part[2][2][PTS];            // fold2/conv5 partial sums [stream][warpgroup][point]
  __shared__ alignas(8) uint64_t full[NSLOT][2];   // [slot][consuming warpgroup]: half-stage landed
  __shared__ alignas(8) uint64_t empty[NSLOT][2];  // [slot][consuming warpgroup]: its four warps are done reading it
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int kC = (kMode == MODE_F16F8) ? CORR_DEFAULT : 0;
  const int64_t total_tiles = tiles_per_img * job.B;
  const int my_tiles =
      ((int64_t)blockIdx.x < total_tiles) ? (int)((total_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x) : 0;

  if (tid == 0) {
    for (int i = 0; i < NSLOT; ++i) {
      tc::mbar_init(&full[i][0], 1);
      tc::mbar_init(&full[i][1], 1);
      tc::mbar_init(&empty[i][0], 4);
      tc::mbar_init(&empty[i][1], 4);
    }
    tc::fence_barrier_init();
  }
  __syncthreads();

  // ===================== producer =====================
  if (tid >= NCONS) {
    tc::setmaxnreg_dec<REG_PRODUCER>();
    if (tid == NCONS) {
      // half-stage g -> slot g % NSLOT, consumed by warpgroup g & 1.  It reuses the slot of half-stage q = g - NSLOT,
      // which warpgroup q & 1 releases on empty[q % NSLOT][q & 1]: that (slot, warpgroup) pair's use number q / 6.
      const uint32_t total_hs = (uint32_t)my_tiles * HS_PER_TILE;
      for (uint32_t g = 0; g < total_hs; ++g) {
        const uint32_t slot = g % NSLOT;
        if (g >= NSLOT) {
          const uint32_t q = g - NSLOT;
          tc::mbar_wait_inline(&empty[slot][q & 1], (q / (2 * NSLOT)) & 1u);
        }
        tc::mbar_arrive_expect_tx(&full[slot][g & 1], HS_BYTES);
        tc::bulk_g2s(s.w[slot], wpk + (size_t)(g % HS_PER_TILE) * HS_BYTES, HS_BYTES, &full[slot][g & 1]);
      }
    }
    return;
  }

  // ===================== consumers (threads [0, NCONS): tid is the consumer thread index) =====================
  tc::setmaxnreg_inc<REG_CONSUMER>();
  const int h = warp >> 2;                       // warpgroup: output features [128h, 128h + 128) of each N block
  const int wi = warp & 3;
  const int r0 = wi * 16 + (lane >> 2);          // accumulator rows r0, r0 + 8
  const int cq = (lane & 3) * 2;                 // accumulator column offset within each 8-column group
  const uint32_t x_base = tc::smem_u32(s.x[0]), w_base = tc::smem_u32(s.w[0]);
  uint32_t g = (uint32_t)h;                      // this warpgroup's half-stages: h, h + 2, ...
  uint32_t ph = 0;                               // phase bit per slot of full[slot][h]
  __half2 amax = __float2half2_rn(0.f);          // running maximum of this thread's fp16 A-operand values (MODE_F16F8)
  float acc[2][64];
  float tmp[64];                                 // MODE_F16F8: corrections of one half-stage

  for (int it = 0; it < my_tiles; ++it) {
    const int64_t tile = (int64_t)blockIdx.x + (int64_t)it * gridDim.x;
    const int b = (int)(tile / tiles_per_img);
    const int64_t n0 = (tile % tiles_per_img) * PTS;
#pragma unroll(kMode == MODE_F16F8 ? 2 : 1)
    for (int sx = 0; sx < 2; ++sx) {
      // ---- fold1/conv1 (3 -> 64, fp32 FMA) into K slice 0: thread -> point tid / 4, features 16 (tid % 4) + [0, 16)
      named_bar_sync(1, NCONS);                  // the previous layer's MMAs are done with the activation buffer
      {
        const int p = tid >> 2, f0 = (tid & 3) * 16;
        const int64_t n = n0 + p;
        float x, y, z, xr, yr, zr;
        point_of(job, b, n, x, y, z, xr, yr, zr);
        if (sx == 0 && (tid & 3) == 0 && job.out_uv && n < job.N) {
          float u, v;
          project(job.trans_mat + b * 12, job.clamp_max, x, y, z, u, v);
          float* o = job.out_uv + ((int64_t)b * job.N + n) * 2;
          o[0] = u; o[1] = v;
        }
        const StreamWeights& sw = sx ? job.l : job.g;
        const float* b1p = sw.b1 + f0;
        const float* w1p = sw.w1 + f0;
        const uint32_t o16 = ptc::pro_base16((uint32_t)p, (uint32_t)(tid & 3));
        const uint32_t o8 = ptc::pro_base8((uint32_t)p, (uint32_t)(tid & 3));
#pragma unroll
        for (int j = 0; j < 16; j += 2) {
          const float2 b1 = __ldg(reinterpret_cast<const float2*>(b1p + j));
          const float2 wx = __ldg(reinterpret_cast<const float2*>(w1p + j));
          const float2 wy = __ldg(reinterpret_cast<const float2*>(w1p + 64 + j));
          const float2 wz = __ldg(reinterpret_cast<const float2*>(w1p + 128 + j));
          float v2[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float a = e ? b1.y : b1.x;
            a = fmaf(xr, e ? wx.y : wx.x, a);
            a = fmaf(yr, e ? wy.y : wy.x, a);
            a = fmaf(zr, e ? wz.y : wz.x, a);
            v2[e] = fmaxf(a, 0.f);
          }
          store_pair<kMode>(s.x[0], ptc::pro_off16(o16, j), ptc::pro_off8(o8, j), v2[0], v2[1], job.act_scale[sx][0][0],
                            job.act_scale[sx][0][1], amax, ((kC >> 1) & 1) != 0);
        }
      }
      tc::fence_proxy_async_smem();
      named_bar_sync(1, NCONS);

#pragma unroll
      for (int layer = 0; layer < 4; ++layer) {
        const int nsl = layer_k(layer) / 64, nnb = layer_n(layer) / 256;
        const bool k1 = ((kC >> (2 * layer)) & 1) != 0, k2 = ((kC >> (2 * layer + 1)) & 1) != 0;
#pragma unroll 1
        for (int t = 0; t < nsl; ++t) {
#pragma unroll
          for (int nb = 0; nb < 2; ++nb) {
            if (nb >= nnb) continue;
            const uint32_t slot = g % NSLOT, par = (ph >> slot) & 1u;
            tc::mbar_wait(&full[slot][h], par);
            ph ^= 1u << slot;
            // descriptor low words of the slice's A tile and the slot's B tile; every other operand of the half-stage is
            // a constant number of 16-byte units (>> 4) further (tc::desc_lo)
            const uint32_t xa = tc::desc_lo(x_base + (uint32_t)t * X_SLICE), wb = tc::desc_lo(w_base + slot * HS_BYTES);
            tc::acc_fence(acc[nb]);
            if constexpr (kMode == MODE_F16F8) tc::acc_fence(tmp);
            tc::wgmma_fence();
            if constexpr (kMode == MODE_BF16X3) {
#pragma unroll
              for (int k = 0; k < 4; ++k)
                tc::wgmma_m64n128_lo<tc::KIND_BF16>(acc[nb], xa + 2u * k, wb + 2u * k, (t | k) ? 1u : 0u);
#pragma unroll
              for (int k = 0; k < 4; ++k)
                tc::wgmma_m64n128_lo<tc::KIND_BF16>(acc[nb], xa + (X_TILE >> 4) + 2u * k, wb + 2u * k, 1u);
#pragma unroll
              for (int k = 0; k < 4; ++k)
                tc::wgmma_m64n128_lo<tc::KIND_BF16>(acc[nb], xa + 2u * k, wb + (W_TILE >> 4) + 2u * k, 1u);
            } else {
#pragma unroll
              for (int k = 0; k < 4; ++k)
                tc::wgmma_m64n128_lo<tc::KIND_F16>(acc[nb], xa + 2u * k, wb + 2u * k, (t | k) ? 1u : 0u);
              // corrections into the zero-initialised side accumulator, in the same commit group; they are added after
              // the wait, so each element still gets main(t), then + corr(t), then main(t + 1)
              if (k1) {
#pragma unroll
                for (int k = 0; k < 2; ++k)
                  tc::wgmma_m64n128_lo<tc::KIND_E5M2>(tmp, xa + (X_TILE >> 4) + 2u * k, wb + (W_TILE >> 4) + 2u * k,
                                                      k ? 1u : 0u);
              }
              if (k2) {
#pragma unroll
                for (int k = 0; k < 2; ++k)
                  tc::wgmma_m64n128_lo<tc::KIND_E5M2>(tmp, xa + ((X_TILE + X8_TILE) >> 4) + 2u * k,
                                                      wb + ((W_TILE + W8_TILE) >> 4) + 2u * k, (k1 || k) ? 1u : 0u);
              }
            }
            tc::wgmma_commit();
            tc::wgmma_wait<0>();
            tc::acc_fence(acc[nb]);
            // this warp is done with the slot; the producer refills it once all four warps are
            if (lane == 0) tc::mbar_arrive(&empty[slot][h]);
            if constexpr (kMode == MODE_F16F8) {
              if (k1 || k2) {
                tc::acc_fence(tmp);
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[nb][i] += tmp[i];
              }
            }
            g += 2;
          }
        }
        named_bar_sync(1, NCONS);                // both warpgroups are done reading this layer's input
        if (layer < 3) {
          // ---- epilogue: bias (+ folded image features), ReLU, operand split -> next layer's input, in place
          const bool gather = (sx == 1 && layer == 2);
          // the next layer reads the e5m2 copy only if it keeps the second correction (not fold2/conv1 by default)
          const bool copy = ((kC >> (2 * layer + 3)) & 1) != 0;
          int off[2][4];
          float wg[2][4];
          if (gather) {
            taps_of(job, b, n0 + r0, off[0], wg[0]);
            taps_of(job, b, n0 + r0 + 8, off[1], wg[1]);
          } else {   // layer 2 of the global stream loads the taps too (see below), and drops them
#pragma unroll
            for (int k = 0; k < 8; ++k) { off[k >> 2][k & 3] = -1; wg[k >> 2][k & 3] = 0.f; }
          }
          const StreamWeights& sw = sx ? job.l : job.g;
          const float* bias_v = layer == 0 ? sw.b2 : (layer == 1 ? sw.b3 : (sx == 0 ? job.gbias + (int64_t)b * kHidden : sw.b4));
          const float sc_lo = job.act_scale[sx][layer + 1][0], sc_hi = job.act_scale[sx][layer + 1][1];
          // Every address of the epilogue is a per-thread base plus an immediate: the parameter and tap pointers point
          // at this thread's first column (feature 128h + cq), the store bases hold its row's swizzle pattern
          // (point_tc_layout.cuh), and N block, column group and row half are offsets from them.
          // MODE_F16F8: the thread's row and column are made opaque here so that the bases are formed in place: the
          // compiler would otherwise hoist them out of the tile loop and keep them live across the MMA loops next to
          // the main and side accumulators, where they spill.  MODE_BF16X3 has the registers to keep them.
          int row = r0, cbase = h * 128 + cq;
          if constexpr (kMode == MODE_F16F8) asm volatile("" : "+r"(row), "+r"(cbase));
          const uint32_t base16 = ptc::epi_base16((uint32_t)cbase >> 7, (uint32_t)row, (uint32_t)cbase & 127u);
          const uint32_t base8 = ptc::epi_base8((uint32_t)cbase >> 7, (uint32_t)row, (uint32_t)cbase & 127u);
          const float* bp = bias_v + cbase;
          // the four taps of rows r0 and r0 + 8 (an outside tap reads the first row of the map with weight 0)
          const float* pm = (job.pfeat ? job.pfeat : job.pmap + (int64_t)b * job.img_h * job.img_w * kHidden) + cbase;
          const float* tp[2][4];
#pragma unroll
          for (int k = 0; k < 8; ++k) tp[k >> 2][k & 3] = pm + max(off[k >> 2][k & 3], 0);
#pragma unroll
          for (int nb = 0; nb < 2; ++nb) {
            if (nb >= nnb) continue;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const float2 bb = __ldg(reinterpret_cast<const float2*>(bp + nb * 256 + 8 * j));
              const float bias[2] = {bb.x, bb.y};
#pragma unroll
              for (int e2 = 0; e2 < 2; ++e2) {
                float v2[2] = {bias[0], bias[1]};
                // only the local stream adds the gather.  MODE_F16F8 compiles each stream's epilogues apart (the stream
                // loop is unrolled), so `gather` is a constant there and the global stream issues no tap loads.
                // MODE_BF16X3 shares layer 2's code between the streams (unrolled, it spills inside its epilogues):
                // its tap loads stay unconditional (every address is valid) so that the compiler can issue them ahead
                // across j; a branch around them per j serialised their L2 round trips.
                if (layer == 2 && (gather || kMode == MODE_BF16X3)) {
                  float2 a = make_float2(0.f, 0.f);
#pragma unroll
                  for (int k = 0; k < 4; ++k) {
                    const float2 m = __ldg(reinterpret_cast<const float2*>(tp[e2][k] + nb * 256 + 8 * j));
                    a.x = fmaf(wg[e2][k], m.x, a.x);
                    a.y = fmaf(wg[e2][k], m.y, a.y);
                  }
                  if (gather) {
                    v2[0] += a.x;
                    v2[1] += a.y;
                  }
                }
                const float va = fmaxf(acc[nb][4 * j + 2 * e2] + v2[0], 0.f);
                const float vb = fmaxf(acc[nb][4 * j + 2 * e2 + 1] + v2[1], 0.f);
                store_pair<kMode>(s.x[0], ptc::epi_off16(base16, nb, j, e2), ptc::epi_off8(base8, nb, j, e2), va, vb,
                                  sc_lo, sc_hi, amax, copy);
              }
            }
          }
          tc::fence_proxy_async_smem();
          named_bar_sync(1, NCONS);
        } else {
          // ---- fold2/conv2 output (256) -> ReLU -> fold2/conv5 dot product
          float pr[2] = {0.f, 0.f};
          const StreamWeights& sw = sx ? job.l : job.g;
          const float* b5p = sw.b5 + (h * 128 + cq);
          const float* w6p = sw.w6 + (h * 128 + cq);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const float2 b5 = __ldg(reinterpret_cast<const float2*>(b5p + 8 * j));
            const float2 w6 = __ldg(reinterpret_cast<const float2*>(w6p + 8 * j));
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float a = fmaxf(acc[0][4 * j + e] + ((e & 1) ? b5.y : b5.x), 0.f);
              pr[e >> 1] = fmaf(a, (e & 1) ? w6.y : w6.x, pr[e >> 1]);
            }
          }
#pragma unroll
          for (int e2 = 0; e2 < 2; ++e2) {
            pr[e2] += __shfl_xor_sync(0xffffffffu, pr[e2], 1);
            pr[e2] += __shfl_xor_sync(0xffffffffu, pr[e2], 2);
          }
          if ((lane & 3) == 0) {
            part[sx][h][r0] = pr[0];
            part[sx][h][r0 + 8] = pr[1];
          }
        }
      }
    }
    named_bar_sync(1, NCONS);
    if (tid < PTS) {
      const int64_t n = n0 + tid;
      if (n < job.N) {
        const float rg = (part[0][0][tid] + part[0][1][tid]) + __ldg(job.g.b6);
        const float rl = (part[1][0][tid] + part[1][1][tid]) + __ldg(job.l.b6);
        if (job.out_global) job.out_global[(int64_t)b * job.N + n] = rg;
        if (job.out_local) job.out_local[(int64_t)b * job.N + n] = rl;
        float r = rg + rl;
        if (job.tanh_out) r = tanhf(r);
        job.out_pred[(int64_t)b * job.N + n] = __fdiv_rn(r, job.out_div);
      }
    }
  }
  if constexpr (kMode == MODE_F16F8) {
    // fp16 range guard: +inf here means an activation exceeded 65504 and the result is meaningless
    if ((__hisinf(__low2half(amax)) || __hisinf(__high2half(amax))) && job.status) atomicOr(job.status, DISN_STATUS_FP16_OVERFLOW);
  }
}

template <int kMode>
int launch_var(disn_ctx* c, const PointJob& job, const void* wpk, int grid, int smem,
               int64_t tiles_per_img) {
  // the attribute belongs to (function, device): set per context, not per process (a second engine on another device
  // in the same process would otherwise launch with the 48 KB default)
  auto key = (const void*)point_tc_kernel<kMode>;
  if (!c->attr_done.count(key)) {
    DISN_CUDA_OK(cudaFuncSetAttribute(point_tc_kernel<kMode>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    c->attr_done.insert(key);
  }
  point_tc_kernel<kMode><<<grid, NTHREADS, smem, c->stream>>>(job, reinterpret_cast<const uint8_t*>(wpk), tiles_per_img);
  return 0;
}

}  // namespace

// Pack both streams' tensor-core layers into the kernel's B-operand half-stage images, in consumption order:
//   stream, layer, K slice t, 256-wide N block nb, half h (output features nb*256 + 128h + [0,128)), 32 KB each:
//   DISN_PREC_BF16X3  [hi | lo] 16 KB bf16 SW128 tiles [128 rows n][64 k];
//   DISN_PREC_F16F8   [fp16 W, SW128, 16 KB | e5m2(w.2^-s1), SW64, 8 KB | e5m2((w - fp16(w)).2^s2), SW64, 8 KB].
//   The exponents follow the layer's weight rms (2^L) so that the e5m2 operands (normal range 2^-14 .. 2^15,
//   2 mantissa bits) sit mid-range for O(1) activations: s1 = 10 + L, s2 = 12 + L; the matching activation
//   multipliers 2^s1 and 2^-s2 go to the kernel.
int tc_pack_weights(disn_ctx* c) {
  const size_t total = (size_t)HS_PER_TILE * HS_BYTES;
  std::vector<uint8_t> img(total, 0), img8(total, 0);
  size_t stage = 0;
  for (int sidx = 0; sidx < 2; ++sidx) {
    const std::string p = sidx ? "sdfprediction_imgfeat" : "sdfprediction";
    const char* names[4] = {"/fold1/conv2/weights", "/fold1/conv3/weights", "/fold2/conv1/weights", "/fold2/conv2/weights"};
    for (int layer = 0; layer < 4; ++layer) {
      auto it = c->weights.find(p + names[layer]);
      DISN_REQUIRE(it != c->weights.end(), "missing variable " + p + names[layer]);
      const int K = layer_k(layer), N = layer_n(layer);
      std::vector<float> w((size_t)K * N);   // rows 0..K-1 of the [Cin,Cout] matrix (point-feature part)
      DISN_CUDA_OK(cudaMemcpyAsync(w.data(), it->second.ptr(), w.size() * sizeof(float), cudaMemcpyDeviceToHost,
                                   c->stream));
      DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
      double ss = 0;
      for (float v : w) ss += (double)v * v;
      const double rms = std::sqrt(ss / (double)w.size());
      const int L = rms > 0 ? (int)std::lround(std::log2(rms)) : -4;
      const int s1 = std::min(24, std::max(-8, 10 + L)), s2 = std::min(28, std::max(-8, 12 + L));
      c->tc_act_scale[sidx][layer][0] = std::ldexp(1.f, s1);
      c->tc_act_scale[sidx][layer][1] = std::ldexp(1.f, -s2);
      for (int t = 0; t < K / 64; ++t)
        for (int nb = 0; nb < N / 256; ++nb, ++stage)
          for (int half = 0; half < 2; ++half) {
            const size_t pos = (size_t)sidx * STAGES_PER_STREAM + kLayerPos[layer] + (size_t)(t * (N / 256) + nb);
            uint8_t* dst = img.data() + (2 * pos + half) * HS_BYTES;
            uint8_t* dst8 = img8.data() + (2 * pos + half) * HS_BYTES;
            for (int nl = 0; nl < 128; ++nl) {
              const int n = nb * 256 + half * 128 + nl;
              for (int k = 0; k < 64; ++k) {
                const float v = w[(size_t)(t * 64 + k) * N + n];
                const uint32_t o16 = tc::sw128_offset(nl, k / 8) + (k % 8) * 2;
                const __nv_bfloat16 hi = __float2bfloat16(v);
                const __nv_bfloat16 lo = __float2bfloat16(v - __bfloat162float(hi));
                memcpy(dst + o16, &hi, 2);
                memcpy(dst + W_TILE + o16, &lo, 2);
                const __half hv = __float2half_rn(v);
                memcpy(dst8 + o16, &hv, 2);
                const uint32_t o8 = tc::sw64_offset(nl, k / 16) + (k % 16);
                dst8[W_TILE + o8] = (uint8_t)__nv_cvt_float_to_fp8(std::ldexp(v, -s1), __NV_SATFINITE, __NV_E5M2);
                dst8[W_TILE + W8_TILE + o8] =
                    (uint8_t)__nv_cvt_float_to_fp8(std::ldexp(v - __half2float(hv), s2), __NV_SATFINITE, __NV_E5M2);
              }
            }
          }
    }
  }
  DISN_REQUIRE(stage == (size_t)2 * STAGES_PER_STREAM, "internal: stage count");
  if (c->tc_weights.ensure(total) || c->tc_weights_f8.ensure(total)) return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(c->tc_weights.as<void>(), img.data(), total, cudaMemcpyHostToDevice, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(c->tc_weights_f8.as<void>(), img8.data(), total, cudaMemcpyHostToDevice, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));   // ordered on the ctx stream (see conv_tc_pack)
  return 0;
}

int launch_point_tc(disn_ctx* c, const PointJob& job_in) {
  const bool f8 = c->cfg.precision == DISN_PREC_F16F8;
  const void* wpk = (f8 ? c->tc_weights_f8 : c->tc_weights).as<void>();
  DISN_REQUIRE(wpk != nullptr, "tensor-core weights not packed (call disn_finalize_weights)");
  PointJob job = job_in;
  memcpy(job.act_scale, c->tc_act_scale, sizeof(job.act_scale));
  const int smem = (int)sizeof(TcSmem) + 1024;
  const int64_t tiles_per_img = (job.N + PTS - 1) / PTS;
  const int64_t total = tiles_per_img * job.B;
  if (total == 0) return 0;
  const int grid = (int)std::min<int64_t>(total, c->num_sms);
  const int rc = f8 ? launch_var<MODE_F16F8>(c, job, wpk, grid, smem, tiles_per_img)
                    : launch_var<MODE_BF16X3>(c, job, wpk, grid, smem, tiles_per_img);
  if (rc) return rc;
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace disn
