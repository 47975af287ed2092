// Fused per-point SDF kernel, fp32 CUDA-core arithmetic (DISN_PREC_FP32): the exact-precision anchor
// of the hot path.  One persistent CTA per SM walks 32-point tiles; for each tile it
//   1. generates / loads the query points (grid mode reproduces test/create_sdf.py:246-255),
//   2. projects them through trans_mat and clamps to [0,clamp_max]  (models/model_normalization.py:241-251),
//   3. runs both point-MLP streams (models/sdfnet.py:69-92, :171-190) with activations resident in
//      shared memory and weights streamed from L2 through a cp.async double buffer; the global embedding
//      enters as the per-image bias `gbias`, the five resampled VGG taps as a 4-tap bilinear gather of the
//      pre-projected 512-channel map `pmap` (tf.contrib.resampler semantics, SURVEY.md Appendix A),
//   4. sums the streams, applies the optional tanh / output scale, and stores 4 bytes per point.
#include "common.cuh"

namespace disn {

namespace {

constexpr int TP = 32;          // points per tile
constexpr int NTHREADS = 256;
constexpr int KC = 16;          // weight rows per cp.async stage
constexpr int ACT_LD = TP;      // activations stored [feature][point]

struct Smem {
  float act0[512 * ACT_LD];     // 64 KB
  float act1[512 * ACT_LD];     // 64 KB
  float wt[2][KC * 512];        // 64 KB
  float px[TP], py[TP], pz[TP]; // MLP input coordinates
  float u[TP], v[TP];           // projected pixel coordinates
  float pred[TP];               // global-stream result
};

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// stage `rows` x N floats of W (row-major [K][N]) starting at row k0 into wt[buf]
template <int N>
__device__ __forceinline__ void stage_weights(float* dst, const float* __restrict__ W, int k0, int K) {
  constexpr int VEC_PER_ROW = N / 4;
  constexpr int TOTAL = KC * VEC_PER_ROW;
  for (int i = threadIdx.x; i < TOTAL; i += NTHREADS) {
    int r = i / VEC_PER_ROW, cvec = i % VEC_PER_ROW;
    if (k0 + r < K) cp_async16(dst + r * N + cvec * 4, W + (int64_t)(k0 + r) * N + cvec * 4);
  }
}

// Dense layer on the tile: out[N][TP] = act( in[K][TP]^T * W[K][N] + init ),  N in {256, 512}.
// Thread tile: PT points x 8 features (features f0..f0+3 and N/2+f0..N/2+f0+3).
// `init(f, ptbase, acc)` seeds the accumulators (bias, folded global bias, or bias + gathered features).
template <int K, int N, bool RELU, class Init>
__device__ __forceinline__ void dense_layer(Smem& s, const float* __restrict__ in, float* __restrict__ out,
                                            const float* __restrict__ W, Init init) {
  constexpr int FG = N / 8;                 // feature groups: 64 (N=512) or 32 (N=256)
  constexpr int PG = NTHREADS / FG;         // point groups: 4 or 8
  constexpr int PT = TP / PG;               // points per thread: 8 or 4
  const int fg = threadIdx.x % FG, pg = threadIdx.x / FG;
  const int f0 = fg * 4, p0 = pg * PT;

  float acc[PT][8];
  init(f0, p0, acc);

  constexpr int NCHUNK = (K + KC - 1) / KC;
  stage_weights<N>(s.wt[0], W, 0, K);
  cp_async_commit();
  for (int ch = 0; ch < NCHUNK; ++ch) {
    if (ch + 1 < NCHUNK) stage_weights<N>(s.wt[(ch + 1) & 1], W, (ch + 1) * KC, K);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const float* wt = s.wt[ch & 1];
    static_assert(K % KC == 0, "layer widths are multiples of the weight stage depth");
#pragma unroll
    for (int kk = 0; kk < KC; ++kk) {
      {
        const int k = ch * KC + kk;
        float a[PT], w[8];
#pragma unroll
        for (int i = 0; i < PT; i += 4)
          *reinterpret_cast<float4*>(&a[i]) = *reinterpret_cast<const float4*>(in + k * ACT_LD + p0 + i);
        *reinterpret_cast<float4*>(&w[0]) = *reinterpret_cast<const float4*>(wt + kk * N + f0);
        *reinterpret_cast<float4*>(&w[4]) = *reinterpret_cast<const float4*>(wt + kk * N + N / 2 + f0);
#pragma unroll
        for (int i = 0; i < PT; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
      }
    }
    __syncthreads();
  }
  // write out[f][p]
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int f = (j < 4) ? (f0 + j) : (N / 2 + f0 + j - 4);
#pragma unroll
    for (int i = 0; i < PT; i += 4) {
      float4 o;
      o.x = RELU ? fmaxf(acc[i + 0][j], 0.f) : acc[i + 0][j];
      o.y = RELU ? fmaxf(acc[i + 1][j], 0.f) : acc[i + 1][j];
      o.z = RELU ? fmaxf(acc[i + 2][j], 0.f) : acc[i + 2][j];
      o.w = RELU ? fmaxf(acc[i + 3][j], 0.f) : acc[i + 3][j];
      *reinterpret_cast<float4*>(out + f * ACT_LD + p0 + i) = o;
    }
  }
  __syncthreads();
}

// one stream of the point MLP on the current tile; returns with s.act1[0..255][TP] = fold2/conv2 output
template <bool LOCAL>
__device__ __forceinline__ void run_stream(Smem& s, const PointJob& job, const StreamWeights& w, int b, int64_t n0) {
  // fold1/conv1: 3 -> 64 (ReLU), into act0[64][TP]
  for (int i = threadIdx.x; i < 64 * TP; i += NTHREADS) {
    int f = i / TP, p = i % TP;
    float v = w.b1[f];
    v = fmaf(s.px[p], w.w1[0 * 64 + f], v);
    v = fmaf(s.py[p], w.w1[1 * 64 + f], v);
    v = fmaf(s.pz[p], w.w1[2 * 64 + f], v);
    s.act0[f * ACT_LD + p] = fmaxf(v, 0.f);
  }
  __syncthreads();
  // fold1/conv2: 64 -> 256
  dense_layer<64, 256, true>(s, s.act0, s.act1, w.w2, [&](int f0, int p0, float (*acc)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float bv = w.b2[(j < 4) ? (f0 + j) : (128 + f0 + j - 4)];
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i][j] = bv;
    }
  });
  // fold1/conv3: 256 -> 512
  dense_layer<256, 512, true>(s, s.act1, s.act0, w.w3, [&](int f0, int p0, float (*acc)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float bv = w.b3[(j < 4) ? (f0 + j) : (256 + f0 + j - 4)];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i][j] = bv;
    }
  });
  // fold2/conv1: (512 point features | folded image features) -> 512
  dense_layer<512, 512, true>(s, s.act0, s.act1, w.w4, [&](int f0, int p0, float (*acc)[8]) {
    if (!LOCAL) {
      const float* gb = job.gbias + (int64_t)b * kHidden;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float bv = gb[(j < 4) ? (f0 + j) : (256 + f0 + j - 4)];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i][j] = bv;
      }
    } else {
      // bias + tf.contrib.resampler gather of the projected map (4 taps, zero outside the map)
      const int Wm = job.img_w, Hm = job.img_h;
      const float* pm = job.pmap + (int64_t)b * Hm * Wm * kHidden;
      float4 blo = *reinterpret_cast<const float4*>(w.b4 + f0);
      float4 bhi = *reinterpret_cast<const float4*>(w.b4 + 256 + f0);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float x = s.u[p0 + i], y = s.v[p0 + i];
        float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
        if (job.pfeat) {     // explicit per-point features (get_decoder): already folded through W[512:1984]
          const int64_t n = n0 + p0 + i;
          if (n < job.N) {
            const float* q = job.pfeat + ((int64_t)b * job.N + n) * kHidden;
            lo = __ldg(reinterpret_cast<const float4*>(q + f0));
            hi = __ldg(reinterpret_cast<const float4*>(q + 256 + f0));
          }
        } else if (x > -1.f && y > -1.f && x < (float)Wm && y < (float)Hm) {
          int fx = (int)floorf(x), fy = (int)floorf(y);
          int cx = fx + 1, cy = fy + 1;
          float dx = (float)cx - x, dy = (float)cy - y;
          float wgt[4] = {dx * dy, (1.f - dx) * (1.f - dy), dx * (1.f - dy), (1.f - dx) * dy};
          int tx[4] = {fx, cx, fx, cx}, ty[4] = {fy, cy, cy, fy};
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            if (tx[t] >= 0 && tx[t] < Wm && ty[t] >= 0 && ty[t] < Hm) {
              const float* q = pm + ((int64_t)ty[t] * Wm + tx[t]) * kHidden;
              float4 a = __ldg(reinterpret_cast<const float4*>(q + f0));
              float4 c = __ldg(reinterpret_cast<const float4*>(q + 256 + f0));
              lo.x = fmaf(wgt[t], a.x, lo.x); lo.y = fmaf(wgt[t], a.y, lo.y);
              lo.z = fmaf(wgt[t], a.z, lo.z); lo.w = fmaf(wgt[t], a.w, lo.w);
              hi.x = fmaf(wgt[t], c.x, hi.x); hi.y = fmaf(wgt[t], c.y, hi.y);
              hi.z = fmaf(wgt[t], c.z, hi.z); hi.w = fmaf(wgt[t], c.w, hi.w);
            }
          }
        }
        acc[i][0] = blo.x + lo.x; acc[i][1] = blo.y + lo.y; acc[i][2] = blo.z + lo.z; acc[i][3] = blo.w + lo.w;
        acc[i][4] = bhi.x + hi.x; acc[i][5] = bhi.y + hi.y; acc[i][6] = bhi.z + hi.z; acc[i][7] = bhi.w + hi.w;
      }
    }
  });
  // fold2/conv2: 512 -> 256
  dense_layer<512, 256, true>(s, s.act1, s.act0, w.w5, [&](int f0, int p0, float (*acc)[8]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float bv = w.b5[(j < 4) ? (f0 + j) : (128 + f0 + j - 4)];
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i][j] = bv;
    }
  });
}

__global__ void __launch_bounds__(NTHREADS, 1) point_fp32_kernel(PointJob job, int64_t tiles_per_img) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  const int64_t total_tiles = tiles_per_img * job.B;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;

  for (int64_t tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int b = (int)(tile / tiles_per_img);
    const int64_t n0 = (tile % tiles_per_img) * TP;
    // ---- points + projection -------------------------------------------------------------------
    if (threadIdx.x < TP) {
      const int p = threadIdx.x;
      const int64_t n = n0 + p;
      float x, y, z, xr, yr, zr, u, v;
      point_of(job, b, n, x, y, z, xr, yr, zr);
      project(job.trans_mat + b * 12, job.clamp_max, x, y, z, u, v);
      s.px[p] = xr; s.py[p] = yr; s.pz[p] = zr;
      s.u[p] = u; s.v[p] = v;
      if (job.out_uv && n < job.N) {
        float* o = job.out_uv + ((int64_t)b * job.N + n) * 2;
        o[0] = u; o[1] = v;
      }
    }
    __syncthreads();

    // ---- global stream ---------------------------------------------------------------------------
    run_stream<false>(s, job, job.g, b, n0);
    {  // fold2/conv5: 256 -> 1 (linear); warp w handles points w*4..w*4+3
      for (int pp = 0; pp < 4; ++pp) {
        int p = warp * 4 + pp;
        float sum = 0.f;
        for (int f = lane; f < 256; f += 32) sum = fmaf(s.act0[f * ACT_LD + p], job.g.w6[f], sum);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) s.pred[p] = sum + job.g.b6[0];
      }
    }
    __syncthreads();
    // ---- local stream -----------------------------------------------------------------------------
    run_stream<true>(s, job, job.l, b, n0);
    {
      for (int pp = 0; pp < 4; ++pp) {
        int p = warp * 4 + pp;
        float sum = 0.f;
        for (int f = lane; f < 256; f += 32) sum = fmaf(s.act0[f * ACT_LD + p], job.l.w6[f], sum);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) {
          const int64_t n = n0 + p;
          if (n < job.N) {
            const float rl = sum + job.l.b6[0];
            if (job.out_global) job.out_global[(int64_t)b * job.N + n] = s.pred[p];
            if (job.out_local) job.out_local[(int64_t)b * job.N + n] = rl;
            float r = s.pred[p] + rl;     // pred_sdf = global + local (:204)
            if (job.tanh_out) r = tanhf(r);
            job.out_pred[(int64_t)b * job.N + n] = __fdiv_rn(r, job.out_div);
          }
        }
      }
    }
    __syncthreads();
  }
}

}  // namespace

int launch_point_fp32(disn_ctx* c, const PointJob& job) {
  if (!c->attr_point_fp32) {   // per context (= per device)
    DISN_CUDA_OK(cudaFuncSetAttribute(point_fp32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)sizeof(Smem)));
    c->attr_point_fp32 = true;
  }
  int64_t tiles_per_img = (job.N + TP - 1) / TP;
  int64_t total = tiles_per_img * job.B;
  if (total == 0) return 0;
  int grid = (int)std::min<int64_t>(total, c->num_sms);
  point_fp32_kernel<<<grid, NTHREADS, sizeof(Smem), c->stream>>>(job, tiles_per_img);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace disn
