// Training of the SDF decoder with the encoder frozen (the reference's train/train_sdf.py with the default flags:
// --img_feat_twostream, bn=False, wd=1e-5, SDF_WEIGHT=10, --mask_weight 4; models/model_normalization.py:169-206,254-299,
// utils/tf_util.py:23-47).  One step:
//   1. encode the batch in groups of 8 (VGG embedding and taps only: the inference folds bake in fold2/conv1, which
//      training changes) and gather the raw [B*N, 1472] point features next to the local stream's layer-3 output;
//   2. forward both streams with the layer activations kept: layer 1 (3 inputs) on the CUDA cores, every other layer a
//      tensor-core GEMM (conv_tc: bf16 hi/lo split operands, three MMAs per product, fp32 accumulation);
//   3. one kernel per image for the loss terms and dpred (TF's gradient conventions), float64 sums in a fixed order;
//   4. backward: dgrad dX = (dZ W^T) . [X > 0] and wgrad dW^T = dZ^T X as tensor-core GEMMs over the padded point axis
//      (split-K partials reduced in a fixed order), bias gradients and layer 1 by chunked float64 column sums, + wd W;
//   5. one Adam kernel over the 24 decoder variables (TF's ApplyAdam, float32, one rounding per operation).
// No step uses a float atomic, so two runs of the same steps are bitwise equal.  The context's fp32 decoder variables
// are the masters Adam updates in place; the encoder's variables are only read.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "common.cuh"

namespace disn {

namespace {
constexpr int kLayers = 6;
constexpr int kVars = 2 * kLayers * 2;                   // 2 streams x 6 layers x (weights, biases)
const char* const kScope[2] = {"sdfprediction", "sdfprediction_imgfeat"};
const char* const kLayer[kLayers] = {"fold1/conv1", "fold1/conv2", "fold1/conv3", "fold2/conv1", "fold2/conv2",
                                     "fold2/conv5"};
constexpr int kCout[kLayers] = {64, 256, 512, 512, 256, 1};
constexpr int kGroup = 8;                                // images per encode
constexpr int kSub = 16;                                 // column-sum chunks per image
constexpr int kCat = kHidden + kLocalFeat;               // 1984: the local stream's fold2/conv1 input
// phases timed by disn_train_phase_ms
enum { PH_ENCODE, PH_GATHER, PH_FORWARD, PH_LOSS, PH_BACKWARD, PH_ADAM, kTrainPhases };

int cin_of(int s, int l, int nc) {
  static const int c[kLayers] = {3, 64, 256, 0, 512, 256};
  return l == 3 ? (s == 0 ? kHidden + nc : kCat) : c[l];
}
std::string var_name(int v) {       // v = (s * 6 + l) * 2 + bias
  const int s = v / (2 * kLayers), l = (v / 2) % kLayers;
  return std::string(kScope[s]) + "/" + kLayer[l] + (v & 1 ? "/biases" : "/weights");
}
}  // namespace

struct TrainState {
  disn_train_config cfg{};
  int nc = 0;
  int64_t off[kVars + 1] = {};        // flat offsets of the variables in grad / m / v
  DevBuffer grad, m, v;               // [off[kVars]] each
  float beta1_power = 0.f, beta2_power = 0.f;
  double vgg_reg = 0.0;               // sum over the frozen VGG kernels of wd * l2_loss(w)
  DevBuffer arena;                    // step scratch
  std::vector<double> host_sums;
  // phase timing of the last step: events recorded at each phase boundary, the phase each interval belongs to (the
  // interval from event i-1 to event i is ev_phase[i]), and the milliseconds summed per phase
  std::vector<cudaEvent_t> ev;
  std::vector<int> ev_phase;
  int n_ev = 0;
  float phase_ms[kTrainPhases] = {};
  ~TrainState() {
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
  }
};

void train_state_free(TrainState* t) { delete t; }

namespace {
// records the end of an interval of phase `phase` on the context's stream (phase -1: the start)
int mark(disn_ctx* c, int phase) {
  TrainState* t = c->train.get();
  if (t->n_ev == (int)t->ev.size()) {
    cudaEvent_t e = nullptr;
    DISN_CUDA_OK(cudaEventCreate(&e));
    t->ev.push_back(e);
    t->ev_phase.push_back(-1);
  }
  t->ev_phase[t->n_ev] = phase;
  DISN_CUDA_OK(cudaEventRecord(t->ev[t->n_ev++], c->stream));
  return 0;
}
// after the stream is synchronised: the milliseconds of each phase of the last step
int sum_phases(TrainState* t) {
  for (float& m : t->phase_ms) m = 0.f;
  for (int i = 1; i < t->n_ev; ++i) {
    float ms = 0.f;
    DISN_CUDA_OK(cudaEventElapsedTime(&ms, t->ev[i - 1], t->ev[i]));
    if (t->ev_phase[i] >= 0) t->phase_ms[t->ev_phase[i]] += ms;
  }
  return 0;
}
}  // namespace

namespace {

struct VarTable {
  float* p[kVars];
  int64_t off[kVars + 1];
};

// the tensors whose squared norms one sumsq_kernel launch forms, by value (one CTA each)
struct SumSqTable {
  const float* p[kVars];
  int64_t n[kVars];
};

// ---------------------------------------------------------------------------------------------------------------------
// forward pieces
// X1[p][co] = relu(x W[0][co] + y W[1][co] + z W[2][co] + b[co])   (fp32 FMAs in k order)
__global__ void layer1_kernel(const float* __restrict__ pts, const float* __restrict__ W, const float* __restrict__ b,
                              float* __restrict__ out, int64_t P) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P * 64; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i >> 6;
    const int co = (int)(i & 63);
    const float* q = pts + p * 3;
    out[i] = fmaxf(fmaf(q[2], W[128 + co], fmaf(q[1], W[64 + co], q[0] * W[co])) + b[co], 0.f);
  }
}

// the global stream's per-image fold2/conv1 bias: gb[b][co] = sum_j emb[b][j] W[512 + j][co] + bias[co]
__global__ void gbias_kernel(const float* __restrict__ emb, const float* __restrict__ W, const float* __restrict__ bias,
                             float* __restrict__ gb, int B, int nc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * kHidden) return;
  const int b = i / kHidden, co = i % kHidden;
  float s = 0.f;
  for (int j = 0; j < nc; ++j) s = fmaf(emb[(int64_t)b * nc + j], W[(int64_t)(kHidden + j) * kHidden + co], s);
  gb[i] = s + bias[co];
}

// X[p][co] = relu(Z[p][co] + gb[image of p][co]) over P rows (padding rows use the last image)
__global__ void add_image_bias_relu_kernel(float* __restrict__ Z, const float* __restrict__ gb, int64_t rows, int64_t N,
                                           int B) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows * kHidden; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i / kHidden;
    const int b = (int)min(p / N, (int64_t)(B - 1));
    Z[i] = fmaxf(Z[i] + gb[b * kHidden + (int)(i % kHidden)], 0.f);
  }
}

// cat[p][0:512] = X3[p]
__global__ void concat_kernel(const float4* __restrict__ x3, float4* __restrict__ cat, int64_t rows) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows * (kHidden / 4); i += (int64_t)gridDim.x * blockDim.x)
    cat[(i / (kHidden / 4)) * (kCat / 4) + i % (kHidden / 4)] = x3[i];
}

// pred[p] = (X5g[p] . w6g + b6g) + (X5l[p] . w6l + b6l): one warp per point, lane sums then a fixed butterfly
__global__ void head_kernel(const float* __restrict__ xg, const float* __restrict__ xl, const float* __restrict__ wg,
                            const float* __restrict__ bg, const float* __restrict__ wl, const float* __restrict__ bl,
                            float* __restrict__ pred, int64_t rows) {
  const int lane = threadIdx.x & 31;
  for (int64_t p = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; p < rows; p += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    float sg = 0.f, sl = 0.f;
    for (int k = lane; k < 256; k += 32) {
      sg = fmaf(xg[p * 256 + k], wg[k], sg);
      sl = fmaf(xl[p * 256 + k], wl[k], sl);
    }
    for (int o = 16; o > 0; o >>= 1) {
      sg += __shfl_xor_sync(0xffffffffu, sg, o);
      sl += __shfl_xor_sync(0xffffffffu, sl, o);
    }
    if (lane == 0) pred[p] = (sg + bg[0]) + (sl + bl[0]);
  }
}

// C[m][n] = act(sum_s ws[s][m][n] + bias[n]) for a forward / dgrad GEMM that conv_tc split along K
__global__ void splitk_sum_kernel(const float* __restrict__ ws, int splits, int64_t MN, int N, const float* __restrict__ bias,
                                  int relu, float* __restrict__ C) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < MN; i += (int64_t)gridDim.x * blockDim.x) {
    float s = ws[i];
    for (int z = 1; z < splits; ++z) s += ws[(int64_t)z * MN + i];
    if (bias) s += bias[i % N];
    C[i] = relu ? fmaxf(s, 0.f) : s;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// loss: one CTA per image, thread t takes samples t, t + 512, ... in order, then a fixed tree (sdf_acc.cu's order).
// gt is the fed ground truth (sdf_val - 0.003).  dpred = d overall_loss / d pred with TF's conventions: the mean's
// gradient g0 = 1000 / (B N) in float32, times the weight mask, times sign(gt * sw - pred) (0 at 0), negated.
constexpr int LOSS_THREADS = 512;
__global__ void __launch_bounds__(LOSS_THREADS) loss_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                            int64_t N, float sw, float mw, float g0,
                                                            float* __restrict__ dpred, double* __restrict__ sums) {
  __shared__ double s_c[LOSS_THREADS], s_w[LOSS_THREADS], s_r[LOSS_THREADS];
  const int b = blockIdx.x, t = threadIdx.x;
  double cnt = 0.0, ws = 0.0, rs = 0.0;
  for (int64_t n = t; n < N; n += LOSS_THREADS) {
    const int64_t i = (int64_t)b * N + n;
    const float g = gt[i], pr = pred[i];
    cnt += (g > 0.f) == (pr > 0.f) ? 1.0 : 0.0;
    const float w = __fadd_rn(__fmul_rn(g <= 0.01f ? 1.f : 0.f, mw), g > 0.01f ? 1.f : 0.f);
    const float d = __fsub_rn(__fmul_rn(g, sw), pr);
    ws += (double)__fmul_rn(fabsf(d), w);
    rs += (double)fabsf(__fsub_rn(g, __fdiv_rn(pr, sw)));
    const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
    dpred[i] = -__fmul_rn(__fmul_rn(g0, w), sg);
  }
  s_c[t] = cnt; s_w[t] = ws; s_r[t] = rs;
  __syncthreads();
  for (int s = LOSS_THREADS / 2; s > 0; s >>= 1) {
    if (t < s) { s_c[t] += s_c[t + s]; s_w[t] += s_w[t + s]; s_r[t] += s_r[t + s]; }
    __syncthreads();
  }
  if (t == 0) { sums[b * 3] = s_c[0]; sums[b * 3 + 1] = s_w[0]; sums[b * 3 + 2] = s_r[0]; }
}

// sq[k] = float64 sum of x^2 over tensor k: one CTA per tensor, strided per thread, then a fixed tree
__global__ void sumsq_kernel(SumSqTable t, double* __restrict__ sq) {
  __shared__ double s[256];
  const float* x = t.p[blockIdx.x];
  const int64_t n = t.n[blockIdx.x];
  double a = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += 256) a += (double)x[i] * (double)x[i];
  s[threadIdx.x] = a;
  __syncthreads();
  for (int k = 128; k > 0; k >>= 1) {
    if ((int)threadIdx.x < k) s[threadIdx.x] += s[threadIdx.x + k];
    __syncthreads();
  }
  if (threadIdx.x == 0) sq[blockIdx.x] = s[0];
}

// ---------------------------------------------------------------------------------------------------------------------
// backward pieces
// dZ5[p][k] = X5[p][k] > 0 ? dpred[p] w6[k] : 0, both streams
__global__ void head_back_kernel(const float* __restrict__ dpred, const float* __restrict__ x, const float* __restrict__ w6,
                                 float* __restrict__ dz, int64_t rows) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows * 256; i += (int64_t)gridDim.x * blockDim.x)
    dz[i] = x[i] > 0.f ? __fmul_rn(dpred[i >> 8], w6[i & 255]) : 0.f;
}

// dX[i] = X[i] > 0 ? dX[i] : 0 (ReLU's gradient passes where its output, equivalently its input, is > 0)
__global__ void relu_mask_kernel(float* __restrict__ dx, const float* __restrict__ x, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (!(x[i] > 0.f)) dx[i] = 0.f;
}

// out[c][r] = in[r][c], [rows, cols] -> [cols, rows], 32 x 32 tiles through shared memory
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t rows, int cols) {
  __shared__ float tile[32][33];
  const int64_t r0 = (int64_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int64_t r = r0 + j;
    const int cc = c0 + threadIdx.x;
    tile[j][threadIdx.x] = (r < rows && cc < cols) ? in[r * cols + cc] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) {
    const int cc = c0 + j;
    const int64_t r = r0 + threadIdx.x;
    if (cc < cols && r < rows) out[(int64_t)cc * rows + r] = tile[threadIdx.x][j];
  }
}

// wgrad: the GEMM gave dW^T [Cout][Cin] as `splits` partials; g[ci][co] = sum_s ws[s][co][ci] + wd W[ci][co]
__global__ void wgrad_sum_kernel(const float* __restrict__ ws, int splits, int cin, int cout, const float* __restrict__ W,
                                 float wd, float* __restrict__ g) {
  const int64_t total = (int64_t)cin * cout, MN = total;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ci = (int)(i / cout), co = (int)(i % cout);
    const int64_t j = (int64_t)co * cin + ci;
    float s = ws[j];
    for (int z = 1; z < splits; ++z) s += ws[(int64_t)z * MN + j];
    g[i] = __fadd_rn(s, __fmul_rn(wd, W[i]));
  }
}

// Column sums of dZ [B*N, C] over points, in float64, in chunks: chunk (b, q) covers points [q*len, (q+1)*len) of image b.
// part[(b * kSub + q) * R + r][c] with R = 4 when pts is given (1, x, y, z multipliers: layer 1's bias and weight
// gradients), else R = 1.
__global__ void colsum_partial_kernel(const float* __restrict__ dz, const float* __restrict__ pts, int C, int64_t N,
                                      double* __restrict__ part) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int chunk = blockIdx.y;               // b * kSub + q
  if (c >= C) return;
  const int b = chunk / kSub, q = chunk % kSub;
  const int64_t len = (N + kSub - 1) / kSub;
  const int64_t n0 = q * len, n1 = min(N, n0 + len);
  double s0 = 0.0, sx = 0.0, sy = 0.0, sz = 0.0;
  for (int64_t n = n0; n < n1; ++n) {
    const int64_t p = (int64_t)b * N + n;
    const double d = dz[p * C + c];
    s0 += d;
    if (pts) { sx += (double)pts[p * 3] * d; sy += (double)pts[p * 3 + 1] * d; sz += (double)pts[p * 3 + 2] * d; }
  }
  const int R = pts ? 4 : 1;
  double* o = part + (int64_t)chunk * R * C + c;
  o[0] = s0;
  if (pts) { o[C] = sx; o[2 * C] = sy; o[3 * C] = sz; }
}

// per-image sums S[b][c] = sum_q part[b][q][0][c] (R = 1 layout), and db[c] = float32(sum_b S[b][c])
__global__ void colsum_final_kernel(const double* __restrict__ part, int C, int B, double* __restrict__ S,
                                    float* __restrict__ db) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double tot = 0.0;
  for (int b = 0; b < B; ++b) {
    double s = 0.0;
    for (int q = 0; q < kSub; ++q) s += part[((int64_t)b * kSub + q) * C + c];
    if (S) S[(int64_t)b * C + c] = s;
    tot += s;
  }
  db[c] = (float)tot;
}

// layer 1 (R = 4 layout): db[c] and dW[i][c] = float32(sum) + wd W[i][c]
__global__ void layer1_final_kernel(const double* __restrict__ part, int nchunks, const float* __restrict__ W, float wd,
                                    float* __restrict__ dW, float* __restrict__ db) {
  const int c = threadIdx.x;              // 64 columns
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < nchunks; ++k)
    for (int r = 0; r < 4; ++r) s[r] += part[((int64_t)k * 4 + r) * 64 + c];
  db[c] = (float)s[0];
  for (int i = 0; i < 3; ++i) dW[i * 64 + c] = __fadd_rn((float)s[i + 1], __fmul_rn(wd, W[i * 64 + c]));
}

// the global stream's embedding rows: dW[512 + j][co] = float32(sum_b emb[b][j] S[b][co]) + wd W[512 + j][co]
__global__ void emb_wgrad_kernel(const float* __restrict__ emb, const double* __restrict__ S, int B, int nc,
                                 const float* __restrict__ W, float wd, float* __restrict__ dW) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= (int64_t)nc * kHidden) return;
  const int j = (int)(i / kHidden), co = (int)(i % kHidden);
  double s = 0.0;
  for (int b = 0; b < B; ++b) s += (double)emb[(int64_t)b * nc + j] * S[(int64_t)b * kHidden + co];
  const int64_t w = (int64_t)(kHidden + j) * kHidden + co;
  dW[w] = __fadd_rn((float)s, __fmul_rn(wd, W[w]));
}

// TF's ApplyAdam (training/training_ops.cc, float32): m += (g - m)(1 - b1); v += (g^2 - v)(1 - b2);
// w -= (m alpha) / (sqrt(v) + eps), alpha = lr sqrt(1 - b2^t) / (1 - b1^t) formed on the host
__global__ void adam_kernel(VarTable t, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, float alpha,
                            float one_b1, float one_b2, float eps) {
  const int64_t total = t.off[kVars];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int k = 0;
    while (t.off[k + 1] <= i) ++k;
    const float gi = g[i];
    const float mi = __fadd_rn(m[i], __fmul_rn(__fsub_rn(gi, m[i]), one_b1));
    const float vi = __fadd_rn(v[i], __fmul_rn(__fsub_rn(__fmul_rn(gi, gi), v[i]), one_b2));
    m[i] = mi;
    v[i] = vi;
    float* w = t.p[k] + (i - t.off[k]);
    *w = __fsub_rn(*w, __fdiv_rn(__fmul_rn(mi, alpha), __fadd_rn(__fsqrt_rn(vi), eps)));
  }
}

int blocks_for(disn_ctx* c, int64_t n, int per = 256) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((n + per - 1) / per, (int64_t)c->num_sms * 16));
}

// the step's device buffers, carved from one arena (P = padded points)
struct StepBufs {
  float *pts, *prot, *tm, *gt, *uv, *emb, *gb, *cat, *pred, *dpred, *dz[2], *dt, *ws;
  float* x[2][5];               // [stream][layer 0..4]: post-ReLU outputs of layers 1-5
  uint8_t *wpk, *xpk;
  double *part, *S, *sums, *sq;
  int64_t ws_elems;
};

size_t carve(char* base, int B, int64_t P, int nc, StepBufs& s) {
  Arena a{base};
  s.pts = a.take<float>(P * 3); s.prot = a.take<float>(P * 3); s.tm = a.take<float>((size_t)B * 12);
  s.gt = a.take<float>(P); s.uv = a.take<float>(P * 2); s.emb = a.take<float>((size_t)B * nc);
  s.gb = a.take<float>((size_t)B * kHidden); s.cat = a.take<float>(P * kCat);
  s.pred = a.take<float>(P); s.dpred = a.take<float>(P);
  for (int st = 0; st < 2; ++st)
    for (int l = 0; l < 5; ++l) s.x[st][l] = a.take<float>(P * kCout[l]);
  s.dz[0] = a.take<float>(P * kHidden); s.dz[1] = a.take<float>(P * kHidden);
  s.dt = a.take<float>(P * kHidden);
  s.ws_elems = (int64_t)16 << 20;
  s.ws = a.take<float>(s.ws_elems);
  s.wpk = a.take<uint8_t>(conv_tc_packed_bytes(kCat, kHidden));
  s.xpk = a.take<uint8_t>(conv_tc_packed_bytes((int)P, kCat));
  s.part = a.take<double>((size_t)B * kSub * 4 * kHidden);
  s.S = a.take<double>((size_t)B * kHidden);
  s.sums = a.take<double>((size_t)B * 3);
  s.sq = a.take<double>(kVars);
  return a.off;
}

// C[M,N] = act(A[M,K] B[K,N] + bias) with B packed in bpk (forward and dgrad; M = the padded point count)
int tc_gemm(disn_ctx* c, const StepBufs& s, const float* A, const uint8_t* bpk, const float* bias, int relu, float* C,
            int64_t M, int N, int K) {
  int splits = 1;
  if (launch_conv_tc(c, A, bpk, bias, C, s.ws, s.ws_elems, (int)M, N, K, 0, 0, 0, relu, &splits)) return -1;
  if (splits > 1) {
    splitk_sum_kernel<<<blocks_for(c, M * N), 256, 0, c->stream>>>(s.ws, splits, M * N, N, bias, relu, C);
    c->launches++;
  }
  return 0;
}

// g[Cin][Cout] = X^T dZ + wd W over the P padded points: dZ^T (transposed into s.dt) times X packed as [P, Cin]
int tc_wgrad(disn_ctx* c, const StepBufs& s, const float* dz, int cout, const float* X, int64_t ldx, int cin, int64_t P,
             const float* W, float wd, float* g) {
  dim3 tb(32, 8), tg((unsigned)((P + 31) / 32), (unsigned)((cout + 31) / 32));
  transpose_kernel<<<tg, tb, 0, c->stream>>>(dz, s.dt, P, cout);
  c->launches++;
  if (conv_tc_pack_device(c, X, (int)P, cin, ldx, false, s.xpk)) return -1;
  int splits = 1;
  if (launch_conv_tc(c, s.dt, s.xpk, nullptr, s.ws, s.ws, s.ws_elems, cout, cin, (int)P, 0, 0, 0, 0, &splits)) return -1;
  wgrad_sum_kernel<<<blocks_for(c, (int64_t)cin * cout), 256, 0, c->stream>>>(s.ws, splits, cin, cout, W, wd, g);
  c->launches++;
  return 0;
}

const float* wt(disn_ctx* c, int s, int l, bool bias) { return c->weights.at(var_name((s * kLayers + l) * 2 + bias)).ptr(); }

// The whole step up to the gradients (flat, in variable order, in t->grad).  Leaves the per-image loss sums in s.sums
// and the squared norms of the decoder kernels in s.sq.
int train_forward_backward(disn_ctx* c, const float* imgs, int H, int Wd, const float* pts, const float* pts_rot,
                           const float* trans_mat, const float* gt, int B, int64_t N, StepBufs& s) {
  TrainState* t = c->train.get();
  const int nc = t->nc;
  const int64_t Pn = (int64_t)B * N;
  const int64_t P = (Pn + 127) / 128 * 128;
  const size_t need = carve(nullptr, B, P, nc, s);
  if (t->arena.ensure(need + 256)) return -1;
  carve(t->arena.as<char>(), B, P, nc, s);
  cudaStream_t st = c->stream;
  // inputs; padding points are zeros (finite activations) and get dpred = 0, so they add nothing to any gradient
  DISN_CUDA_OK(cudaMemsetAsync(s.pts, 0, (size_t)P * 3 * 4, st));
  DISN_CUDA_OK(cudaMemsetAsync(s.prot, 0, (size_t)P * 3 * 4, st));
  DISN_CUDA_OK(cudaMemsetAsync(s.dpred, 0, (size_t)P * 4, st));
  DISN_CUDA_OK(cudaMemsetAsync(s.cat, 0, (size_t)P * kCat * 4, st));
  DISN_CUDA_OK(cudaMemcpyAsync(s.pts, pts, (size_t)Pn * 12, cudaMemcpyHostToDevice, st));
  DISN_CUDA_OK(cudaMemcpyAsync(s.prot, pts_rot ? pts_rot : pts, (size_t)Pn * 12, cudaMemcpyHostToDevice, st));
  DISN_CUDA_OK(cudaMemcpyAsync(s.tm, trans_mat, (size_t)B * 48, cudaMemcpyHostToDevice, st));
  DISN_CUDA_OK(cudaMemcpyAsync(s.gt, gt, (size_t)Pn * 4, cudaMemcpyHostToDevice, st));
  // 1. encode in groups, keep the embeddings, gather the raw point features into cat[:, 512:]
  t->n_ev = 0;
  if (mark(c, -1)) return -1;
  for (int b0 = 0; b0 < B; b0 += kGroup) {
    const int gb = std::min(kGroup, B - b0);
    if (encoder_run(c, imgs + (size_t)b0 * H * Wd * 3, gb, H, Wd, 3, false, true)) return -1;
    DISN_CUDA_OK(cudaMemcpyAsync(s.emb + (size_t)b0 * nc, c->emb.as<float>(), (size_t)gb * nc * 4, cudaMemcpyDeviceToDevice,
                                 st));
    if (mark(c, PH_ENCODE)) return -1;
    if (gather_point_feat(c, s.pts + (int64_t)b0 * N * 3, s.tm + b0 * 12, gb, N, s.uv, s.cat + (int64_t)b0 * N * kCat + kHidden,
                          kCat))
      return -1;
    if (mark(c, PH_GATHER)) return -1;
  }
  // 2. forward
  for (int k = 0; k < 2; ++k) {
    float* const* x = s.x[k];
    layer1_kernel<<<blocks_for(c, P * 64), 256, 0, st>>>(s.prot, wt(c, k, 0, 0), wt(c, k, 0, 1), x[0], P);
    c->launches++;
    for (int l = 1; l < 5; ++l) {
      const float* W = wt(c, k, l, 0);
      const float* b = wt(c, k, l, 1);
      const int cin = l == 3 ? (k == 0 ? kHidden : kCat) : cin_of(k, l, nc);   // global layer 4: the point-feature rows
      const float* A = (l == 3 && k == 1) ? s.cat : x[l - 1];
      if (conv_tc_pack_device(c, W, cin, kCout[l], kCout[l], false, s.wpk)) return -1;
      if (l == 3 && k == 0) {
        gbias_kernel<<<(B * kHidden + 255) / 256, 256, 0, st>>>(s.emb, W, b, s.gb, B, nc);
        if (tc_gemm(c, s, A, s.wpk, nullptr, 0, x[l], P, kCout[l], cin)) return -1;
        add_image_bias_relu_kernel<<<blocks_for(c, P * kHidden), 256, 0, st>>>(x[l], s.gb, P, N, B);
        c->launches += 2;
      } else {
        if (tc_gemm(c, s, A, s.wpk, b, 1, x[l], P, kCout[l], cin)) return -1;
      }
      if (l == 2 && k == 1) {
        concat_kernel<<<blocks_for(c, P * kHidden / 4), 256, 0, st>>>(reinterpret_cast<const float4*>(x[l]),
                                                                         reinterpret_cast<float4*>(s.cat), P);
        c->launches++;
      }
    }
  }
  head_kernel<<<blocks_for(c, P * 32), 256, 0, st>>>(s.x[0][4], s.x[1][4], wt(c, 0, 5, 0), wt(c, 0, 5, 1), wt(c, 1, 5, 0),
                                                     wt(c, 1, 5, 1), s.pred, P);
  c->launches++;
  if (mark(c, PH_FORWARD)) return -1;
  // 3. loss terms and dpred (padding rows keep dpred = 0)
  const float g0 = 1000.0f / (float)Pn;                      // float32, as TF's Mean gradient
  loss_kernel<<<B, LOSS_THREADS, 0, st>>>(s.pred, s.gt, N, t->cfg.sdf_weight, t->cfg.mask_weight, g0, s.dpred, s.sums);
  c->launches++;
  // squared norms of the decoder kernels before the update (the regularization term)
  {
    SumSqTable sq{};
    for (int i = 0; i < kVars / 2; ++i) {
      const auto& w = c->weights.at(var_name(2 * i));
      sq.p[i] = w.ptr();
      sq.n[i] = w.numel;
    }
    sumsq_kernel<<<kVars / 2, 256, 0, st>>>(sq, s.sq);
    c->launches++;
  }
  if (mark(c, PH_LOSS)) return -1;
  // 4. backward, stream by stream; grad(v) = t->grad + off[v]
  const float wd = t->cfg.wd;
  auto G = [&](int k, int l, bool bias) { return t->grad.as<float>() + t->off[(k * kLayers + l) * 2 + bias]; };
  for (int k = 0; k < 2; ++k) {
    float* const* x = s.x[k];
    // head: dw6 = X5^T dpred (+ wd w6), db6 = sum dpred, dZ5 = dpred w6 . [X5 > 0]
    if (tc_wgrad(c, s, s.dpred, 1, x[4], 256, 256, P, wt(c, k, 5, 0), wd, G(k, 5, 0))) return -1;
    colsum_partial_kernel<<<dim3(1, B * kSub), 32, 0, st>>>(s.dpred, nullptr, 1, N, s.part);
    colsum_final_kernel<<<1, 32, 0, st>>>(s.part, 1, B, nullptr, G(k, 5, 1));
    head_back_kernel<<<blocks_for(c, P * 256), 256, 0, st>>>(s.dpred, x[4], wt(c, k, 5, 0), s.dz[0], P);
    c->launches += 3;
    int cur = 0;
    for (int l = 4; l >= 1; --l) {
      const int cout = kCout[l];
      const float* dz = s.dz[cur];
      const float* W = wt(c, k, l, 0);
      const bool emb_rows = (l == 3 && k == 0);
      const int cin = l == 3 ? (k == 0 ? kHidden : kCat) : cin_of(k, l, nc);
      const float* X = (l == 3 && k == 1) ? s.cat : x[l - 1];
      // bias (and, for the global fold2/conv1, the per-image sums its embedding rows need)
      colsum_partial_kernel<<<dim3((cout + 127) / 128, B * kSub), 128, 0, st>>>(dz, nullptr, cout, N, s.part);
      colsum_final_kernel<<<(cout + 127) / 128, 128, 0, st>>>(s.part, cout, B, emb_rows ? s.S : nullptr, G(k, l, 1));
      c->launches += 2;
      if (emb_rows) {
        emb_wgrad_kernel<<<(nc * kHidden + 255) / 256, 256, 0, st>>>(s.emb, s.S, B, nc, W, wd, G(k, l, 0));
        c->launches++;
      }
      if (tc_wgrad(c, s, dz, cout, X, l == 3 && k == 1 ? kCat : cin, cin, P, W, wd, G(k, l, 0))) return -1;
      // dX = (dZ W[:Cin']^T) . [X > 0], Cin' = the rows fed by the previous layer
      const int cprev = kCout[l - 1];
      if (conv_tc_pack_device(c, W, cout, cprev, cout, true, s.wpk)) return -1;
      if (tc_gemm(c, s, dz, s.wpk, nullptr, 0, s.dz[cur ^ 1], P, cprev, cout)) return -1;
      relu_mask_kernel<<<blocks_for(c, P * cprev), 256, 0, st>>>(s.dz[cur ^ 1], x[l - 1], P * cprev);
      c->launches++;
      cur ^= 1;
    }
    // layer 1: db1 and dW1 = [x y z]^T dZ1 by column sums (3 inputs), over the real points only
    colsum_partial_kernel<<<dim3(1, B * kSub), 64, 0, st>>>(s.dz[cur], s.prot, 64, N, s.part);
    layer1_final_kernel<<<1, 64, 0, st>>>(s.part, B * kSub, wt(c, k, 0, 0), wd, G(k, 0, 0), G(k, 0, 1));
    c->launches += 2;
  }
  if (mark(c, PH_BACKWARD)) return -1;
  DISN_CUDA_OK(cudaGetLastError());
  return 0;
}

// the five reported values from the per-image sums and the squared kernel norms (host, float64 sums in image order, each
// value rounded to float32 as TF reports it): accuracy, sdf_loss_realvalue, sdf_loss, regularization, overall_loss
void reported(const TrainState* t, const double* sums, const double* sq, int B, int64_t Pn, double* out) {
  double cnt = 0.0, ws = 0.0, rs = 0.0;
  for (int b = 0; b < B; ++b) { cnt += sums[b * 3]; ws += sums[b * 3 + 1]; rs += sums[b * 3 + 2]; }
  double reg = t->vgg_reg;
  for (int i = 0; i < kVars / 2; ++i) reg += (double)t->cfg.wd * sq[i] / 2;
  const float acc = (float)cnt / (float)Pn;
  const float real = (float)(rs / (double)Pn);
  const float loss = (float)(ws / (double)Pn) * 1000.0f;
  const float regf = (float)reg;
  out[0] = acc; out[1] = real; out[2] = loss; out[3] = regf; out[4] = (float)(loss + regf);
}

int step_checks(disn_ctx* c, const float* imgs, const float* pts, const float* trans_mat, const float* gt, int B, int64_t N,
                int H, int W, int C) {
  DISN_REQUIRE(c && imgs && pts && trans_mat && gt, "null argument");
  DISN_REQUIRE(c->train, "disn_train_begin has not been called");
  DISN_REQUIRE(B >= 1 && N >= 1 && C == 3, "train_step: B >= 1, N >= 1, 3-channel images");
  DISN_REQUIRE((int64_t)B * N <= ((int64_t)1 << 24), "train_step: B * N <= 2^24 points");
  DISN_REQUIRE(B <= 65535 / kSub, "train_step: B <= " + std::to_string(65535 / kSub) + " images per step");
  for (int v = 0; v < kVars; ++v) {
    auto it = c->weights.find(var_name(v));
    DISN_REQUIRE(it != c->weights.end() && it->second.numel == c->train->off[v + 1] - c->train->off[v],
                 "variable " + var_name(v) + " is missing or changed size since disn_train_begin");
  }
  (void)H; (void)W;
  return 0;
}

// after a step the encoded state (embedding-only encodes, and projected maps / folded bias of old decoder weights) and
// every packed form of the decoder are stale
void invalidate_inference(disn_ctx* c) {
  c->enc_B = 0;
  c->enc_stale = true;
  c->weights_dirty = true;
  for (int l = 0; l < 5; ++l) c->enc_tc_weights.erase("proj" + std::to_string(l));
  c->enc_tc_weights.erase("decoder_proj");
  // a full encode's graph (key[4] = embedding_only = 0) replays the erased projection packs, and its warm key would have
  // the next full encode captured before they are repacked; the embedding-only graph of the training encodes reads no
  // decoder variable and stays
  const bool full_graph = c->enc_graph_key.size() > 4 && c->enc_graph_key[4] == 0;
  const bool full_warm = c->enc_warm_key.size() > 4 && c->enc_warm_key[4] == 0;
  if (full_graph) encoder_graph_reset(c);
  else if (full_warm) c->enc_warm_key.clear();
}

}  // namespace
}  // namespace disn

using namespace disn;

extern "C" {

void disn_default_train_config(disn_train_config* cfg) {
  if (!cfg) return;
  cfg->beta1 = 0.5f;
  cfg->beta2 = 0.999f;
  cfg->epsilon = 1e-8f;
  cfg->wd = 1e-5f;
  cfg->mask_weight = 4.0f;
  cfg->sdf_weight = 10.0f;
}

int disn_train_begin(disn_ctx* c, const disn_train_config* cfg) {
  DISN_REQUIRE(c && cfg, "null argument");
  DISN_REQUIRE(cfg->beta1 >= 0.f && cfg->beta1 < 1.f && cfg->beta2 >= 0.f && cfg->beta2 < 1.f && cfg->epsilon > 0.f &&
                   std::isfinite(cfg->wd) && std::isfinite(cfg->mask_weight) && std::isfinite(cfg->sdf_weight),
               "train_begin: beta1, beta2 in [0,1), epsilon > 0, finite wd / mask_weight / sdf_weight");
  DISN_REQUIRE(c->cfg.tanh_out == 0, "train_begin: training with --tanh is not implemented");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  if (c->weights_dirty && disn_finalize_weights(c)) return -1;     // checks the decoder's names and shapes
  std::unique_ptr<TrainState, TrainStateDeleter> t(new TrainState());
  t->cfg = *cfg;
  t->nc = c->cfg.num_classes;
  for (int v = 0; v < kVars; ++v) {
    const int s = v / (2 * kLayers), l = (v / 2) % kLayers;
    const int64_t n = (v & 1) ? kCout[l] : (int64_t)cin_of(s, l, t->nc) * kCout[l];
    DISN_REQUIRE(c->weights.at(var_name(v)).numel == n, "variable " + var_name(v) + " has the wrong size");
    t->off[v + 1] = t->off[v] + n;
  }
  const size_t bytes = (size_t)t->off[kVars] * sizeof(float);
  if (t->grad.ensure(bytes) || t->m.ensure(bytes) || t->v.ensure(bytes)) return -1;
  DISN_CUDA_OK(cudaMemsetAsync(t->grad.as<float>(), 0, bytes, c->stream));
  DISN_CUDA_OK(cudaMemsetAsync(t->m.as<float>(), 0, bytes, c->stream));
  DISN_CUDA_OK(cudaMemsetAsync(t->v.as<float>(), 0, bytes, c->stream));
  t->beta1_power = cfg->beta1;        // TF creates the powers with the betas and multiplies them after each step
  t->beta2_power = cfg->beta2;
  // the frozen encoder's share of the regularization: every vgg_16 kernel (slim.l2_regularizer, conv and fc layers)
  std::vector<std::string> vgg;
  for (const auto& kv : c->weights)
    if (kv.first.rfind("vgg_16/", 0) == 0 && kv.first.size() > 8 && kv.first.compare(kv.first.size() - 8, 8, "/weights") == 0)
      vgg.push_back(kv.first);
  DISN_REQUIRE(vgg.size() <= kVars, "train_begin: more vgg_16 kernels than expected");
  if (!vgg.empty()) {
    SumSqTable tb{};
    for (size_t i = 0; i < vgg.size(); ++i) {
      const auto& w = c->weights.at(vgg[i]);
      tb.p[i] = w.ptr();
      tb.n[i] = w.numel;
    }
    DevBuffer tmp;
    if (tmp.ensure(kVars * sizeof(double))) return -1;
    double* d_sq = tmp.as<double>();
    sumsq_kernel<<<(unsigned)vgg.size(), 256, 0, c->stream>>>(tb, d_sq);
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
    std::vector<double> sq(vgg.size());
    DISN_CUDA_OK(cudaMemcpyAsync(sq.data(), d_sq, sq.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
    for (double q : sq) t->vgg_reg += (double)cfg->wd * q / 2;     // std::map order: the names' order
  }
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  c->train = std::move(t);
  return 0;
}

int disn_train_step(disn_ctx* c, const float* imgs, int32_t H, int32_t W, int32_t C, const float* pts, const float* pts_rot,
                    const float* trans_mat, const float* sdf_gt, int32_t B, int64_t N, float lr, double* losses) {
  if (int rc = step_checks(c, imgs, pts, trans_mat, sdf_gt, B, N, H, W, C)) return rc;
  DISN_REQUIRE(losses && std::isfinite(lr), "train_step: losses and a finite lr");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  TrainState* t = c->train.get();
  StepBufs s{};
  const int rc = train_forward_backward(c, imgs, H, W, pts, pts_rot, trans_mat, sdf_gt, B, N, s);
  invalidate_inference(c);      // also on failure: the encoder buffers hold a training batch
  if (rc) return rc;
  // 5. Adam, TF's float32 alpha
  const float alpha = lr * sqrtf(1.f - t->beta2_power) / (1.f - t->beta1_power);   // host float32, no contraction
  VarTable vt;
  for (int v = 0; v < kVars; ++v) { vt.p[v] = c->weights.at(var_name(v)).ptr(); vt.off[v] = t->off[v]; }
  vt.off[kVars] = t->off[kVars];
  adam_kernel<<<blocks_for(c, t->off[kVars]), 256, 0, c->stream>>>(vt, t->grad.as<float>(), t->m.as<float>(), t->v.as<float>(),
                                                                  alpha, 1.f - t->cfg.beta1, 1.f - t->cfg.beta2,
                                                                  t->cfg.epsilon);
  c->launches++;
  DISN_CUDA_OK(cudaGetLastError());
  if (mark(c, PH_ADAM)) return -1;
  t->host_sums.resize((size_t)B * 3 + kVars / 2);
  DISN_CUDA_OK(cudaMemcpyAsync(t->host_sums.data(), s.sums, (size_t)B * 3 * sizeof(double), cudaMemcpyDeviceToHost,
                               c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(t->host_sums.data() + B * 3, s.sq, (kVars / 2) * sizeof(double), cudaMemcpyDeviceToHost,
                               c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  if (sum_phases(t)) return -1;
  t->beta1_power = t->beta1_power * t->cfg.beta1;
  t->beta2_power = t->beta2_power * t->cfg.beta2;
  reported(t, t->host_sums.data(), t->host_sums.data() + B * 3, B, (int64_t)B * N, losses);
  return 0;
}

// name -> (device pointer or host scalar, element count, slot: 0 variable, 1 Adam, 2 Adam_1, 3 beta power, 4 another
// loaded variable, read only)
static int train_slot(disn_ctx* c, const char* name, float** dev, float** host, int64_t* n, int* slot) {
  DISN_REQUIRE(c && name, "null argument");
  DISN_REQUIRE(c->train, "disn_train_begin has not been called");
  TrainState* t = c->train.get();
  std::string nm(name);
  *dev = nullptr; *host = nullptr; *slot = 3; *n = 1;
  if (nm == "beta1_power") { *host = &t->beta1_power; return 0; }
  if (nm == "beta2_power") { *host = &t->beta2_power; return 0; }
  *slot = 0;
  if (nm.size() > 7 && nm.compare(nm.size() - 7, 7, "/Adam_1") == 0) { *slot = 2; nm.resize(nm.size() - 7); }
  else if (nm.size() > 5 && nm.compare(nm.size() - 5, 5, "/Adam") == 0) { *slot = 1; nm.resize(nm.size() - 5); }
  for (int v = 0; v < kVars; ++v)
    if (var_name(v) == nm) {
      *n = t->off[v + 1] - t->off[v];
      *dev = *slot == 0 ? c->weights.at(nm).ptr() : (*slot == 1 ? t->m : t->v).as<float>() + t->off[v];
      return 0;
    }
  auto it = c->weights.find(name);     // any other loaded variable (the frozen encoder's): read only
  DISN_REQUIRE(it != c->weights.end() && *slot == 0, "unknown training variable " + std::string(name));
  *slot = 4;
  *n = it->second.numel;
  *dev = it->second.ptr();
  return 0;
}

int disn_train_get(disn_ctx* c, const char* name, float* out, int64_t n) {
  float *dev, *host;
  int64_t have = 0;
  int slot = 0;
  if (int rc = train_slot(c, name, &dev, &host, &have, &slot)) return rc;
  DISN_REQUIRE(out && n == have, std::string("train_get: ") + name + " has " + std::to_string(have) + " elements");
  if (host) { *out = *host; return 0; }
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  DISN_CUDA_OK(cudaMemcpyAsync(out, dev, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

int disn_train_set(disn_ctx* c, const char* name, const float* data, int64_t n) {
  float *dev, *host;
  int64_t have = 0;
  int slot = 0;
  if (int rc = train_slot(c, name, &dev, &host, &have, &slot)) return rc;
  DISN_REQUIRE(data && n == have, std::string("train_set: ") + name + " has " + std::to_string(have) + " elements");
  DISN_REQUIRE(slot != 4, std::string("train_set: ") + name + " is not a decoder variable, slot or beta power");
  if (host) { *host = *data; return 0; }
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  DISN_CUDA_OK(cudaMemcpyAsync(dev, data, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  if (slot == 0) invalidate_inference(c);     // a decoder variable changed
  return 0;
}

int disn_train_phase_ms(disn_ctx* c, float* ms) {
  DISN_REQUIRE(c && ms, "null argument");
  DISN_REQUIRE(c->train, "disn_train_begin has not been called");
  for (int i = 0; i < kTrainPhases; ++i) ms[i] = c->train->phase_ms[i];
  return 0;
}

int disn_train_var_name(int32_t i, char* out, int64_t capacity) {
  DISN_REQUIRE(i >= 0 && i < kVars && out, "train_var_name: index in [0, 24)");
  const std::string n = var_name(i);
  DISN_REQUIRE(capacity > (int64_t)n.size(), "train_var_name: buffer too small");
  memcpy(out, n.c_str(), n.size() + 1);
  return 0;
}

}  // extern "C"

#ifdef DISN_DIAGNOSTICS
// Diagnostic: one step's gradients without the update -> grads [total] (variables in disn_train_var_name order, each
// row-major as TF stores it), pred [B*N], acts (NULL or [2][5][B*N][width] of the stream layer outputs, widths
// 64, 256, 512, 512, 256) and the five reported values.  The encoded state is dropped as by disn_train_step.
extern "C" int disn_debug_train_grads(disn_ctx* c, const float* imgs, int32_t H, int32_t W, int32_t C, const float* pts,
                                      const float* pts_rot, const float* trans_mat, const float* sdf_gt, int32_t B, int64_t N,
                                      float* grads, float* pred, float* acts, double* losses) {
  using namespace disn;
  if (int rc = step_checks(c, imgs, pts, trans_mat, sdf_gt, B, N, H, W, C)) return rc;
  DISN_REQUIRE(grads && pred && losses, "null argument");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  TrainState* t = c->train.get();
  StepBufs s{};
  const int rc = train_forward_backward(c, imgs, H, W, pts, pts_rot, trans_mat, sdf_gt, B, N, s);
  invalidate_inference(c);
  if (rc) return rc;
  const int64_t Pn = (int64_t)B * N;
  std::vector<double> h((size_t)B * 3 + kVars / 2);
  DISN_CUDA_OK(cudaMemcpyAsync(grads, t->grad.as<float>(), (size_t)t->off[kVars] * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(pred, s.pred, (size_t)Pn * 4, cudaMemcpyDeviceToHost, c->stream));
  if (acts) {
    float* o = acts;
    for (int k = 0; k < 2; ++k)
      for (int l = 0; l < 5; ++l) {
        DISN_CUDA_OK(cudaMemcpyAsync(o, s.x[k][l], (size_t)Pn * kCout[l] * 4, cudaMemcpyDeviceToHost, c->stream));
        o += Pn * kCout[l];
      }
  }
  DISN_CUDA_OK(cudaMemcpyAsync(h.data(), s.sums, (size_t)B * 3 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(h.data() + B * 3, s.sq, (kVars / 2) * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  if (sum_phases(t)) return -1;
  reported(t, h.data(), h.data() + B * 3, B, Pn, losses);
  return 0;
}
#endif  // DISN_DIAGNOSTICS
