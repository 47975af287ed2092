// C ABI of the DISN hot-path library (see include/disn_b200.h for the reference call sites).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

#include "adaptive_common.cuh"
#include "common.cuh"

namespace disn {
static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
}  // namespace disn

using namespace disn;

disn_ctx::~disn_ctx() {
  encoder_graph_reset(this);
  for (cudaEvent_t e : sdf_ev)
    if (e) cudaEventDestroy(e);
  for (cudaEvent_t e : ad_ev)
    if (e) cudaEventDestroy(e);
  for (cudaEvent_t e : am_ev)
    if (e) cudaEventDestroy(e);
  for (cudaEvent_t e : obj_ev)
    if (e) cudaEventDestroy(e);
  if (own_stream && stream) cudaStreamDestroy(stream);
}

extern "C" {

const char* disn_last_error(void) { return g_err.c_str(); }

void disn_default_config(disn_config* cfg) {
  if (!cfg) return;
  cfg->device = 0;
  cfg->img_h = 137; cfg->img_w = 137;
  cfg->vgg_in = 224;
  cfg->num_classes = 1024;
  cfg->clamp_max = 136.0f;
  cfg->sdf_weight = 10.0f;
  cfg->tanh_out = 0;
  cfg->precision = DISN_PREC_FP32;
  cfg->max_batch = 1;
}

int disn_create(const disn_config* cfg, disn_ctx** out) {
  DISN_REQUIRE(cfg && out, "null config/out");
  DISN_REQUIRE(cfg->max_batch >= 1 && cfg->max_batch <= 8, "max_batch in [1,8]");
  DISN_REQUIRE(cfg->img_h > 1 && cfg->img_w > 1 && cfg->num_classes % 4 == 0, "bad image/embedding size");
  // the tensor-core point kernel addresses one image's projected map with 32-bit element offsets (point_tc.cu taps_of)
  DISN_REQUIRE((int64_t)cfg->img_h * cfg->img_w * kHidden < ((int64_t)1 << 31),
               "feature map too large: img_h * img_w * 512 must stay below 2^31 (" + std::to_string(cfg->img_h) + " x " +
                   std::to_string(cfg->img_w) + " given)");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    set_error(std::string("no CUDA device: the DISN path has no CPU fallback (") + cudaGetErrorString(e) + ")");
    return -1;
  }
  DISN_REQUIRE(cfg->device >= 0 && cfg->device < ndev, "device ordinal out of range");
  DISN_CUDA_OK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  DISN_CUDA_OK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9) {
    set_error("this library is built for sm_90a (H100) only; device is sm_" + std::to_string(prop.major) +
              std::to_string(prop.minor));
    return -1;
  }
  std::unique_ptr<disn_ctx> c(new disn_ctx());   // a failure below frees everything created so far
  c->cfg = *cfg;
  c->num_sms = prop.multiProcessorCount;
  cudaStream_t s = nullptr;      // a failed create may still write the handle: only a created stream goes in c
  DISN_CUDA_OK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  c->stream = s;
  c->own_stream = true;
  if (c->d_tm.ensure(sizeof(float) * 12 * 8) || c->d_status.ensure(sizeof(int)) || c->h_status.ensure(sizeof(int)))
    return -1;
  DISN_CUDA_OK(cudaMemset(c->d_status.as<int>(), 0, sizeof(int)));
  *c->h_status.as<int>() = 0;
  *out = c.release();
  return 0;
}

void disn_destroy(disn_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->cfg.device);
  cudaStreamSynchronize(c->stream);
  delete c;
}

}  // extern "C"

// Call after a synchronisation of c->stream: turns failure bits the kernels raised into a loud error.
int disn::check_status(disn_ctx* c) {
  int* h = c->h_status.as<int>();
  const int st = *h;
  if (st == 0) return 0;
  *h = 0;
  cudaMemsetAsync(c->d_status.as<int>(), 0, sizeof(int), c->stream);
  if (st & DISN_STATUS_FP16_OVERFLOW) {
    set_error("DISN_PREC_F16F8: an MLP activation exceeded the fp16 range (65504); the result is invalid -- "
              "use DISN_PREC_BF16X3 (fp32 range) for these weights");
    return -4;
  }
  if (st & DISN_STATUS_BAD_INDEX) {
    set_error("eval_grid_indexed: a grid index lies outside [0, (sdf_res+1)^3); the result is invalid");
    return -4;
  }
  set_error("kernel reported status " + std::to_string(st));
  return -4;
}

extern "C" {

int disn_set_stream(disn_ctx* c, void* cuda_stream) {
  DISN_REQUIRE(c, "null ctx");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
  if (cuda_stream) {
    c->stream = (cudaStream_t)cuda_stream;
    c->own_stream = false;
  } else {
    DISN_CUDA_OK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    c->own_stream = true;
  }
  return 0;
}

int disn_synchronize(disn_ctx* c) {
  DISN_REQUIRE(c, "null ctx");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return check_status(c);     // asynchronous (DISN_DEVICE_PTR) launches report here
}

int disn_set_precision(disn_ctx* c, int32_t precision) {
  DISN_REQUIRE(c, "null ctx");
  DISN_REQUIRE(precision == DISN_PREC_FP32 || precision == DISN_PREC_BF16X3 || precision == DISN_PREC_F16F8,
               "unknown precision");
  c->cfg.precision = precision;
  return 0;
}

int64_t disn_launch_count(disn_ctx* c) { return c ? c->launches : 0; }

int disn_load_weight(disn_ctx* c, const char* name, const float* data, const int64_t* shape, int32_t ndim) {
  DISN_REQUIRE(c && name && data && shape && ndim >= 1 && ndim <= 4, "bad load_weight arguments");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  int64_t numel = 1;
  std::vector<int64_t> shp(shape, shape + ndim);
  for (int i = 0; i < ndim; ++i) { DISN_REQUIRE(shape[i] > 0, "non-positive dim"); numel *= shape[i]; }
  DevTensor& t = c->weights[name];
  if (t.numel != numel) t.buf = DevBuffer();      // a weight of another size gets an allocation of exactly its size
  if (t.buf.ensure(numel * sizeof(float))) return -1;
  t.shape = shp;
  t.numel = numel;
  DISN_CUDA_OK(cudaMemcpyAsync(t.ptr(), data, numel * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));   // caller-owned host buffer; ordered on the ctx stream
  c->weights_dirty = true;
  c->enc_B = 0;     // encoder products (taps, gbias, pmap) belong to the previous weights: force a new disn_encode
  c->enc_tc_weights.clear();     // packed encoder weights follow the fp32 masters
  encoder_graph_reset(c);    // the graph replays launches that read the old packed images
  return 0;
}

static int check_shape(disn_ctx* c, const std::string& name, std::initializer_list<int64_t> want) {
  auto it = c->weights.find(name);
  DISN_REQUIRE(it != c->weights.end(), "missing variable " + name);
  std::vector<int64_t> w(want);
  // accept [1,1,Cin,Cout] or [Cin,Cout] for 1x1 convs
  const auto& s = it->second.shape;
  int64_t nw = 1, ns = 1;
  for (auto v : w) nw *= v;
  for (auto v : s) ns *= v;
  DISN_REQUIRE(nw == ns && s.back() == w.back(), "variable " + name + " has the wrong shape");
  return 0;
}

int disn_finalize_weights(disn_ctx* c) {
  DISN_REQUIRE(c, "null ctx");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const int nc = c->cfg.num_classes;
  for (const char* sc : {"sdfprediction", "sdfprediction_imgfeat"}) {
    std::string p(sc);
    int64_t cat = (p == "sdfprediction") ? 512 + nc : 512 + kLocalFeat;
    if (check_shape(c, p + "/fold1/conv1/weights", {3, 64})) return -2;
    if (check_shape(c, p + "/fold1/conv2/weights", {64, 256})) return -2;
    if (check_shape(c, p + "/fold1/conv3/weights", {256, 512})) return -2;
    if (check_shape(c, p + "/fold2/conv1/weights", {cat, 512})) return -2;
    if (check_shape(c, p + "/fold2/conv2/weights", {512, 256})) return -2;
    if (check_shape(c, p + "/fold2/conv5/weights", {256, 1})) return -2;
    for (const char* l : {"fold1/conv1", "fold1/conv2", "fold1/conv3", "fold2/conv1", "fold2/conv2", "fold2/conv5"})
      DISN_REQUIRE(c->weights.count(p + "/" + l + "/biases"), "missing variable " + p + "/" + l + "/biases");
    // the point kernels read these biases by output feature straight from the tensors
    const struct { const char* l; int64_t n; } widths[5] = {
        {"fold1/conv1", 64}, {"fold1/conv2", 256}, {"fold1/conv3", 512}, {"fold2/conv1", 512}, {"fold2/conv2", 256}};
    for (const auto& e : widths)
      DISN_REQUIRE(c->weights.at(p + "/" + e.l + "/biases").numel == e.n, "mis-shaped variable " + p + "/" + e.l + "/biases");
  }
  if (tc_pack_weights(c)) return -1;
  c->weights_dirty = false;
  return 0;
}

int disn_encode(disn_ctx* c, const float* imgs, int32_t B, int32_t H, int32_t W, int32_t C, uint32_t flags) {
  DISN_REQUIRE(c && imgs, "null ctx/imgs");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  DISN_REQUIRE(B <= c->cfg.max_batch, "batch exceeds max_batch of the context");
  if (c->weights_dirty && disn_finalize_weights(c)) return -1;
  if (encoder_run(c, imgs, B, H, W, C, (flags & DISN_DEVICE_PTR) != 0)) return -1;
  c->enc_stale = false;
  if (!(flags & DISN_DEVICE_PTR)) DISN_CUDA_OK(cudaStreamSynchronize(c->stream));   // caller-owned host buffer
  return 0;
}

int disn_get_encoded(disn_ctx* c, int32_t what, float* out, int64_t out_elems) {
  DISN_REQUIRE(c && out, "null ctx/out");
  DISN_REQUIRE(c->enc_B > 0, not_encoded(c));
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  static const int tapHW[5] = {224, 112, 56, 28, 14};
  const float* src = nullptr;
  int64_t n = 0, B = c->enc_B;
  if (what == 0) { src = c->emb.as<float>(); n = B * c->cfg.num_classes; }
  else if (what >= 1 && what <= 5) {
    src = c->taps[what - 1].as<float>();
    n = B * tapHW[what - 1] * tapHW[what - 1] * kTapC[what - 1];
  }
  else if (what == 6) { src = c->pmap.as<float>(); n = B * c->cfg.img_h * c->cfg.img_w * kHidden; }
  else if (what == 7) { src = c->gbias.as<float>(); n = B * kHidden; }
  else if (what == 8) { src = c->img_rs.as<float>(); n = B * c->cfg.vgg_in * c->cfg.vgg_in * 3; }
  DISN_REQUIRE(src, "unknown `what`");
  DISN_REQUIRE(out_elems == n, "output buffer has the wrong number of elements");
  DISN_CUDA_OK(cudaMemcpyAsync(out, src, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

static const float* W(disn_ctx* c, const std::string& n) { return c->weights.at(n).ptr(); }

static void fill_stream(disn_ctx* c, const std::string& p, StreamWeights& s) {
  s.w1 = W(c, p + "/fold1/conv1/weights"); s.b1 = W(c, p + "/fold1/conv1/biases");
  s.w2 = W(c, p + "/fold1/conv2/weights"); s.b2 = W(c, p + "/fold1/conv2/biases");
  s.w3 = W(c, p + "/fold1/conv3/weights"); s.b3 = W(c, p + "/fold1/conv3/biases");
  s.w4 = W(c, p + "/fold2/conv1/weights"); s.b4 = W(c, p + "/fold2/conv1/biases");
  s.w5 = W(c, p + "/fold2/conv2/weights"); s.b5 = W(c, p + "/fold2/conv2/biases");
  s.w6 = W(c, p + "/fold2/conv5/weights"); s.b6 = W(c, p + "/fold2/conv5/biases");
}

}  // extern "C"
int disn::ensure_point_scratch(disn_ctx* c, int64_t pts) {
  const size_t n = (size_t)pts * sizeof(float);
  return c->d_pts.ensure(3 * n) || c->d_pts_rot.ensure(3 * n) || c->d_out.ensure(n) || c->d_uv.ensure(2 * n) ? -1 : 0;
}

// Device-visible alias of a caller buffer that is pinned (cudaHostAlloc / cudaHostRegister / torch pin_memory), else
// nullptr.  With unified addressing the kernel epilogue can store its 4 B per point straight into such memory over PCIe
// (~1 GB/s at 2.5e8 points/s), so the host result needs no device scratch and no device->host copy after the kernel.
static float* pinned_alias(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  if (a.type == cudaMemoryTypeHost && a.devicePointer) return static_cast<float*>(a.devicePointer);
  return nullptr;
}

int disn::run_point_job(disn_ctx* c, PointJob& job) {
  if (!job.gbias) job.gbias = c->gbias.as<float>();
  if (!job.pmap) job.pmap = c->pmap.as<float>();
  job.img_h = c->cfg.img_h; job.img_w = c->cfg.img_w;
  job.clamp_max = c->cfg.clamp_max;
  job.tanh_out = c->cfg.tanh_out;
  fill_stream(c, "sdfprediction", job.g);
  fill_stream(c, "sdfprediction_imgfeat", job.l);
  job.status = c->d_status.as<int>();
  if (c->cfg.precision == DISN_PREC_FP32 ? launch_point_fp32(c, job) : launch_point_tc(c, job)) return -1;
  // the status word travels to the pinned mirror behind the kernel; whoever synchronises next checks it
  DISN_CUDA_OK(cudaMemcpyAsync(c->h_status.as<int>(), job.status, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  return 0;
}

extern "C" {

int disn_eval_points(disn_ctx* c, const float* pts, const float* pts_rot, const float* trans_mat, int32_t B,
                     int64_t N, float* out_pred, float* out_uv, uint32_t flags) {
  DISN_REQUIRE(c && pts && trans_mat && out_pred, "null argument");
  DISN_REQUIRE(c->enc_B > 0, not_encoded(c));
  DISN_REQUIRE(B == c->enc_B, "batch differs from the encoded batch");
  DISN_REQUIRE(N >= 0, "negative N");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  if (N == 0) return 0;
  PointJob job{};
  job.B = B; job.N = N; job.out_div = 1.0f;
  if (flags & DISN_DEVICE_PTR) {
    job.pts = pts; job.pts_rot = (pts_rot && pts_rot != pts) ? pts_rot : nullptr;
    job.trans_mat = trans_mat; job.out_pred = out_pred; job.out_uv = out_uv;
    return run_point_job(c, job);
  }
  if (ensure_point_scratch(c, (int64_t)B * N)) return -1;
  float* pred_alias = pinned_alias(out_pred);
  float* uv_alias = out_uv ? pinned_alias(out_uv) : nullptr;
  size_t nb = (size_t)B * N * 3 * sizeof(float);
  DISN_CUDA_OK(cudaMemcpyAsync(c->d_pts.as<float>(), pts, nb, cudaMemcpyHostToDevice, c->stream));
  job.pts = c->d_pts.as<float>();
  if (pts_rot && pts_rot != pts) {
    DISN_CUDA_OK(cudaMemcpyAsync(c->d_pts_rot.as<float>(), pts_rot, nb, cudaMemcpyHostToDevice, c->stream));
    job.pts_rot = c->d_pts_rot.as<float>();
  }
  DISN_CUDA_OK(cudaMemcpyAsync(c->d_tm.as<float>(), trans_mat, (size_t)B * 12 * sizeof(float), cudaMemcpyHostToDevice,
                               c->stream));
  job.trans_mat = c->d_tm.as<float>();
  job.out_pred = pred_alias ? pred_alias : c->d_out.as<float>();
  job.out_uv = out_uv ? (uv_alias ? uv_alias : c->d_uv.as<float>()) : nullptr;
  if (run_point_job(c, job)) return -1;
  if (!pred_alias)
    DISN_CUDA_OK(cudaMemcpyAsync(out_pred, job.out_pred, (size_t)B * N * sizeof(float), cudaMemcpyDeviceToHost,
                                 c->stream));
  if (out_uv && !uv_alias)
    DISN_CUDA_OK(cudaMemcpyAsync(out_uv, job.out_uv, (size_t)B * N * 2 * sizeof(float), cudaMemcpyDeviceToHost,
                                 c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return check_status(c);
}

// numpy.linspace(start, stop, num) in float64, then cast to float32 (test/create_sdf.py:247-254):
// y[i] = start + i*step with step = (stop-start)/(num-1), last element forced to stop.
static void linspace_f32(double start, double stop, int num, float* out) {
  if (num == 1) { out[0] = (float)start; return; }
  const double div = (double)(num - 1);
  const double delta = stop - start;
  volatile double step = delta / div;
  for (int i = 0; i < num; ++i) {
    volatile double prod = (double)i * step;   // volatile: no FMA contraction, match numpy's two roundings
    out[i] = (float)(prod + start);
  }
  out[num - 1] = (float)stop;
}

int disn_eval_grid(disn_ctx* c, const double* sdf_params, const float* trans_mat, int32_t B, int32_t sdf_res,
                   int32_t z0, int32_t z1, float* out_sdf, uint32_t flags) {
  DISN_REQUIRE(c && sdf_params && trans_mat && out_sdf, "null argument");
  DISN_REQUIRE(c->enc_B > 0, not_encoded(c));
  DISN_REQUIRE(B == c->enc_B, "batch differs from the encoded batch");
  DISN_REQUIRE(sdf_res >= 1, "sdf_res >= 1");
  const int R = sdf_res + 1;
  DISN_REQUIRE(z0 >= 0 && z1 <= R && z0 <= z1, "z range outside [0, sdf_res+1]");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const int64_t N = (int64_t)(z1 - z0) * R * R;
  if (N == 0) return 0;
  if (grid_axes(c, sdf_params, B, R)) return -1;

  PointJob job{};
  job.B = B; job.N = N; job.R = R; job.z0 = z0; job.axes = c->d_axes.as<float>();
  job.out_div = c->cfg.sdf_weight;   // correctly rounded r / 10 like the reference's float64 divide + float32 pack (create_sdf.py:285,299)
  if (flags & DISN_DEVICE_PTR) {
    job.trans_mat = trans_mat;
    job.out_pred = out_sdf;
    return run_point_job(c, job);
  }
  DISN_CUDA_OK(cudaMemcpyAsync(c->d_tm.as<float>(), trans_mat, (size_t)B * 12 * sizeof(float), cudaMemcpyHostToDevice,
                               c->stream));
  job.trans_mat = c->d_tm.as<float>();
  if (float* alias = pinned_alias(out_sdf)) {     // pinned caller buffer: the kernel writes the host grid directly
    job.out_pred = alias;
    if (run_point_job(c, job)) return -1;
    DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
    return check_status(c);
  }
  if (ensure_point_scratch(c, (int64_t)B * N)) return -1;
  job.out_pred = c->d_out.as<float>();
  if (run_point_job(c, job)) return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(out_sdf, job.out_pred, (size_t)B * N * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return check_status(c);
}

int disn_write_dist(const char* path, int32_t res, const double* bbox, const float* values) {
  DISN_REQUIRE(path && bbox && values && res >= 1, "bad write_dist arguments");
  FILE* f = fopen(path, "wb");
  if (!f) { set_error(std::string("cannot open ") + path); return -3; }
  int32_t hdr[3] = {-res, res, res};
  const size_t n = (size_t)(res + 1) * (res + 1) * (res + 1);
  bool ok = fwrite(hdr, sizeof(int32_t), 3, f) == 3 && fwrite(bbox, sizeof(double), 6, f) == 6 &&
            fwrite(values, sizeof(float), n, f) == n;
  ok = (fclose(f) == 0) && ok;
  if (!ok) { set_error(std::string("short write to ") + path); return -3; }
  return 0;
}

int disn_cam_estimate(disn_ctx* c, const float* imgs, int32_t B, int32_t H, int32_t W, int32_t C, const float* K,
                      float* out_rt, float* out_trans_mat) {
  DISN_REQUIRE(c && imgs && out_trans_mat, "null argument");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  DISN_REQUIRE(B >= 1 && B <= c->cfg.max_batch, "batch exceeds max_batch of the context");
  float *dK, *dRT, *dTM;
  auto carve = [&](char* base) {
    Arena a{base};
    dK = a.take<float>(9);
    dRT = a.take<float>((size_t)B * 12);
    dTM = a.take<float>((size_t)B * 12);
    return a.off;
  };
  if (c->nn_scratch.ensure(carve(nullptr))) return -1;
  carve(c->nn_scratch.as<char>());
  if (cam_predict(c, imgs, B, H, W, C, K, dK, dRT, dTM)) return -1;
  if (out_rt) DISN_CUDA_OK(cudaMemcpyAsync(out_rt, dRT, (size_t)B * 12 * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(out_trans_mat, dTM, (size_t)B * 12 * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

int disn_nn_distance(disn_ctx* c, const float* xyz1, const float* xyz2, int32_t B, int32_t N, int32_t M, float* dist1,
                     int32_t* idx1, float* dist2, int32_t* idx2) {
  DISN_REQUIRE(c && xyz1 && xyz2 && dist1 && idx1 && dist2 && idx2, "null argument");
  DISN_REQUIRE(B >= 1 && N >= 1 && M >= 1, "NnDistance requires non-empty point sets of shape (batch,#points,3)");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const size_t n1 = (size_t)B * N, n2 = (size_t)B * M;
  float *d1, *d2, *o1, *o2;
  int *i1, *i2;
  auto carve = [&](char* base) {
    Arena a{base};
    d1 = a.take<float>(n1 * 3);
    d2 = a.take<float>(n2 * 3);
    o1 = a.take<float>(n1);
    o2 = a.take<float>(n2);
    i1 = a.take<int>(n1);
    i2 = a.take<int>(n2);
    return a.off;
  };
  if (c->nn_scratch.ensure(carve(nullptr))) return -1;
  carve(c->nn_scratch.as<char>());
  DISN_CUDA_OK(cudaMemcpyAsync(d1, xyz1, n1 * 3 * 4, cudaMemcpyHostToDevice, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(d2, xyz2, n2 * 3 * 4, cudaMemcpyHostToDevice, c->stream));
  if (nn_distance(c, d1, N, d2, M, B, o1, i1, o2, i2)) return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(dist1, o1, n1 * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(idx1, i1, n1 * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(dist2, o2, n2 * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(idx2, i2, n2 * 4, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return 0;
}

int disn_write_obj(const char* path, const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces) {
  DISN_REQUIRE(path && (verts || n_verts == 0) && (faces || n_faces == 0) && n_verts >= 0 && n_faces >= 0,
               "bad write_obj arguments");
  FILE* f = fopen(path, "w");
  if (!f) { set_error(std::string("cannot open ") + path); return -3; }
  std::vector<char> buf(1 << 20);
  setvbuf(f, buf.data(), _IOFBF, buf.size());
  fprintf(f, "# Generated by the DISN marching-cubes post-pass\n# Number of vertices: %lld\n# Number of faces: %lld\n",
          (long long)n_verts, (long long)n_faces);
  for (int64_t i = 0; i < n_verts; ++i) fprintf(f, "v %g %g %g\n", verts[3 * i], verts[3 * i + 1], verts[3 * i + 2]);
  for (int64_t i = 0; i < n_faces; ++i)
    fprintf(f, "f %d %d %d\n", faces[3 * i] + 1, faces[3 * i + 1] + 1, faces[3 * i + 2] + 1);
  bool ok = !ferror(f);
  ok = (fclose(f) == 0) && ok;
  if (!ok) { set_error(std::string("short write to ") + path); return -3; }
  return 0;
}

// staging of a host SDF grid for marching cubes (persistent, grows)
static int mc_input(disn_ctx* c, const float* sdf, int32_t R, uint32_t flags, const float** d_sdf) {
  if (flags & DISN_DEVICE_PTR) { *d_sdf = sdf; return 0; }
  const size_t bytes = (size_t)R * R * R * sizeof(float);
  if (c->d_mc_in.ensure(bytes)) return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(c->d_mc_in.as<float>(), sdf, bytes, cudaMemcpyHostToDevice, c->stream));
  *d_sdf = c->d_mc_in.as<float>();
  return 0;
}

int disn_mc_run(disn_ctx* c, const float* sdf, int32_t R, const double* bbox, float iso, uint32_t flags,
                int64_t* n_verts, int64_t* n_faces) {
  DISN_REQUIRE(c && sdf && bbox, "null argument");
  DISN_REQUIRE(R >= 2, "need at least 2 samples per axis");
  DISN_REQUIRE((int64_t)R * R * R * 3 < (int64_t)1 << 32, "grid too large for 32-bit vertex ids");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const float* d_sdf = nullptr;
  int rc = mc_input(c, sdf, R, flags, &d_sdf);
  if (!rc) rc = mc_run(c, d_sdf, R, bbox, iso);
  return finish_mesh_call(c, rc, n_verts, n_faces);
}

int disn_mc_fetch(disn_ctx* c, float* verts, int32_t* faces) {
  DISN_REQUIRE(c, "null ctx");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  return c->mesh.fetch(c->stream, verts, faces);
}

int disn_mesh_counts(disn_ctx* c, int64_t* n_verts, int64_t* n_faces) {
  DISN_REQUIRE(c && n_verts && n_faces, "null argument");
  *n_verts = c->mesh.nv();
  *n_faces = c->mesh.nf();
  return 0;
}

int disn_mc_write_obj(disn_ctx* c, const char* path) {
  DISN_REQUIRE(c && path, "null argument");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const int64_t nv = c->mesh.nv(), nf = c->mesh.nf();
  std::vector<float> v((size_t)nv * 3);
  std::vector<int32_t> f((size_t)nf * 3);
  if (c->mesh.fetch(c->stream, v.data(), f.data())) return -1;
  return disn_write_obj(path, v.data(), nv, f.data(), nf);
}

int disn_marching_cubes(disn_ctx* c, const float* sdf, int32_t R, const double* bbox, float iso, float* verts,
                        int64_t* n_verts, int32_t* faces, int64_t* n_faces, uint32_t flags) {
  DISN_REQUIRE(c && sdf && bbox && n_verts && n_faces, "null argument");
  int64_t nv = 0, nf = 0;
  const int rc = disn_mc_run(c, sdf, R, bbox, iso, flags, &nv, &nf);
  if (rc) return rc;
  if (verts == nullptr || faces == nullptr) { *n_verts = nv; *n_faces = nf; return 0; }     // counting call
  if (*n_verts < nv || *n_faces < nf) { set_error("marching_cubes: output buffers too small"); return -2; }
  *n_verts = nv; *n_faces = nf;
  return c->mesh.fetch(c->stream, verts, faces);
}

int disn_mesh_load(disn_ctx* c, const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces) {
  DISN_REQUIRE(c, "null ctx");
  DISN_REQUIRE(n_verts >= 0 && n_faces >= 0 && (verts || n_verts == 0) && (faces || n_faces == 0),
               "bad mesh_load arguments");
  DISN_REQUIRE(n_verts < ((int64_t)1 << 31) && 3 * n_faces < ((int64_t)1 << 31), "mesh too large for 32-bit indices");
  for (int64_t i = 0; i < 3 * n_faces; ++i)
    if (faces[i] < 0 || faces[i] >= n_verts)
      DISN_REQUIRE(false, "face " + std::to_string(i / 3) + " references vertex " + std::to_string(faces[i]) +
                              " outside [0, " + std::to_string(n_verts) + ")");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  return finish_mesh_call(c, mesh_load(c, verts, n_verts, faces, n_faces), nullptr, nullptr);
}

int disn_mesh_clean(disn_ctx* c, double dist_thresh, double num_thresh, int32_t* face_component, int64_t* n_components,
                    int64_t* n_kept, int64_t* n_verts, int64_t* n_faces) {
  DISN_REQUIRE(c, "null ctx");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  return mesh_clean(c, dist_thresh, num_thresh, face_component, n_components, n_kept, n_verts, n_faces);
}

int disn_mesh_sdf(disn_ctx* c, int32_t res, const double* bbox, double expand_rate, double sigma, float* out,
                  double* bbox_out, uint32_t flags) {
  DISN_REQUIRE(c && out, "null argument");
  DISN_REQUIRE(res >= 1, "mesh_sdf: res >= 1");
  DISN_REQUIRE((int64_t)(res + 1) * (res + 1) * (res + 1) <= INT32_MAX,
               "mesh_sdf: (res+1)^3 grid points must fit a 32-bit index (res <= 1289)");
  DISN_REQUIRE(std::isfinite(sigma) && sigma >= 0.0, "mesh_sdf: sigma must be finite and >= 0");
  DISN_REQUIRE(bbox || (std::isfinite(expand_rate) && expand_rate > 0.0), "mesh_sdf: expand_rate must be finite and > 0");
  if (bbox)
    for (int a = 0; a < 3; ++a)
      DISN_REQUIRE(std::isfinite(bbox[a]) && std::isfinite(bbox[3 + a]) && bbox[a] < bbox[3 + a],
                   "mesh_sdf: box min must be below max on every axis");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  return mesh_sdf(c, res, bbox, expand_rate, sigma, out, bbox_out, (flags & DISN_DEVICE_PTR) != 0);
}

int disn_mesh_sdf_phase_ms(disn_ctx* c, float* ms) {
  DISN_REQUIRE(c && ms, "null argument");
  for (int i = 0; i < 4; ++i) ms[i] = c->sdf_phase_ms[i];
  return 0;
}

int disn_mesh_part_areas(disn_ctx* c, const int32_t* part_ids, int32_t n_parts, int64_t* part_q, int32_t* shift) {
  DISN_REQUIRE(c, "null ctx");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  return mesh_part_areas(c, part_ids, n_parts, part_q, shift);
}

int disn_mesh_normalize(disn_ctx* c, const int32_t* part_ids, int32_t n_parts, const int64_t* amounts,
                        const double* draws, int64_t n_draws, const double* given, double* centroid, double* m,
                        double* samples) {
  DISN_REQUIRE(c, "null ctx");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  return mesh_normalize(c, part_ids, n_parts, amounts, draws, n_draws, given, centroid, m, samples);
}

int disn_field(disn_ctx* c, int32_t R, float** out_dev) {
  DISN_REQUIRE(c && out_dev, "null argument");
  DISN_REQUIRE(R >= 2 && (int64_t)R * R * R <= INT32_MAX, "field: 2 <= R and R^3 < 2^31");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  if (c->d_field.ensure((size_t)R * R * R * sizeof(float))) return -1;
  *out_dev = c->d_field.as<float>();
  return 0;
}

int disn_sdf_band_count(disn_ctx* c, const float* sdf, int32_t R, float iso, const float* edges, uint32_t flags,
                        int64_t* counts) {
  DISN_REQUIRE(c && sdf && edges && counts, "null argument");
  DISN_REQUIRE(R >= 2 && (int64_t)R * R * R < INT32_MAX, "sdf_band_count: 2 <= R and R^3 < 2^31 - 1");
  // the four index lists share one buffer of R^3 entries: it holds them all only when no point lies in two bands
  for (int a = 0; a < 4; ++a) {
    const float la = edges[2 * a], ha = edges[2 * a + 1];
    DISN_REQUIRE(!std::isnan(la) && !std::isnan(ha), "sdf_band_count: band edges must not be NaN");
    for (int b = a + 1; b < 4; ++b) {
      const float lb = edges[2 * b], hb = edges[2 * b + 1];
      const bool empty = !(la < ha) || !(lb < hb);
      DISN_REQUIRE(empty || ha <= lb || hb <= la,
                   "sdf_band_count: bands " + std::to_string(a) + " and " + std::to_string(b) + " overlap");
    }
  }
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  return band_count(c, sdf, R, iso, edges, (flags & DISN_DEVICE_PTR) != 0, counts);
}

int disn_sdf_band_gather(disn_ctx* c, const float* axes, const int64_t* choices, const int64_t* k, float* out) {
  DISN_REQUIRE(c && axes && k && ((choices && out) || k[0] + k[1] + k[2] + k[3] == 0), "null argument");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  return band_gather(c, axes, choices, k, out);
}

int disn_sdf_strided(disn_ctx* c, const float* sdf, int32_t R, int32_t reduce, uint32_t flags, float* out) {
  DISN_REQUIRE(c && sdf && out, "null argument");
  DISN_REQUIRE(R >= 2 && (int64_t)R * R * R <= INT32_MAX && reduce >= 1, "sdf_strided: 2 <= R, R^3 < 2^31, reduce >= 1");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  return sdf_strided(c, sdf, R, reduce, (flags & DISN_DEVICE_PTR) != 0, out);
}

int disn_eval_grid_resident(disn_ctx* c, const double* sdf_params, const float* trans_mat, int32_t B, int32_t sdf_res,
                            float** out_dev) {
  DISN_REQUIRE(c && sdf_params && trans_mat && out_dev, "null argument");
  DISN_REQUIRE(sdf_res >= 1 && B >= 1, "sdf_res >= 1, B >= 1");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  const int R = sdf_res + 1;
  if (c->d_grid.ensure((size_t)B * R * R * R * sizeof(float))) return -1;
  float* tm = c->d_tm.as<float>();
  DISN_CUDA_OK(cudaMemcpyAsync(tm, trans_mat, (size_t)B * 12 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  const int rc = disn_eval_grid(c, sdf_params, tm, B, sdf_res, 0, R, c->d_grid.as<float>(), DISN_DEVICE_PTR);
  if (rc) return rc;
  *out_dev = c->d_grid.as<float>();
  return 0;
}

int disn_eval_grid_indexed(disn_ctx* c, const double* sdf_params, const float* trans_mat, int32_t image, int32_t sdf_res,
                           const int32_t* idx, int64_t n, float* out, uint32_t flags) {
  DISN_REQUIRE(c && sdf_params && trans_mat && ((idx && out) || n == 0), "null argument");
  DISN_REQUIRE(c->enc_B > 0, not_encoded(c));
  DISN_REQUIRE(image >= 0 && image < c->enc_B, "image outside the encoded batch");
  DISN_REQUIRE(sdf_res >= 1 && (int64_t)(sdf_res + 1) * (sdf_res + 1) * (sdf_res + 1) <= INT32_MAX,
               "eval_grid_indexed: 1 <= sdf_res and (sdf_res+1)^3 < 2^31");
  DISN_REQUIRE(n >= 0, "negative n");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  if (n == 0) return 0;
  const int R = sdf_res + 1;
  if (grid_axes(c, sdf_params, 1, R)) return -1;
  if (flags & DISN_DEVICE_PTR) return eval_grid_points(c, image, R, trans_mat, idx, n, out);
  const int64_t R3 = (int64_t)R * R * R;
  for (int64_t i = 0; i < n; ++i)
    DISN_REQUIRE(idx[i] >= 0 && idx[i] < R3, "eval_grid_indexed: index " + std::to_string(idx[i]) + " at position " +
                                                 std::to_string(i) + " lies outside [0, (sdf_res+1)^3)");
  if (c->d_idx.ensure((size_t)n * sizeof(int32_t)) || ensure_point_scratch(c, n)) return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(c->d_idx.as<int32_t>(), idx, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, c->stream));
  DISN_CUDA_OK(cudaMemcpyAsync(c->d_tm.as<float>(), trans_mat, 12 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  if (eval_grid_points(c, image, R, c->d_tm.as<float>(), c->d_idx.as<int32_t>(), n, c->d_out.as<float>())) return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(out, c->d_out.as<float>(), (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return check_status(c);
}

int disn_eval_grid_adaptive(disn_ctx* c, const double* sdf_params, const float* trans_mat, int32_t image, int32_t sdf_res,
                            float iso, double band, float** grid_dev, int64_t* level_counts, int32_t* n_levels) {
  DISN_REQUIRE(c && sdf_params && trans_mat && grid_dev && level_counts && n_levels, "null argument");
  DISN_REQUIRE(c->enc_B > 0, not_encoded(c));
  DISN_REQUIRE(image >= 0 && image < c->enc_B, "image outside the encoded batch");
  DISN_REQUIRE(sdf_res >= 1 && (int64_t)(sdf_res + 1) * (sdf_res + 1) * (sdf_res + 1) <= INT32_MAX,
               "eval_grid_adaptive: 1 <= sdf_res and (sdf_res+1)^3 < 2^31");
  DISN_REQUIRE(std::isfinite(iso), "eval_grid_adaptive: iso must be finite");
  DISN_REQUIRE(!std::isnan(band) && band >= 0.0, "eval_grid_adaptive: band must be >= 0 (+inf evaluates every point)");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  if (grid_axes(c, sdf_params, 1, sdf_res + 1)) return -1;
  DISN_CUDA_OK(cudaMemcpyAsync(c->d_tm.as<float>(), trans_mat, 12 * sizeof(float), cudaMemcpyHostToDevice, c->stream));
  if (adaptive_run(c, nullptr, image, c->d_tm.as<float>(), sdf_res, sdf_params, iso, band, level_counts, n_levels))
    return -1;
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  if (const int rc = check_status(c)) return rc;
  *grid_dev = c->ad_grid.as<float>();
  return 0;
}

}  // extern "C"

// End of a call that builds the resident mesh: on failure the resident mesh is emptied (it may be half replaced or built
// from invalid values), and the resident counts are reported either way, so a caller's view of the slot always matches
// what disn_mc_fetch copies.
int disn::finish_mesh_call(disn_ctx* c, int rc, int64_t* n_verts, int64_t* n_faces) {
  if (rc) {
    c->mesh.clear();
    c->am_nv = -1;
  }
  if (n_verts) *n_verts = c->mesh.nv();
  if (n_faces) *n_faces = c->mesh.nf();
  return rc;
}

extern "C" {

int disn_mesh_grid_adaptive(disn_ctx* c, const double* sdf_params, const float* trans_mat, int32_t image, int32_t sdf_res,
                            float iso, double band, int64_t* level_counts, int32_t* n_levels, int64_t* n_verts,
                            int64_t* n_faces) {
  DISN_REQUIRE(c && sdf_params && trans_mat && level_counts && n_levels, "null argument");
  DISN_REQUIRE(c->enc_B > 0, not_encoded(c));
  DISN_REQUIRE(image >= 0 && image < c->enc_B, "image outside the encoded batch");
  DISN_REQUIRE(sdf_res >= 1 && sdf_res <= 2048, "mesh_grid_adaptive: 1 <= sdf_res <= 2048");
  DISN_REQUIRE(std::isfinite(iso), "mesh_grid_adaptive: iso must be finite");
  DISN_REQUIRE(!std::isnan(band) && band >= 0.0, "mesh_grid_adaptive: band must be >= 0 (+inf evaluates every point)");
  const int64_t R = sdf_res + 1;
  DISN_REQUIRE(coarse_stride(sdf_res) > 1 || (R * R * R <= INT32_MAX && 3 * R * R * R < ((int64_t)1 << 32)),
               "mesh_grid_adaptive: an odd sdf_res (no power of two divides it) evaluates the dense grid, which needs "
               "(sdf_res+1)^3 < 2^31 and 3 (sdf_res+1)^3 < 2^32 (sdf_res <= 1125)");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  int rc = grid_axes(c, sdf_params, 1, sdf_res + 1);
  if (!rc && cudaMemcpyAsync(c->d_tm.as<float>(), trans_mat, 12 * sizeof(float), cudaMemcpyHostToDevice, c->stream)) {
    set_error("mesh_grid_adaptive: trans_mat upload failed");
    rc = -1;
  }
  if (!rc && coarse_stride(sdf_res) == 1) {     // the dense grid, as disn_eval_grid_adaptive evaluates it, then MC
    c->am_nv = -1;                              // the mesher's diagnostics describe no call until its next one
    c->am_edges_sorted = nullptr;
    rc = adaptive_run(c, nullptr, image, c->d_tm.as<float>(), sdf_res, sdf_params, iso, band, level_counts, n_levels);
    if (!rc) rc = mc_run(c, c->ad_grid.as<float>(), (int)R, sdf_params, iso);
  } else if (!rc) {
    rc = adaptive_mesh_run(c, nullptr, image, c->d_tm.as<float>(), sdf_res, sdf_params, iso, band, level_counts, n_levels);
  }
  if (!rc && cudaStreamSynchronize(c->stream) != cudaSuccess) {
    set_error("mesh_grid_adaptive: stream synchronisation failed");
    rc = -1;
  }
  if (!rc) rc = check_status(c);    // the f16f8 overflow status: the mesh was built from invalid values
  return finish_mesh_call(c, rc, n_verts, n_faces);
}

// ---- cross-process device buffers (multi-GPU gather without a collective) -------------------------------------------
// Rank 0 allocates the whole-grid buffer and exports a CUDA IPC handle; the other ranks (one process per GPU) open it and
// pass `ptr + slab offset` as the DISN_DEVICE_PTR output of disn_eval_grid, so the kernel's epilogue stores every
// SDF value straight into rank 0's HBM over NVLink (peer stores) while it computes: compute and gather are one kernel.
int disn_shared_alloc(disn_ctx* c, int64_t bytes, void** dev_ptr, unsigned char* handle64) {
  DISN_REQUIRE(c && dev_ptr && handle64 && bytes > 0, "bad shared_alloc arguments");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  void* p = nullptr;
  DISN_CUDA_OK(cudaMalloc(&p, (size_t)bytes));
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { cudaFree(p); set_error(std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(e)); return -1; }
  memcpy(handle64, &h, 64);
  *dev_ptr = p;
  return 0;
}

int disn_shared_open(disn_ctx* c, const unsigned char* handle64, void** dev_ptr) {
  DISN_REQUIRE(c && handle64 && dev_ptr, "bad shared_open arguments");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  DISN_CUDA_OK(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}

int disn_shared_close(disn_ctx* c, void* dev_ptr, int32_t owner) {
  DISN_REQUIRE(c && dev_ptr, "bad shared_close arguments");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  if (owner) DISN_CUDA_OK(cudaFree(dev_ptr));
  else DISN_CUDA_OK(cudaIpcCloseMemHandle(dev_ptr));
  return 0;
}

int disn_fetch(disn_ctx* c, const void* dev, void* host, int64_t bytes) {
  DISN_REQUIRE(c && dev && host && bytes >= 0, "bad fetch arguments");
  DISN_CUDA_OK(cudaSetDevice(c->cfg.device));
  DISN_CUDA_OK(cudaMemcpyAsync(host, dev, (size_t)bytes, cudaMemcpyDeviceToHost, c->stream));
  DISN_CUDA_OK(cudaStreamSynchronize(c->stream));
  return check_status(c);
}

}  // extern "C"

void disn::axis_table(double start, double stop, int num, float* out) { linspace_f32(start, stop, num, out); }

// axis tables (host float64 linspace -> float32): B*3*R floats, re-uploaded only when the boxes / resolution change (keeps
// repeated calls free of host syncs)
int disn::grid_axes(disn_ctx* c, const double* sdf_params, int B, int R) {
  const size_t axes_bytes = (size_t)8 * 3 * R * sizeof(float);
  if (axes_bytes > c->d_axes.bytes()) c->axes_key.clear();   // a new allocation holds no tables yet
  if (c->d_axes.ensure(axes_bytes)) return -1;
  std::vector<double> key(sdf_params, sdf_params + (size_t)B * 6);
  key.push_back((double)R);
  if (key != c->axes_key) {
    std::vector<float> axes((size_t)B * 3 * R);
    for (int b = 0; b < B; ++b)
      for (int a = 0; a < 3; ++a)
        linspace_f32(sdf_params[b * 6 + a], sdf_params[b * 6 + 3 + a], R, &axes[((size_t)b * 3 + a) * R]);
    DISN_CUDA_OK(cudaMemcpyAsync(c->d_axes.as<float>(), axes.data(), axes.size() * sizeof(float), cudaMemcpyHostToDevice,
                                 c->stream));
    DISN_CUDA_OK(cudaStreamSynchronize(c->stream));   // `axes` is a stack-owned staging buffer
    c->axes_key = key;
  }
  return 0;
}

namespace disn {
namespace {

constexpr int ROW_THREADS = 256;
constexpr int64_t ROW_CHUNK = (int64_t)1 << 24;   // grid points per network call (12 B of coordinates each)

// x,y,z rows of points [j0, j0 + n) from the axis tables: grid point idx[j] (an index outside the grid raises the status
// and reads point 0), or point j of the stride-s lattice.  The floats are the ones grid mode reads, so explicit-point
// evaluation of the rows gives grid mode's values.
template <class Index>
__global__ void __launch_bounds__(ROW_THREADS) grid_rows_kernel(const Index* __restrict__ idx, int64_t j0, int64_t n, int R,
                                                                int s, const float* __restrict__ axes,
                                                                float* __restrict__ xyz, int* __restrict__ status) {
  const int64_t j = (int64_t)blockIdx.x * ROW_THREADS + threadIdx.x;
  if (j >= n) return;
  int x, y, z;
  if (idx) {
    int64_t i = (int64_t)idx[j0 + j];
    if ((uint64_t)i >= (uint64_t)R * R * R) {
      atomicOr(status, DISN_STATUS_BAD_INDEX);
      i = 0;
    }
    x = (int)(i % R); y = (int)((i / R) % R); z = (int)(i / ((int64_t)R * R));
  } else {
    const int M = (R - 1) / s + 1;
    const int64_t i = j0 + j;
    x = (int)(i % M) * s; y = (int)((i / M) % M) * s; z = (int)(i / ((int64_t)M * M)) * s;
  }
  xyz[j * 3 + 0] = axes[x]; xyz[j * 3 + 1] = axes[R + y]; xyz[j * 3 + 2] = axes[2 * R + z];
}

}  // namespace

// One image of the encoded batch as a batch of one: its gbias / pmap rows, its matrix and the first axis tables.  The
// dense grid runs in grid mode; listed and lattice points go through explicit-point rows, one chunk at a time.
template <class Index>
int eval_grid_points(disn_ctx* c, int image, int R, const float* d_tm, const Index* idx, int64_t n, float* out, int s) {
  if (n == 0) return 0;
  PointJob job{};
  job.B = 1;
  job.gbias = c->gbias.as<float>() + (int64_t)image * kHidden;
  job.pmap = c->pmap.as<float>() + (int64_t)image * c->cfg.img_h * c->cfg.img_w * kHidden;
  job.trans_mat = d_tm;
  job.out_div = c->cfg.sdf_weight;
  if (!idx && s == 1) {
    job.N = n; job.R = R; job.z0 = 0; job.axes = c->d_axes.as<float>();
    job.out_pred = out;
    return run_point_job(c, job);
  }
  const int64_t chunk = std::min<int64_t>(n, ROW_CHUNK);
  if (c->d_rows.ensure((size_t)chunk * 3 * sizeof(float))) return -1;
  for (int64_t j0 = 0; j0 < n; j0 += chunk) {
    const int64_t m = std::min<int64_t>(chunk, n - j0);
    grid_rows_kernel<Index><<<(unsigned)((m + ROW_THREADS - 1) / ROW_THREADS), ROW_THREADS, 0, c->stream>>>(
        idx, j0, m, R, s, c->d_axes.as<float>(), c->d_rows.as<float>(), c->d_status.as<int>());
    c->launches++;
    DISN_CUDA_OK(cudaGetLastError());
    job.N = m; job.pts = c->d_rows.as<float>(); job.pts_rot = nullptr;
    job.out_pred = out + j0;
    if (run_point_job(c, job)) return -1;
  }
  return 0;
}
template int eval_grid_points<int32_t>(disn_ctx*, int, int, const float*, const int32_t*, int64_t, float*, int);
template int eval_grid_points<unsigned long long>(disn_ctx*, int, int, const float*, const unsigned long long*, int64_t,
                                                  float*, int);

}  // namespace disn
