// Shared declarations for the DISN library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <set>
#include <string>
#include <utility>
#include <vector>

#include "../../include/disn_b200.h"

namespace disn {

void set_error(const std::string& msg);

#define DISN_CUDA_OK(expr)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      ::disn::set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " at " + \
                        __FILE__ + ":" + std::to_string(__LINE__));                          \
      return -1;                                                                             \
    }                                                                                        \
  } while (0)

#define DISN_REQUIRE(cond, msg)                          \
  do {                                                   \
    if (!(cond)) {                                       \
      ::disn::set_error(std::string("invalid argument: ") + (msg)); \
      return -2;                                         \
    }                                                    \
  } while (0)

// Sole owner of one device (cudaMalloc) or pinned host (cudaMallocHost) allocation: move-only, freed on destruction.
template <bool Pinned>
class Buffer {
 public:
  Buffer() = default;
  Buffer(Buffer&& o) noexcept : p_(o.p_), bytes_(o.bytes_) { o.p_ = nullptr; o.bytes_ = 0; }
  Buffer& operator=(Buffer&& o) noexcept { std::swap(p_, o.p_); std::swap(bytes_, o.bytes_); return *this; }
  Buffer(const Buffer&) = delete;
  Buffer& operator=(const Buffer&) = delete;
  ~Buffer() { release(); }

  // Grow only: when `need` exceeds the capacity, drops the old allocation (its contents are NOT kept) and allocates
  // exactly need + slack bytes.  A failed allocation leaves the buffer empty and returns -1; the next call retries.
  int ensure(size_t need, size_t slack = 0) {
    if (need <= bytes_) return 0;
    release();
    void* p = nullptr;
    DISN_CUDA_OK(Pinned ? cudaMallocHost(&p, need + slack) : cudaMalloc(&p, need + slack));
    p_ = p;
    bytes_ = need + slack;
    return 0;
  }
  template <class T> T* as() const { return static_cast<T*>(p_); }
  size_t bytes() const { return bytes_; }

 private:
  void release() {
    if (p_) { if (Pinned) cudaFreeHost(p_); else cudaFree(p_); }
    p_ = nullptr;
    bytes_ = 0;
  }
  void* p_ = nullptr;
  size_t bytes_ = 0;
};
using DevBuffer = Buffer<false>;
using PinnedBuffer = Buffer<true>;

// Carves 256-byte aligned pieces out of one allocation.  With a null base every take returns nullptr and only `off`
// advances, so running the same takes first on nullptr sizes the allocation they are then carved from.
struct Arena {
  char* base;
  size_t off = 0;
  template <class T> T* take(size_t n) {
    T* p = reinterpret_cast<T*>(base ? base + off : nullptr);
    off += (n * sizeof(T) + 255) & ~(size_t)255;
    return p;
  }
};

// Lock-free union-find over an int32 parent array (mesh_clean.cu: faces; mesh_sdf.cu: grid points).
// Root of x with intermediate pointer jumping.  parent[x] <= x always holds (a root is only ever hooked under a smaller
// root), so the root of a component is its smallest face.  Concurrent jumps only replace a pointer by an ancestor.
__device__ __forceinline__ int32_t uf_find(volatile int32_t* parent, int32_t x) {
  int32_t cur = parent[x];
  if (cur != x) {
    int32_t prev = x, next;
    while (cur > (next = parent[cur])) {
      parent[prev] = next;
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

// hook the larger root under the smaller one; a failed CAS means the root moved: continue from its new parent
__device__ __forceinline__ void uf_union(int32_t* parent, int32_t a, int32_t b) {
  int32_t ra = uf_find(parent, a), rb = uf_find(parent, b);
  while (ra != rb) {
    if (ra < rb) {
      const int32_t old = atomicCAS(&parent[rb], rb, ra);
      if (old == rb) break;
      rb = old;
    } else {
      const int32_t old = atomicCAS(&parent[ra], ra, rb);
      if (old == ra) break;
      ra = old;
    }
  }
}

// Root of x by a read-only walk (for the flattening pass: a pointer-jumping store from another thread could otherwise
// overwrite the root this thread stored).
__device__ __forceinline__ int32_t uf_root(const int32_t* parent, int32_t x) {
  volatile const int32_t* p = parent;
  int32_t n;
  while ((n = p[x]) != x) x = n;
  return x;
}

struct DevTensor {
  DevBuffer buf;
  std::vector<int64_t> shape;
  int64_t numel = 0;
  float* ptr() const { return buf.as<float>(); }
};

// VGG-16 topology (reference spec: models/CNN/vgg.py:187-196)
static const int kNumConv = 13;
static const int kTapLayer[5] = {1, 3, 6, 9, 12};  // conv1_2, conv2_2, conv3_3, conv4_3, conv5_3
static const int kTapC[5] = {64, 128, 256, 512, 512};
static const int kLocalFeat = 1472;
static const int kHidden = 512;

// One stream of the point MLP (models/sdfnet.py:69-92 / :171-190) after the algebraic folds.
struct StreamWeights {
  const float* w1; const float* b1;   // fold1/conv1 [3,64]
  const float* w2; const float* b2;   // fold1/conv2 [64,256]
  const float* w3; const float* b3;   // fold1/conv3 [256,512]
  const float* w4;                    // fold2/conv1 rows 0..511 [512,512] (point-feature part)
  const float* b4;                    // fold2/conv1 biases [512] (local stream; global uses gbias)
  const float* w5; const float* b5;   // fold2/conv2 [512,256]
  const float* w6; const float* b6;   // fold2/conv5 [256,1]
};

struct PointJob {
  // inputs
  const float* pts;       // [B,N,3] or nullptr (grid mode)
  const float* pts_rot;   // [B,N,3] or nullptr (= pts)
  const float* trans_mat; // [B,4,3] device
  const float* axes;      // grid mode: [B,3,R] float32 linspace tables (x,y,z)
  int32_t R;              // grid mode: points per axis
  int32_t z0;             // grid mode: first z plane; point n is grid point z0*R^2 + n (the dense slab)
  int64_t N;              // points per image in this call
  int32_t B;
  // per-image encoder products
  const float* gbias;     // [B,512]
  const float* pmap;      // [B,img_h,img_w,512]
  const float* pfeat;     // explicit-feature decoder (get_decoder): [B,N,512] per-point folded local features replace the
                          // gather of pmap; nullptr on the fused path
  int32_t img_h, img_w;
  float clamp_max;
  float out_div;          // result divisor: 1 (eval_points) or sdf_weight (eval_grid)
  int32_t tanh_out;
  StreamWeights g, l;
  // DISN_PREC_F16F8: power-of-two multipliers of the e5m2 correction operands, [stream][layer]{(a-h(a)) scale, a scale}
  float act_scale[2][4][2];
  // outputs
  float* out_pred;        // [B,N]
  float* out_uv;          // [B,N,2] or nullptr
  float* out_global;      // [B,N] pred_sdf_value_global (raw stream output) or nullptr
  float* out_local;       // [B,N] pred_sdf_value_local or nullptr
  int* status;            // device word the kernels OR failure bits into (DISN_STATUS_*), or nullptr
};

constexpr int DISN_STATUS_FP16_OVERFLOW = 1;   // DISN_PREC_F16F8: an activation exceeded fp16's range
constexpr int DISN_STATUS_BAD_INDEX = 2;       // eval_grid_points: a listed index outside [0, R^3) (evaluated as point 0)

// query point n of image b of a point job: (x, y, z) is projected, (xr, yr, zr) feeds the MLP; zeros past the end
__device__ __forceinline__ void point_of(const PointJob& job, int b, int64_t n, float& x, float& y, float& z, float& xr,
                                         float& yr, float& zr) {
  x = y = z = xr = yr = zr = 0.f;
  if (n >= job.N) return;
  if (job.pts) {
    const float* q = job.pts + ((int64_t)b * job.N + n) * 3;
    x = q[0]; y = q[1]; z = q[2];
    if (job.pts_rot) {
      const float* r = job.pts_rot + ((int64_t)b * job.N + n) * 3;
      xr = r[0]; yr = r[1]; zr = r[2];
    } else { xr = x; yr = y; zr = z; }
  } else {
    const int R = job.R;
    const int ix = (int)(n % R);
    const int64_t tt = n / R;
    const int iy = (int)(tt % R);
    const int iz = (int)(tt / R) + job.z0;
    const float* ax = job.axes + (int64_t)b * 3 * R;
    x = ax[ix]; y = ax[R + iy]; z = ax[2 * R + iz];
    xr = x; yr = y; zr = z;
  }
}

// image coordinates of a point (models/model_normalization.py:241-251): [x,y,z,1] . T (T: [4,3], fp32 multiply-adds in
// k order like a plain matmul), divided by the depth and clamped to [0, clamp_max]
__device__ __forceinline__ void project(const float* T, float clamp_max, float x, float y, float z, float& u, float& v) {
  const float q0 = fmaf(z, T[6], fmaf(y, T[3], x * T[0])) + T[9];
  const float q1 = fmaf(z, T[7], fmaf(y, T[4], x * T[1])) + T[10];
  const float q2 = fmaf(z, T[8], fmaf(y, T[5], x * T[2])) + T[11];
  u = fminf(clamp_max, fmaxf(0.f, q0 / q2));
  v = fminf(clamp_max, fmaxf(0.f, q1 / q2));
}

// The device-resident mesh the mesh calls share: vertices [nv,3] float32 and faces [nf,3] int32 (0-based), plus a spare
// pair that cleaning compacts into.  The counts always describe arrays that are allocated and written: a writer calls
// replace(), which empties the mesh before it makes room, writes through verts() / faces() and then commit()s the counts,
// so a writer that fails in between leaves the empty mesh.  The arrays grow only, with 25 % + 1024 elements of slack.
class ResidentMesh {
 public:
  int64_t nv() const { return nv_; }
  int64_t nf() const { return nf_; }
  float* verts() const { return verts_.as<float>(); }
  int32_t* faces() const { return faces_.as<int32_t>(); }

  int replace(int64_t nv, int64_t nf) {
    clear();
    return grow(verts_, faces_, nv, nf);
  }
  void commit(int64_t nv, int64_t nf) { nv_ = nv; nf_ = nf; }
  void clear() { nv_ = nf_ = 0; }

  // room for a mesh built from the resident one; the resident mesh is untouched until swap_spare makes the spare pair
  // resident with the given counts
  int reserve_spare(int64_t nv, int64_t nf) { return grow(spare_verts_, spare_faces_, nv, nf); }
  float* spare_verts() const { return spare_verts_.as<float>(); }
  int32_t* spare_faces() const { return spare_faces_.as<int32_t>(); }
  void swap_spare(int64_t nv, int64_t nf) {
    std::swap(verts_, spare_verts_);
    std::swap(faces_, spare_faces_);
    commit(nv, nf);
  }

  // copies the mesh to host arrays of nv()*3 floats / nf()*3 int32 (an array is copied only when the mesh has entries
  // of its kind and its pointer is non-null) on `stream`, then synchronises with it
  int fetch(cudaStream_t stream, float* verts, int32_t* faces) const {
    if (nv_ && verts)
      DISN_CUDA_OK(cudaMemcpyAsync(verts, verts_.as<float>(), (size_t)nv_ * 3 * sizeof(float), cudaMemcpyDeviceToHost,
                                   stream));
    if (nf_ && faces)
      DISN_CUDA_OK(cudaMemcpyAsync(faces, faces_.as<int32_t>(), (size_t)nf_ * 3 * sizeof(int32_t),
                                   cudaMemcpyDeviceToHost, stream));
    DISN_CUDA_OK(cudaStreamSynchronize(stream));
    return 0;
  }

 private:
  static int grow(DevBuffer& verts, DevBuffer& faces, int64_t nv, int64_t nf) {
    const size_t vb = 3 * sizeof(float), fb = 3 * sizeof(int32_t);
    return verts.ensure(nv * vb, (nv / 4 + 1024) * vb) || faces.ensure(nf * fb, (nf / 4 + 1024) * fb) ? -1 : 0;
  }
  DevBuffer verts_, faces_, spare_verts_, spare_faces_;
  int64_t nv_ = 0, nf_ = 0;
};

}  // namespace disn

// Every allocation of the context is a buffer member: deleting the context frees them all.
struct disn_ctx {
  ~disn_ctx();                  // destroys the encoder graph and the stream if the context owns it (api.cu)
  disn_config cfg;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  std::map<std::string, disn::DevTensor> weights;
  bool weights_dirty = true;
  int64_t launches = 0;
  int num_sms = 132;            // cudaDevAttrMultiProcessorCount of cfg.device, read once in disn_create
  bool attr_conv_tc = false, attr_point_fp32 = false;   // cudaFuncSetAttribute done on this device
  std::set<const void*> attr_done;                      // ... for the point_tc_kernel instantiations

  // encoder state
  int32_t enc_B = 0;
  int32_t alloc_B = 0;          // batch the encoder buffers are sized for
  disn::DevBuffer img_in;       // [B,H,W,3] as uploaded
  disn::DevBuffer img_rs;       // [B,224,224,3]
  disn::DevBuffer act[2];       // ping-pong activations
  disn::DevBuffer taps[5];
  disn::DevBuffer proj[5];      // per-level projected maps [B,h,h,512]
  disn::DevBuffer fc_a;         // [B,4096]
  disn::DevBuffer fc_b;         // [B,4096]
  disn::DevBuffer partial;      // split-K partials (fc layers)
  disn::DevBuffer splitk_ws;    // split-K partials (conv / projection GEMMs)
  disn::DevBuffer emb;          // [B,num_classes]
  disn::DevBuffer gbias;        // [B,512]
  disn::DevBuffer pmap;         // [B,img_h,img_w,512]
  cudaGraphExec_t enc_graph_exec = nullptr;   // captured encoder launch sequence (encoder_run)
  std::vector<int64_t> enc_graph_key, enc_warm_key;
  int64_t enc_graph_launches = 0;
  // scratch for host-pointer calls
  disn::DevBuffer d_pts, d_pts_rot, d_out, d_uv;
  disn::DevBuffer d_tm;         // [max_batch,4,3]
  disn::DevBuffer d_status;     // device status word (PointJob::status)
  disn::PinnedBuffer h_status;  // pinned host mirror, copied behind every point-kernel launch
  disn::DevBuffer d_axes;       // [max_batch,3,R]
  std::vector<double> axes_key; // (sdf_params, R) the tables in d_axes were built from
  // bf16x3 packed weights (tensor-core path)
  disn::DevBuffer tc_weights;          // bf16 hi/lo stage images of the point MLP (DISN_PREC_BF16X3)
  disn::DevBuffer tc_weights_f8;       // fp16 + e5m2 stage images (DISN_PREC_F16F8)
  float tc_act_scale[2][4][2] = {};
  std::map<std::string, disn::DevBuffer> enc_tc_weights;   // packed bf16 hi/lo stage images of the encoder GEMMs
  // the mesh that marching cubes, the coarse-to-fine mesher, mesh_load and the OBJ reader write and the other mesh calls
  // read or change in place
  disn::ResidentMesh mesh;
  // marching cubes: persistent scratch (mc.cu)
  disn::DevBuffer mc_code, mc_vbase, mc_chunk, mc_sums, mc_totals;
  disn::PinnedBuffer mc_totals_host;
  // small-part cleaning of the resident mesh (mesh_clean.cu): scratch arena and the totals read back once per clean; both
  // grow only
  disn::DevBuffer cl_arena;
  disn::PinnedBuffer cl_totals_host;
  // signed distance field of the resident mesh (mesh_sdf.cu): scratch arena (BVH, edge bits, union-find parents, the
  // distance grid of host-output calls), pinned staging (mesh statistics, axis tables) and the phase timing events
  disn::DevBuffer sdf_arena;
  disn::PinnedBuffer sdf_host;
  cudaEvent_t sdf_ev[5] = {};
  float sdf_phase_ms[4] = {};
  // resident field of the preprocessing chain (disn_field): mesh_sdf writes it, marching cubes and the samplers read it
  disn::DevBuffer d_field;
  // surface-sample normalisation (mesh_normalize.cu): scratch arena and pinned statistics words
  disn::DevBuffer nm_arena;
  disn::PinnedBuffer nm_host;
  // band / strided sampling of a field (sdf_sample.cu): host-field staging, flags and scan scratch, the four compacted
  // index lists, their counts, and the gather staging; smp_src / smp_R / smp_n describe the lists of the last band count
  disn::DevBuffer smp_in, smp_flag, smp_scan, smp_list, smp_counts, smp_gather;
  disn::PinnedBuffer smp_host;
  const float* smp_src = nullptr;
  int32_t smp_R = 0;
  int64_t smp_n[4] = {};
  // device-resident SDF grid of disn_eval_grid_resident and host staging for the marching-cubes input
  disn::DevBuffer d_grid;
  disn::DevBuffer d_idx;        // host-index staging of disn_eval_grid_indexed
  disn::DevBuffer d_rows;       // eval_grid_points: x,y,z rows of one chunk of listed grid points
  // coarse-to-fine refinement (adaptive.cu), one set for the grid and the mesher: block states of every level, the coarse
  // lattice values, each level's active blocks, the sort buffers of the level lists (the mesher's crossing cells reuse
  // them), sort scratch, the network's value chunk, device counters with their pinned mirror
  disn::DevBuffer ad_state, ad_coarse, ad_active[4], ad_keys[2], ad_sort_tmp, ad_vals, ad_cnt;
  disn::PinnedBuffer ad_host;
  // coarse-to-fine grid (adaptive.cu): the filled grid, one byte per point (1 = evaluated), host-field staging and the
  // phase events; ad_R / ad_levels describe the last call
  disn::DevBuffer ad_grid, ad_mark, ad_field;
  cudaEvent_t ad_ev[7] = {};
  int32_t ad_R = 0, ad_levels = 0;
  disn::DevBuffer d_mc_in;
  // coarse-to-fine mesh without a dense grid (adaptive_mesh.cu): each level's value table, the crossing edges, cases and
  // face offsets of the cells, scan scratch and the phase events.  am_nv: vertices of the last call (-1: none or failed),
  // am_edges_sorted: its sorted crossing edges (vertex v = edge of rank v)
  disn::DevBuffer am_table[4], am_edges[2], am_case, am_tri, am_sums;
  cudaEvent_t am_ev[4] = {};
  int64_t am_nv = -1;
  const unsigned long long* am_edges_sorted = nullptr;
  // OBJ reader (obj_read.cu): the file's bytes in pinned staging and on the device, the per-line arrays (line starts,
  // record types, scanned counts, usemtl max-scan, select / scan scratch), the per-face and per-coordinate lists (face
  // materials, host-converted coordinates), counters with their pinned mirror, the host side of the coordinate list, the
  // per-face part ids and the part names of the last read (obj_none: the part of the faces before any usemtl), phase
  // events and times (upload, line starts, classify, parse; host conversion and parts in [4])
  disn::PinnedBuffer obj_host;
  disn::DevBuffer obj_bytes, obj_arena, obj_lists, obj_small;
  disn::PinnedBuffer obj_small_host, obj_list_host, obj_part_ids;
  std::vector<std::string> obj_names;
  std::vector<bool> obj_none;
  bool obj_parts_ready = false;
  int64_t obj_part_faces = 0, obj_host_tokens = 0, obj_overflows = 0;
  cudaEvent_t obj_ev[5] = {};
  float obj_phase_ms[5] = {};
  // nn_distance / cam scratch (persistent, grows)
  disn::DevBuffer nn_scratch;
  disn::DevBuffer dec_scratch;  // explicit-feature decoder staging (decoder.cu)
  disn::DevBuffer d_gt, d_acc;  // disn_sdf_metrics: host-call staging of the samples' values and the per-image sums
};

namespace disn {
// encoder.cu
int encoder_alloc(disn_ctx* c, int B);
int encoder_run(disn_ctx* c, const float* imgs, int B, int H, int W, int C, bool device_ptr,
                bool embedding_only = false);
void encoder_graph_reset(disn_ctx* c);
// api.cu
int run_point_job(disn_ctx* c, PointJob& job);    // fills weights / encoder products / status and launches per cfg.precision
int ensure_point_scratch(disn_ctx* c, int64_t pts);
int check_status(disn_ctx* c);    // after a synchronisation: the kernels' status bits as an error (and clears them)
// encoder.cu helpers reused by the explicit-feature decoder
int encoder_gemv(disn_ctx* c, const float* x, const float* W, const float* bias, float* out, int B, int K, int N, int relu);
int encoder_gemm_plain(disn_ctx* c, const std::string& wname, const float* A, const float* Bm, const float* bias, float* C,
                       int M, int N, int K, int relu);
// point_fp32.cu
int launch_point_fp32(disn_ctx* c, const PointJob& job);
// point_tc.cu
int tc_pack_weights(disn_ctx* c);
int launch_point_tc(disn_ctx* c, const PointJob& job);
// conv_tc.cu
int conv_tc_pack(disn_ctx* c, const float* d_w, int K, int N, DevBuffer& out);
int launch_conv_tc(disn_ctx* c, const float* A, const uint8_t* wpk, const float* bias, float* C, float* ws,
                   int64_t ws_elems, int M, int N, int K, int H, int W, int Cin, int relu, int* splits_out);
// cam.cu
// the pose heads on the embeddings d_emb [B, num_classes] (device) -> pred_RT and pred_trans_mat [B,4,3] (device)
int launch_cam_heads(disn_ctx* c, int B, const float* d_emb, const float* d_K, float* d_rt, float* d_tm);
// the embedding-only encode of host imgs [B,H,W,C], then the heads with intrinsics K (host float[9], NULL = the reference's
// constant) staged in d_K: pred_RT and pred_trans_mat [B,4,3] in the caller's device buffers (disn_cam_estimate/_metrics)
int cam_predict(disn_ctx* c, const float* imgs, int B, int H, int W, int C, const float* K, float* d_K, float* d_rt,
                float* d_tm);
// chamfer.cu
int nn_distance(disn_ctx* c, const float* d_xyz1, int n, const float* d_xyz2, int m, int B, float* d_dist1,
                int* d_idx1, float* d_dist2, int* d_idx2);
// mc.cu: the mesh of d_sdf [R,R,R] (3 R^3 < 2^32) becomes the resident mesh
int mc_run(disn_ctx* c, const float* d_sdf, int R, const double* bbox, float iso);
// in-place exclusive scan of d[0..n) on c->stream, total -> *d_total (device); `sums` = scan_scratch_elems(n) words
int64_t scan_scratch_elems(int64_t n);
int exclusive_scan(disn_ctx* c, uint32_t* d, int64_t n, uint32_t* d_total, uint32_t* sums);
// mesh_clean.cu: uploads a host mesh whose arguments disn_mesh_load accepted
int mesh_load(disn_ctx* c, const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces);
int mesh_clean(disn_ctx* c, double dist_thresh, double num_thresh, int32_t* face_component, int64_t* n_components,
               int64_t* n_kept, int64_t* n_verts, int64_t* n_faces);
// mesh_sdf.cu
int mesh_sdf(disn_ctx* c, int32_t res, const double* bbox, double expand_rate, double sigma, float* out,
             double* bbox_out, bool device_out);
// mesh_normalize.cu
int mesh_part_areas(disn_ctx* c, const int32_t* part_ids, int32_t n_parts, int64_t* part_q, int32_t* shift);
int mesh_normalize(disn_ctx* c, const int32_t* part_ids, int32_t n_parts, const int64_t* amounts, const double* draws,
                   int64_t n_draws, const double* given, double* centroid_out, double* m_out, double* samples_out);
// sdf_sample.cu
int band_count(disn_ctx* c, const float* sdf, int32_t R, float iso, const float* edges, bool device_ptr, int64_t* counts);
int band_gather(disn_ctx* c, const float* axes, const int64_t* choices, const int64_t* k, float* out);
int sdf_strided(disn_ctx* c, const float* sdf, int32_t R, int32_t reduce, bool device_ptr, float* out);
// api.cu: numpy.linspace(start, stop, num) in float64 cast to float32 (the grid coordinates of eval_grid and mesh_sdf)
void axis_table(double start, double stop, int num, float* out);
// api.cu: the float32 axis tables of B boxes in c->d_axes (uploaded only when boxes or R change)
int grid_axes(disn_ctx* c, const double* sdf_params, int B, int R);
// api.cu: n grid points of encoded image `image` -> out[0..n) (device) = pred/sdf_weight, bitwise disn_eval_grid's values.
// Point j is grid point idx[j] = (z*R + y)*R + x (device; Index = int32_t or unsigned long long), or with idx == nullptr
// point j of the stride-s lattice in (z, y, x) order (s = 1: the dense grid).  The axis tables of the image's box must be
// in c->d_axes (grid_axes with B = 1); d_tm: the image's [4,3] matrix on the device.  A listed index outside [0, R^3)
// raises DISN_STATUS_BAD_INDEX and is evaluated as point 0.
template <class Index>
int eval_grid_points(disn_ctx* c, int image, int R, const float* d_tm, const Index* idx, int64_t n, float* out, int s = 1);
// adaptive.cu: coarse-to-fine grid of one image; values come from `field` (device [R,R,R]) when it is non-null, else from
// the network (eval_grid_points, with d_tm and the axis tables as above).  The filled grid stays in c->ad_grid, the
// evaluated-point marks in c->ad_mark.
int adaptive_run(disn_ctx* c, const float* field, int image, const float* d_tm, int32_t res, const double* sdf_params,
                 float iso, double band, int64_t* level_counts, int32_t* n_levels);
// adaptive_mesh.cu: the mesh of adaptive_run's grid followed by mc_run, built from the surface blocks alone (s0 >= 2);
// field / image / d_tm as for adaptive_run.  The mesh becomes the resident mesh (c->mesh).
int adaptive_mesh_run(disn_ctx* c, const float* field, int image, const float* d_tm, int32_t res, const double* sdf_params,
                      float iso, double band, int64_t* level_counts, int32_t* n_levels);
// api.cu: the end of a call that builds the resident mesh from rc: empties the mesh on failure, reports its counts
int finish_mesh_call(disn_ctx* c, int rc, int64_t* n_verts, int64_t* n_faces);
// bytes held by the buffers of adaptive_mesh_run
size_t adaptive_mesh_bytes(const disn_ctx* c);
// obj_read.cu: one OBJ coordinate token -> float32 as Python's float() and numpy's float64 -> float32 cast (-1 outside the
// reader's grammar; *overflow set when a finite value becomes a float32 infinity)
int obj_token_to_float(const char* s, int64_t len, float* out, bool* overflow);
}  // namespace disn
