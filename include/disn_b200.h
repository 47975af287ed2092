/*
 * disn_b200.h -- C ABI of the H100-native (sm_90a) DISN SDF-inference hot path.
 *
 * The reference has no FFI on this path (it is a Python-built TF-1.x graph); the entry points
 * below are what a replacement of that graph binds, one per reference call site
 * (paths relative to the reference repo):
 *
 *   disn_create / disn_destroy      <-> tf.Session + model.get_model graph build
 *                                       (test/create_sdf.py:152-176, models/model_normalization.py:47)
 *   disn_load_weight                <-> tf.train.Saver.restore by variable name (test/create_sdf.py:180-192);
 *                                       names/shapes = SURVEY.md 8a "checkpoint variable names"
 *   disn_encode                     <-> image resize + vgg_16 + 5 tap resizes
 *                                       (models/model_normalization.py:65-77,171-183; models/CNN/vgg.py:182-218)
 *   disn_eval_points                <-> one sess.run([pred_sdf, ref_img, sample_img_points], feed_dict)
 *                                       (test/create_sdf.py:262-275): get_img_points (:241-251), resampler x5,
 *                                       sdfnet.get_sdf_basic2 (models/sdfnet.py:69-92),
 *                                       sdfnet.get_sdf_basic2_imgfeat_twostream (:171-190), sum, optional tanh
 *   disn_eval_grid                  <-> the whole chunk loop of test_one_epoch (test/create_sdf.py:241-285):
 *                                       linspace/meshgrid grid, SPLIT_SIZE sess.runs, reassembly, /SDF_WEIGHT
 *   disn_write_dist                 <-> to_binary (test/create_sdf.py:292-303)
 *   disn_marching_cubes(+_to_obj)   <-> os.system("./isosurface/computeMarchingCubes <dist> <obj> -i <iso>")
 *                                       (test/create_sdf.py:319-323)
 *
 * Conventions: every function returns 0 on success, non-zero on failure with a thread-local message
 * in disn_last_error(); the caller owns all buffers; all tensors are float32, row-major, NHWC / [B,N,C]
 * exactly as the reference feeds them.  Pointers are HOST pointers unless DISN_DEVICE_PTR is set in
 * `flags`, in which case points / trans_mat / outputs are device pointers on the context's device and
 * the call is asynchronous on the context's stream.  One context = one CUDA device + one stream;
 * a context is not thread-safe, distinct contexts are independent.
 */
#ifndef DISN_B200_H
#define DISN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct disn_ctx disn_ctx;

enum {
  DISN_DEVICE_PTR = 1,   /* data pointers are device pointers; call is async on the ctx stream */
};

/* arithmetic used by the fused point kernel */
enum {
  DISN_PREC_FP32 = 0,    /* CUDA-core fp32 FMA (exact restatement of the reference arithmetic) */
  DISN_PREC_BF16X3 = 1,  /* tensor cores (wgmma), bf16 hi/lo split operands, 3 MMAs per product, fp32 accumulate */
  DISN_PREC_F16F8 = 2,   /* wgmma: fp16 main product + two e5m2 (2x rate) correction products, fp32
                            accumulate: 2 MMA-units per product instead of 3; activations must stay below 65504 */
};

typedef struct disn_config {
  int32_t device;        /* CUDA device ordinal */
  int32_t img_h, img_w;  /* FLAGS.img_h / img_w (137): size the feature taps are resized to */
  int32_t vgg_in;        /* get_model img_size (224) */
  int32_t num_classes;   /* FLAGS.num_classes (1024): width of the global embedding */
  float clamp_max;       /* 136.0: upper clamp of projected pixel coordinates */
  float sdf_weight;      /* SDF_WEIGHT (10.0): eval_grid divides by it */
  int32_t tanh_out;      /* FLAGS.tanh */
  int32_t precision;     /* DISN_PREC_* */
  int32_t max_batch;     /* images per encode call the context pre-allocates for (>=1) */
} disn_config;

void disn_default_config(disn_config* cfg);

int disn_create(const disn_config* cfg, disn_ctx** out);
void disn_destroy(disn_ctx* ctx);
const char* disn_last_error(void);

/* Run the ctx on an externally owned CUDA stream (cudaStream_t passed as void*). NULL = own stream. */
int disn_set_stream(disn_ctx* ctx, void* cuda_stream);
int disn_synchronize(disn_ctx* ctx);
int disn_set_precision(disn_ctx* ctx, int32_t precision);

/* Weights by TF variable name, HWIO layout as TF stores them. Host pointer. Missing variables keep
 * their previous value (zero on a fresh context), mirroring the reference's tolerant restore. */
int disn_load_weight(disn_ctx* ctx, const char* name, const float* data, const int64_t* shape, int32_t ndim);
/* Re-derive the packed / split forms the kernels read (call after the last disn_load_weight). */
int disn_finalize_weights(disn_ctx* ctx);

/* imgs: [B,H,W,C] (C = 3; H,W = 137 or vgg_in), host pointer (synchronous) or, with DISN_DEVICE_PTR,
 * device pointer (asynchronous on the ctx stream). Keeps per-image features on the device. */
int disn_encode(disn_ctx* ctx, const float* imgs, int32_t B, int32_t H, int32_t W, int32_t C, uint32_t flags);
/* Fetch encoder products to host (tests / get_model end_points).
 * what: 0 = img_embedding [B,num_classes]; 1..5 = raw VGG tap conv{1_2,2_2,3_3,4_3,5_3} [B,h,h,C];
 *       6 = projected local map [B,img_h,img_w,512]; 7 = global-stream folded bias [B,512];
 *       8 = resized input image [B,vgg_in,vgg_in,3]. */
int disn_get_encoded(disn_ctx* ctx, int32_t what, float* out, int64_t out_elems);

/* One sess.run: pts[B,N,3] (projection input, `sample_pc`), pts_rot[B,N,3] (MLP input, `sample_pc_rot`;
 * NULL = same as pts), trans_mat[B,4,3] -> out_pred[B,N,1] (=pred_sdf, NOT divided by sdf_weight),
 * out_uv[B,N,2] (=sample_img_points) or NULL. B must equal the last disn_encode batch. */
int disn_eval_points(disn_ctx* ctx, const float* pts, const float* pts_rot, const float* trans_mat,
                     int32_t B, int64_t N, float* out_pred, float* out_uv, uint32_t flags);

/* Dense grid: sdf_params host double[B,6] = [xmin,ymin,zmin,xmax,ymax,zmax], trans_mat [B,4,3],
 * resolution R = sdf_res+1 points per axis, z-planes [z0,z1) -> out_sdf[B,(z1-z0),R,R] = pred/sdf_weight
 * (x fastest, z slowest, i.e. the reference's reassembled `result`). Grid coordinates are generated on
 * the device from float64 linspace tables cast to float32, bit-identical to the reference's host grid. */
int disn_eval_grid(disn_ctx* ctx, const double* sdf_params, const float* trans_mat, int32_t B,
                   int32_t sdf_res, int32_t z0, int32_t z1, float* out_sdf, uint32_t flags);

/* .dist writer: int32 {-res,res,res}, double bbox[6], float32 values[(res+1)^3]. Host values. */
int disn_write_dist(const char* path, int32_t res, const double* bbox, const float* values);

/* OBJ writer in the conventions of the reference's mesher output (demo/result.obj): comment header with
 * the counts, `v x y z` (%g), 1-based `f i j k`. Host arrays; faces are 0-based on input. */
int disn_write_obj(const char* path, const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces);

/* Marching cubes of sdf[R,R,R] (z,y,x) at iso over bbox. Two-call protocol: pass verts=faces=NULL to
 * get counts, then call again with buffers of n_verts*3 floats / n_faces*3 int32 (0-based).
 * sdf is a host pointer unless DISN_DEVICE_PTR. Vertices are welded (shared per grid edge) and ordered
 * by (z,y,x,axis) of their edge; faces by cell index. */
int disn_marching_cubes(disn_ctx* ctx, const float* sdf, int32_t R, const double* bbox, float iso,
                        float* verts, int64_t* n_verts, int32_t* faces, int64_t* n_faces, uint32_t flags);

/* Device-resident variant of the driver's tail (test/create_sdf.py:277-323 without the .dist round trip through the
 * file system): disn_eval_grid_resident leaves the whole [B,R,R,R] grid (pred/sdf_weight) in HBM and returns its device
 * address (valid until the next call on this context); disn_mc_run meshes one [R,R,R] field (device pointer with
 * DISN_DEVICE_PTR, e.g. grid + b*R^3, or a host array) and keeps the welded mesh in HBM; disn_mc_fetch copies it to host
 * buffers of n_verts*3 floats / n_faces*3 int32; disn_mc_write_obj writes it in disn_write_obj's format; disn_fetch is
 * a synchronous device->host copy on the context's stream (e.g. to keep the .dist artefact). */
int disn_eval_grid_resident(disn_ctx* ctx, const double* sdf_params, const float* trans_mat, int32_t B,
                            int32_t sdf_res, float** out_dev);
int disn_mc_run(disn_ctx* ctx, const float* sdf, int32_t R, const double* bbox, float iso, uint32_t flags,
                int64_t* n_verts, int64_t* n_faces);
int disn_mc_fetch(disn_ctx* ctx, float* verts, int32_t* faces);
int disn_mc_write_obj(disn_ctx* ctx, const char* path);
int disn_fetch(disn_ctx* ctx, const void* dev, void* host, int64_t bytes);

/* Estimated-camera path (reference: demo/demo.py:195-258 cam_evl, cam_est/model_cam.py:47-109, models/posenet.py:91-124):
 * imgs host [B,H,W,3] -> VGG-16 embedding (the context's `vgg_16/...` weights = the camera checkpoint's) -> three FC
 * heads (`cameraprediction/{scale,ortho6d,translation}/fc{1,2,3}/{weights,biases}`) -> pred_RT [B,4,3] (or NULL) and
 * pred_trans_mat = pred_RT . K^T [B,4,3].  K: host float[9] row-major intrinsics, NULL = the reference constant
 * [[149.84375,0,68.5],[0,149.84375,68.5],[0,0,1]] (cam_est/model_cam.py:28). */
int disn_cam_estimate(disn_ctx* ctx, const float* imgs, int32_t B, int32_t H, int32_t W, int32_t C, const float* K,
                      float* out_rt, float* out_trans_mat);

/* Chamfer nearest-neighbour distances, the reference's NnDistance op (models/tf_ops/nn_distance/tf_nndistance.cpp:
 * 21-43; called at test/test_cd_emd.py:300, test/test_f_score.py:253): xyz1 [B,N,3], xyz2 [B,M,3] host float32 ->
 * dist1 [B,N] (squared L2 to the nearest point of xyz2), idx1 [B,N] int32, dist2 [B,M], idx2 [B,M].
 * Bit-identical to the reference CPU kernel (float32 arithmetic, first minimum wins). */
int disn_nn_distance(disn_ctx* ctx, const float* xyz1, const float* xyz2, int32_t B, int32_t N, int32_t M,
                     float* dist1, int32_t* idx1, float* dist2, int32_t* idx2);

/* Approximate earth mover's distance, the reference's ApproxMatch / MatchCost ops (models/tf_ops/approxmatch/
 * tf_approxmatch.cpp:23-85, 86-107; called at test/test_cd_emd.py:307-308): xyz1 [B,N,3], xyz2 [B,M,3] host float32.
 * disn_approx_match -> match [B,N,M] float32 (element (k,l): mass moved from point k of xyz1 to point l of xyz2 -- the CPU
 * op's k*M+l indexing) and/or cost [B] = MatchCost of that match; either output may be NULL (cost only: `match` never leaves
 * HBM).  disn_match_cost = the MatchCost op for a caller-supplied match.  Same arithmetic as the reference CPU kernels
 * (float64 sums in a fixed order, expf of a float32 exponent): equal to them within the float64 summation order. */
int disn_approx_match(disn_ctx* ctx, const float* xyz1, const float* xyz2, int32_t B, int32_t N, int32_t M,
                      float* match_out, float* cost_out);
int disn_match_cost(disn_ctx* ctx, const float* xyz1, const float* xyz2, const float* match, int32_t B, int32_t N, int32_t M,
                    float* cost);

/* Multi-GPU result gather without a collective (one process per GPU, SURVEY.md 8e "peer-direct stores from the kernel
 * epilogue into the root's buffer"): rank 0 calls disn_shared_alloc (cudaMalloc + CUDA IPC handle, 64 bytes), ships the
 * handle to the other ranks, which disn_shared_open it and pass `ptr + byte offset of their z-slab` as the
 * DISN_DEVICE_PTR output of disn_eval_grid: the fused kernel then writes each SDF value over NVLink into rank 0's HBM.
 * disn_shared_close: owner = 1 frees (rank 0), owner = 0 unmaps (the others). */
int disn_shared_alloc(disn_ctx* ctx, int64_t bytes, void** dev_ptr, unsigned char* handle64);
int disn_shared_open(disn_ctx* ctx, const unsigned char* handle64, void** dev_ptr);
int disn_shared_close(disn_ctx* ctx, void* dev_ptr, int32_t owner);

/* IoU evaluator of the reference (test/test_iou.py:208-233 iou_pymesh): both triangle meshes (host float32 verts
 * [nv,3], int32 0-based faces [nf,3]) are voxelised at cell 2/dim (restated pymesh.VoxelGrid: a cell centred at k*cell is
 * occupied iff it overlaps a triangle), the corners of the occupied cells are binned with ((v+1.1)/2.4*dim) truncated, and
 * the counts of the AND / OR of the two dim^3 occupancy grids are returned (IoU = intersection / union; dim = 110 in the
 * reference).  occ1_out / occ2_out: optional uint8[dim^3] copies of the occupancy grids (index order [x][y][z]). */
int disn_iou(disn_ctx* ctx, const float* verts1, int64_t nv1, const int32_t* faces1, int64_t nf1, const float* verts2,
             int64_t nv2, const int32_t* faces2, int64_t nf2, int32_t dim, int64_t* intersection, int64_t* uni,
             uint8_t* occ1_out, uint8_t* occ2_out);

/* Graph intermediates and the encoder/decoder split point of the reference (models/model_normalization.py:38-45,169-206,
 * 223-238); host pointers, synchronous, not the hot path:
 *   disn_eval_points_ex  = disn_eval_points + out_global / out_local [B,N,1] (end_points['pred_sdf_value_global'/'_local']);
 *   disn_point_img_feat  = end_points['point_img_feat'] [B,N,1472] (5x resize-to-137 + resampler, concat conv1..conv5)
 *                          and sample_img_points [B,N,2] (or NULL) for pts [B,N,3], trans_mat [B,4,3]; needs disn_encode;
 *   disn_eval_features   = get_decoder: pts_rot [B,N,3], global_feat [B,num_classes], point_feat [B,N,1472] -> out_pred
 *                          [B,N,1] = global + local (raw: no tanh, no /sdf_weight), out_global / out_local or NULL;
 *                          needs the weights only. flags must be 0. */
int disn_eval_points_ex(disn_ctx* ctx, const float* pts, const float* pts_rot, const float* trans_mat, int32_t B, int64_t N,
                        float* out_pred, float* out_uv, float* out_global, float* out_local);
int disn_point_img_feat(disn_ctx* ctx, const float* pts, const float* trans_mat, int32_t B, int64_t N, float* out_feat,
                        float* out_uv);
int disn_eval_features(disn_ctx* ctx, const float* pts_rot, const float* global_feat, const float* point_feat, int32_t B,
                       int64_t N, float* out_pred, float* out_global, float* out_local, uint32_t flags);

/* Kernel launch counter (bench's gpu_launches): number of this library's kernels launched so far. */
int64_t disn_launch_count(disn_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* DISN_B200_H */
