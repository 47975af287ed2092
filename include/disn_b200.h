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
 *   disn_mesh_load / disn_mesh_clean <-> clean_single_mesh (postprocessing/clean_smallparts.py:38-54):
 *                                       pymesh.separate_mesh, keep rule, pymesh.merge_meshes
 *   disn_mesh_sdf                   <-> os.system("computeDistanceField <obj> res res res -s -e <e> -o X.dist -m 1 [-g s]")
 *                                       (preprocessing/create_point_sdf_grid.py:200-210)
 *   disn_mesh_part_areas / disn_mesh_normalize <-> get_normalize_mesh (preprocessing/create_point_sdf_grid.py:169-198)
 *   disn_obj_read / disn_obj_parts  <-> pymesh.load_mesh (test/test_cd_emd.py:180-250, test/test_iou.py:210,220,
 *                                       postprocessing/clean_smallparts.py:28,39) and trimesh.load_mesh(process=False)
 *                                       (preprocessing/create_point_sdf_grid.py:172, create_point_sdf_fullgrid.py:166)
 *   disn_field / disn_sdf_band_count / disn_sdf_band_gather <-> the field between create_one_sdf, create_one_cube_obj
 *                                       and sample_sdf (:74-113, :200-252); disn_sdf_strided <-> the strided sample_sdf
 *                                       of create_point_sdf_fullgrid.py:70-96
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

enum {
  DISN_OBJ_PARTS = 1,               /* disn_obj_read: also record per-face material parts for disn_obj_parts */
  DISN_ERR_OBJ_UNSUPPORTED = -5,    /* disn_obj_read: the file cannot be opened, lies outside the reader's grammar or is
                                       invalid; disn_last_error() names the path, the line and the reason */
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
  int32_t img_h, img_w;  /* FLAGS.img_h / img_w (137): size the feature taps are resized to;
                            disn_create refuses img_h * img_w * 512 >= 2^31 */
  int32_t vgg_in;        /* get_model img_size (224) */
  int32_t num_classes;   /* FLAGS.num_classes (1024): width of the global embedding */
  float clamp_max;       /* 136.0: upper clamp of projected pixel coordinates (the reference's constant, whatever
                            img_h / img_w are) */
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
 * DISN_DEVICE_PTR, e.g. grid + b*R^3, or a host array; 2 <= R and 3 R^3 < 2^32) and keeps the welded mesh in HBM as the
 * resident mesh.  Once its arguments are accepted, *n_verts / *n_faces (each may be NULL) receive the resident mesh's
 * counts, also on failure: a failed call (out of memory, a CUDA error) leaves the resident mesh empty.  disn_mc_fetch
 * copies the resident mesh to host buffers of n_verts*3 floats / n_faces*3 int32; disn_mesh_counts reports its counts
 * from host-side state (no device work, no synchronisation); disn_mc_write_obj writes it in disn_write_obj's format;
 * disn_fetch is a synchronous device->host copy on the context's stream (e.g. to keep the .dist artefact). */
int disn_eval_grid_resident(disn_ctx* ctx, const double* sdf_params, const float* trans_mat, int32_t B,
                            int32_t sdf_res, float** out_dev);

/* Indexed grid: the grid points idx[0..n) (int32 linear indices (z*R + y)*R + x, any order, R = sdf_res+1, R^3 < 2^31) of
 * encoded image `image`, with sdf_params host double[6] (that image's box) and trans_mat [4,3] -> out[n] = pred/sdf_weight.
 * Every value is bitwise the value disn_eval_grid produces at that point, in every precision.  idx, trans_mat and out are
 * host pointers (indices checked on the host), or device pointers with DISN_DEVICE_PTR (asynchronous; an index outside
 * the grid is reported by the next synchronising call).  The DISN_PREC_F16F8 overflow status works as for disn_eval_grid. */
int disn_eval_grid_indexed(disn_ctx* ctx, const double* sdf_params, const float* trans_mat, int32_t image, int32_t sdf_res,
                           const int32_t* idx, int64_t n, float* out, uint32_t flags);

/* Coarse-to-fine grid of encoded image `image` (DESIGN.md 4.9): the network is evaluated on the stride-s0 lattice (s0 =
 * the largest power of two <= 16 dividing sdf_res) and then only inside blocks whose corners straddle iso or lie within
 * band * (s/2) * |h| of it; every other point is the trilinear interpolation of an inactive block's corners.  The complete
 * [R,R,R] grid stays in HBM (*grid_dev, valid until the next call; mesh it with disn_mc_run and DISN_DEVICE_PTR).  For a
 * 1-Lipschitz field and band >= 1 its marching-cubes mesh equals the dense grid's; band = +inf evaluates every point.
 * sdf_params host double[6], trans_mat host [4,3]; level_counts (at least 5 entries) receives the points evaluated by
 * the coarse lattice and by each level, *n_levels their number.  iso must be finite and band >= 0.  Synchronises once
 * per level. */
int disn_eval_grid_adaptive(disn_ctx* ctx, const double* sdf_params, const float* trans_mat, int32_t image,
                            int32_t sdf_res, float iso, double band, float** grid_dev, int64_t* level_counts,
                            int32_t* n_levels);
/* Coarse-to-fine mesh of encoded image `image` without a dense grid (DESIGN.md 4.10): the levels of
 * disn_eval_grid_adaptive, with the evaluated values kept in tables proportional to their number, then marching cubes on
 * the cells that can cross iso only.  The welded mesh becomes the resident mesh (disn_mc_fetch, disn_mc_write_obj,
 * disn_mesh_clean) and equals, bit for bit, the mesh disn_mc_run makes of disn_eval_grid_adaptive's grid: vertices, faces,
 * their order and level_counts (at least 5 entries; *n_levels their number), in every precision and for every band.
 * 1 <= sdf_res <= 2048, iso finite, band >= 0.  An odd sdf_res (s0 = 1) evaluates the dense grid as
 * disn_eval_grid_adaptive does and needs sdf_res <= 1125.  Refuses meshes with 2^31 or more vertices or faces.  Once the
 * arguments are accepted, *n_verts / *n_faces (each may be NULL) receive the resident mesh's counts, also on failure: a
 * failed call (out of memory, a refused size, the DISN_PREC_F16F8 overflow status) leaves the resident mesh empty.
 * Synchronises once per level and twice for the mesh. */
int disn_mesh_grid_adaptive(disn_ctx* ctx, const double* sdf_params, const float* trans_mat, int32_t image,
                            int32_t sdf_res, float iso, double band, int64_t* level_counts, int32_t* n_levels,
                            int64_t* n_verts, int64_t* n_faces);
int disn_mc_run(disn_ctx* ctx, const float* sdf, int32_t R, const double* bbox, float iso, uint32_t flags,
                int64_t* n_verts, int64_t* n_faces);
int disn_mc_fetch(disn_ctx* ctx, float* verts, int32_t* faces);
int disn_mesh_counts(disn_ctx* ctx, int64_t* n_verts, int64_t* n_faces);
int disn_mc_write_obj(disn_ctx* ctx, const char* path);
int disn_fetch(disn_ctx* ctx, const void* dev, void* host, int64_t bytes);

/* Small-part removal, the reference's clean_single_mesh (postprocessing/clean_smallparts.py:38-54), on the resident mesh
 * of disn_mc_run / disn_mesh_load; disn_mc_fetch and disn_mc_write_obj then return the cleaned mesh.
 *   disn_mesh_load: uploads a host mesh (verts [n_verts,3] float32, faces [n_faces,3] int32 0-based) into that slot; a
 *     face index outside [0, n_verts) is an error and leaves the resident mesh as it was.  Once the arguments are
 *     accepted, a failed call (out of memory, a CUDA error) leaves the resident mesh empty.
 *   disn_mesh_clean: components = faces connected through shared undirected edges {a,b}, a != b (PyMesh "face"
 *     connectivity), numbered in order of their smallest face; n_c = distinct vertices of component c; centroid from
 *     fixed-point sums (round(v * 2^32) in int64); keep c iff n_c > max n_c * num_thresh and |centroid| < dist_thresh
 *     (the reference uses 0.5 / 0.3).  The result holds the kept faces and the vertices they reference, both in their
 *     original order (a vertex shared by two kept components appears once).  face_component: NULL or host int32
 *     [n_faces before cleaning] of component numbers.  Outputs: component count, kept components, and the cleaned
 *     mesh's n_verts / n_faces (each pointer may be NULL).  A context without a mesh holds the empty mesh.  Refuses a
 *     mesh with max |coordinate| * n_verts >= 2^30 (int64 range of the sums) and leaves it resident unchanged. */
int disn_mesh_load(disn_ctx* ctx, const float* verts, int64_t n_verts, const int32_t* faces, int64_t n_faces);
int disn_mesh_clean(disn_ctx* ctx, double dist_thresh, double num_thresh, int32_t* face_component, int64_t* n_components,
                    int64_t* n_kept, int64_t* n_verts, int64_t* n_faces);

/* OBJ file -> the resident mesh, parsed on the device (create_sdf.read_obj / read_obj_parts; pymesh.load_mesh /
 * trimesh.load_mesh(process=False) in the reference).  On success the context is in the state disn_mesh_load of
 * read_obj's arrays leaves: verts [V,3] float32 (each coordinate float64-rounded, then float32-rounded), faces [F,3] int32
 * 0-based.  The grammar: ASCII; lines end at \n, \r\n or a lone \r; tokens split on space, \t, \v, \f, \x1c-\x1f; `v`
 * records take tokens 1-3 as [+-]?(digits[.digits?]|.digits)([eE][+-]?digits)? or inf / infinity / nan; `f` records have
 * exactly three corners whose text before the first '/' is [+-]?digits (at most 18) in [1, V], V counted over the whole
 * file; other records are ignored.  Anything else returns DISN_ERR_OBJ_UNSUPPORTED and leaves the resident mesh empty,
 * as does every other failure (CUDA and allocation errors keep their ordinary codes).  *n_verts / *n_faces / *n_parts
 * (each may be NULL) receive the resident counts and the number of parts.
 * disn_obj_parts (after a read with DISN_OBJ_PARTS): part_ids [n_faces] int32 = the part of each face, parts numbered in
 * order of their first face; a face's part is the material name of the last `usemtl` line before it (its second token,
 * or "" when it has none).  Part p's name is names[name_offsets[p] .. the next part's non-negative offset, or
 * name_offsets[n_parts]); the part of faces before any usemtl has offset -1.  Any of part_ids / name_offsets / names may
 * be NULL (name_offsets[n_parts] is the bytes names needs).
 * disn_obj_read_stats: counts[2] = coordinates of the last read converted on the host (those outside the device's exact
 * rule), coordinates whose finite float64 value overflowed float32; phase_ms[5] = upload, line starts, classification,
 * parse (device events) and host conversion + parts (host clock) of the last successful read. */
int disn_obj_read(disn_ctx* ctx, const char* path, uint32_t flags, int64_t* n_verts, int64_t* n_faces, int32_t* n_parts);
int disn_obj_parts(disn_ctx* ctx, int32_t* part_ids, int64_t* name_offsets, char* names, int64_t names_capacity);
int disn_obj_read_stats(disn_ctx* ctx, int64_t* counts, float* phase_ms);

/* Signed distance field of the resident mesh (disn_mesh_load / disn_mc_run / disn_mesh_clean), the reference's
 * computeDistanceField -s (preprocessing/create_point_sdf_grid.py:200-210): R = res+1 points per axis over bbox
 * (NULL = cube around the mesh AABB scaled by expand_rate; the box used is written to bbox_out[6] if non-NULL),
 * sign by exterior flood fill with wall threshold sigma.  out: host float[R,R,R] (z,y,x), or a device pointer
 * with DISN_DEVICE_PTR (e.g. straight into disn_mc_run).  Grid points are disn_eval_grid's (float64 linspace cast to
 * float32); distances are exact point-triangle distances in float64 rounded once to float32; a point is exterior when
 * it is farther than sigma from the mesh and connected to the box boundary through grid edges that cross no face
 * (DESIGN.md 4.7).  The call synchronises with the context's stream.
 * disn_mesh_sdf_phase_ms: milliseconds of the last call's four phases (BVH build, distance, edge rasterisation, flood
 * fill and sign) into ms[4]. */
int disn_mesh_sdf(disn_ctx* ctx, int32_t res, const double* bbox, double expand_rate, double sigma, float* out,
                  double* bbox_out, uint32_t flags);
int disn_mesh_sdf_phase_ms(disn_ctx* ctx, float* ms);

/* Surface-sample normalisation of the resident mesh, the reference's get_normalize_mesh
 * (preprocessing/create_point_sdf_grid.py:169-198: per-part sample counts int32(area_i * 16384 / area_sum) at :172-189,
 * trimesh.sample.sample_surface, centroid and max norm of the samples, (v - c) / m).  Definitions (DESIGN.md 4.8): face
 * areas in float64, quantised to int64 Q_f = rint(a_f * 2^shift) and scanned exactly per part.
 *   disn_mesh_part_areas: part_ids host int32 [n_faces] in [0, n_parts) (NULL: one part) -> part_q [n_parts] (the part
 *     totals of Q_f) and the shift.  The caller derives the amounts n_p = floor(Q_p * 16384 / sum Q) and draws the
 *     random numbers in sample_surface's order.
 *   disn_mesh_normalize: amounts [n_parts], draws host double [n_draws][3] = (face pick, r1, r2) per sample, parts in
 *     order, n_draws = sum of the amounts; writes centroid [3] and m (float64, the reference's norm_params) and the
 *     samples [n_draws][3] float64 if non-NULL, and replaces the resident vertices by float32((v - c) / m).  given:
 *     NULL, or double[4] = (c, m) to skip the sampling and only transform the vertices
 *     (create_point_sdf_fullgrid.py:163-183, where part_ids / amounts / draws are ignored).
 * Errors leave the resident mesh unchanged: no faces, n_parts outside [1, n_faces], non-finite vertices, a part id out of
 * range, an amount outside [0, 2^31), an amount on a zero-area part, a draw count that differs from the amounts' sum, no samples, draws outside [0, 1),
 * max |sample| * n_draws >= 2^30 (int64 range of the centroid sums) or m = 0. */
int disn_mesh_part_areas(disn_ctx* ctx, const int32_t* part_ids, int32_t n_parts, int64_t* part_q, int32_t* shift);
int disn_mesh_normalize(disn_ctx* ctx, const int32_t* part_ids, int32_t n_parts, const int64_t* amounts,
                        const double* draws, int64_t n_draws, const double* given, double* centroid, double* m,
                        double* samples);

/* Resident field of the per-object preprocessing chain (preprocessing/create_point_sdf_grid.py:213-246): a context-owned
 * device buffer of R^3 floats (valid until the next disn_field call with a larger R), passed with DISN_DEVICE_PTR to
 * disn_mesh_sdf (write), disn_mc_run (create_one_cube_obj, :248-252) and the samplers below, so the field never leaves
 * HBM except as samples. */
int disn_field(disn_ctx* ctx, int32_t R, float** out_dev);

/* Band sampling, the reference's sample_sdf (preprocessing/create_point_sdf_grid.py:74-113), in two calls around the
 * host's np.random.randint draws:
 *   disn_sdf_band_count: sdf [R,R,R] (host, or device with DISN_DEVICE_PTR; a device field must stay valid until the
 *     gather), iso and edges [4][2] = (lo, hi) as float32 -> counts [4] of the points with lo <= float32(sdf - iso) < hi;
 *     each band's flat indices are kept on the device in ascending order.  The bands must be disjoint (the four lists
 *     share one buffer of R^3 entries): NaN edges or two non-empty intervals that overlap are an error;
 *   disn_sdf_band_gather: axes host float [3][R] (the x, y, z tables of the host function), choices host int64 (k[0]
 *     indices into band 0, then band 1, ...) -> out [sum k][4] float32 rows (x, y, z, sdf).
 * Strided sampling, create_point_sdf_fullgrid.py:70-96: out [M,M,M] with M = (R-1)/reduce + 1 holds every reduce-th
 * value on each axis. */
int disn_sdf_band_count(disn_ctx* ctx, const float* sdf, int32_t R, float iso, const float* edges, uint32_t flags,
                        int64_t* counts);
int disn_sdf_band_gather(disn_ctx* ctx, const float* axes, const int64_t* choices, const int64_t* k, float* out);
int disn_sdf_strided(disn_ctx* ctx, const float* sdf, int32_t R, int32_t reduce, uint32_t flags, float* out);

/* Estimated-camera path (reference: demo/demo.py:195-258 cam_evl, cam_est/model_cam.py:47-109, models/posenet.py:91-124):
 * imgs host [B,H,W,3] -> VGG-16 embedding (the context's `vgg_16/...` weights = the camera checkpoint's) -> three FC
 * heads (`cameraprediction/{scale,ortho6d,translation}/fc{1,2,3}/{weights,biases}`) -> pred_RT [B,4,3] (or NULL) and
 * pred_trans_mat = pred_RT . K^T [B,4,3].  K: host float[9] row-major intrinsics, NULL = the reference constant
 * [[149.84375,0,68.5],[0,149.84375,68.5],[0,0,1]] (cam_est/model_cam.py:28). */
int disn_cam_estimate(disn_ctx* ctx, const float* imgs, int32_t B, int32_t H, int32_t W, int32_t C, const float* K,
                      float* out_rt, float* out_trans_mat);

/* Camera checkpoint score (cam_est/train_sdf_cam.py:459-565 eval_one_epoch, cam_est/model_cam.py:111-239): the
 * prediction of disn_cam_estimate on imgs, then per image b over the N points pts [B,N,3] (host float32) with the ground
 * truth trans_mat and RT (the view file's regress_mat) [B,4,3], h = [p, 1]:
 *   sums[b][0] = sum |h.pred_RT - h.RT|^2                          (rotpc_loss = total / 2)
 *   sums[b][1] = sum |xy_pred - xy_gt|^2, xy = (h.M)[:2] / (h.M)[2] (rot2d_loss = total / 2 / 10000)
 *   sums[b][2] = sum sqrt(|h.pred_RT - h.RT|^2)                    (rot3d_dist_all = sums[b][2] / N)
 *   sums[b][3] = sum sqrt(|clamp(xy_gt) - clamp(xy_pred)|^2), clamp to [0, 136]  (rot2d_dist_all = sums[b][3] / N)
 *   sums[b][4] = sum over the 12 entries of (pred_trans_mat - trans_mat)^2     (rotmatrix_loss = total / (12 B))
 * Float32 terms, one rounding per op; float64 sums in a fixed order (repeated calls are bitwise equal).  out_rt and
 * out_trans_mat (either may be NULL) receive disn_cam_estimate's bits.  B in [1, max_batch], N >= 1. */
int disn_cam_metrics(disn_ctx* ctx, const float* imgs, int32_t B, int32_t H, int32_t W, int32_t C, const float* K,
                     const float* pts, int64_t N, const float* trans_mat, const float* RT, float* out_rt,
                     float* out_trans_mat, double* sums);

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

/* One reference mesh against V meshes (the views of test/test_iou.py:165-206 iou_cat, one call per object): the reference
 * is voxelised once, the V views in one launch, and the V intersection / union counts come back from one synchronise.
 * View v has vertices [vert_offsets[v], vert_offsets[v+1]) of verts and faces [face_offsets[v], face_offsets[v+1]) of
 * faces, whose ids are local to the view.  intersection[v] / uni[v] equal disn_iou(ref, view v) bit for bit (disn_iou is
 * the V = 1 case).  occ_out: optional uint8[(V+1)*dim^3], the reference's grid then the views'.  Refused before anything
 * is launched: null pointers, dim outside [2,512], V < 1, offsets that do not start at 0 or decrease, a mesh without
 * faces, a face id outside its own mesh (the message names the view).  Scratch per call: (V+1) windows of
 * (1.2 dim + 8)^3 bits and (V+1) grids of dim^3 bits. */
int disn_iou_views(disn_ctx* ctx, const float* ref_verts, int64_t ref_nv, const int32_t* ref_faces, int64_t ref_nf,
                   int32_t V, const float* verts, const int64_t* vert_offsets, const int32_t* faces,
                   const int64_t* face_offsets, int32_t dim, int64_t* intersection, int64_t* uni, uint8_t* occ_out);

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

/* Checkpoint score at ground-truth samples, the metrics test/test_sdf_acc.py prints (models/model_normalization.py:
 * 279-299, non-binary branch).  pts [B,N,3] (pts_rot = pts, as without --rot), trans_mat [B,4,3] and gt [B,N] (the
 * loader's sdf_val) of the encoded batch; pred: NULL or [B,N], receiving pred_sdf bitwise equal to disn_eval_points's.
 * With g = float32(gt - iso_offset) (the driver's sdf_val - 0.003) and p = pred, per image b:
 *   count[b] = #{(g > 0) == (p > 0)};
 *   wsum[b]  = float64 sum of |g * sdf_weight - p| * w, w = mask_weight if g <= 0.01 else 1;
 *   rsum[b]  = float64 sum of |g - p / sdf_weight|;
 * each term formed in float32 with correctly rounded operations in TF's order, the sums in a fixed order (repeated calls
 * are bitwise equal).  Batch values: accuracy = float32(sum count) / float32(B*N), sdf_loss = float32(sum wsum / (B*N))
 * * 1000 in float32, sdf_loss_realvalue = float32(sum rsum / (B*N)).  Host pointers (synchronous), or device pointers
 * for every array with DISN_DEVICE_PTR (asynchronous; the DISN_PREC_F16F8 overflow status is then reported by the next
 * synchronising call).  N >= 1, B = the encoded batch, sdf_weight non-zero, all three scalars finite. */
int disn_sdf_metrics(disn_ctx* ctx, const float* pts, const float* trans_mat, const float* gt, int32_t B, int64_t N,
                     float iso_offset, float sdf_weight, float mask_weight, uint32_t flags, float* pred, int64_t* count,
                     double* wsum, double* rsum);

/* Decoder training with the encoder frozen (train/train_sdf.py with --img_feat_twostream, bn=False; models/
 * model_normalization.py:169-206,254-299; DESIGN.md 4.12).  The 24 decoder variables (weights and biases of fold1/conv1-3
 * and fold2/conv1,2,5 in sdfprediction and sdfprediction_imgfeat) of the context are the fp32 masters; TF's Adam updates
 * them in place.
 *   disn_train_begin: checks the decoder variables, zeroes the Adam slots, sets beta1_power = beta1, beta2_power = beta2
 *     and computes the frozen VGG kernels' share of the regularization.  Needs every vgg_16 variable loaded that will
 *     count (slim.l2_regularizer over its 16 kernels).  Not with tanh_out.
 *   disn_train_step: one sess.run of the train op on host arrays imgs [B,H,W,3], pts [B,N,3] (`sample_pc`, projected),
 *     pts_rot [B,N,3] (`sample_pc_rot`, the MLP input; NULL = pts), trans_mat [B,4,3], sdf_gt [B,N] (the fed `sdf`:
 *     the loader's sdf_val - 0.003), learning rate lr -> losses[5] = accuracy, sdf_loss_realvalue, sdf_loss,
 *     regularization, overall_loss of the forward pass before the update (float32 values as TF reports them, widened).
 *     Encodes in groups of 8 images.  Afterwards the encoded state is dropped: every call that needs it fails with an
 *     error naming the stale state until the next disn_encode, which uses the updated weights.  Synchronous.
 *   disn_train_get / disn_train_set: by TF name -- a decoder variable, `<var>/Adam`, `<var>/Adam_1`, `beta1_power`,
 *     `beta2_power` -- n = the element count.  Setting a variable drops the encoded state as a step does.
 *     Any other loaded variable (the frozen encoder's) can be read, not set.
 *   disn_train_var_name: the i-th decoder variable's name (i in [0,24)), the order of the diagnostic gradients.
 *   disn_train_phase_ms: device-event milliseconds of the last step's phases into ms[6]: encode (VGG-16 and the
 *     embedding copy, all groups), gather (point features), forward, loss (with the regularization norms), backward,
 *     Adam (0 after the gradient diagnostic). */
typedef struct disn_train_config {
  float beta1, beta2, epsilon;   /* AdamOptimizer(lr, beta1=FLAGS.beta1): 0.5, 0.999, 1e-8 */
  float wd;                      /* weight decay of every kernel (1e-5) */
  float mask_weight;             /* FLAGS.mask_weight (4) */
  float sdf_weight;              /* SDF_WEIGHT (10) */
} disn_train_config;
void disn_default_train_config(disn_train_config* cfg);
int disn_train_begin(disn_ctx* ctx, const disn_train_config* cfg);
int disn_train_step(disn_ctx* ctx, const float* imgs, int32_t H, int32_t W, int32_t C, const float* pts, const float* pts_rot,
                    const float* trans_mat, const float* sdf_gt, int32_t B, int64_t N, float lr, double* losses);
int disn_train_get(disn_ctx* ctx, const char* name, float* out, int64_t n);
int disn_train_set(disn_ctx* ctx, const char* name, const float* data, int64_t n);
int disn_train_var_name(int32_t i, char* out, int64_t capacity);
int disn_train_phase_ms(disn_ctx* ctx, float* ms);

/* Kernel launch counter (bench's gpu_launches): number of this library's kernels launched so far. */
int64_t disn_launch_count(disn_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* DISN_B200_H */
