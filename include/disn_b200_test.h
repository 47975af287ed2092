/* Diagnostics of the DISN library: building blocks, probes and debug harnesses used by tests/ and tools/.
 * They live in libdisn_b200_test.so (the product library libdisn_b200.so does not export them). */
#ifndef DISN_B200_TEST_H
#define DISN_B200_TEST_H
#include "disn_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* Diagnostic: one warpgroup-MMA GEMM D[128x256] = A[128x64] * B[256x64]^T (bf16, four m64n128 blocks), `passes` times
 * accumulated; D_out[c][64h + r][j] = D[64c + r][128h + j] (c, h in {0,1}). Host pointers. */
int disn_tc_selftest(int device, const float* A, const float* B, int passes, float* D_out);
/* Diagnostic: mixed-kind accumulation used by DISN_PREC_F16F8 -- D = fp16(A16).fp16(B16)^T (mode bit 0) +
 * e5m2(A8).e5m2(B8)^T (mode bit 1) summed in fp32, D_out laid out as above; A8q/B8q return the e5m2 values actually used. */
int disn_tc_selftest_mixed(int device, const float* A16, const float* B16, const float* A8, const float* B8, int mode,
                           float* A8q, float* B8q, float* D_out);

/* Diagnostic: one encoder GEMM (plain when H == 0, else the 3x3 SAME im2col view of NHWC A[M/(H*W),H,W,Cin]) through
 * the fp32 CUDA-core kernel and through the tensor-core kernel; host pointers, outputs [M,N]. */
int disn_debug_gemm(disn_ctx* ctx, const float* A, const float* Wt, const float* bias, int M, int N, int K, int H, int W,
                    int Cin, int relu, float* out_fp32, float* out_tc);

/* Diagnostic: prints the achievable L2 -> shared-memory bulk-copy streaming rate (bytes/clk/SM) for a sweep of
 * ring depths, stage sizes and cluster multicast widths (the weight-streaming pattern of the tensor-core kernel). */
int disn_tc_stream_probe(int device);
/* Diagnostic: prints the issue cost (cycles) of the mbarrier / wgmma synchronisation instructions of the consumers. */
int disn_tc_op_probe(int device);

/* Diagnostic of the tensor-core point kernel: the packed weight image of operand mode `precision` (DISN_PREC_BF16X3 or
 * DISN_PREC_F16F8) -> image[nbytes] (host; nbytes must be the packed size, 132 half-stages of 32 KB in consumption order,
 * see tc_pack_weights) and the e5m2 activation multipliers [stream][layer]{(a - h(a)) scale, a scale} -> act_scale[16]. */
int disn_debug_tc_weights(disn_ctx* ctx, int32_t precision, int64_t nbytes, uint8_t* image, float* act_scale);

/* Diagnostics of the coarse-to-fine grid (disn_eval_grid_adaptive):
 *   disn_adaptive_mask: points [first, first + n) of the last call's evaluated-point mask -> out uint8[n] (1 = evaluated);
 *   disn_adaptive_from_field: the same refinement with values read from field [R,R,R] (host, or device with
 *     DISN_DEVICE_PTR) instead of the network; sdf_params[6] gives the box (the spacing of the band);
 *   disn_adaptive_phase_ms: device-event milliseconds of the last call's phases -- coarse lattice (or the dense grid),
 *     each level, fill -- into ms (at least 6 entries), *n their number. */
int disn_adaptive_mask(disn_ctx* ctx, int64_t first, int64_t n, uint8_t* out);
int disn_adaptive_from_field(disn_ctx* ctx, const float* field, int32_t sdf_res, const double* sdf_params, float iso,
                             double band, uint32_t flags, float** grid_dev, int64_t* level_counts, int32_t* n_levels);
int disn_adaptive_phase_ms(disn_ctx* ctx, float* ms, int32_t* n);

/* Diagnostics of the coarse-to-fine mesh (disn_mesh_grid_adaptive):
 *   disn_mesh_adaptive_from_field: the same mesh with values read from field [R,R,R] (host, or device with
 *     DISN_DEVICE_PTR) instead of the network, (sdf_res+1)^3 < 2^31, sdf_res even;
 *   disn_mesh_adaptive_phase_ms: device-event milliseconds of the last call's phases -- levels, candidate cells, mesh --
 *     into ms[3];
 *   disn_mesh_adaptive_bytes: bytes held by the call's buffers (the resident mesh not included);
 *   disn_mesh_adaptive_edges: the edge ids ((z*R + y)*R + x)*3 + axis of vertices [first, first + n) of the last call. */
int disn_mesh_adaptive_from_field(disn_ctx* ctx, const float* field, int32_t sdf_res, const double* sdf_params, float iso,
                                  double band, uint32_t flags, int64_t* level_counts, int32_t* n_levels, int64_t* n_verts,
                                  int64_t* n_faces);
int disn_mesh_adaptive_phase_ms(disn_ctx* ctx, float* ms);
int disn_mesh_adaptive_bytes(disn_ctx* ctx, int64_t* bytes);
int disn_mesh_adaptive_edges(disn_ctx* ctx, int64_t first, int64_t n, int64_t* out);

/* Diagnostic: the OBJ reader's host coordinate converter (Python's float() then numpy's float64 -> float32 cast) on n
 * tokens text[offsets[i] .. offsets[i] + lengths[i]) -> out[n]; a token outside the reader's grammar is an error naming
 * it.  Needs no device. */
int disn_debug_obj_tokens(const char* text, const int64_t* offsets, const int32_t* lengths, int64_t n, float* out);

/* Diagnostic: the camera-pose heads of disn_cam_estimate on a caller's embedding emb [B, num_classes] (host) instead of
 * the encoder's; K [3,3] row-major (NULL = the default intrinsics) -> out_rt and out_trans_mat [B,4,3] (host).  The
 * context's encoder products are left as they are. */
int disn_debug_cam_heads(disn_ctx* ctx, const float* emb, int32_t B, const float* K, float* out_rt, float* out_trans_mat);

/* Diagnostic of decoder training: disn_train_step's gradients of overall_loss without the Adam update -> grads (the 24
 * variables in disn_train_var_name order, each row-major as TF stores it, wd * W included), pred [B*N], acts (NULL or the
 * ten layer outputs after ReLU, stream-major, each [B*N][64 | 256 | 512 | 512 | 256]) and losses[5].  Drops the encoded
 * state as a step does. */
int disn_debug_train_grads(disn_ctx* ctx, const float* imgs, int32_t H, int32_t W, int32_t C, const float* pts,
                           const float* pts_rot, const float* trans_mat, const float* sdf_gt, int32_t B, int64_t N,
                           float* grads, float* pred, float* acts, double* losses);

#ifdef __cplusplus
}
#endif
#endif /* DISN_B200_TEST_H */
