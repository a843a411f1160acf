/*
 * sdb200.h -- C ABI of libsdb200.so, the H100-native (sm_90a) implementation of the
 * SceneDreamer per-pixel render hot path.
 *
 * Conventions
 *   - every pointer named d_* is a DEVICE pointer owned by the caller; nothing is allocated,
 *     freed or retained by the library (no ownership transfer, re-entrant; the only process-wide
 *     state is a launch counter and the optional diagnostics pointer; the library links against
 *     the CUDA runtime only -- no cuBLAS / cuDNN);
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *   - every entry point returns 0 on success, a positive cudaError_t on a CUDA failure, or a
 *     negative SDB_E* code for an argument error; no exceptions cross the ABI.  The Python
 *     mirrors turn non-zero codes into RuntimeError like the reference's TORCH_CHECKs do;
 *   - there is NO CPU fallback: without a CUDA device the compute entry points return an error.
 *
 * Each entry point cites the reference interface it replaces (paths relative to the reference
 * repository root).  INTEGRATION.md shows the binding a maintainer would add on the reference
 * side.
 */
#ifndef SDB200_H
#define SDB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SDB_OK 0
#define SDB_EINVAL (-1)      /* bad argument (null pointer, size <= 0, ...)            */
#define SDB_EUNSUPPORTED (-2) /* valid in the reference, not supported here (see docs) */

/* Library / build information.  Safe to call without a GPU. */
int sdb_version(void);                 /* 10000*major + 100*minor + patch                 */
const char *sdb_build_info(void);      /* "sm_90a nvcc X.Y ..." -- static string          */
const char *sdb_error_string(int code);/* cudaGetErrorString for >0, own text for <0      */

/* --------------------------------------------------------------------------------------------
 * a1. Ray / voxel intersection, perspective camera.
 * Replaces voxlib.ray_voxel_intersection_perspective
 *   (imaginaire/model_utils/gancraft/voxlib/voxlib.cpp:11,26;
 *    ray_voxel_intersection.cu:253-325 host wrapper, :52-235 kernel).
 * The camera frame (fwd/side/up) is derived on the host from cam_dir/cam_up exactly as the
 * reference does (:279-284); cam_* are HOST pointers to 3 floats.
 *   d_voxel      int32, dims[3] with element strides[3] (any strides, like the reference)
 *   d_voxel_id   int32  [H, W, M]        (reference shape [H,W,M,1])
 *   d_depth2     float  [2, H, W, M]     (entry t, exit t; NaN in unfilled slots)
 *   d_raydirs    float  [H, W, 3]
 * ------------------------------------------------------------------------------------------ */
int sdb_ray_voxel_intersection_perspective(
    const int32_t *d_voxel, const int64_t dims[3], const int64_t strides[3],
    const float cam_ori[3], const float cam_dir[3], const float cam_up[3],
    float cam_f, const float cam_c[2], const int32_t img_dims[2], int32_t max_samples,
    int32_t *d_voxel_id, float *d_depth2, float *d_raydirs, void *stream);

/* The same traversal with an optional empty-space bound (bit-identical results, fewer steps): the
 * walk's per-axis event times are pure functions of the cell index, so from a cell above the
 * highest occupied voxel of its column block the state after leaving that empty box is computed
 * directly instead of cell by cell (DESIGN.md 3.1).  d_height_bound: int16 [nbx * nbz] from
 * sdb_build_height_bound (nb = ceil(dim / 2^block_log2) over dims[1], dims[2]); NULL = plain walk.
 * The bound must describe THIS volume's current contents (rebuild after any edit).               */
int64_t sdb_height_bound_elems(const int64_t dims[3], int32_t block_log2);
int sdb_build_height_bound(const int32_t *d_voxel, const int64_t dims[3], const int64_t strides[3], int32_t block_log2,
                           int16_t *d_height_bound, void *stream);
int sdb_ray_voxel_intersection_perspective_ex(
    const int32_t *d_voxel, const int64_t dims[3], const int64_t strides[3],
    const float cam_ori[3], const float cam_dir[3], const float cam_up[3],
    float cam_f, const float cam_c[2], const int32_t img_dims[2], int32_t max_samples,
    int32_t *d_voxel_id, float *d_depth2, float *d_raydirs, const int16_t *d_height_bound, int32_t block_log2,
    void *stream);

/* Row bands of one frame as ONE call (multi-GPU single-frame sharding, DESIGN.md 6): output row v of the
 * img_dims[0]-row result is frame row band[0] + (v / band[1]) * band[2] + v % band[1], i.e. bands of band[1] rows
 * starting at frame row band[0], band[2] frame rows apart; cam_c is the principal point of the WHOLE frame.  Every
 * ray is computed exactly as the whole-frame call computes it (c0 - row is exact in float32).                  */
int sdb_ray_voxel_intersection_perspective_bands(
    const int32_t *d_voxel, const int64_t dims[3], const int64_t strides[3],
    const float cam_ori[3], const float cam_dir[3], const float cam_up[3],
    float cam_f, const float cam_c[2], const int32_t img_dims[2], int32_t max_samples, const int32_t band[3],
    int32_t *d_voxel_id, float *d_depth2, float *d_raydirs, const int16_t *d_height_bound, int32_t block_log2,
    void *stream);

/* Host-only helper (no GPU needed): the camera frame the call above derives. */
void sdb_camera_frame(const float cam_dir[3], const float cam_up[3], float fwd[3], float side[3], float up[3]);

/* --------------------------------------------------------------------------------------------
 * a6/a7. Multi-resolution hash / tiled grid encoding, float32 (float16 tables: the _f16 pair below).
 * Replace _gridencoder.grid_encode_forward / grid_encode_backward
 *   (gridencoder/src/bindings.cpp:5-8, gridencoder.h:12-13, gridencoder.cu:423-478).
 * Same argument meaning as the reference: caller pre-allocates everything;
 *   d_inputs [B,D] in [0,1]; d_embeddings [sum T_l, C]; d_offsets int32 [L+1];
 *   d_outputs [L,B,C]; d_dy_dx [B, L*D*C] (only touched when calc_grad_inputs);
 *   backward: d_grad [L,B,C], d_grad_embeddings pre-zeroed, d_grad_inputs [B,D].
 * D in {2,3,4,5}, C in {1,2,4,8} (else SDB_EUNSUPPORTED, the reference throws).
 * Unlike the reference (legacy default stream, gridencoder.cu:351) the launch goes to `stream`.
 * ------------------------------------------------------------------------------------------ */
int sdb_grid_encode_forward(
    const float *d_inputs, const float *d_embeddings, const int32_t *d_offsets, float *d_outputs,
    uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
    int calc_grad_inputs, float *d_dy_dx, uint32_t gridtype, int align_corners, void *stream);

int sdb_grid_encode_backward(
    const float *d_grad, const float *d_inputs, const float *d_embeddings, const int32_t *d_offsets,
    float *d_grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
    int calc_grad_inputs, const float *d_dy_dx, float *d_grad_inputs, uint32_t gridtype,
    int align_corners, void *stream);

/* The same two calls on a float16 table -- the reference under autocast (gridencoder/grid.py:38-39 casts the
 * embeddings to half when C is even; the binding dispatches on the table's dtype, gridencoder.cu:442-444, 473-475):
 * d_embeddings / d_outputs / d_dy_dx / d_grad / d_grad_embeddings / d_grad_inputs are IEEE half, d_inputs stays float32.
 * Arithmetic as c10::Half performs it (every operator rounds its result to half), so outputs and dy_dx are
 * bit-identical to the reference; the table gradient uses half2 atomics like the reference (:299-305).
 * C in {2,4,8} (odd C never reaches this path in the reference; SDB_EUNSUPPORTED).                              */
int sdb_grid_encode_forward_f16(
    const float *d_inputs, const void *d_embeddings, const int32_t *d_offsets, void *d_outputs,
    uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
    int calc_grad_inputs, void *d_dy_dx, uint32_t gridtype, int align_corners, void *stream);
int sdb_grid_encode_backward_f16(
    const void *d_grad, const float *d_inputs, const void *d_embeddings, const int32_t *d_offsets,
    void *d_grad_embeddings, uint32_t B, uint32_t D, uint32_t C, uint32_t L, float S, uint32_t H,
    int calc_grad_inputs, const void *d_dy_dx, void *d_grad_inputs, uint32_t gridtype,
    int align_corners, void *stream);

/* --------------------------------------------------------------------------------------------
 * a9. Positional encoding along one dimension of a contiguous tensor viewed as [pre, post]
 * -> [pre, stride, post], stride = 2*ndegrees (+1 if incl_orig).
 * Replace voxlib.positional_encoding / positional_encoding_backward
 *   (voxlib.cpp:20,22,29-30; positional_encoding_kernel.cu:40-118).
 * ------------------------------------------------------------------------------------------ */
int sdb_positional_encoding(const float *d_in, float *d_out, int64_t pre, int64_t post,
                            int32_t ndegrees, int incl_orig, void *stream);
int sdb_positional_encoding_backward(const float *d_out_grad, const float *d_out, float *d_in_grad,
                                     int64_t pre, int64_t post, int32_t ndegrees, int incl_orig,
                                     void *stream);

/* --------------------------------------------------------------------------------------------
 * voxlib surface: sparse tri-linear interpolation at world coordinates (GANcraft block features;
 * SceneDreamer never calls it, gancraft_base.py:442 does).  Replace
 *   voxlib.sp_trilinear_worldcoord / sp_trilinear_worldcoord_backward
 *   (voxlib.cpp:15,17,27-28; sp_trilinear_worldcoord_kernel.cu:48-338, host :351-437, :453-520).
 *   d_feature [M, C] fp32 (row i = feature of corner id i, or id i+1 with ign_zero);
 *   d_corner_lut int32 volume, element (a,b,c) at a*strides[0] + b*strides[1] + c*strides[2];
 *   d_worldcoord [E, 3] fp32 contiguous; d_out [E, C]; d_out_grad [E, C]; d_feature_grad [M, C]
 *   (zeroed by the call, then accumulated with atomics like the reference).
 * ------------------------------------------------------------------------------------------ */
int sdb_sp_trilinear_worldcoord(const float *d_feature, int64_t M, int32_t C, const int32_t *d_corner_lut,
                                const int64_t lut_dims[3], const int64_t lut_strides[3],
                                const float *d_worldcoord, int64_t E, int ign_zero, float *d_out, void *stream);
int sdb_sp_trilinear_worldcoord_backward(const float *d_out_grad, int64_t M, int32_t C,
                                         const int32_t *d_corner_lut, const int64_t lut_dims[3],
                                         const int64_t lut_strides[3], const float *d_worldcoord, int64_t E,
                                         int ign_zero, float *d_feature_grad, void *stream);

/* --------------------------------------------------------------------------------------------
 * a2-a5, a8, a10-a12. Fused per-pixel render: sampling -> labels -> hash-grid features ->
 * style-modulated sigma/colour MLP (wgmma tensor cores) -> front-to-back compositing + sky
 * blend.  Replaces the body of Generator._forward_perpix and the tile loop around it
 *   (imaginaire/generators/scenedreamer.py:285-428, :600-628; mc_utils.py:82-161;
 *    model_utils/layers.py:92-126, :241-271; gridencoder.cu:75-224).
 * See sdb_render_params below and DESIGN.md for layouts.
 * The fused kernels (render, sky, training forward and gradient chains) keep their fp32 layer
 * accumulators in a library-owned device buffer per (device, stream), allocated on the first
 * launch that needs it: under CUDA-graph capture such a launch returns SDB_EUNSUPPORTED, so run
 * one launch of the same size on the stream before capturing.
 * ------------------------------------------------------------------------------------------ */
typedef struct sdb_render_params {
    /* rays (outputs of a1): n_img images of H x W rays, R = n_img*H*W, row-major like the reference */
    int32_t n_img, H, W;
    int32_t M;                   /* slots per ray (num_blocks_early_stop), 1..8               */
    int32_t S;                   /* samples per ray (num_samples), 1..64; S+1 strata points   */
    const int32_t *d_voxel_id;   /* [R, M]                                                    */
    const float *d_depth2;       /* [n_img][2][H*W][M] (reference layout [N,2,H,W,M,1])       */
    const float *d_raydirs;      /* [R, 3]                                                    */
    const float *d_cam_ori;      /* [n_img, 3] device, or NULL: take cam_ori_value (n_img == 1) */
    float voxel_dims[3];         /* normalisation of world coords (scenedreamer.py:298-299)   */
    const float *d_global_enc;   /* [n_img, 2] device: scene code = encoder dims 3,4 (:300-302)*/
    float sample_depth;          /* mc_utils.py:107                                           */
    float dists_scale;           /* scenedreamer.py:373                                       */
    /* sampling positions along the ray.  Deterministic branch (mc_utils.py:118-120):
       d_fractions[S+1] = linspace(0,1,S+3)[1:-1], d_uniforms = NULL.  Stratified branch
       (:122-125): d_uniforms [R, S+1] in [0,1) and d_fractions[S+1] = linspace(0,1,S+2)[:-1].  */
    const float *d_fractions;
    const float *d_uniforms;
    /* label translation: reduced label per Minecraft id with ignore already mapped to dirt
       (mc_utils.py:241-246); labels must be < 15                                              */
    const int32_t *d_label_lut;
    int32_t n_lut;
    /* hash grid, D=5, C=8, every level hashed with T = 2^log2_T entries:
       d_table  = raw 5-D table [L*T, 8] (exact reference arithmetic, 32 corners / level), or
       d_table3 = per-scene pre-blended table from sdb_preblend_table (8 corners / level;
                  needs n_img == 1 or identical global_enc).  Exactly one is non-NULL.         */
    const float *d_table;
    const float *d_table3;
    int32_t L;                   /* 16                                                        */
    int32_t log2_T;
    float level_S;               /* log2(per_level_scale)                                     */
    int32_t base_res;
    /* MLP weights packed by sdb_pack_mlp(): one pack per image (style code), stride bytes     */
    const void *d_mlp_pack;
    int64_t mlp_pack_stride;     /* 0 = all images share one pack                             */
    int32_t precision;           /* must match the pack: 0 = fp16 x1, 1 = bf16 x3, 2 = fp16 x3 */
    /* sky: SKYMLP output per ray [R, 64] and the per-image mean [n_img, 64]                   */
    const float *d_sky;
    const float *d_sky_avg;
    /* outputs */
    float *d_net_out;            /* [R, 64]                                                   */
    float *d_depth_out;          /* [R] sum w*t (scenedreamer.py:816) or NULL                 */
    float *d_total_weight;       /* [R] or NULL                                               */
    float *d_weights_out;        /* [R, S] compositing weights (scenedreamer.py:373-376) or NULL */
    float *d_rand_depth_out;     /* [R, S] sample depths after the NaN guard (:346-352) or NULL */
    /* scratch: sdb_render_workspace_bytes(n_img, H, W) bytes                                  */
    void *d_workspace;
    /* early termination (sdb_render_rays_forward only): a 16x8 ray tile stops marching once the
       transmittance exp(-sum e) of every live ray in it is below this value; the samples not
       shaded have compositing weight < threshold (reported as 0 in d_weights_out).  0 = off =
       the reference's arithmetic sample for sample.  The training forward ignores it.          */
    float early_stop_transmittance;
    /* camera origin BY VALUE, used when d_cam_ori == NULL (one image): the reference hands the pose
       of a frame over from the host (scenedreamer.py:569-586); by value it rides in the launch
       instead of a host->device copy the stream would have to wait for                          */
    float cam_ori_value[3];
} sdb_render_params;

int64_t sdb_render_workspace_bytes(int32_t n_img, int32_t H, int32_t W);
/* d_workspace after the call (int32): [0] live (not sky-only) 16x8 ray tiles, [1] tile-steps executed
   (live tiles x S minus what early termination skipped) -- diagnostics / bench bookkeeping.        */
int sdb_render_rays_forward(const sdb_render_params *p, void *stream);

/* Per-scene collapse of the two constant encoder dimensions (inference only):
 * table3[l][i] = sum_j w_j(l) * table[l][i ^ K_j(l)], j over the 4 (dim3,dim4) corners.
 * d_table [L*T, 8] -> d_table3 [L*T, 8].  (DESIGN.md section 2, "parity-preserving work
 * reductions"; valid because every level is hashed and T is a power of two.)
 * d_global_enc: 2 floats on the device.                                                       */
int sdb_preblend_table(const float *d_table, float *d_table3, int32_t L, int32_t log2_T, float level_S,
                       int32_t base_res, const float *d_global_enc, void *stream);

/* Size in bytes of the packed MLP image for a precision mode, and the packer.  Inputs are DEVICE
 * fp32 row-major matrices of the style-modulated network for ONE style code:
 *   w1 [256,128] b1 [256]; emb [n_labels<=15, 256] (row k = fc_m_a.weight[:, k]);
 *   wh [5][256,256] (fc_2..fc_6: weight * alpha per input column) bh [5][256] (beta);
 *   wsig [256] bsig [1]; wout [64,256] bout [64].                                             */
int64_t sdb_mlp_pack_bytes(int32_t precision);
int sdb_pack_mlp(const float *d_w1, const float *d_b1, const float *d_emb, int32_t n_labels,
                 const float *d_wh, const float *d_bh, const float *d_wsig, const float *d_bsig,
                 const float *d_wout, const float *d_bout, int32_t precision, void *d_pack, void *stream);

/* --------------------------------------------------------------------------------------------
 * a9. Sky branch on the tensor-core engine: PE(raydir, 5 degrees, incl. orig) -> SKYMLP -> sky
 * features per ray + the per-image mean.  Replaces voxlib.positional_encoding + SKYMLP.forward +
 * torch.mean on the hot path (scenedreamer.py:368-370, :592-598; gancraft_base.py:150-169).
 *   pack: sdb_pack_sky_mlp() with w1 [256,33], b1 [256] (= fc1.bias + fc_z_a(z)), wh [4][256,256],
 *         bh [4][256], wout [64,256], bout [64] (device fp32) for ONE style code;
 *   d_raydirs [n_img*H*W, 3]; d_sky [n_img*H*W, 64]; d_sky_avg [n_img, 64];
 *   d_workspace: sdb_sky_workspace_bytes(n_img, H, W) bytes.
 * ------------------------------------------------------------------------------------------ */
int64_t sdb_sky_pack_bytes(int32_t precision);
int sdb_pack_sky_mlp(const float *d_w1, const float *d_b1, const float *d_wh, const float *d_bh,
                     const float *d_wout, const float *d_bout, int32_t precision, void *d_pack, void *stream);
int64_t sdb_sky_workspace_bytes(int32_t n_img, int32_t H, int32_t W);
int sdb_sky_forward(const float *d_raydirs, int32_t n_img, int32_t H, int32_t W, const void *d_sky_pack,
                    int64_t pack_stride, int32_t precision, float *d_sky, float *d_sky_avg, void *d_workspace,
                    void *stream);

/* --------------------------------------------------------------------------------------------
 * a7 + backward of a8/a10/a11: training.  sdb_render_rays_train_forward is sdb_render_rays_forward
 * (fp16x3, pre-blended table: p->d_table3, p->precision == 2) that additionally writes a RECORD of
 * the pass into caller-owned device memory: per-sample hash-grid coordinates and features, the six
 * hidden activations (bf16) with their LeakyReLU sign words, sigma, interval length and the colour
 * head output.  sdb_render_rays_backward turns dL/d net_out into every parameter gradient of the
 * per-pixel path -- what torch.autograd produces for Generator._forward_perpix in the reference
 * (imaginaire/generators/scenedreamer.py:313-428 under train.py; kernel_grid_backward /
 * kernel_input_backward gridencoder.cu:227-343 for the table and the scene code):
 *   1. compositing backward (volum_rendering_relu, clamp, sky blend; mc_utils.py:154-161,
 *      scenedreamer.py:373-413)                       -> dL/dc, dL/dsigma per sample, dL/dsky;
 *   2. the data-gradient chain of LightningMLP on the wgmma engine (transposed weights, bf16x3)
 *      -> dZ of every layer (bf16 record) and dL/d features;
 *   3. table backward through the pre-blended 3-D table (vector red.add), un-blend to the raw 5-D
 *      table, and the scene-code gradient;
 *   4. weight gradients: dZ^T * A over all samples on the tensor cores (hand-written wgmma kernel: the
 *      bf16 records are MMA-ready tiles, fp32 accumulators in registers; csrc/wgrad.cu).
 * The same sdb_render_params as the forward call must be passed (same rays, uniforms, packs).
 * The call is fully asynchronous: the live-tile count of the recorded pass stays on the device (record
 * header), every kernel is launched over the record's capacity and reads it there.
 * ------------------------------------------------------------------------------------------ */
int64_t sdb_render_train_record_bytes(int32_t n_img, int32_t H, int32_t W, int32_t S);
int sdb_render_rays_train_forward(const sdb_render_params *p, void *d_record, void *stream);

/* Packed TRANSPOSED weights for step 2 (bf16 hi/lo): w1 [256,128], wh [5][256,256] (style-modulated,
 * as for sdb_pack_mlp), wsig [256], wout [64,256]; device fp32 for ONE style code.              */
int64_t sdb_mlp_backward_pack_bytes(void);
int sdb_pack_mlp_backward(const float *d_w1, const float *d_wh, const float *d_wsig, const float *d_wout,
                          void *d_pack, void *stream);

typedef struct sdb_render_grads {
    const float *d_grad_net_out;   /* in  [R, 64]  dL/d net_out                                     */
    const void *d_bwd_pack;        /* in  sdb_pack_mlp_backward image(s)                            */
    int64_t bwd_pack_stride;       /*     0 = all images share one pack                             */
    const float *d_table;          /* in  raw 5-D table [L*T, 8] (for the scene-code gradient)      */
    /* outputs (all written, none accumulated into)                                                 */
    float *d_grad_table;           /* [L*T, 8]  dL/d hash_encoder.embeddings                        */
    float *d_grad_global_enc;      /* [2]       dL/d scene code (summed over images)                */
    float *d_grad_w1ext;           /* [256, 144] cols 0..127 fc_1.weight, 128+k fc_m_a.weight[:,k], 143 fc_1.bias */
    float *d_grad_wh;              /* [5][256, 272] cols 0..255 dL/dW' (modulated weight), col 256 dL/dbeta        */
    float *d_grad_wsig;            /* [8, 272]  row 0: cols 0..255 fc_sigma.weight, col 256 fc_sigma.bias          */
    float *d_grad_wout;            /* [64, 272] cols 0..255 fc_out_c.weight, col 256 fc_out_c.bias                 */
    float *d_grad_sky;             /* [R, 64]   dL/d sky features per ray                           */
    float *d_grad_sky_avg;         /* [n_img, 64]                                                   */
    void *d_workspace;             /* sdb_render_backward_workspace_bytes() bytes                   */
} sdb_render_grads;

int64_t sdb_render_backward_workspace_bytes(int32_t n_img, int32_t H, int32_t W, int32_t S, int32_t L, int32_t log2_T);
int sdb_render_rays_backward(const sdb_render_params *p, const void *d_record, const sdb_render_grads *g, void *stream);

/* --------------------------------------------------------------------------------------------
 * a9 under autograd.  sdb_sky_train_forward = sdb_sky_forward (fp16x3, ONE style code / image)
 * that also records PE(raydir), the five hidden activations (bf16) and their LeakyReLU sign
 * words; sdb_sky_backward turns dL/d sky [R,64] (ray order; the contribution of the frame mean
 * already added by the caller) into the SKYMLP weight gradients (gancraft_base.py:150-169 under
 * torch.autograd): gradient chain + weight gradients on the tensor-core engine.
 *   d_grad_w1ext [256, 48]: cols 0..32 fc1.weight, col 47 the layer-0 bias (fc1.bias + fc_z_a(z));
 *   d_grad_wh [4][256, 272]: fc2..fc5 (cols 0..255 weight, col 256 bias); d_grad_wout [64, 272].
 *   backward pack: sdb_pack_sky_mlp_backward(wh [4][256,256], wout [64,256]).
 * ------------------------------------------------------------------------------------------ */
int64_t sdb_sky_train_record_bytes(int32_t n_img, int32_t H, int32_t W);
int sdb_sky_train_forward(const float *d_raydirs, int32_t n_img, int32_t H, int32_t W, const void *d_sky_pack,
                          float *d_sky, float *d_sky_avg, void *d_workspace, void *d_record, void *stream);
int64_t sdb_sky_backward_pack_bytes(void);
int sdb_pack_sky_mlp_backward(const float *d_wh, const float *d_wout, void *d_pack, void *stream);
int64_t sdb_sky_backward_workspace_bytes(int32_t n_img, int32_t H, int32_t W);
int sdb_sky_backward(int32_t n_img, int32_t H, int32_t W, const void *d_record, const float *d_grad_sky,
                     const void *d_bwd_pack, float *d_grad_w1ext, float *d_grad_wh, float *d_grad_wout,
                     void *d_workspace, void *stream);

/* --------------------------------------------------------------------------------------------
 * f1. RenderCNN + tanh on the tensor cores: per-pixel feature map -> image.
 * Replaces Base3DGenerator._forward_global = RenderCNN.forward + tanh
 *   (imaginaire/generators/gancraft_base.py:172-225, :588-603) for the WHOLE padded frame at once
 *   (the reference's tile loop, scenedreamer.py:600-628, computes the same function tile by tile).
 *   pack: sdb_cnn_pack() from the reference's `denoiser.*` tensors (device fp32, their shapes):
 *         conv1 [256,64,1,1]+[256]; conv2a, conv3a [256,256,3,3]+[256]; conv2b, conv3b [256,256,3,3];
 *         conv4a, conv4b [256,256,1,1]+[256]; conv4 [3,256,1,1]+[3];
 *   d_mod [4][256] = fc_z_cond(z) for ONE style code (the four `adapt` chunks, gancraft_base.py:208-209);
 *   d_net_out [H][W][64] fp32 (the fused kernel's net_out) -> d_rgb [3][H][W] = tanh(raw), d_rgb_raw
 *   [3][H][W] or NULL;  precision 2 = fp16 hi/lo split x3 (fp32-grade, parity), 0 = one fp16 pass;
 *   d_workspace: sdb_cnn_workspace_bytes() bytes; workspace_ready = 0 on the first call for a given
 *   (workspace, H, W, precision) -- the call then clears the zero borders -- and 1 afterwards.
 * ------------------------------------------------------------------------------------------ */
int64_t sdb_cnn_pack_bytes(int32_t precision);
int sdb_cnn_pack(const float *d_w1, const float *d_b1, const float *d_w2a, const float *d_b2a, const float *d_w2b,
                 const float *d_w3a, const float *d_b3a, const float *d_w3b, const float *d_w4a, const float *d_b4a,
                 const float *d_w4b, const float *d_b4b, const float *d_w4, const float *d_b4, int32_t precision,
                 void *d_pack, void *stream);
int64_t sdb_cnn_workspace_bytes(int32_t H, int32_t W, int32_t precision);
int sdb_cnn_forward(const float *d_net_out, int32_t H, int32_t W, const void *d_pack, const float *d_mod,
                    int32_t precision, float *d_rgb, float *d_rgb_raw, void *d_workspace, int32_t workspace_ready,
                    void *stream);

/* --------------------------------------------------------------------------------------------
 * a8 (training): the style modulation of LightningMLP's five ModLinear layers for ONE style code, folded into plain
 * weights, forward and backward (imaginaire/model_utils/layers.py:241-271 as used at :92-126):
 *   alpha = weight_alpha z + bias_alpha [I], beta = weight_beta z + bias_beta [O], W' = W * alpha (per input column).
 * d_params / d_grads: 25 device pointers, float32, contiguous, in the order
 *   weight[0..4] [O,I], weight_alpha[0..4] [I,Cz], bias_alpha[0..4] [I], weight_beta[0..4] [O,Cz], bias_beta[0..4] [O]
 * (layers fc_2 .. fc_6).  forward: d_alpha [5,I], d_wh [5,O,I], d_bh [5,O] (= beta).  backward: from d_g_wh [5,O,I] and
 * d_g_bh [5,O] every parameter gradient (d_grads, same order, OVERWRITTEN) and d_dz [Cz]; d_dalpha [5,I] is scratch.
 * Replaces ~110 ATen launches per training view of the torch formulation (the backward is host-bound there).
 * ------------------------------------------------------------------------------------------ */
int sdb_modulate_forward(const void *const d_params[25], const float *d_z, int32_t O, int32_t I, int32_t Cz, float *d_alpha,
                         float *d_wh, float *d_bh, void *stream);
int sdb_modulate_backward(const void *const d_params[25], void *const d_grads[25], const float *d_z, const float *d_alpha,
                          const float *d_g_wh, const float *d_g_bh, int32_t O, int32_t I, int32_t Cz, float *d_dalpha,
                          float *d_dz, void *stream);

/* --------------------------------------------------------------------------------------------
 * f2. The Adam step of the hash table in one pass over (param, grad, exp_avg,
 * exp_avg_sq) -- torch.optim.Adam's arithmetic and state (imaginaire/utils/trainer.py:297-323,
 * configs/scenedreamer_train.yaml:36-61: betas (0, 0.999), eps 1e-7, no weight decay / amsgrad).
 * n elements (multiple of 4, 16-byte aligned arrays); step = count AFTER the increment (>= 1); the
 * hyper-parameters are doubles (Python floats): 1 - beta, the bias corrections and lr / bc1 are formed
 * in double and narrowed last, as torch does.
 * With beta1 == 0 entries whose gradient is exactly 0 only decay exp_avg_sq (param / exp_avg are
 * not read) -- identical to the dense formula.
 * ------------------------------------------------------------------------------------------ */
int sdb_adam_step(float *d_param, const float *d_grad, float *d_exp_avg, float *d_exp_avg_sq, int64_t n, double lr,
                  double beta1, double beta2, double eps, int64_t step, void *stream);

/* --------------------------------------------------------------------------------------------
 * f4. Rejection statistics of the training camera sampler, one pass on the
 * device (Generator._get_batch, imaginaire/generators/scenedreamer.py:127-142):
 *   d_stats[0] = mean of the non-NaN first-hit entry depths depth2[0, :, :, 0]
 *   d_stats[1] = -sum_k p_k log(p_k + 1e-10), p_k = share of rays whose first voxel id is k (n_bins = 680)
 * d_voxel_id [H*W, M] int32, d_depth2 [2][H*W][M]; d_workspace: sdb_pose_stats_workspace_bytes().
 * ------------------------------------------------------------------------------------------ */
int64_t sdb_pose_stats_workspace_bytes(int32_t n_bins);
int sdb_pose_stats(const int32_t *d_voxel_id, const float *d_depth2, int32_t H, int32_t W, int32_t M, int32_t n_bins,
                   float *d_stats, void *d_workspace, void *stream);

/* --------------------------------------------------------------------------------------------
 * f3. Voxel world of a scene from its bird's-eye-view maps, built in HBM.
 * Replaces the CPU scatter passes, the per-tree Python loop and the 1-4 GB host->device copy of
 * PCGVoxelGenerator.next_world (imaginaire/model_utils/pcg_gen.py:83-174).
 *   sdb_world_build: d_hq / d_label int32 [X, Z] (quantised height index, block id per column);
 *     tree instances d_inst int32 [n_inst, 4] = (h, x, z, model) in the reference's iteration order,
 *     models concatenated in d_models with dims d_mdim [n_models, 3] and offsets d_moff int64;
 *     -> d_world int32 [SH, X, Z] (scratch), d_heightmap int64 [X, Z], d_minmax int32[2] = {gnd, top}.
 *   sdb_world_truncate: d_voxel_t [sky - gnd, X, Z] = world[gnd:sky] (tree keys decoded).
 * ------------------------------------------------------------------------------------------ */
int sdb_world_build(const int32_t *d_hq, const int32_t *d_label, int32_t X, int32_t Z, int32_t SH, const int32_t *d_inst,
                    int32_t n_inst, const int32_t *d_models, const int32_t *d_mdim, const int64_t *d_moff,
                    int32_t *d_world, int64_t *d_heightmap, int32_t *d_minmax, void *stream);
int sdb_world_truncate(const int32_t *d_world, int32_t X, int32_t Z, int32_t gnd, int32_t sky, int32_t *d_voxel_t, void *stream);

/* Kernels this library has launched in this process so far (every launch is counted; memsets and
 * library GEMMs are not).  bench.py reads it around its timed region for `gpu_launches`.          */
int64_t sdb_launch_count(void);

/* Diagnostics only: byte offsets inside the training record / backward workspace (20 int64, see render_train.cu). */
int sdb_debug_train_layout(int32_t n_img, int32_t H, int32_t W, int32_t S, int32_t L, int32_t log2_T, int64_t *out);

/* Diagnostics only: host-mapped (pinned) int32[64] progress buffer written by CTA 0 of the fused
 * kernels (role, step, layer markers); pass NULL to disable (default).                          */
void sdb_debug_set_progress_buffer(void *mapped);

/* tensor-core (wgmma) self test: C[128,N] = A[128,K] * B[N,K]^T with the exact smem descriptors the
 * fused kernel uses.  d_a, d_b fp32 inputs (rounded to fp16/bf16 inside), d_c fp32 output.
 * variant 0 = the layout the library uses; 1 = LBO/SBO swapped (diagnostic only).              */
int sdb_tc_selftest(const float *d_a, const float *d_b, float *d_c, int32_t N, int32_t K,
                    int32_t use_bf16, int32_t variant, void *stream);

/* Diagnostic: C[128, G] = X^T Y for X [128 samples, 128], Y [128 samples, G] (fp32 in, bf16 inside) with both operands
 * read MN-major from the activation tile layout of the fused kernels (samples = reduction dimension); variant 0 / 1 =
 * the two assignments of the descriptor's LBO / SBO fields.                                                          */
int sdb_tc_selftest_mn(const float *d_x, const float *d_y, float *d_c, int32_t G, int32_t variant, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SDB200_H */
