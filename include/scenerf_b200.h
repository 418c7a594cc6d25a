/*
 * scenerf_b200 -- C ABI of the Hopper (sm_90a) ray renderer that replaces the hot path of
 * astra-vision/SceneRF: `SceneRF.render_rays_batch` (reference scenerf/models/scenerf.py:392-471, BundleFusion twin
 * scenerf/models/scenerf_bf.py:420-494) and everything below it.
 *
 * The reference has no FFI: its boundary is a bound Python method.  This header is the boundary a maintainer binds
 * instead (ctypes stub in INTEGRATION.md; scenerf_b200/renderer.py is that binding).  Conventions:
 *   - plain C, no torch types; every `*_dev` pointer is a CUDA device pointer, every `*_host` pointer host memory;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream); no call synchronises the device
 *     except the *_host entry points;
 *   - no hidden device allocations: packed buffers and workspace are supplied by the caller (sizes from the
 *     *_bytes functions); the library never falls back to a CPU path;
 *   - return value 0 = ok, otherwise an SRF_E_* code and a message in srf_last_error() (thread-local).
 * The reference raises Python exceptions for bad shapes (torch) -- the Python binding turns non-zero codes into
 * RuntimeError / ValueError.
 */
#ifndef SCENERF_B200_H
#define SCENERF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SRF_ABI_VERSION 2
#define SRF_NUM_SCALES 5   /* x_rgb keys "1_1","1_2","1_4","1_8","1_16" (unet2d_sphere.py:200-206) */
#define SRF_NUM_BLOCKS 3   /* ResnetFC n_blocks (scenerf.py:100-114) */
#define SRF_D_HIDDEN 512
#define SRF_D_X 42         /* 39 positional-encoding + 3 view direction (scenerf.py:101) */
#define SRF_MAX_GAUSSIANS 8

enum srf_status {
  SRF_OK = 0,
  SRF_E_INVALID = 1,   /* bad argument / shape */
  SRF_E_WORKSPACE = 2, /* workspace or packed buffer too small */
  SRF_E_CUDA = 3,      /* CUDA runtime error (message has the cudaError string) */
  SRF_E_UNSUPPORTED = 4
};

enum srf_precision {
  SRF_PREC_FP32 = 0, /* SIMT fp32 FMA everywhere: strict mode, matches the reference to float32 round-off */
  SRF_PREC_FP16_TC = 1, /* wgmma tensor cores: fp16 operands, fp32 accumulate ("fast mode") */
  SRF_PREC_FP32_TC = 2  /* wgmma tensor cores at float32-grade accuracy: every fp32 operand is carried as an fp16
                           hi/lo pair (22 mantissa bits), all four partial products accumulate in fp32.
                           The precision-matched mode for the reference's fp32 sgemm (resnetfc.py:54-63,133-164);
                           needs an SRF_PYR_FP32 pyramid and srf_pack_weights_tc_split() output */
};

enum srf_dataset { SRF_KITTI = 0, SRF_BUNDLEFUSION = 1 };

/* Storage of the packed feature pyramid.  FP32 is required by SRF_PREC_FP32.  FP16 halves the bytes of every bilinear
 * tap (one 128-bit load per 8 channels) for the tensor-core mode, whose operands are rounded to fp16 anyway. */
enum srf_pyramid_format { SRF_PYR_FP32 = 0, SRF_PYR_FP16 = 1 };

/* The 22 tensors of one ResnetFC exactly as nn.Linear stores them: weight (out,in) row-major fp32, bias (out).
 * Reference: scenerf/models/resnetfc.py:66-131; state-dict names in comments. */
typedef struct srf_mlp_weights {
  int d_out;                               /* 4 for `mlp`, 2 for `mlp_gaussian` */
  int d_latent;                            /* 2480 = sum of pyramid channels */
  const float* lin_in_w;                   /* lin_in.weight   (512, 42)   */
  const float* lin_in_b;                   /* lin_in.bias     (512)       */
  const float* lin_z_w[SRF_NUM_BLOCKS];    /* lin_z.b.weight  (512, 2480) */
  const float* lin_z_b[SRF_NUM_BLOCKS];    /* lin_z.b.bias    (512)       */
  const float* fc0_w[SRF_NUM_BLOCKS];      /* blocks.b.fc_0.weight (512,512) */
  const float* fc0_b[SRF_NUM_BLOCKS];
  const float* fc1_w[SRF_NUM_BLOCKS];      /* blocks.b.fc_1.weight (512,512) */
  const float* fc1_b[SRF_NUM_BLOCKS];
  const float* lin_out_w;                  /* lin_out.weight  (d_out, 512) */
  const float* lin_out_b;
  const void* tc_packed;                   /* srf_pack_weights_tc() output, or NULL if SRF_PREC_FP16_TC is not used */
  const void* tc_split_packed;             /* srf_pack_weights_tc_split() output, or NULL if SRF_PREC_FP32_TC is not used */
} srf_mlp_weights;

/* Feature pyramid of ONE input image, repacked channels-last ([H][W][C] fp32) by srf_pack_pyramid().
 * Reference input: x_rgb dict of CHW tensors, consumed at scenerf.py:522-525 / utils.py:232-247. */
typedef struct srf_pyramid {
  const void* hwc[SRF_NUM_SCALES];   /* [H][W][C] of float (format 0) or IEEE half (format 1) */
  int C[SRF_NUM_SCALES], H[SRF_NUM_SCALES], W[SRF_NUM_SCALES];
  int format;                        /* srf_pyramid_format */
  const void* latent_table;          /* optional: srf_build_latent_table() output for the MAIN network (`mlp`), else NULL */
  const void* latent_table_gauss;    /* optional: the same for `mlp_gaussian` (its own lin_z weights), else NULL */
  int latent_table_format;           /* srf_pyramid_format of the table rows: FP16 is used by SRF_PREC_FP16_TC, FP32 by SRF_PREC_FP32_TC */
} srf_pyramid;

/* Hyper-parameters the path reads from the module (scenerf.py:23-115) + per-call camera and pose. */
typedef struct srf_config {
  int dataset;               /* srf_dataset: selects the +1.5 / +0.5 constant (scenerf.py:592 vs scenerf_bf.py:606) */
  int n_pts_uni;             /* U */
  int n_gaussians;           /* G */
  int n_pts_per_gaussian;    /* P ; samples per ray S = U + G*P */
  float max_sample_depth;
  float base_std;            /* self.std */
  float som_sigma;
  int sphere_W, sphere_H;    /* out_img_W / out_img_H */
  int d_latent;              /* total pyramid channels (ResnetFC d_latent); 0 means the reference's 2480 */
  float v_angle_min, v_angle_max, h_angle_min, h_angle_max; /* SphericalMapping angles incl. add_fov */
  float K[9];                /* cam_K row-major */
  float inv_K[9];            /* torch.inverse(cam_K) (scenerf.py:401) -- supplied by the caller so that it is bit-equal */
  float T[16];               /* T_source2infer row-major */
  int precision;             /* srf_precision */
  uint64_t seed;             /* in-kernel Philox seed when noise pointers are NULL */
  int flags;                 /* SRF_FLAG_* */
  int ray_offset;            /* index of this call's first ray inside the frame it belongs to: the Philox counter of ray i
                                is (seed, ray_offset + i, sample), so a frame rendered in shards (several calls, several
                                GPUs: scenerf_b200/dist.py) draws exactly the noise of the unsharded call */
} srf_config;

#define SRF_FLAG_HIDDEN_FP16 2       /* tensor-core path: the residual hidden state h travels between ResNet blocks as
                                       fp16 instead of fp32 (GEMM accumulation stays fp32).  Halves the
                                       L2 traffic of the epilogues; h is rounded to fp16 as the next GEMM's operand
                                       anyway, measured effect on depth/colour error < 15 % of the fp16-mode error */
#define SRF_FLAG_TF32_MATMUL 8      /* float32 path, training (needs SRF_FLAG_SAVE_ACTIVATIONS in the forward): the GEMMs of the
                                       forward and of srf_render_rays_backward run on tensor cores as wgmma tf32
                                       (float32 storage, 10-bit mantissa operands, float32 accumulate) -- the regime of the
                                       reference's own torch 1.7.1 defaults on Ampere-class GPUs.  Not bit-compatible with
                                       the strict float32 mode; tolerances in DESIGN.md 6.3. */
#define SRF_FLAG_SAVE_ACTIVATIONS 4 /* float32 path, training: srf_render_rays keeps the ResnetFC pre-activations of both MLP
                                       passes in its workspace (24.4 KB per sample point) so that srf_render_rays_backward
                                       does not recompute the forward.  Outputs are bit-identical with and without it. */
#define SRF_FLAG_SKIP_ZERO_CHUNKS 1 /* tensor-core path: skip K-chunks of lin_z whose gathered features are all
                                       zero for the whole 128-point tile (bit-identical result) */

/* Outputs of render_rays_batch: the 12-key dict of scenerf.py:456-469.  Any pointer may be NULL (not written);
 * inference callers need only depth and color.  All fp32, ray order = input order, samples sorted by distance. */
typedef struct srf_outputs {
  float* depth;                 /* (R)   */
  float* color;                 /* (R,3) */
  float* gaussian_means;        /* (R,G) */
  float* gaussian_stds;         /* (R,G) */
  float* weights_at_depth;      /* (R)   */
  float* closest_pts_to_depths; /* (R)   */
  float* loss_kl;               /* (R)   */
  float* alphas;                /* (R,S) */
  float* som_vars;              /* (R,G) */
  float* densities;             /* (R,S) */
  float* weights;               /* (R,S) */
  float* depth_volumes;         /* (R,S) */
  float* som_means;             /* (R,G) extra: RaySOM new_means (ray_som_kl.py:78), not part of the dict */
  int32_t* dbg_sphere_main;     /* (R*S,2) extra: rounded sphere coords of the main pass (parity diagnostics) */
  int32_t* dbg_sphere_gauss;    /* (R*G,2) */
} srf_outputs;

int srf_abi_version(void);
const char* srf_last_error(void);
/* sizeof() of the ABI structs as the library was compiled: 0 srf_config, 1 srf_pyramid, 2 srf_mlp_weights,
 * 3 srf_outputs -- lets a foreign-language binding verify its struct layout at load time. */
size_t srf_sizeof(int which);

/* --- one-time packing ------------------------------------------------------------------------------------- */
size_t srf_pyramid_bytes(const int* C, const int* H, const int* W, int format);
/* CHW fp32 (device) -> HWC fp32 / fp16 (srf_pyramid_format) into dst_dev; fills *out.  Replaces nothing in the reference: it is the layout
 * change that makes the 4-tap gather of utils.py:239-245 read contiguous channels. */
int srf_pack_pyramid(const float* const* chw_dev, const int* C, const int* H, const int* W, int format, void* dst_dev,
                     size_t dst_bytes, srf_pyramid* out, void* stream);

size_t srf_tc_weights_bytes(int d_out, int d_latent);
/* fp32 nn.Linear tensors -> fp16 K-major, 128B-swizzled shared-memory stage images in MMA consumption order. */
int srf_pack_weights_tc(const srf_mlp_weights* w, void* dst_dev, size_t dst_bytes, void* stream);
/* The same stage images for SRF_PREC_FP32_TC: every weight is scaled by a power of two 2^s (max|w| 2^s in
 * [2^13, 2^14), exact, undone in the epilogues) and stored as two fp16 images, hi = rn(w 2^s) and lo = rn(w 2^s - hi). */
size_t srf_tc_split_weights_bytes(int d_out, int d_latent);
int srf_pack_weights_tc_split(const srf_mlp_weights* w, void* dst_dev, size_t dst_bytes, void* stream);

/* Pre-projected latents (optional, once per image and network).  SphericalMapping.from_pixels rounds the sphere
 * coordinates to integers (spherical_mapping.py:115), so the 2480-channel latent of a sample point -- and therefore
 * lin_z[b](z) of resnetfc.py:148-150 -- is a function of the integer sphere pixel only.  The table holds
 * lin_z[b].weight . z(pixel) (3 x 512 values) for every pixel that can have a valid bilinear tap (+ one zero row); with
 * `pyr->latent_table` (`latent_table_gauss`) set, the tensor-core modes skip the three lin_z GEMM passes of the main
 * (gaussian-proposal) network -- 70.5 % of the per-point FLOPs -- and add the table row in the epilogue.  A table
 * belongs to ONE network: build it with that network's weights.  Exact in real arithmetic; rounding differs from the dense
 * path at float32 round-off (fp32 table) / fp16 round-off (fp16 table).  pyr must be an SRF_PYR_FP32 pack.
 * Sizes: table (sphere_W+1)*(sphere_H+1)*1536 values (config B: 1.4 GB fp16 / 2.8 GB fp32); workspace 2 KB per texel. */
size_t srf_latent_table_bytes(const srf_config* cfg, int format);
size_t srf_latent_table_workspace_bytes(const srf_pyramid* pyr);
int srf_build_latent_table(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w, int format,
                           void* table_dev, size_t table_bytes, void* workspace_dev, size_t workspace_bytes, void* stream);

/* --- the hot path ----------------------------------------------------------------------------------------- */
size_t srf_render_workspace_bytes(const srf_config* cfg, int n_rays);

/* SceneRF.render_rays_batch (scenerf.py:392-471) for one chunk-free batch of rays.
 *   pixels_dev (R,2) fp32 (x,y);  noise_u_dev (R,U) U[0,1) or NULL;  noise_n_dev (R,G*P) N(0,1) or NULL
 *   (the two RNG draws of utils.py:84 and utils.py:208-211; NULL = Philox from cfg->seed). */
int srf_render_rays(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w_main,
                    const srf_mlp_weights* w_gauss, const float* pixels_dev, int n_rays, const float* noise_u_dev,
                    const float* noise_n_dev, const srf_outputs* out, void* workspace_dev, size_t workspace_bytes,
                    void* stream);

/* Same call with HOST buffers for pixels and outputs (pinned or pageable): H2D of the rays, render, D2H of the
 * requested outputs, stream synchronised on return.  out_host pointers are host pointers. */
int srf_render_rays_host(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w_main,
                         const srf_mlp_weights* w_gauss, const float* pixels_host, int n_rays,
                         const srf_outputs* out_host, void* workspace_dev, size_t workspace_bytes, void* stream);
size_t srf_render_host_workspace_bytes(const srf_config* cfg, int n_rays);

/* SceneRF.predict (scenerf.py:505-547): points already in the infer-camera frame.
 *   cam_pts_dev (n_cols*n_per,3); viewdir_dev (n_cols,3) shared by the n_per points of a column;
 *   raw_out_dev (n, d_out) = ResnetFC output before activation, or NULL;
 *   density_dev (n) = softplus(out[3]-1), color_dev (n,3) = sigmoid(out[:3]) (d_out==4 only), or NULL. */
size_t srf_predict_workspace_bytes(const srf_config* cfg, int n_points);
int srf_predict(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w, const float* cam_pts_dev,
                const float* viewdir_dev, int n_cols, int n_per, float* raw_out_dev, float* density_dev,
                float* color_dev, int32_t* dbg_sphere_dev, void* workspace_dev, size_t workspace_bytes,
                void* stream);

/* --- next row: backward pass (training drop-in) ----------------------------------------------------------------------
 * What torch.autograd computes for SceneRF.render_rays_batch (scenerf.py:392-748; consumers of the gradients: the losses
 * of scenerf.py:243-320).  float32 precision and an SRF_PYR_FP32 pyramid only.  Call srf_render_rays first with ALL 12
 * dict outputs plus `som_means` requested and keep its workspace untouched: the backward reads the forward's
 * intermediates (sorted distances, sample points, raw MLP outputs) from it.
 *   noise_n_dev     : the same (R,G*P) tensor the forward got, or NULL when the forward drew Philox noise (same cfg->seed)
 *   fwd_out         : the forward's outputs;  grad_out: cotangents with the same shapes, NULL members = zero.
 *                     `som_vars` cotangents are ignored: RaySOM statistics are not differentiated (their only consumer logs
 *                     them detached, scenerf.py:222-227); everything else matches autograd (scenerf.py:662 detach included).
 *   grad_main/gauss : float32 device buffers shaped like the weights (srf_mlp_weights used as a pointer table, packed_tc
 *                     ignored); gradients are ACCUMULATED into them (zero them for a fresh gradient).
 *   grad_pyr_chw[5] : float32 CHW buffers shaped like the caller's feature maps; accumulated with atomics.
 * Parameter gradients are bit-reproducible run to run; feature-map gradients up to float atomics ordering. */
size_t srf_render_backward_workspace_bytes(const srf_config* cfg, int n_rays);
int srf_render_rays_backward(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w_main,
                             const srf_mlp_weights* w_gauss, int n_rays, const float* noise_n_dev,
                             const srf_outputs* fwd_out, const srf_outputs* grad_out, const void* fwd_workspace_dev,
                             size_t fwd_workspace_bytes, const srf_mlp_weights* grad_main,
                             const srf_mlp_weights* grad_gauss, float* const* grad_pyr_chw, void* workspace_dev,
                             size_t workspace_bytes, void* stream);

/* --- next row: TSDF fusion of the rendered depth sweeps ----------------------------------------------------------
 * TSDFVolume.integrate of the reference (scenerf/data/utils/fusion.py:219-324, the CPU / numba semantics that
 * scripts/reconstruction/depth2tsdf.py:87-103 runs): volumes are (dims[0],dims[1],dims[2]) C-order fp32 device arrays
 * owned by the caller.  srf_tsdf_reset = constructor state (tsdf 255, weight 0, colour 0; fusion.py:55-58).
 *   origin[3] float32 volume origin; voxel_size; inv_cam_pose_host[16] = inverse(cam_pose) row-major float64 (the
 *   reference inverts in float64, fusion.py:265); cam_intr_host[9] row-major float32; depth_dev (H,W) float32;
 *   color_dev (H,W,3) float32 or uint8 (color_is_u8). */
int srf_tsdf_reset(float* tsdf_dev, float* weight_dev, float* color_dev, const int* dims, void* stream);
int srf_tsdf_integrate(float* tsdf_dev, float* weight_dev, float* color_dev, const int* dims, const float* origin,
                       double voxel_size, const double* inv_cam_pose_host, const float* cam_intr_host,
                       const float* depth_dev, const void* color_dev_im, int color_is_u8, int im_h, int im_w,
                       double trunc_margin, float obs_weight, void* stream);

/* Merge volume B into A (same dims) with integrate's fold rule: keep A where |A| < |B|, else B's distance and colour;
 * weights add.  Used when the poses of one sweep are integrated on several GPUs: merging the ranks' volumes in pose
 * order equals integrating all poses sequentially (fusion.py:212-216): distances and weights bit for bit, colours
 * except on float32-exact distance ties between observations of different ranks (either minimal observation). */
int srf_tsdf_merge(float* tsdf_a, float* weight_a, float* color_a, const float* tsdf_b, const float* weight_b,
                   const float* color_b, const int* dims, void* stream);

/* --- next row: mesh extraction from the fused volume ---------------------------------------------------------------
 * TSDFVolume.get_mesh / get_point_cloud of the reference (fusion.py:333-379): marching cubes at level 0 over the
 * (dims[0],dims[1],dims[2]) C-order tsdf volume, on the device (DESIGN.md 6.6).  A voxel is inside iff its value is < 0
 * (unobserved voxels hold 255: outside).  mask_dev: (X,Y,Z) uint8 or NULL; voxels whose mask is 0 read as 1.0 (the
 * volume itself is not written).  Output order does not depend on thread scheduling: vertices by owning grid point in
 * C order (then +x, +y, +z edge), faces by cell in C order.
 * Two calls on the same workspace:
 *   srf_tsdf_mesh_count_host : counts vertices and faces; synchronises the stream (host results, hence _host).
 *   srf_tsdf_mesh_emit       : writes verts_dev (V,3) float32 world coordinates float32(v*float32(voxel_size) + origin),
 *                              normals_dev (V,3) float32 unit gradients toward increasing tsdf (0 where the gradient is 0),
 *                              colors_dev (V,3) uint8 (r,g,b) unfolded from color_dev at the rounded index,
 *                              faces_dev (F,3) int32 vertex ids; normals / colors / faces may be NULL (not written).
 * A volume with a dimension < 2 gives an empty mesh; volumes whose counts could overflow int32 are rejected. */
size_t srf_tsdf_mesh_workspace_bytes(const int* dims);
int srf_tsdf_mesh_count_host(const float* tsdf_dev, const uint8_t* mask_dev, const int* dims, void* ws, size_t ws_bytes,
                             long long* n_verts, long long* n_faces, void* stream);
int srf_tsdf_mesh_emit(const float* tsdf_dev, const float* color_dev, const uint8_t* mask_dev, const int* dims,
                       const float* origin, double voxel_size, const void* ws, size_t ws_bytes, float* verts_dev,
                       float* normals_dev, uint8_t* colors_dev, int32_t* faces_dev, void* stream);

/* --- evaluation metrics on the device (DESIGN.md 6.7) ----------------------------------------------------------------
 * srf_eval_confusion: one pass over a (dims[0],dims[1],dims[2]) C-order volume.  The prediction is either
 *   - the occupancy of tsdf2occ (eval_sr.py:11-17, eval_sc_bf.py:117-123): pred_dev NULL, tsdf_dev float32, occupied iff
 *     double(|tsdf|) < th_dev[index along th_axis] and |tsdf| != 255; th_dev holds dims[th_axis] float64 thresholds
 *     (computed by the caller with the reference's expression and clamps); occ_dev (uint8 0/1) is written if non-NULL;
 *   - or pred_dev, an array of the srf_eval_dtype pred_dtype (tsdf_dev, th_dev, occ_dev unused).
 * target_dev: uint8 labels, 255 = not evaluated (NULL in occupancy mode: only occ_dev is written).  mask_dev: uint8 0/1 or NULL.
 * hist_dev: srf_eval_hist_len(dims, n_classes, per_z) int64 counters, zeroed here and then filled:
 *   hist[zh][m][tb][pb], zh = z slice (per_z != 0) or 0, m = 0 every voxel / 1 voxels with mask 1,
 *   tb = target bucket (label l < n_classes -> l, any other label but 255 -> n_classes; 255 is not counted),
 *   pb = pred bucket (value j in [0, n_classes) -> j, other value > 0 -> n_classes, the rest -> n_classes + 1).
 *   The tsdf occupancy counts as pred 1 (n_classes + 0 when n_classes == 1).
 * max_z_dev (one int): the largest z holding a label other than 0 and 255, -1 if none. */
enum srf_eval_dtype { SRF_EVAL_U8 = 0, SRF_EVAL_I32 = 1, SRF_EVAL_I64 = 2, SRF_EVAL_F32 = 3, SRF_EVAL_F64 = 4 };
#define SRF_EVAL_MAX_CLASSES 64
size_t srf_eval_hist_len(const int* dims, int n_classes, int per_z);
int srf_eval_confusion(const float* tsdf_dev, const void* pred_dev, int pred_dtype, const uint8_t* target_dev,
                       const uint8_t* mask_dev, const int* dims, int n_classes, int th_axis, const double* th_dev, int per_z,
                       long long* hist_dev, int* max_z_dev, uint8_t* occ_dev, void* stream);
/* generate_sc_gt_bf.py:307-309: out_dev = 255, then 0 where tsdf > float32(voxel_size), then 1 where |tsdf| <
 * float32(voxel_size), both only where tsdf != 255 (float32 comparisons). */
int srf_eval_sc_label(const float* tsdf_dev, const int* dims, double voxel_size, uint8_t* out_dev, void* stream);
/* F.interpolate(size=(out_h,out_w), mode="bilinear", align_corners=False) of one row-major float32 image. */
int srf_resize_bilinear(const float* src_dev, int in_h, int in_w, float* dst_dev, int out_h, int out_w, void* stream);
/* compute_depth_errors (loss/depth_metrics.py) of n (gt, pred) float32 pairs; pred is clamped to [1e-3, 80] on the fly
 * (the inputs are not written).  Sums in float64 with a fixed order.  The frame's (abs_rel, sq_rel, rmse, rmse_log,
 * a1, a2, a3) -- the first four rounded to float32 as the reference returns them -- are written to frame_dev[7] if
 * non-NULL and added to buckets_dev[slot*8 + 0..6], and buckets_dev[slot*8 + 7] += 1 (frame count), if buckets_dev is
 * non-NULL.  Nothing synchronises.  ws: srf_depth_errors_workspace_bytes() bytes. */
size_t srf_depth_errors_workspace_bytes(void);
int srf_depth_errors(const float* gt_dev, const float* pred_dev, long long n, void* ws, size_t ws_bytes, double* buckets_dev,
                     int slot, double* frame_dev, void* stream);

/* Novel-view colour metrics (scripts/evaluation/eval_color.py / eval_color_bf.py), DESIGN.md 6.8.  Images are (h,w,3)
 * row-major float32 in [0,1], as eval_color.py passes them.
 * srf_psnr_ssim: skimage 0.18.1 peak_signal_noise_ratio(data_range=1) -- 10*log10(1/mse), the squared difference formed in
 *   float32, inf for identical images -- and structural_similarity(multichannel=True, data_range=1): per channel, 7x7 box
 *   means in float64, S over the interior [3, h-4] x [3, w-4], mean of the three channel means.  Both sides >= 7 (skimage
 *   raises below).  frame_dev[2] = (psnr, ssim) if non-NULL; buckets_dev rows of 4 doubles [psnr, ssim, lpips, n]:
 *   row slot += (psnr, ssim, 0, 1) if non-NULL.  Sums in a fixed order: bit-identical from run to run.  Nothing
 *   synchronises.  ws: srf_psnr_ssim_workspace_bytes(h, w) bytes (0 for a side below 7).
 * srf_lpips_vgg: lpips 0.1 LPIPS(net="vgg", version="0.1") of one pair of [0,1] images: the (x-0.5)*2 of compute_lpips,
 *   the scaling layer (x - shift[c]) / scale[c] (3 host floats each), torchvision VGG16 features[0:30] (13 conv3x3+ReLU on the srf_conv3x3_hwc kernel, 4 max-pools 2x2 floor),
 *   the head at the five taps (relu1_2 .. relu5_3): f / (sqrt(sum_c f^2) + 1e-10), squared difference, dot lin[k]
 *   (64/128/256/512/512 floats), spatial mean; *out_dev (one float32) = the sum of the five means.
 *   w9_dev[13]: [9][Cout][Cin] (tap = ky*3 + kx), values rounded to the nearest tf32 by the caller; Cin = 32 for conv1_1
 *   (RGB then 29 zero channels), the previous Cout otherwise.  bias_dev[13]: (Cout).  Device pointers 16-byte aligned.
 *   Sides in [16, 8192].  ws: srf_lpips_workspace_bytes(h, w) bytes.  Nothing synchronises. */
size_t srf_psnr_ssim_workspace_bytes(int h, int w);
int srf_psnr_ssim(const float* img_dev, const float* gt_dev, int h, int w, void* ws, size_t ws_bytes, double* buckets_dev, int slot,
                  double* frame_dev, void* stream);
size_t srf_lpips_workspace_bytes(int h, int w);
int srf_lpips_vgg(const float* img0_dev, const float* img1_dev, int h, int w, const float* const* w9_dev, const float* const* bias_dev,
                  const float* const* lin_dev, const float* shift_host, const float* scale_host, void* ws, size_t ws_bytes, float* out_dev,
                  void* stream);

/* --- next row: image-side glue of the novel-view sweep (scripts/reconstruction/generate_novel_depths.py:103-152) ---
 * The reference renders an x-major stride-`scale` pixel grid (gw x gh rays, ray = ix*gh + iy), reshapes, transposes
 * and F.interpolate(bilinear)s to (H,W).  srf_upsample_render does that in one pass from the render outputs:
 * depth_xm (gw*gh) -> depth_out (H,W); color_xm (gw*gh,3) -> color_out (H,W,3).  Either pair may be NULL.
 * gw==W && gh==H is the scale-1 case (transpose only).  color_mode: 0 raw, 1 clamp to [0,1] (:144),
 * 2 = the PNG round trip the reference's TSDF stage sees: float32(uint8(c*255))/255*255 (depth2tsdf.py:19-26,98),
 * 3 = the PNG round trip eval_color.py scores: float32(uint8(c*255))/255, in [0,1] (render_colors.py:123-127, eval_color.py:93-94). */
int srf_upsample_render(const float* depth_xm, const float* color_xm, int gw, int gh, int out_h, int out_w,
                        float* depth_out, float* color_out, int color_mode, void* stream);

/* --- next row (producer side): DecoderSphere.get_sphere_feature, scenerf/models/unet2d_sphere.py:138-166 ------------------
 * x_chw_dev (C,h,w) float32 image-plane feature map of ONE image; pix_dev (n,2) float32 image pixels and
 * pix_sphere_dev (n,2) int64 sphere pixels as SphericalMapping.from_pixels returns them (spherical_mapping.py:80-93);
 * out_dev: (C,out_H,out_W) like the reference, or (out_H,out_W,C) when out_hwc != 0, with
 * out_W = round(out_img_W/scale), out_H = round(out_img_H/scale) (Python round, half to even: query them with
 * srf_sphere_feature_dims).  Sphere cells hit by several pixels keep the LAST pixel in index order (what the reference's
 * index_put_ does on one CPU thread; on CUDA torch leaves it undefined).  workspace: out_W*out_H ints. */
void srf_sphere_feature_dims(int out_img_W, int out_img_H, int scale, int* out_W, int* out_H);
int srf_sphere_feature(const float* x_chw_dev, int C, int h, int w, const float* pix_dev, const long long* pix_sphere_dev,
                       int n_pixels, int scale, int out_img_W, int out_img_H, float* out_dev, int out_hwc,
                       void* workspace_dev, size_t workspace_bytes, void* stream);

/* --- next row (producer side): the convolutional tail of the spherical decoder, channels-last ------------------------------------
 * `UpSampleBN` / `BasicBlock` of scenerf/models/unet2d_sphere.py:9-57 as applied by `DecoderSphere.forward` (:167-206), whose five
 * outputs are the x_rgb pyramid.  All maps are [H][W][C] float32 with a channel stride `ld` that is a multiple of 4 (padding
 * channels hold zeros); BatchNorm is applied in eval mode, folded by the caller into per-channel scale / shift.
 *   srf_upsample_concat_hwc : F.interpolate(x, size=(H,W), bilinear, align_corners=True) of the coarser map x (h,w,Cx) concatenated
 *                             in front of skip (H,W,Cs) -> out (H,W,ld_out), channels [Cx+Cs, ld_out) zeroed      (unet2d_sphere.py:47-56)
 *   srf_conv3x3_hwc         : y = LeakyReLU_slope( conv3x3(in; dilation = padding = dil) * scale + shift (+ residual) ); slope 1 = none.
 *                             w9_dev: weights repacked [9][Cout][ld_in] (tap = ky*3 + kx; Conv2d.weight[co][ci][ky][kx]), zero for
 *                             padded ci.  Writes out32_dev (H,W,ld32) float32 and/or out16_dev (H,W,ld16) IEEE half -- with
 *                             ld = Cout these ARE the buffers srf_pyramid.hwc[] points to (no CHW->HWC pass).  wgmma tf32
 *                             implicit GEMM, operands read as fp32 with a 10-bit mantissa (cuDNN's default allow_tf32 regime).  The
 *                             tensor core truncates; feed it tensors already rounded to the nearest tf32 value (w9 rounded by the
 *                             caller; round_out != 0 stores out32 rounded because it feeds another convolution; the concat kernel
 *                             always rounds) and the truncation is exact -- 6.7x less error through the 35 chained convolutions. */
int srf_upsample_concat_hwc(const float* x_dev, int h, int w, int Cx, int ld_x, const float* skip_dev, int Cs, int ld_skip, int H, int W,
                            float* out_dev, int ld_out, void* stream);
int srf_conv3x3_hwc(const float* in_dev, int H, int W, int ld_in, const float* w9_dev, int Cout, int dil, const float* scale_dev,
                    const float* shift_dev, const float* residual_dev, int ld_res, float slope, int round_out, float* out32_dev, int ld32,
                    void* out16_dev, int ld16, void* stream);

/* Diagnostic: one GEMM of the training path, C[M x N] = epilogue(A[M x K] * B[N x K]^T) with float32 device operands.
 * use_tf32 != 0 runs the wgmma tf32 kernel (csrc/gemm_tf32.cu), 0 the float32 SIMT kernel (csrc/gemm.cu).
 * bias (N) / mask (M x N, keeps values where mask > 0) / residual (M x N) may be NULL; splitk_ws enables split-K. */
int srf_debug_gemm(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K, const float* bias,
                   const float* mask, int ldm, const float* residual, int ldr, int accumulate, float* splitk_ws,
                   size_t splitk_ws_floats, int use_tf32, void* stream);

/* Diagnostic (not part of the reference-facing surface): run the tensor-core point MLP of srf_predict but stop each
 * 128-point tile after layer `layer` of the tile program (mlp_tc.cu: 1 lin_in+lin_z0, 2 fc0_0, 4 fc1_0+lin_z1,
 * 5 fc0_1, 7 fc1_1+lin_z2, 8 fc0_2, 9 fc1_2, 10 lin_out) and write the raw fp32 accumulator rows to
 * acc_out_dev (ceil(n/128)*128, 512).  With cfg->precision == SRF_PREC_FP32_TC a tile holds 64 points: rows
 * 128t..128t+63 are the high-part products of points 64t..64t+63, rows 128t+64..128t+127 their low-part products,
 * both in units of the weight scale 2^s (acc_out_dev has ceil(n/64)*128 rows). */
int srf_debug_tc_layer(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w,
                       const float* cam_pts_dev, const float* viewdir_dev, int n_cols, int n_per, int layer,
                       float* acc_out_dev, void* workspace_dev, size_t workspace_bytes, void* stream);

/* Device-side timing of the point-MLP passes of the calls that follow on this thread (CUDA events recorded on the
 * call's stream around the mlp_gaussian pass and the main mlp pass).  srf_last_mlp_ms waits for the end events of
 * the most recent call and returns the elapsed milliseconds (-1 if that pass did not run). */
void srf_set_profiling(int on);
int srf_last_mlp_ms(float* gauss_ms, float* main_ms);

/* Diagnostic: non-zero once the mbarrier watchdog of a TMA-fed tensor-core kernel fired (readable even after the
 * resulting device trap): 0x40000000 | warp << 24 | (barrier smem offset & 0xFFFFF) << 4 | kernel << 1 | parity, where
 * kernel is 0 for the point MLP (point_mlp_tc_kernel), 1 for the tf32 GEMM (gemm_tf32_nt_kernel) and 2 for the decoder's
 * convolution (conv3x3_tf32_kernel). */
int srf_debug_watchdog_flag(void);

/* Number of kernels the last srf_render_rays / srf_predict call on this thread launched (bench "gpu_launches"). */
int srf_last_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* SCENERF_B200_H */
