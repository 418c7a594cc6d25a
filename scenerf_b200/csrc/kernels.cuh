// Host-side launchers of the scenerf_b200 kernels (definitions in the .cu files of this directory).
#pragma once
#include "common.cuh"

namespace srf {

// ray_kernels.cu
void launch_ray_setup(const DevParams& p, const float* pixels, int R, float* unit, float* viewdir, float* gauss_pts,
                      cudaStream_t st);
void launch_sample_sort(const DevParams& p, int R, const float* unit, const float* gauss_raw, const float* noise_u,
                        const float* noise_n, float* means, float* stds, float* t_sorted, float* depth_volume,
                        float* pts, cudaStream_t st);
void launch_composite_som(const DevParams& p, int R, const float* raw, const float* t_sorted,
                          const float* depth_volume, const float* means, const float* stds, const srf_outputs& out,
                          cudaStream_t st);

// pack.cu
void launch_chw_to_hwc(const float* src, void* dst, int C, int H, int W, bool fp16, cudaStream_t st);

// tsdf.cu : TSDF integration of rendered depth sweeps (reference: data/utils/fusion.py:219-324, CPU path)
void launch_tsdf_reset(float* tsdf, float* weight, float* color, long long n, cudaStream_t st);
void launch_tsdf_integrate(const int* dims, const float* origin, double voxel_size, const double* inv_pose, const float* intr,
                           int im_h, int im_w, double trunc, float obs_weight, int color_is_u8, float* tsdf, float* weight,
                           float* color, const float* depth, const void* color_im, cudaStream_t st);

// mesh.cu : marching cubes over a TSDF volume (reference: data/utils/fusion.py:333-379)
size_t mesh_workspace_bytes(const int* dims);
void launch_mesh_count(const float* tsdf, const unsigned char* mask, const int* dims, void* ws, cudaStream_t st);
cudaError_t mesh_read_totals(const int* dims, const void* ws, int* n_verts, int* n_tris, cudaStream_t st);
void launch_mesh_emit(const float* tsdf, const float* color, const unsigned char* mask, const int* dims, const float* origin,
                      double voxel_size, const void* ws, float* verts, float* normals, unsigned char* colors, int* faces,
                      cudaStream_t st);

// image_ops.cu : resampling of x-major renders into images, TSDF volume merge
void launch_upsample_render(const float* depth_xm, const float* color_xm, int gw, int gh, int H, int W, float* depth_out,
                            float* color_out, int color_mode, cudaStream_t st);
void launch_tsdf_merge(float* tsdf_a, float* weight_a, float* color_a, const float* tsdf_b, const float* weight_b,
                       const float* color_b, long long n, cudaStream_t st);

// sphere_feature.cu : image-plane feature map -> sphere grid (unet2d_sphere.py:138-166)
void launch_sphere_feature(const float* x, int C, int h, int w, const float* pix, const long long* pix_sphere, int n, int scale,
                           int oW, int oH, int* winner, float* out, int out_hwc, cudaStream_t st);

inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Mapped host flag of the mbarrier watchdog of the sm_90a kernels (tma.cuh), readable even after the resulting device
// trap: 0, or 0x40000000 | warp << 24 | (barrier smem offset & 0xFFFFF) << 4 | kernel << 1 | parity, where kernel is
// 0 for point_mlp_tc_kernel, 1 for gemm_tf32_nt_kernel, 2 for conv3x3_tf32_kernel and 3 for the split (3xTF32)
// gemm_tf32_nt_kernel.
int watchdog_flag();
int* watchdog_device_flag();   // the device address the kernels write (allocated on first use; null if that failed)

// gemm.cu : float32 SIMT GEMM (see the file header for operand layouts and the epilogue)
struct GemmArgs {
  const float* A = nullptr; int lda = 0; bool at = false; bool relu_a = false;
  const float* B = nullptr; int ldb = 0; bool bt = false; bool relu_b = false;
  float* C = nullptr; int ldc = 0; int M = 0, N = 0, K = 0;
  const float* bias = nullptr; const float* mask = nullptr; int ldm = 0; const float* R = nullptr; int ldr = 0; int accumulate = 0;
  const int* skip_if_zero = nullptr;   // device flag: when *flag == 0 the launch does nothing (an all-zero K-segment of the latent)
  // tf32 kernel only: the latent axis (K when seg_mode == 1, N when seg_mode == 2) is the concatenation of the 5 pyramid
  // scales [seg_off[s], seg_off[s+1]); k-blocks / column tiles that lie entirely in scales with seg_flags[s] == 0 are
  // skipped on the device (their inputs are exact zeros / their outputs are never read).  One launch instead of five.
  const int* seg_flags = nullptr; int seg_mode = 0; int seg_off[6] = {0, 0, 0, 0, 0, 0};
  float* splitk_ws = nullptr; size_t splitk_ws_floats = 0;   // optional scratch: enables deterministic split-K for long-K, few-tile shapes
  float* relu_out = nullptr; int ld_relu = 0;   // tf32 kernel only: the epilogue also stores max(result, 0) here (the next GEMM's A operand)
};
int launch_gemm(const GemmArgs& g, cudaStream_t st);
// The seg_* fields as the tf32 kernel and the split-K reduce read them: mode 0 none, 1 dead k-blocks, 2 dead column tiles
// of kSegTileN (the tf32 kernel's N tile).
constexpr int kSegTileN = 128;
struct SegInfo { const int* flags; int mode; int off[6]; };
// true when [lo, hi) of the latent axis touches only scales whose flag is 0
__device__ __forceinline__ bool seg_dead(const SegInfo& sg, int lo, int hi) {
#pragma unroll
  for (int s = 0; s < 5; ++s)
    if (lo < sg.off[s + 1] && hi > sg.off[s] && sg.flags[s] != 0) return false;
  return true;
}
// Deterministic split-K of the weight-gradient shapes (few output tiles, long K): slice z of K (k_per long, a multiple of
// the kernel's k granularity) goes to g.splitk_ws + z*M*N, then launch_splitk_reduce adds the slices in z order into C.
// Only for plain products (no bias / mask / residual) of fewer than 96 tiles with K >= 1024: about two waves over the
// SMs, at most `cap` slices, as many as fit g.splitk_ws_floats.  splits == 1: no split (k_per = K).
struct SplitK { int splits, k_per; };
SplitK plan_splitk(const GemmArgs& g, int tiles, int k_gran, int cap);
void launch_splitk_reduce(const GemmArgs& g, int splits, const SegInfo& sg, cudaStream_t st);
// SM count of the current device (cached; 132 on an H100 SXM): sizes waves, split-K factors and point chunks
int device_sm_count();
// per-thread count of kernels launched by the float32 / tf32 MLP paths (gemm.cu, gemm_tf32.cu, mlp_simt.cu);
// the run_* entry points report the difference as their launch count (srf_last_launch_count)
int& launch_counter();    // 0, or -1 for an operand-layout combination that is not instantiated

// gemm_tf32.cu : the same contract on tensor cores (wgmma .tf32, float32 operands read in place); NT layout only
// (at=false, bt=true, no operand ReLU).  split: the 3xTF32 kernel (hi.hi + hi.lo + lo.hi, float32-grade products).
// Returns 0, or -1 when the shape cannot be expressed as TMA tensor maps.
int launch_gemm_tf32(const GemmArgs& g, cudaStream_t st, bool split = false);

// mlp_simt.cu : float32 point MLP (gather + positional encoding + ResnetFC) and its backward, n points in chunks.
//   pts (n,3) infer-frame points; viewdir (n/n_per,3); raw_out (n,d_out).  The run_* functions return the number of
//   kernel launches, or -1 for a workspace that is too small or an engine the call cannot use.
// GEMM engine of the chain: SIMT float32 FMAs (gemm.cu), or for its NT products wgmma tf32 (gemm_tf32.cu) or the split
// 3xTF32 wgmma kernel of float32-grade accuracy (fp32tc); the two tensor-core engines are training only and arrange the
// operands the same way.
enum class MatmulEngine { simt, tf32, fp32tc };
inline bool tensor_cores(MatmulEngine e) { return e != MatmulEngine::simt; }
// workspace of run_point_mlp_simt; save_activations: also enough for a training forward (tf32: its ReLU'd operands)
size_t simt_workspace_bytes(int d_latent, int n_points, bool save_activations);
size_t mlp_saved_bytes(int d_latent, int n_points);            // activation store of one pass (SRF_FLAG_SAVE_ACTIVATIONS)
size_t mlp_backward_workspace_bytes(int d_latent, int n_points);
// saved == NULL: inference (SIMT engine only).  saved = a store of mlp_saved_bytes: the training forward, which keeps the
// activations there for run_point_mlp_backward_simt; raw outputs are bit-identical to inference on the SIMT engine.
int run_point_mlp_simt(const DevParams& p, const srf_mlp_weights& w, const float* pts, const float* viewdir, int n, int n_per,
                       float* raw_out, int32_t* dbg_sphere, void* saved, MatmulEngine e, void* workspace, size_t ws_bytes,
                       cudaStream_t st);
// grads: same layout as the weights, pyramid grads CHW; both accumulated into.  saved_base: the store the training
// forward wrote for the same points, or NULL: the forward is then recomputed chunk by chunk (SIMT engine only).
int run_point_mlp_backward_simt(const DevParams& p, const srf_mlp_weights& w, const srf_mlp_weights& gw, float* const* grad_pyr_chw,
                                const float* pts, const float* viewdir, int n, int n_per, const float* g_raw, const void* saved_base,
                                MatmulEngine e, void* workspace, size_t ws_bytes, cudaStream_t st);

// backward.cu : per-ray backward of the compositing (reference: torch.autograd through scenerf.py:392-748)
void launch_ray_backward(const DevParams& p, int R, const float* raw, const float* t_sorted, const float* unit,
                         const float* gauss_raw, const float* noise_n, const srf_outputs& fwd, const srf_outputs& cot,
                         float* graw_main, float* graw_gauss, cudaStream_t st);

// mlp_tc.cu : wgmma tensor-core point MLP.
//   split != 0: the fp32-grade layout (hi + lo fp16 images of W 2^s, see mlp_tc.cu) read through w.tc_split_packed
size_t tc_weights_bytes(int d_out, int d_latent, int split);
int pack_weights_tc(const srf_mlp_weights& w, void* dst, size_t bytes, int split, cudaStream_t st);
constexpr int kTcFlagPreproj = 1 << 29; // internal bit: this pass may use DevParams::preproj (the table of ITS network)
constexpr int kTcFlagSplit = 1 << 30;   // internal bit of the `flags` argument of run_point_mlp_tc*: split (fp32-grade) mode
size_t tc_workspace_bytes(int d_latent, int n_points);
int run_point_mlp_tc(const DevParams& p, const srf_mlp_weights& w, const float* pts, const float* viewdir, int n,
                     int n_per, float* raw_out, int32_t* dbg_sphere, int flags, void* workspace, size_t ws_bytes,
                     cudaStream_t st);

// conv_tf32.cu : the spherical decoder's 3x3 (dilated) convolutions as a wgmma .tf32 implicit GEMM on channels-last maps
//   (unet2d_sphere.py:9-57) + the UpSampleBN front end (bilinear align_corners=True upsample of the coarser map, concat with the skip map)
int launch_conv3x3_tf32(const float* in, int H, int W, int Cin, const float* w9, int Cout, int dil, const float* scale, const float* shift,
                        const float* residual, int ld_res, float slope, int round_out, float* out32, int ld32, void* out16, int ld16,
                        cudaStream_t st);
void launch_upsample_concat(const float* x, int h, int w, int Cx, int ldx, const float* skip, int Cs, int lds, int H, int W, float* out, int ld,
                            cudaStream_t st);

// preproj.cu : pre-projected latent table  table[(sy,sx)][block][512] = lin_z[block].weight . z(sphere pixel)  (see file header)
size_t preproj_rows(int sphere_W, int sphere_H);
size_t preproj_table_bytes(int sphere_W, int sphere_H, int fp16);
size_t preproj_workspace_bytes(const int* H, const int* W);
int run_preproject(const DevParams& p, const srf_mlp_weights& w, int fp16, void* table, size_t table_bytes, void* workspace,
                   size_t ws_bytes, cudaStream_t st);

// metrics.cu : evaluation (occupancy confusion histograms, completion-target labels, depth errors)
size_t eval_hist_len(const int* dims, int n_classes, int per_z);
void launch_eval_confusion(const float* tsdf, const void* pred, int pred_dtype, const uint8_t* target, const uint8_t* mask,
                           const int* dims, int n_classes, int th_axis, const double* th, int per_z, unsigned long long* hist,
                           int* max_z, uint8_t* occ, cudaStream_t st);
void launch_eval_sc_label(const float* tsdf, long long n, float voxel_size, uint8_t* out, cudaStream_t st);
size_t depth_errors_workspace_bytes();
void launch_depth_errors(const float* gt, const float* pred, long long n, void* ws, double* bucket, int slot, double* frame,
                         cudaStream_t st);
// color_metrics.cu : novel-view colour metrics (eval_color.py): PSNR + SSIM of one (H,W,3) pair (two launches, float64
// partials in ws, frame = (psnr, ssim), bucket row slot of [psnr, ssim, lpips, n] += (psnr, ssim, -, 1)), and LPIPS-VGG.
size_t psnr_ssim_workspace_bytes(int H, int W);
void launch_psnr_ssim(const float* img, const float* gt, int H, int W, void* ws, double* bucket, int slot, double* frame, cudaStream_t st);
size_t lpips_workspace_bytes(int H, int W);
// w9[13]: [9][Cout][Cin] tf32-rounded weights (Cin 32 for conv1_1: RGB + zero channels), bias[13], lin[5] (64..512);
// shift/scale: 3 host floats each.  *out = the pair's LPIPS (float32).  Returns the launch count, or launch_conv3x3_tf32's
// error (-1 shape, -2 driver entry point missing).
int run_lpips_vgg(const float* img0, const float* img1, int H, int W, const float* const* w9, const float* const* bias,
                  const float* const* lin, const float* shift, const float* scale, void* workspace, float* out, cudaStream_t st);
// image_ops.cu : F.interpolate(size=(out_h,out_w), mode="bilinear", align_corners=False) of one (in_h,in_w) float32 image
void launch_resize_bilinear(const float* src, int in_h, int in_w, float* dst, int out_h, int out_w, cudaStream_t st);

// diagnostic: stop every tile after `debug_layer` (1,2,4,5,7,8,9,10 -- see the tile program in mlp_tc.cu) and dump the
// raw fp32 accumulator to debug_acc: (n_tiles*64, 512), point i at row i; split mode (ceil(n/32)*64, 512), point i at
// row 64 (i/32) + i%32 with all four partial products (rows 64 (i/32) + 32..63 untouched); only points i < n
int run_point_mlp_tc_debug(const DevParams& p, const srf_mlp_weights& w, const float* pts, const float* viewdir, int n,
                           int n_per, float* raw_out, int32_t* dbg_sphere, int flags, void* workspace, size_t ws_bytes,
                           int debug_layer, float* debug_acc, cudaStream_t st);

}  // namespace srf
