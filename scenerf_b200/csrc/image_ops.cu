// Image-side glue of the novel-view sweep ("next" row 8f-4): the reference renders a stride-`scale` pixel grid in
// x-major ray order, reshapes to (gw, gh), transposes and bilinearly upsamples to the full image
// (scripts/reconstruction/generate_novel_depths.py:103-147), writes depth .npy + colour .png, and depth2tsdf.py:95-101
// reads them back.  Here the x-major render buffers are resampled straight into the (H,W) / (H,W,3) images that
// TSDF integration consumes, including (optionally) the 8-bit quantisation of the PNG round trip.
// HBM-bound elementwise work: 4 taps read (L2-resident, the source is <= 1/scale^2 of the output) + 16 B written per pixel.
#include "kernels.cuh"

namespace srf {

// torch.nn.functional.interpolate(mode="bilinear", align_corners=False): ATen area_pixel_compute_source_index
// (UpSample.h) -> src = scale*(dst+0.5)-0.5 clamped at 0, scale = in/out in float; lambda1 = src - floor, lambda0 = 1-lambda1;
// value = wy0*(wx0*v00 + wx1*v01) + wy1*(wx0*v10 + wx1*v11).
struct Tap { int i0, i1; float w0, w1; };
// FMA: ATen's CPU kernel as compiled (src = fma(scale, dst+0.5, -0.5)); otherwise separately rounded operations
template <bool FMA = false>
__device__ __forceinline__ Tap source_tap(int dst, int in_size, int out_size) {
  const float scale = __fdiv_rn((float)in_size, (float)out_size);
  float src = FMA ? __fmaf_rn(scale, __fadd_rn((float)dst, 0.5f), -0.5f) : __fsub_rn(__fmul_rn(scale, __fadd_rn((float)dst, 0.5f)), 0.5f);
  if (src < 0.f) src = 0.f;
  Tap t;
  t.i0 = min((int)src, in_size - 1);
  t.i1 = t.i0 + (t.i0 < in_size - 1 ? 1 : 0);
  t.w1 = fminf(fmaxf(__fsub_rn(src, (float)t.i0), 0.f), 1.f);
  t.w0 = __fsub_rn(1.f, t.w1);
  return t;
}
__device__ __forceinline__ float blend(float v00, float v01, float v10, float v11, const Tap& tx, const Tap& ty) {
  const float r0 = __fadd_rn(__fmul_rn(v00, tx.w0), __fmul_rn(v01, tx.w1));
  const float r1 = __fadd_rn(__fmul_rn(v10, tx.w0), __fmul_rn(v11, tx.w1));
  return __fadd_rn(__fmul_rn(r0, ty.w0), __fmul_rn(r1, ty.w1));
}

// depth_xm (gw*gh), color_xm (gw*gh,3): ray r = ix*gh + iy (x-major grid).  Outputs row-major (H,W) and (H,W,3).
// color_mode: 0 raw, 1 clamp to [0,1], 2 PNG round trip ((u8(c*255)/255)*255, a float image in [0,255] as depth2tsdf.py:98 builds)
__global__ void upsample_render_kernel(const float* __restrict__ depth_xm, const float* __restrict__ color_xm, int gw, int gh,
                                       int H, int W, float* __restrict__ depth_out, float* __restrict__ color_out, int color_mode) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W) return;
  const int y = i / W, x = i % W;
  float d, c[3];
  if (gw == W && gh == H) {      // scale == 1: plain transpose (generate_novel_depths.py:136-138)
    const int r = x * gh + y;
    if (depth_xm) d = depth_xm[r];
    if (color_xm) { c[0] = color_xm[3 * r]; c[1] = color_xm[3 * r + 1]; c[2] = color_xm[3 * r + 2]; }
  } else {
    const Tap tx = source_tap(x, gw, W), ty = source_tap(y, gh, H);
    const int r00 = tx.i0 * gh + ty.i0, r01 = tx.i1 * gh + ty.i0, r10 = tx.i0 * gh + ty.i1, r11 = tx.i1 * gh + ty.i1;
    if (depth_xm) d = blend(depth_xm[r00], depth_xm[r01], depth_xm[r10], depth_xm[r11], tx, ty);
    if (color_xm) {
#pragma unroll
      for (int k = 0; k < 3; ++k)
        c[k] = blend(color_xm[3 * r00 + k], color_xm[3 * r01 + k], color_xm[3 * r10 + k], color_xm[3 * r11 + k], tx, ty);
    }
  }
  if (depth_xm && depth_out) depth_out[i] = d;
  if (color_xm && color_out) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      float v = c[k];
      if (color_mode >= 1) v = fminf(fmaxf(v, 0.f), 1.f);
      if (color_mode == 2) {
        const float q = (float)(unsigned char)(int)__fmul_rn(v, 255.f);    // matplotlib to_rgba(bytes=True): (x*255).astype(uint8)
        v = __fmul_rn(__fdiv_rn(q, 255.f), 255.f);                          // depth2tsdf.py:23,98: float32(u8)/255.0*255.0
      }
      color_out[3 * (size_t)i + k] = v;
    }
  }
}

// Merge volume B (later observations) into A (earlier ones) with the fold rule of fusion.py:212-216: keep A where
// |A| < |B|, else take B's distance and colour; weights add.  Contiguous pose ranges merged in order reproduce the
// sequential integration: distances and weights bit for bit; the colour can differ only where two observations from
// different ranges have distances that round to the same float32 (the sequential fold compares the stored float32
// with the incoming float64, the merge sees two float32) -- both answers are an observation of minimal |distance|.
__global__ void tsdf_merge_kernel(float* __restrict__ tsdf_a, float* __restrict__ weight_a, float* __restrict__ color_a,
                                  const float* __restrict__ tsdf_b, const float* __restrict__ weight_b,
                                  const float* __restrict__ color_b, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float wb = weight_b[i];
  if (wb == 0.f) return;                     // B never observed this voxel
  const float a = tsdf_a[i], b = tsdf_b[i];
  weight_a[i] = weight_a[i] + wb;
  if (!(fabsf(a) < fabsf(b))) { tsdf_a[i] = b; color_a[i] = color_b[i]; }
}

// One float32 image resized with F.interpolate(size=(out_h, out_w), mode="bilinear", align_corners=False), as
// generate_sc_gt_bf.py:296-297 resizes each source depth -- a CPU tensor there, so the arithmetic is that of ATen's CPU
// kernel as built: the source index and each 2-tap lerp contract into one FMA (a*wa + b*wb -> fma(a, wa, b*wb)), outer
// (y) lerp of the two inner (x) lerps.  The tap indices and weights are those of source_tap, which is the size= form:
// ATen takes scale = float(in)/out.  The scale_factor= form (recompute_scale_factor unset) takes scale = 1/scale_factor
// instead, which differs in the last bits whenever in/out is not what 1/scale_factor rounds to.
__device__ __forceinline__ float lerp_fma(float a, float wa, float b, float wb) { return __fmaf_rn(a, wa, __fmul_rn(b, wb)); }

__global__ void resize_bilinear_kernel(const float* __restrict__ src, int in_h, int in_w, float* __restrict__ dst, int out_h,
                                       int out_w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= out_h * out_w) return;
  const int y = i / out_w, x = i % out_w;
  const Tap tx = source_tap<true>(x, in_w, out_w), ty = source_tap<true>(y, in_h, out_h);
  const float* r0 = src + (size_t)ty.i0 * in_w;
  const float* r1 = src + (size_t)ty.i1 * in_w;
  dst[i] = lerp_fma(lerp_fma(r0[tx.i0], tx.w0, r0[tx.i1], tx.w1), ty.w0, lerp_fma(r1[tx.i0], tx.w0, r1[tx.i1], tx.w1), ty.w1);
}

void launch_resize_bilinear(const float* src, int in_h, int in_w, float* dst, int out_h, int out_w, cudaStream_t st) {
  const int n = out_h * out_w;
  resize_bilinear_kernel<<<(n + 255) / 256, 256, 0, st>>>(src, in_h, in_w, dst, out_h, out_w);
}

void launch_upsample_render(const float* depth_xm, const float* color_xm, int gw, int gh, int H, int W, float* depth_out,
                            float* color_out, int color_mode, cudaStream_t st) {
  const int n = H * W;
  upsample_render_kernel<<<(n + 255) / 256, 256, 0, st>>>(depth_xm, color_xm, gw, gh, H, W, depth_out, color_out, color_mode);
}
void launch_tsdf_merge(float* tsdf_a, float* weight_a, float* color_a, const float* tsdf_b, const float* weight_b,
                       const float* color_b, long long n, cudaStream_t st) {
  tsdf_merge_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(tsdf_a, weight_a, color_a, tsdf_b, weight_b, color_b, n);
}

}  // namespace srf
