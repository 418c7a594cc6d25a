// 3x3 (dilated) convolution of the spherical decoder on tensor cores, channels-last in and out -- the producer tail of the feature
// pyramid (SURVEY 8f-3).  Reference: scenerf/models/unet2d_sphere.py:9-57 (`BasicBlock`, `UpSampleBN`: Conv2d 3x3 with
// padding = dilation, BatchNorm2d in eval mode, LeakyReLU(0.01), residual add), applied five times by `DecoderSphere.forward`
// (:167-206); its outputs "1_1".."1_16" ARE the x_rgb pyramid the ray renderer gathers from (scenerf.py:522-525).
//
// Implicit GEMM, no im2col buffer:  out[p, co] = sum_{tap} sum_{ci} in[p + d*(tap - 1), ci] * W[tap][co][ci].
//   M tile = 128 consecutive pixels of one image row, N tile = 128 output channels, K loop = 9 taps x Cin/32 blocks.
//   A tiles come from a 3-D tensor map over the [H][W][C] input: box {32 ch, 128 px, 1 row} at (c0, x0 + dx, y + dy) --
//   TMA's out-of-bounds zero fill IS the convolution's zero padding (negative / too large coordinates), and the box lands
//   in shared memory as the same 128-row x 128-byte swizzled tile a plain GEMM would stage.
//   B tiles: 2-D map over the weights repacked [tap][co][ci] (ci padded to a multiple of 4), box {32, 128} at (c0, tap*Cout + n0).
//   wgmma .tf32 (fp32 operands read in place, 10-bit mantissa -- the regime of the reference's own cuDNN default
//   `allow_tf32=True` on Ampere-class GPUs) through the tf32 tile mainloop of tma.cuh: two consumer warpgroups that each
//   accumulate 64 pixels x 128 channels in registers.
//   The tensor core TRUNCATES the 13 low mantissa bits of what it reads; through the decoder's 35 chained convolutions that
//   bias compounds (1.3 % relative L2 on the finest map of the test network).  So every tensor that feeds a convolution is
//   stored already ROUNDED TO NEAREST tf32 (weights at pack time, the concat buffer, intermediate activations: `round_out`),
//   which makes the truncation exact: 0.2 % relative L2, 6.7x better, at no cost.  The pyramid maps themselves stay unrounded.
//   Epilogue (from the accumulator registers): y = acc*scale[co] + shift[co] (conv bias + eval-mode BatchNorm folded on the host),
//   (+ residual[p, co]), LeakyReLU, store fp32 [H][W][C] and/or fp16 [H][W][C] -- i.e. straight into the packed pyramid
//   layout of srf_pyramid (no CHW -> HWC pass).
// Roofline: tensor (tf32 = half the f16 rate); 2*9*Cin*Cout flops per pixel.
#include <cuda_fp16.h>
#include "kernels.cuh"
#include "tma.cuh"

namespace srf {
namespace conv {

using namespace tf32;

struct ConvArgs {
  int H, W, Cin, Cout;            // Cin as stored (channel stride of the input, multiple of 4; padded channels hold zeros)
  int dil;                        // dilation = padding
  const float* scale;             // (Cout) folded BatchNorm scale, or all ones
  const float* shift;             // (Cout) folded conv bias / BatchNorm shift
  const float* residual;          // [H][W][ld_res] or null
  int ld_res;
  float slope;                    // LeakyReLU negative slope; 1.0 = no activation
  int round_out;                  // store out32 rounded to the nearest tf32 (it feeds another convolution)
  float* out32; int ld32;         // [H][W][ld32] or null
  __half* out16; int ld16;        // [H][W][ld16] or null
  int* err;
};

// nearest value with a 10-bit mantissa (ties away from zero; finite inputs)
__device__ __forceinline__ float round_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

__global__ void __launch_bounds__(kThreads, 1)
conv3x3_tf32_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ ConvArgs a) {
  const int xt = (a.W + kBM - 1) / kBM;
  const int y = blockIdx.y / xt, x0 = (blockIdx.y % xt) * kBM;
  const int n0 = blockIdx.x * kBN;
  const int kb = (a.Cin + kBK - 1) / kBK;                                 // channel blocks per tap
  int j = 0;                                                              // the producer's k-block cursor
  float acc[64];
  if (!mainloop<kWatchConvTf32>(&tmA, &tmB, 9 * kb, a.err, acc, [&](uint32_t sA, uint32_t sB, uint32_t bar) {
        const int tap = j / kb, cb = j - tap * kb;
        const int dy = (tap / 3 - 1) * a.dil, dx = (tap % 3 - 1) * a.dil;
        tma_load_3d(sA, &tmA, cb * kBK, x0 + dx, y + dy, bar);      // OOB -> zeros = the conv padding
        tma_load_2d(sB, &tmB, cb * kBK, tap * a.Cout + n0, bar);
        ++j;
      }))
    return;
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int w = t >> 5, l = t & 31;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int px = x0 + (wg - 1) * 64 + 16 * w + (l >> 2) + 8 * half;
    if (px >= a.W) continue;
    const size_t pix = (size_t)y * a.W + px;
#pragma unroll
    for (int c8 = 0; c8 < kBN / 8; ++c8) {
      const int co = n0 + 8 * c8 + 2 * (l & 3);
      if (co >= a.Cout) break;                              // Cout % 4 == 0: co + 1 < Cout as well
      const float2 sc = __ldg(reinterpret_cast<const float2*>(a.scale + co)), sh = __ldg(reinterpret_cast<const float2*>(a.shift + co));
      float2 o = make_float2(fmaf(acc[4 * c8 + 2 * half], sc.x, sh.x), fmaf(acc[4 * c8 + 2 * half + 1], sc.y, sh.y));
      if (a.residual) {
        const float2 t2 = *reinterpret_cast<const float2*>(a.residual + pix * a.ld_res + co);
        o.x += t2.x; o.y += t2.y;
      }
      o.x = o.x > 0.f ? o.x : o.x * a.slope; o.y = o.y > 0.f ? o.y : o.y * a.slope;
      if (a.out16) *reinterpret_cast<__half2*>(a.out16 + pix * a.ld16 + co) = __floats2half2_rn(o.x, o.y);
      if (a.out32) {
        if (a.round_out) { o.x = round_tf32(o.x); o.y = round_tf32(o.y); }
        *reinterpret_cast<float2*>(a.out32 + pix * a.ld32 + co) = o;
      }
    }
  }
}

// UpSampleBN front end (unet2d_sphere.py:47-56): F.interpolate(x, size=(H, W), bilinear, align_corners=True) of the coarser
// map, concatenated in front of the skip map: out[y][x] = [ up(x)(Cx) | skip(Cs) | zero padding to ld ], all channels-last.
__global__ void upsample_concat_kernel(const float* __restrict__ x, int h, int w, int Cx, int ldx, const float* __restrict__ skip, int Cs,
                                       int lds, int H, int W, float* __restrict__ out, int ld) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)H * W * ld;
  if (idx >= total) return;
  const int c = (int)(idx % ld);
  const size_t pix = idx / ld;
  const int ox = (int)(pix % W), oy = (int)(pix / W);
  float v = 0.f;
  if (c < Cx) {
    // ATen area_pixel_compute_source_index, align_corners=True: src = dst * (in - 1) / (out - 1)  (scale computed in float)
    const float sy = (H > 1) ? (float)(h - 1) / (float)(H - 1) : 0.f, sx = (W > 1) ? (float)(w - 1) / (float)(W - 1) : 0.f;
    const float fy = __fmul_rn(sy, (float)oy), fx = __fmul_rn(sx, (float)ox);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = y0 + (y0 < h - 1 ? 1 : 0), x1 = x0 + (x0 < w - 1 ? 1 : 0);
    const float ly = __fsub_rn(fy, (float)y0), lx = __fsub_rn(fx, (float)x0);
    const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
    const float v00 = x[((size_t)y0 * w + x0) * ldx + c], v01 = x[((size_t)y0 * w + x1) * ldx + c];
    const float v10 = x[((size_t)y1 * w + x0) * ldx + c], v11 = x[((size_t)y1 * w + x1) * ldx + c];
    // ATen upsample_bilinear2d: h0lambda * (w0lambda * v00 + w1lambda * v01) + h1lambda * (w0lambda * v10 + w1lambda * v11)
    v = __fadd_rn(__fmul_rn(hy, __fadd_rn(__fmul_rn(hx, v00), __fmul_rn(lx, v01))), __fmul_rn(ly, __fadd_rn(__fmul_rn(hx, v10), __fmul_rn(lx, v11))));
  } else if (c < Cx + Cs) {
    v = skip[pix * lds + (c - Cx)];
  }
  out[idx] = round_tf32(v);            // this buffer only feeds the level's first convolution
}

}  // namespace conv

// in: [H][W][Cin] float32 (Cin = channel stride, multiple of 4, 16-byte aligned); w9: [9][Cout][Cin] float32 (tap = ky*3 + kx).
// Returns 0, -1 (shape / alignment not expressible as tensor maps, or more than 65535 row tiles H * ceil(W/128)), -2 (driver
// entry point missing).
int launch_conv3x3_tf32(const float* in, int H, int W, int Cin, const float* w9, int Cout, int dil, const float* scale, const float* shift,
                        const float* residual, int ld_res, float slope, int round_out, float* out32, int ld32, void* out16, int ld16,
                        cudaStream_t st) {
  if (H < 1 || W < 1 || Cin < 4 || (Cin % 4) || Cout < 4 || (Cout % 4) || dil < 1 || !al16(in) || !al16(w9) || !al16(scale) || !al16(shift)) return -1;
  if ((long long)H * ((W + tf32::kBM - 1) / tf32::kBM) > 65535) return -1;     // one row tile per gridDim.y index (limit 65535)
  if ((out32 && (!al16(out32) || ld32 % 4)) || (out16 && ((reinterpret_cast<uintptr_t>(out16) & 7) || ld16 % 4)) || (residual && (!al16(residual) || ld_res % 4)))
    return -1;
  CUtensorMap tmA, tmB;
  const cuuint64_t dims_a[3] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H}, strides_a[2] = {(cuuint64_t)Cin * 4, (cuuint64_t)W * Cin * 4};
  const cuuint64_t dims_b[2] = {(cuuint64_t)Cin, (cuuint64_t)9 * Cout}, strides_b[1] = {(cuuint64_t)Cin * 4};
  const cuuint32_t box_a[3] = {(cuuint32_t)tf32::kBK, (cuuint32_t)tf32::kBM, 1}, box_b[2] = {(cuuint32_t)tf32::kBK, (cuuint32_t)tf32::kBN};
  int rc = encode_tensor_map_f32(&tmA, in, 3, dims_a, strides_a, box_a);
  if (rc == 0) rc = encode_tensor_map_f32(&tmB, w9, 2, dims_b, strides_b, box_b);
  if (rc) return rc;
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(conv::conv3x3_tf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tf32::kSmemBytes); attr = true; }
  conv::ConvArgs a;
  a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.dil = dil; a.scale = scale; a.shift = shift; a.residual = residual; a.ld_res = ld_res;
  a.slope = slope; a.round_out = round_out; a.out32 = out32; a.ld32 = ld32; a.out16 = reinterpret_cast<__half*>(out16); a.ld16 = ld16; a.err = watchdog_device_flag();
  const dim3 grid((Cout + tf32::kBN - 1) / tf32::kBN, (unsigned)(H * ((W + tf32::kBM - 1) / tf32::kBM)));
  conv::conv3x3_tf32_kernel<<<grid, tf32::kThreads, tf32::kSmemBytes, st>>>(tmA, tmB, a);
  return 0;
}

void launch_upsample_concat(const float* x, int h, int w, int Cx, int ldx, const float* skip, int Cs, int lds, int H, int W, float* out, int ld,
                            cudaStream_t st) {
  const size_t total = (size_t)H * W * ld;
  conv::upsample_concat_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, h, w, Cx, ldx, skip, Cs, lds, H, W, out, ld);
}

}  // namespace srf
