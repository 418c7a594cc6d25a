// Novel-view colour metrics on the device (DESIGN.md 6.8): the per-image numbers of scripts/evaluation/eval_color.py /
// eval_color_bf.py, which score a rendered colour image against the source frame.
//   psnr_ssim : skimage 0.18.1 peak_signal_noise_ratio(data_range=1) and structural_similarity(multichannel=True,
//               data_range=1) of one (H,W,3) float32 pair in one pass.  float64 arithmetic as skimage's; the squared
//               difference is formed in float32 as skimage forms it for float32 inputs.  Block partials in a fixed
//               order, so the results depend on the shape only and repeat bit for bit.
//   lpips     : lpips 0.1 LPIPS(net="vgg", version="0.1") -- scaling layer, the 13 conv3x3+ReLU of torchvision's
//               VGG16 features[0:30] on launch_conv3x3_tf32 (conv_tf32.cu, unchanged), 2x2 floor max-pools, and the
//               head (unit-normalise each tap over channels, squared difference, 1x1 lin, spatial mean, sum of 5).
#include "kernels.cuh"

namespace srf {

namespace {

// ---- PSNR / SSIM --------------------------------------------------------------------------------------------------
// 7x7 window (skimage win_size=7, uniform_filter).  skimage keeps only S[3:-3, 3:-3]: every window of that interior lies
// inside the image, so the filter's boundary mode (scipy 'reflect') never reaches a kept value and a tile loads only
// in-image pixels.
constexpr int kWin = 7, kPad = 3;
constexpr int kTW = 32, kTH = 8;                 // interior outputs per block
constexpr int kSsimThreads = kTW * kTH;          // one output per thread per channel
constexpr int kInW = kTW + 2 * kPad, kInH = kTH + 2 * kPad;
constexpr int kSsimSums = 4;                      // S sum of channels 0..2, float32 squared-difference sum

__device__ __forceinline__ void block_sum(double (*red)[kSsimThreads], double* v, int n, double* dst) {
  const int t = threadIdx.x;
#pragma unroll
  for (int k = 0; k < n; ++k) red[k][t] = v[k];
  __syncthreads();
  for (int w = kSsimThreads / 2; w > 0; w >>= 1) {
    if (t < w)
#pragma unroll
      for (int k = 0; k < n; ++k) red[k][t] += red[k][t + w];
    __syncthreads();
  }
  if (t < n) dst[t] = red[t][0];
}

__global__ void __launch_bounds__(kSsimThreads) psnr_ssim_partial_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                                         int H, int W, double* __restrict__ partial) {
  __shared__ float sa[3][kInH][kInW], sb[3][kInH][kInW];
  __shared__ double v[5][kTH][kInW];              // vertical 7-sums of x, y, x^2, y^2, xy
  __shared__ double red[kSsimSums][kSsimThreads];
  const int t = threadIdx.x;
  const int gx0 = blockIdx.x * kTW, gy0 = blockIdx.y * kTH;   // input origin; outputs start at (+3, +3)
  for (int i = t; i < kInH * kInW; i += kSsimThreads) {
    const int r = i / kInW, c = i % kInW, gy = gy0 + r, gx = gx0 + c;
    const bool in = gy < H && gx < W;
    const size_t o = ((size_t)gy * W + gx) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      sa[ch][r][c] = in ? a[o + ch] : 0.f;
      sb[ch][r][c] = in ? b[o + ch] : 0.f;
    }
  }
  __syncthreads();
  const int r = t / kTW, c = t % kTW;
  const bool valid = gy0 + kPad + r <= H - 1 - kPad && gx0 + kPad + c <= W - 1 - kPad;
  double acc[kSsimSums] = {0.0, 0.0, 0.0, 0.0};
  const double cov_norm = 49.0 / 48.0;            // NP / (NP - 1), use_sample_covariance
  const double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03; // (K1 * data_range) ** 2, (K2 * data_range) ** 2
  for (int ch = 0; ch < 3; ++ch) {
    for (int i = t; i < kTH * kInW; i += kSsimThreads) {
      const int rr = i / kInW, cc = i % kInW;
      double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int k = 0; k < kWin; ++k) {
        const double x = sa[ch][rr + k][cc], y = sb[ch][rr + k][cc];
        // products of two floats are exact in float64
        s[0] = __dadd_rn(s[0], x); s[1] = __dadd_rn(s[1], y);
        s[2] = __dadd_rn(s[2], __dmul_rn(x, x)); s[3] = __dadd_rn(s[3], __dmul_rn(y, y)); s[4] = __dadd_rn(s[4], __dmul_rn(x, y));
      }
#pragma unroll
      for (int q = 0; q < 5; ++q) v[q][rr][cc] = s[q];
    }
    __syncthreads();
    if (valid) {
      double u[5];
#pragma unroll
      for (int q = 0; q < 5; ++q) {
        double s = 0.0;
#pragma unroll
        for (int k = 0; k < kWin; ++k) s = __dadd_rn(s, v[q][r][c + k]);
        u[q] = __ddiv_rn(s, 49.0);
      }
      const double ux = u[0], uy = u[1];
      const double vx = __dmul_rn(cov_norm, __dsub_rn(u[2], __dmul_rn(ux, ux)));
      const double vy = __dmul_rn(cov_norm, __dsub_rn(u[3], __dmul_rn(uy, uy)));
      const double vxy = __dmul_rn(cov_norm, __dsub_rn(u[4], __dmul_rn(ux, uy)));
      const double A1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), C1), A2 = __dadd_rn(__dmul_rn(2.0, vxy), C2);
      const double B1 = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), C1), B2 = __dadd_rn(__dadd_rn(vx, vy), C2);
      acc[ch] = __ddiv_rn(__dmul_rn(A1, A2), __dmul_rn(B1, B2));
    }
    __syncthreads();
  }
  // PSNR: every element of the image once, grid-stride in linear block order
  const long long n = (long long)H * W * 3;
  const long long blk = (long long)blockIdx.y * gridDim.x + blockIdx.x, nblk = (long long)gridDim.x * gridDim.y;
  for (long long i = blk * kSsimThreads + t; i < n; i += nblk * kSsimThreads) {
    const float d = __fsub_rn(a[i], b[i]);
    acc[3] = __dadd_rn(acc[3], (double)__fmul_rn(d, d));
  }
  block_sum(red, acc, kSsimSums, partial + blk * kSsimSums);
}

// one block: partials in block order; frame = (psnr, ssim); bucket row [psnr, ssim, lpips, n] += (psnr, ssim, -, 1)
__global__ void __launch_bounds__(kSsimThreads) psnr_ssim_final_kernel(const double* __restrict__ partial, int n_blocks, int H, int W,
                                                                       double* __restrict__ bucket, int slot, double* __restrict__ frame) {
  __shared__ double red[kSsimSums][kSsimThreads];
  __shared__ double tot[kSsimSums];
  double s[kSsimSums] = {0.0, 0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < n_blocks; i += kSsimThreads)
#pragma unroll
    for (int k = 0; k < kSsimSums; ++k) s[k] += partial[(size_t)i * kSsimSums + k];
  block_sum(red, s, kSsimSums, tot);
  __syncthreads();
  if (threadIdx.x != 0) return;
  const double n_in = (double)(H - 2 * kPad) * (double)(W - 2 * kPad);
  // np.mean over the three channel values: ((m0 + m1) + m2) / 3
  const double ssim = (tot[0] / n_in + tot[1] / n_in + tot[2] / n_in) / 3.0;
  const double mse = tot[3] / ((double)H * W * 3.0);
  const double psnr = 10.0 * log10(1.0 / mse);    // identical images: 1/0 = inf
  if (frame) { frame[0] = psnr; frame[1] = ssim; }
  if (bucket) {
    bucket[slot * 4 + 0] += psnr;
    bucket[slot * 4 + 1] += ssim;
    bucket[slot * 4 + 3] += 1.0;
  }
}

// ---- LPIPS-VGG ----------------------------------------------------------------------------------------------------
constexpr int kLpipsLayers = 5;
constexpr int kPrepC = 32;           // conv1_1 input channels as stored: RGB + 29 zero channels (one 32-wide k-block)
constexpr int kHeadThreads = 256, kHeadBlocks = 256;   // fixed: the summation order depends on the shape only
constexpr int kHeadWarps = kHeadThreads / 32;
constexpr int kMaxC4PerLane = 512 / 4 / 32;

__device__ __forceinline__ float round_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// compute_lpips: (img - 0.5) * 2, then ScalingLayer (x - shift) / scale, float32; stored channels-last and rounded to the
// nearest tf32 because it feeds a convolution
__global__ void lpips_prep_kernel(const float* __restrict__ img, int n_pix, float s0, float s1, float s2, float k0, float k1, float k2,
                                  float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix * (kPrepC / 4)) return;
  const int p = i / (kPrepC / 4), q = i % (kPrepC / 4);
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  if (q == 0) {
    const float sh[3] = {s0, s1, s2}, sc[3] = {k0, k1, k2};
    float v[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float x = __fmul_rn(__fsub_rn(img[(size_t)p * 3 + ch], 0.5f), 2.f);
      v[ch] = round_tf32(__fdiv_rn(__fsub_rn(x, sh[ch]), sc[ch]));
    }
    o = make_float4(v[0], v[1], v[2], 0.f);
  }
  reinterpret_cast<float4*>(out)[i] = o;
}

// nn.MaxPool2d(2, 2) (floor mode) on [H][W][C]; the inputs are tf32-rounded already, so the outputs are too
__global__ void maxpool2x2_hwc_kernel(const float* __restrict__ in, int H, int W, int C, float* __restrict__ out) {
  const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Ho * Wo * C4) return;
  const int c4 = (int)(i % C4);
  const long long p = i / C4;
  const int x = (int)(p % Wo), y = (int)(p / Wo);
  const float4* r0 = reinterpret_cast<const float4*>(in + ((size_t)(2 * y) * W + 2 * x) * C) + c4;
  const float4* r1 = reinterpret_cast<const float4*>(in + ((size_t)(2 * y + 1) * W + 2 * x) * C) + c4;
  const float4 a = r0[0], b = r0[C4], c = r1[0], d = r1[C4];
  reinterpret_cast<float4*>(out)[i] = make_float4(fmaxf(fmaxf(a.x, b.x), fmaxf(c.x, d.x)), fmaxf(fmaxf(a.y, b.y), fmaxf(c.y, d.y)),
                                                  fmaxf(fmaxf(a.z, b.z), fmaxf(c.z, d.z)), fmaxf(fmaxf(a.w, b.w), fmaxf(c.w, d.w)));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// one warp per pixel: n = sqrt(sum_c f^2) + 1e-10 for both taps, d = sum_c lin_c (f0/n0 - f1/n1)^2 in float32 (the
// reference's dtype); the per-pixel values summed in float64, warp by warp, into one partial per block
__global__ void __launch_bounds__(kHeadThreads) lpips_head_kernel(const float* __restrict__ f0, const float* __restrict__ f1, int n_pix,
                                                                  int C, const float* __restrict__ lin, double* __restrict__ partial) {
  __shared__ double red[kHeadWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C4 = C / 4;
  double acc = 0.0;
  for (int p = blockIdx.x * kHeadWarps + warp; p < n_pix; p += gridDim.x * kHeadWarps) {
    const float4* a4 = reinterpret_cast<const float4*>(f0 + (size_t)p * C);
    const float4* b4 = reinterpret_cast<const float4*>(f1 + (size_t)p * C);
    float4 a[kMaxC4PerLane], b[kMaxC4PerLane];
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxC4PerLane; ++j) {
      const int c4 = lane + 32 * j;
      a[j] = c4 < C4 ? a4[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
      b[j] = c4 < C4 ? b4[c4] : make_float4(0.f, 0.f, 0.f, 0.f);
      sa += a[j].x * a[j].x + a[j].y * a[j].y + a[j].z * a[j].z + a[j].w * a[j].w;
      sb += b[j].x * b[j].x + b[j].y * b[j].y + b[j].z * b[j].z + b[j].w * b[j].w;
    }
    const float na = __fadd_rn(sqrtf(warp_sum(sa)), 1e-10f), nb = __fadd_rn(sqrtf(warp_sum(sb)), 1e-10f);
    float d = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxC4PerLane; ++j) {
      const int c4 = lane + 32 * j;
      if (c4 >= C4) break;
      const float4 w = reinterpret_cast<const float4*>(lin)[c4];
      const float ex = __fsub_rn(__fdiv_rn(a[j].x, na), __fdiv_rn(b[j].x, nb)), ey = __fsub_rn(__fdiv_rn(a[j].y, na), __fdiv_rn(b[j].y, nb));
      const float ez = __fsub_rn(__fdiv_rn(a[j].z, na), __fdiv_rn(b[j].z, nb)), ew = __fsub_rn(__fdiv_rn(a[j].w, na), __fdiv_rn(b[j].w, nb));
      d += w.x * (ex * ex) + w.y * (ey * ey) + w.z * (ez * ez) + w.w * (ew * ew);
    }
    d = warp_sum(d);
    acc += (double)d;                 // identical across the warp's lanes
  }
  if (lane == 0) red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < kHeadWarps; ++w) s += red[w];
    partial[blockIdx.x] = s;
  }
}

// the five spatial means (partials in block order) summed in layer order, rounded to float32 like the reference's value
struct TapPixels { int n[kLpipsLayers]; };
__global__ void lpips_final_kernel(const double* __restrict__ partial, const TapPixels n_pix, float* __restrict__ out) {
  __shared__ double mean[kLpipsLayers];
  if (threadIdx.x < kLpipsLayers) {
    double s = 0.0;
    for (int b = 0; b < kHeadBlocks; ++b) s += partial[threadIdx.x * kHeadBlocks + b];
    mean[threadIdx.x] = s / (double)n_pix.n[threadIdx.x];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int k = 0; k < kLpipsLayers; ++k) v += mean[k];
    *out = (float)v;
  }
}

__global__ void fill_ones_kernel(float* p, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 1.f;
}

inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

struct LpipsWs {
  float* ones;                        // conv scale (512)
  float* buf[2][2];                   // [image][ping/pong], H*W*64 floats each
  double* partial;                    // [5][kHeadBlocks]
};

size_t carve_lpips(int H, int W, unsigned char* base, LpipsWs* ws) {
  size_t off = 0;
  auto take = [&](size_t bytes) { unsigned char* p = base + off; off += al256(bytes); return p; };
  LpipsWs w;
  w.ones = reinterpret_cast<float*>(take(512 * sizeof(float)));
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) w.buf[i][j] = reinterpret_cast<float*>(take((size_t)H * W * 64 * sizeof(float)));
  w.partial = reinterpret_cast<double*>(take((size_t)kLpipsLayers * kHeadBlocks * sizeof(double)));
  if (ws) *ws = w;
  return off;
}

}  // namespace

size_t psnr_ssim_workspace_bytes(int H, int W) {
  const size_t nb = (size_t)((W - 2 * kPad + kTW - 1) / kTW) * ((H - 2 * kPad + kTH - 1) / kTH);
  return nb * kSsimSums * sizeof(double);
}

void launch_psnr_ssim(const float* img, const float* gt, int H, int W, void* ws, double* bucket, int slot, double* frame, cudaStream_t st) {
  const dim3 grid((W - 2 * kPad + kTW - 1) / kTW, (H - 2 * kPad + kTH - 1) / kTH);
  psnr_ssim_partial_kernel<<<grid, kSsimThreads, 0, st>>>(img, gt, H, W, (double*)ws);
  psnr_ssim_final_kernel<<<1, kSsimThreads, 0, st>>>((const double*)ws, (int)(grid.x * grid.y), H, W, bucket, slot, frame);
}

// VGG16 features[0:30]: five stages of (2, 2, 3, 3, 3) conv3x3+ReLU, a 2x2 max-pool before stages 2..5; the tap is the
// last ReLU of each stage
static const int kStageConvs[kLpipsLayers] = {2, 2, 3, 3, 3};
static const int kStageC[kLpipsLayers] = {64, 128, 256, 512, 512};

size_t lpips_workspace_bytes(int H, int W) { return carve_lpips(H, W, nullptr, nullptr); }

int run_lpips_vgg(const float* img0, const float* img1, int H, int W, const float* const* w9, const float* const* bias,
                  const float* const* lin, const float* shift, const float* scale, void* workspace, float* out, cudaStream_t st) {
  LpipsWs ws;
  carve_lpips(H, W, reinterpret_cast<unsigned char*>(workspace), &ws);
  int launches = 0;
  fill_ones_kernel<<<2, 256, 0, st>>>(ws.ones, 512);
  ++launches;
  const float* img[2] = {img0, img1};
  float* cur[2];
  float* spare[2];
  for (int i = 0; i < 2; ++i) {
    cur[i] = ws.buf[i][0];
    spare[i] = ws.buf[i][1];
    const int n = H * W * (kPrepC / 4);
    lpips_prep_kernel<<<(n + 255) / 256, 256, 0, st>>>(img[i], H * W, shift[0], shift[1], shift[2], scale[0], scale[1], scale[2], cur[i]);
    ++launches;
  }
  int h = H, w = W, cin = kPrepC, layer = 0;
  TapPixels n_pix;
  for (int s = 0; s < kLpipsLayers; ++s) {
    if (s > 0) {
      for (int i = 0; i < 2; ++i) {
        const long long n = (long long)(h / 2) * (w / 2) * (cin / 4);
        maxpool2x2_hwc_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(cur[i], h, w, cin, spare[i]);
        ++launches;
        float* t = cur[i]; cur[i] = spare[i]; spare[i] = t;
      }
      h /= 2;
      w /= 2;
    }
    const int cout = kStageC[s];
    for (int k = 0; k < kStageConvs[s]; ++k, ++layer) {
      for (int i = 0; i < 2; ++i) {
        const int rc = launch_conv3x3_tf32(cur[i], h, w, cin, w9[layer], cout, 1, ws.ones, bias[layer], nullptr, 0, 0.f, 1, spare[i], cout,
                                           nullptr, 0, st);
        if (rc) return rc == -2 ? -2 : -1;
        ++launches;
        float* t = cur[i]; cur[i] = spare[i]; spare[i] = t;
      }
      cin = cout;
    }
    lpips_head_kernel<<<kHeadBlocks, kHeadThreads, 0, st>>>(cur[0], cur[1], h * w, cout, lin[s], ws.partial + s * kHeadBlocks);
    ++launches;
    n_pix.n[s] = h * w;
  }
  lpips_final_kernel<<<1, 32, 0, st>>>(ws.partial, n_pix, out);
  return launches + 1;
}

}  // namespace srf
