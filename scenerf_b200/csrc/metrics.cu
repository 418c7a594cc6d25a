// Evaluation metrics on the device (DESIGN.md 6.7): the numbers the reference computes on the host after a
// reconstruction or a novel-depth render.
//   confusion : tsdf2occ (scripts/evaluation/eval_sr.py:11-17, eval_sc_bf.py:117-123) or a given prediction, against
//               uint8 target labels, into joint (target bucket x pred bucket) histograms -- per z slice when asked, once
//               without and once with a mask.  Every number SSCMetrics (loss/sscMetrics.py:361-529) reports follows
//               from these integer counts; integer atomics make them independent of the thread schedule.
//   sc_label  : the BundleFusion completion target (scripts/reconstruction/generate_sc_gt_bf.py:307-309).
//   depth     : compute_depth_errors (loss/depth_metrics.py) with float64 block sums, a fixed-order second pass and the
//               frame's 7 values added into a caller-chosen bucket slot on the device.
#include "kernels.cuh"

namespace srf {

namespace {

constexpr int kHistThreads = 256;

template <typename T>
__device__ __forceinline__ double as_double(T v) { return (double)v; }

// pred bucket of one value: j for v == j (j < C), C for any other v > 0, C+1 for the rest (v <= 0 or NaN)
template <typename T>
__device__ __forceinline__ int pred_bucket(T v, int C) {
  const double d = as_double(v);
  if (d >= 0.0 && d < (double)C && d == floor(d)) return (int)d;
  return d > 0.0 ? C : C + 1;
}

// grid-stride over the volume (C order: z fastest).  hist[zh][m][tb][pb], m = 0 unmasked / 1 masked,
// tb = target bucket 0..C (C = a label >= C other than 255), pb = pred bucket 0..C+1.
// PRED: -1 = occupancy from the tsdf, otherwise a srf_eval_dtype of the pred array.
template <int PRED, typename T>
__global__ void __launch_bounds__(kHistThreads) confusion_kernel(
    const float* __restrict__ tsdf, const T* __restrict__ pred, const uint8_t* __restrict__ target,
    const uint8_t* __restrict__ mask, int X, int Y, int Z, int C, int th_axis, const double* __restrict__ th,
    int per_z, unsigned long long* __restrict__ hist, int* __restrict__ max_z, uint8_t* __restrict__ occ_out) {
  extern __shared__ unsigned int sh[];
  const int TB = C + 1, PB = C + 2, per_m = TB * PB;
  const int n_sh = (per_z ? Z : 1) * 2 * per_m;
  for (int i = threadIdx.x; i < n_sh; i += blockDim.x) sh[i] = 0u;
  __shared__ int sh_max_z;
  if (threadIdx.x == 0) sh_max_z = -1;
  __syncthreads();
  const long long n = (long long)X * Y * Z;
  const int occ_bucket = C > 1 ? 1 : C;
  int my_max_z = -1;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(i % Z);
    int pb;
    if (PRED < 0) {
      const float t = tsdf[i];
      const float a = fabsf(t);
      const int ti = th_axis == 0 ? (int)(i / ((long long)Y * Z)) : th_axis == 1 ? (int)((i / Z) % Y) : z;
      // numpy compares the float32 |tsdf| with the float64 table in float64 (exact promotion)
      const bool o = ((double)a < th[ti]) && (a != 255.f);
      if (occ_out) occ_out[i] = o ? 1 : 0;
      pb = o ? occ_bucket : 0;
    } else {
      pb = pred_bucket(pred[i], C);
    }
    const int tv = target ? target[i] : 255;            // no target: occupancy only
    if (tv != 0 && tv != 255) my_max_z = max(my_max_z, z);
    // most voxels of a volume share a few counters: one shared atomic per distinct counter of the warp
    const int key = tv == 255 ? -1 : (per_z ? z : 0) * 2 * per_m + (tv < C ? tv : C) * PB + pb;
    const unsigned act = __activemask(), lane = threadIdx.x & 31;
    const unsigned peers = __match_any_sync(act, key);
    if (key >= 0 && __ffs(peers) - 1 == (int)lane) atomicAdd(sh + key, (unsigned)__popc(peers));
    if (mask) {
      const int mkey = mask[i] ? key : -1;
      const unsigned mpeers = __match_any_sync(act, mkey);
      if (mkey >= 0 && __ffs(mpeers) - 1 == (int)lane) atomicAdd(sh + mkey + per_m, (unsigned)__popc(mpeers));
    }
  }
  for (int o = 16; o > 0; o >>= 1) my_max_z = max(my_max_z, __shfl_xor_sync(0xffffffffu, my_max_z, o));
  if ((threadIdx.x & 31) == 0 && my_max_z >= 0) atomicMax(&sh_max_z, my_max_z);
  __syncthreads();
  for (int i = threadIdx.x; i < n_sh; i += blockDim.x)
    if (sh[i]) atomicAdd(hist + i, (unsigned long long)sh[i]);
  if (threadIdx.x == 0 && sh_max_z >= 0) atomicMax(max_z, sh_max_z);
}

// generate_sc_gt_bf.py:307-309: 255 everywhere, 0 where tsdf > vs, 1 where |tsdf| < vs (both away from 255).  numpy
// compares the float32 grid with the Python float voxel_size in float32 (a Python scalar does not promote an array).
__global__ void sc_label_kernel(const float* __restrict__ tsdf, long long n, float vs, uint8_t* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float t = tsdf[i];
  uint8_t o = 255;
  if (t != 255.f) {
    if (t > vs) o = 0;
    if (fabsf(t) < vs) o = 1;
  }
  out[i] = o;
}

constexpr int kDepthThreads = 256;
constexpr int kDepthBlocks = 256;   // fixed: the summation order depends on n only, not on the device
constexpr int kDepthSums = 7;

// sums: abs_rel, sq_rel, squared error, squared log error (float32 terms as numpy forms them) and the a1/a2/a3 counts
__global__ void __launch_bounds__(kDepthThreads) depth_partial_kernel(const float* __restrict__ gt, const float* __restrict__ pred,
                                                                      long long n, double* __restrict__ partial) {
  double s[kDepthSums] = {0, 0, 0, 0, 0, 0, 0};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float g = gt[i];
    float p = pred[i];
    if (p < 1e-3f) p = 1e-3f;             // depth_metrics.py: pred[pred < min_depth] = min_depth (float32 compare)
    if (p > 80.f) p = 80.f;
    const float r0 = __fdiv_rn(g, p), r1 = __fdiv_rn(p, g);
    const bool nan = (r0 != r0) || (r1 != r1);           // np.maximum propagates NaN: such a ratio passes no threshold
    const float th = fmaxf(r0, r1);
    const float d = __fsub_rn(g, p);
    const float d2 = __fmul_rn(d, d);
    const float lg = __fsub_rn(logf(g), logf(p));
    s[0] += (double)__fdiv_rn(fabsf(d), g);
    s[1] += (double)__fdiv_rn(d2, g);
    s[2] += (double)d2;
    s[3] += (double)__fmul_rn(lg, lg);
    s[4] += (!nan && th < 1.25f) ? 1.0 : 0.0;
    s[5] += (!nan && th < 1.5625f) ? 1.0 : 0.0;       // 1.25 ** 2, exact in float32
    s[6] += (!nan && th < 1.953125f) ? 1.0 : 0.0;     // 1.25 ** 3
  }
  __shared__ double red[kDepthSums][kDepthThreads];
#pragma unroll
  for (int k = 0; k < kDepthSums; ++k) red[k][threadIdx.x] = s[k];
  __syncthreads();
  for (int w = kDepthThreads / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) {
#pragma unroll
      for (int k = 0; k < kDepthSums; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x < kDepthSums) partial[blockIdx.x * kDepthSums + threadIdx.x] = red[threadIdx.x][0];
}

// one block: the partials in block order, then the frame's values in the reference's dtypes (float32 means and square
// roots for the first four, float64 fractions for a1..a3), added to bucket[slot] = 7 sums + a frame count
__global__ void __launch_bounds__(kDepthThreads) depth_final_kernel(const double* __restrict__ partial, int n_blocks, long long n,
                                                                    double* __restrict__ bucket, int slot, double* __restrict__ frame) {
  __shared__ double tot[kDepthSums];
  if (threadIdx.x < kDepthSums) {
    double a = 0.0;
    for (int b = 0; b < n_blocks; ++b) a += partial[b * kDepthSums + threadIdx.x];
    tot[threadIdx.x] = a;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const double dn = (double)n;
  double v[kDepthSums];
  v[0] = (double)(float)(tot[0] / dn);
  v[1] = (double)(float)(tot[1] / dn);
  v[2] = (double)sqrtf((float)(tot[2] / dn));
  v[3] = (double)sqrtf((float)(tot[3] / dn));
  for (int k = 4; k < kDepthSums; ++k) v[k] = tot[k] / dn;
  for (int k = 0; k < kDepthSums; ++k) {
    if (frame) frame[k] = v[k];
    if (bucket) bucket[slot * (kDepthSums + 1) + k] += v[k];
  }
  if (bucket) bucket[slot * (kDepthSums + 1) + kDepthSums] += 1.0;
}

template <int PRED, typename T>
void launch_confusion_t(const float* tsdf, const void* pred, const uint8_t* target, const uint8_t* mask, const int* dims, int C,
                        int th_axis, const double* th, int per_z, unsigned long long* hist, int* max_z, uint8_t* occ,
                        int n_sm, cudaStream_t st) {
  const size_t sh = eval_hist_len(dims, C, per_z) * sizeof(unsigned int);
  auto k = confusion_kernel<PRED, T>;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh);
  const long long n = (long long)dims[0] * dims[1] * dims[2];
  // a few blocks per SM: each block flushes its whole histogram once, so more blocks cost more global atomics
  long long blocks = (n + kHistThreads * 8 - 1) / (kHistThreads * 8);
  blocks = blocks < 4LL * n_sm ? blocks : 4LL * n_sm;
  if (blocks < 1) blocks = 1;
  k<<<(unsigned)blocks, kHistThreads, sh, st>>>(tsdf, (const T*)pred, target, mask, dims[0], dims[1], dims[2], C, th_axis, th,
                                               per_z, hist, max_z, occ);
}

}  // namespace

size_t eval_hist_len(const int* dims, int n_classes, int per_z) {
  return (size_t)(per_z ? dims[2] : 1) * 2 * (n_classes + 1) * (n_classes + 2);
}

void launch_eval_confusion(const float* tsdf, const void* pred, int pred_dtype, const uint8_t* target, const uint8_t* mask,
                           const int* dims, int n_classes, int th_axis, const double* th, int per_z, unsigned long long* hist,
                           int* max_z, uint8_t* occ, cudaStream_t st) {
  int dev = 0, n_sm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
  cudaMemsetAsync(hist, 0, eval_hist_len(dims, n_classes, per_z) * sizeof(unsigned long long), st);
  cudaMemsetAsync(max_z, 0xff, sizeof(int), st);            // -1: no labelled voxel
  switch (pred ? pred_dtype : -1) {
    case -1: launch_confusion_t<-1, float>(tsdf, nullptr, target, mask, dims, n_classes, th_axis, th, per_z, hist, max_z, occ, n_sm, st); break;
    case SRF_EVAL_U8: launch_confusion_t<0, uint8_t>(nullptr, pred, target, mask, dims, n_classes, 0, nullptr, per_z, hist, max_z, nullptr, n_sm, st); break;
    case SRF_EVAL_I32: launch_confusion_t<1, int32_t>(nullptr, pred, target, mask, dims, n_classes, 0, nullptr, per_z, hist, max_z, nullptr, n_sm, st); break;
    case SRF_EVAL_I64: launch_confusion_t<2, long long>(nullptr, pred, target, mask, dims, n_classes, 0, nullptr, per_z, hist, max_z, nullptr, n_sm, st); break;
    case SRF_EVAL_F32: launch_confusion_t<3, float>(nullptr, pred, target, mask, dims, n_classes, 0, nullptr, per_z, hist, max_z, nullptr, n_sm, st); break;
    default: launch_confusion_t<4, double>(nullptr, pred, target, mask, dims, n_classes, 0, nullptr, per_z, hist, max_z, nullptr, n_sm, st); break;
  }
}

void launch_eval_sc_label(const float* tsdf, long long n, float voxel_size, uint8_t* out, cudaStream_t st) {
  sc_label_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(tsdf, n, voxel_size, out);
}

size_t depth_errors_workspace_bytes() { return (size_t)kDepthBlocks * kDepthSums * sizeof(double); }

void launch_depth_errors(const float* gt, const float* pred, long long n, void* ws, double* bucket, int slot, double* frame,
                         cudaStream_t st) {
  long long blocks = (n + kDepthThreads - 1) / kDepthThreads;
  blocks = blocks < kDepthBlocks ? blocks : kDepthBlocks;
  if (blocks < 1) blocks = 1;
  depth_partial_kernel<<<(unsigned)blocks, kDepthThreads, 0, st>>>(gt, pred, n, (double*)ws);
  depth_final_kernel<<<1, 32, 0, st>>>((const double*)ws, (int)blocks, n, bucket, slot, frame);
}

}  // namespace srf
