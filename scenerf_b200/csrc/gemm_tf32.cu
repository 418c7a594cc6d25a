// TF32 tensor-core GEMM for the training path:  C[M x N] = epilogue( A[M x K] * B[N x K]^T ),  A and B float32, both
// K-contiguous ("NT"), accumulation in float32.  wgmma .tf32 reads the float32 operands straight from shared memory (top 19
// bits), so there is no conversion pass: 2-D TMA tensor copies (128-byte swizzle) stage 128 x 32 float tiles of A
// and B through the tf32 tile mainloop of tma.cuh, and the two consumer warpgroups (rows 0-63 / 64-127 of the tile) apply
// the same epilogue as gemm.cu (bias, ReLU mask, residual, accumulate) straight from registers.  One output tile per CTA;
// split-K over gridDim.z with fixed-order reduction for the weight-gradient shapes.
// SPLIT = true is the same kernel on the 3xTF32 mainloop (tma.cuh): hi.hi + hi.lo + lo.hi per k-step, products of
// float32-grade accuracy from raw float32 operands (the fp32tc training engine); tiles, epilogue and split-K are shared.
#include "kernels.cuh"
#include "tma.cuh"

namespace srf {
namespace tf32 {

static_assert(kBN == kSegTileN, "segment mode 2 skips whole column tiles of this kernel");

template <bool SPLIT>
__global__ void __launch_bounds__(kThreads, 1)
gemm_tf32_nt_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, float* C, int ldc, int M, int N,
                    int K, const float* __restrict__ bias, const float* __restrict__ mask, int ldm, const float* R, int ldr,
                    int accumulate, int k_per, const int* __restrict__ skip, const __grid_constant__ SegInfo sg, int* err,
                    float* relu_out, int ld_relu) {
  if (skip && *skip == 0) return;
  if (sg.mode == 2 && seg_dead(sg, blockIdx.x * kBN, min(N, (int)(blockIdx.x + 1) * kBN))) return;   // dead column tile
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * kBN;
  const int kbeg = blockIdx.z * k_per;
  const int kend = min(K, kbeg + k_per);
  const int nk = (kend - kbeg + kBK - 1) / kBK;
  if (gridDim.z > 1) C += (size_t)blockIdx.z * M * ldc;

  // K-segmented mode: k-blocks that lie entirely in dead scales are not streamed; n_live = number of blocks that are
  auto dead = [&](int k0) { return sg.mode == 1 && seg_dead(sg, k0, min(kend, k0 + kBK)); };
  int n_live = nk;
  if (sg.mode == 1) {
    n_live = 0;
    for (int k0 = kbeg; k0 < kend; k0 += kBK) n_live += dead(k0) ? 0 : 1;
  }
  int k0 = kbeg;                                             // the producer's cursor: first k of the next block
  float acc[64];
  if (!mainloop<SPLIT ? kWatchGemmFp32tc : kWatchGemmTf32, SPLIT>(&tmA, &tmB, n_live, err, acc, [&](uint32_t sA, uint32_t sB, uint32_t bar) {
        while (dead(k0)) k0 += kBK;
        tma_load_2d(sA, &tmA, k0, m0, bar);
        tma_load_2d(sB, &tmB, k0, n0, bar);
        k0 += kBK;
      }))
    return;
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int w = t >> 5, l = t & 31;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int gm = m0 + (wg - 1) * 64 + 16 * w + (l >> 2) + 8 * half;
    if (gm >= M) continue;
#pragma unroll
    for (int c8 = 0; c8 < kBN / 8; ++c8) {
      const int gn = n0 + 8 * c8 + 2 * (l & 3);
      if (gn >= N) break;                                    // N % 4 == 0: gn + 1 < N as well
      float2 o = make_float2(acc[4 * c8 + 2 * half], acc[4 * c8 + 2 * half + 1]);
      if (bias) { const float2 t2 = *reinterpret_cast<const float2*>(bias + gn); o.x += t2.x; o.y += t2.y; }
      if (mask) {
        const float2 t2 = *reinterpret_cast<const float2*>(mask + (size_t)gm * ldm + gn);
        o.x = t2.x > 0.f ? o.x : 0.f; o.y = t2.y > 0.f ? o.y : 0.f;
      }
      if (R) { const float2 t2 = *reinterpret_cast<const float2*>(R + (size_t)gm * ldr + gn); o.x += t2.x; o.y += t2.y; }
      float2* dst = reinterpret_cast<float2*>(C + (size_t)gm * ldc + gn);
      if (accumulate) { const float2 t2 = *dst; o.x += t2.x; o.y += t2.y; }
      *dst = o;
      if (relu_out)          // the consumer GEMM reads its A operand as stored: hand it the ReLU'd activations directly
        *reinterpret_cast<float2*>(relu_out + (size_t)gm * ld_relu + gn) = make_float2(fmaxf(o.x, 0.f), fmaxf(o.y, 0.f));
    }
  }
}

}  // namespace tf32

// rows x K float32 matrix with row stride ld (elements): box = 128 rows x 32 floats
static bool encode_f32(CUtensorMap* tm, const float* base, int rows, int K, int ld) {
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows}, strides[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {(cuuint32_t)tf32::kBK, (cuuint32_t)tf32::kBM};
  return encode_tensor_map_f32(tm, base, 2, dims, strides, box) == 0;
}

template <bool SPLIT>
static int launch(const GemmArgs& g, const CUtensorMap& tmA, const CUtensorMap& tmB, cudaStream_t st) {
  constexpr size_t smem = SPLIT ? tf32::kSplitSmemBytes : tf32::kSmemBytes;
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(tf32::gemm_tf32_nt_kernel<SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); attr = true; }
  int* err = watchdog_device_flag();
  dim3 grid((g.N + tf32::kBN - 1) / tf32::kBN, (g.M + tf32::kBM - 1) / tf32::kBM);
  SegInfo sg;
  sg.flags = g.seg_flags; sg.mode = g.seg_flags ? g.seg_mode : 0;
  for (int i = 0; i < 6; ++i) sg.off[i] = g.seg_off[i];
  // the relu_out store needs the finished sum, so such a call is never split
  const SplitK sk = g.relu_out ? SplitK{1, g.K} : plan_splitk(g, grid.x * grid.y, tf32::kBK, 32);
  if (sk.splits > 1) {
    grid.z = sk.splits;
    tf32::gemm_tf32_nt_kernel<SPLIT><<<grid, tf32::kThreads, smem, st>>>(tmA, tmB, g.splitk_ws, g.N, g.M, g.N, g.K, nullptr, nullptr, 0,
                                                                        nullptr, 0, 0, sk.k_per, g.skip_if_zero, sg, err, nullptr, 0);
    launch_splitk_reduce(g, sk.splits, sg, st);
    launch_counter() += 2;
  } else {
    ++launch_counter();
    tf32::gemm_tf32_nt_kernel<SPLIT><<<grid, tf32::kThreads, smem, st>>>(tmA, tmB, g.C, g.ldc, g.M, g.N, g.K, g.bias, g.mask, g.ldm, g.R,
                                                                        g.ldr, g.accumulate, g.K, g.skip_if_zero, sg, err, g.relu_out,
                                                                        g.ld_relu);
  }
  return 0;
}

// Only the NT layout with un-transformed operands (at=false, bt=true, no relu_a / relu_b).  Returns 0, or -1 when the
// shape cannot go through TMA (unaligned rows) -- the caller then falls back to launch_gemm.
int launch_gemm_tf32(const GemmArgs& g, cudaStream_t st, bool split) {
  if (g.at || !g.bt || g.relu_a || g.relu_b) return -1;
  if ((g.lda % 4) || (g.ldb % 4) || (g.ldc % 4) || (g.N % 4) || !al16(g.A) || !al16(g.B) || !al16(g.C)) return -1;
  if ((g.bias && !al16(g.bias)) || (g.mask && (!al16(g.mask) || g.ldm % 4)) || (g.R && (!al16(g.R) || g.ldr % 4))) return -1;
  if (g.relu_out && (!al16(g.relu_out) || g.ld_relu % 4)) return -1;
  CUtensorMap tmA, tmB;
  if (!encode_f32(&tmA, g.A, g.M, g.K, g.lda) || !encode_f32(&tmB, g.B, g.N, g.K, g.ldb)) return -1;
  return split ? launch<true>(g, tmA, tmB, st) : launch<false>(g, tmA, tmB, st);
}

}  // namespace srf
