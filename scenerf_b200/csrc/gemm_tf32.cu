// TF32 tensor-core GEMM for the training path:  C[M x N] = epilogue( A[M x K] * B[N x K]^T ),  A and B float32, both
// K-contiguous ("NT"), accumulation in float32.  wgmma .tf32 reads the float32 operands straight from shared memory (top 19
// bits), so there is no conversion pass: TMA (cp.async.bulk.tensor.2d, 128-byte swizzle) stages 128 x 32 float tiles of A
// and B into a 3-stage mbarrier ring, and two consumer warpgroups (rows 0-63 / 64-127 of the tile) each issue 4 wgmma
// m64n128k8 per stage into a 64 x 128 register accumulator, then apply the same epilogue as gemm.cu (bias, ReLU mask,
// residual, accumulate) straight from registers.  One output tile per CTA; split-K over gridDim.z with fixed-order
// reduction for the weight-gradient shapes.
#include <cuda.h>
#include "kernels.cuh"
#include "wgmma.cuh"

namespace srf {
namespace tf32 {

constexpr int kBM = 128, kBN = 128, kBK = 32, kStages = 3;
constexpr uint32_t kTileBytes = kBM * kBK * 4;            // 16 KB
constexpr int kThreads = 384;                             // warpgroup 0: TMA producer (one thread); 1, 2: MMA + epilogue

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
// bounded wait: a protocol bug must not hang the GPU
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* err) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 2000000000LL) { if (err) atomicExch(err, (int)(0x54000000u | (bar & 0xFFFFFF))); __trap(); }
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}

struct SegInfo { const int* flags; int mode; int off[6]; };
// true when [lo, hi) of the latent axis touches only scales whose flag is 0
__device__ __forceinline__ bool seg_dead(const SegInfo& sg, int lo, int hi) {
#pragma unroll
  for (int s = 0; s < 5; ++s)
    if (lo < sg.off[s + 1] && hi > sg.off[s] && sg.flags[s] != 0) return false;
  return true;
}

__global__ void __launch_bounds__(kThreads, 1)
gemm_tf32_nt_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, float* C, int ldc, int M, int N,
                    int K, const float* __restrict__ bias, const float* __restrict__ mask, int ldm, const float* R, int ldr,
                    int accumulate, int k_per, const int* __restrict__ skip, const __grid_constant__ SegInfo sg, int* err,
                    float* relu_out, int ld_relu) {
  if (skip && *skip == 0) return;
  if (sg.mode == 2 && seg_dead(sg, blockIdx.x * kBN, min(N, (int)(blockIdx.x + 1) * kBN))) return;   // dead column tile
  extern __shared__ unsigned char smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;            // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t sA = base, sB = base + kStages * kTileBytes;
  const uint32_t bars = sB + kStages * kTileBytes;                        // full[kStages], empty[kStages]
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * kBN;
  const int kbeg = blockIdx.z * k_per;
  const int kend = min(K, kbeg + k_per);
  const int nk = (kend - kbeg + kBK - 1) / kBK;
  if (gridDim.z > 1) C += (size_t)blockIdx.z * M * ldc;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");   // descriptor fetch off the first load's path
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
    for (int s = 0; s < kStages; ++s) { mbar_init(bars + 8u * s, 1); mbar_init(bars + 8u * (kStages + s), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // K-segmented mode: k-blocks that lie entirely in dead scales are skipped by producer and consumers alike (same predicate,
  // same order, so the ring stays in step); n_live = number of blocks actually streamed
  int n_live = nk;
  if (sg.mode == 1) {
    n_live = 0;
    for (int i = 0; i < nk; ++i) n_live += seg_dead(sg, kbeg + i * kBK, min(kend, kbeg + (i + 1) * kBK)) ? 0 : 1;
  }
  if (wg == 0) {
    if (t == 0) {
      int j = 0;
      for (int i = 0; i < nk; ++i) {
        if (sg.mode == 1 && seg_dead(sg, kbeg + i * kBK, min(kend, kbeg + (i + 1) * kBK))) continue;
        const int s = j % kStages;
        mbar_wait(bars + 8u * (kStages + s), (((uint32_t)(j / kStages)) & 1u) ^ 1u, err);
        mbar_arrive_expect_tx(bars + 8u * s, 2 * kTileBytes);
        tma_load_2d(sA + s * kTileBytes, &tmA, kbeg + i * kBK, m0, bars + 8u * s);
        tma_load_2d(sB + s * kTileBytes, &tmB, kbeg + i * kBK, n0, bars + 8u * s);
        ++j;
      }
    }
    return;
  }
  // consumer warpgroup: rows (wg - 1) * 64 .. +63 of the tile (the A tile's 64-row half starts 8 KB further)
  const uint32_t a_off = (uint32_t)(wg - 1) * 64u * 128u;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int j = 0; j < n_live; ++j) {
    const int s = j % kStages;
    mbar_wait(bars + 8u * s, ((uint32_t)(j / kStages)) & 1u, err);
    gmma::fence();
#pragma unroll
    for (int k4 = 0; k4 < kBK / 8; ++k4)     // +32 bytes per k-step of 8 floats inside the swizzle row
      gmma::mma_tf32_n128(acc, gmma::desc_sw128(sA + s * kTileBytes + a_off + k4 * 32), gmma::desc_sw128(sB + s * kTileBytes + k4 * 32),
                          (j > 0 || k4 > 0) ? 1 : 0);
    gmma::commit();
    // this stage's MMAs stay in flight; the previous stage has completed and goes back to the producer
    gmma::wait<1>();
    if (t == 0 && j > 0) mbar_arrive(bars + 8u * (kStages + (j - 1) % kStages));
  }
  gmma::wait<0>();
  gmma::fence_regs(acc);
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

__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ part, int splits, float* __restrict__ C, int ldc, int M, int N, int accumulate,
                     const int* __restrict__ skip, const __grid_constant__ SegInfo sg) {
  if (skip && *skip == 0) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * N) return;
  if (sg.mode == 2) {                                      // columns of a dead tile were never written by the GEMM
    const int t0 = (i % N) / kBN * kBN;
    if (seg_dead(sg, t0, min(N, t0 + kBN))) return;
  }
  float v = 0.f;
  for (int z = 0; z < splits; ++z) v += part[(size_t)z * M * N + i];
  float* dst = C + (size_t)(i / N) * ldc + (i % N);
  *dst = accumulate ? (*dst + v) : v;
}

}  // namespace tf32

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn tf32_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}
// rows x K float32 matrix with row stride ld (elements): box = box_rows rows x 32 floats, 128-byte swizzle
static bool encode_f32(CUtensorMap* tm, const float* base, int rows, int K, int ld, int box_rows = tf32::kBM) {
  EncodeTiledFn fn = tf32_encode_fn();
  if (!fn) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {(cuuint32_t)tf32::kBK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int* g_tf32_err = nullptr;       // mapped host flag written by the watchdog
int tf32_watchdog_flag() { return g_tf32_err ? *reinterpret_cast<volatile int*>(g_tf32_err) : 0; }

// Only the NT layout with un-transformed operands (at=false, bt=true, no relu_a / relu_b).  Returns 0, or -1 when the
// shape cannot go through TMA (unaligned rows) -- the caller then falls back to launch_gemm.
int launch_gemm_tf32(const GemmArgs& g, cudaStream_t st) {
  if (g.at || !g.bt || g.relu_a || g.relu_b) return -1;
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if ((g.lda % 4) || (g.ldb % 4) || (g.ldc % 4) || (g.N % 4) || !al16(g.A) || !al16(g.B) || !al16(g.C)) return -1;
  if ((g.bias && !al16(g.bias)) || (g.mask && (!al16(g.mask) || g.ldm % 4)) || (g.R && (!al16(g.R) || g.ldr % 4))) return -1;
  if (g.relu_out && (!al16(g.relu_out) || g.ld_relu % 4)) return -1;
  if (!g_tf32_err) {
    int* h = nullptr;
    if (cudaHostAlloc(&h, sizeof(int), cudaHostAllocMapped) == cudaSuccess) { *h = 0; cudaHostGetDevicePointer(&g_tf32_err, h, 0); }
  }
  CUtensorMap tmA, tmB;
  if (!encode_f32(&tmA, g.A, g.M, g.K, g.lda) || !encode_f32(&tmB, g.B, g.N, g.K, g.ldb)) return -1;
  static bool attr = false;
  const size_t smem = 2 * tf32::kStages * tf32::kTileBytes + 1024 + 64;
  if (!attr) { cudaFuncSetAttribute(tf32::gemm_tf32_nt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); attr = true; }
  dim3 grid((g.N + tf32::kBN - 1) / tf32::kBN, (g.M + tf32::kBM - 1) / tf32::kBM);
  tf32::SegInfo sg;
  sg.flags = g.seg_flags; sg.mode = g.seg_flags ? g.seg_mode : 0;
  for (int i = 0; i < 6; ++i) sg.off[i] = g.seg_off[i];
  const int tiles = grid.x * grid.y;
  int splits = 1;
  if (g.splitk_ws && !g.bias && !g.mask && !g.R && !g.relu_out && tiles < 96 && g.K >= 1024) {
    splits = (2 * device_sm_count() + tiles - 1) / tiles;     // ~2 waves
    if (splits > 32) splits = 32;
    while (splits > 1 && (size_t)splits * g.M * g.N > g.splitk_ws_floats) --splits;
  }
  if (splits > 1) {
    const int k_per = ((g.K + splits - 1) / splits + tf32::kBK - 1) / tf32::kBK * tf32::kBK;
    splits = (g.K + k_per - 1) / k_per;
    grid.z = splits;
    tf32::gemm_tf32_nt_kernel<<<grid, tf32::kThreads, smem, st>>>(tmA, tmB, g.splitk_ws, g.N, g.M, g.N, g.K, nullptr, nullptr, 0, nullptr, 0,
                                                                  0, k_per, g.skip_if_zero, sg, g_tf32_err, nullptr, 0);
    tf32::splitk_reduce_kernel<<<(g.M * g.N + 255) / 256, 256, 0, st>>>(g.splitk_ws, splits, g.C, g.ldc, g.M, g.N, g.accumulate,
                                                                        g.skip_if_zero, sg);
    launch_counter() += 2;
  } else {
    ++launch_counter();
    tf32::gemm_tf32_nt_kernel<<<grid, tf32::kThreads, smem, st>>>(tmA, tmB, g.C, g.ldc, g.M, g.N, g.K, g.bias, g.mask, g.ldm, g.R, g.ldr,
                                                                  g.accumulate, g.K, g.skip_if_zero, sg, g_tf32_err, g.relu_out, g.ld_relu);
  }
  return 0;
}

}  // namespace srf
