// Hopper mbarrier / TMA primitives of the sm_90a kernels (mlp_tc.cu, gemm_tf32.cu, conv_tf32.cu), the bounded barrier
// wait with its watchdog, and the tf32 tile mainloop that gemm_tf32.cu and conv_tf32.cu share.
#pragma once
#include <cuda.h>
#include "wgmma.cuh"

namespace srf {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}

// Kernel field of the watchdog code (see watchdog_flag in kernels.cuh).
constexpr uint32_t kWatchPointMlp = 0, kWatchGemmTf32 = 1, kWatchConvTf32 = 2, kWatchGemmFp32tc = 3;

// Bounded wait: a protocol bug must not hang the GPU -- after ~2 s the watchdog records the barrier and traps.
template <uint32_t KERNEL>
__device__ __noinline__ void mbar_timeout(int* error_flag, uint32_t bar, uint32_t parity) {
  if (error_flag)
    atomicExch(error_flag, (int)(0x40000000u | ((bar & 0xFFFFF) << 4) | (KERNEL << 1) | (parity & 1) | ((threadIdx.x >> 5) << 24)));
  __threadfence_system();
  __trap();
}
template <uint32_t KERNEL>
__device__ __forceinline__ void mbar_spin(uint32_t bar, uint32_t parity, int* error_flag) {
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) mbar_timeout<KERNEL>(error_flag, bar, parity);
  }
}
template <uint32_t KERNEL>
__device__ __noinline__ void mbar_wait_spin(uint32_t bar, uint32_t parity, int* error_flag) { mbar_spin<KERNEL>(bar, parity, error_flag); }
// The point MLP runs at the register limit, so its spin loop is out of line.  In the tf32 ring the call sits on the
// wake-up path of every wait that misses: an out-of-line spin there made `bench.py --workload decoder` 6 % slower
// (H100 80GB HBM3, 700 W power limit).
template <uint32_t KERNEL>
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* error_flag) {
  if (mbar_try_wait(bar, parity)) return;
  if constexpr (KERNEL == kWatchPointMlp)
    mbar_wait_spin<KERNEL>(bar, parity, error_flag);
  else
    mbar_spin<KERNEL>(bar, parity, error_flag);
}

__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, int c2, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// Host: encodes a float32 tensor map of rank 2 or 3 (dims[0] innermost; strides: byte strides of dims 1..rank-1) with
// 128-byte swizzle, L2_256B promotion and zero fill out of bounds.  Returns 0, -1 (rejected by the driver) or -2 (the
// driver has no tensor-map encoder).
int encode_tensor_map_f32(CUtensorMap* tm, const float* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                          const cuuint32_t* box);

// The tf32 tile mainloop: one 128 x 128 output tile per CTA, K streamed in blocks of 32 floats (one 128-byte swizzle row)
// through a 3-stage ring.  Thread 0 of warpgroup 0 is the TMA producer: per k-block it waits for the stage's `empty`
// barrier, arms its `full` barrier for the A and B tiles (16 KB each, 128 rows x 128 bytes, SWIZZLE_128B) and has the
// kernel's functor issue the copies.  Warpgroups 1 and 2 are the consumers, rows 0-63 / 64-127 of the tile (the A tile's
// 64-row half starts 8 KB further): per stage they wait on `full`, issue 4 wgmma m64n128k8 into a 64 x 128 register
// accumulator and commit; the stage's MMAs stay in flight while the previous stage, now complete (wait_group 1), goes
// back to the producer (`empty` counts one arrival per consumer warpgroup).
//
// SPLIT (3xTF32, float32-grade products from float32 operands): a second ring holds lo = x - trunc_tf32(x) of every
// landed A and B tile, and each k-step issues three MMAs, hi.hi + hi.lo + lo.hi, into a k-block partial that is added
// to the accumulator in float32 (see the consumer loop).  The landed tile itself is the hi operand: wgmma .tf32 reads
// only the top 19 bits of a float32, i.e. trunc_tf32(x).  lo is exact
// in float32 (x and trunc_tf32(x) share sign and exponent), |lo| < 2^-10 |x|, and the tensor core's truncation of lo to
// tf32 loses less than 2^-20 |x|.  Where x - trunc_tf32(x) is 0 (x is a tf32 value) or NaN (x = +-Inf), lo = x 2^-24
// instead: a same-signed stand-in 2^-24 |x| away from the exact 0, inside the 2^-20 |x| above.  Then no correction
// product is Inf * 0 or Inf - Inf where the float32 product is +-Inf, and Inf and NaN reach the sum as they do on the
// SIMT kernel.  Per product the dropped lo.lo term and the two truncated lo operands stay below 3 2^-20 |a||b|.  The
// split is element-wise, so it uses the landed tile's swizzled offsets and the MMA descriptors of both rings are the same.
// Warps 1-3 of warpgroup 0 split: per k-block they wait on `full`, write lo, fence the generic-proxy stores against the
// async proxy the MMAs read through (fence.proxy.async), and arrive on the stage's `split` barrier (one arrival per
// splitter thread); the consumers wait on `split` instead of `full`.  The lo slots of stage s are free when `full(s)`
// completes: the producer re-arms it only after both consumers released the stage's previous MMAs on `empty(s)`.
namespace tf32 {

constexpr int kBM = 128, kBN = 128, kBK = 32, kStages = 3;
constexpr uint32_t kTileBytes = kBM * kBK * 4;                      // 16 KB
constexpr int kThreads = 384;                                       // warpgroup 0: producer; 1, 2: MMA + epilogue
constexpr size_t kSmemBytes = 2 * kStages * kTileBytes + 1024 + 64; // A and B rings, 1024-byte round-up, barriers
constexpr int kSplitters = 96;                                      // SPLIT: warps 1-3 of warpgroup 0
constexpr size_t kSplitSmemBytes = 4 * kStages * kTileBytes + 1024 + 128;   // + the A_lo and B_lo rings and `split` barriers
static_assert(kSplitSmemBytes <= 227 * 1024, "the split ring must fit the 227 KB of shared memory an H100 block may use");

// lo = x - trunc_tf32(x); x 2^-24 where that is 0 or NaN (see above)
__device__ __forceinline__ float tf32_lo(float x) {
  const float lo = x - __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
  return fabsf(lo) > 0.f ? lo : x * 0x1p-24f;   // false for 0 and for NaN (x = +-Inf, or x NaN)
}

// issue(sA, sB, bar) loads the next k-block's A and B tiles to shared addresses sA, sB, completing on bar; it is called
// by the producer thread only, nk times, in order.  Returns false in warpgroup 0, true in the consumer warpgroups,
// whose acc then holds the finished accumulator.
template <uint32_t KERNEL, bool SPLIT = false, class Issue>
__device__ __forceinline__ bool mainloop(const CUtensorMap* tmA, const CUtensorMap* tmB, int nk, int* err, float (&acc)[64],
                                         Issue&& issue) {
  extern __shared__ unsigned char smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;      // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t sA = base, sB = base + kStages * kTileBytes;
  constexpr uint32_t kLo = 2 * kStages * kTileBytes;                // SPLIT: A_lo / B_lo slot = hi slot + kLo
  // full[kStages], empty[kStages] (SPLIT: then split[kStages])
  const uint32_t bars = sB + kStages * kTileBytes + (SPLIT ? kLo : 0u);
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmA)) : "memory");   // descriptor fetch off the first load's path
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmB)) : "memory");
    for (int s = 0; s < kStages; ++s) {
      mbar_init(bars + 8u * s, 1); mbar_init(bars + 8u * (kStages + s), 2);
      if constexpr (SPLIT) mbar_init(bars + 8u * (2 * kStages + s), kSplitters);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (t == 0) {
      for (int j = 0; j < nk; ++j) {
        const int s = j % kStages;
        mbar_wait<KERNEL>(bars + 8u * (kStages + s), (((uint32_t)(j / kStages)) & 1u) ^ 1u, err);
        mbar_arrive_expect_tx(bars + 8u * s, 2 * kTileBytes);
        issue(sA + s * kTileBytes, sB + s * kTileBytes, bars + 8u * s);
      }
    } else if constexpr (SPLIT) {
      if (t >= 32) {
        const int i0 = t - 32;
        for (int j = 0; j < nk; ++j) {
          const int s = j % kStages;
          mbar_wait<KERNEL>(bars + 8u * s, ((uint32_t)(j / kStages)) & 1u, err);
          // the stage's A slot, then its B slot kStages slots further: the same loop covers both (2 x 1024 float4)
          for (int i = i0; i < 2 * (int)(kTileBytes / 16); i += kSplitters) {
            const uint32_t off = s * kTileBytes + (i >= (int)(kTileBytes / 16) ? kStages * kTileBytes - kTileBytes : 0u) + 16u * i;
            const float4* src = reinterpret_cast<const float4*>(smem_raw + (sA + off - smem_u32(smem_raw)));
            float4* dst = reinterpret_cast<float4*>(smem_raw + (sA + kLo + off - smem_u32(smem_raw)));
            const float4 v = *src;
            *dst = make_float4(tf32_lo(v.x), tf32_lo(v.y), tf32_lo(v.z), tf32_lo(v.w));
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the MMAs read lo through the async proxy
          mbar_arrive(bars + 8u * (2 * kStages + s));
        }
      }
    }
    return false;
  }
  const uint32_t a_off = (uint32_t)(wg - 1) * 64u * 128u;
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  if constexpr (SPLIT) {
    // The tensor core's accumulator truncates, once per MMA.  Three MMAs per k-step into one running sum would truncate
    // it 3 ceil(K/8) times, a loss that leans towards zero; instead each k-block's 12 MMAs go to a fresh partial `blk`
    // that is added to acc in float32 (rounded to nearest).  That add needs the block's MMAs complete (wait_group 0),
    // so the stage goes back to the producer right away; the other consumer warpgroup keeps the tensor core busy.
    float blk[64];
    for (int j = 0; j < nk; ++j) {
      const int s = j % kStages;
      mbar_wait<KERNEL>(bars + 8u * (2 * kStages + s), ((uint32_t)(j / kStages)) & 1u, err);
      gmma::fence();
#pragma unroll
      for (int k4 = 0; k4 < kBK / 8; ++k4) {
        const uint32_t a = sA + s * kTileBytes + a_off + k4 * 32, b = sB + s * kTileBytes + k4 * 32;
        gmma::mma_tf32_n128(blk, gmma::desc_sw128(a), gmma::desc_sw128(b), k4 > 0 ? 1 : 0);
        gmma::mma_tf32_n128(blk, gmma::desc_sw128(a), gmma::desc_sw128(b + kLo), 1);
        gmma::mma_tf32_n128(blk, gmma::desc_sw128(a + kLo), gmma::desc_sw128(b), 1);
      }
      gmma::commit();
      gmma::wait<0>();
      gmma::fence_regs(blk);
      if (t == 0) mbar_arrive(bars + 8u * (kStages + s));
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] += blk[i];
    }
    return true;
  }
  for (int j = 0; j < nk; ++j) {
    const int s = j % kStages;
    mbar_wait<KERNEL>(bars + 8u * s, ((uint32_t)(j / kStages)) & 1u, err);
    gmma::fence();
#pragma unroll
    for (int k4 = 0; k4 < kBK / 8; ++k4)     // +32 bytes per k-step of 8 floats inside the swizzle row
      gmma::mma_tf32_n128(acc, gmma::desc_sw128(sA + s * kTileBytes + a_off + k4 * 32), gmma::desc_sw128(sB + s * kTileBytes + k4 * 32),
                          (j > 0 || k4 > 0) ? 1 : 0);
    gmma::commit();
    gmma::wait<1>();
    if (t == 0 && j > 0) mbar_arrive(bars + 8u * (kStages + (j - 1) % kStages));
  }
  gmma::wait<0>();
  gmma::fence_regs(acc);
  return true;
}

}  // namespace tf32
}  // namespace srf
