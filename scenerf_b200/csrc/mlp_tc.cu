// Fused point-MLP on Hopper tensor cores (sm_90a): one persistent kernel does, per 64-row tile, projection -> integer
// sphere coords -> positional encoding -> 5-scale bilinear gather -> the whole ResnetFC (lin_in, 3 x [lin_z, fc_0, fc_1],
// lin_out) with wgmma (fp16 operands, fp32 accumulators in registers).  The (N x 2522) x_in matrix of the reference
// (scenerf/models/scenerf.py:527-531) and all hidden activations never touch HBM: gathered features / activations are
// produced straight into 128B-swizzled shared-memory A tiles, weights are streamed as pre-swizzled stage images by
// cp.async.bulk (TMA engine) through an mbarrier ring.
//
// Reference computed here: scenerf.py:505-531 (predict up to mlp(x_in)), resnetfc.py:54-63,133-164.
//
// Tile program (A chunk = 64 rows x 64 k, fp16, K-major SW128; each A chunk meets the 128 x 64 weight images of the
// warpgroup's two N-quarters):
//   L0  lin_in   1 chunk   fresh   ACC  = x Win^T
//   L1  lin_z0   KZ chunks acc     ACC += z Wz0^T                  -> E1: h = ACC + c0            ; A = relu(h)
//   L2  fc_0     8 chunks  fresh   ACC  = relu(h) W0^T             -> E2: net = ACC + b0          ; A = relu(net)
//   L3  fc_1     8 chunks  fresh   ACC  = relu(net) W1^T
//   L4  lin_z1   KZ        acc     ACC += z Wz1^T                  -> E1: h = h + ACC + c1 ...
//   ... (blocks 1, 2) ...
//   L9  fc_1     8         fresh                                   -> E3: h = h + ACC + b1_2      ; A = relu(h)
//   L10 lin_out  8 (N=16)  fresh   ACC[:, :16] = relu(h) Wout^T    -> E4: out = ACC + bout
// Biases are folded into the epilogues as cumulative vectors c_b.
//
// Threads: two warpgroups (256 threads, 1 CTA / SM).  Warpgroup g owns output columns [256 g, 256 g + 256) of every
// 512-wide layer as two 64 x 128 register accumulators (wgmma m64n128k16), streams ITS weight images through its own
// ring (one thread issues the bulk copies, running a ring's depth ahead of its MMAs), and runs the epilogues of its
// columns from registers.  Both warpgroups produce the shared A tiles together: geometry, positional encoding, the
// latent gather (overlapping the MMAs of the previous latent chunk) and the activations written by the epilogues.
// The fp32 hidden state h (64 x 512) does not fit next to the accumulators: it lives in a per-CTA scratch that stays
// L2-resident, in the accumulator's register order (each thread reads back exactly what it wrote).
//
// Split (fp32-grade) mode: every fp32 operand x is carried as fp16 hi = rn(x) and lo = rn(x - hi), and the split is
// carried along K: a tile holds 64 points, every A chunk exists twice (A_hi, A_lo: 64 rows each), every weight image
// is followed by the image of its low parts, and each image meets both A parts, all into the same registers:
//   D = A_hi W_hi^T + A_lo W_hi^T + A_hi W_lo^T + A_lo W_lo^T
// So each 16 KB image streamed from L2 serves 64 points (the weight stream bounds this kernel), and the epilogue
// finishes its rows as in fp16 mode.  The ring holds 3 single-image slots per warpgroup; the x chunk and the latent
// double buffer live in activation chunks that are idle while they are used (Smem<true>, zpass).  Each fc layer sums
// its K in two halves (flush), which keeps the accumulation round-off at the level of two MMAs per k-step.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include "kernels.cuh"
#include "tma.cuh"

namespace srf {
namespace tc {

constexpr int kTileM = 64;                        // MMA rows = points per tile (both modes)
constexpr int kChunkK = 64;                       // fp16 elements per A/B row = 128 bytes = one SW128 atom row
constexpr int kAChunkBytes = kTileM * 128;        // 8 KB: one A chunk (split mode: one part of it)
constexpr int kBRows = 128, kBSlotBytes = kBRows * 128;   // one weight image: 128 rows (N) x 64 k = 16 KB
constexpr int kHiddenChunks = kHidden / kChunkK;  // 8
constexpr int kQuarters = kHidden / kBRows;       // 4 N-quarters of 128
constexpr int kOutN = 16;                         // lin_out padded to N = 16
constexpr int kOutImgBytes = kOutN * 128;         // 2 KB
constexpr int kThreads = 256;                     // two warpgroups
constexpr int kNumBias = 8;                       // c0,c1,c2, b_fc0[0..2], b_fc1_2, b_out(padded)
constexpr size_t kHeaderBytes = (size_t)kNumBias * kHidden * sizeof(float);   // 16 KB
constexpr int kNumLayers = 11;
// split-mode blobs: the power-of-two weight scale 2^s and its inverse live in unused entries of the b_out header row
constexpr int kScaleSlot = 7 * kHidden + 256, kInvScaleSlot = 7 * kHidden + 257;
// per-CTA scratch (floats): the fp32 hidden state (2 warpgroups x 2 quarters x 64 registers x 128 threads), then, in
// split mode, the partial sums of the first half of an fc layer's K loop (same layout; see flush)
constexpr size_t kScratchFloats = (size_t)2 * kTileM * kHidden;   // 256 KB per CTA

// dynamic shared memory carve-up, per mode.  An A chunk is 64 rows x 64 k; in split mode it is the 8 KB of high parts
// followed by the 8 KB of low parts, so row r of the low part is row r + 64 of the chunk.
template <bool SPLIT>
struct Smem {
  static constexpr int kParts = SPLIT ? 2 : 1;
  static constexpr int kAStride = kParts * kAChunkBytes;                      // bytes per A chunk (hi + lo)
  static constexpr int kAct = 0;                                              // 8 A chunks: activations of the current layer
  // x chunk (positional encoding | view direction) and the latent double buffer.  fp16: regions of their own.  split:
  // aliases of activation chunks 0 and 1-2, which no MMA reads while they are in use (see zpass)
  static constexpr int kX = SPLIT ? kAct : kAct + kHiddenChunks * kAStride;
  static constexpr int kZ = SPLIT ? kAct + kAStride : kX + kAStride;
  static constexpr int kSlots = SPLIT ? 3 : 4;                                // per warpgroup, one 16 KB weight image each
  static constexpr int kRingBytes = kSlots * kBSlotBytes;
  static constexpr int kRing = SPLIT ? kAct + kHiddenChunks * kAStride : kZ + 2 * kAStride;
  static constexpr int kBar = kRing + 2 * kRingBytes;                         // full[2][4]
  static constexpr int kSph = kBar + 2 * 4 * 8;                               // short2 (sx,sy) per point
  static constexpr int kMask = kSph + kTileM * 4;                             // active latent chunks of the tile
  static constexpr int kTotal = kMask + 16;
};
// the fp16 carve-up: 64 KB activations, 8 KB x, 16 KB latents, 2 x 64 KB rings
static_assert(Smem<false>::kRing == 88 * 1024 && Smem<false>::kTotal + 1024 <= 232448, "shared memory budget (fp16)");
// split: 128 KB activations (x and latents inside), 2 x 48 KB rings.  The latent buffers stay clear of the x chunk
// (lin_in's last MMAs may still read it when lin_z0's first gather starts) and of activation chunk 7 (fc_1's last)
using SmemSplit = Smem<true>;
static_assert(SmemSplit::kRing == 128 * 1024 && SmemSplit::kTotal + 1024 <= 232448, "shared memory budget (split)");
static_assert(SmemSplit::kZ >= SmemSplit::kX + SmemSplit::kAStride &&
              SmemSplit::kZ + 2 * SmemSplit::kAStride <= SmemSplit::kAct + 7 * SmemSplit::kAStride, "split latent buffers");

struct Layer { int chunks_is_kz, chunks, fresh, signal, is_out; };
// chunks_is_kz: number of chunks = KZ (runtime) instead of `chunks`
__constant__ Layer kLayers[kNumLayers] = {
    {0, 1, 1, 0, 0}, {1, 0, 0, 1, 0},                       // lin_in, lin_z0
    {0, 8, 1, 1, 0}, {0, 8, 1, 0, 0}, {1, 0, 0, 1, 0},      // fc0_0, fc1_0, lin_z1
    {0, 8, 1, 1, 0}, {0, 8, 1, 0, 0}, {1, 0, 0, 1, 0},      // fc0_1, fc1_1, lin_z2
    {0, 8, 1, 1, 0}, {0, 8, 1, 1, 0},                       // fc0_2, fc1_2
    {0, 8, 1, 1, 1}};                                       // lin_out

struct KernelArgs {
  const float* pts;        // (n,3)
  const float* viewdir;    // (n/n_per,3)
  int n, n_per, n_tiles, kz;
  const unsigned char* wblob;   // header (biases) + stage images
  float* scratch;          // gridDim.x * kScratchFloats
  float* raw_out;          // (n, d_out)
  int d_out;
  int32_t* dbg_sphere;     // (n,2) or null
  int skip_zero;           // SRF_FLAG_SKIP_ZERO_CHUNKS
  int hidden_fp16;         // SRF_FLAG_HIDDEN_FP16: the hidden state travels between blocks as fp16
  const unsigned char* preproj;  // pre-projected latent table (preproj.cu) or null: rows of 3 x 512 values (fp16 in fp16 mode, fp32 in
                                 // split mode); when set, the lin_z GEMMs are not executed and E1 adds the row of the point's sphere pixel
  int pre_W1, pre_H1;      // sphere_W + 1, sphere_H + 1: row = sy * pre_W1 + sx inside, pre_W1 * pre_H1 (the zero row) outside
  int debug_layer;         // -1, or: stop every tile after this layer's ACC is complete and dump it
  float* debug_acc;        // (n_tiles*64, 512)
  int* error_flag;         // set to non-zero by the watchdog
};

// ---------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// The 2 x 10.9 MB of weight images are re-read by every CTA for every tile while the feature pyramid streams through
// L2 once per frame: ask L2 to keep the weights (evict_last) so that the stream sees L2-hit latency.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
               ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar), "l"(policy)
               : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t a) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(a) : "memory");
}
// {relu(lo), relu(hi)} -> packed fp16x2 in one instruction (the ReLU of the reference rides on the conversion)
__device__ __forceinline__ uint32_t pack_relu_half2(float lo, float hi) {
  uint32_t d;
  asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
  return d;
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}
// split mode: (a, b) -> packed fp16 high parts rn(x) and packed low parts rn(x - rn(x)); hi + lo carries 22 mantissa
// bits (the low part goes subnormal below |x| ~ 2^-3, absolute error <= 2^-25 there)
__device__ __forceinline__ void split_half2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// byte offset of (row, 16-byte granule g) inside a 128B-swizzled K-major tile whose rows are 128 bytes
__device__ __forceinline__ uint32_t sw128_offset(int row, int g) { return (uint32_t)(row * 128 + ((g ^ (row & 7)) << 4)); }

__device__ __forceinline__ int layer_chunks(int l, int kz) { return kLayers[l].chunks_is_kz ? kz : kLayers[l].chunks; }
// chunk c of a lin_z layer is active for this tile?  (mask bit c; all ones when skipping is off)
__device__ __forceinline__ bool chunk_active(int l, int c, uint64_t mask) { return !kLayers[l].chunks_is_kz || ((mask >> c) & 1ull); }

// which pyramid scales touch K-chunk c (channels [64c, 64c+64))
__device__ __forceinline__ uint64_t chunk_mask_for_scales(const DevParams& p, uint32_t scale_bits, int kz) {
  uint64_t m = 0;
  for (int c = 0; c < kz; ++c) {
    const int lo = c * kChunkK, hi = lo + kChunkK;
    for (int s = 0; s < kScales; ++s)
      if (((scale_bits >> s) & 1u) && p.ch_off[s] < hi && p.ch_off[s + 1] > lo) m |= 1ull << c;
  }
  return m;
}

// byte offset of the first image of chunk k of layer l inside the image region of the blob
//   parts = 1 (fp16 images) or 2 (split mode: every image is followed by the image of the fp16 low parts)
__device__ __forceinline__ size_t chunk_image_offset(int l, int k, int kz, int parts) {
  size_t off = 0;
  for (int i = 0; i < l; ++i) off += (size_t)layer_chunks(i, kz) * (kLayers[i].is_out ? kOutImgBytes : kQuarters * kBSlotBytes);
  return (off + (size_t)k * (kLayers[l].is_out ? kOutImgBytes : kQuarters * kBSlotBytes)) * (size_t)parts;
}

// ---------------------------------------------------------------------------------------------------------------
// Weight stream of one warpgroup.  A stage ("slot") is, for a 512-wide layer, one 16 KB image of chunk k: in fp16 mode
// that of one of the warpgroup's two N-quarters, in split mode the hi or the lo image of one of them (slot j = 2 q +
// part, the blob's order); for lin_out, the 16 x 64 image(s) of chunk k (hi + lo, 4 KB, in split mode; warpgroup 0
// only).  The order is the tile program's order; lin_z chunks not in the tile's mask are skipped.
// ---------------------------------------------------------------------------------------------------------------
template <int kWideSlots>      // slots per chunk of a 512-wide layer: 2 (fp16) or 4 (split)
struct Cursor {
  int l = 0, k = 0, j = 0;
  // move to the first slot at or after (l, k, j) that exists; false when the tile's stream is exhausted
  __device__ __forceinline__ bool normalize(int kz, uint64_t mask, int last_layer, int wg) {
    while (l <= last_layer) {
      if (l == kNumLayers - 1 && wg != 0) return false;
      if (j >= (kLayers[l].is_out ? 1 : kWideSlots)) { j = 0; ++k; }
      if (k >= layer_chunks(l, kz)) { k = 0; ++l; continue; }
      if (!chunk_active(l, k, mask)) { ++k; continue; }
      return true;
    }
    return false;
  }
};

// next active latent chunk of lin_z layer l after chunk c (-1: none)
__device__ __forceinline__ int next_active(int kz, uint64_t mask, int c) {
  for (++c; c < kz; ++c)
    if ((mask >> c) & 1ull) return c;
  return -1;
}

// ---------------------------------------------------------------------------------------------------------------
// The kernel
// ---------------------------------------------------------------------------------------------------------------
// PRE: the latent-table variant (a.preproj set): no lin_z chunk exists in the tile program and the E1 epilogues add table rows.
template <bool H16, bool SPLIT, bool PRE>
__global__ void __launch_bounds__(kThreads, 1)
point_mlp_tc_kernel(const __grid_constant__ DevParams p, const __grid_constant__ KernelArgs a) {
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  // SWIZZLE_128B tiles need 1024-byte alignment; the launch reserves 1 KB of slack for this round-up
  unsigned char* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  const uint32_t smem_base = smem_u32(smem);
  const int tid = threadIdx.x;
  const int wg = tid >> 7, t = tid & 127, w = t >> 5, lane = tid & 31;
  using L = Smem<SPLIT>;
  constexpr int kParts = L::kParts;                     // weight images per (chunk, quarter) and A parts: hi (+ lo)
  constexpr int kPts = kTileM;                          // points per tile
  constexpr int kWideSlots = 2 * kParts;                // ring slots per chunk of a 512-wide layer
  constexpr int kSlots = L::kSlots;                     // 4 (fp16) or 3 (split)
  constexpr int kAStride = L::kAStride;
  constexpr int kSmemAct = L::kAct, kSmemX = L::kX, kSmemZ = L::kZ;
  const uint32_t ring = smem_base + L::kRing + (uint32_t)wg * L::kRingBytes;
  auto full_bar = [&](int s) { return smem_base + L::kBar + 8u * (uint32_t)(wg * 4 + s); };
  short2* sph_smem = reinterpret_cast<short2*>(smem + L::kSph);
  volatile unsigned long long* mask_smem = reinterpret_cast<volatile unsigned long long*>(smem + L::kMask);

  if (tid == 0) {
    for (int s = 0; s < 8; ++s) mbar_init(smem_base + L::kBar + 8u * s, 1);
    fence_barrier_init();
  }
  __syncthreads();

  const int kz = a.kz;
  const int last_layer = (a.debug_layer >= 0) ? a.debug_layer : (kNumLayers - 1);
  const unsigned char* images = a.wblob + kHeaderBytes;
  const float* bias = reinterpret_cast<const float*>(a.wblob);
  float* scratch = a.scratch + (size_t)blockIdx.x * kScratchFloats;
  float* hbuf = scratch + (size_t)wg * (2 * 64 * 128);             // [j][reg][thread] of this warpgroup
  [[maybe_unused]] float* pbuf = scratch + (size_t)(2 + wg) * (2 * 64 * 128);       // split: first-half partial sums, same order
  const uint64_t policy = l2_policy_evict_last();

  // ---- weight stream: producer (thread 0 of the warpgroup) and consumer positions -----------------------------
  Cursor<kWideSlots> pc;
  bool p_live = false;
  uint32_t ppos = 0, cpos = 0, done = 0;                // slots issued / consumed / known complete (whole kernel)
  uint64_t mask = 0;
  auto produce = [&]() {
    if (t != 0) return;
    while (p_live && ppos < done + (uint32_t)kSlots) {
      const bool is_out = kLayers[pc.l].is_out != 0;
      const unsigned char* src = images + chunk_image_offset(pc.l, pc.k, kz, kParts) + (is_out ? 0 : (size_t)(kWideSlots * wg + pc.j) * kBSlotBytes);
      const uint32_t bytes = is_out ? (uint32_t)(kOutImgBytes * kParts) : (uint32_t)kBSlotBytes;
      const int s = (int)(ppos % kSlots);
      mbar_arrive_expect_tx(full_bar(s), bytes);
      bulk_g2s(ring + (uint32_t)s * kBSlotBytes, src, bytes, full_bar(s), policy);
      ++ppos;
      ++pc.j;
      p_live = pc.normalize(kz, mask, last_layer, wg);
    }
  };
  float acc0[64], acc1[64], acco[8];
  // wait for the next slot and issue its MMAs: A chunk at a_addr, 4 k-steps of 16 (x hi/lo parts in split mode)
  auto wait_slot = [&]() -> uint32_t {
    const int s = (int)(cpos % kSlots);
    mbar_wait<kWatchPointMlp>(full_bar(s), (cpos / kSlots) & 1u, a.error_flag);
    return ring + (uint32_t)s * kBSlotBytes;
  };
  // all but the newest commit group have completed: their slots are refilled (one commit group per slot)
  auto release1 = [&]() {
    gmma::wait<1>();
    done = cpos - 1;
    produce();
  };
  // split mode: one weight image (hi or lo part of W) against both parts of the A chunk, into the same registers;
  // over the image pair of a quarter this is A_hi W_hi + A_lo W_hi + A_hi W_lo + A_lo W_lo.  One slot, one commit group.
  auto mma_image = [&](float (&acc)[64], uint64_t ad_hi, uint64_t ad_lo, bool fresh) __attribute__((always_inline)) {
    const uint64_t bd = gmma::desc_sw128(wait_slot());
    gmma::fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      gmma::mma_f16_n128(acc, ad_hi + 2 * k, bd + 2 * k, (fresh && k == 0) ? 0 : 1);
      gmma::mma_f16_n128(acc, ad_lo + 2 * k, bd + 2 * k, 1);
    }
    gmma::commit();
    ++cpos;
  };
  auto mma_pair = [&](uint32_t a_addr, bool fresh) {          // both quarters of the warpgroup: 2 slots, 2 commit groups (split: 4, 4)
    const uint64_t ad = gmma::desc_sw128(a_addr);
    if constexpr (SPLIT) {
      const uint64_t ad_lo = gmma::desc_sw128(a_addr + kAChunkBytes);
      mma_image(acc0, ad, ad_lo, fresh);
      release1();
      mma_image(acc0, ad, ad_lo, false);
      release1();
      mma_image(acc1, ad, ad_lo, fresh);
      release1();
      mma_image(acc1, ad, ad_lo, false);
    } else {
      {
        const uint32_t b = wait_slot();
        gmma::fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) gmma::mma_f16_n128(acc0, ad + 2 * k, gmma::desc_sw128(b) + 2 * k, (fresh && k == 0) ? 0 : 1);
        gmma::commit();
        ++cpos;
      }
      release1();
      {
        const uint32_t b = wait_slot();
        gmma::fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) gmma::mma_f16_n128(acc1, ad + 2 * k, gmma::desc_sw128(b) + 2 * k, (fresh && k == 0) ? 0 : 1);
        gmma::commit();
        ++cpos;
      }
    }
  };
  // lin_out: one slot (split mode: the hi and lo images, each against both A parts)
  auto mma_out = [&](uint32_t a_addr, bool fresh) {
    const uint64_t ad = gmma::desc_sw128(a_addr);
    [[maybe_unused]] const uint64_t ad_lo = gmma::desc_sw128(a_addr + kAChunkBytes);
    const uint32_t b = wait_slot();
    gmma::fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int part = 0; part < kParts; ++part) {
        const uint64_t bd = gmma::desc_sw128(b + part * kOutImgBytes) + 2 * k;
        gmma::mma_f16_n16(acco, ad + 2 * k, bd, (fresh && k == 0 && part == 0) ? 0 : 1);
        if constexpr (SPLIT) gmma::mma_f16_n16(acco, ad_lo + 2 * k, bd, 1);
      }
    gmma::commit();
    ++cpos;
  };
  auto retire1 = release1;
  // every commit group has completed: the accumulators may be read
  auto retire0 = [&]() {
    gmma::wait<0>();
    gmma::fence_regs(acc0); gmma::fence_regs(acc1); gmma::fence_regs(acco);
    done = cpos;
    produce();
  };
  auto sync_all = [&]() { named_bar_sync(1, kThreads); };
  // split mode: every MMA rounds its sum into the accumulator, and the four products per k-step put twice as many
  // MMAs on one accumulator as the 32-point row layout did (about sqrt(2) more round-off, measured layer by layer).
  // Each fc layer therefore sums its K in two halves: after chunk 3 the accumulators go to pbuf and restart from
  // zero; the epilogue adds the two halves.
  auto flush = [&]() {
    retire0();
#pragma unroll
    for (int i2 = 0; i2 < 32; ++i2) {
      reinterpret_cast<float2*>(pbuf)[(size_t)i2 * 128 + t] = make_float2(acc0[2 * i2], acc0[2 * i2 + 1]);
      reinterpret_cast<float2*>(pbuf)[(size_t)(32 + i2) * 128 + t] = make_float2(acc1[2 * i2], acc1[2 * i2 + 1]);
    }
#pragma unroll
    for (int i = 0; i < 64; ++i) { acc0[i] = 0.0f; acc1[i] = 0.0f; }
  };

  const short2* sph_cur = sph_smem;
  const int erow0 = 16 * w + (lane >> 2);                // accumulator rows of this thread: erow0, erow0 + 8
  const int ecol = 2 * (lane & 3);                       // + 8 c8 (+ 128 j + 256 wg)

  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    const int row0 = tile * kPts;
    // ---------------- front-end: geometry of the tile's points ---------------------------------------------------
    if (tid == 0) mask_smem[0] = 0ull;
    sync_all();
    {
      uint32_t my_scales = 0;
      if (tid < kPts) {
        const int gi = row0 + tid;
        int sx = kSphereInvalid, sy = kSphereInvalid;
        if (gi < a.n) {
          point_to_sphere(p, a.pts[(size_t)gi * 3 + 0], a.pts[(size_t)gi * 3 + 1], a.pts[(size_t)gi * 3 + 2], sx, sy);
          if (a.dbg_sphere) { a.dbg_sphere[(size_t)gi * 2 + 0] = sx; a.dbg_sphere[(size_t)gi * 2 + 1] = sy; }
        }
        // 16-bit storage: anything beyond +-32767 can only address zero padding (sphere grids are <= 16384 wide)
        sph_smem[tid] = make_short2((short)max(min(sx, 32767), -32768), (short)max(min(sy, 32767), -32768));
        if (a.skip_zero) {
#pragma unroll
          for (int s = 0; s < kScales; ++s) my_scales |= scale_taps(p, s, sx, sy).any ? (1u << s) : 0u;
        }
      }
      if (a.skip_zero && tid < ((kPts + 31) & ~31)) {
        const uint32_t wbits = __reduce_or_sync(0xffffffffu, my_scales);
        if (lane == 0) {
          const unsigned long long bits = chunk_mask_for_scales(p, wbits, kz);
          if (bits) atomicOr((unsigned long long*)mask_smem, bits);
        }
      }
    }
    sync_all();
    mask = PRE ? 0ull : (a.skip_zero ? mask_smem[0] : ~0ull);
    // weight stream of this tile: prime the ring (every slot of the previous tile has completed)
    pc = Cursor<kWideSlots>();
    p_live = pc.normalize(kz, mask, last_layer, wg);
    produce();

    // pre-projected latents: table rows of the two points whose accumulator rows this thread finishes
    const unsigned char* pre_row[2] = {nullptr, nullptr};
    if constexpr (PRE) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const short2 sp = sph_cur[(erow0 + 8 * hh) % kPts];
        const bool in = sp.x >= 0 && sp.x < a.pre_W1 && sp.y >= 0 && sp.y < a.pre_H1;
        const size_t ridx = in ? (size_t)sp.y * a.pre_W1 + sp.x : (size_t)a.pre_W1 * a.pre_H1;
        pre_row[hh] = a.preproj + ridx * (size_t)(SRF_NUM_BLOCKS * kHidden * (SPLIT ? 4 : 2));
      }
    }

    // ---------------- x chunk = [pe(39) | viewdir(3) | 0] as fp16 ----------------------------------------------------
    if (tid < 2 * kPts) {
      // two threads per point: thread tid < kPts writes granules 0-2 (x,y,z + the first 21 encodings), the other
      // granules 3-7 (the other 15 encodings, the view direction, zero padding)
      const bool first = tid < kPts;
      const int xrow = first ? tid : tid - kPts;
      const int gi = row0 + xrow;
      const uint32_t slot_addr = smem_base + kSmemX;
      float qx = 0.f, qy = 0.f, qz = 0.f;
      if (gi < a.n) { qx = a.pts[(size_t)gi * 3 + 0]; qy = a.pts[(size_t)gi * 3 + 1]; qz = a.pts[(size_t)gi * 3 + 2]; }
      const float kPi = 3.14159274101257324f, kHalfPi = 1.57079637050628662f;
      auto sel3 = [](int i, float v0, float v1, float v2) { return i == 0 ? v0 : (i == 1 ? v1 : v2); };   // no indexed register arrays
      // value of x_in index idx (0..63) for this row: pe.py:32-43 order, then viewdir, then zeros.  idx is a run-time value
      // (the granules are produced by a rolled loop, so the kernel holds 8 copies of sinf instead of 36)
      auto xval = [&](int idx, const float* vd) -> float {
        if (gi >= a.n) return 0.0f;
        if (idx < 3) return sel3(idx, qx, qy, qz);
        if (idx < 3 + 36) {
          const int j = idx - 3, fp = j / 3, cc = j - 3 * fp;    // fp = 2*k + phase
          float arg = fmul(sel3(cc, qx, qy, qz), kPi * (float)(1 << (fp >> 1)));    // pi * 2^k: exact scaling of the fp32 constant
          if (fp & 1) arg = fadd(kHalfPi, arg);
          return sinf(arg);
        }
        if (idx < kDX) return sel3(idx - 39, vd[0], vd[1], vd[2]);
        return 0.0f;
      };
      float vd[3] = {0.f, 0.f, 0.f};
      if (!first && gi < a.n) {
        const float* vp = a.viewdir + (size_t)(gi / a.n_per) * 3;
        vd[0] = vp[0]; vd[1] = vp[1]; vd[2] = vp[2];
      }
      const int g_end = first ? 3 : 8;
#pragma unroll 1
      for (int g = first ? 0 : 3; g < g_end; ++g) {
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = xval(8 * g + j, vd);
        if constexpr (SPLIT) {
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) split_half2(v[2 * j], v[2 * j + 1], hi[j], lo[j]);
          sts128(slot_addr + sw128_offset(xrow, g), hi[0], hi[1], hi[2], hi[3]);
          sts128(slot_addr + sw128_offset(xrow + kPts, g), lo[0], lo[1], lo[2], lo[3]);
        } else {
          sts128(slot_addr + sw128_offset(xrow, g), pack_half2(v[0], v[1]), pack_half2(v[2], v[3]), pack_half2(v[4], v[5]),
                 pack_half2(v[6], v[7]));
        }
      }
    }
    fence_proxy_async_smem();
    sync_all();

    // ---------------- latent gather: chunk c of z into an A chunk -------------------------------------------------
    // thread -> kItems items per chunk: points (tid/8) + 32*i, granule (8 channels = 16 B of fp16) g = tid % 8.
    // Per point only (element offset of the north-west tap, x/y fractional weights, 4 validity bits) is kept in
    // registers for the current scale; the 4 tap weights are re-derived (same products as scale_taps) per chunk.
    constexpr int kItems = kPts / 32;
    int cur_scale = -1;
    int t_off[kItems];          // offset of tap 0 (may be "virtual" when tap 0 itself is out of range)
    uint32_t t_ok[kItems];      // bit t = tap t in range
    float t_w[kItems], t_n[kItems];
    int dxo = 0, dyo = 0;       // element strides to the east / south tap
    auto gather = [&](int c, uint32_t zaddr) {
      const int g = tid & 7;
      const int ch = c * kChunkK + g * 8;                     // first of this thread's 8 channels
      auto emit_vals = [&](int row, const float (&v)[8]) {
        if constexpr (SPLIT) {
          uint32_t hi[4], lo[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) split_half2(v[2 * j], v[2 * j + 1], hi[j], lo[j]);
          sts128(zaddr + sw128_offset(row, g), hi[0], hi[1], hi[2], hi[3]);
          sts128(zaddr + sw128_offset(row + kPts, g), lo[0], lo[1], lo[2], lo[3]);
        } else {
          sts128(zaddr + sw128_offset(row, g), pack_half2(v[0], v[1]), pack_half2(v[2], v[3]), pack_half2(v[4], v[5]), pack_half2(v[6], v[7]));
        }
      };
      int s = -1;
#pragma unroll
      for (int i = 0; i < kScales; ++i)
        if (ch >= p.ch_off[i] && ch < p.ch_off[i + 1]) s = i;
      if (s >= 0 && s != cur_scale) {
        dxo = p.C[s]; dyo = p.W[s] * p.C[s];
#pragma unroll
        for (int i = 0; i < kItems; ++i) {
          const short2 sp16 = sph_cur[(tid >> 3) + 32 * i];
          const Taps tp = scale_taps(p, s, sp16.x, sp16.y);
          t_ok[i] = (tp.off[0] >= 0 ? 1u : 0u) | (tp.off[1] >= 0 ? 2u : 0u) | (tp.off[2] >= 0 ? 4u : 0u) | (tp.off[3] >= 0 ? 8u : 0u);
          // off[t] = off0 + (t&1)*dxo + (t>>1)*dyo for in-range taps -> recover off0 from any valid tap
          int o0 = 0;
          if (tp.off[0] >= 0) o0 = tp.off[0];
          else if (tp.off[1] >= 0) o0 = tp.off[1] - dxo;
          else if (tp.off[2] >= 0) o0 = tp.off[2] - dyo;
          else if (tp.off[3] >= 0) o0 = tp.off[3] - dxo - dyo;
          t_off[i] = o0;
          t_w[i] = tp.fx; t_n[i] = tp.fy;
        }
        cur_scale = s;
      }
      const char* fbytes = (s >= 0) ? reinterpret_cast<const char*>(p.feat[s]) : nullptr;
      const int ch_in = (s >= 0) ? ch - p.ch_off[s] : 0;
      const bool f16 = p.feat_fp16 != 0;
#pragma unroll
      for (int u = 0; u < kItems; ++u) {
        const int row = (tid >> 3) + 32 * u;
        float acc[8];
        const uint32_t ok = (s >= 0) ? t_ok[u] : 0u;
        if (!ok) {
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e] = 0.0f;
          emit_vals(row, acc);
          continue;
        }
        const float wx = t_w[u], ny = t_n[u];
        const float e_ = fsub(1.0f, wx), so = fsub(1.0f, ny);
        const float tw4[4] = {fmul(so, e_), fmul(so, wx), fmul(ny, e_), fmul(ny, wx)};     // nw, ne, sw, se
        float v[4][8];
#pragma unroll
        for (int tp = 0; tp < 4; ++tp) {
          if ((ok >> tp) & 1u) {
            const size_t eidx = (size_t)(ch_in + t_off[u] + (tp & 1) * dxo + (tp >> 1) * dyo);
            if (f16) {
              const uint4 raw = __ldg(reinterpret_cast<const uint4*>(fbytes + eidx * 2));
              const uint32_t rw[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&rw[q]));
                v[tp][2 * q] = f.x; v[tp][2 * q + 1] = f.y;
              }
            } else {
              const float4* src = reinterpret_cast<const float4*>(fbytes + eidx * 4);
              const float4 a0 = __ldg(src), a1 = __ldg(src + 1);
              v[tp][0] = a0.x; v[tp][1] = a0.y; v[tp][2] = a0.z; v[tp][3] = a0.w;
              v[tp][4] = a1.x; v[tp][5] = a1.y; v[tp][6] = a1.z; v[tp][7] = a1.w;
            }
          } else {
#pragma unroll
            for (int e = 0; e < 8; ++e) v[tp][e] = 0.0f;
          }
        }
        // out = ((v_nw*nw + v_ne*ne) + v_sw*sw) + v_se*se : separate roundings like ATen's CPU kernel
        // (an out-of-range tap contributes an exact +0)
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          acc[e] = fmul(v[0][e], tw4[0]);
#pragma unroll
          for (int tp = 1; tp < 4; ++tp) acc[e] = fadd(acc[e], fmul(v[tp][e], tw4[tp]));
        }
        emit_vals(row, acc);
      }
    };
    // one lin_z layer: the active chunks in order, chunk i+1 gathered while the MMAs of chunk i run
    auto zpass = [&]() {
      cur_scale = -1;
      int c = next_active(kz, mask, -1);
      if (c < 0) return;
      // split mode: the latent buffers are activation chunks 1-2.  Each warpgroup has retired all but its newest commit
      // group (chunk 7 of fc_1, or lin_in's x chunk); once both warpgroups are here no MMA reads chunks 1-2 any more
      if constexpr (SPLIT) sync_all();
      gather(c, smem_base + kSmemZ);
      fence_proxy_async_smem();
      sync_all();
      for (int zi = 0; c >= 0; ++zi) {
        const int cn = next_active(kz, mask, c);
        mma_pair(smem_base + kSmemZ + (uint32_t)(zi & 1) * kAStride, false);
        if (cn >= 0) gather(cn, smem_base + kSmemZ + (uint32_t)((zi + 1) & 1) * kAStride);
        retire0();
        fence_proxy_async_smem();
        sync_all();
        c = cn;
      }
    };

    // ---------------- epilogue of the warpgroup's 256 columns: registers -> [+bias (+h) (+table)] -> A = relu -------
    //   register i of accumulator j: row erow0 + 8 ((i/2) % 2), column 256 wg + 128 j + 8 (i/4) + ecol + (i % 2)
    //   h is kept in register order: element (j, i) of thread t at hbuf[(j * 64 + i) * 128 + t]
    auto epilogue = [&](auto use_h_c, auto write_h_c, auto use_p_c, int bias_idx) __attribute__((always_inline)) {
      constexpr bool USE_H = decltype(use_h_c)::value, WRITE_H = decltype(write_h_c)::value, USE_P = decltype(use_p_c)::value;
      // split: every epilogue but block 0's E1 (after lin_in + lin_z0) follows an fc layer, whose first half is in pbuf
      constexpr bool PART = SPLIT && (USE_H || !WRITE_H);
      [[maybe_unused]] const float inv_scale = SPLIT ? __ldg(bias + kInvScaleSlot) : 1.0f;
      // split mode: the row is passed through an opaque move so that the swizzled store addresses derived from it are
      // recomputed in every epilogue; held in registers across the tile (as the compiler would otherwise), they spill
      int erow = erow0;
      if constexpr (SPLIT) asm volatile("mov.b32 %0, %0;" : "+r"(erow));
      auto finish = [&](float (&acc)[64], int j) __attribute__((always_inline)) {
#pragma unroll
        for (int i2 = 0; i2 < 32; ++i2) {
          const int i = 2 * i2, hh = i2 & 1;
          const int row = erow + 8 * hh;
          const int col = 256 * wg + 128 * j + 8 * (i2 >> 1) + ecol;
          float r0 = acc[i], r1 = acc[i + 1];
          if constexpr (PART) {
            const float2 f = reinterpret_cast<const float2*>(pbuf)[(size_t)(j * 32 + i2) * 128 + t];
            r0 += f.x; r1 += f.y;
          }
          if constexpr (SPLIT) { r0 *= inv_scale; r1 *= inv_scale; }   // the four products are in units of 2^s
          if constexpr (!USE_P) {
            const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + (size_t)bias_idx * kHidden + col));
            r0 += bb.x; r1 += bb.y;
          }
          [[maybe_unused]] float2* hp = reinterpret_cast<float2*>(hbuf) + (size_t)(j * 32 + i2) * 128 + t;
          [[maybe_unused]] __half2* hp16 = reinterpret_cast<__half2*>(hbuf) + (size_t)(j * 32 + i2) * 128 + t;
          if constexpr (USE_H) {
            if constexpr (H16) { const float2 f = __half22float2(*hp16); r0 += f.x; r1 += f.y; }
            else { const float2 f = *hp; r0 += f.x; r1 += f.y; }
          }
          if constexpr (USE_P) {
            if constexpr (SPLIT) {
              const float2 f = __ldg(reinterpret_cast<const float2*>(pre_row[hh] + ((size_t)bias_idx * kHidden + col) * 4));
              r0 += f.x; r1 += f.y;
            } else {
              const float2 f = __half22float2(__ldg(reinterpret_cast<const __half2*>(pre_row[hh] + ((size_t)bias_idx * kHidden + col) * 2)));
              r0 += f.x; r1 += f.y;
            }
          }
          if constexpr (WRITE_H) {
            if constexpr (H16) *hp16 = __floats2half2_rn(r0, r1);
            else *hp = make_float2(r0, r1);
          }
          const uint32_t addr = smem_base + kSmemAct + (uint32_t)(col >> 6) * kAStride;
          const uint32_t inrow = (uint32_t)((((col & 63) >> 3) ^ (row & 7)) << 4) + (uint32_t)((col & 7) * 2);
          if constexpr (SPLIT) {
            uint32_t hi, lo;
            split_half2(fmaxf(r0, 0.0f), fmaxf(r1, 0.0f), hi, lo);
            sts32(addr + (uint32_t)row * 128 + inrow, hi);
            sts32(addr + (uint32_t)(row + kPts) * 128 + inrow, lo);     // row r of the low part
          } else {
            sts32(addr + (uint32_t)row * 128 + inrow, pack_relu_half2(r0, r1));
          }
        }
      };
      finish(acc0, 0);
      finish(acc1, 1);
    };
    // epilogue boundary: every MMA of both warpgroups that reads the A tile has completed before it is overwritten,
    // and the new tile is visible to the async proxy before the next layer's MMAs
    auto epi = [&](auto use_h_c, auto write_h_c, auto use_p_c, int bias_idx) __attribute__((always_inline)) {
      retire0();
      sync_all();
      epilogue(use_h_c, write_h_c, use_p_c, bias_idx);
      fence_proxy_async_smem();
      sync_all();
    };
    // debug: raw accumulator of the current layer.  fp16: row r of tile t to row 64 t + r.  split: the layout of the
    // former 32-point tiles (hi-part rows, then lo-part rows): point i to row 64 (i / 32) + i % 32, the complete
    // accumulator (all four products); the low rows stay as the caller left them.  Only points i < n are written.
    auto dump_acc = [&](bool out, bool part) {
      retire0();
      if (out && wg != 0) return;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float* dst;
        if constexpr (SPLIT) {
          const int gi = row0 + erow0 + 8 * hh;
          if (gi >= a.n) continue;
          dst = a.debug_acc + ((size_t)(gi >> 5) * 64 + (gi & 31)) * kHidden;
        } else {
          dst = a.debug_acc + ((size_t)tile * kTileM + erow0 + 8 * hh) * kHidden;
        }
        if (out) {
#pragma unroll
          for (int c8 = 0; c8 < 2; ++c8) { dst[8 * c8 + ecol] = acco[4 * c8 + 2 * hh]; dst[8 * c8 + ecol + 1] = acco[4 * c8 + 2 * hh + 1]; }
        } else {
#pragma unroll
          for (int c8 = 0; c8 < 16; ++c8) {
            const int col = 256 * wg + 8 * c8 + ecol;
            float v[4] = {acc0[4 * c8 + 2 * hh], acc0[4 * c8 + 2 * hh + 1], acc1[4 * c8 + 2 * hh], acc1[4 * c8 + 2 * hh + 1]};
            if constexpr (SPLIT) {
              if (part) {                      // the first half of the fc layer's K sum (flush)
                const int i2 = 2 * c8 + hh;
                const float2 p0 = reinterpret_cast<const float2*>(pbuf)[(size_t)i2 * 128 + t];
                const float2 p1 = reinterpret_cast<const float2*>(pbuf)[(size_t)(32 + i2) * 128 + t];
                v[0] += p0.x; v[1] += p0.y; v[2] += p1.x; v[3] += p1.y;
              }
            }
            dst[col] = v[0]; dst[col + 1] = v[1];
            dst[col + 128] = v[2]; dst[col + 129] = v[3];
          }
        }
      }
    };

    // ---------------- the tile program ---------------------------------------------------------------------------
    using T = std::true_type;
    using F = std::false_type;
    using P = std::integral_constant<bool, PRE>;
    mma_pair(smem_base + kSmemX, true);                           // lin_in
    retire1();
    if (!PRE) zpass();                                            // lin_z0
    if (a.debug_layer == 1) { dump_acc(false, false); continue; }
    bool stop = false;
    for (int b = 0; b < SRF_NUM_BLOCKS; ++b) {
      if (b == 0) epi(F{}, T{}, P{}, b);                          // E1 -> A = relu(h)
      else epi(T{}, T{}, P{}, b);
#pragma unroll 1
      for (int k = 0; k < kHiddenChunks; ++k) {                                                                         // fc_0
        mma_pair(smem_base + kSmemAct + (uint32_t)k * kAStride, k == 0);
        retire1();
        if (SPLIT && k == kHiddenChunks / 2 - 1) flush();
      }
      if (a.debug_layer == 2 + 3 * b) { dump_acc(false, true); stop = true; break; }
      epi(F{}, F{}, F{}, 3 + b);                                  // E2 -> A = relu(net)
#pragma unroll 1
      for (int k = 0; k < kHiddenChunks; ++k) {                                                                         // fc_1
        mma_pair(smem_base + kSmemAct + (uint32_t)k * kAStride, k == 0);
        retire1();
        if (SPLIT && k == kHiddenChunks / 2 - 1) flush();
      }
      if (b < SRF_NUM_BLOCKS - 1) {
        if (!PRE) zpass();                                        // lin_z(b+1) accumulates onto fc_1
        if (a.debug_layer == 4 + 3 * b) { dump_acc(false, true); stop = true; break; }
      } else if (a.debug_layer == 9) { dump_acc(false, true); stop = true; break; }
    }
    if (stop) continue;
    epi(T{}, F{}, F{}, 6);                                        // E3 -> A = relu(h)
    if (wg == 0) {
#pragma unroll 1
      for (int k = 0; k < kHiddenChunks; ++k) { mma_out(smem_base + kSmemAct + (uint32_t)k * kAStride, k == 0); retire1(); }   // lin_out
      if (a.debug_layer == 10) { dump_acc(true, false); continue; }
      retire0();
      // ---------------- E4: out = ACC[:, :d_out] + b_out ------------------------------------------------------
      const float* bo = bias + (size_t)7 * kHidden;
      const float inv_scale = SPLIT ? __ldg(bias + kInvScaleSlot) : 1.0f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int row = erow0 + 8 * ((i >> 1) & 1);
        const int col = 8 * (i >> 2) + ecol + (i & 1);
        float v = acco[i];
        if constexpr (SPLIT) v *= inv_scale;
        const int gi = row0 + row;
        if (gi < a.n && col < a.d_out) a.raw_out[(size_t)gi * a.d_out + col] = v + __ldg(bo + col);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Weight packing: nn.Linear fp32 (out,in) -> header of epilogue bias vectors + fp16 stage images in consumption order
// ---------------------------------------------------------------------------------------------------------------
struct PackArgs {
  srf_mlp_weights w;
  int kz;
  int parts;               // 1: fp16 images; 2: split mode, image (q, part) at index q*2 + part, part 0 = rn(W 2^s), 1 = rn(W 2^s - hi)
};

__device__ __forceinline__ const float* layer_weight(const srf_mlp_weights& w, int l, int& K) {
  K = kHidden;
  switch (l) {
    case 0: K = kDX; return w.lin_in_w;
    case 1: K = w.d_latent; return w.lin_z_w[0];
    case 2: return w.fc0_w[0];
    case 3: return w.fc1_w[0];
    case 4: K = w.d_latent; return w.lin_z_w[1];
    case 5: return w.fc0_w[1];
    case 6: return w.fc1_w[1];
    case 7: K = w.d_latent; return w.lin_z_w[2];
    case 8: return w.fc0_w[2];
    case 9: return w.fc1_w[2];
    default: return w.lin_out_w;
  }
}

// split mode: largest |w| over the 11 weight matrices -> power-of-two scale 2^s with max|w| 2^s in [2^13, 2^14), so
// that the fp16 low parts of typical weights are normal numbers (unscaled, |w| ~ 0.06 has a subnormal low part).
// Scaling by a power of two and its inverse in the epilogue are exact.
__global__ void weight_absmax_kernel(const __grid_constant__ PackArgs pa, unsigned int* __restrict__ max_bits) {
  float m = 0.0f;
  for (int l = 0; l < kNumLayers; ++l) {
    int K;
    const float* W = layer_weight(pa.w, l, K);
    const size_t n = (size_t)(l == kNumLayers - 1 ? pa.w.d_out : kHidden) * K;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(W[i]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(max_bits, __float_as_uint(m));       // non-negative floats order like their bits
}
__global__ void weight_scale_kernel(const unsigned int* __restrict__ max_bits, float* __restrict__ hdr, int split) {
  float scale = 1.0f;
  if (split) {
    const float m = __uint_as_float(*max_bits);
    int e = 0;
    if (m > 0.0f && isfinite(m)) { frexpf(m, &e); e = 14 - e; }        // m < 2^e0  ->  m 2^(14-e0) < 2^14
    e = max(-40, min(40, e));
    scale = ldexpf(1.0f, e);
  }
  hdr[kScaleSlot] = scale;
  hdr[kInvScaleSlot] = 1.0f / scale;
}

// one thread per 16-byte granule of the image region
__global__ void pack_images_kernel(const __grid_constant__ PackArgs pa, const float* __restrict__ hdr, unsigned char* __restrict__ images,
                                   size_t n_granules) {
  const size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= n_granules) return;
  size_t byte = gid * 16;
  const int parts = pa.parts;
  const float scale = hdr[kScaleSlot];
  // locate the layer
  int l = 0;
  size_t off = 0;
  for (; l < kNumLayers; ++l) {
    const size_t sz = (size_t)layer_chunks(l, pa.kz) * (kLayers[l].is_out ? kOutImgBytes : kQuarters * kBSlotBytes) * parts;
    if (byte < off + sz) break;
    off += sz;
  }
  const size_t rel = byte - off;
  const bool is_out = kLayers[l].is_out;
  const size_t img_bytes = is_out ? kOutImgBytes : kBSlotBytes;
  const size_t chunk_bytes = (is_out ? 1 : kQuarters) * img_bytes * parts;
  const int c = (int)(rel / chunk_bytes);
  const size_t in_chunk = rel % chunk_bytes;
  const int img = (int)(in_chunk / img_bytes);          // q * parts + part
  const int q = img / parts, part = img % parts;
  const size_t in_img = in_chunk % img_bytes;
  const int row = (int)(in_img / 128);
  const int gpos = (int)((in_img % 128) / 16);
  const int g = gpos ^ (row & 7);                      // logical granule stored at this swizzled position
  const int n = q * kBRows + row;                      // output unit
  int K;
  const float* W = layer_weight(pa.w, l, K);
  const int n_rows = is_out ? pa.w.d_out : kHidden;
  __align__(16) __half hv[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int k = c * kChunkK + g * 8 + j;
    const float v = ((n < n_rows && k < K) ? W[(size_t)n * K + k] : 0.0f) * scale;
    const __half hi = __float2half_rn(v);
    hv[j] = part == 0 ? hi : __float2half_rn(v - __half2float(hi));
  }
  *reinterpret_cast<uint4*>(images + byte) = *reinterpret_cast<const uint4*>(hv);
}

__global__ void pack_header_kernel(const __grid_constant__ PackArgs pa, float* __restrict__ hdr) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= kHidden) return;
  const srf_mlp_weights& w = pa.w;
  // cumulative biases folded into the epilogues (see file header)
  hdr[0 * kHidden + j] = w.lin_in_b[j] + w.lin_z_b[0][j];
  hdr[1 * kHidden + j] = w.fc1_b[0][j] + w.lin_z_b[1][j];
  hdr[2 * kHidden + j] = w.fc1_b[1][j] + w.lin_z_b[2][j];
  hdr[3 * kHidden + j] = w.fc0_b[0][j];
  hdr[4 * kHidden + j] = w.fc0_b[1][j];
  hdr[5 * kHidden + j] = w.fc0_b[2][j];
  hdr[6 * kHidden + j] = w.fc1_b[2][j];
  hdr[7 * kHidden + j] = (j < w.d_out) ? w.lin_out_b[j] : 0.0f;
}

static size_t images_bytes(int kz, int parts = 1) {
  size_t b = 0;
  const int chunks[kNumLayers] = {1, kz, 8, 8, kz, 8, 8, kz, 8, 8, 8};
  for (int l = 0; l < kNumLayers; ++l) b += (size_t)chunks[l] * (l == kNumLayers - 1 ? kOutImgBytes : kQuarters * kBSlotBytes);
  return b * (size_t)parts;
}

}  // namespace tc

static inline int kz_of(int d_latent) { return (d_latent + tc::kChunkK - 1) / tc::kChunkK; }

size_t tc_weights_bytes(int d_out, int d_latent, int split) {
  (void)d_out;
  // + 256: slack; the last 4 bytes of the blob are the absmax scratch word of the split pack
  return tc::kHeaderBytes + tc::images_bytes(kz_of(d_latent), split ? 2 : 1) + 256;
}

int pack_weights_tc(const srf_mlp_weights& w, void* dst, size_t bytes, int split, cudaStream_t st) {
  const int kz = kz_of(w.d_latent);
  if (kz > 64 || w.d_out < 1 || w.d_out > tc::kOutN || (w.d_latent % 8)) return 1;
  const size_t need = tc_weights_bytes(w.d_out, w.d_latent, split);
  if (bytes < need) return 1;
  tc::PackArgs pa;
  pa.w = w;
  pa.kz = kz;
  pa.parts = split ? 2 : 1;
  float* hdr = reinterpret_cast<float*>(dst);
  unsigned int* max_bits = reinterpret_cast<unsigned int*>(reinterpret_cast<unsigned char*>(dst) + need - 4);
  tc::pack_header_kernel<<<(kHidden + 127) / 128, 128, 0, st>>>(pa, hdr);
  if (split) {
    cudaMemsetAsync(max_bits, 0, 4, st);
    tc::weight_absmax_kernel<<<296, 256, 0, st>>>(pa, max_bits);
  }
  tc::weight_scale_kernel<<<1, 1, 0, st>>>(max_bits, hdr, split ? 1 : 0);
  const size_t n_gran = tc::images_bytes(kz, pa.parts) / 16;
  tc::pack_images_kernel<<<(unsigned)((n_gran + 255) / 256), 256, 0, st>>>(
      pa, hdr, reinterpret_cast<unsigned char*>(dst) + tc::kHeaderBytes, n_gran);
  return 0;
}

static int num_sms() { return device_sm_count(); }

using TcKernelFn = void (*)(const DevParams, const tc::KernelArgs);
constexpr int kNumTcKernels = 6;
// index: 0 = fp32 hidden state, 1 = fp16 hidden state, 2 = split mode; +3 = latent table
static TcKernelFn tc_kernel_at(int i) {
  static const TcKernelFn table[kNumTcKernels] = {
      tc::point_mlp_tc_kernel<false, false, false>, tc::point_mlp_tc_kernel<true, false, false>, tc::point_mlp_tc_kernel<false, true, false>,
      tc::point_mlp_tc_kernel<false, false, true>,  tc::point_mlp_tc_kernel<true, false, true>,  tc::point_mlp_tc_kernel<false, true, true>};
  return table[i];
}
static TcKernelFn tc_kernel(bool h16, bool split, bool pre) { return tc_kernel_at((split ? 2 : (h16 ? 1 : 0)) + (pre ? 3 : 0)); }

constexpr int kMaxTcCtas = 256;
size_t tc_workspace_bytes(int d_latent, int n_points) {
  (void)d_latent; (void)n_points;
  // hidden-state / partial-sum scratch for up to kMaxTcCtas CTAs + slack
  return (size_t)kMaxTcCtas * tc::kScratchFloats * sizeof(float) + 256;
}

int run_point_mlp_tc_debug(const DevParams& p, const srf_mlp_weights& w, const float* pts, const float* viewdir, int n,
                           int n_per, float* raw_out, int32_t* dbg_sphere, int flags, void* workspace, size_t ws_bytes,
                           int debug_layer, float* debug_acc, cudaStream_t st) {
  if (ws_bytes < tc_workspace_bytes(p.d_latent, n)) return -1;
  if (debug_layer >= 0 && !(debug_layer < tc::kNumLayers && debug_layer != 0 && debug_layer != 3 && debug_layer != 6))
    return -2;                         // layers without an accumulator-complete point cannot be dumped
  const bool split = (flags & kTcFlagSplit) != 0;
  // + 1 KB: slack for the kernel's round-up to 1024-byte alignment
  auto smem_of = [](bool s) { return (size_t)(s ? tc::Smem<true>::kTotal : tc::Smem<false>::kTotal) + 1024; };
  const size_t smem = smem_of(split);
  static bool attr_set = false;
  if (!attr_set) {
    for (int i = 0; i < kNumTcKernels; ++i)
      cudaFuncSetAttribute(tc_kernel_at(i), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_of(i % 3 == 2));
    attr_set = true;
  }
  tc::KernelArgs a;
  a.pts = pts; a.viewdir = viewdir; a.n = n; a.n_per = n_per;
  a.n_tiles = (n + tc::kTileM - 1) / tc::kTileM;
  a.kz = kz_of(p.d_latent);
  a.wblob = reinterpret_cast<const unsigned char*>(split ? w.tc_split_packed : w.tc_packed);
  if (!a.wblob) return -3;
  a.scratch = reinterpret_cast<float*>(workspace);
  a.raw_out = raw_out; a.d_out = w.d_out; a.dbg_sphere = dbg_sphere;
  a.skip_zero = (flags & SRF_FLAG_SKIP_ZERO_CHUNKS) ? 1 : 0;
  a.hidden_fp16 = (!split && (flags & SRF_FLAG_HIDDEN_FP16)) ? 1 : 0;
  // pre-projected latent table: only for the pass the caller marks (the table belongs to ONE network) and only in the
  // element type this mode reads (fp16 rows in fp16 mode, fp32 rows in split mode)
  a.preproj = nullptr; a.pre_W1 = p.sphere_W + 1; a.pre_H1 = p.sphere_H + 1;
  if ((flags & kTcFlagPreproj) && p.preproj && (p.preproj_fp16 != 0) == !split) {
    a.preproj = reinterpret_cast<const unsigned char*>(p.preproj);
    a.skip_zero = 0;
  }
  a.debug_layer = debug_layer; a.debug_acc = debug_acc;
  a.error_flag = watchdog_device_flag();
  // persistent: one CTA per SM (the shared-memory footprint allows no second one), tiles round-robin
  int grid = a.n_tiles < num_sms() ? a.n_tiles : num_sms();
  if (grid > kMaxTcCtas) grid = kMaxTcCtas;
  if (grid < 1) return 0;                       // no point: nothing launched
  tc_kernel(a.hidden_fp16 != 0, split, a.preproj != nullptr)<<<grid, tc::kThreads, smem, st>>>(p, a);
  return 1;
}

int run_point_mlp_tc(const DevParams& p, const srf_mlp_weights& w, const float* pts, const float* viewdir, int n,
                     int n_per, float* raw_out, int32_t* dbg_sphere, int flags, void* workspace, size_t ws_bytes,
                     cudaStream_t st) {
  return run_point_mlp_tc_debug(p, w, pts, viewdir, n, n_per, raw_out, dbg_sphere, flags, workspace, ws_bytes, -1,
                                nullptr, st);
}

}  // namespace srf
