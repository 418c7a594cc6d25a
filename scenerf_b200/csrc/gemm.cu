// float32 SIMT GEMM family used by the strict-precision forward and backward of the point MLP (mlp_simt.cu).
//   C[M x N] = epilogue( sum_k a(m,k) * b(k,n) ),  k ascending, one fmaf chain per output (the summation order does
//   not depend on the tile shape, so both kernels below give bit-identical results)
//   AT=false: A stored [M][K] (lda)   AT=true : A stored [K][M] (lda)
//   BT=true : B stored [N][K] (ldb)   BT=false: B stored [K][N] (ldb)
//   epilogue: v = acc (+bias[n]); if mask: v = mask[m][n] > 0 ? v : 0; if R: v += R[m][n]; if accumulate: v += C[m][n]
//   R may alias C (R == C, ldr == ldc): the thread that writes C[m][n] is the only one that reads R[m][n], and it reads
//   it first, so the residual add works in place (R and C are not __restrict__).  The float32 forward relies on this
//   (mlp_simt.cu: h = h + lin_z(z) and h = h + fc_1(relu(net)) in one buffer).
// gemm128_kernel: 128x128x16 tiles, 8x8 outputs per thread, float4 global/shared accesses, register-prefetched double
// buffering -- the hot one (needs 16-byte aligned rows).  gemm64_kernel: 64x64x16, scalar loads, any shape (lin_in K=42,
// lin_out M=4 ...).  FP32-FMA-bound: 2*M*N*K flops against SMs (132 on an H100 SXM) x 128 lanes x 2 x clock.
#include "kernels.cuh"

namespace srf {

template <bool AT, bool BT, bool RELU_A, bool RELU_B>
__global__ void __launch_bounds__(256)
gemm64_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb, float* C, int ldc, int M, int N, int K,
              const float* __restrict__ bias, const float* __restrict__ mask, int ldm, const float* R, int ldr, int accumulate,
              int k_per, const int* __restrict__ skip) {
  if (skip && *skip == 0) return;                            // the whole K-segment is known to be zero (see GemmArgs::skip_if_zero)
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4] = {};
  const int kbeg = blockIdx.z * k_per;                       // split-K as in gemm128_kernel
  if (gridDim.z > 1) { K = min(K, kbeg + k_per); C += (size_t)blockIdx.z * M * ldc; }
  for (int k0 = kbeg; k0 < K; k0 += 16) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int idx = threadIdx.x + e * 256;
      {
        const int rr = AT ? (idx & 63) : (idx >> 4), kk = AT ? (idx >> 6) : (idx & 15);
        const int gm = m0 + rr, gk = k0 + kk;
        float a = 0.f;
        if (gm < M && gk < K) a = AT ? A[(size_t)gk * lda + gm] : A[(size_t)gm * lda + gk];
        if (RELU_A) a = fmaxf(a, 0.f);
        As[kk][rr] = a;
      }
      {
        const int rr = BT ? (idx >> 4) : (idx & 63), kk = BT ? (idx & 15) : (idx >> 6);
        const int gn = n0 + rr, gk = k0 + kk;
        float b = 0.f;
        if (gn < N && gk < K) b = BT ? B[(size_t)gn * ldb + gk] : B[(size_t)gk * ldb + gn];
        if (RELU_B) b = fmaxf(b, 0.f);
        Bs[kk][rr] = b;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[gn];
      if (mask) v = (mask[(size_t)gm * ldm + gn] > 0.f) ? v : 0.f;
      if (R) v += R[(size_t)gm * ldr + gn];
      if (accumulate) v += C[(size_t)gm * ldc + gn];
      C[(size_t)gm * ldc + gn] = v;
    }
  }
}

constexpr int kBM = 128, kBN = 128, kBK = 16, kPitch = kBM + 4;

// Loads one 128 x 16 operand tile into registers (2 float4 per thread) and stores it as S[k][x] (x = m or n).
//   ROWK=true : operand stored [x][k] (float4 along k, transposed on the way into shared memory)
//   ROWK=false: operand stored [k][x] (float4 along x)
template <bool ROWK, bool RELU>
struct TileLoader {
  float4 v[2];
  __device__ __forceinline__ void load(const float* __restrict__ P, int ld, int x0, int X, int k0, int K) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int f = threadIdx.x + i * 256;
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      if (ROWK) {
        const int row = f >> 2, kq = f & 3;
        const int gx = x0 + row, gk = k0 + kq * 4;
        if (gx < X && gk < K) t = *reinterpret_cast<const float4*>(P + (size_t)gx * ld + gk);      // K % 4 == 0
      } else {
        const int kk = f >> 5, xq = f & 31;
        const int gk = k0 + kk, gx = x0 + xq * 4;
        if (gk < K && gx < X) t = *reinterpret_cast<const float4*>(P + (size_t)gk * ld + gx);      // X % 4 == 0
      }
      if (RELU) { t.x = fmaxf(t.x, 0.f); t.y = fmaxf(t.y, 0.f); t.z = fmaxf(t.z, 0.f); t.w = fmaxf(t.w, 0.f); }
      v[i] = t;
    }
  }
  __device__ __forceinline__ void store(float (*S)[kPitch]) const {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int f = threadIdx.x + i * 256;
      if (ROWK) {
        const int row = f >> 2, kq = f & 3;
        S[kq * 4 + 0][row] = v[i].x; S[kq * 4 + 1][row] = v[i].y; S[kq * 4 + 2][row] = v[i].z; S[kq * 4 + 3][row] = v[i].w;
      } else {
        const int kk = f >> 5, xq = f & 31;
        *reinterpret_cast<float4*>(&S[kk][xq * 4]) = v[i];
      }
    }
  }
};

// gridDim.z > 1: split-K.  Slice z handles k in [z*k_per, (z+1)*k_per) and stores its plain partial sums to
// C + z*M*ldc (C is then a scratch buffer, no epilogue); splitk_reduce_kernel adds the slices in fixed order.
template <bool AT, bool BT, bool RELU_A, bool RELU_B>
__global__ void __launch_bounds__(256, 2)
gemm128_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B, int ldb, float* C, int ldc, int M, int N, int K,
               const float* __restrict__ bias, const float* __restrict__ mask, int ldm, const float* R, int ldr, int accumulate,
               int k_per, const int* __restrict__ skip) {
  if (skip && *skip == 0) return;
  __shared__ __align__(16) float As[2][kBK][kPitch];
  __shared__ __align__(16) float Bs[2][kBK][kPitch];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * kBM, n0 = blockIdx.x * kBN;
  TileLoader<!AT, RELU_A> la;
  TileLoader<BT, RELU_B> lb;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const int kbeg = blockIdx.z * k_per;
  if (gridDim.z > 1) { K = min(K, kbeg + k_per); C += (size_t)blockIdx.z * M * ldc; }
  la.load(A, lda, m0, M, kbeg, K);
  lb.load(B, ldb, n0, N, kbeg, K);
  la.store(As[0]);
  lb.store(Bs[0]);
  __syncthreads();
  int buf = 0;
  for (int k0 = kbeg; k0 < K; k0 += kBK) {
    const bool more = k0 + kBK < K;
    if (more) { la.load(A, lda, m0, M, k0 + kBK, K); lb.load(B, ldb, n0, N, k0 + kBK, K); }
#pragma unroll
    for (int kk = 0; kk < kBK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (more) {
      la.store(As[buf ^ 1]);
      lb.store(Bs[buf ^ 1]);
      __syncthreads();
      buf ^= 1;
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gm = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (gm >= M) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gn = n0 + h * 64 + tx * 4;
      if (gn >= N) continue;                                           // N % 4 == 0
      float4 v = make_float4(acc[i][h * 4 + 0], acc[i][h * 4 + 1], acc[i][h * 4 + 2], acc[i][h * 4 + 3]);
      if (bias) { const float4 t = *reinterpret_cast<const float4*>(bias + gn); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
      if (mask) {
        const float4 t = *reinterpret_cast<const float4*>(mask + (size_t)gm * ldm + gn);
        v.x = t.x > 0.f ? v.x : 0.f; v.y = t.y > 0.f ? v.y : 0.f; v.z = t.z > 0.f ? v.z : 0.f; v.w = t.w > 0.f ? v.w : 0.f;
      }
      if (R) { const float4 t = *reinterpret_cast<const float4*>(R + (size_t)gm * ldr + gn); v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
      float4* dst = reinterpret_cast<float4*>(C + (size_t)gm * ldc + gn);
      if (accumulate) { const float4 t = *dst; v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w; }
      *dst = v;
    }
  }
}

// C[m][n] = (accumulate ? C[m][n] : 0) + sum_z part[z][m][n]   (z ascending: deterministic)
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ part, int splits, float* __restrict__ C, int ldc, int M, int N, int accumulate,
                     const int* __restrict__ skip, const __grid_constant__ SegInfo sg) {
  if (skip && *skip == 0) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * N) return;
  if (sg.mode == 2) {                                      // columns of a dead tile were never written by the GEMM
    const int t0 = (i % N) / kSegTileN * kSegTileN;
    if (seg_dead(sg, t0, min(N, t0 + kSegTileN))) return;
  }
  const int m = i / N, n = i % N;
  float v = 0.f;
  for (int z = 0; z < splits; ++z) v += part[(size_t)z * M * N + i];
  float* dst = C + (size_t)m * ldc + n;
  *dst = accumulate ? (*dst + v) : v;
}

void launch_splitk_reduce(const GemmArgs& g, int splits, const SegInfo& sg, cudaStream_t st) {
  splitk_reduce_kernel<<<(g.M * g.N + 255) / 256, 256, 0, st>>>(g.splitk_ws, splits, g.C, g.ldc, g.M, g.N, g.accumulate, g.skip_if_zero, sg);
}

SplitK plan_splitk(const GemmArgs& g, int tiles, int k_gran, int cap) {
  SplitK sk{1, g.K};
  if (!g.splitk_ws || g.bias || g.mask || g.R || tiles >= 96 || g.K < 1024) return sk;
  int splits = (2 * device_sm_count() + tiles - 1) / tiles;     // ~2 waves
  if (splits > cap) splits = cap;
  while (splits > 1 && (size_t)splits * g.M * g.N > g.splitk_ws_floats) --splits;
  if (splits > 1) {
    sk.k_per = ((g.K + splits - 1) / splits + k_gran - 1) / k_gran * k_gran;
    sk.splits = (g.K + sk.k_per - 1) / sk.k_per;             // still >= 2: k_per < K for K >= 1024, k_gran <= 32
  }
  return sk;
}

int device_sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
      n = 132;                 // no device visible (size queries on a build machine): H100 SXM
      cudaGetLastError();
    }
  }
  return n;
}

int& launch_counter() {
  static thread_local int c = 0;
  return c;
}

template <bool AT, bool BT, bool RA, bool RB>
static void dispatch(const GemmArgs& g, cudaStream_t st) {
  bool fast = (g.lda % 4 == 0) && (g.ldb % 4 == 0) && (g.ldc % 4 == 0) && (g.N % 4 == 0) && al16(g.A) && al16(g.B) && al16(g.C);
  if (!AT) fast = fast && (g.K % 4 == 0);          // float4 along k of A
  else fast = fast && (g.M % 4 == 0);              // float4 along m of A
  if (BT) fast = fast && (g.K % 4 == 0);
  if (g.bias) fast = fast && al16(g.bias);
  if (g.mask) fast = fast && al16(g.mask) && (g.ldm % 4 == 0);
  if (g.R) fast = fast && al16(g.R) && (g.ldr % 4 == 0);
  fast = fast && g.M >= 64 && g.N >= 64;
  // the SIMT kernels write every column: segment mode 0 for the reduce, whatever a tf32-mode fallback call carries in seg_*
  const SegInfo no_seg{};
  if (fast) {
    dim3 grid((g.N + kBN - 1) / kBN, (g.M + kBM - 1) / kBM);
    // weight-gradient shapes (few output tiles, long K): split K over gridDim.z into the caller's scratch
    const SplitK sk = plan_splitk(g, grid.x * grid.y, kBK, 16);
    if (sk.splits > 1) {
      grid.z = sk.splits;
      gemm128_kernel<AT, BT, RA, RB><<<grid, 256, 0, st>>>(g.A, g.lda, g.B, g.ldb, g.splitk_ws, g.N, g.M, g.N, g.K, nullptr, nullptr, 0,
                                                           nullptr, 0, 0, sk.k_per, g.skip_if_zero);
      launch_splitk_reduce(g, sk.splits, no_seg, st);
      launch_counter() += 2;
    } else {
      ++launch_counter();
      gemm128_kernel<AT, BT, RA, RB><<<grid, 256, 0, st>>>(g.A, g.lda, g.B, g.ldb, g.C, g.ldc, g.M, g.N, g.K, g.bias, g.mask, g.ldm,
                                                           g.R, g.ldr, g.accumulate, g.K, g.skip_if_zero);
    }
  } else {
    dim3 grid((g.N + 63) / 64, (g.M + 63) / 64);
    const SplitK sk = plan_splitk(g, grid.x * grid.y, 16, 64);
    if (sk.splits > 1) {
      grid.z = sk.splits;
      gemm64_kernel<AT, BT, RA, RB><<<grid, 256, 0, st>>>(g.A, g.lda, g.B, g.ldb, g.splitk_ws, g.N, g.M, g.N, g.K, nullptr, nullptr, 0,
                                                          nullptr, 0, 0, sk.k_per, g.skip_if_zero);
      launch_splitk_reduce(g, sk.splits, no_seg, st);
      launch_counter() += 2;
    } else {
      ++launch_counter();
      gemm64_kernel<AT, BT, RA, RB><<<grid, 256, 0, st>>>(g.A, g.lda, g.B, g.ldb, g.C, g.ldc, g.M, g.N, g.K, g.bias, g.mask, g.ldm,
                                                          g.R, g.ldr, g.accumulate, g.K, g.skip_if_zero);
    }
  }
}

int launch_gemm(const GemmArgs& g, cudaStream_t st) {
  const int key = (g.at ? 8 : 0) | (g.bt ? 4 : 0) | (g.relu_a ? 2 : 0) | (g.relu_b ? 1 : 0);
  switch (key) {
    case 4: dispatch<false, true, false, false>(g, st); return 0;       // forward  C = A W^T
    case 6: dispatch<false, true, true, false>(g, st); return 0;        // forward  C = relu(A) W^T
    case 0: dispatch<false, false, false, false>(g, st); return 0;      // dX = dY W
    case 9: dispatch<true, false, false, true>(g, st); return 0;        // dW += dY^T relu(X)
    case 8: dispatch<true, false, false, false>(g, st); return 0;       // dW += dY^T X
    default: return -1;
  }
}

}  // namespace srf
