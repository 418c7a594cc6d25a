// float32 SIMT implementation of the point MLP: projection + integer sphere coords + positional encoding +
// 5-scale bilinear gather (materialised as x_in for a chunk of points) followed by ResnetFC as plain fp32 GEMMs.
// This is the STRICT mode (srf_precision::SRF_PREC_FP32): every multiply-add is an fp32 FMA, so it tracks the
// reference (cuBLAS/MKL sgemm, scenerf/models/resnetfc.py:133-164) to float32 round-off.  It is also the device-side
// yardstick the tensor-core kernel is compared against at sizes the CPU oracle cannot reach.
//
// Reference: scenerf.py:505-547 (predict), utils.py:232-247,298-315, spherical_mapping.py:80-115, pe.py:32-43.
#include "kernels.cuh"

namespace srf {

// points per pass: one wave of 2 CTAs per SM of the GEMM chain's 128 x 128 tiles (4 column tiles of the 512-wide layers)
// -> 66 row tiles = 8448 points = 264 CTAs on the 132 SMs of an H100 SXM (x_in chunk 86 MB)
static int simt_chunk() { return (2 * device_sm_count() / 4 > 0 ? 2 * device_sm_count() / 4 : 1) * 128; }
#define kChunk (simt_chunk())

static inline int xin_ld(int d_latent) { return ((d_latent + kDX + 31) / 32) * 32; }

// one warp per point: [ z (d_latent) | pe (39) | viewdir (3) | 0-pad ]
__global__ void __launch_bounds__(256)
build_xin_kernel(const __grid_constant__ DevParams p, const float* __restrict__ pts, const float* __restrict__ viewdir,
                 int n, int n_per, int point0, float* __restrict__ X, int ld, int32_t* __restrict__ dbg_sphere,
                 int* __restrict__ scale_any) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= n) return;                       // whole warp
  const int gi = point0 + i;
  const float x = pts[(size_t)gi * 3 + 0], y = pts[(size_t)gi * 3 + 1], z = pts[(size_t)gi * 3 + 2];
  int sx, sy;
  point_to_sphere(p, x, y, z, sx, sy);
  if (dbg_sphere && lane == 0) { dbg_sphere[(size_t)gi * 2 + 0] = sx; dbg_sphere[(size_t)gi * 2 + 1] = sy; }
  float* row = X + (size_t)i * ld;
#pragma unroll
  for (int s = 0; s < kScales; ++s) {
    const Taps t = scale_taps(p, s, sx, sy);
    if (scale_any && t.any && lane == 0 && scale_any[s] == 0) atomicOr(&scale_any[s], 1);
    const float* f = reinterpret_cast<const float*>(p.feat[s]);
    float* dst = row + p.ch_off[s];
    for (int c = lane; c < p.C[s]; c += 32) {
      float acc = 0.0f;
      if (t.any) {
        const float v0 = t.off[0] >= 0 ? __ldg(f + t.off[0] + c) : 0.0f;
        const float v1 = t.off[1] >= 0 ? __ldg(f + t.off[1] + c) : 0.0f;
        const float v2 = t.off[2] >= 0 ? __ldg(f + t.off[2] + c) : 0.0f;
        const float v3 = t.off[3] >= 0 ? __ldg(f + t.off[3] + c) : 0.0f;
        acc = fadd(fadd(fadd(fmul(v0, t.w[0]), fmul(v1, t.w[1])), fmul(v2, t.w[2])), fmul(v3, t.w[3]));
      }
      dst[c] = acc;
    }
  }
  if (lane == 0) {
    float* xp = row + p.d_latent;
    positional_encoding(x, y, z, [&](int k, float v) { xp[k] = v; });
    const float* vd = viewdir + (size_t)(gi / n_per) * 3;
    xp[kDPE + 0] = vd[0]; xp[kDPE + 1] = vd[1]; xp[kDPE + 2] = vd[2];
    for (int k = p.d_latent + kDX; k < ld; ++k) row[k] = 0.0f;
  }
}

// lin_out: N = d_out (2 or 4) outputs per row, K = 512: one warp per row.
__global__ void __launch_bounds__(256)
lin_out_kernel(const float* __restrict__ Hh, const float* __restrict__ W, const float* __restrict__ bias,
               float* __restrict__ out, int M, int d_out) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= M) return;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k = lane; k < kHidden; k += 32) {
    const float a = fmaxf(Hh[(size_t)i * kHidden + k], 0.0f);
#pragma unroll
    for (int o = 0; o < 4; ++o)
      if (o < d_out) acc[o] = fmaf(a, W[o * kHidden + k], acc[o]);
  }
#pragma unroll
  for (int o = 0; o < 4; ++o) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], s);
  }
  if (lane == 0)
    for (int o = 0; o < d_out; ++o) out[(size_t)i * d_out + o] = acc[o] + bias[o];
}

void launch_build_xin(const DevParams& p, const float* pts, const float* viewdir, int m, int n_per, int point0, float* X, int ld,
                      int32_t* dbg_sphere, int* scale_any, cudaStream_t st) {
  if (scale_any) cudaMemsetAsync(scale_any, 0, kScales * sizeof(int), st);
  build_xin_kernel<<<(m + 7) / 8, 256, 0, st>>>(p, pts, viewdir, m, n_per, point0, X, ld, dbg_sphere, scale_any);
  ++launch_counter();
}

void launch_lin_out(const float* Hh, const float* W, const float* bias, float* out, int M, int d_out, cudaStream_t st) {
  lin_out_kernel<<<(M + 7) / 8, 256, 0, st>>>(Hh, W, bias, out, M, d_out);
  ++launch_counter();
}

size_t simt_workspace_bytes(int d_latent, int n_points) {
  const size_t chunk = (size_t)(n_points < kChunk ? n_points : kChunk);
  return chunk * ((size_t)xin_ld(d_latent) + 2 * kHidden) * sizeof(float) + 512;
}

// C[M x N] = (accumulate ? C : 0) + ( relu?(A)[M x K] * W[N x K]^T + bias )   (gemm.cu)
template <bool kRelu>
static void gemm(const float* A, int lda, const float* W, int ldw, const float* b, float* C, int M, int N, int K,
                 int accumulate, cudaStream_t st, const int* skip = nullptr) {
  GemmArgs g;
  g.skip_if_zero = skip;
  g.A = A; g.lda = lda; g.relu_a = kRelu; g.B = W; g.ldb = ldw; g.bt = true; g.C = C; g.ldc = N; g.M = M; g.N = N; g.K = K;
  g.bias = b; g.accumulate = accumulate;
  launch_gemm(g, st);
}

int run_point_mlp_simt(const DevParams& p, const srf_mlp_weights& w, const float* pts, const float* viewdir, int n,
                       int n_per, float* raw_out, int32_t* dbg_sphere, void* workspace, size_t ws_bytes,
                       cudaStream_t st) {
  if (ws_bytes < simt_workspace_bytes(p.d_latent, n)) return -1;
  const int ld = xin_ld(p.d_latent);
  float* X = reinterpret_cast<float*>(workspace);
  const int chunk_cap = n < kChunk ? n : kChunk;
  float* Hh = X + (size_t)chunk_cap * ld;
  float* Nn = Hh + (size_t)chunk_cap * kHidden;
  int* scale_any = reinterpret_cast<int*>(Nn + (size_t)chunk_cap * kHidden);
  const int c0 = launch_counter();
  for (int p0 = 0; p0 < n; p0 += kChunk) {
    const int m = (n - p0) < kChunk ? (n - p0) : kChunk;
    launch_build_xin(p, pts, viewdir, m, n_per, p0, X, ld, dbg_sphere, scale_any, st);
    // h = lin_in(x)                               (resnetfc.py:148)
    gemm<false>(X + p.d_latent, ld, w.lin_in_w, kDX, w.lin_in_b, Hh, m, kHidden, kDX, 0, st);
    for (int b = 0; b < SRF_NUM_BLOCKS; ++b) {
      // h = h + lin_z[b](z)                       (resnetfc.py:152-158)
      // one K-segment per pyramid scale; a scale no point of the chunk reaches is all zeros and is skipped on the device
      for (int s = 0; s < kScales; ++s) {
        gemm<false>(X + p.ch_off[s], ld, w.lin_z_w[b] + p.ch_off[s], p.d_latent, s == 0 ? w.lin_z_b[b] : nullptr, Hh, m, kHidden,
                    p.C[s], 1, st, s == 0 ? nullptr : scale_any + s);
      }
      // net = fc_0(relu(h)); h = h + fc_1(relu(net))   (resnetfc.py:54-63)
      gemm<true>(Hh, kHidden, w.fc0_w[b], kHidden, w.fc0_b[b], Nn, m, kHidden, kHidden, 0, st);
      gemm<true>(Nn, kHidden, w.fc1_w[b], kHidden, w.fc1_b[b], Hh, m, kHidden, kHidden, 1, st);
    }
    // out = lin_out(relu(h))                      (resnetfc.py:163)
    launch_lin_out(Hh, w.lin_out_w, w.lin_out_b, raw_out + (size_t)p0 * w.d_out, m, w.d_out, st);
  }
  return launch_counter() - c0;
}

}  // namespace srf
