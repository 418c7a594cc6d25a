// float32 implementation of the point MLP and of its backward: projection + integer sphere coords + positional encoding +
// 5-scale bilinear gather (materialised as x_in for a chunk of points) followed by ResnetFC as plain fp32 GEMMs.
// This is the STRICT mode (srf_precision::SRF_PREC_FP32): every multiply-add is an fp32 FMA, so it tracks the
// reference (cuBLAS/MKL sgemm, scenerf/models/resnetfc.py:133-164) to float32 round-off.  It is also the device-side
// yardstick the tensor-core kernel is compared against at sizes the CPU oracle cannot reach, and the forward and backward
// of training (SRF_FLAG_TF32_MATMUL moves the NT products of training onto the wgmma tf32 kernel, gemm_tf32.cu;
// SRF_FLAG_FP32TC_MATMUL onto its split 3xTF32 variant, which keeps float32-grade products).
//
// Every decision about how the ResnetFC chain is sequenced lives here: the chunk sizes of inference and training, the
// layout of the saved activations, ONE forward (inference, training forward and the backward's recompute) and ONE
// backward block loop (both GEMM engines).
//
// Backward order, per chunk of points: recompute the forward keeping the pre-activations (or read them from the store
// of the training forward), then the GEMM chain backwards (dX = dY W, dW += dY^T X, db += colsum dY), then scatter
// d latent into the CHW feature-map gradients with atomics.  Parameter gradients are deterministic (no atomics, fixed
// chunk order); feature-map gradients use float atomicAdd.
//
// Reference: scenerf.py:505-547 (predict), utils.py:232-247,298-315, spherical_mapping.py:80-115, pe.py:32-43.
#include "kernels.cuh"

namespace srf {

// Inference: points per pass: one wave of 2 CTAs per SM of the GEMM chain's 128 x 128 tiles (4 column tiles of the
// 512-wide layers) -> 66 row tiles = 8448 points = 264 CTAs on the 132 SMs of an H100 SXM (x_in chunk 86 MB)
static int simt_chunk() { return (2 * device_sm_count() / 4 > 0 ? 2 * device_sm_count() / 4 : 1) * 128; }
// Training: points per pass of the forward and the backward.  Round 1 used 9472 (74 row tiles x 4 column tiles = one wave
// of 296 CTAs) -- and paid for it with ~700 launches per 1200-ray training step; the GEMM kernels are grid-size agnostic,
// so a pass now covers a whole training call (81.6 k points fit: ~40 KB of workspace per point) and the launch count
// drops ~8x.  SRF_TRAIN_CHUNK overrides (multiple of 128).
static int train_chunk() {
  static int v = 0;
  if (!v) {
    const char* e = getenv("SRF_TRAIN_CHUNK");
    v = e ? atoi(e) : 98304;
    if (v < 128) v = 128;
    v = (v + 127) / 128 * 128;
  }
  return v;
}
constexpr size_t kSplitKFloats = (size_t)4 * 512 * 2528;     // split-K scratch of the weight-gradient GEMMs (20 MB)

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

// gb[n] += sum_m dY[m][n], deterministic two-stage: kColSegs row segments (grid.y) -> part[seg][n], then a fixed-order sum
constexpr int kColSegs = 64;
__global__ void __launch_bounds__(256)
colsum_partial_kernel(const float* __restrict__ dY, int ld, int M, int N, float* __restrict__ part) {
  __shared__ float sh[8][32];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), rl = threadIdx.x >> 5;
  const int rows_per = (M + kColSegs - 1) / kColSegs;
  const int r0 = blockIdx.y * rows_per, r1 = min(M, r0 + rows_per);
  float s = 0.f;
  if (c < N)
    for (int m = r0 + rl; m < r1; m += 8) s += dY[(size_t)m * ld + c];
  sh[rl][threadIdx.x & 31] = s;
  __syncthreads();
  if (rl == 0 && c < N) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sh[k][threadIdx.x & 31];
    part[(size_t)blockIdx.y * N + c] = t;
  }
}
__global__ void __launch_bounds__(256)
colsum_final_kernel(const float* __restrict__ part, int N, float* __restrict__ gb) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= N) return;
  float t = 0.f;
  for (int s = 0; s < kColSegs; ++s) t += part[(size_t)s * N + c];
  gb[c] += t;
}

// dst[c][r] = relu?(src[r][c])   (rows x cols -> cols x rows; dst row stride ldd >= rows)
template <bool RELU>
__global__ void __launch_bounds__(256)
transpose_kernel(const float* __restrict__ src, int lds, int rows, int cols, float* __restrict__ dst, int ldd) {
  __shared__ float t[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty + i * 8, c = c0 + tx;
    float v = (r < rows && c < cols) ? src[(size_t)r * lds + c] : 0.f;
    if (RELU) v = fmaxf(v, 0.f);
    t[ty + i * 8][tx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + i * 8, r = r0 + tx;
    if (c < cols && r < rows) dst[(size_t)c * ldd + r] = t[tx][ty + i * 8];
  }
}
__global__ void __launch_bounds__(256) relu_kernel(const float4* __restrict__ src, float4* __restrict__ dst, size_t n4) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 v = src[i];
  v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
  dst[i] = v;
}

// dh[m][c] = (h3[m][c] > 0) ? sum_o g[m][o] * Wout[o][c] : 0        (lin_out backward w.r.t. its input)
__global__ void __launch_bounds__(256)
lin_out_dx_kernel(const float* __restrict__ g, int d_out, const float* __restrict__ Wout, const float* __restrict__ h3,
                  float* __restrict__ dh, int M) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * kHidden) return;
  const int m = i / kHidden, c = i % kHidden;
  float v = 0.f;
  for (int o = 0; o < d_out; ++o) v = fmaf(g[(size_t)m * d_out + o], Wout[o * kHidden + c], v);
  dh[i] = (h3[i] > 0.f) ? v : 0.f;
}

// feature-map gradient: grad_chw[s][c][pixel] += w_tap * dz[point][ch_off[s] + c]   (one warp per point)
struct PyrGrad { float* chw[kScales]; };
__global__ void __launch_bounds__(256)
scatter_latent_kernel(const __grid_constant__ DevParams p, const float* __restrict__ pts, int n, int point0,
                      const float* __restrict__ dZ, int ld, PyrGrad gp) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= n) return;
  const int gi = point0 + i;
  int sx, sy;
  point_to_sphere(p, pts[(size_t)gi * 3 + 0], pts[(size_t)gi * 3 + 1], pts[(size_t)gi * 3 + 2], sx, sy);
  const float* row = dZ + (size_t)i * ld;
#pragma unroll
  for (int s = 0; s < kScales; ++s) {
    const Taps t = scale_taps(p, s, sx, sy);
    if (!t.any) continue;
    const int C = p.C[s];
    const size_t plane = (size_t)p.H[s] * p.W[s];
    float* g = gp.chw[s];
    for (int c = lane; c < C; c += 32) {
      const float v = row[p.ch_off[s] + c];
      if (v == 0.f) continue;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (t.off[k] >= 0) atomicAdd(g + (size_t)c * plane + t.off[k] / C, t.w[k] * v);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// one warp per point: X[i] = [ gathered latent (d_latent) | positional encoding (39) | viewdir (3) | 0-pad ], row stride ld
//   scale_any (5 ints, or NULL): set to 1 for every scale at which some point of the chunk has an in-range bilinear tap.
//   Scales whose flag stays 0 contribute exact zeros to x_in (quirk Q2: out-of-range normalised coordinates), so the
//   lin_z GEMMs skip their K-segment -- bit-identical results.
static void launch_build_xin(const DevParams& p, const float* pts, const float* viewdir, int m, int n_per, int point0, float* X,
                             int ld, int32_t* dbg_sphere, int* scale_any, cudaStream_t st) {
  if (scale_any) cudaMemsetAsync(scale_any, 0, kScales * sizeof(int), st);
  build_xin_kernel<<<(m + 7) / 8, 256, 0, st>>>(p, pts, viewdir, m, n_per, point0, X, ld, dbg_sphere, scale_any);
  ++launch_counter();
}

static void colsum(const float* dY, int ld, int M, int N, float* gb, float* scratch, cudaStream_t st) {
  colsum_partial_kernel<<<dim3((N + 31) / 32, kColSegs), 256, 0, st>>>(dY, ld, M, N, scratch);
  colsum_final_kernel<<<(N + 255) / 256, 256, 0, st>>>(scratch, N, gb);
  launch_counter() += 2;
}

template <bool RELU>
static void transpose(const float* src, int lds, int rows, int cols, float* dst, int ldd, cudaStream_t st) {
  transpose_kernel<RELU><<<dim3((cols + 31) / 32, (rows + 31) / 32), 256, 0, st>>>(src, lds, rows, cols, dst, ldd);
  ++launch_counter();
}

// One GEMM of the chain: C[M x N] = epilogue(op(A) op(B)) with gemm.cu's operand layouts; g carries the epilogue and
// scratch fields.  A tensor-core engine puts an NT product without operand ReLU on the wgmma kernel (fp32tc: its split
// 3xTF32 variant); every other product,
// and a shape that kernel cannot take, runs on the SIMT kernels, and relu_out is then filled by a separate pass over C
// (the callers keep ldc == ld_relu == N).
template <bool AT, bool BT, bool RA = false, bool RB = false>
static void gemm(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K, GemmArgs g, MatmulEngine e,
                 cudaStream_t st) {
  g.A = A; g.lda = lda; g.at = AT; g.relu_a = RA; g.B = B; g.ldb = ldb; g.bt = BT; g.relu_b = RB;
  g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = K;
  if (tensor_cores(e) && launch_gemm_tf32(g, st, e == MatmulEngine::fp32tc) == 0) return;
  launch_gemm(g, st);
  if (g.relu_out) {
    const size_t n4 = (size_t)M * N / 4;
    relu_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float4*>(C), reinterpret_cast<float4*>(g.relu_out), n4);
    ++launch_counter();
  }
}

// The latent axis of a tf32 product is the five pyramid scales: the kernel skips the k-blocks (mode 1) or the column
// tiles (mode 2) that lie in scales whose flag is 0.
static void set_segments(GemmArgs& g, const int* flags, int mode, const int* ch_off) {
  g.seg_flags = flags; g.seg_mode = mode;
  for (int i = 0; i <= kScales; ++i) g.seg_off[i] = ch_off[i];
}

// ---------------------------------------------------------------------------------------------------------------
// Activations of the chain, the ones the backward reads: X = x_in (ld), PRE[b] = h + lin_z[b](z), NET[b] =
// fc_0(relu(PRE[b])), H3 = h after block 2 (512 each), and the 5 scale flags of each chunk (8 ints per chunk).
// whole_pass: the rows of every point of a pass (the store of SRF_FLAG_SAVE_ACTIVATIONS, laid out X (n,ld) |
// PRE[0] NET[0] PRE[1] NET[1] PRE[2] NET[2] H3 (n,512) | flags); otherwise the buffers of one chunk, reused by every chunk.
struct Acts {
  float* X; float* PRE[3]; float* NET[3]; float* H3; int* flags;
  bool whole_pass;
  // the view of chunk c, which starts at point p0
  Acts chunk(int p0, int c, int ld) const {
    Acts a = *this;
    if (!whole_pass) return a;
    a.X += (size_t)p0 * ld;
    for (int b = 0; b < 3; ++b) { a.PRE[b] += (size_t)p0 * kHidden; a.NET[b] += (size_t)p0 * kHidden; }
    a.H3 += (size_t)p0 * kHidden;
    a.flags += c * 8;
    return a;
  }
};
static inline size_t n_chunks_train(int n) { return ((size_t)n + train_chunk() - 1) / train_chunk(); }
size_t mlp_saved_bytes(int d_latent, int n_points) {
  return (size_t)n_points * ((size_t)xin_ld(d_latent) + 7 * kHidden) * sizeof(float) + n_chunks_train(n_points) * 8 * sizeof(int) + 256;
}
static Acts saved_view(void* base, int d_latent, int n) {
  Acts a;
  float* q = reinterpret_cast<float*>(base);
  a.X = q; q += (size_t)n * xin_ld(d_latent);
  for (int b = 0; b < 3; ++b) { a.PRE[b] = q; q += (size_t)n * kHidden; a.NET[b] = q; q += (size_t)n * kHidden; }
  a.H3 = q; q += (size_t)n * kHidden;
  a.flags = reinterpret_cast<int*>(q);
  a.whole_pass = true;
  return a;
}

// the training forward keeps its activations in the store; on a tensor-core engine it needs two ReLU'd operand buffers per chunk
static size_t relu_scratch_bytes(int n_points) {
  return (size_t)2 * (size_t)(n_points < train_chunk() ? n_points : train_chunk()) * kHidden * sizeof(float) + 256;
}
size_t simt_workspace_bytes(int d_latent, int n_points, bool save_activations) {
  const size_t chunk = (size_t)(n_points < simt_chunk() ? n_points : simt_chunk());
  const size_t infer = chunk * ((size_t)xin_ld(d_latent) + 2 * kHidden) * sizeof(float) + 512;
  if (!save_activations) return infer;
  const size_t relu = relu_scratch_bytes(n_points);
  return infer > relu ? infer : relu;
}

// resnetfc.py:133-164 for the m rows of one chunk (x_in in a.X, its scale flags in a.flags): h = lin_in(x), then per
// block PRE[b] = h + lin_z[b](z), NET[b] = fc_0(relu(PRE[b])), h = PRE[b] + fc_1(relu(NET[b])); H3 = h after block 2.
// The residual always enters as the epilogue's R operand, which gemm.cu allows to alias C, so inference runs the same
// arithmetic in two buffers (PRE[b] = H3 = h, NET[b] = net) and training keeps every activation apart.
// tf32 / fp32tc: relu_scratch holds 2 x m x 512 floats -- the tensor-core GEMM reads its A operand as stored, so the producing
// GEMM's epilogue also stores the ReLU'd activations the next GEMM consumes.
static void resnetfc_forward(const DevParams& p, const srf_mlp_weights& w, const Acts& a, int ld, int m, MatmulEngine e,
                             float* relu_scratch, cudaStream_t st) {
  const int H = kHidden, DL = p.d_latent;
  const bool tc = tensor_cores(e);
  GemmArgs o;
  o.bias = w.lin_in_b;
  gemm<false, true>(a.X + DL, ld, w.lin_in_w, kDX, a.PRE[0], H, m, H, kDX, o, e, st);                        // h = lin_in(x)
  for (int b = 0; b < SRF_NUM_BLOCKS; ++b) {
    const float* h = (b == 0) ? a.PRE[0] : a.H3;
    if (tc) {
      float* relu2 = relu_scratch + (size_t)m * H;
      o = GemmArgs(); o.bias = w.lin_z_b[b]; o.R = h; o.ldr = H; o.relu_out = relu_scratch; o.ld_relu = H;
      set_segments(o, a.flags, 1, p.ch_off);
      gemm<false, true>(a.X, ld, w.lin_z_w[b], DL, a.PRE[b], H, m, H, DL, o, e, st);                         // pre = h + lin_z(z); relu(pre) on the side
      o = GemmArgs(); o.bias = w.fc0_b[b]; o.relu_out = relu2; o.ld_relu = H;
      gemm<false, true>(relu_scratch, H, w.fc0_w[b], H, a.NET[b], H, m, H, H, o, e, st);                     // net = fc_0(relu(pre)); relu(net) on the side
      o = GemmArgs(); o.bias = w.fc1_b[b]; o.R = a.PRE[b]; o.ldr = H;
      gemm<false, true>(relu2, H, w.fc1_w[b], H, a.H3, H, m, H, H, o, e, st);                                // h = pre + fc_1(relu(net))
    } else {
      for (int s = 0; s < kScales; ++s) {                                                                     // pre = h + lin_z(z), one K-segment per scale
        o = GemmArgs();
        if (s == 0) { o.bias = w.lin_z_b[b]; o.R = h; o.ldr = H; }
        else { o.accumulate = 1; o.skip_if_zero = a.flags + s; }
        gemm<false, true>(a.X + p.ch_off[s], ld, w.lin_z_w[b] + p.ch_off[s], DL, a.PRE[b], H, m, H, p.C[s], o, e, st);
      }
      o = GemmArgs(); o.bias = w.fc0_b[b];
      gemm<false, true, true>(a.PRE[b], H, w.fc0_w[b], H, a.NET[b], H, m, H, H, o, e, st);                   // net = fc_0(relu(pre))
      o = GemmArgs(); o.bias = w.fc1_b[b]; o.R = a.PRE[b]; o.ldr = H;
      gemm<false, true, true>(a.NET[b], H, w.fc1_w[b], H, a.H3, H, m, H, H, o, e, st);                       // h = pre + fc_1(relu(net))
    }
  }
}

int run_point_mlp_simt(const DevParams& p, const srf_mlp_weights& w, const float* pts, const float* viewdir, int n, int n_per,
                       float* raw_out, int32_t* dbg_sphere, void* saved, MatmulEngine e, void* workspace, size_t ws_bytes,
                       cudaStream_t st) {
  const int ld = xin_ld(p.d_latent);
  int chunk;
  Acts a;
  float* relu_scratch = nullptr;
  if (saved) {                             // training forward: the activations of the whole pass go to the store
    if (tensor_cores(e)) {
      if (ws_bytes < relu_scratch_bytes(n)) return -1;
      relu_scratch = reinterpret_cast<float*>(workspace);
    }
    chunk = train_chunk();
    a = saved_view(saved, p.d_latent, n);
  } else {                                 // inference: one chunk's x_in, h and net in the workspace
    if (e != MatmulEngine::simt || ws_bytes < simt_workspace_bytes(p.d_latent, n, false)) return -1;
    chunk = simt_chunk();
    const size_t cap = (size_t)(n < chunk ? n : chunk);
    float* Hh = reinterpret_cast<float*>(workspace) + cap * ld;
    float* Nn = Hh + cap * kHidden;
    a = Acts{reinterpret_cast<float*>(workspace), {Hh, Hh, Hh}, {Nn, Nn, Nn}, Hh, reinterpret_cast<int*>(Nn + cap * kHidden), false};
  }
  const int c0 = launch_counter();
  for (int p0 = 0, c = 0; p0 < n; p0 += chunk, ++c) {
    const int m = (n - p0) < chunk ? (n - p0) : chunk;
    const Acts ac = a.chunk(p0, c, ld);
    launch_build_xin(p, pts, viewdir, m, n_per, p0, ac.X, ld, dbg_sphere, ac.flags, st);
    resnetfc_forward(p, w, ac, ld, m, e, relu_scratch, st);
    lin_out_kernel<<<(m + 7) / 8, 256, 0, st>>>(ac.H3, w.lin_out_w, w.lin_out_b, raw_out + (size_t)p0 * w.d_out, m, w.d_out);  // resnetfc.py:163
    ++launch_counter();
  }
  return launch_counter() - c0;
}

// ---------------------------------------------------------------------------------------------------------------
size_t mlp_backward_workspace_bytes(int d_latent, int n_points) {
  const size_t m = (size_t)(n_points < train_chunk() ? n_points : train_chunk());
  // + tensor-core engines: transposed copies (2 x [512][m], X^T [ld][m]) and the transposed weights (6 x 512x512, 3 x 512 x d_latent)
  const size_t tf32_extra = ((size_t)2 * kHidden * (m + 4) + (size_t)xin_ld(d_latent) * (m + 4) + (size_t)6 * kHidden * kHidden +
                             (size_t)3 * kHidden * d_latent) * sizeof(float);
  return m * ((size_t)2 * xin_ld(d_latent) + 10 * kHidden) * sizeof(float) + kSplitKFloats * sizeof(float) + 512 + tf32_extra;
}

// The products of the backward chain, each written once for both engines.  SIMT: TN / NN kernels on the activations and
// weights as stored.  tf32 / fp32tc: every product is NT -- dW = (dY^T)(relu(X)^T)^T with K = m from transposed copies of the
// chunk, dX = dY (W^T)^T from the transposed weights.
struct ChainBackward {
  const DevParams& p;
  MatmulEngine e;
  int m, mq;                 // rows of the chunk; row stride of the transposed copies (16-byte aligned rows)
  float* SK;                 // split-K scratch
  float* Tt0; float* Tt1;    // tensor cores: dY^T, relu(X)^T
  const float* Xt;           // tensor cores: z^T of the chunk
  cudaStream_t st;

  GemmArgs accumulate_splitk() const {
    GemmArgs o;
    o.accumulate = 1; o.splitk_ws = SK; o.splitk_ws_floats = kSplitKFloats;
    return o;
  }
  // gW[M x N] += dY[m x M]^T relu?(X)[m x N]
  template <bool RELU>
  void wgrad(const float* dY, int ldy, const float* X, int ldx, float* gW, int M, int N, MatmulEngine eng) const {
    if (tensor_cores(eng)) {
      transpose<false>(dY, ldy, m, M, Tt0, mq, st);
      transpose<RELU>(X, ldx, m, N, Tt1, mq, st);
      gemm<false, true>(Tt0, mq, Tt1, mq, gW, N, M, N, m, accumulate_splitk(), eng, st);
    } else {
      gemm<true, false, false, RELU>(dY, ldy, X, ldx, gW, N, M, N, m, accumulate_splitk(), eng, st);
    }
  }
  // dX[m x 512] = (dY[m x 512] W) * (mask > 0) + R for a 512 x 512 weight W (WT = W^T)
  void dgrad(const float* dY, const float* W, const float* WT, const float* mask, const float* R, float* dX) const {
    const int H = kHidden;
    GemmArgs o;
    o.mask = mask; o.ldm = H;
    if (R) { o.R = R; o.ldr = H; }
    if (tensor_cores(e)) gemm<false, true>(dY, H, WT, H, dX, H, m, H, H, o, e, st);
    else gemm<false, false>(dY, H, W, H, dX, H, m, H, H, o, e, st);
  }
  // lin_z, whose input is the latent z (the first d_latent columns of X): gW += dY^T z, then dZ (+)= dY W (W = lin_z
  // weight, WT = W^T).  SIMT: both products per pyramid scale, a scale no point reaches returning at its flag; tensor cores: one
  // launch each, the kernel skipping the column tiles of such scales.
  void latent(const float* dY, const float* X, int ld, const float* W, const float* WT, float* gW, float* dZ, int accumulate,
              const int* flags) const {
    const int H = kHidden, DL = p.d_latent;
    if (tensor_cores(e)) {
      transpose<false>(dY, H, m, H, Tt0, mq, st);
      GemmArgs o = accumulate_splitk();
      set_segments(o, flags, 2, p.ch_off);
      gemm<false, true>(Tt0, mq, Xt, mq, gW, DL, H, DL, m, o, e, st);
      o = GemmArgs(); o.accumulate = accumulate;
      set_segments(o, flags, 2, p.ch_off);
      gemm<false, true>(dY, H, WT, H, dZ, ld, m, DL, H, o, e, st);
      return;
    }
    for (int s = 0; s < kScales; ++s) {
      GemmArgs o = accumulate_splitk();
      o.skip_if_zero = s ? flags + s : nullptr;
      gemm<true, false>(dY, H, X + p.ch_off[s], ld, gW + p.ch_off[s], DL, H, p.C[s], m, o, e, st);
      o = GemmArgs(); o.accumulate = accumulate; o.skip_if_zero = s ? flags + s : nullptr;
      gemm<false, false>(dY, H, W + p.ch_off[s], DL, dZ + p.ch_off[s], ld, m, p.C[s], H, o, e, st);
    }
  }
};

int run_point_mlp_backward_simt(const DevParams& p, const srf_mlp_weights& w, const srf_mlp_weights& gw, float* const* grad_pyr_chw,
                                const float* pts, const float* viewdir, int n, int n_per, const float* g_raw, const void* saved_base,
                                MatmulEngine e, void* workspace, size_t ws_bytes, cudaStream_t st) {
  if (ws_bytes < mlp_backward_workspace_bytes(p.d_latent, n)) return -1;
  if (!saved_base && tensor_cores(e)) return -1;   // the recompute is the SIMT chain: tensor-core gradients need that engine's forward store
  const int ld = xin_ld(p.d_latent), H = kHidden, DL = p.d_latent;
  const size_t cap = (size_t)(n < train_chunk() ? n : train_chunk());
  Acts chunk_acts;                                         // recompute buffers of one chunk
  chunk_acts.X = reinterpret_cast<float*>(workspace);
  float* dZ = chunk_acts.X + cap * ld;
  float* q = dZ + cap * ld;
  for (int b = 0; b < 3; ++b) { chunk_acts.PRE[b] = q; q += cap * H; chunk_acts.NET[b] = q; q += cap * H; }
  chunk_acts.H3 = q; q += cap * H;
  float* dH = q; q += cap * H;
  float* dN = q; q += cap * H;
  float* dP = q; q += cap * H;
  float* SK = q; q += kSplitKFloats;
  chunk_acts.flags = reinterpret_cast<int*>(q); q += 128;
  chunk_acts.whole_pass = false;
  // tensor-core engines' scratch
  const int mp = (int)((cap + 3) / 4 * 4);
  float* Tt0 = q; q += (size_t)H * mp;
  float* Tt1 = q; q += (size_t)H * mp;
  float* Xt = q; q += (size_t)ld * mp;
  float* WT0[3]; float* WT1[3]; float* WTZ[3];
  for (int b = 0; b < 3; ++b) { WT0[b] = q; q += (size_t)H * H; WT1[b] = q; q += (size_t)H * H; WTZ[b] = q; q += (size_t)H * DL; }
  if (tensor_cores(e)) {
    for (int b = 0; b < 3; ++b) {                          // W^T so that dX = dY W becomes an NT product
      transpose<false>(w.fc0_w[b], H, H, H, WT0[b], H, st);
      transpose<false>(w.fc1_w[b], H, H, H, WT1[b], H, st);
      transpose<false>(w.lin_z_w[b], DL, H, DL, WTZ[b], H, st);
    }
  }
  const Acts acts = saved_base ? saved_view(const_cast<void*>(saved_base), p.d_latent, n) : chunk_acts;
  auto G = [](const float* c) { return const_cast<float*>(c); };
  PyrGrad gp;
  for (int s = 0; s < kScales; ++s) gp.chw[s] = grad_pyr_chw[s];
  const int c0 = launch_counter();
  for (int p0 = 0, c = 0; p0 < n; p0 += train_chunk(), ++c) {
    const int m = (n - p0) < train_chunk() ? (n - p0) : train_chunk();
    const float* g_out = g_raw + (size_t)p0 * w.d_out;
    const Acts a = acts.chunk(p0, c, ld);
    if (!saved_base) {                                     // forward recompute, keeping the pre-activations
      launch_build_xin(p, pts, viewdir, m, n_per, p0, a.X, ld, nullptr, a.flags, st);
      resnetfc_forward(p, w, a, ld, m, MatmulEngine::simt, nullptr, st);
    }
    const ChainBackward bw{p, e, m, (m + 3) / 4 * 4, SK, Tt0, Tt1, Xt, st};
    // lin_out (M = d_out) and lin_in (N = 42) are narrow products: SIMT kernels in both modes
    bw.wgrad<true>(g_out, w.d_out, a.H3, H, G(gw.lin_out_w), w.d_out, H, MatmulEngine::simt);              // gW_out += g^T relu(h3)
    colsum(g_out, w.d_out, m, w.d_out, G(gw.lin_out_b), SK, st);
    lin_out_dx_kernel<<<(m * H + 255) / 256, 256, 0, st>>>(g_out, w.d_out, w.lin_out_w, a.H3, dH, m);
    ++launch_counter();
    if (tensor_cores(e)) transpose<false>(a.X, ld, m, DL, Xt, bw.mq, st);                            // z^T, once per chunk
    for (int b = 2; b >= 0; --b) {
      bw.wgrad<true>(dH, H, a.NET[b], H, G(gw.fc1_w[b]), H, H, e);                                           // gW_fc1 += dh^T relu(net)
      colsum(dH, H, m, H, G(gw.fc1_b[b]), SK, st);
      bw.dgrad(dH, w.fc1_w[b], WT1[b], a.NET[b], nullptr, dN);                                               // dnet = (dh W_fc1) * (net>0)
      bw.wgrad<true>(dN, H, a.PRE[b], H, G(gw.fc0_w[b]), H, H, e);                                           // gW_fc0 += dnet^T relu(pre)
      colsum(dN, H, m, H, G(gw.fc0_b[b]), SK, st);
      bw.dgrad(dN, w.fc0_w[b], WT0[b], a.PRE[b], dH, dP);                                                    // dpre = dh + (dnet W_fc0) * (pre>0)
      bw.latent(dP, a.X, ld, w.lin_z_w[b], WTZ[b], G(gw.lin_z_w[b]), dZ, b == 2 ? 0 : 1, a.flags);           // gW_linz += dpre^T z; dz (+)= dpre W_linz
      colsum(dP, H, m, H, G(gw.lin_z_b[b]), SK, st);
      float* tmp = dH; dH = dP; dP = tmp;                                                                    // dh <- dpre
    }
    bw.wgrad<false>(dH, H, a.X + DL, ld, G(gw.lin_in_w), H, kDX, MatmulEngine::simt);                       // gW_in += dh^T x
    colsum(dH, H, m, H, G(gw.lin_in_b), SK, st);
    scatter_latent_kernel<<<(m + 7) / 8, 256, 0, st>>>(p, pts, m, p0, dZ, ld, gp);
    ++launch_counter();
  }
  return launch_counter() - c0;
}

}  // namespace srf
