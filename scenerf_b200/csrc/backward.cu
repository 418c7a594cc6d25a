// Backward pass of the ray-render path ("next" row 8f-1 of the hot-path contract): what torch.autograd computes for
// SceneRF.render_rays_batch (scenerf/models/scenerf.py:392-748), hand-written.  float32 SIMT, the backward twin of
// mlp_simt.cu / ray_kernels.cu (strict mode); a tensor-core backward is the follow-up.
//
// Gradient structure (forward op file:line -> what is differentiated):
//   scenerf.py:662      main-MLP inputs detached: no gradient into sample positions through the MLP
//   utils.py:204-214    t = mean + eps*std (clamped at 0.1: clamped samples carry no gradient), depth_volume = t*unit_z
//   scenerf.py:704-748  compositing (cumprod backward as torch: reverse cumsum of grad*out divided by the input)
//   ray_som_kl.py:64-92 loss_kl differentiates gauss_means / gauss_stds only; som_vars is NOT differentiated here
//   scenerf.py:533-536,473-481 ; scenerf.py:585-594   heads (sigmoid, softplus(x-1), relu(.)+c)
//   resnetfc.py:133-164 ResnetFC;  utils.py:232-247  grid_sample(bilinear, zeros) w.r.t. the 5 feature maps
//
// Order: ray_backward_kernel (per ray: cotangents -> d raw MLP outputs of both passes)  ->  per chunk of points:
// recompute the float32 forward keeping pre-activations, then the GEMM chain backwards (dX = dY W, dW += dY^T X,
// db += colsum dY), then scatter d latent into the CHW feature-map gradients with atomics.
// Parameter gradients are deterministic (no atomics, fixed chunk order); feature-map gradients use float atomicAdd.
#include "kernels.cuh"

namespace srf {

constexpr int kBwdWarps = 4;
constexpr int kMaxSB = 256;
// Points per pass of the GEMM chain.  Round 1 used 9472 (74 row tiles x 4 column tiles = one wave of 296 CTAs) -- and paid for it with
// ~700 launches per 1200-ray training step; the GEMM kernels are grid-size agnostic, so a pass now covers a whole training call
// (81.6 k points fit: ~40 KB of workspace per point) and the launch count drops ~8x.  SRF_TRAIN_CHUNK overrides (multiple of 128).
static int chunk_b() {
  static int v = 0;
  if (!v) {
    const char* e = getenv("SRF_TRAIN_CHUNK");
    v = e ? atoi(e) : 98304;
    if (v < 128) v = 128;
    v = (v + 127) / 128 * 128;
  }
  return v;
}
#define kChunkB (chunk_b())
constexpr size_t kSplitKFloats = (size_t)4 * 512 * 2528;     // split-K scratch of the weight-gradient GEMMs (20 MB)

struct RayBwdSmem {
  float t[kMaxSB], z[kMaxSB], sg[kMaxSB], al[kMaxSB], T[kMaxSB], gw[kMaxSB], ga[kMaxSB], gtt[kMaxSB], gt[kMaxSB], gz[kMaxSB];
};

// one warp per ray
template <int kMaxG>
__global__ void __launch_bounds__(kBwdWarps * 32)
ray_backward_kernel(const __grid_constant__ DevParams p, int R, const float* __restrict__ raw,      // (R*S,4) main MLP output
                    const float* __restrict__ t_sorted, const float* __restrict__ unit, const float* __restrict__ gauss_raw,
                    const float* __restrict__ noise_n, srf_outputs fwd, srf_outputs cot,
                    float* __restrict__ graw_main,      // (R*S,4)
                    float* __restrict__ graw_gauss) {   // (R*G,2)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  RayBwdSmem& sm = reinterpret_cast<RayBwdSmem*>(smem_raw)[threadIdx.x >> 5];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * kBwdWarps + warp;
  if (r >= R) return;
  const int S = p.S, G = p.G, P = p.P;
  const size_t base = (size_t)r * S;
  const float uz = unit[r * 3 + 2];

  for (int j = lane; j < S; j += 32) {
    sm.t[j] = fmaxf(t_sorted[base + j], 0.0f);
    sm.z[j] = fwd.depth_volumes[base + j];
    sm.sg[j] = fwd.densities[base + j];
    sm.al[j] = fwd.alphas[base + j];
  }
  __syncwarp();
  // transmittance before each sample (same segment scan as the forward kernel)
  const int spt = (S + 31) >> 5;
  const int j0 = min(S, lane * spt), j1 = min(S, j0 + spt);
  float seg = 1.0f;
  for (int j = j0; j < j1; ++j) seg *= fadd(fsub(1.0f, sm.al[j]), 1e-10f);
  float incl = seg;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl *= v;
  }
  float Tacc = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) Tacc = 1.0f;
  for (int j = j0; j < j1; ++j) { sm.T[j] = Tacc; Tacc *= fadd(fsub(1.0f, sm.al[j]), 1e-10f); }
  __syncwarp();
  // arg-min sample of |depth - z| (scenerf.py:730-735), first index wins
  const float depth = fwd.depth[r];
  float best = __int_as_float(0x7f800000);
  int best_j = 0x7fffffff;
  for (int j = lane; j < S; j += 32) {
    const float d = fabsf(fsub(depth, sm.z[j]));
    if (d < best) { best = d; best_j = j; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oj = __shfl_xor_sync(0xffffffffu, best_j, o);
    if (ob < best || (ob == best && oj < best_j)) { best = ob; best_j = oj; }
  }
  const float dz_star = fsub(depth, sm.z[best_j]);
  const float sgn = (dz_star > 0.f) ? 1.f : ((dz_star < 0.f) ? -1.f : 0.f);
  const float c_closest = cot.closest_pts_to_depths ? cot.closest_pts_to_depths[r] : 0.f;
  const float c_wad = cot.weights_at_depth ? cot.weights_at_depth[r] : 0.f;
  const float gd = (cot.depth ? cot.depth[r] : 0.f) + sgn * c_closest;
  float cc[3] = {0.f, 0.f, 0.f};
  if (cot.color) { cc[0] = cot.color[r * 3]; cc[1] = cot.color[r * 3 + 1]; cc[2] = cot.color[r * 3 + 2]; }

  for (int j = lane; j < S; j += 32) {
    const float4 o = reinterpret_cast<const float4*>(raw)[base + j];
    const float c0 = sigmoidf_ref(o.x), c1 = sigmoidf_ref(o.y), c2 = sigmoidf_ref(o.z);
    const float w = fwd.weights[base + j];
    float gw = (cot.weights ? cot.weights[base + j] : 0.f) + gd * sm.z[j] + cc[0] * c0 + cc[1] * c1 + cc[2] * c2;
    float gz = (cot.depth_volumes ? cot.depth_volumes[base + j] : 0.f) + gd * w;
    if (j == best_j) { gw += c_wad; gz -= sgn * c_closest; }
    sm.gw[j] = gw;
    sm.gz[j] = gz;
    sm.ga[j] = (cot.alphas ? cot.alphas[base + j] : 0.f) + gw * sm.T[j];
    sm.gtt[j] = gw * sm.al[j] * sm.T[j];
    // colour head: d sigmoid
    float4 g;
    g.x = cc[0] * w * c0 * (1.f - c0);
    g.y = cc[1] * w * c1 * (1.f - c1);
    g.z = cc[2] * w * c2 * (1.f - c2);
    g.w = 0.f;
    reinterpret_cast<float4*>(graw_main)[base + j] = g;
  }
  __syncwarp();
  // suffix_k = sum_{j>k} gtt_j   (cumprod backward); ga_k -= suffix_k / s_k
  float segsum = 0.f;
  for (int j = j0; j < j1; ++j) segsum += sm.gtt[j];
  float incl_r = segsum;                         // inclusive scan from the right over lanes
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_down_sync(0xffffffffu, incl_r, o);
    if (lane + o < 32) incl_r += v;
  }
  float suffix = __shfl_down_sync(0xffffffffu, incl_r, 1);
  if (lane == 31) suffix = 0.f;
  for (int j = j1 - 1; j >= j0; --j) {
    sm.ga[j] -= suffix / fadd(fsub(1.0f, sm.al[j]), 1e-10f);
    suffix += sm.gtt[j];
  }
  __syncwarp();
  // alpha = 1 - exp(-delta*sigma)
  for (int j = lane; j < S; j += 32) {
    const float delta = (j == 0) ? sm.t[0] : fsub(sm.t[j], sm.t[j - 1]);
    const float E = expf(-fmul(delta, sm.sg[j]));
    const float ga = sm.ga[j];
    sm.gtt[j] = ga * sm.sg[j] * E;               // reuse: g_delta
    const float gsig = (cot.densities ? cot.densities[base + j] : 0.f) + ga * delta * E;
    const float x3 = fsub(raw[(base + j) * 4 + 3], 1.0f);
    const float dsoft = (x3 > 20.0f) ? 1.0f : fdiv(1.0f, fadd(1.0f, expf(-x3)));
    graw_main[(base + j) * 4 + 3] = gsig * dsoft;
  }
  __syncwarp();
  for (int j = lane; j < S; j += 32) {
    float gt = sm.gtt[j] - ((j + 1 < S) ? sm.gtt[j + 1] : 0.f);
    if (t_sorted[base + j] < 0.f) gt = 0.f;      // scenerf.py:707 (never active: samples are >= 0.1)
    sm.gt[j] = gt + sm.gz[j] * uz;               // depth_volume = t * unit_z (utils.py:216)
  }
  __syncwarp();
  // route to the gaussian that produced each sample (utils.py:204-214)
  float gm[kMaxG], gs[kMaxG];
#pragma unroll
  for (int g = 0; g < kMaxG; ++g) { gm[g] = 0.f; gs[g] = 0.f; }
  for (int i = lane; i < G * P; i += 32) {
    const int g = i / P;
    const float m = fwd.gaussian_means[(size_t)r * G + g], s = fwd.gaussian_stds[(size_t)r * G + g];
    const float e = noise_n ? noise_n[(size_t)r * G * P + i] : philox_normal(p.seed, (uint32_t)r + p.ray0, (uint32_t)i);
    const float t = fadd(m, fmul(e, s));
    if (t < 0.1f) continue;
    int lo = 0, hi = S;                          // lower_bound of t in the sorted distances (same float as the forward wrote)
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (sm.t[mid] < t) lo = mid + 1; else hi = mid; }
    const float gt = (lo < S) ? sm.gt[lo] : 0.f;
#pragma unroll
    for (int k = 0; k < kMaxG; ++k) if (k == g) { gm[k] += gt; gs[k] += gt * e; }
  }
#pragma unroll
  for (int g = 0; g < kMaxG; ++g) { gm[g] = warp_sum(gm[g]); gs[g] = warp_sum(gs[g]); }
  if (lane == 0) {
    const float c_kl = cot.loss_kl ? cot.loss_kl[r] : 0.f;
    for (int g = 0; g < G; ++g) {
      const size_t ig = (size_t)r * G + g;
      const float m1 = fwd.gaussian_means[ig], s1 = fwd.gaussian_stds[ig];
      const float m2 = fwd.som_means[ig], nv = fwd.som_vars[ig];
      const float mean_diff = fabsf(fsub(m1, m2));
      const float var_diff = fabsf(fsub(sqrtf(fmul(s1, s1)), sqrtf(nv)));
      const bool mask = (mean_diff > 0.1f) && (var_diff > 0.1f) && (nv > 0.0f);
      float s2 = sqrtf(nv);
      if (s2 < 1.5f) s2 = 1.5f;
      float g_mean = gm[0], g_std = gs[0];
#pragma unroll
      for (int k = 1; k < kMaxG; ++k) if (k == g) { g_mean = gm[k]; g_std = gs[k]; }
      g_mean += cot.gaussian_means ? cot.gaussian_means[ig] : 0.f;
      g_std += cot.gaussian_stds ? cot.gaussian_stds[ig] : 0.f;
      if (mask) {
        const float gk = c_kl / (float)G;
        g_mean += gk * (m1 - m2) / (s2 * s2);
        g_std += gk * (-(s2 / (s1 * s1)) / (s2 / s1 + 1e-8f) + s1 / (s2 * s2));
      }
      const float m0 = linspace_at(p.g_start, p.g_end, G, g);
      const float o0 = gauss_raw[ig * 2 + 0], o1 = gauss_raw[ig * 2 + 1];
      graw_gauss[ig * 2 + 0] = (fadd(m0, o0) > 0.f) ? g_mean : 0.f;
      graw_gauss[ig * 2 + 1] = (fadd(o1, p.base_std) > 0.f) ? g_std : 0.f;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
struct GemmOpt {
  const float* bias = nullptr;
  const float* mask = nullptr; int ldm = 0;
  const float* R = nullptr; int ldr = 0;
  int accumulate = 0;
  float* splitk_ws = nullptr; size_t splitk_ws_floats = 0;
  const int* skip = nullptr;
  const int* seg_flags = nullptr; int seg_mode = 0; const int* seg_off = nullptr;     // tf32 kernel: fused per-scale segments
  float* relu_out = nullptr; int ld_relu = 0;                                         // tf32 kernel: also store max(result, 0)
};
// SRF_FLAG_TF32_MATMUL: NT GEMMs without operand ReLU go to the wgmma tf32 kernel (gemm_tf32.cu); the callers
// below arrange their operands accordingly (ReLU'd / transposed copies).  Set per call by the run_* entry points.
static thread_local bool g_tf32 = false;

static void relu_copy_2d(const float* src, int lds, float* dst, int ldd, int M, int N, cudaStream_t st);
template <bool AT, bool BT, bool RA, bool RB>
static void gemm(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K, const GemmOpt& o,
                 cudaStream_t st) {
  GemmArgs g;
  g.A = A; g.lda = lda; g.at = AT; g.relu_a = RA; g.B = B; g.ldb = ldb; g.bt = BT; g.relu_b = RB;
  g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = K;
  g.bias = o.bias; g.mask = o.mask; g.ldm = o.ldm; g.R = o.R; g.ldr = o.ldr; g.accumulate = o.accumulate;
  g.splitk_ws = o.splitk_ws; g.splitk_ws_floats = o.splitk_ws_floats; g.skip_if_zero = o.skip;
  if (o.seg_flags) { g.seg_flags = o.seg_flags; g.seg_mode = o.seg_mode; for (int i = 0; i < 6; ++i) g.seg_off[i] = o.seg_off[i]; }
  g.relu_out = o.relu_out; g.ld_relu = o.ld_relu;
  if (g_tf32 && !AT && BT && !RA && !RB && launch_gemm_tf32(g, st) == 0) return;
  launch_gemm(g, st);
  if (o.relu_out) relu_copy_2d(C, ldc, o.relu_out, o.ld_relu, M, N, st);      // SIMT fallback of a tf32-mode call
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
static void colsum(const float* dY, int ld, int M, int N, float* gb, float* scratch, cudaStream_t st) {
  colsum_partial_kernel<<<dim3((N + 31) / 32, kColSegs), 256, 0, st>>>(dY, ld, M, N, scratch);
  colsum_final_kernel<<<(N + 255) / 256, 256, 0, st>>>(scratch, N, gb);
  launch_counter() += 2;
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
template <bool RELU>
static void transpose(const float* src, int lds, int rows, int cols, float* dst, int ldd, cudaStream_t st) {
  transpose_kernel<RELU><<<dim3((cols + 31) / 32, (rows + 31) / 32), 256, 0, st>>>(src, lds, rows, cols, dst, ldd);
  ++launch_counter();
}
__global__ void __launch_bounds__(256) relu_kernel(const float4* __restrict__ src, float4* __restrict__ dst, size_t n4) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 v = src[i];
  v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
  dst[i] = v;
}
static void relu_copy(const float* src, float* dst, size_t n, cudaStream_t st) {
  relu_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float4*>(src), reinterpret_cast<float4*>(dst), n / 4);
  ++launch_counter();
}
static void relu_copy_2d(const float* src, int lds, float* dst, int ldd, int M, int N, cudaStream_t st) {
  if (lds == N && ldd == N) { relu_copy(src, dst, (size_t)M * N, st); return; }
  for (int m = 0; m < M; ++m) relu_copy(src + (size_t)m * lds, dst + (size_t)m * ldd, (size_t)N, st);     // not used by the callers here
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

static inline int xin_ld_b(int d_latent) { return ((d_latent + kDX + 31) / 32) * 32; }

size_t mlp_backward_workspace_bytes(int d_latent, int n_points) {
  const size_t m = (size_t)(n_points < kChunkB ? n_points : kChunkB);
  // + tf32 mode: transposed copies (2 x [512][m], X^T [ld][m]) and the transposed weights (6 x 512x512, 3 x 512 x d_latent)
  const size_t tf32_extra = ((size_t)2 * kHidden * (m + 4) + (size_t)xin_ld_b(d_latent) * (m + 4) + (size_t)6 * kHidden * kHidden +
                             (size_t)3 * kHidden * d_latent) * sizeof(float);
  return m * ((size_t)2 * xin_ld_b(d_latent) + 10 * kHidden) * sizeof(float) + kSplitKFloats * sizeof(float) + 512 + tf32_extra;
}

// Activations of the float32 forward that the backward needs, for ALL points of a pass (SRF_FLAG_SAVE_ACTIVATIONS): the
// training forward writes them once and the backward skips its recompute.  Layout: X (n,ld) | PRE[3] NET[3] H3 (n,512) |
// per-chunk scale flags (8 ints per chunk).
struct SavedActs { float* X; float* PRE[3]; float* NET[3]; float* H3; int* flags; };
static inline size_t n_chunks_b(int n) { return ((size_t)n + kChunkB - 1) / kChunkB; }
size_t mlp_forward_save_scratch_bytes(int n_points) {           // two ReLU'd operand buffers of one pass (tf32 mode)
  return (size_t)2 * (size_t)(n_points < kChunkB ? n_points : kChunkB) * kHidden * sizeof(float) + 256;
}
size_t mlp_saved_bytes(int d_latent, int n_points) {
  return (size_t)n_points * ((size_t)xin_ld_b(d_latent) + 7 * kHidden) * sizeof(float) + n_chunks_b(n_points) * 8 * sizeof(int) + 256;
}
static SavedActs saved_view(void* base, int d_latent, int n) {
  SavedActs a;
  float* q = reinterpret_cast<float*>(base);
  a.X = q; q += (size_t)n * xin_ld_b(d_latent);
  for (int b = 0; b < 3; ++b) { a.PRE[b] = q; q += (size_t)n * kHidden; a.NET[b] = q; q += (size_t)n * kHidden; }
  a.H3 = q; q += (size_t)n * kHidden;
  a.flags = reinterpret_cast<int*>(q);
  return a;
}

// resnetfc.py:133-164 for m points keeping the pre-activations: PRE[b] = h + lin_z_b(z), NET[b] = fc_0(relu(PRE[b])),
// H3 = h after block 2.
// relu_scratch: m x 512 floats, used only in tf32 mode (the tensor-core GEMM takes its A operand as stored, so the
// ReLU'd activations are materialised first).
static void forward_chunk(const DevParams& p, const srf_mlp_weights& w, const float* X, int ld, float* const* PRE, float* const* NET,
                         float* H3, int m, const int* scale_any, float* relu_scratch, cudaStream_t st) {
  const int H = kHidden, DL = p.d_latent;
  GemmOpt o;
  o.bias = w.lin_in_b;
  gemm<false, true, false, false>(X + DL, ld, w.lin_in_w, kDX, PRE[0], H, m, H, kDX, o, st);                   // h0 = lin_in(x)
  for (int b = 0; b < 3; ++b) {
    if (g_tf32 && relu_scratch) {                                                                              // one launch, dead scales' k-blocks skipped in the kernel
      o = GemmOpt(); o.bias = w.lin_z_b[b]; o.R = (b == 0) ? PRE[0] : H3; o.ldr = H;
      o.seg_flags = scale_any; o.seg_mode = 1; o.seg_off = p.ch_off;
      o.relu_out = relu_scratch; o.ld_relu = H;                                                                // relu(pre): fc_0's operand, from this epilogue
      gemm<false, true, false, false>(X, ld, w.lin_z_w[b], DL, PRE[b], H, m, H, DL, o, st);
    } else
    for (int s = 0; s < kScales; ++s) {                                                                        // pre = h + lin_z(z), one K-segment per scale
      o = GemmOpt();
      if (s == 0) { o.bias = w.lin_z_b[b]; o.R = (b == 0) ? PRE[0] : H3; o.ldr = H; }
      else { o.accumulate = 1; o.skip = scale_any + s; }
      gemm<false, true, false, false>(X + p.ch_off[s], ld, w.lin_z_w[b] + p.ch_off[s], DL, PRE[b], H, m, H, p.C[s], o, st);
    }
    if (g_tf32 && relu_scratch) {
      float* relu2 = relu_scratch + (size_t)m * H;
      o = GemmOpt(); o.bias = w.fc0_b[b]; o.relu_out = relu2; o.ld_relu = H;
      gemm<false, true, false, false>(relu_scratch, H, w.fc0_w[b], H, NET[b], H, m, H, H, o, st);              // net = fc_0(relu(pre)); relu(net) on the side
      o = GemmOpt(); o.bias = w.fc1_b[b]; o.R = PRE[b]; o.ldr = H;
      gemm<false, true, false, false>(relu2, H, w.fc1_w[b], H, H3, H, m, H, H, o, st);                         // h = pre + fc_1(relu(net))
    } else {
      o = GemmOpt(); o.bias = w.fc0_b[b];
      gemm<false, true, true, false>(PRE[b], H, w.fc0_w[b], H, NET[b], H, m, H, H, o, st);                     // net = fc_0(relu(pre))
      o = GemmOpt(); o.bias = w.fc1_b[b]; o.R = PRE[b]; o.ldr = H;
      gemm<false, true, true, false>(NET[b], H, w.fc1_w[b], H, H3, H, m, H, H, o, st);                         // h = pre + fc_1(relu(net))
    }
  }
}

// Training forward of one pass: same arithmetic as run_point_mlp_simt (bit-identical raw outputs), activations kept.
int run_point_mlp_forward_save(const DevParams& p, const srf_mlp_weights& w, const float* pts, const float* viewdir, int n, int n_per,
                               float* raw_out, int32_t* dbg_sphere, void* saved_base, int tf32_matmul, void* scratch, size_t scratch_bytes,
                               cudaStream_t st) {
  const int ld = xin_ld_b(p.d_latent), H = kHidden;
  g_tf32 = tf32_matmul != 0;
  float* relu_scratch = reinterpret_cast<float*>(scratch);
  if (g_tf32 && scratch_bytes < mlp_forward_save_scratch_bytes(n)) return -1;
  const SavedActs a = saved_view(saved_base, p.d_latent, n);
  const int c0 = launch_counter();
  int chunk = 0;
  for (int p0 = 0; p0 < n; p0 += kChunkB, ++chunk) {
    const int m = (n - p0) < kChunkB ? (n - p0) : kChunkB;
    float* X = a.X + (size_t)p0 * ld;
    float* PRE[3]; float* NET[3];
    for (int b = 0; b < 3; ++b) { PRE[b] = a.PRE[b] + (size_t)p0 * H; NET[b] = a.NET[b] + (size_t)p0 * H; }
    float* H3 = a.H3 + (size_t)p0 * H;
    int* flags = a.flags + chunk * 8;
    launch_build_xin(p, pts, viewdir, m, n_per, p0, X, ld, dbg_sphere, flags, st);
    forward_chunk(p, w, X, ld, PRE, NET, H3, m, flags, relu_scratch, st);
    launch_lin_out(H3, w.lin_out_w, w.lin_out_b, raw_out + (size_t)p0 * w.d_out, m, w.d_out, st);
  }
  return launch_counter() - c0;
}

// grads: same layout as the weights (accumulated into); pyramid grads CHW (accumulated into).  saved_base: activations of
// run_point_mlp_forward_save for the same points, or NULL (the forward is then recomputed chunk by chunk).
// Returns launches or -1.
int run_point_mlp_backward_simt(const DevParams& p, const srf_mlp_weights& w, const srf_mlp_weights& gw, float* const* grad_pyr_chw,
                                const float* pts, const float* viewdir, int n, int n_per, const float* g_raw, const void* saved_base,
                                int tf32_matmul, void* workspace, size_t ws_bytes, cudaStream_t st) {
  if (ws_bytes < mlp_backward_workspace_bytes(p.d_latent, n)) return -1;
  g_tf32 = tf32_matmul != 0;
  const int ld = xin_ld_b(p.d_latent), H = kHidden, DL = p.d_latent;
  const size_t cap = (size_t)(n < kChunkB ? n : kChunkB);
  float* Xc = reinterpret_cast<float*>(workspace);
  float* dZ = Xc + cap * ld;
  float* PREc[3]; float* NETc[3];
  float* q = dZ + cap * ld;
  for (int b = 0; b < 3; ++b) { PREc[b] = q; q += cap * H; NETc[b] = q; q += cap * H; }
  float* H3c = q; q += cap * H;
  float* dH = q; q += cap * H;
  float* dN = q; q += cap * H;
  float* dP = q; q += cap * H;
  float* SK = q; q += kSplitKFloats;
  int* flags_c = reinterpret_cast<int*>(q); q += 128;
  // tf32 mode scratch
  const int mp = (int)((cap + 3) / 4 * 4);                 // row stride of the transposed activations (16-byte aligned rows)
  float* Tt0 = q; q += (size_t)H * mp;                     // dY^T
  float* Tt1 = q; q += (size_t)H * mp;                     // relu(X)^T
  float* Xt = q; q += (size_t)ld * mp;                     // z^T (all latent columns)
  float* WT0[3]; float* WT1[3]; float* WTZ[3];
  for (int b = 0; b < 3; ++b) { WT0[b] = q; q += (size_t)H * H; WT1[b] = q; q += (size_t)H * H; WTZ[b] = q; q += (size_t)H * DL; }
  if (g_tf32) {
    for (int b = 0; b < 3; ++b) {                          // W^T so that dX = dY W becomes an NT product
      transpose<false>(w.fc0_w[b], H, H, H, WT0[b], H, st);
      transpose<false>(w.fc1_w[b], H, H, H, WT1[b], H, st);
      transpose<false>(w.lin_z_w[b], DL, H, DL, WTZ[b], H, st);
    }
  }
  SavedActs sv;
  if (saved_base) sv = saved_view(const_cast<void*>(saved_base), p.d_latent, n);
  auto G = [](const float* c) { return const_cast<float*>(c); };
  PyrGrad gp;
  for (int s = 0; s < kScales; ++s) gp.chw[s] = grad_pyr_chw[s];
  const int c0 = launch_counter();
  int chunk = 0;
  for (int p0 = 0; p0 < n; p0 += kChunkB, ++chunk) {
    const int m = (n - p0) < kChunkB ? (n - p0) : kChunkB;
    const float* g_out = g_raw + (size_t)p0 * w.d_out;
    float* X = Xc; float* H3 = H3c; int* scale_any = flags_c;
    float* PRE[3] = {PREc[0], PREc[1], PREc[2]};
    float* NET[3] = {NETc[0], NETc[1], NETc[2]};
    GemmOpt o;
    if (saved_base) {
      X = sv.X + (size_t)p0 * ld; H3 = sv.H3 + (size_t)p0 * H; scale_any = sv.flags + chunk * 8;
      for (int b = 0; b < 3; ++b) { PRE[b] = sv.PRE[b] + (size_t)p0 * H; NET[b] = sv.NET[b] + (size_t)p0 * H; }
    } else {
      // ---- forward recompute, keeping pre-activations (resnetfc.py:133-164) ----
      launch_build_xin(p, pts, viewdir, m, n_per, p0, X, ld, nullptr, scale_any, st);
      forward_chunk(p, w, X, ld, PRE, NET, H3, m, scale_any, dN, st);
    }
    // ---- backward ----
    o = GemmOpt(); o.accumulate = 1; o.splitk_ws = SK; o.splitk_ws_floats = kSplitKFloats;
    gemm<true, false, false, true>(g_out, w.d_out, H3, H, G(gw.lin_out_w), H, w.d_out, H, m, o, st);           // gW_out += g^T relu(h3)
    colsum(g_out, w.d_out, m, w.d_out, G(gw.lin_out_b), SK, st);
    lin_out_dx_kernel<<<(m * H + 255) / 256, 256, 0, st>>>(g_out, w.d_out, w.lin_out_w, H3, dH, m);
    ++launch_counter();
    if (g_tf32) {
      // every product as NT on tensor cores: dW = (dY^T)(relu(X)^T)^T with K = m, dX = dY (W^T)^T
      const int mq = (m + 3) / 4 * 4;
      transpose<false>(X, ld, m, DL, Xt, mq, st);                                                              // z^T, once per chunk
      for (int b = 2; b >= 0; --b) {
        transpose<false>(dH, H, m, H, Tt0, mq, st);
        transpose<true>(NET[b], H, m, H, Tt1, mq, st);
        o = GemmOpt(); o.accumulate = 1; o.splitk_ws = SK; o.splitk_ws_floats = kSplitKFloats;
        gemm<false, true, false, false>(Tt0, mq, Tt1, mq, G(gw.fc1_w[b]), H, H, H, m, o, st);                  // gW_fc1 += dh^T relu(net)
        colsum(dH, H, m, H, G(gw.fc1_b[b]), SK, st);
        o = GemmOpt(); o.mask = NET[b]; o.ldm = H;
        gemm<false, true, false, false>(dH, H, WT1[b], H, dN, H, m, H, H, o, st);                              // dnet = (dh W_fc1) * (net>0)
        transpose<false>(dN, H, m, H, Tt0, mq, st);
        transpose<true>(PRE[b], H, m, H, Tt1, mq, st);
        o = GemmOpt(); o.accumulate = 1; o.splitk_ws = SK; o.splitk_ws_floats = kSplitKFloats;
        gemm<false, true, false, false>(Tt0, mq, Tt1, mq, G(gw.fc0_w[b]), H, H, H, m, o, st);                  // gW_fc0 += dnet^T relu(pre)
        colsum(dN, H, m, H, G(gw.fc0_b[b]), SK, st);
        o = GemmOpt(); o.mask = PRE[b]; o.ldm = H; o.R = dH; o.ldr = H;
        gemm<false, true, false, false>(dN, H, WT0[b], H, dP, H, m, H, H, o, st);                              // dpre = dh + (dnet W_fc0) * (pre>0)
        transpose<false>(dP, H, m, H, Tt0, mq, st);
        // latent axis = output columns here: column tiles that lie in dead scales are skipped in the kernel (one launch each)
        o = GemmOpt(); o.accumulate = 1; o.splitk_ws = SK; o.splitk_ws_floats = kSplitKFloats;
        o.seg_flags = scale_any; o.seg_mode = 2; o.seg_off = p.ch_off;
        gemm<false, true, false, false>(Tt0, mq, Xt, mq, G(gw.lin_z_w[b]), DL, H, DL, m, o, st);                // gW_linz += dpre^T z
        o = GemmOpt(); o.accumulate = (b == 2) ? 0 : 1; o.seg_flags = scale_any; o.seg_mode = 2; o.seg_off = p.ch_off;
        gemm<false, true, false, false>(dP, H, WTZ[b], H, dZ, ld, m, DL, H, o, st);                             // dz (+)= dpre W_linz
        colsum(dP, H, m, H, G(gw.lin_z_b[b]), SK, st);
        float* tmp = dH; dH = dP; dP = tmp;
      }
    } else
    for (int b = 2; b >= 0; --b) {
      o = GemmOpt(); o.accumulate = 1; o.splitk_ws = SK; o.splitk_ws_floats = kSplitKFloats;
      gemm<true, false, false, true>(dH, H, NET[b], H, G(gw.fc1_w[b]), H, H, H, m, o, st);                     // gW_fc1 += dh^T relu(net)
      colsum(dH, H, m, H, G(gw.fc1_b[b]), SK, st);
      o = GemmOpt(); o.mask = NET[b]; o.ldm = H;
      gemm<false, false, false, false>(dH, H, w.fc1_w[b], H, dN, H, m, H, H, o, st);                           // dnet = (dh W_fc1) * (net>0)
      o = GemmOpt(); o.accumulate = 1; o.splitk_ws = SK; o.splitk_ws_floats = kSplitKFloats;
      gemm<true, false, false, true>(dN, H, PRE[b], H, G(gw.fc0_w[b]), H, H, H, m, o, st);                     // gW_fc0 += dnet^T relu(pre)
      colsum(dN, H, m, H, G(gw.fc0_b[b]), SK, st);
      o = GemmOpt(); o.mask = PRE[b]; o.ldm = H; o.R = dH; o.ldr = H;
      gemm<false, false, false, false>(dN, H, w.fc0_w[b], H, dP, H, m, H, H, o, st);                           // dpre = dh + (dnet W_fc0) * (pre>0)
      for (int s = 0; s < kScales; ++s) {
        o = GemmOpt(); o.accumulate = 1; o.splitk_ws = SK; o.splitk_ws_floats = kSplitKFloats; o.skip = s ? scale_any + s : nullptr;
        gemm<true, false, false, false>(dP, H, X + p.ch_off[s], ld, G(gw.lin_z_w[b]) + p.ch_off[s], DL, H, p.C[s], m, o, st);   // gW_linz += dpre^T z
        o = GemmOpt(); o.accumulate = (b == 2) ? 0 : 1; o.skip = s ? scale_any + s : nullptr;
        gemm<false, false, false, false>(dP, H, w.lin_z_w[b] + p.ch_off[s], DL, dZ + p.ch_off[s], ld, m, p.C[s], H, o, st);      // dz (+)= dpre W_linz
      }
      colsum(dP, H, m, H, G(gw.lin_z_b[b]), SK, st);
      float* tmp = dH; dH = dP; dP = tmp;                                                                      // dh <- dpre
    }
    o = GemmOpt(); o.accumulate = 1; o.splitk_ws = SK; o.splitk_ws_floats = kSplitKFloats;
    gemm<true, false, false, false>(dH, H, X + DL, ld, G(gw.lin_in_w), kDX, H, kDX, m, o, st);                 // gW_in += dh^T x
    colsum(dH, H, m, H, G(gw.lin_in_b), SK, st);
    scatter_latent_kernel<<<(m + 7) / 8, 256, 0, st>>>(p, pts, m, p0, dZ, ld, gp);
    ++launch_counter();
  }
  return launch_counter() - c0;
}

void launch_ray_backward(const DevParams& p, int R, const float* raw, const float* t_sorted, const float* unit,
                         const float* gauss_raw, const float* noise_n, const srf_outputs& fwd, const srf_outputs& cot,
                         float* graw_main, float* graw_gauss, cudaStream_t st) {
  const int blocks = (R + kBwdWarps - 1) / kBwdWarps;
  const size_t smem = kBwdWarps * sizeof(RayBwdSmem);
  if (p.G <= 4) {
    cudaFuncSetAttribute(ray_backward_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    ray_backward_kernel<4><<<blocks, kBwdWarps * 32, smem, st>>>(p, R, raw, t_sorted, unit, gauss_raw, noise_n, fwd, cot, graw_main, graw_gauss);
  } else {
    cudaFuncSetAttribute(ray_backward_kernel<kMaxGaussians>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    ray_backward_kernel<kMaxGaussians><<<blocks, kBwdWarps * 32, smem, st>>>(p, R, raw, t_sorted, unit, gauss_raw, noise_n, fwd, cot, graw_main, graw_gauss);
  }
}

}  // namespace srf
