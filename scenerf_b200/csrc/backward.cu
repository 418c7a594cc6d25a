// Backward pass of the ray-render path ("next" row 8f-1 of the hot-path contract): what torch.autograd computes for
// SceneRF.render_rays_batch (scenerf/models/scenerf.py:392-748), hand-written: the compositing half.  The ResnetFC half
// (the float32 chain backwards and the scatter into the feature-map gradients) is in mlp_simt.cu.
//
// Gradient structure (forward op file:line -> what is differentiated):
//   scenerf.py:662      main-MLP inputs detached: no gradient into sample positions through the MLP
//   utils.py:204-214    t = mean + eps*std (clamped at 0.1: clamped samples carry no gradient), depth_volume = t*unit_z
//   scenerf.py:704-748  compositing (cumprod backward as torch: reverse cumsum of grad*out divided by the input)
//   ray_som_kl.py:64-92 loss_kl differentiates gauss_means / gauss_stds only; som_vars is NOT differentiated here
//   scenerf.py:533-536,473-481 ; scenerf.py:585-594   heads (sigmoid, softplus(x-1), relu(.)+c)
//   resnetfc.py:133-164 ResnetFC;  utils.py:232-247  grid_sample(bilinear, zeros) w.r.t. the 5 feature maps
//
// Order: ray_backward_kernel (per ray: cotangents -> d raw MLP outputs of both passes)  ->  run_point_mlp_backward_simt
// for each of the two MLP passes.
#include "kernels.cuh"

namespace srf {

constexpr int kBwdWarps = 4;
constexpr int kMaxSB = 256;

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
