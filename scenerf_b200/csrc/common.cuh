// Shared device-side definitions for the SceneRF ray-render kernels (sm_90a).
//
// The per-point geometry below restates, operation by operation, what the reference does in
//   utils.py:298-315 (cam_pts_2_pix), spherical_mapping.py:8-18,80-115 (pixel -> integer sphere coords),
//   pe.py:32-43 (positional encoding) and utils.py:232-247 + ATen grid_sampler_2d (bilinear taps),
// using explicit round-to-nearest intrinsics so that nvcc never contracts a multiply-add the reference performs as
// two roundings (at |x*f| ~ 1e4 rad one float32 ulp is 1e-3 rad -- fusing would change sin() in the third digit).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/scenerf_b200.h"

namespace srf {

constexpr int kScales = SRF_NUM_SCALES;
constexpr int kHidden = SRF_D_HIDDEN;
constexpr int kDX = SRF_D_X;        // 42
constexpr int kDPE = 39;
constexpr int kMaxGaussians = SRF_MAX_GAUSSIANS;

// Everything a kernel needs to know about one render call; passed by value (__grid_constant__).
struct DevParams {
  float K[9], invK[9], T[16];
  float v_min, v_fov, h_min, h_fov;
  float sphW1, sphH1;                 // float(sphere_W - 1), float(sphere_H - 1)
  int sphere_W, sphere_H;
  float max_depth, base_std, add_const, som_sigma;
  float g_start, g_end;               // float32(step/2), float32(max_depth - step/2), step = max_depth/n_gaussians (scenerf.py:554-560)
  float uni_step;                     // float32((max_depth - 0.2)/U)  (utils.py:77)
  float two_sig2;                     // float32(2*som_sigma**2)       (ray_som_kl.py:91)
  int U, G, P, S;
  // pyramid (channels-last)
  const void* feat[kScales];          // [H][W][C] float, or __half when feat_fp16
  int feat_fp16;
  int C[kScales], H[kScales], W[kScales];
  int ch_off[kScales + 1];            // prefix sums of C
  float normW[kScales], normH[kScales];   // grid normaliser: (W,H) for scale 1, (W//s, H//s) otherwise (scenerf.py:522-525)
  float halfW[kScales], halfH[kScales];   // float(W_t/2), float(H_t/2): ATen CPU unnormalise scaling factor
  int d_latent;                       // sum C
  uint64_t seed;
  const void* preproj;                // srf_pyramid.latent_table (pre-projected lin_z of the network of THIS pass) or null
  const void* preproj_gauss;          // srf_pyramid.latent_table_gauss (api.cu moves it into `preproj` for the proposal pass)
  int preproj_fp16;
  uint32_t ray0;                      // srf_config.ray_offset: Philox counter of ray r is (seed, ray0 + r, sample)
};

__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }

// (3x3 row-major) * (x,y,z), left-to-right accumulation like the oracle's _mm3.
__device__ __forceinline__ void mat3_mul(const float* M, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = fadd(fadd(fmul(M[0], x), fmul(M[1], y)), fmul(M[2], z));
  oy = fadd(fadd(fmul(M[3], x), fmul(M[4], y)), fmul(M[5], z));
  oz = fadd(fadd(fmul(M[6], x), fmul(M[7], y)), fmul(M[8], z));
}

// utils.py:272-282: T (4x4 row-major) applied to (x,y,z,1).
__device__ __forceinline__ void rigid_transform(const float* T, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = fadd(fadd(fadd(fmul(T[0], x), fmul(T[1], y)), fmul(T[2], z)), T[3]);
  oy = fadd(fadd(fadd(fmul(T[4], x), fmul(T[5], y)), fmul(T[6], z)), T[7]);
  oz = fadd(fadd(fadd(fmul(T[8], x), fmul(T[9], y)), fmul(T[10], z)), T[11]);
}

// utils.py:177-182 / utils.py:134-138: d = inv_K[:3,:3] [px,py,1]; unit = d / max(|d|, 1e-12).
__device__ __forceinline__ void pixel_direction(const DevParams& p, float px, float py, float* d, float* unit) {
  mat3_mul(p.invK, px, py, 1.0f, d[0], d[1], d[2]);
  float n = sqrtf(fadd(fadd(fmul(d[0], d[0]), fmul(d[1], d[1])), fmul(d[2], d[2])));
  n = fmaxf(n, 1e-12f);
  unit[0] = fdiv(d[0], n); unit[1] = fdiv(d[1], n); unit[2] = fdiv(d[2], n);
}

constexpr int kSphereInvalid = -(1 << 28);   // any value far outside every feature map -> all taps masked

// cam point (infer frame) -> rounded integer sphere coordinates.
//   utils.py:298-315 : pix = (K p).xy / (K p).z if (K p).z > 0 else (-1,-1)
//   spherical_mapping.py:80-115 : c = inv_K [pix,1]; v = acos(-c.y/|c|)/pi*180; h = 180 - atan2(c.z,c.x)/pi*180;
//                                 s = round((angle - min)/fov * (size-1))   (half-to-even, then .long())
__device__ __forceinline__ void point_to_sphere(const DevParams& p, float x, float y, float z, int& sx, int& sy) {
  float hx, hy, hz;
  mat3_mul(p.K, x, y, z, hx, hy, hz);
  float pixx = -1.0f, pixy = -1.0f;
  if (hz > 0.0f) { pixx = fdiv(hx, hz); pixy = fdiv(hy, hz); }
  float cx, cy, cz;
  mat3_mul(p.invK, pixx, pixy, 1.0f, cx, cy, cz);
  const float dist = sqrtf(fadd(fadd(fmul(cx, cx), fmul(cy, cy)), fmul(cz, cz)));
  const float kPi = 3.14159274101257324f;   // float32(math.pi)
  const float v = fmul(fdiv(acosf(fdiv(-cy, dist)), kPi), 180.0f);
  const float h = fsub(180.0f, fmul(fdiv(atan2f(cz, cx), kPi), 180.0f));
  const float fx = fmul(fdiv(fsub(h, p.h_min), p.h_fov), p.sphW1);
  const float fy = fmul(fdiv(fsub(v, p.v_min), p.v_fov), p.sphH1);
  // rintf == round-half-to-even == torch.round.  Non-finite / absurd values can only ever address zero padding.
  sx = (fabsf(fx) < 1e8f) ? __float2int_rn(fx) : kSphereInvalid;
  sy = (fabsf(fy) < 1e8f) ? __float2int_rn(fy) : kSphereInvalid;
}

// pe.py:32-43: out[0..2] = x ; out[3 + j*3 + c] = sin(x_c * f_{j/2} + phase_{j%2}), f_k = pi 2^k, phase = {0, pi/2}.
template <typename Store>
__device__ __forceinline__ void positional_encoding(float x, float y, float z, Store&& store) {
  const float kPi = 3.14159274101257324f;
  const float kHalfPi = 1.57079637050628662f;   // float32(np.pi * 0.5)
  const float c[3] = {x, y, z};
  store(0, x); store(1, y); store(2, z);
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const float f = kPi * (float)(1 << k);      // exact power-of-two scaling of float32(pi)
#pragma unroll
    for (int ph = 0; ph < 2; ++ph) {
#pragma unroll
      for (int cc = 0; cc < 3; ++cc) {
        float arg = fmul(c[cc], f);
        if (ph) arg = fadd(kHalfPi, arg);
        store(3 + (2 * k + ph) * 3 + cc, sinf(arg));
      }
    }
  }
}

// Bilinear taps of one scale for integer sphere coords (utils.py:237 normalise, ATen CPU grid_sampler_2d:
// ix = (g+1)*(W/2) - 0.5 ; x_w = floor(ix) ; w = ix - x_w ; e = 1 - w ; weights nw=s*e, ne=s*w, sw=n*e, se=n*w).
struct Taps {
  int off[4];     // element offset of the tap's first channel in the HWC map, or -1 if the tap is out of range
  float w[4];     // nw, ne, sw, se
  float fx, fy;   // fractional x / y position (w and n below): w[] = {(1-fy)(1-fx), (1-fy)fx, fy(1-fx), fy fx}
  bool any;
};

__device__ __forceinline__ Taps scale_taps(const DevParams& p, int s, int sx, int sy) {
  Taps t;
  const float gx = fsub(fmul(fdiv((float)sx, p.normW[s]), 2.0f), 1.0f);
  const float gy = fsub(fmul(fdiv((float)sy, p.normH[s]), 2.0f), 1.0f);
  float ix = fsub(fmul(fadd(gx, 1.0f), p.halfW[s]), 0.5f);
  float iy = fsub(fmul(fadd(gy, 1.0f), p.halfH[s]), 0.5f);
  const int W = p.W[s], H = p.H[s], C = p.C[s];
  // clamp far-out-of-range coordinates (all taps masked anyway) so the float->int conversion is well defined
  ix = fminf(fmaxf(ix, -4.0f), (float)W + 4.0f);
  iy = fminf(fmaxf(iy, -4.0f), (float)H + 4.0f);
  const float xw = floorf(ix), yn = floorf(iy);
  const float w = fsub(ix, xw), e = fsub(1.0f, w);
  const float n = fsub(iy, yn), so = fsub(1.0f, n);
  const int x0 = (int)xw, y0 = (int)yn;
  t.w[0] = fmul(so, e); t.w[1] = fmul(so, w); t.w[2] = fmul(n, e); t.w[3] = fmul(n, w);
  t.fx = w; t.fy = n;
  t.any = false;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int xx = x0 + (k & 1), yy = y0 + (k >> 1);
    const bool ok = (xx >= 0) && (xx < W) && (yy >= 0) && (yy < H);
    t.off[k] = ok ? (yy * W + xx) * C : -1;
    t.any |= ok;
  }
  return t;
}

// ---- Philox4x32-10 (counter-based RNG for the perf path when no noise tensors are supplied) -------------------
__device__ __forceinline__ uint4 philox4x32(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0; key.y += W1;
  }
  return ctr;
}
__device__ __forceinline__ float u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }   // [0,1)


// ---- helpers shared by the forward ray kernels (ray_kernels.cu) and the backward pass (backward.cu) --------------
__device__ __forceinline__ float linspace_at(float start, float end, int steps, int i) {
  // ATen linspace: lower half start + step*i, upper half end - step*(steps-1-i)
  if (steps == 1) return start;
  const float step = fdiv(fsub(end, start), (float)(steps - 1));
  return (i < steps / 2) ? fadd(start, fmul(step, (float)i)) : fsub(end, fmul(step, (float)(steps - 1 - i)));
}

__device__ __forceinline__ float philox_uniform(uint64_t seed, uint32_t ray, uint32_t idx, uint32_t stream) {
  const uint4 o = philox4x32(make_uint4(ray, idx >> 2, stream, 0u), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const uint32_t v[4] = {o.x, o.y, o.z, o.w};
  return u01(v[idx & 3]);
}
__device__ __forceinline__ float philox_normal(uint64_t seed, uint32_t ray, uint32_t idx) {
  const uint4 o = philox4x32(make_uint4(ray, idx >> 1, 2u, 0u), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const float u1 = ((float)(((idx & 1) ? o.z : o.x) >> 8) + 1.0f) * (1.0f / 16777216.0f);   // (0,1]
  const float u2 = u01((idx & 1) ? o.w : o.y);
  return sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float sigmoidf_ref(float x) { return fdiv(1.0f, fadd(1.0f, expf(-x))); }
__device__ __forceinline__ float softplusf_ref(float x) { return (x > 20.0f) ? x : log1pf(expf(x)); }

}  // namespace srf
