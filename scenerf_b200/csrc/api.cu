// extern "C" boundary of libscenerf_b200.so (declarations + contract: include/scenerf_b200.h).
// Sequences the kernels of one render_rays_batch call on the caller's stream:
//   ray_setup -> point MLP (mlp_gaussian, R*G points) -> sample_sort -> point MLP (mlp, R*S points) -> composite_som
// which is scenerf/models/scenerf.py:598-700 (batchify_depth_and_color) without the Python chunk loop of :419-442.
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cmath>
#include "kernels.cuh"

namespace {

thread_local char g_err[512] = "";
thread_local int g_launches = 0;

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int check_cuda(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(SRF_E_CUDA, "%s: %s (watchdog flag 0x%x)", what, cudaGetErrorString(e), srf::watchdog_flag());
  return SRF_OK;
}

inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// bump allocator over the caller-supplied workspace
struct Arena {
  unsigned char* base;
  size_t cap, off;
  template <typename T>
  T* take(size_t count) {
    T* p = reinterpret_cast<T*>(base + off);
    off += align256(count * sizeof(T));
    return p;
  }
};

int validate(const srf_config* cfg, const srf_pyramid* pyr) {
  if (!cfg) return fail(SRF_E_INVALID, "cfg is NULL");
  if (cfg->n_gaussians < 1 || cfg->n_gaussians > SRF_MAX_GAUSSIANS)
    return fail(SRF_E_INVALID, "n_gaussians=%d outside [1,%d]", cfg->n_gaussians, SRF_MAX_GAUSSIANS);
  if (cfg->n_pts_uni < 1 || cfg->n_pts_per_gaussian < 1)
    return fail(SRF_E_INVALID, "n_pts_uni=%d n_pts_per_gaussian=%d must be >= 1", cfg->n_pts_uni,
                cfg->n_pts_per_gaussian);
  const int S = cfg->n_pts_uni + cfg->n_gaussians * cfg->n_pts_per_gaussian;
  if (S > 256) return fail(SRF_E_INVALID, "samples per ray S=%d exceeds 256", S);
  if (cfg->sphere_W < 2 || cfg->sphere_H < 2 || cfg->sphere_W > 16384 || cfg->sphere_H > 16384)
    return fail(SRF_E_INVALID, "sphere grid %dx%d outside [2,16384]", cfg->sphere_W, cfg->sphere_H);
  if (cfg->precision != SRF_PREC_FP32 && cfg->precision != SRF_PREC_FP16_TC && cfg->precision != SRF_PREC_FP32_TC)
    return fail(SRF_E_INVALID, "unknown precision %d", cfg->precision);
  if (pyr) {
    if (cfg->precision != SRF_PREC_FP16_TC && pyr->format != SRF_PYR_FP32)
      return fail(SRF_E_INVALID, "precision=FP32 / FP32_TC needs a pyramid packed as SRF_PYR_FP32");
    for (int s = 0; s < SRF_NUM_SCALES; ++s) {
      if (!pyr->hwc[s] || pyr->C[s] < 1 || pyr->H[s] < 1 || pyr->W[s] < 1)
        return fail(SRF_E_INVALID, "pyramid scale %d is empty", s);
      if (pyr->C[s] % 8) return fail(SRF_E_INVALID, "pyramid scale %d: C=%d must be a multiple of 8", s, pyr->C[s]);
    }
  }
  return SRF_OK;
}

int validate_weights(const srf_mlp_weights* w, int d_out, int d_latent, int precision) {
  if (!w) return fail(SRF_E_INVALID, "weights are NULL");
  if (w->d_out != d_out) return fail(SRF_E_INVALID, "ResnetFC d_out=%d, expected %d", w->d_out, d_out);
  if (w->d_latent != d_latent)
    return fail(SRF_E_INVALID, "ResnetFC d_latent=%d but the pyramid has %d channels", w->d_latent, d_latent);
  if (precision == SRF_PREC_FP16_TC && !w->tc_packed)
    return fail(SRF_E_INVALID, "precision=FP16_TC needs srf_pack_weights_tc() output in tc_packed");
  if (precision == SRF_PREC_FP32_TC && !w->tc_split_packed)
    return fail(SRF_E_INVALID, "precision=FP32_TC needs srf_pack_weights_tc_split() output in tc_split_packed");
  if (precision == SRF_PREC_FP32) {
    bool ok = w->lin_in_w && w->lin_in_b && w->lin_out_w && w->lin_out_b;
    for (int b = 0; b < SRF_NUM_BLOCKS; ++b)
      ok = ok && w->lin_z_w[b] && w->lin_z_b[b] && w->fc0_w[b] && w->fc0_b[b] && w->fc1_w[b] && w->fc1_b[b];
    if (!ok) return fail(SRF_E_INVALID, "a ResnetFC tensor pointer is NULL");
  }
  return SRF_OK;
}

srf::DevParams make_params(const srf_config* cfg, const srf_pyramid* pyr) {
  srf::DevParams p;
  memset(&p, 0, sizeof(p));
  memcpy(p.K, cfg->K, sizeof(p.K));
  memcpy(p.invK, cfg->inv_K, sizeof(p.invK));
  memcpy(p.T, cfg->T, sizeof(p.T));
  // python: h_fov = abs(h_max - h_min) in double, cast to fp32 when it meets the tensor (spherical_mapping.py:68-69,108-109)
  p.v_min = cfg->v_angle_min;
  p.h_min = cfg->h_angle_min;
  p.v_fov = (float)fabs((double)cfg->v_angle_max - (double)cfg->v_angle_min);
  p.h_fov = (float)fabs((double)cfg->h_angle_max - (double)cfg->h_angle_min);
  p.sphere_W = cfg->sphere_W;
  p.sphere_H = cfg->sphere_H;
  p.sphW1 = (float)(cfg->sphere_W - 1);
  p.sphH1 = (float)(cfg->sphere_H - 1);
  p.max_depth = cfg->max_sample_depth;
  p.base_std = cfg->base_std;
  p.add_const = cfg->dataset == SRF_KITTI ? 1.5f : 0.5f;
  p.som_sigma = cfg->som_sigma;
  const double step = (double)cfg->max_sample_depth * 1.0 / cfg->n_gaussians;          // scenerf.py:554
  p.g_start = (float)(step / 2);
  p.g_end = (float)((double)cfg->max_sample_depth - step / 2);
  p.uni_step = (float)(((double)cfg->max_sample_depth - 0.2) / cfg->n_pts_uni);        // utils.py:77
  p.two_sig2 = (float)(2.0 * (double)cfg->som_sigma * (double)cfg->som_sigma);
  p.U = cfg->n_pts_uni;
  p.G = cfg->n_gaussians;
  p.P = cfg->n_pts_per_gaussian;
  p.S = p.U + p.G * p.P;
  p.seed = cfg->seed;
  p.ray0 = (uint32_t)cfg->ray_offset;
  if (pyr) {
    int off = 0;
    for (int s = 0; s < SRF_NUM_SCALES; ++s) {
      const int scale = 1 << s;
      p.feat[s] = pyr->hwc[s];
      p.feat_fp16 = pyr->format == SRF_PYR_FP16;
      p.C[s] = pyr->C[s]; p.H[s] = pyr->H[s]; p.W[s] = pyr->W[s];
      p.ch_off[s] = off;
      off += pyr->C[s];
      // scenerf.py:522-525: scale 1 normalised by (out_img_W, out_img_H), scale s by (W//s, H//s)
      p.normW[s] = (float)(cfg->sphere_W / scale);
      p.normH[s] = (float)(cfg->sphere_H / scale);
      p.halfW[s] = (float)(pyr->W[s] / 2.0);
      p.halfH[s] = (float)(pyr->H[s] / 2.0);
    }
    p.ch_off[SRF_NUM_SCALES] = off;
    p.d_latent = off;
    p.preproj = pyr->latent_table;
    p.preproj_gauss = pyr->latent_table_gauss;
    p.preproj_fp16 = pyr->latent_table_format == SRF_PYR_FP16;
  }
  return p;
}

// save_activations: the float32 pass is a training forward (SRF_FLAG_SAVE_ACTIVATIONS)
size_t mlp_workspace_bytes(int precision, int d_latent, int n_points, bool save_activations) {
  return precision == SRF_PREC_FP32 ? srf::simt_workspace_bytes(d_latent, n_points, save_activations)
                                    : srf::tc_workspace_bytes(d_latent, n_points);
}

// optional device-side timing of the two point-MLP passes (bench.py roofline): events on the launching stream
thread_local bool g_profiling = false;
thread_local cudaEvent_t g_ev[4] = {nullptr, nullptr, nullptr, nullptr};   // gauss begin/end, main begin/end
thread_local bool g_ev_valid[2] = {false, false};

void prof_record(int which, cudaStream_t st) {
  if (!g_profiling) return;
  if (!g_ev[which]) cudaEventCreate(&g_ev[which]);
  cudaEventRecord(g_ev[which], st);
  if (which & 1) g_ev_valid[which >> 1] = true;
}

// the GEMM engine the matmul flags select (training); validate_matmul has refused both flags together
srf::MatmulEngine matmul_engine(int flags) {
  if (flags & SRF_FLAG_FP32TC_MATMUL) return srf::MatmulEngine::fp32tc;
  return (flags & SRF_FLAG_TF32_MATMUL) ? srf::MatmulEngine::tf32 : srf::MatmulEngine::simt;
}
int validate_matmul(const srf_config* cfg, const char* who) {
  if ((cfg->flags & SRF_FLAG_TF32_MATMUL) && (cfg->flags & SRF_FLAG_FP32TC_MATMUL))
    return fail(SRF_E_INVALID, "%s: SRF_FLAG_TF32_MATMUL and SRF_FLAG_FP32TC_MATMUL select different GEMM engines; set one", who);
  return SRF_OK;
}

// the tensor-core pass of network w: its flags (split mode, latent table) and its DevParams.  A latent table belongs to
// one network: the main pass (d_out 4) reads latent_table, the proposal pass latent_table_gauss
int tc_pass(const srf::DevParams& p, int precision, int flags, const srf_mlp_weights& w, srf::DevParams& pp) {
  int f = flags & ~(srf::kTcFlagSplit | srf::kTcFlagPreproj);
  if (precision == SRF_PREC_FP32_TC) f |= srf::kTcFlagSplit;
  pp = p;
  pp.preproj = (w.d_out == 4) ? p.preproj : p.preproj_gauss;
  if (pp.preproj) f |= srf::kTcFlagPreproj;
  return f;
}

int run_mlp(const srf::DevParams& p, int precision, int flags, const srf_mlp_weights& w, const float* pts,
            const float* viewdir, int n, int n_per, float* raw, int32_t* dbg, void* ws, size_t ws_bytes,
            cudaStream_t st, void* saved = nullptr) {
  int l;
  const int pass = (w.d_out == 4) ? 1 : 0;
  prof_record(2 * pass, st);
  if (precision == SRF_PREC_FP32) {
    // SRF_FLAG_TF32_MATMUL / SRF_FLAG_FP32TC_MATMUL apply to the training forward only
    const srf::MatmulEngine e = saved ? matmul_engine(flags) : srf::MatmulEngine::simt;
    l = srf::run_point_mlp_simt(p, w, pts, viewdir, n, n_per, raw, dbg, saved, e, ws, ws_bytes, st);
  } else {
    srf::DevParams pp;
    const int f = tc_pass(p, precision, flags, w, pp);
    l = srf::run_point_mlp_tc(pp, w, pts, viewdir, n, n_per, raw, dbg, f, ws, ws_bytes, st);
  }
  if (l < 0) return fail(SRF_E_WORKSPACE, "point-MLP workspace too small (%zu bytes)", ws_bytes);
  prof_record(2 * pass + 1, st);
  g_launches += l;
  return check_cuda("point MLP");
}

int pyramid_channels(const srf_pyramid* pyr) {
  int c = 0;
  for (int s = 0; s < SRF_NUM_SCALES; ++s) c += pyr->C[s];
  return c;
}

struct RayWorkspace {
  float *unit, *viewdir, *gauss_pts, *gauss_raw, *means, *stds, *t_sorted, *depth_volume, *pts, *raw;
  void* mlp_ws;
  size_t mlp_ws_bytes;
  void *saved_main, *saved_gauss;     // SRF_FLAG_SAVE_ACTIVATIONS (float32 training forward), else NULL
};

size_t carve(const srf_config* cfg, int R, int d_latent, unsigned char* base, RayWorkspace* out) {
  const size_t G = cfg->n_gaussians, S = cfg->n_pts_uni + G * cfg->n_pts_per_gaussian;
  Arena a{base, 0, 0};
  RayWorkspace w;
  w.unit = a.take<float>((size_t)R * 3);
  w.viewdir = a.take<float>((size_t)R * 3);
  w.gauss_pts = a.take<float>((size_t)R * G * 3);
  w.gauss_raw = a.take<float>((size_t)R * G * 2);
  w.means = a.take<float>((size_t)R * G);
  w.stds = a.take<float>((size_t)R * G);
  w.t_sorted = a.take<float>((size_t)R * S);
  w.depth_volume = a.take<float>((size_t)R * S);
  w.pts = a.take<float>((size_t)R * S * 3);
  w.raw = a.take<float>((size_t)R * S * 4);
  const bool save = (cfg->flags & SRF_FLAG_SAVE_ACTIVATIONS) && cfg->precision == SRF_PREC_FP32;
  const size_t m1 = mlp_workspace_bytes(cfg->precision, d_latent, (int)((size_t)R * S), save);
  const size_t m2 = mlp_workspace_bytes(cfg->precision, d_latent, (int)((size_t)R * G), save);
  w.mlp_ws_bytes = m1 > m2 ? m1 : m2;
  w.mlp_ws = a.take<unsigned char>(w.mlp_ws_bytes);
  w.saved_main = w.saved_gauss = nullptr;
  if (save) {
    w.saved_main = a.take<unsigned char>(srf::mlp_saved_bytes(d_latent, (int)((size_t)R * S)));
    w.saved_gauss = a.take<unsigned char>(srf::mlp_saved_bytes(d_latent, (int)((size_t)R * G)));
  }
  if (out) *out = w;
  return a.off;
}

constexpr int kDefaultLatent = 2480;

}  // namespace

extern "C" {

int srf_abi_version(void) { return SRF_ABI_VERSION; }
const char* srf_last_error(void) { return g_err; }
int srf_last_launch_count(void) { return g_launches; }
int srf_debug_watchdog_flag(void) { return srf::watchdog_flag(); }
void srf_set_profiling(int on) { g_profiling = on != 0; }
int srf_last_mlp_ms(float* gauss_ms, float* main_ms) {
  float* dst[2] = {gauss_ms, main_ms};
  for (int i = 0; i < 2; ++i) {
    if (!dst[i]) continue;
    *dst[i] = -1.0f;
    if (!g_ev_valid[i]) continue;
    if (cudaEventSynchronize(g_ev[2 * i + 1]) != cudaSuccess) return check_cuda("srf_last_mlp_ms");
    cudaEventElapsedTime(dst[i], g_ev[2 * i], g_ev[2 * i + 1]);
  }
  return SRF_OK;
}
size_t srf_sizeof(int which) {
  switch (which) {
    case 0: return sizeof(srf_config);
    case 1: return sizeof(srf_pyramid);
    case 2: return sizeof(srf_mlp_weights);
    case 3: return sizeof(srf_outputs);
    default: return 0;
  }
}

size_t srf_pyramid_bytes(const int* C, const int* H, const int* W, int format) {
  size_t b = 0;
  const size_t esz = format == SRF_PYR_FP16 ? 2 : 4;
  for (int s = 0; s < SRF_NUM_SCALES; ++s) b += align256((size_t)C[s] * H[s] * W[s] * esz);
  return b;
}

int srf_pack_pyramid(const float* const* chw_dev, const int* C, const int* H, const int* W, int format, void* dst_dev,
                     size_t dst_bytes, srf_pyramid* out, void* stream) {
  if (!chw_dev || !C || !H || !W || !dst_dev || !out) return fail(SRF_E_INVALID, "srf_pack_pyramid: NULL argument");
  if (format != SRF_PYR_FP32 && format != SRF_PYR_FP16) return fail(SRF_E_INVALID, "srf_pack_pyramid: format %d", format);
  if (dst_bytes < srf_pyramid_bytes(C, H, W, format))
    return fail(SRF_E_WORKSPACE, "srf_pack_pyramid: dst has %zu bytes, need %zu", dst_bytes, srf_pyramid_bytes(C, H, W, format));
  const size_t esz = format == SRF_PYR_FP16 ? 2 : 4;
  out->format = format;
  out->latent_table = nullptr;
  out->latent_table_gauss = nullptr;
  out->latent_table_format = 0;
  unsigned char* d = reinterpret_cast<unsigned char*>(dst_dev);
  for (int s = 0; s < SRF_NUM_SCALES; ++s) {
    if (!chw_dev[s] || C[s] < 1 || H[s] < 1 || W[s] < 1) return fail(SRF_E_INVALID, "srf_pack_pyramid: scale %d empty", s);
    srf::launch_chw_to_hwc(chw_dev[s], d, C[s], H[s], W[s], format == SRF_PYR_FP16, (cudaStream_t)stream);
    out->hwc[s] = d;
    out->C[s] = C[s]; out->H[s] = H[s]; out->W[s] = W[s];
    d += align256((size_t)C[s] * H[s] * W[s] * esz);
  }
  return check_cuda("srf_pack_pyramid");
}

size_t srf_tc_weights_bytes(int d_out, int d_latent) { return srf::tc_weights_bytes(d_out, d_latent, 0); }
size_t srf_tc_split_weights_bytes(int d_out, int d_latent) { return srf::tc_weights_bytes(d_out, d_latent, 1); }

static int pack_tc_common(const srf_mlp_weights* w, void* dst_dev, size_t dst_bytes, int split, void* stream, const char* who) {
  if (!w || !dst_dev) return fail(SRF_E_INVALID, "%s: NULL argument", who);
  bool ok = w->lin_in_w && w->lin_in_b && w->lin_out_w && w->lin_out_b;
  for (int b = 0; b < SRF_NUM_BLOCKS; ++b)
    ok = ok && w->lin_z_w[b] && w->lin_z_b[b] && w->fc0_w[b] && w->fc0_b[b] && w->fc1_w[b] && w->fc1_b[b];
  if (!ok) return fail(SRF_E_INVALID, "%s: a ResnetFC tensor pointer is NULL", who);
  const size_t need = srf::tc_weights_bytes(w->d_out, w->d_latent, split);
  if (dst_bytes < need) return fail(SRF_E_WORKSPACE, "%s: dst has %zu bytes, need %zu", who, dst_bytes, need);
  const int rc = srf::pack_weights_tc(*w, dst_dev, dst_bytes, split, (cudaStream_t)stream);
  if (rc) return fail(SRF_E_INVALID, "%s: unsupported shape (d_out=%d d_latent=%d)", who, w->d_out, w->d_latent);
  return check_cuda(who);
}
int srf_pack_weights_tc_split(const srf_mlp_weights* w, void* dst_dev, size_t dst_bytes, void* stream) {
  return pack_tc_common(w, dst_dev, dst_bytes, 1, stream, "srf_pack_weights_tc_split");
}

int srf_pack_weights_tc(const srf_mlp_weights* w, void* dst_dev, size_t dst_bytes, void* stream) {
  return pack_tc_common(w, dst_dev, dst_bytes, 0, stream, "srf_pack_weights_tc");
}

size_t srf_latent_table_bytes(const srf_config* cfg, int format) {
  if (!cfg || cfg->sphere_W < 1 || cfg->sphere_H < 1) return 0;
  return srf::preproj_table_bytes(cfg->sphere_W, cfg->sphere_H, format == SRF_PYR_FP16);
}
size_t srf_latent_table_workspace_bytes(const srf_pyramid* pyr) { return pyr ? srf::preproj_workspace_bytes(pyr->H, pyr->W) : 0; }

int srf_build_latent_table(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w_main, int format,
                           void* table_dev, size_t table_bytes, void* workspace_dev, size_t workspace_bytes, void* stream) {
  g_launches = 0;
  if (int rc = validate(cfg, pyr)) return rc;
  if (!pyr || !w_main || !table_dev || !workspace_dev) return fail(SRF_E_INVALID, "srf_build_latent_table: NULL argument");
  if (pyr->format != SRF_PYR_FP32) return fail(SRF_E_INVALID, "srf_build_latent_table: needs an SRF_PYR_FP32 pyramid");
  if (format != SRF_PYR_FP32 && format != SRF_PYR_FP16) return fail(SRF_E_INVALID, "srf_build_latent_table: format %d", format);
  const int d_latent = pyramid_channels(pyr);
  if (int rc = validate_weights(w_main, w_main->d_out, d_latent, SRF_PREC_FP32)) return rc;
  if (table_bytes < srf_latent_table_bytes(cfg, format) || workspace_bytes < srf_latent_table_workspace_bytes(pyr))
    return fail(SRF_E_WORKSPACE, "srf_build_latent_table: table %zu / workspace %zu bytes, need %zu / %zu", table_bytes, workspace_bytes,
                srf_latent_table_bytes(cfg, format), srf_latent_table_workspace_bytes(pyr));
  srf_pyramid plain = *pyr;
  plain.latent_table = nullptr;
  plain.latent_table_gauss = nullptr;
  const srf::DevParams p = make_params(cfg, &plain);
  const int l = srf::run_preproject(p, *w_main, format == SRF_PYR_FP16, table_dev, table_bytes, workspace_dev, workspace_bytes,
                                    (cudaStream_t)stream);
  if (l < 0) return fail(SRF_E_INVALID, "srf_build_latent_table: unsupported shape");
  g_launches = l;
  return check_cuda("srf_build_latent_table");
}

size_t srf_render_workspace_bytes(const srf_config* cfg, int n_rays) {
  if (!cfg || n_rays < 0) return 0;
  return carve(cfg, n_rays, cfg->d_latent > 0 ? cfg->d_latent : kDefaultLatent, nullptr, nullptr) + 4096;
}

int srf_render_rays(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w_main,
                    const srf_mlp_weights* w_gauss, const float* pixels_dev, int n_rays, const float* noise_u_dev,
                    const float* noise_n_dev, const srf_outputs* out, void* workspace_dev, size_t workspace_bytes,
                    void* stream) {
  g_launches = 0;
  if (int rc = validate(cfg, pyr)) return rc;
  if (int rc = validate_matmul(cfg, "srf_render_rays")) return rc;
  if (!pyr || !out) return fail(SRF_E_INVALID, "srf_render_rays: pyramid / outputs are NULL");
  if (n_rays == 0) return SRF_OK;                      // empty batch: nothing to write (reference returns empty cats)
  if (n_rays < 0 || !pixels_dev) return fail(SRF_E_INVALID, "srf_render_rays: n_rays=%d pixels=%p", n_rays, (const void*)pixels_dev);
  const int d_latent = pyramid_channels(pyr);
  if (int rc = validate_weights(w_main, 4, d_latent, cfg->precision)) return rc;
  if (int rc = validate_weights(w_gauss, 2, d_latent, cfg->precision)) return rc;
  RayWorkspace ws;
  const size_t need = carve(cfg, n_rays, d_latent, reinterpret_cast<unsigned char*>(workspace_dev), &ws);
  if (!workspace_dev || workspace_bytes < need)
    return fail(SRF_E_WORKSPACE, "srf_render_rays: workspace has %zu bytes, need %zu", workspace_bytes, need);
  const cudaStream_t st = (cudaStream_t)stream;
  const srf::DevParams p = make_params(cfg, pyr);
  const int R = n_rays, G = p.G, S = p.S;

  srf::launch_ray_setup(p, pixels_dev, R, ws.unit, ws.viewdir, ws.gauss_pts, st);
  ++g_launches;
  if (int rc = check_cuda("ray_setup")) return rc;
  if (int rc = run_mlp(p, cfg->precision, cfg->flags, *w_gauss, ws.gauss_pts, ws.viewdir, R * G, G, ws.gauss_raw,
                       out->dbg_sphere_gauss, ws.mlp_ws, ws.mlp_ws_bytes, st, ws.saved_gauss))
    return rc;
  float* means = out->gaussian_means ? out->gaussian_means : ws.means;
  float* stds = out->gaussian_stds ? out->gaussian_stds : ws.stds;
  float* dv = out->depth_volumes ? out->depth_volumes : ws.depth_volume;
  srf::launch_sample_sort(p, R, ws.unit, ws.gauss_raw, noise_u_dev, noise_n_dev, means, stds, ws.t_sorted, dv, ws.pts, st);
  ++g_launches;
  if (int rc = check_cuda("sample_sort")) return rc;
  if (int rc = run_mlp(p, cfg->precision, cfg->flags, *w_main, ws.pts, ws.viewdir, R * S, S, ws.raw,
                       out->dbg_sphere_main, ws.mlp_ws, ws.mlp_ws_bytes, st, ws.saved_main))
    return rc;
  srf::launch_composite_som(p, R, ws.raw, ws.t_sorted, dv, means, stds, *out, st);
  ++g_launches;
  return check_cuda("composite_som");
}

size_t srf_render_host_workspace_bytes(const srf_config* cfg, int n_rays) {
  if (!cfg || n_rays < 0) return 0;
  const size_t G = cfg->n_gaussians, S = cfg->n_pts_uni + G * cfg->n_pts_per_gaussian;
  // staging for pixels + every output the caller may request
  const size_t stage = align256((size_t)n_rays * 2 * 4) + 6 * align256((size_t)n_rays * 4 * 4) +
                       3 * align256((size_t)n_rays * G * 4) + 4 * align256((size_t)n_rays * S * 4);
  return srf_render_workspace_bytes(cfg, n_rays) + stage + 4096;
}

int srf_render_rays_host(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w_main,
                         const srf_mlp_weights* w_gauss, const float* pixels_host, int n_rays,
                         const srf_outputs* out_host, void* workspace_dev, size_t workspace_bytes, void* stream) {
  if (!cfg || !out_host) return fail(SRF_E_INVALID, "srf_render_rays_host: NULL argument");
  if (n_rays == 0) return SRF_OK;
  if (n_rays < 0 || !pixels_host) return fail(SRF_E_INVALID, "srf_render_rays_host: bad rays");
  if (!workspace_dev || workspace_bytes < srf_render_host_workspace_bytes(cfg, n_rays))
    return fail(SRF_E_WORKSPACE, "srf_render_rays_host: workspace has %zu bytes, need %zu", workspace_bytes,
                srf_render_host_workspace_bytes(cfg, n_rays));
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t R = n_rays, G = cfg->n_gaussians, S = cfg->n_pts_uni + G * cfg->n_pts_per_gaussian;
  Arena a{reinterpret_cast<unsigned char*>(workspace_dev), 0, 0};
  float* pix = a.take<float>(R * 2);
  srf_outputs dev;
  memset(&dev, 0, sizeof(dev));
  struct Item { float* const* host; float** devp; size_t count; };
  const Item items[] = {
      {&out_host->depth, &dev.depth, R}, {&out_host->color, &dev.color, R * 3},
      {&out_host->gaussian_means, &dev.gaussian_means, R * G}, {&out_host->gaussian_stds, &dev.gaussian_stds, R * G},
      {&out_host->weights_at_depth, &dev.weights_at_depth, R}, {&out_host->closest_pts_to_depths, &dev.closest_pts_to_depths, R},
      {&out_host->loss_kl, &dev.loss_kl, R}, {&out_host->alphas, &dev.alphas, R * S},
      {&out_host->som_vars, &dev.som_vars, R * G}, {&out_host->densities, &dev.densities, R * S},
      {&out_host->weights, &dev.weights, R * S}, {&out_host->depth_volumes, &dev.depth_volumes, R * S},
      {&out_host->som_means, &dev.som_means, R * G}};
  for (const Item& it : items)
    if (*it.host) *it.devp = a.take<float>(it.count);
  if (cudaMemcpyAsync(pix, pixels_host, R * 2 * sizeof(float), cudaMemcpyHostToDevice, st) != cudaSuccess)
    return check_cuda("H2D pixels");
  const int rc = srf_render_rays(cfg, pyr, w_main, w_gauss, pix, n_rays, nullptr, nullptr, &dev,
                                 reinterpret_cast<unsigned char*>(workspace_dev) + a.off, workspace_bytes - a.off, stream);
  if (rc) return rc;
  for (const Item& it : items)
    if (*it.host) cudaMemcpyAsync(*it.host, *it.devp, it.count * sizeof(float), cudaMemcpyDeviceToHost, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) return check_cuda("srf_render_rays_host sync");
  return check_cuda("srf_render_rays_host");
}

size_t srf_predict_workspace_bytes(const srf_config* cfg, int n_points) {
  if (!cfg || n_points < 0) return 0;
  return mlp_workspace_bytes(cfg->precision, cfg->d_latent > 0 ? cfg->d_latent : kDefaultLatent, n_points, false) + align256((size_t)n_points * 4 * 4) + 4096;
}

__global__ void activate_kernel(const float* __restrict__ raw, int n, float* __restrict__ density,
                                float* __restrict__ color) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 o = reinterpret_cast<const float4*>(raw)[i];
  if (color) {
    color[(size_t)i * 3 + 0] = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-o.x)));
    color[(size_t)i * 3 + 1] = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-o.y)));
    color[(size_t)i * 3 + 2] = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-o.z)));
  }
  if (density) {
    const float x = __fsub_rn(o.w, 1.0f);
    density[i] = (x > 20.0f) ? x : log1pf(expf(x));
  }
}

int srf_predict(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w, const float* cam_pts_dev,
                const float* viewdir_dev, int n_cols, int n_per, float* raw_out_dev, float* density_dev,
                float* color_dev, int32_t* dbg_sphere_dev, void* workspace_dev, size_t workspace_bytes,
                void* stream) {
  g_launches = 0;
  if (int rc = validate(cfg, pyr)) return rc;
  if (!pyr || !w) return fail(SRF_E_INVALID, "srf_predict: NULL argument");
  if (n_cols == 0 || n_per == 0) return SRF_OK;
  if (n_cols < 0 || n_per < 0 || !cam_pts_dev || !viewdir_dev) return fail(SRF_E_INVALID, "srf_predict: bad points");
  const int d_latent = pyramid_channels(pyr);
  if (int rc = validate_weights(w, w->d_out, d_latent, cfg->precision)) return rc;
  if (w->d_out != 2 && w->d_out != 4) return fail(SRF_E_INVALID, "srf_predict: d_out=%d", w->d_out);
  if ((density_dev || color_dev) && w->d_out != 4)
    return fail(SRF_E_INVALID, "srf_predict: density/color need a d_out=4 network");
  const int n = n_cols * n_per;
  Arena a{reinterpret_cast<unsigned char*>(workspace_dev), 0, 0};
  float* raw = raw_out_dev ? raw_out_dev : a.take<float>((size_t)n * 4);
  const size_t mlp_bytes = mlp_workspace_bytes(cfg->precision, d_latent, n, false);
  if (!workspace_dev || workspace_bytes < a.off + mlp_bytes)
    return fail(SRF_E_WORKSPACE, "srf_predict: workspace has %zu bytes, need %zu", workspace_bytes, a.off + mlp_bytes);
  const srf::DevParams p = make_params(cfg, pyr);
  const cudaStream_t st = (cudaStream_t)stream;
  if (int rc = run_mlp(p, cfg->precision, cfg->flags, *w, cam_pts_dev, viewdir_dev, n, n_per, raw, dbg_sphere_dev,
                       reinterpret_cast<unsigned char*>(workspace_dev) + a.off, workspace_bytes - a.off, st))
    return rc;
  if (density_dev || color_dev) {
    activate_kernel<<<(n + 255) / 256, 256, 0, st>>>(raw, n, density_dev, color_dev);
    ++g_launches;
  }
  return check_cuda("srf_predict");
}

size_t srf_render_backward_workspace_bytes(const srf_config* cfg, int n_rays) {
  if (!cfg || n_rays < 0) return 0;
  const size_t G = cfg->n_gaussians, S = cfg->n_pts_uni + G * cfg->n_pts_per_gaussian;
  const int d_latent = cfg->d_latent > 0 ? cfg->d_latent : kDefaultLatent;
  const size_t m1 = srf::mlp_backward_workspace_bytes(d_latent, (int)((size_t)n_rays * S));
  const size_t m2 = srf::mlp_backward_workspace_bytes(d_latent, (int)((size_t)n_rays * G));
  return align256((size_t)n_rays * S * 4 * 4) + align256((size_t)n_rays * G * 2 * 4) + (m1 > m2 ? m1 : m2) + 4096;
}

int srf_render_rays_backward(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w_main,
                             const srf_mlp_weights* w_gauss, int n_rays, const float* noise_n_dev,
                             const srf_outputs* fwd_out, const srf_outputs* grad_out, const void* fwd_workspace_dev,
                             size_t fwd_workspace_bytes, const srf_mlp_weights* grad_main,
                             const srf_mlp_weights* grad_gauss, float* const* grad_pyr_chw, void* workspace_dev,
                             size_t workspace_bytes, void* stream) {
  g_launches = 0;
  if (int rc = validate(cfg, pyr)) return rc;
  if (int rc = validate_matmul(cfg, "srf_render_rays_backward")) return rc;
  if (!pyr || !fwd_out || !grad_out || !grad_main || !grad_gauss || !grad_pyr_chw)
    return fail(SRF_E_INVALID, "srf_render_rays_backward: NULL argument");
  if (cfg->precision != SRF_PREC_FP32 || pyr->format != SRF_PYR_FP32)
    return fail(SRF_E_INVALID, "srf_render_rays_backward: float32 precision and an fp32 pyramid are required");
  if (n_rays == 0) return SRF_OK;
  if (n_rays < 0) return fail(SRF_E_INVALID, "srf_render_rays_backward: n_rays=%d", n_rays);
  if (!fwd_out->depth || !fwd_out->alphas || !fwd_out->weights || !fwd_out->densities || !fwd_out->depth_volumes ||
      !fwd_out->gaussian_means || !fwd_out->gaussian_stds || !fwd_out->som_vars || !fwd_out->som_means)
    return fail(SRF_E_INVALID, "srf_render_rays_backward: the forward must have produced depth, alphas, weights, densities, "
                               "depth_volumes, gaussian_means, gaussian_stds, som_vars and som_means");
  const int d_latent = pyramid_channels(pyr);
  if (int rc = validate_weights(w_main, 4, d_latent, cfg->precision)) return rc;
  if (int rc = validate_weights(w_gauss, 2, d_latent, cfg->precision)) return rc;
  if (int rc = validate_weights(grad_main, 4, d_latent, cfg->precision)) return rc;
  if (int rc = validate_weights(grad_gauss, 2, d_latent, cfg->precision)) return rc;
  for (int s = 0; s < SRF_NUM_SCALES; ++s)
    if (!grad_pyr_chw[s]) return fail(SRF_E_INVALID, "srf_render_rays_backward: grad_pyr_chw[%d] is NULL", s);
  RayWorkspace fw;
  const size_t fneed = carve(cfg, n_rays, d_latent, reinterpret_cast<unsigned char*>(const_cast<void*>(fwd_workspace_dev)), &fw);
  if (!fwd_workspace_dev || fwd_workspace_bytes < fneed)
    return fail(SRF_E_WORKSPACE, "srf_render_rays_backward: forward workspace has %zu bytes, need %zu", fwd_workspace_bytes, fneed);
  srf_config c2 = *cfg;
  c2.d_latent = d_latent;
  const size_t need = srf_render_backward_workspace_bytes(&c2, n_rays);
  if (!workspace_dev || workspace_bytes < need)
    return fail(SRF_E_WORKSPACE, "srf_render_rays_backward: workspace has %zu bytes, need %zu", workspace_bytes, need);
  const cudaStream_t st = (cudaStream_t)stream;
  const srf::DevParams p = make_params(cfg, pyr);
  const int R = n_rays, G = p.G, S = p.S;
  Arena a{reinterpret_cast<unsigned char*>(workspace_dev), 0, 0};
  float* graw_main = a.take<float>((size_t)R * S * 4);
  float* graw_gauss = a.take<float>((size_t)R * G * 2);
  const size_t mlp_ws_bytes = workspace_bytes - a.off - 2048;
  void* mlp_ws = a.take<unsigned char>(mlp_ws_bytes);
  const srf::MatmulEngine e = matmul_engine(cfg->flags);
  if (srf::tensor_cores(e) && !fw.saved_main)
    return fail(SRF_E_INVALID, "srf_render_rays_backward: %s needs SRF_FLAG_SAVE_ACTIVATIONS (forward and backward must "
                               "see the same activations)", e == srf::MatmulEngine::tf32 ? "SRF_FLAG_TF32_MATMUL" : "SRF_FLAG_FP32TC_MATMUL");
  srf::launch_ray_backward(p, R, fw.raw, fw.t_sorted, fw.unit, fw.gauss_raw, noise_n_dev, *fwd_out, *grad_out, graw_main,
                           graw_gauss, st);
  ++g_launches;
  if (int rc = check_cuda("ray_backward")) return rc;
  int l = srf::run_point_mlp_backward_simt(p, *w_main, *grad_main, grad_pyr_chw, fw.pts, fw.viewdir, R * S, S, graw_main, fw.saved_main,
                                           e, mlp_ws, mlp_ws_bytes, st);
  if (l < 0) return fail(SRF_E_WORKSPACE, "srf_render_rays_backward: MLP backward workspace too small");
  g_launches += l;
  if (int rc = check_cuda("main MLP backward")) return rc;
  l = srf::run_point_mlp_backward_simt(p, *w_gauss, *grad_gauss, grad_pyr_chw, fw.gauss_pts, fw.viewdir, R * G, G, graw_gauss,
                                       fw.saved_gauss, e, mlp_ws, mlp_ws_bytes, st);
  if (l < 0) return fail(SRF_E_WORKSPACE, "srf_render_rays_backward: MLP backward workspace too small");
  g_launches += l;
  return check_cuda("gaussian MLP backward");
}

int srf_tsdf_reset(float* tsdf_dev, float* weight_dev, float* color_dev, const int* dims, void* stream) {
  if (!tsdf_dev || !weight_dev || !color_dev || !dims || dims[0] < 1 || dims[1] < 1 || dims[2] < 1)
    return fail(SRF_E_INVALID, "srf_tsdf_reset: bad argument");
  srf::launch_tsdf_reset(tsdf_dev, weight_dev, color_dev, (long long)dims[0] * dims[1] * dims[2], (cudaStream_t)stream);
  return check_cuda("srf_tsdf_reset");
}

int srf_tsdf_integrate(float* tsdf_dev, float* weight_dev, float* color_dev, const int* dims, const float* origin,
                       double voxel_size, const double* inv_cam_pose_host, const float* cam_intr_host,
                       const float* depth_dev, const void* color_dev_im, int color_is_u8, int im_h, int im_w,
                       double trunc_margin, float obs_weight, void* stream) {
  if (!tsdf_dev || !weight_dev || !color_dev || !dims || !origin || !inv_cam_pose_host || !cam_intr_host || !depth_dev ||
      !color_dev_im)
    return fail(SRF_E_INVALID, "srf_tsdf_integrate: NULL argument");
  if (dims[0] < 1 || dims[1] < 1 || dims[2] < 1 || im_h < 1 || im_w < 1 || !(voxel_size > 0))
    return fail(SRF_E_INVALID, "srf_tsdf_integrate: bad shape (%d,%d,%d) image %dx%d voxel %g", dims[0], dims[1], dims[2], im_h, im_w, voxel_size);
  srf::launch_tsdf_integrate(dims, origin, voxel_size, inv_cam_pose_host, cam_intr_host, im_h, im_w, trunc_margin, obs_weight,
                             color_is_u8, tsdf_dev, weight_dev, color_dev, depth_dev, color_dev_im, (cudaStream_t)stream);
  g_launches = 1;
  return check_cuda("srf_tsdf_integrate");
}

int srf_tsdf_merge(float* tsdf_a, float* weight_a, float* color_a, const float* tsdf_b, const float* weight_b,
                   const float* color_b, const int* dims, void* stream) {
  if (!tsdf_a || !weight_a || !color_a || !tsdf_b || !weight_b || !color_b || !dims || dims[0] < 1 || dims[1] < 1 || dims[2] < 1)
    return fail(SRF_E_INVALID, "srf_tsdf_merge: bad argument");
  srf::launch_tsdf_merge(tsdf_a, weight_a, color_a, tsdf_b, weight_b, color_b, (long long)dims[0] * dims[1] * dims[2],
                         (cudaStream_t)stream);
  g_launches = 1;
  return check_cuda("srf_tsdf_merge");
}

namespace {
// 0 = ok; otherwise the failure already recorded.  *empty = a dimension < 2 (no cell: an empty mesh)
int mesh_dims(const char* fn, const int* dims, bool* empty) {
  if (!dims || dims[0] < 1 || dims[1] < 1 || dims[2] < 1)
    return fail(SRF_E_INVALID, "%s: bad dims", fn);
  const long long n = (long long)dims[0] * dims[1] * dims[2];
  // the scanned counts are int32: at most 3 vertices per grid point and 10 faces per cell
  if (n > 0x7fffffffLL / 10)
    return fail(SRF_E_INVALID, "%s: volume (%d,%d,%d) too large for int32 vertex / face counts", fn, dims[0], dims[1], dims[2]);
  *empty = dims[0] < 2 || dims[1] < 2 || dims[2] < 2;
  return SRF_OK;
}
}  // namespace

size_t srf_tsdf_mesh_workspace_bytes(const int* dims) {
  bool empty;
  if (mesh_dims("srf_tsdf_mesh_workspace_bytes", dims, &empty)) return 0;
  return srf::mesh_workspace_bytes(dims);
}

int srf_tsdf_mesh_count_host(const float* tsdf_dev, const uint8_t* mask_dev, const int* dims, void* ws, size_t ws_bytes,
                             long long* n_verts, long long* n_faces, void* stream) {
  bool empty;
  if (int rc = mesh_dims("srf_tsdf_mesh_count_host", dims, &empty)) return rc;
  if (!tsdf_dev || !n_verts || !n_faces) return fail(SRF_E_INVALID, "srf_tsdf_mesh_count_host: NULL argument");
  if (empty) {
    *n_verts = *n_faces = 0;
    return SRF_OK;
  }
  if (!ws || ws_bytes < srf::mesh_workspace_bytes(dims))
    return fail(SRF_E_WORKSPACE, "srf_tsdf_mesh_count_host: workspace %zu bytes < %zu", ws_bytes, srf::mesh_workspace_bytes(dims));
  srf::launch_mesh_count(tsdf_dev, mask_dev, dims, ws, (cudaStream_t)stream);
  g_launches = 4;
  if (int rc = check_cuda("srf_tsdf_mesh_count_host")) return rc;
  int nv = 0, nt = 0;
  const cudaError_t e = srf::mesh_read_totals(dims, ws, &nv, &nt, (cudaStream_t)stream);
  if (e != cudaSuccess) return fail(SRF_E_CUDA, "srf_tsdf_mesh_count_host: %s", cudaGetErrorString(e));
  *n_verts = nv;
  *n_faces = nt;
  return SRF_OK;
}

int srf_tsdf_mesh_emit(const float* tsdf_dev, const float* color_dev, const uint8_t* mask_dev, const int* dims,
                       const float* origin, double voxel_size, const void* ws, size_t ws_bytes, float* verts_dev,
                       float* normals_dev, uint8_t* colors_dev, int32_t* faces_dev, void* stream) {
  bool empty;
  if (int rc = mesh_dims("srf_tsdf_mesh_emit", dims, &empty)) return rc;
  if (!tsdf_dev || !origin || !verts_dev || (colors_dev && !color_dev))
    return fail(SRF_E_INVALID, "srf_tsdf_mesh_emit: NULL argument");
  if (empty) return SRF_OK;
  if (!ws || ws_bytes < srf::mesh_workspace_bytes(dims))
    return fail(SRF_E_WORKSPACE, "srf_tsdf_mesh_emit: workspace %zu bytes < %zu", ws_bytes, srf::mesh_workspace_bytes(dims));
  srf::launch_mesh_emit(tsdf_dev, color_dev, mask_dev, dims, origin, voxel_size, ws, verts_dev, normals_dev, colors_dev,
                        faces_dev, (cudaStream_t)stream);
  g_launches = faces_dev ? 2 : 1;
  return check_cuda("srf_tsdf_mesh_emit");
}

int srf_upsample_render(const float* depth_xm, const float* color_xm, int gw, int gh, int out_h, int out_w,
                        float* depth_out, float* color_out, int color_mode, void* stream) {
  if (gw < 1 || gh < 1 || out_h < 1 || out_w < 1 || color_mode < 0 || color_mode > 3)
    return fail(SRF_E_INVALID, "srf_upsample_render: bad shape grid %dx%d -> %dx%d mode %d", gw, gh, out_w, out_h, color_mode);
  if ((!depth_xm || !depth_out) && (!color_xm || !color_out))
    return fail(SRF_E_INVALID, "srf_upsample_render: nothing to do (need a depth pair or a colour pair)");
  srf::launch_upsample_render(depth_out ? depth_xm : nullptr, color_out ? color_xm : nullptr, gw, gh, out_h, out_w, depth_out,
                              color_out, color_mode, (cudaStream_t)stream);
  g_launches = 1;
  return check_cuda("srf_upsample_render");
}

size_t srf_eval_hist_len(const int* dims, int n_classes, int per_z) {
  if (!dims || dims[0] < 1 || dims[1] < 1 || dims[2] < 1 || n_classes < 1 || n_classes > SRF_EVAL_MAX_CLASSES) return 0;
  return srf::eval_hist_len(dims, n_classes, per_z);
}

int srf_eval_confusion(const float* tsdf_dev, const void* pred_dev, int pred_dtype, const uint8_t* target_dev,
                       const uint8_t* mask_dev, const int* dims, int n_classes, int th_axis, const double* th_dev, int per_z,
                       long long* hist_dev, int* max_z_dev, uint8_t* occ_dev, void* stream) {
  if (!dims || dims[0] < 1 || dims[1] < 1 || dims[2] < 1) return fail(SRF_E_INVALID, "srf_eval_confusion: bad dims");
  if (n_classes < 1 || n_classes > SRF_EVAL_MAX_CLASSES)
    return fail(SRF_E_INVALID, "srf_eval_confusion: n_classes=%d outside [1,%d]", n_classes, SRF_EVAL_MAX_CLASSES);
  if (!hist_dev || !max_z_dev || (!target_dev && (pred_dev || !occ_dev)))
    return fail(SRF_E_INVALID, "srf_eval_confusion: NULL argument");
  if (pred_dev) {
    if (pred_dtype < SRF_EVAL_U8 || pred_dtype > SRF_EVAL_F64)
      return fail(SRF_E_INVALID, "srf_eval_confusion: unknown pred_dtype %d", pred_dtype);
  } else {
    if (!tsdf_dev || !th_dev) return fail(SRF_E_INVALID, "srf_eval_confusion: occupancy mode needs tsdf_dev and th_dev");
    if (th_axis < 0 || th_axis > 2) return fail(SRF_E_INVALID, "srf_eval_confusion: th_axis=%d outside [0,2]", th_axis);
  }
  // one block's histogram lives in shared memory as 32-bit counters
  const size_t sh = srf::eval_hist_len(dims, n_classes, per_z) * sizeof(unsigned int);
  if (sh > 200 * 1024)
    return fail(SRF_E_INVALID, "srf_eval_confusion: %zu histogram bytes per block exceed 200 KB (per_z=%d, n_classes=%d, Z=%d)", sh,
                per_z, n_classes, dims[2]);
  srf::launch_eval_confusion(tsdf_dev, pred_dev, pred_dtype, target_dev, mask_dev, dims, n_classes, th_axis, th_dev, per_z,
                             (unsigned long long*)hist_dev, max_z_dev, occ_dev, (cudaStream_t)stream);
  g_launches = 1;
  return check_cuda("srf_eval_confusion");
}

int srf_eval_sc_label(const float* tsdf_dev, const int* dims, double voxel_size, uint8_t* out_dev, void* stream) {
  if (!tsdf_dev || !out_dev || !dims || dims[0] < 1 || dims[1] < 1 || dims[2] < 1)
    return fail(SRF_E_INVALID, "srf_eval_sc_label: bad argument");
  srf::launch_eval_sc_label(tsdf_dev, (long long)dims[0] * dims[1] * dims[2], (float)voxel_size, out_dev, (cudaStream_t)stream);
  g_launches = 1;
  return check_cuda("srf_eval_sc_label");
}

int srf_resize_bilinear(const float* src_dev, int in_h, int in_w, float* dst_dev, int out_h, int out_w, void* stream) {
  if (!src_dev || !dst_dev || in_h < 1 || in_w < 1 || out_h < 1 || out_w < 1 || (long long)out_h * out_w > 0x7fffffffLL)
    return fail(SRF_E_INVALID, "srf_resize_bilinear: bad argument %dx%d -> %dx%d", in_h, in_w, out_h, out_w);
  srf::launch_resize_bilinear(src_dev, in_h, in_w, dst_dev, out_h, out_w, (cudaStream_t)stream);
  g_launches = 1;
  return check_cuda("srf_resize_bilinear");
}

size_t srf_depth_errors_workspace_bytes(void) { return srf::depth_errors_workspace_bytes(); }

int srf_depth_errors(const float* gt_dev, const float* pred_dev, long long n, void* ws, size_t ws_bytes, double* buckets_dev,
                     int slot, double* frame_dev, void* stream) {
  if (!gt_dev || !pred_dev || n < 1) return fail(SRF_E_INVALID, "srf_depth_errors: bad argument (n=%lld)", n);
  if (!buckets_dev && !frame_dev) return fail(SRF_E_INVALID, "srf_depth_errors: nothing to write (buckets and frame are NULL)");
  if (buckets_dev && slot < 0) return fail(SRF_E_INVALID, "srf_depth_errors: slot=%d < 0", slot);
  if (!ws || ws_bytes < srf::depth_errors_workspace_bytes())
    return fail(SRF_E_WORKSPACE, "srf_depth_errors: workspace %zu bytes < %zu", ws_bytes, srf::depth_errors_workspace_bytes());
  srf::launch_depth_errors(gt_dev, pred_dev, n, ws, buckets_dev, slot, frame_dev, (cudaStream_t)stream);
  g_launches = 2;
  return check_cuda("srf_depth_errors");
}

size_t srf_psnr_ssim_workspace_bytes(int h, int w) { return h >= 7 && w >= 7 ? srf::psnr_ssim_workspace_bytes(h, w) : 0; }

int srf_psnr_ssim(const float* img_dev, const float* gt_dev, int h, int w, void* ws, size_t ws_bytes, double* buckets_dev, int slot,
                  double* frame_dev, void* stream) {
  if (!img_dev || !gt_dev) return fail(SRF_E_INVALID, "srf_psnr_ssim: NULL image");
  // skimage: "win_size exceeds image extent" below a side of 7
  if (h < 7 || w < 7 || (long long)h * w > 0x7fffffffLL / 3)
    return fail(SRF_E_INVALID, "srf_psnr_ssim: image %dx%d (each side must be at least 7, the SSIM window)", h, w);
  if (!buckets_dev && !frame_dev) return fail(SRF_E_INVALID, "srf_psnr_ssim: nothing to write (buckets and frame are NULL)");
  if (buckets_dev && slot < 0) return fail(SRF_E_INVALID, "srf_psnr_ssim: slot=%d < 0", slot);
  if (!ws || ws_bytes < srf::psnr_ssim_workspace_bytes(h, w))
    return fail(SRF_E_WORKSPACE, "srf_psnr_ssim: workspace %zu bytes < %zu", ws_bytes, srf::psnr_ssim_workspace_bytes(h, w));
  srf::launch_psnr_ssim(img_dev, gt_dev, h, w, ws, buckets_dev, slot, frame_dev, (cudaStream_t)stream);
  g_launches = 2;
  return check_cuda("srf_psnr_ssim");
}

static bool lpips_shape_ok(int h, int w) { return h >= 16 && w >= 16 && h <= 8192 && w <= 8192; }

size_t srf_lpips_workspace_bytes(int h, int w) { return lpips_shape_ok(h, w) ? srf::lpips_workspace_bytes(h, w) : 0; }

int srf_lpips_vgg(const float* img0_dev, const float* img1_dev, int h, int w, const float* const* w9_dev, const float* const* bias_dev,
                  const float* const* lin_dev, const float* shift_host, const float* scale_host, void* ws, size_t ws_bytes, float* out_dev,
                  void* stream) {
  if (!img0_dev || !img1_dev || !w9_dev || !bias_dev || !lin_dev || !shift_host || !scale_host || !out_dev)
    return fail(SRF_E_INVALID, "srf_lpips_vgg: NULL argument");
  if (!lpips_shape_ok(h, w))
    return fail(SRF_E_INVALID, "srf_lpips_vgg: image %dx%d (each side must be in [16, 8192]: four 2x2 pools leave the last tap a pixel)", h, w);
  for (int i = 0; i < 13; ++i)
    if (!w9_dev[i] || !bias_dev[i] || !srf::al16(w9_dev[i]) || !srf::al16(bias_dev[i]))
      return fail(SRF_E_INVALID, "srf_lpips_vgg: conv %d weight / bias NULL or not 16-byte aligned", i);
  for (int k = 0; k < 5; ++k)
    if (!lin_dev[k] || !srf::al16(lin_dev[k])) return fail(SRF_E_INVALID, "srf_lpips_vgg: lin%d NULL or not 16-byte aligned", k);
  if (!srf::al16(ws)) return fail(SRF_E_INVALID, "srf_lpips_vgg: the workspace must be 16-byte aligned");
  if (!ws || ws_bytes < srf::lpips_workspace_bytes(h, w))
    return fail(SRF_E_WORKSPACE, "srf_lpips_vgg: workspace %zu bytes < %zu", ws_bytes, srf::lpips_workspace_bytes(h, w));
  const int l = srf::run_lpips_vgg(img0_dev, img1_dev, h, w, w9_dev, bias_dev, lin_dev, shift_host, scale_host, ws, out_dev,
                                   (cudaStream_t)stream);
  if (l == -2) return fail(SRF_E_UNSUPPORTED, "srf_lpips_vgg: cuTensorMapEncodeTiled is not available");
  if (l < 0) return fail(SRF_E_INVALID, "srf_lpips_vgg: a convolution of the %dx%d image cannot be expressed as tensor maps", h, w);
  g_launches = l;
  return check_cuda("srf_lpips_vgg");
}

int srf_debug_gemm(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K, const float* bias,
                   const float* mask, int ldm, const float* residual, int ldr, int accumulate, float* splitk_ws,
                   size_t splitk_ws_floats, int use_tf32, void* stream) {
  if (!A || !B || !C || M < 1 || N < 1 || K < 1) return fail(SRF_E_INVALID, "srf_debug_gemm: bad argument");
  if (use_tf32 < 0 || use_tf32 > 2) return fail(SRF_E_INVALID, "srf_debug_gemm: use_tf32=%d (0 simt, 1 tf32, 2 split 3xTF32)", use_tf32);
  srf::GemmArgs g;
  g.A = A; g.lda = lda; g.B = B; g.ldb = ldb; g.bt = true; g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = K;
  g.bias = bias; g.mask = mask; g.ldm = ldm; g.R = residual; g.ldr = ldr; g.accumulate = accumulate;
  g.splitk_ws = splitk_ws; g.splitk_ws_floats = splitk_ws_floats;
  const int rc = use_tf32 ? srf::launch_gemm_tf32(g, (cudaStream_t)stream, use_tf32 == 2) : srf::launch_gemm(g, (cudaStream_t)stream);
  static const char* const kName[3] = {"simt", "tf32", "split 3xTF32"};
  if (rc) return fail(SRF_E_INVALID, "srf_debug_gemm: shape not supported by the %s kernel", kName[use_tf32]);
  g_launches = 1;
  return check_cuda("srf_debug_gemm");
}

static int py_round_div(int a, int b) {            // Python round(a / b): half to even
  const double q = (double)a / (double)b;
  return (int)nearbyint(q);
}

void srf_sphere_feature_dims(int out_img_W, int out_img_H, int scale, int* out_W, int* out_H) {
  if (out_W) *out_W = scale > 0 ? py_round_div(out_img_W, scale) : 0;
  if (out_H) *out_H = scale > 0 ? py_round_div(out_img_H, scale) : 0;
}

int srf_sphere_feature(const float* x_chw_dev, int C, int h, int w, const float* pix_dev, const long long* pix_sphere_dev,
                       int n_pixels, int scale, int out_img_W, int out_img_H, float* out_dev, int out_hwc,
                       void* workspace_dev, size_t workspace_bytes, void* stream) {
  if (!x_chw_dev || !pix_dev || !pix_sphere_dev || !out_dev || !workspace_dev)
    return fail(SRF_E_INVALID, "srf_sphere_feature: NULL argument");
  if (C < 1 || h < 1 || w < 1 || n_pixels < 0 || scale < 1 || out_img_W < 1 || out_img_H < 1)
    return fail(SRF_E_INVALID, "srf_sphere_feature: bad shape C=%d h=%d w=%d n=%d scale=%d", C, h, w, n_pixels, scale);
  int oW, oH;
  srf_sphere_feature_dims(out_img_W, out_img_H, scale, &oW, &oH);
  if (oW < 1 || oH < 1) return fail(SRF_E_INVALID, "srf_sphere_feature: empty sphere grid at scale %d", scale);
  if (workspace_bytes < (size_t)oW * oH * sizeof(int))
    return fail(SRF_E_WORKSPACE, "srf_sphere_feature: workspace has %zu bytes, need %zu", workspace_bytes, (size_t)oW * oH * sizeof(int));
  srf::launch_sphere_feature(x_chw_dev, C, h, w, pix_dev, pix_sphere_dev, n_pixels, scale, oW, oH,
                             reinterpret_cast<int*>(workspace_dev), out_dev, out_hwc, (cudaStream_t)stream);
  g_launches = 3;
  return check_cuda("srf_sphere_feature");
}

int srf_upsample_concat_hwc(const float* x_dev, int h, int w, int Cx, int ld_x, const float* skip_dev, int Cs, int ld_skip, int H, int W,
                            float* out_dev, int ld_out, void* stream) {
  if (!x_dev || !skip_dev || !out_dev || h < 1 || w < 1 || H < 1 || W < 1 || Cx < 1 || Cs < 0 || ld_x < Cx || ld_skip < Cs ||
      ld_out < Cx + Cs)
    return fail(SRF_E_INVALID, "srf_upsample_concat_hwc: bad argument (x %dx%dx%d/%d, skip %dx%dx%d/%d, out ld %d)", h, w, Cx, ld_x, H, W, Cs,
                ld_skip, ld_out);
  srf::launch_upsample_concat(x_dev, h, w, Cx, ld_x, skip_dev, Cs, ld_skip, H, W, out_dev, ld_out, (cudaStream_t)stream);
  g_launches = 1;
  return check_cuda("srf_upsample_concat_hwc");
}

int srf_conv3x3_hwc(const float* in_dev, int H, int W, int ld_in, const float* w9_dev, int Cout, int dil, const float* scale_dev,
                    const float* shift_dev, const float* residual_dev, int ld_res, float slope, int round_out, float* out32_dev, int ld32,
                    void* out16_dev, int ld16, void* stream) {
  if (!in_dev || !w9_dev || !scale_dev || !shift_dev || (!out32_dev && !out16_dev))
    return fail(SRF_E_INVALID, "srf_conv3x3_hwc: NULL argument");
  if ((out32_dev && ld32 < Cout) || (out16_dev && ld16 < Cout) || (residual_dev && ld_res < Cout))
    return fail(SRF_E_INVALID, "srf_conv3x3_hwc: a channel stride is smaller than Cout=%d", Cout);
  const int rc = srf::launch_conv3x3_tf32(in_dev, H, W, ld_in, w9_dev, Cout, dil, scale_dev, shift_dev, residual_dev, ld_res, slope, round_out,
                                          out32_dev, ld32, out16_dev, ld16, (cudaStream_t)stream);
  if (rc == -2) return fail(SRF_E_UNSUPPORTED, "srf_conv3x3_hwc: cuTensorMapEncodeTiled is not available");
  if (rc) return fail(SRF_E_INVALID, "srf_conv3x3_hwc: shape or alignment not supported (H=%d W=%d ld_in=%d Cout=%d dil=%d; strides must be "
                                     "multiples of 4 floats, pointers 16-byte aligned, H*ceil(W/128) <= 65535)", H, W, ld_in, Cout, dil);
  g_launches = 1;
  return check_cuda("srf_conv3x3_hwc");
}

int srf_debug_tc_layer(const srf_config* cfg, const srf_pyramid* pyr, const srf_mlp_weights* w,
                       const float* cam_pts_dev, const float* viewdir_dev, int n_cols, int n_per, int layer,
                       float* acc_out_dev, void* workspace_dev, size_t workspace_bytes, void* stream) {
  g_launches = 0;
  if (int rc = validate(cfg, pyr)) return rc;
  if (!pyr || !w || !cam_pts_dev || !viewdir_dev || !acc_out_dev || n_cols < 1 || n_per < 1)
    return fail(SRF_E_INVALID, "srf_debug_tc_layer: bad argument");
  const int d_latent = pyramid_channels(pyr);
  const bool split = cfg->precision == SRF_PREC_FP32_TC;
  if (int rc = validate_weights(w, w->d_out, d_latent, split ? SRF_PREC_FP32_TC : SRF_PREC_FP16_TC)) return rc;
  // the same pass as srf_predict's: this network's latent table when the pyramid carries one
  srf::DevParams pp;
  const int f = tc_pass(make_params(cfg, pyr), cfg->precision, cfg->flags, *w, pp);
  const int l = srf::run_point_mlp_tc_debug(pp, *w, cam_pts_dev, viewdir_dev, n_cols * n_per, n_per, nullptr, nullptr, f,
                                            workspace_dev, workspace_bytes, layer, acc_out_dev, (cudaStream_t)stream);
  if (l == -1) return fail(SRF_E_WORKSPACE, "srf_debug_tc_layer: workspace too small");
  if (l < 0) return fail(SRF_E_INVALID, "srf_debug_tc_layer: layer %d has no accumulator-complete point", layer);
  g_launches += l;
  return check_cuda("srf_debug_tc_layer");
}

}  // extern "C"
