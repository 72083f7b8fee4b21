#include "engine.h"

#include <algorithm>
#include <atomic>
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "container.h"

namespace uhdr_b200 {

int fmt_planes(int fmt) {
  switch (fmt) {
    case F_P010: return 2;
    case F_YUV420: case F_YUV444: case F_YUV422: case F_YUV444_10: return 3;
    case F_Y400: case F_RGBA8888: case F_RGBAF16: case F_RGBA1010102: case F_RGB888: return 1;
  }
  return 0;
}

void fmt_plane_geom(int fmt, int w, int h, int i, int* pw, int* ph, int* esz) {
  *pw = w; *ph = h; *esz = 1;
  switch (fmt) {
    case F_P010:
      *esz = 2;
      if (i == 1) { *pw = ((w + 1) / 2) * 2; *ph = (h + 1) / 2; }
      break;
    case F_YUV420:
      if (i > 0) { *pw = (w + 1) / 2; *ph = (h + 1) / 2; }
      break;
    case F_YUV422:
      if (i > 0) *pw = (w + 1) / 2;
      break;
    case F_YUV444_10: *esz = 2; break;
    case F_RGBA8888: case F_RGBA1010102: *esz = 4; break;
    case F_RGBAF16: *esz = 8; break;
    case F_RGB888: *esz = 3; break;
    default: break;
  }
}

static inline int align_up(int v, int a) { return (v + a - 1) / a * a; }

int alloc_dev_image(Workspace& ws, int fmt, int w, int h, int stride_align, DevImage* out) {
  memset(out, 0, sizeof *out);
  out->v.fmt = fmt;
  out->v.w = w;
  out->v.h = h;
  out->cg = out->ct = out->range = -1;
  const int np = fmt_planes(fmt);
  if (np == 0) return fail(E_UNSUPPORTED, "unsupported image format %d", fmt);
  const int ystride = align_up(w, stride_align);
  for (int i = 0; i < np; i++) {
    int pw, ph, esz;
    fmt_plane_geom(fmt, w, h, i, &pw, &ph, &esz);
    int stride = i == 0 ? ystride : (fmt == F_P010 ? ystride : align_up(pw, stride_align > 1 ? stride_align / 2 : 1));
    if (fmt == F_YUV444 || fmt == F_YUV444_10) stride = ystride;
    // 8 spare rows: the JPEG block stage reads whole 8-row blocks
    void* p = ws.dalloc((size_t)stride * (ph + 8) * esz);
    if (!p) return E_MEM;
    // bytes between the plane width and its stride must be defined: the JPEG block stage reads
    // whole 8-sample blocks, and the reference's internal copies are zero initialised
    // (uhdr_memory_block, ultrahdr_api.cpp:50-117)
    if (pw % 8 != 0 || fmt == F_RGB888)
      if (cudaMemsetAsync(p, 0, (size_t)stride * (ph + 8) * esz, ws.stream()) != cudaSuccess)
        return fail(E_ERROR, "cudaMemsetAsync failed");
    out->v.p[i] = p;
    out->v.stride[i] = stride;
  }
  return E_OK;
}

// rows that are tight on both sides go as one linear copy (one DMA descriptor instead of one per row)
static cudaError_t copy_plane_async(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height,
                                    cudaMemcpyKind kind, cudaStream_t s) {
  if (dpitch == width && spitch == width) return cudaMemcpyAsync(dst, src, width * height, kind, s);
  return cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, kind, s);
}

int upload_image(Workspace& ws, const uhdr_raw_image_t& src, DevImage* out, cudaMemcpyKind kind) {
  if (src.w == 0 || src.h == 0) return fail(E_INVALID_PARAM, "image has zero dimension");
  int rc = alloc_dev_image(ws, src.fmt, src.w, src.h, 64, out);
  if (rc) return rc;
  out->cg = src.cg;
  out->ct = src.ct;
  out->range = src.range;
  out->v.full_range = src.range == UHDR_CR_FULL_RANGE;
  const int np = fmt_planes(src.fmt);
  for (int i = 0; i < np; i++) {
    if (!src.planes[i]) return fail(E_INVALID_PARAM, "plane %d of the image is a null pointer", i);
    int pw, ph, esz;
    fmt_plane_geom(src.fmt, src.w, src.h, i, &pw, &ph, &esz);
    if ((int)src.stride[i] < pw) pw = src.stride[i];
    CUDA_TRY(copy_plane_async((void*)out->v.p[i], (size_t)out->v.stride[i] * esz, src.planes[i],
                              (size_t)src.stride[i] * esz, (size_t)pw * esz, ph, kind, ws.stream()));
  }
  return E_OK;
}

int download_image(Workspace& ws, const DevImage& src, uhdr_raw_image_t* dst) {
  const int np = fmt_planes(src.v.fmt);
  for (int i = 0; i < np; i++) {
    int pw, ph, esz;
    fmt_plane_geom(src.v.fmt, src.v.w, src.v.h, i, &pw, &ph, &esz);
    if ((int)dst->stride[i] < pw) pw = dst->stride[i];
    CUDA_TRY(copy_plane_async(dst->planes[i], (size_t)dst->stride[i] * esz, src.v.p[i],
                              (size_t)src.v.stride[i] * esz, (size_t)pw * esz, ph,
                              cudaMemcpyDeviceToHost, ws.stream()));
  }
  return E_OK;
}

// ------------------------------------------------------------------------------------------------
int generate_gainmap_dev(Workspace& ws, const DevImage& sdr, const DevImage& hdr,
                         const uhdr_b200_gm_config_t& cfg, int map_align, GainmapJob* job) {
  // format checks, jpegr.cpp:537-562
  if (sdr.v.fmt != F_YUV444 && sdr.v.fmt != F_YUV422 && sdr.v.fmt != F_YUV420 && sdr.v.fmt != F_RGBA8888)
    return fail(E_UNSUPPORTED, "generate gainmap method expects sdr intent color format to be one of "
                "{YCbCr444, YCbCr422, YCbCr420, RGBA8888}. Received %d", sdr.v.fmt);
  if (hdr.v.fmt != F_P010 && hdr.v.fmt != F_YUV444_10 && hdr.v.fmt != F_RGBA1010102 && hdr.v.fmt != F_RGBAF16)
    return fail(E_UNSUPPORTED, "generate gainmap method expects hdr intent color format to be one of "
                "{P010, 30bppYCbCr444, RGBA1010102, RGBAHalfFloat}. Received %d", hdr.v.fmt);
  if (hdr.ct < 0 || hdr.ct > 3)
    return fail(E_UNSUPPORTED, "No implementation available for converting transfer characteristics %d to linear", hdr.ct);
  if (sdr.v.w != hdr.v.w || sdr.v.h != hdr.v.h)
    return fail(E_INVALID_PARAM, "sdr intent resolution %dx%d and hdr intent resolution %dx%d do not match",
                sdr.v.w, sdr.v.h, hdr.v.w, hdr.v.h);
  GainmapGenParams p;
  memset(&p, 0, sizeof p);
  p.hdr = hdr.v;
  p.sdr = sdr.v;
  p.hdr_ct = hdr.ct;
  if (!luminance_coeffs(hdr.cg, p.lum))
    return fail(E_UNSUPPORTED, "No implementation available for calculating luminance for color gamut %d", hdr.cg);
  const float hdr_white_nits = reference_display_peak_nits(hdr.ct);
  // gamut side selection, jpegr.cpp:605-638 (UHDR_WRITE_XMP is off: kWriteXmpMetadata == false)
  bool use_sdr_cg = true;
  bool ident = true;
  if (sdr.cg != hdr.cg) {
    use_sdr_cg = !(hdr.cg == UHDR_CG_BT_2100 || (hdr.cg == UHDR_CG_DISPLAY_P3 && sdr.cg != UHDR_CG_BT_2100));
    const bool ok = use_sdr_cg ? gamut_matrix(sdr.cg, hdr.cg, p.gamut, &ident)
                               : gamut_matrix(hdr.cg, sdr.cg, p.gamut, &ident);
    if (!ok) return fail(E_UNSUPPORTED, "No implementation available for gamut conversion from %d to %d", hdr.cg, sdr.cg);
  }
  p.gamut_on_hdr = use_sdr_cg ? 1 : 0;
  p.gamut_identity = ident ? 1 : 0;
  if (!yuv2rgb_coeffs(sdr.cg, p.sdr_y2r))  // :640-648
    return fail(E_UNSUPPORTED, "No implementation available for converting yuv to rgb for color gamut %d", sdr.cg);
  if (cfg.sdr_is_601) yuv2rgb_coeffs(UHDR_CG_DISPLAY_P3, p.sdr_y2r);  // :688-690
  if (!yuv2rgb_coeffs(hdr.cg, p.hdr_y2r))
    return fail(E_UNSUPPORTED, "No implementation available for converting yuv to rgb for color gamut %d", hdr.cg);
  if (!luminance_coeffs(sdr.cg, p.lum))  // luminanceFn = getLuminanceFn(sdr_intent->cg), :660
    return fail(E_UNSUPPORTED, "No implementation available for computing luminance for color gamut %d", sdr.cg);
  p.use_luminance = cfg.use_luminance;
  // map geometry :692-706
  int scale = cfg.scale_factor;
  if (scale <= 0) return fail(E_INVALID_PARAM, "invalid gainmap scale factor %d", scale);
  int mw = sdr.v.w / scale, mh = sdr.v.h / scale;
  if (mw == 0 || mh == 0) {
    int sf = sdr.v.w < sdr.v.h ? sdr.v.w : sdr.v.h;
    scale = sf >= 8 ? sf / 8 : 1;
    mw = sdr.v.w / scale;
    mh = sdr.v.h / scale;
  }
  p.scale = scale;
  p.map_w = mw;
  p.map_h = mh;
  p.nch = cfg.multichannel ? 3 : 1;
  p.sdr_nits = 203.0f;
  p.hdr_nits = hdr.ct == UHDR_CT_LINEAR ? 203.0f : hdr_white_nits;
  p.luts = ws.luts();
  int rc = E_OK;
  if (job->map.v.p[0]) {  // caller-provided destination (device-pointer stage API): geometry checked, pixels written there
    if (job->map.v.stride[0] < mw) return fail(E_INVALID_PARAM, "gain map destination stride %d is smaller than its width %d", job->map.v.stride[0], mw);
    job->map.v.fmt = cfg.multichannel ? F_RGB888 : F_Y400;
    job->map.v.w = mw;
    job->map.v.h = mh;
  } else {
    rc = alloc_dev_image(ws, cfg.multichannel ? F_RGB888 : F_Y400, mw, mh, map_align, &job->map);
  }
  if (rc) return rc;
  job->map.cg = hdr.cg;  // :714-716: initialised with the hdr intent's colour aspects
  job->map.ct = hdr.ct;
  job->map.range = hdr.range;
  p.dst = (uint8_t*)job->map.v.p[0];
  p.dst_stride = job->map.v.stride[0];
  job->nch = p.nch;
  job->hdr_white_nits = hdr_white_nits;
  job->gamma = cfg.gamma;
  job->target_nits = cfg.target_disp_peak_nits;
  job->use_base_cg = use_sdr_cg ? 1 : 0;
  job->onepass = cfg.preset == UHDR_USAGE_REALTIME;
  if (job->onepass) {
    p.min_boost = 1.0f;
    p.max_boost = hdr_white_nits / 203.0f;
    p.log2_min = std::log2(p.min_boost);  // float overloads: jpegr.cpp has `using namespace std`
    p.log2_max = std::log2(p.max_boost);
    p.gamma = cfg.gamma;
    {
      const double range = (double)(p.log2_max - p.log2_min);
      const double inv = 1.0 / range;   // IEEE division on the host: correctly rounded
      p.inv_log2_range = (range != 0.0 && std::isfinite(range) && std::isfinite(inv)) ? inv : 0.0;
    }
    if (gainmap_fast_eligible(p, true)) {
      unsigned* sched = (unsigned*)ws.dalloc(64);
      if (!sched) return E_MEM;
      CUDA_TRY(cudaMemsetAsync(sched, 0, 4, ws.stream()));
      TIMED(ws, "gainmap_onepass", launch_gainmap_fast(p, true, sched, ws.stream()));
    } else
      TIMED(ws, "gainmap_onepass", launch_gainmap_onepass(p, ws.stream()));
    return E_OK;
  }
  p.minmax = (unsigned*)ws.dalloc(128);
  float* d_minmax_f = (float*)ws.dalloc(64);
  job->h_minmax = (float*)ws.halloc(64);
  if (!p.minmax || !d_minmax_f || !job->h_minmax) return E_MEM;
  GainmapFinalizeParams f;
  f.minmax = p.minmax;
  f.minmax_f = d_minmax_f;
  f.nch = p.nch;
  f.has_user_max = cfg.max_content_boost != FLT_MAX;
  f.has_user_min = cfg.min_content_boost != FLT_MIN;
  f.log2_user_max = f.has_user_max ? std::log2(cfg.max_content_boost) : 0.0f;
  f.log2_user_min = f.has_user_min ? std::log2(cfg.min_content_boost) : 0.0f;
  // Two-pass on the fast kernels.  Scale 1: a statistics pass leaves only the extremes of the quotient (hdr+eps)/(sdr+eps)
  // per class (dark or not), and a code pass recomputes every quotient and maps it to its byte, taking the log2 in fp32
  // wherever the byte provably does not depend on more.  Scales 2 / 4: the float plane carries the quotient (sign = dark
  // pixel) to k_affine_q.  UHDR_B200_GAINS_PLANE=1 keeps the log2 in pass 1 and a plane of gains (measurement / triage).
  static const bool keep_gains_plane = getenv("UHDR_B200_GAINS_PLANE") != nullptr;
  job->exact_word = nullptr;
  p.gamma = cfg.gamma;
  // the code pass stores bytes like the one-pass kernel: gamma 1 and its conditions on dst
  const bool q2 = p.scale == 1 && !keep_gains_plane && gainmap_fast_eligible(p, true);
  if (q2) {
    CUDA_TRY(launch_init_q_keys(p.minmax, ws.stream()));
    // words 8 and 10: tile tickets of the two passes, 9: exact-path count (all zeroed by init_q_keys)
    TIMED(ws, "gainmap_pass1", launch_gainmap_q2(p, f, false, p.minmax + 8, nullptr, ws.stream()));
    TIMED(ws, "gainmap_affine", launch_gainmap_q2(p, f, true, p.minmax + 10, p.minmax + 9, ws.stream()));
    job->exact_word = reinterpret_cast<unsigned*>(job->h_minmax + 8);
    job->values = (unsigned long long)mw * mh * p.nch;
    CUDA_TRY(cudaMemcpyAsync(job->exact_word, p.minmax + 9, sizeof(unsigned), cudaMemcpyDeviceToHost, ws.stream()));
    CUDA_TRY(cudaMemcpyAsync(job->h_minmax, d_minmax_f, 6 * sizeof(float), cudaMemcpyDeviceToHost, ws.stream()));
    return E_OK;
  }
  p.gains = (float*)ws.dalloc(sizeof(float) * (size_t)mw * mh * p.nch);
  if (!p.gains) return E_MEM;
  AffineParams a;
  a.gains = p.gains;
  a.minmax_f = d_minmax_f;
  a.dst = p.dst;
  a.map_w = mw;
  a.map_h = mh;
  a.nch = p.nch;
  a.dst_stride = p.dst_stride;
  a.gamma = cfg.gamma;
  const bool pass1_fast = gainmap_fast_eligible(p, false), affine_fast = affine_fast_eligible(a);
  const bool q_mode = p.scale != 1 && pass1_fast && affine_fast && !keep_gains_plane;
  if (q_mode) {
    p.store_q = 1;
    CUDA_TRY(launch_init_q_keys(p.minmax, ws.stream()));
    TIMED(ws, "gainmap_pass1", launch_gainmap_fast(p, false, p.minmax + 8, ws.stream()));
    count_launches(1);
    TIMED(ws, "gainmap_affine", launch_affine_q(a, f, p.minmax + 9, ws.stream()));
    job->exact_word = reinterpret_cast<unsigned*>(job->h_minmax + 8);
    job->values = (unsigned long long)mw * mh * p.nch;
    CUDA_TRY(cudaMemcpyAsync(job->exact_word, p.minmax + 9, sizeof(unsigned), cudaMemcpyDeviceToHost, ws.stream()));
  } else {
    CUDA_TRY(launch_gainmap_init_minmax(p.minmax, ws.stream()));
    if (pass1_fast)
      TIMED(ws, "gainmap_pass1", launch_gainmap_fast(p, false, p.minmax + 8, ws.stream()));  // word 8: tile tickets, zeroed by init_minmax
    else
      TIMED(ws, "gainmap_pass1", launch_gainmap_pass1(p, ws.stream()));
    if (affine_fast) {  // clamp / hints folded into the affine pass
      count_launches(1);
      TIMED(ws, "gainmap_affine", launch_affine_fast(a, f, ws.stream()));
    } else {
      TIMED(ws, "gainmap_finalize", launch_gainmap_finalize(f, ws.stream()));
      TIMED(ws, "gainmap_affine", launch_gainmap_affine(a, ws.stream()));
    }
  }
  CUDA_TRY(cudaMemcpyAsync(job->h_minmax, d_minmax_f, 6 * sizeof(float), cudaMemcpyDeviceToHost, ws.stream()));
  return E_OK;
}

static std::atomic<unsigned long long> g_affine_values{0}, g_affine_exact{0};
void gainmap_affine_stats(unsigned long long out[2]) {
  out[0] = g_affine_values.load();
  out[1] = g_affine_exact.load();
}

void finish_gainmap_metadata(const GainmapJob& job, uhdr_gainmap_metadata_t* md) {
  const float kSdrWhiteNits = 203.0f;
  if (job.exact_word) {   // k_affine_q ran: how many values needed the fp64 log2
    g_affine_values.fetch_add(job.values);
    g_affine_exact.fetch_add(*job.exact_word);
  }
  if (job.onepass) {  // jpegr.cpp:724-734
    for (int i = 0; i < 3; i++) {
      md->max_content_boost[i] = job.hdr_white_nits / kSdrWhiteNits;
      md->min_content_boost[i] = 1.0f;
      md->gamma[i] = job.gamma;
      md->offset_sdr[i] = 0.0f;
      md->offset_hdr[i] = 0.0f;
    }
    md->hdr_capacity_min = 1.0f;
    md->hdr_capacity_max = job.target_nits != -1.0f ? job.target_nits / kSdrWhiteNits : md->max_content_boost[0];
  } else {            // :1031-1048, float exp2 (using namespace std)
    for (int i = 0; i < 3; i++) {
      const int c = job.nch == 3 ? i : 0;
      md->max_content_boost[i] = std::exp2(job.h_minmax[3 + c]);
      md->min_content_boost[i] = std::exp2(job.h_minmax[c]);
      md->gamma[i] = job.gamma;
      md->offset_sdr[i] = 1e-7f;
      md->offset_hdr[i] = 1e-7f;
    }
    md->hdr_capacity_min = 1.0f;
    md->hdr_capacity_max = job.target_nits != -1.0f ? job.target_nits / kSdrWhiteNits : job.hdr_white_nits / kSdrWhiteNits;
  }
  md->use_base_cg = job.use_base_cg;
}

// ------------------------------------------------------------------------------------------------
namespace {
// applyGainMap launches since process start: k_apply_lin1, k_apply_fast, k_apply_gainmap, k_resize_map
std::atomic<unsigned long long> g_apply_routes[4];
}  // namespace
void apply_route_stats(unsigned long long out[4]) {
  for (int i = 0; i < 4; i++) out[i] = g_apply_routes[i].load(std::memory_order_relaxed);
}

bool map_needs_resize(int w, int h, int map_w, int map_h) {  // :1652-1671
  const float pa = (float)w / h, ga = (float)map_w / map_h;
  return std::fabs(pa - ga) / pa > 0.01f;
}

int resize_map_dev(Workspace& ws, const DevImage& map, int w, int h, DevImage* rs) {
  if (!rs->v.p[0] && alloc_dev_image(ws, map.v.fmt, w, h, 64, rs))
    return fail(E_UNSUPPORTED, "encountered error while resizing the gainmap image from %ux%u to %ux%u", map.v.w, map.v.h, w, h);
  ResizeMapParams r;
  r.src = (const uint8_t*)map.v.p[0];
  r.src_w = map.v.w; r.src_h = map.v.h; r.src_stride = map.v.stride[0];
  r.bpp = map.v.fmt == F_RGBA8888 ? 4 : (map.v.fmt == F_RGB888 ? 3 : 1);
  r.dst = (uint8_t*)rs->v.p[0];
  r.dst_w = w; r.dst_h = h; r.dst_stride = rs->v.stride[0];
  TIMED(ws, "resize_gainmap", launch_resize_map(r, ws.stream()));
  g_apply_routes[3].fetch_add(1, std::memory_order_relaxed);
  rs->cg = map.cg; rs->ct = map.ct; rs->range = map.range;
  return E_OK;
}

static size_t idw_table_floats(int sdr_w, int map_w, int* scale_int, float* scale_f) {
  const float scale = (float)sdr_w / map_w;
  const bool integer = scale == std::floor(scale);
  *scale_int = integer ? (int)(size_t)scale : 0;
  *scale_f = scale;
  return integer && *scale_int > 1 ? (size_t)16 * *scale_int * *scale_int : 0;
}

size_t apply_table_floats(const DevImage& sdr, const DevImage& map) {
  int si;
  float sf;
  return 3 * 1024 + idw_table_floats(sdr.v.w, map.v.w, &si, &sf) + 768 + 4;
}

int apply_gainmap_dev(Workspace& ws, const DevImage& sdr, const DevImage& map_in,
                      const uhdr_gainmap_metadata_t& md, int out_ct, float max_display_boost,
                      DevImage* dst) {
  return apply_gainmap_region(&ws, ws.stream(), ws.luts(), sdr, map_in, md, out_ct, max_display_boost, dst, nullptr,
                              nullptr, nullptr);
}

int apply_gainmap_region(Workspace* ws, cudaStream_t stream, const float* luts, const DevImage& sdr,
                         const DevImage& map_in, const uhdr_gainmap_metadata_t& md, int out_ct,
                         float max_display_boost, DevImage* dst, const ApplyRegion* region, float* h_tab,
                         float* d_tab) {
  DevImage map = map_in;
  // validation, jpegr.cpp:1538-1614
  if (!dst || !dst->v.p[0])
    return fail(E_INVALID_PARAM, "apply gainmap method received nullptr for destination image or plane pointer");
  if (dst->v.stride[0] < dst->v.w)
    return fail(E_INVALID_PARAM, "destination stride (%u) cannot be less than image width (%u)", dst->v.stride[0], dst->v.w);
  if (out_ct != UHDR_CT_LINEAR && out_ct != UHDR_CT_HLG && out_ct != UHDR_CT_PQ)
    return fail(E_INVALID_PARAM, "apply gainmap method expects output color transfer to be one of "
                "{UHDR_CT_LINEAR, UHDR_CT_HLG, UHDR_CT_PQ}. Received %d", out_ct);
  if ((out_ct == UHDR_CT_LINEAR && dst->v.fmt != F_RGBAF16) || (out_ct != UHDR_CT_LINEAR && dst->v.fmt != F_RGBA1010102))
    return fail(E_INVALID_PARAM, "unsupported destination pixel format %d for output color transfer %d", dst->v.fmt, out_ct);
  // :1585 uhdr_validate_gainmap_metadata_descriptor.  The kernels rely on it: hdr_capacity_max == hdr_capacity_min
  // gives a NaN weight, and gamma < 0 an infinite gain-LUT input whose table index overflows
  if (int rc = validate_metadata(md)) return rc;
  if (sdr.v.fmt != F_YUV444 && sdr.v.fmt != F_YUV422 && sdr.v.fmt != F_YUV420 && sdr.v.fmt != F_RGB888 && sdr.v.fmt != F_RGBA8888)
    return fail(E_UNSUPPORTED, "apply gainmap method expects base image color format to be one of "
                "{YCbCr444, YCbCr422, YCbCr420, RGB888, RGBA8888}. Received %d", sdr.v.fmt);
  if (map.v.fmt != F_Y400 && map.v.fmt != F_RGB888 && map.v.fmt != F_RGBA8888)
    return fail(E_UNSUPPORTED, "apply gainmap method expects gainmap image color format to be one of "
                "{YCbCr400, RGB888, RGBA8888}. Received %d", map.v.fmt);
  ApplyParams p;
  memset(&p, 0, sizeof p);
  const int sdr_cg = sdr.cg == UHDR_CG_UNSPECIFIED ? (int)UHDR_CG_BT_709 : sdr.cg;
  const int hdr_cg = map.cg == UHDR_CG_UNSPECIFIED ? sdr_cg : map.cg;
  dst->cg = hdr_cg;
  bool ident = true;
  if (!gamut_matrix(hdr_cg, sdr_cg, p.gamut, &ident))
    return fail(E_ERROR, "No implementation available for converting from gamut %d to %d", sdr_cg, hdr_cg);
  p.gamut_on_sdr = md.use_base_cg ? 0 : 1;
  p.gamut_identity = ident ? 1 : 0;
  if (map_needs_resize(sdr.v.w, sdr.v.h, map.v.w, map.v.h)) {  // resize_image(gainmap_img, sdr_intent->w, sdr_intent->h)
    if (!ws) return fail(E_ERROR, "the gain map of a region render must have the base image's aspect ratio");
    DevImage rs;
    rs.v.p[0] = nullptr;
    if (int rc = resize_map_dev(*ws, map, sdr.v.w, sdr.v.h, &rs)) return rc;
    map = rs;
  }
  const size_t idw_floats = idw_table_floats(sdr.v.w, map.v.w, &p.scale_int, &p.scale_f);
  float display_boost = max_display_boost < md.hdr_capacity_max ? max_display_boost : md.hdr_capacity_max;
  float weight;
  if (display_boost != md.hdr_capacity_max) {  // :1680-1689, float log2 (using namespace std)
    weight = (std::log2(display_boost) - std::log2(md.hdr_capacity_min)) /
             (std::log2(md.hdr_capacity_max) - std::log2(md.hdr_capacity_min));
    weight = weight < 0.0f ? 0.0f : (weight > 1.0f ? 1.0f : weight);
  } else {
    weight = 1.0f;
  }
  // per-call tables: IDW (only needed for integer scale > 1) and the gain LUT
  GainmapMetadata m;
  static_assert(sizeof(GainmapMetadata) == sizeof(uhdr_gainmap_metadata_t), "layout");
  memcpy(&m, &md, sizeof m);
  const size_t tab_floats = 3 * 1024 + idw_floats + 768 + 4;  // + zeroed tile-counter words
  if (!h_tab) {
    h_tab = (float*)ws->halloc(sizeof(float) * tab_floats);
    d_tab = (float*)ws->dalloc(sizeof(float) * tab_floats);
    if (!h_tab || !d_tab) return E_MEM;
  }
  memset(h_tab + tab_floats - 4, 0, 4 * sizeof(float));
  build_gain_lut(m, weight, h_tab);
  {  // scale-1 shortcut table: gain-map byte -> gain factor.  mapUintToFloat (b / 255.0f), IDW
     // weights {1,0,0,0} and GainLUT::getGainFactor's index (gamma 1) composed on the host
    float* g8 = h_tab + 3 * 1024 + idw_floats;
    for (int c = 0; c < 3; c++)
      for (int b = 0; b < 256; b++) {
        const float g = static_cast<float>(b) / 255.0f;
        int32_t idx = static_cast<int32_t>(g * (1024 - 1) + 0.5);
        idx = idx < 0 ? 0 : (idx > 1023 ? 1023 : idx);
        g8[c * 256 + b] = h_tab[c * 1024 + idx];
      }
  }
  if (idw_floats) {
    build_idw_tables(p.scale_int, h_tab + 3 * 1024);   // straight into the pinned staging block
  }
  CUDA_TRY(cudaMemcpyAsync(d_tab, h_tab, sizeof(float) * tab_floats, cudaMemcpyHostToDevice, stream));
  p.gain_lut = d_tab;
  p.idw = d_tab + 3 * 1024;
  const bool single = metadata_single_channel(m);
  double max_off = 0.0;
  for (int c = 0; c < 3; c++) {
    p.gamma_inv[c] = 1.0f / md.gamma[single ? 0 : c];
    p.off_sdr[c] = md.offset_sdr[c];
    p.off_hdr[c] = md.offset_hdr[c];
    max_off = std::max(max_off, (double)md.offset_sdr[c]);
  }
  {  // a channel is (linear base + offset) * factor - offset, then a gamut row (sum of |coefficients| < 2.4), with
     // the linear base <= 1: below FLT_MAX / 4 nothing overflows, and without inf no NaN (0 * inf, inf - inf) occurs
    double max_f = 0.0;
    for (int i = 0; i < 3 * 1024; i++) max_f = std::max(max_f, (double)h_tab[i]);
    p.nan_possible = !(max_f * (1.0 + max_off) * 4.0 < (double)FLT_MAX);
  }
  yuv2rgb_coeffs(UHDR_CG_DISPLAY_P3, p.y2r);
  p.sdr = sdr.v;
  p.map = (const uint8_t*)map.v.p[0];
  p.map_w = map.v.w;
  p.map_h = map.v.h;
  p.map_stride = map.v.stride[0];
  p.map_bpp = map.v.fmt == F_RGBA8888 ? 4 : (map.v.fmt == F_RGB888 ? 3 : 1);
  p.map_nch = map.v.fmt == F_Y400 ? 1 : 3;
  p.out_ct = out_ct;
  p.out_nits = out_ct == UHDR_CT_HLG ? 1000.0f : 10000.0f;
  p.luts = luts;
  p.dst = (void*)dst->v.p[0];
  p.dst_stride = dst->v.stride[0];
  if (region) {  // the scale above is the whole image's
    p.sdr.w = region->w;
    p.sdr.h = region->h;
    p.ox = region->ox;
    p.oy = region->oy;
  }
  const bool fast = apply_fast_eligible(p);
  if (ws) ws->t_begin("apply_gainmap");
  const cudaError_t e = fast ? launch_apply_fast(p, d_tab + 3 * 1024 + idw_floats, stream) : launch_apply_gainmap(p, stream);
  if (ws) ws->t_end();
  CUDA_TRY(e);
  g_apply_routes[!fast ? 2 : p.scale_int == 1 && out_ct == UHDR_CT_LINEAR ? 0 : 1].fetch_add(1, std::memory_order_relaxed);
  return E_OK;
}

// ------------------------------------------------------------------------------------------------
int tonemap_dev(Workspace& ws, const DevImage& hdr, DevImage* sdr) {
  // jpegr.cpp:1986-2037
  if (hdr.v.fmt != F_P010 && hdr.v.fmt != F_YUV444_10 && hdr.v.fmt != F_RGBA1010102 && hdr.v.fmt != F_RGBAF16)
    return fail(E_UNSUPPORTED, "tonemap method expects hdr intent color format to be one of "
                "{P010, 30bppYCbCr444, RGBA1010102, RGBAHalfFloat}. Received %d", hdr.v.fmt);
  if (hdr.v.fmt == F_P010 && sdr->v.fmt != F_YUV420)
    return fail(E_UNSUPPORTED, "tonemap method expects sdr intent color format to be YCbCr420 if hdr intent is P010. Received %d", sdr->v.fmt);
  if (hdr.v.fmt == F_YUV444_10 && sdr->v.fmt != F_YUV444)
    return fail(E_UNSUPPORTED, "tonemap method expects sdr intent color format to be YCbCr444 if hdr intent is 30bppYCbCr444. Received %d", sdr->v.fmt);
  if ((hdr.v.fmt == F_RGBA1010102 || hdr.v.fmt == F_RGBAF16) && sdr->v.fmt != F_RGBA8888)
    return fail(E_UNSUPPORTED, "tonemap method expects sdr intent color format to be RGBA8888 if hdr intent is RGBA1010102 or RGBAHalfFloat. Received %d", sdr->v.fmt);
  TonemapParams p;
  memset(&p, 0, sizeof p);
  if (!yuv2rgb_coeffs(hdr.cg, p.y2r))
    return fail(E_UNSUPPORTED, "No implementation available for converting yuv to rgb for color gamut %d", hdr.cg);
  const float nits = reference_display_peak_nits(hdr.ct);
  if (nits == -1.0f)
    return fail(E_UNSUPPORTED, "received invalid peak brightness %f nits for hdr reference display with color transfer %d", nits, hdr.ct);
  sdr->cg = UHDR_CG_DISPLAY_P3;  // :2117-2119
  sdr->ct = UHDR_CT_SRGB;
  sdr->range = UHDR_CR_FULL_RANGE;
  bool ident = true;
  gamut_matrix(UHDR_CG_DISPLAY_P3, hdr.cg, p.gamut, &ident);
  p.gamut_identity = ident;
  p.hdr = hdr.v;
  p.hdr_ct = hdr.ct;
  p.headroom = nits / 203.0f;
  p.normalized = hdr.ct != UHDR_CT_LINEAR;
  p.luts = ws.luts();
  for (int i = 0; i < 3; i++) {
    p.dst[i] = (uint8_t*)sdr->v.p[i];
    p.dst_stride[i] = sdr->v.stride[i];
  }
  p.dst_fmt = sdr->v.fmt;
  TIMED(ws, "tonemap", launch_tonemap(p, ws.stream()));
  return E_OK;
}

int convert_yuv_dev(Workspace& ws, DevImage* img, int src_cg, int dst_cg, bool in_place) {
  // jpegr.cpp:436-518.  The reference converts its own deep copy of the intent in place; a device
  // image that must survive the call (resident encoder inputs) is converted into workspace scratch
  // and *img is redirected to it.
  if (src_cg < 0 || src_cg > 2) return fail(E_INVALID_PARAM, "Unrecognized src color gamut %d", src_cg);
  if (dst_cg < 0 || dst_cg > 2) return fail(E_INVALID_PARAM, "Unrecognized dest color gamut %d", dst_cg);
  if (src_cg == dst_cg) return E_OK;
  if (img->v.fmt != F_YUV420 && img->v.fmt != F_YUV444)
    return fail(E_UNSUPPORTED, "No implementation available for performing gamut conversion for color format %d", img->v.fmt);
  YuvConvParams p;
  yuv_matrix(src_cg, dst_cg, p.m);
  DevImage dst = *img;
  if (!in_place) {
    int rc = alloc_dev_image(ws, img->v.fmt, img->v.w, img->v.h, 64, &dst);
    if (rc) return rc;
    dst.cg = img->cg; dst.ct = img->ct; dst.range = img->range;
    dst.v.full_range = img->v.full_range;
  }
  for (int i = 0; i < 3; i++) {
    p.p[i] = (const uint8_t*)img->v.p[i];
    p.stride[i] = img->v.stride[i];
    p.d[i] = (uint8_t*)dst.v.p[i];
    p.dstride[i] = dst.v.stride[i];
  }
  *img = dst;
  p.w = img->v.w;
  p.h = img->v.h;
  p.fmt = img->v.fmt;
  TIMED(ws, "yuv_convert", launch_yuv_convert(p, ws.stream()));
  return E_OK;
}

int rgb_to_ycbcr_dev(Workspace& ws, const DevImage& rgb, DevImage* out) {
  if (rgb.v.fmt != F_RGBA8888 && rgb.v.fmt != F_RGB888)
    return fail(E_UNSUPPORTED, "convert_raw_input_to_ycbcr: unsupported packed format %d", rgb.v.fmt);
  RgbToYccParams p;
  memset(&p, 0, sizeof p);
  if (!rgb2yuv_coeffs(rgb.cg, p.k)) return fail(E_ERROR, "internal error : cannot convert packed rgb of color gamut %d to yuv", rgb.cg);
  int rc = alloc_dev_image(ws, F_YUV444, rgb.v.w, rgb.v.h, 64, out);
  if (rc) return rc;
  out->cg = rgb.cg;
  out->ct = rgb.ct;
  out->range = UHDR_CR_FULL_RANGE;
  out->v.full_range = 1;
  p.src = (const uint8_t*)rgb.v.p[0];
  p.src_stride = rgb.v.stride[0];
  p.bpp = rgb.v.fmt == F_RGBA8888 ? 4 : 3;
  for (int i = 0; i < 3; i++) p.dst[i] = (uint8_t*)out->v.p[i];
  p.dst_stride = out->v.stride[0];
  p.w = rgb.v.w;
  p.h = rgb.v.h;
  TIMED(ws, "rgb_to_ycbcr", launch_rgb_to_ycc(p, ws.stream()));
  return E_OK;
}

}  // namespace uhdr_b200
