// extern "C" stage entry points with HOST buffers (include/uhdr_b200.h): upload, run the device
// stage, download, synchronise.  These are what the parity tests call through ctypes.
#include <cstring>
#include <mutex>

#include "engine.h"

using namespace uhdr_b200;

namespace {
// one workspace per calling thread, created on first use and kept (arenas are rewound per call)
Workspace* tls_workspace() {
  static thread_local Workspace* ws = nullptr;
  if (!ws) {
    ws = new Workspace();
    if (ws->init() != E_OK) {
      delete ws;
      ws = nullptr;
    }
  }
  if (ws) ws->rewind();
  return ws;
}
}  // namespace

extern "C" {

UHDR_API const char* uhdr_b200_last_error(void) { return last_error(); }

UHDR_API int uhdr_b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

UHDR_API unsigned long long uhdr_b200_kernel_launches(void) { return launch_count(); }

UHDR_API size_t uhdr_b200_lut_blob_floats(void) { return kLutTotalFloats; }
UHDR_API int uhdr_b200_build_lut_blob(float* host_out) {
  build_lut_blob(host_out);
  return E_OK;
}
UHDR_API int uhdr_b200_install_lut_blob_dev(const void* device_ptr) {
  return install_luts_from_device(device_ptr);
}
UHDR_API int uhdr_b200_get_lut_blob(float* host_out) { return read_back_luts(host_out); }

UHDR_API int uhdr_b200_probe_log2(const float* in, float* out, int n) {
  Workspace* ws = tls_workspace();
  if (!ws) return E_ERROR;
  float* d_in = (float*)ws->dalloc((size_t)n * 4);
  float* d_out = (float*)ws->dalloc((size_t)n * 4);
  if (!d_in || !d_out) return E_MEM;
  CUDA_TRY(cudaMemcpyAsync(d_in, in, (size_t)n * 4, cudaMemcpyHostToDevice, ws->stream()));
  CUDA_TRY(launch_log2_probe(d_in, d_out, n, ws->stream()));
  CUDA_TRY(cudaMemcpyAsync(out, d_out, (size_t)n * 4, cudaMemcpyDeviceToHost, ws->stream()));
  return ws->sync();
}

UHDR_API void uhdr_b200_generate_stats(unsigned long long out[2]) {
  if (out) gainmap_affine_stats(out);
}

UHDR_API int uhdr_b200_probe_log2_fast(unsigned first_bits, unsigned count, float* worst) {
  Workspace* ws = tls_workspace();
  if (!ws || !worst) return E_ERROR;
  float* d_w = (float*)ws->dalloc(64);
  if (!d_w) return E_MEM;
  CUDA_TRY(cudaMemsetAsync(d_w, 0, 4, ws->stream()));
  CUDA_TRY(launch_log2_fast_probe(first_bits, count, d_w, ws->stream()));
  CUDA_TRY(cudaMemcpyAsync(worst, d_w, 4, cudaMemcpyDeviceToHost, ws->stream()));
  return ws->sync();
}

UHDR_API void uhdr_b200_tonemap_stats(unsigned long long out[2]) {
  if (out) tonemap_screen_stats(out);
}

UHDR_API void uhdr_b200_apply_stats(unsigned long long out[4]) {
  if (out) apply_route_stats(out);
}

UHDR_API int uhdr_b200_probe_pow_fast(unsigned first_bits, unsigned count, float* worst) {
  Workspace* ws = tls_workspace();
  if (!ws || !worst) return E_ERROR;
  float* d_w = (float*)ws->dalloc(64);
  if (!d_w) return E_MEM;
  CUDA_TRY(cudaMemsetAsync(d_w, 0, 4, ws->stream()));
  CUDA_TRY(launch_pow_fast_probe(first_bits, count, d_w, ws->stream()));
  CUDA_TRY(cudaMemcpyAsync(worst, d_w, 4, cudaMemcpyDeviceToHost, ws->stream()));
  return ws->sync();
}

UHDR_API int uhdr_b200_probe_powf(const float* in, float y, float* out, int n) {
  Workspace* ws = tls_workspace();
  if (!ws) return E_ERROR;
  float* d_in = (float*)ws->dalloc((size_t)n * 4);
  float* d_out = (float*)ws->dalloc((size_t)n * 4);
  if (!d_in || !d_out) return E_MEM;
  CUDA_TRY(cudaMemcpyAsync(d_in, in, (size_t)n * 4, cudaMemcpyHostToDevice, ws->stream()));
  CUDA_TRY(launch_powf_probe(d_in, y, d_out, n, ws->stream()));
  CUDA_TRY(cudaMemcpyAsync(out, d_out, (size_t)n * 4, cudaMemcpyDeviceToHost, ws->stream()));
  return ws->sync();
}

UHDR_API int uhdr_b200_generate_gainmap(const uhdr_raw_image_t* sdr, const uhdr_raw_image_t* hdr,
                                        const uhdr_b200_gm_config_t* cfg,
                                        uhdr_gainmap_metadata_t* md_out,
                                        uhdr_raw_image_t* gainmap_out) {
  if (!sdr || !hdr || !cfg || !md_out || !gainmap_out || !gainmap_out->planes[0])
    return fail(E_INVALID_PARAM, "received nullptr argument");
  Workspace* ws = tls_workspace();
  if (!ws) return E_ERROR;
  DevImage dsdr, dhdr;
  int rc = upload_image(*ws, *sdr, &dsdr);
  if (rc) return rc;
  rc = upload_image(*ws, *hdr, &dhdr);
  if (rc) return rc;
  GainmapJob job;
  rc = generate_gainmap_dev(*ws, dsdr, dhdr, *cfg, 64, &job);
  if (rc) return rc;
  gainmap_out->fmt = (uhdr_img_fmt_t)job.map.v.fmt;
  gainmap_out->cg = (uhdr_color_gamut_t)job.map.cg;
  gainmap_out->ct = (uhdr_color_transfer_t)job.map.ct;
  gainmap_out->range = (uhdr_color_range_t)job.map.range;
  gainmap_out->w = job.map.v.w;
  gainmap_out->h = job.map.v.h;
  gainmap_out->stride[0] = job.map.v.w;
  rc = download_image(*ws, job.map, gainmap_out);
  if (rc) return rc;
  rc = ws->sync();
  if (rc) return rc;
  finish_gainmap_metadata(job, md_out);
  return E_OK;
}

UHDR_API int uhdr_b200_apply_gainmap(const uhdr_raw_image_t* sdr, const uhdr_raw_image_t* gainmap,
                                     const uhdr_gainmap_metadata_t* md, int output_ct, int output_fmt,
                                     float max_display_boost, uhdr_raw_image_t* dest) {
  (void)output_fmt;
  if (!sdr || !gainmap || !md) return fail(E_INVALID_PARAM, "received nullptr argument");
  if (dest == nullptr || dest->planes[UHDR_PLANE_PACKED] == nullptr)
    return fail(E_INVALID_PARAM, "apply gainmap method received nullptr for destination image or plane pointer");
  if (dest->stride[UHDR_PLANE_PACKED] < dest->w)
    return fail(E_INVALID_PARAM, "destination stride (%u) cannot be less than image width (%u)",
                dest->stride[UHDR_PLANE_PACKED], dest->w);
  Workspace* ws = tls_workspace();
  if (!ws) return E_ERROR;
  DevImage dsdr, dmap, ddst;
  int rc = upload_image(*ws, *sdr, &dsdr);
  if (rc) return rc;
  rc = upload_image(*ws, *gainmap, &dmap);
  if (rc) return rc;
  rc = alloc_dev_image(*ws, dest->fmt, sdr->w, sdr->h, 64, &ddst);
  if (rc) return rc;
  rc = apply_gainmap_dev(*ws, dsdr, dmap, *md, output_ct, max_display_boost, &ddst);
  if (rc) return rc;
  dest->cg = (uhdr_color_gamut_t)ddst.cg;
  rc = download_image(*ws, ddst, dest);
  if (rc) return rc;
  return ws->sync();
}

UHDR_API int uhdr_b200_tonemap(const uhdr_raw_image_t* hdr, uhdr_raw_image_t* sdr) {
  if (!hdr || !sdr) return fail(E_INVALID_PARAM, "received nullptr argument");
  Workspace* ws = tls_workspace();
  if (!ws) return E_ERROR;
  DevImage dhdr, dsdr;
  int rc = upload_image(*ws, *hdr, &dhdr);
  if (rc) return rc;
  rc = alloc_dev_image(*ws, sdr->fmt, hdr->w, hdr->h, 64, &dsdr);
  if (rc) return rc;
  rc = tonemap_dev(*ws, dhdr, &dsdr);
  if (rc) return rc;
  sdr->cg = (uhdr_color_gamut_t)dsdr.cg;
  sdr->ct = (uhdr_color_transfer_t)dsdr.ct;
  sdr->range = (uhdr_color_range_t)dsdr.range;
  rc = download_image(*ws, dsdr, sdr);
  if (rc) return rc;
  return ws->sync();
}

UHDR_API int uhdr_b200_convert_yuv(uhdr_raw_image_t* image, int src_cg, int dst_cg) {
  if (!image) return fail(E_INVALID_PARAM, "received nullptr argument");
  Workspace* ws = tls_workspace();
  if (!ws) return E_ERROR;
  DevImage d;
  int rc = upload_image(*ws, *image, &d);
  if (rc) return rc;
  rc = convert_yuv_dev(*ws, &d, src_cg, dst_cg);
  if (rc) return rc;
  rc = download_image(*ws, d, image);
  if (rc) return rc;
  return ws->sync();
}

// ---- device-pointer stage entry points (include/uhdr_b200.h, "Internal FFI" of SURVEY section 8b) ----------
// Descriptors carry DEVICE pointers; kernels are enqueued on the caller's stream; nothing crosses PCIe.
namespace {
DevImage dev_view(const uhdr_raw_image_t& d) {
  DevImage v;
  memset(&v, 0, sizeof v);
  v.v.fmt = d.fmt;
  v.v.w = d.w;
  v.v.h = d.h;
  for (int i = 0; i < 3; i++) {
    v.v.p[i] = d.planes[i];
    v.v.stride[i] = d.stride[i];
  }
  v.v.full_range = d.range == UHDR_CR_FULL_RANGE;
  v.cg = d.cg;
  v.ct = d.ct;
  v.range = d.range;
  return v;
}
// The calling thread's workspace (scratch arenas) on the caller's stream for one call.  The arenas were
// rewound on entry: device scratch of the previous call is protected by stream order, but its pinned host
// staging (the per-call gain tables of applyGainMap) may still be waiting for its H2D copy, so a new call
// first waits for the event the previous one left behind.
struct StreamScope {
  Workspace* ws;
  cudaStream_t st;
  static cudaEvent_t& last_event() {
    static thread_local cudaEvent_t e = nullptr;
    return e;
  }
  StreamScope(Workspace* w, void* stream) : ws(w), st((cudaStream_t)stream) {
    if (!ws) return;
    if (last_event()) cudaEventSynchronize(last_event());
    ws->use_external_stream(st);
  }
  ~StreamScope() {
    if (!ws) return;
    if (!last_event()) cudaEventCreateWithFlags(&last_event(), cudaEventDisableTiming);
    if (last_event()) cudaEventRecord(last_event(), st);
    ws->clear_external_stream();
  }
};
}  // namespace

UHDR_API int uhdr_b200_generate_gainmap_dev(const uhdr_raw_image_t* sdr, const uhdr_raw_image_t* hdr, const uhdr_b200_gm_config_t* cfg,
                                            uhdr_gainmap_metadata_t* md_out, uhdr_raw_image_t* gainmap, void* stream) {
  if (!sdr || !hdr || !cfg || !md_out || !gainmap || !gainmap->planes[0]) return fail(E_INVALID_PARAM, "received nullptr argument");
  Workspace* ws = tls_workspace();
  if (!ws) return E_ERROR;
  StreamScope scope(ws, stream);
  GainmapJob job;
  job.map.v.p[0] = gainmap->planes[0];
  job.map.v.stride[0] = gainmap->stride[0];
  int rc = generate_gainmap_dev(*ws, dev_view(*sdr), dev_view(*hdr), *cfg, 64, &job);
  if (rc) return rc;
  gainmap->fmt = (uhdr_img_fmt_t)job.map.v.fmt;
  gainmap->cg = (uhdr_color_gamut_t)job.map.cg;
  gainmap->ct = (uhdr_color_transfer_t)job.map.ct;
  gainmap->range = (uhdr_color_range_t)job.map.range;
  gainmap->w = job.map.v.w;
  gainmap->h = job.map.v.h;
  // the two-pass preset derives the metadata from the image-wide min / max: those six floats are the only
  // bytes that travel, and the stream has to be drained for them; the one-pass metadata is known up front
  if (!job.onepass && (rc = ws->sync())) return rc;
  finish_gainmap_metadata(job, md_out);
  return E_OK;
}

UHDR_API int uhdr_b200_apply_gainmap_dev(const uhdr_raw_image_t* sdr, const uhdr_raw_image_t* gainmap, const uhdr_gainmap_metadata_t* md,
                                         int output_ct, float max_display_boost, uhdr_raw_image_t* dest, void* stream) {
  if (!sdr || !gainmap || !md || !dest || !dest->planes[0]) return fail(E_INVALID_PARAM, "received nullptr argument");
  Workspace* ws = tls_workspace();
  if (!ws) return E_ERROR;
  StreamScope scope(ws, stream);
  DevImage dd = dev_view(*dest);
  dd.v.w = sdr->w;
  dd.v.h = sdr->h;
  int rc = apply_gainmap_dev(*ws, dev_view(*sdr), dev_view(*gainmap), *md, output_ct, max_display_boost, &dd);
  if (rc) return rc;
  dest->w = sdr->w;
  dest->h = sdr->h;
  dest->cg = (uhdr_color_gamut_t)dd.cg;
  dest->ct = (uhdr_color_transfer_t)output_ct;
  dest->range = UHDR_CR_FULL_RANGE;
  return E_OK;
}

UHDR_API int uhdr_b200_tonemap_dev(const uhdr_raw_image_t* hdr, uhdr_raw_image_t* sdr, void* stream) {
  if (!hdr || !sdr || !sdr->planes[0]) return fail(E_INVALID_PARAM, "received nullptr argument");
  Workspace* ws = tls_workspace();
  if (!ws) return E_ERROR;
  StreamScope scope(ws, stream);
  DevImage ds = dev_view(*sdr);
  ds.v.w = hdr->w;
  ds.v.h = hdr->h;
  int rc = tonemap_dev(*ws, dev_view(*hdr), &ds);
  if (rc) return rc;
  sdr->w = hdr->w;
  sdr->h = hdr->h;
  sdr->cg = (uhdr_color_gamut_t)ds.cg;
  sdr->ct = (uhdr_color_transfer_t)ds.ct;
  sdr->range = (uhdr_color_range_t)ds.range;
  return E_OK;
}

UHDR_API int uhdr_b200_convert_yuv_dev(uhdr_raw_image_t* image, int src_cg, int dst_cg, void* stream) {
  if (!image) return fail(E_INVALID_PARAM, "received nullptr argument");
  Workspace* ws = tls_workspace();
  if (!ws) return E_ERROR;
  StreamScope scope(ws, stream);
  DevImage d = dev_view(*image);
  return convert_yuv_dev(*ws, &d, src_cg, dst_cg, /*in_place=*/true);
}

}  // extern "C"
