// extern "C" stage entry points with HOST buffers (include/uhdr_b200.h): upload, run the device
// stage, download, synchronise.  These are what the parity tests call through ctypes.
#include <cmath>
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

#include "codec.h"

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

UHDR_API void uhdr_b200_jpeg_encode_stats(unsigned long long out[10]) {
  if (out) jpeg_encode_stats(out);
}

UHDR_API void uhdr_b200_jpeg_encode_batch_stats(unsigned long long out[2]) {
  if (out) jpeg_encode_batch_stats(out);
}

UHDR_API void uhdr_b200_device_state_stats(unsigned long long out[2]) {
  if (out) device_state_stats(out);
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

// ---- whole-file codec on device images -------------------------------------------------------------------
}  // extern "C"
namespace uhdr_b200 {
// One codec per host thread and device (a handle is bound to the device that was current when it was made): a
// decode needs its second workspace and parked helper thread.  settle() first: an earlier decode's writes into a
// caller's planes may still read this codec's scratch.
int dev_codec(JpegRCodec** out) {
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  static thread_local std::vector<std::unique_ptr<JpegRCodec>> per_device;
  if ((int)per_device.size() <= dev) per_device.resize(dev + 1);
  std::unique_ptr<JpegRCodec>& c = per_device[dev];
  if (!c) {
    c.reset(new JpegRCodec());
    if (int rc = c->init()) {
      c.reset();
      return rc;
    }
  }
  if (int rc = c->settle()) return rc;
  c->ws().rewind();
  *out = c.get();
  return E_OK;
}

// the descriptor's planes: present, stride >= plane width, device memory of the current device, aligned to their
// element (a sample of the planar formats, a pixel of the packed ones; RGB888 is read byte by byte)
int check_dev_planes(const uhdr_raw_image_t& img, const char* what) {
  const int np = fmt_planes(img.fmt);
  if (np == 0) return fail(E_INVALID_PARAM, "%s: unsupported image format %d", what, img.fmt);
  for (int i = 0; i < np; i++) {
    int pw, ph, esz;
    fmt_plane_geom(img.fmt, img.w, img.h, i, &pw, &ph, &esz);
    if (!img.planes[i]) return fail(E_INVALID_PARAM, "%s: plane %d is a null pointer", what, i);
    if ((int)img.stride[i] < pw) return fail(E_INVALID_PARAM, "%s: plane %d stride %u < width %d", what, i, img.stride[i], pw);
    const int align = img.fmt == UHDR_IMG_FMT_24bppRGB888 ? 1 : esz;
    if ((uintptr_t)img.planes[i] % align)
      return fail(E_INVALID_PARAM, "%s: plane %d at %p is not aligned to its %d-byte elements", what, i, img.planes[i], align);
  }
  return E_OK;
}
int check_dev_memory(const uhdr_raw_image_t& img, const char* what) {
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  for (int i = 0; i < fmt_planes(img.fmt); i++) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, img.planes[i]) != cudaSuccess) {
      cudaGetLastError();
      return fail(E_INVALID_PARAM, "%s: plane %d at %p is not a CUDA pointer", what, i, img.planes[i]);
    }
    if (a.type != cudaMemoryTypeDevice || a.device != dev)
      return fail(E_INVALID_PARAM, "%s: plane %d at %p is not device memory of device %d", what, i, img.planes[i], dev);
  }
  return E_OK;
}
}  // namespace uhdr_b200

namespace {
// The batched entry points' items: grow-only per thread and item type, so a batch of the same or a smaller size
// takes no heap
template <class Item>
Item* batch_items(int n) {
  static thread_local std::vector<Item> its;
  if ((int)its.size() < n) its.resize(n);
  return its.data();
}

// the batched calls' scratch budget per group: 4 GiB, or UHDR_B200_BATCH_GROUP_BYTES
size_t batch_group_bytes() {
  size_t group = size_t(4) << 30;
  if (const char* e = getenv("UHDR_B200_BATCH_GROUP_BYTES")) group = strtoull(e, nullptr, 10);
  return group;
}

// The batched entry points' tail: run(group bytes) unless `rc` (dev_codec's code) already ends the call, that call-level
// error given to every item without one of its own, each item's status, and the first failing item's code and message
// ("<what> <index>: ")
template <class In, class Item, class Run>
int run_batch(In* items, Item* its, int n, int rc, Run run, const char* what = "item") {
  if (!rc) rc = run(batch_group_bytes());
  std::string call_err = rc ? last_error() : "";
  int first = -1;
  for (int i = 0; i < n; i++) {
    Item& b = its[i];
    if (rc && !b.rc) batch_fail(b, rc, call_err.c_str());
    items[i].status = b.rc;
    if (b.rc && first < 0) first = i;
  }
  if (first < 0) return E_OK;
  return fail(its[first].rc, "%s %d: %s", what, first, its[first].err);
}
}  // namespace

extern "C" {
namespace {
bool valid_scale(int k) { return k == 1 || k == 2 || k == 4 || k == 8; }
// the probed sizes at 1/k: libjpeg's output size of a scale_denom = k decode, ceil(size / k)
void scale_dims(DecodedInfo* info, int k) {
  info->width = (info->width + k - 1) / k;
  info->height = (info->height + k - 1) / k;
  info->gm_width = (info->gm_width + k - 1) / k;
  info->gm_height = (info->gm_height + k - 1) / k;
}
int check_out(const void* out, size_t* out_size) {
  if (!out || !out_size) return fail(E_INVALID_PARAM, "received nullptr for the output buffer");
  return E_OK;
}
}  // namespace

// the checks of uhdr_b200_decode_dev (k = 1) and uhdr_b200_decode_scaled_dev that need no device, sizes against the 1/k
// ones; *info: the probed file at 1/k
static int check_decode_args(const void* data, size_t size, int k, int out_ct, float max_display_boost, const uhdr_raw_image_t* dest,
                             const uhdr_raw_image_t* gainmap, DecodedInfo* out) {
  // uhdr_dec_set_image, uhdr_dec_set_out_max_display_boost and uhdr_decode's checks, in their order
  if (!data) return fail(E_INVALID_PARAM, "received nullptr for compressed img->data field");
  if (!dest) return fail(E_INVALID_PARAM, "received nullptr for destination image");
  if (!std::isfinite(max_display_boost) || max_display_boost < 1.0f)
    return fail(E_INVALID_PARAM, "invalid display boost %f, expects to be >= 1.0f}", max_display_boost);
  DecodedInfo& info = *out;
  int rc = JpegRCodec().probe((const uint8_t*)data, size, &info);  // host only
  if (rc) return rc;
  scale_dims(&info, k);
  const int fmt = dest->fmt;
  if ((fmt == UHDR_IMG_FMT_32bppRGBA1010102 && out_ct != UHDR_CT_HLG && out_ct != UHDR_CT_PQ) ||
      (fmt == UHDR_IMG_FMT_64bppRGBAHalfFloat && out_ct != UHDR_CT_LINEAR) ||
      (fmt == UHDR_IMG_FMT_32bppRGBA8888 && out_ct != UHDR_CT_SRGB) ||
      (fmt != UHDR_IMG_FMT_32bppRGBA1010102 && fmt != UHDR_IMG_FMT_64bppRGBAHalfFloat && fmt != UHDR_IMG_FMT_32bppRGBA8888))
    return fail(E_INVALID_PARAM, "unsupported output pixel format and output color transfer pair");
  if ((int)dest->w != info.width || (int)dest->h != info.height)
    return fail(E_INVALID_PARAM, "destination image is %ux%u, the primary image %dx%d", dest->w, dest->h, info.width, info.height);
  if ((rc = check_dev_planes(*dest, "destination"))) return rc;
  if (gainmap) {
    if ((int)gainmap->w != info.gm_width || (int)gainmap->h != info.gm_height)
      return fail(E_INVALID_PARAM, "gain-map image is %ux%u, the gain map %dx%d", gainmap->w, gainmap->h, info.gm_width,
                  info.gm_height);
    if (!gainmap->planes[0] || gainmap->stride[0] < gainmap->w)
      return fail(E_INVALID_PARAM, "gain-map image: null plane or stride %u < width %u", gainmap->stride[0], gainmap->w);
  }
  return E_OK;
}

// ... and those that need the device, after dev_codec()
static int check_decode_memory(const uhdr_raw_image_t* dest, const uhdr_raw_image_t* gainmap, const DecodedInfo& info) {
  int rc = check_dev_memory(*dest, "destination");
  if (rc) return rc;
  if (gainmap) {
    uhdr_raw_image_t g = *gainmap;
    g.fmt = info.gm_channels == 1 ? UHDR_IMG_FMT_8bppYCbCr400 : UHDR_IMG_FMT_32bppRGBA8888;  // what the call writes
    if ((rc = check_dev_planes(g, "gain-map image")) || (rc = check_dev_memory(g, "gain-map image"))) return rc;
  }
  return E_OK;
}

static int decode_dev(const void* data, size_t size, int k, int out_ct, float max_display_boost, uhdr_raw_image_t* dest,
                      uhdr_raw_image_t* gainmap, uhdr_gainmap_metadata_t* metadata_out, void* stream) {
  DecodedInfo info;
  int rc = check_decode_args(data, size, k, out_ct, max_display_boost, dest, gainmap, &info);
  if (rc) return rc;
  JpegRCodec* c = nullptr;
  if ((rc = dev_codec(&c))) return rc;
  if ((rc = check_decode_memory(dest, gainmap, info))) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  return c->decode((const uint8_t*)data, size, out_ct, dest->fmt, max_display_boost, dest, gainmap, metadata_out, &info, &st, k);
}

UHDR_API int uhdr_b200_decode_dev(const void* data, size_t size, int out_ct, float max_display_boost, uhdr_raw_image_t* dest,
                                  uhdr_raw_image_t* gainmap, uhdr_gainmap_metadata_t* metadata_out, void* stream) {
  return decode_dev(data, size, 1, out_ct, max_display_boost, dest, gainmap, metadata_out, stream);
}

UHDR_API int uhdr_b200_decode_scaled_dev(const void* data, size_t size, int k, int out_ct, float max_display_boost,
                                         uhdr_raw_image_t* dest, uhdr_raw_image_t* gainmap,
                                         uhdr_gainmap_metadata_t* metadata_out, void* stream) {
  if (!valid_scale(k)) return fail(E_INVALID_PARAM, "scale denominator %d, expects 1, 2, 4 or 8", k);
  return decode_dev(data, size, k, out_ct, max_display_boost, dest, gainmap, metadata_out, stream);
}

UHDR_API int uhdr_b200_decode_batch_dev(uhdr_b200_decode_item_t* items, int n, int k, int out_ct, float max_display_boost,
                                        void* stream) {
  if (!items) return fail(E_INVALID_PARAM, "received nullptr for the items");
  if (n < 1) return fail(E_INVALID_PARAM, "received %d items, expects at least 1", n);
  if (!valid_scale(k)) return fail(E_INVALID_PARAM, "scale denominator %d, expects 1, 2, 4 or 8", k);
  DecodeBatchItem* its = batch_items<DecodeBatchItem>(n);
  for (int i = 0; i < n; i++) {
    const uhdr_b200_decode_item_t& in = items[i];
    DecodeBatchItem& b = its[i];
    b.data = (const uint8_t*)in.data;
    b.size = in.size;
    b.dest = in.dest_dev;
    b.gainmap = in.gainmap_dev;
    b.md_out = in.metadata_out;
    b.rc = check_decode_args(in.data, in.size, k, out_ct, max_display_boost, in.dest_dev, in.gainmap_dev, &b.info);
    if (b.rc) snprintf(b.err, sizeof b.err, "%s", last_error());
  }
  JpegRCodec* c = nullptr;
  return run_batch(items, its, n, dev_codec(&c), [&](size_t group) {
    for (int i = 0; i < n; i++) {
      DecodeBatchItem& b = its[i];
      if (!b.rc && (b.rc = check_decode_memory(b.dest, b.gainmap, b.info))) snprintf(b.err, sizeof b.err, "%s", last_error());
    }
    return c->decode_batch(its, n, k, out_ct, max_display_boost, (cudaStream_t)stream, group);
  });
}

UHDR_API int uhdr_b200_scaled_dims(const void* data, size_t size, int k, unsigned* w, unsigned* h, unsigned* gm_w,
                                   unsigned* gm_h) {
  if (!valid_scale(k)) return fail(E_INVALID_PARAM, "scale denominator %d, expects 1, 2, 4 or 8", k);
  if (!data || !w || !h || !gm_w || !gm_h) return fail(E_INVALID_PARAM, "received nullptr argument");
  DecodedInfo info;
  int rc = JpegRCodec().probe((const uint8_t*)data, size, &info);  // host only, no device needed
  if (rc) return rc;
  scale_dims(&info, k);
  *w = info.width;
  *h = info.height;
  *gm_w = info.gm_width;
  *gm_h = info.gm_height;
  return E_OK;
}

UHDR_API int uhdr_b200_encode_dev(const uhdr_raw_image_t* hdr, const uhdr_raw_image_t* sdr, const uhdr_b200_gm_config_t* cfg,
                                  int base_quality, const void* exif, size_t exif_size, void* out, size_t cap,
                                  size_t* out_size, void* stream) {
  // uhdr_enc_set_raw_image per intent, the setters' ranges for the configuration, then uhdr_encode
  if (!hdr) return fail(E_INVALID_PARAM, "received nullptr for raw image handle");
  int rc = validate_raw_intent(*hdr, UHDR_HDR_IMG);
  if (rc) return rc;
  if (sdr) {
    if ((rc = validate_raw_intent(*sdr, UHDR_SDR_IMG))) return rc;
    if (sdr->w != hdr->w || sdr->h != hdr->h)
      return fail(E_INVALID_PARAM, "image resolutions mismatch: hdr intent: %dx%d, sdr intent: %dx%d", hdr->w, hdr->h, sdr->w, sdr->h);
  }
  if (!cfg) return fail(E_INVALID_PARAM, "received nullptr for the gain-map configuration");
  // the setters' ranges (uhdr_enc_set_quality, _gainmap_scale_factor, _gainmap_gamma, _preset,
  // _min_max_content_boost, _target_display_peak_brightness); FLT_MIN / FLT_MAX / -1 = unset pass as they do there
  if (base_quality < 0 || base_quality > 100 || cfg->quality < 0 || cfg->quality > 100)
    return fail(E_INVALID_PARAM, "invalid quality factor %d / %d, expects in range [0-100]", base_quality, cfg->quality);
  if (cfg->scale_factor <= 0 || cfg->scale_factor > 128)
    return fail(E_INVALID_PARAM, "gainmap scale factor is expected to be in range (0, 128], received %d", cfg->scale_factor);
  if (!std::isfinite(cfg->gamma) || cfg->gamma <= 0.0f)
    return fail(E_INVALID_PARAM, "unsupported gainmap gamma %f, expects to be > 0", cfg->gamma);
  if (cfg->preset != UHDR_USAGE_REALTIME && cfg->preset != UHDR_USAGE_BEST_QUALITY)
    return fail(E_INVALID_PARAM, "invalid preset %d, expects one of {UHDR_USAGE_REALTIME, UHDR_USAGE_BEST_QUALITY}", cfg->preset);
  const float mn = cfg->min_content_boost, mx = cfg->max_content_boost, nits = cfg->target_disp_peak_nits;
  if (!std::isfinite(mn) || !std::isfinite(mx))
    return fail(E_INVALID_PARAM, "received an argument with value either NaN or infinite. Configured min boost %f, max boost %f", mx, mn);
  if (mx < mn)
    return fail(E_INVALID_PARAM, "Invalid min boost / max boost configuration. configured max boost %f is less than min boost %f", mx, mn);
  if (mn <= 0.0f) return fail(E_INVALID_PARAM, "Invalid min boost configuration %f, expects > 0.0f", mn);
  if (nits != -1.0f && (!std::isfinite(nits) || nits < 203.0f || nits > 10000.0f))
    return fail(E_INVALID_PARAM, "unexpected target display peak brightness nits %f, expects to be with in range [%f, %f]", nits,
                203.0f, 10000.0f);
  if (exif_size && !exif) return fail(E_INVALID_PARAM, "received nullptr for exif->data field");
  if ((rc = check_out(out, out_size))) return rc;
  if ((rc = check_dev_planes(*hdr, "hdr intent")) || (sdr && (rc = check_dev_planes(*sdr, "sdr intent")))) return rc;
  JpegRCodec* c = nullptr;
  if ((rc = dev_codec(&c))) return rc;
  if ((rc = check_dev_memory(*hdr, "hdr intent")) || (sdr && (rc = check_dev_memory(*sdr, "sdr intent")))) return rc;
  // on the caller's stream: the inputs are read after its earlier work; the call returns with the file complete
  c->ws().use_external_stream((cudaStream_t)stream);
  const DevImage dh = dev_view(*hdr), ds = sdr ? dev_view(*sdr) : DevImage{};
  uhdr_b200_gm_config_t gcfg = *cfg;
  gcfg.sdr_is_601 = 0;     // what uhdr_encode passes to generateGainMap
  gcfg.use_luminance = 1;
  rc = c->encode(dh, sdr ? &ds : nullptr, gcfg, base_quality, (const uint8_t*)exif, exif_size, (uint8_t*)out, cap, out_size,
                 /*caller_planes=*/true);
  if (rc) c->ws().sync();  // an error return can leave work in flight that reads the workspace
  c->ws().clear_external_stream();
  return rc;
}

UHDR_API int uhdr_b200_transcode(const void* data, size_t size, const uhdr_b200_transcode_config_t* cfg, void* out, size_t cap,
                                 size_t* out_size) {
  if (!data) return fail(E_INVALID_PARAM, "received nullptr for compressed img->data field");
  if (!cfg) return fail(E_INVALID_PARAM, "received nullptr for the transcode configuration");
  int rc = check_out(out, out_size);
  if (rc) return rc;
  if (!valid_scale(cfg->k)) return fail(E_INVALID_PARAM, "scale denominator %d, expects 1, 2, 4 or 8", cfg->k);
  if (cfg->base_quality < 0 || cfg->base_quality > 100 || cfg->gainmap_quality < 0 || cfg->gainmap_quality > 100)
    return fail(E_INVALID_PARAM, "invalid quality factor %d / %d, expects in range [0-100]", cfg->base_quality, cfg->gainmap_quality);
  DecodedInfo info;
  if ((rc = JpegRCodec().probe((const uint8_t*)data, size, &info))) return rc;  // host only
  JpegRCodec* c = nullptr;
  if ((rc = dev_codec(&c))) return rc;
  return c->transcode((const uint8_t*)data, size, info, *cfg, (uint8_t*)out, cap, out_size);
}

UHDR_API int uhdr_b200_transcode_batch(uhdr_b200_transcode_item_t* items, int n, const uhdr_b200_transcode_config_t* cfg) {
  // uhdr_b200_transcode's call-level checks, before any device work
  if (!items) return fail(E_INVALID_PARAM, "received nullptr for the items");
  if (n < 1) return fail(E_INVALID_PARAM, "received %d items, expects at least 1", n);
  if (!cfg) return fail(E_INVALID_PARAM, "received nullptr for the transcode configuration");
  if (!valid_scale(cfg->k)) return fail(E_INVALID_PARAM, "scale denominator %d, expects 1, 2, 4 or 8", cfg->k);
  if (cfg->base_quality < 0 || cfg->base_quality > 100 || cfg->gainmap_quality < 0 || cfg->gainmap_quality > 100)
    return fail(E_INVALID_PARAM, "invalid quality factor %d / %d, expects in range [0-100]", cfg->base_quality, cfg->gainmap_quality);
  TranscodeBatchItem* its = batch_items<TranscodeBatchItem>(n);
  for (int i = 0; i < n; i++) {
    const uhdr_b200_transcode_item_t& in = items[i];
    TranscodeBatchItem& b = its[i];
    b.data = (const uint8_t*)in.data;
    b.size = in.size;
    b.out = (uint8_t*)in.out;
    b.cap = in.cap;
    b.out_size = 0;
    // uhdr_b200_transcode's per-file checks, in its order
    b.rc = !in.data ? fail(E_INVALID_PARAM, "received nullptr for compressed img->data field")
                    : !in.out ? fail(E_INVALID_PARAM, "received nullptr for the output buffer")
                              : JpegRCodec().probe(b.data, b.size, &b.info);   // host only
    if (b.rc) snprintf(b.err, sizeof b.err, "%s", last_error());
  }
  JpegRCodec* c = nullptr;
  const int rc = run_batch(items, its, n, dev_codec(&c), [&](size_t group) { return c->transcode_batch(its, n, *cfg, group); });
  // out_size: bytes written, or with UHDR_CODEC_MEM_ERROR the size needed (0 when the file was not assembled)
  for (int i = 0; i < n; i++) items[i].out_size = !its[i].rc || its[i].rc == E_MEM ? its[i].out_size : 0;
  return rc;
}

namespace {
// uhdr_b200_transcode_ladder's argument checks of the file, which touch no rung
int ladder_args(const void* data, const uhdr_b200_transcode_rung_t* rungs, int n) {
  if (!data) return fail(E_INVALID_PARAM, "received nullptr for compressed img->data field");
  if (!rungs) return fail(E_INVALID_PARAM, "received nullptr for the rungs");
  if (n < 1 || n > kLadderMaxRungs) return fail(E_INVALID_PARAM, "received %d rungs, expects 1 to %d", n, kLadderMaxRungs);
  return E_OK;
}

// Both ladder entry points: per file its argument checks (its status, no rung touched), then per rung
// uhdr_b200_transcode's argument checks in its order, then the file's probe (host only), whose error goes to every rung
// still valid; the device work when some rung is valid; the call-level error given to every rung without one of its
// own; each rung's status and out_size, and each file's status: what uhdr_b200_transcode_ladder returns for it alone.
// The return value is the first failing file's status, and the last error its message, named "file <i>: " when
// `name_files`.
int run_ladders(uhdr_b200_transcode_file_t* files, int n, bool name_files) {
  LadderFile* lf = batch_items<LadderFile>(n);
  int nr = 0;
  for (int i = 0; i < n; i++) {
    const uhdr_b200_transcode_file_t& in = files[i];
    lf[i].rc = ladder_args(in.data, in.rungs, in.n);
    if (lf[i].rc) snprintf(lf[i].err, sizeof lf[i].err, "%s", last_error());
    lf[i].r0 = nr;
    lf[i].nr = lf[i].rc ? 0 : in.n;
    nr += lf[i].nr;
  }
  TranscodeBatchItem* its = batch_items<TranscodeBatchItem>(nr);
  bool any = false;
  for (int f = 0; f < n; f++) {
    LadderFile& F = lf[f];
    if (F.rc) continue;
    const uhdr_b200_transcode_file_t& in = files[f];
    F.data = (const uint8_t*)in.data;
    bool valid = false;
    for (int i = 0; i < F.nr; i++) {
      const uhdr_b200_transcode_rung_t& r = in.rungs[i];
      const uhdr_b200_transcode_config_t& cfg = r.cfg;
      TranscodeBatchItem& b = its[F.r0 + i];
      b.data = F.data;
      b.size = in.size;
      b.cfg = cfg;
      b.out = (uint8_t*)r.out;
      b.cap = r.cap;
      b.out_size = 0;
      // uhdr_b200_transcode's argument checks, in its order
      b.rc = !r.out ? fail(E_INVALID_PARAM, "received nullptr for the output buffer")
             : !valid_scale(cfg.k) ? fail(E_INVALID_PARAM, "scale denominator %d, expects 1, 2, 4 or 8", cfg.k)
             : cfg.base_quality < 0 || cfg.base_quality > 100 || cfg.gainmap_quality < 0 || cfg.gainmap_quality > 100
                 ? fail(E_INVALID_PARAM, "invalid quality factor %d / %d, expects in range [0-100]", cfg.base_quality,
                        cfg.gainmap_quality)
                 : E_OK;
      if (b.rc) snprintf(b.err, sizeof b.err, "%s", last_error());
      valid |= !b.rc;
    }
    F.info = DecodedInfo();
    if (valid) {
      if (const int prc = JpegRCodec().probe(F.data, in.size, &F.info)) {
        for (int i = 0; i < F.nr; i++)
          if (!its[F.r0 + i].rc) batch_fail(its[F.r0 + i], prc, last_error());
        valid = false;
      }
    }
    for (int i = 0; i < F.nr; i++) its[F.r0 + i].info = F.info;
    any |= valid;
  }
  JpegRCodec* c = nullptr;
  int rc = any ? dev_codec(&c) : E_OK;
  if (!rc && any) rc = c->transcode_ladders(lf, n, its, batch_group_bytes());
  const std::string call_err = rc ? last_error() : "";
  int first = -1;
  for (int f = 0; f < n; f++) {
    LadderFile& F = lf[f];
    if (F.rc) {
      files[f].status = F.rc;
      if (first < 0) first = f;
      continue;
    }
    int fr = -1;
    for (int i = 0; i < F.nr; i++) {
      TranscodeBatchItem& b = its[F.r0 + i];
      if (rc && !b.rc) batch_fail(b, rc, call_err.c_str());
      uhdr_b200_transcode_rung_t& r = files[f].rungs[i];
      r.status = b.rc;
      // out_size: bytes written, or with UHDR_CODEC_MEM_ERROR the size needed (0 when the file was not assembled)
      r.out_size = !b.rc || b.rc == E_MEM ? b.out_size : 0;
      if (b.rc && fr < 0) fr = i;
    }
    files[f].status = fr < 0 ? E_OK : its[F.r0 + fr].rc;
    if (fr >= 0) snprintf(F.err, sizeof F.err, "rung %d: %s", fr, its[F.r0 + fr].err);
    if (fr >= 0 && first < 0) first = f;
  }
  if (first < 0) return E_OK;
  if (name_files) return fail(files[first].status, "file %d: %s", first, lf[first].err);
  return fail(files[first].status, "%s", lf[first].err);
}
}  // namespace

UHDR_API int uhdr_b200_transcode_ladder(const void* data, size_t size, uhdr_b200_transcode_rung_t* rungs, int n) {
  if (int rc = ladder_args(data, rungs, n)) return rc;
  uhdr_b200_transcode_file_t f{data, size, rungs, n, 0};
  return run_ladders(&f, 1, false);
}

UHDR_API int uhdr_b200_transcode_ladders(uhdr_b200_transcode_file_t* files, int n) {
  if (!files) return fail(E_INVALID_PARAM, "received nullptr for the files");
  if (n < 1) return fail(E_INVALID_PARAM, "received %d files, expects at least 1", n);
  return run_ladders(files, n, true);
}

UHDR_API int uhdr_b200_jpeg_encode_dev(const uhdr_raw_image_t* img, int quality, const void* icc, size_t icc_size, void* out,
                                       size_t cap, size_t* out_size, void* stream) {
  if (!img) return fail(E_INVALID_PARAM, "received nullptr argument");
  if (img->w == 0 || img->h == 0) return fail(E_INVALID_PARAM, "image has zero dimension");
  int rc = check_out(out, out_size);
  if (rc) return rc;
  if ((rc = check_dev_planes(*img, "image"))) return rc;
  JpegRCodec* c = nullptr;
  if ((rc = dev_codec(&c))) return rc;
  if ((rc = check_dev_memory(*img, "image"))) return rc;
  c->ws().use_external_stream((cudaStream_t)stream);
  rc = compress_image_dev(c->ws(), dev_view(*img), quality, icc, icc_size, /*caller_planes=*/true, (uint8_t*)out, cap,
                          out_size);
  if (rc) c->ws().sync();
  c->ws().clear_external_stream();
  return rc;
}

}  // extern "C"
