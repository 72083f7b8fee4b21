// Device-resident JPEG/R images (uhdr_b200_image_*, include/uhdr_b200.h): both JPEGs are decoded once, at open, and
// any rectangle of the result is then rendered for any display boost and output transfer by the apply kernel (or the
// colour conversion of an SRGB output) alone.  A render reads the base planes and the map with absolute coordinates
// and writes the caller's destination relative to the rectangle, so it equals that crop of uhdr_b200_decode_dev /
// uhdr_b200_decode_scaled_dev.
#include <cmath>
#include <cstring>

#include "codec.h"

using namespace uhdr_b200;

struct uhdr_b200_image {
  // per-render tables (GainLUT, IDW, scale-1 byte tables) depend on the boost: a small ring of pinned staging /
  // device copies, each free again once the event recorded behind its render has completed
  static constexpr int kSlots = 4;
  int dev = -1;
  int w = 0, h = 0, gm_w = 0, gm_h = 0;   // the 1/k image and the gain map as decoded
  const float* luts = nullptr;
  DevImage sdr{}, map{};                  // own memory; map resized to the base image's size when its aspect differs
  uhdr_gainmap_metadata_t md{};
  YccToRgbaParams rgba{};                 // SRGB renders: all but the region and destination
  size_t tab_floats = 0;
  float* h_tab[kSlots] = {};
  float* d_tab[kSlots] = {};
  cudaEvent_t done[kSlots] = {};
  bool used[kSlots] = {};
  int next = 0;
  // exactly sized blocks: the planes, map and device tables in one, the staging tables in the other; a release
  // parks them like a handle's (uhdr_b200_trim_cache)
  Arena dmem{false, 4096}, hmem{true, 4096};

  ~uhdr_b200_image() {
    for (int i = 0; i < kSlots; i++)
      if (done[i]) {
        if (used[i]) cudaEventSynchronize(done[i]);
        cudaEventDestroy(done[i]);
      }
  }
};

namespace {
size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// the device that was current at open, for the length of a call
struct DeviceScope {
  int prev = -1, dev;
  explicit DeviceScope(int d) : dev(d) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceScope() {
    if (prev >= 0 && prev != dev) cudaSetDevice(prev);
  }
};

// one plane of `src` (device memory) into `dst` at `pitch` bytes
int copy_plane(const DevImage& src, int i, void* dst, size_t pitch, cudaStream_t s) {
  int pw, ph, esz;
  fmt_plane_geom(src.v.fmt, src.v.w, src.v.h, i, &pw, &ph, &esz);
  CUDA_TRY(cudaMemcpy2DAsync(dst, pitch, src.v.p[i], (size_t)src.v.stride[i] * esz, (size_t)pw * esz, ph,
                             cudaMemcpyDeviceToDevice, s));
  return E_OK;
}

// the object's layout, its allocation and the copies of what the codec decoded, on c's stream
int make_resident(JpegRCodec& c, const DevImage& sdr, const DevImage& map, uhdr_b200_image* img) {
  Workspace& ws = c.ws();
  const int np = fmt_planes(sdr.v.fmt);
  const bool resize = map_needs_resize(sdr.v.w, sdr.v.h, map.v.w, map.v.h);
  const int mw = resize ? sdr.v.w : map.v.w, mh = resize ? sdr.v.h : map.v.h;
  const int mesz = map.v.fmt == F_Y400 ? 1 : 4;
  size_t off[5], pitch[4], total = 0;
  for (int i = 0; i < np; i++) {   // strides of 64 pixels, like alloc_dev_image; Cb and Cr share one
    int pw, ph, esz;
    fmt_plane_geom(sdr.v.fmt, sdr.v.w, sdr.v.h, i, &pw, &ph, &esz);
    pitch[i] = align_up(pw, 64);
    off[i] = total;
    total += align_up(pitch[i] * ph, 256);
  }
  pitch[3] = align_up(mw, 64);
  off[3] = total;
  total += align_up(pitch[3] * mesz * mh, 256);
  DevImage probe_map = map;
  probe_map.v.w = mw;
  probe_map.v.h = mh;
  img->tab_floats = apply_table_floats(sdr, probe_map);
  const size_t tab_bytes = align_up(img->tab_floats * sizeof(float), 256);
  off[4] = total;
  total += uhdr_b200_image::kSlots * tab_bytes;
  char* base = (char*)img->dmem.alloc(total);
  char* hbase = (char*)img->hmem.alloc(uhdr_b200_image::kSlots * tab_bytes);
  if (!base || !hbase) return E_MEM;
  img->sdr = sdr;
  for (int i = 0; i < np; i++) {
    img->sdr.v.p[i] = base + off[i];
    img->sdr.v.stride[i] = (int)pitch[i];
    if (int rc = copy_plane(sdr, i, base + off[i], pitch[i], ws.stream())) return rc;
  }
  img->map = map;
  img->map.v.p[0] = base + off[3];
  img->map.v.stride[0] = (int)pitch[3];
  img->map.v.w = mw;
  img->map.v.h = mh;
  if (resize) {  // once, here: applyGainMap then sees a map of the base image's size
    if (int rc = resize_map_dev(ws, map, mw, mh, &img->map)) return rc;
  } else if (int rc = copy_plane(map, 0, base + off[3], pitch[3] * mesz, ws.stream())) {
    return rc;
  }
  for (int i = 0; i < uhdr_b200_image::kSlots; i++) {
    img->d_tab[i] = (float*)(base + off[4] + i * tab_bytes);
    img->h_tab[i] = (float*)(hbase + i * tab_bytes);
    CUDA_TRY(cudaEventCreateWithFlags(&img->done[i], cudaEventDisableTiming));
  }
  // k_ycc_to_rgba as decode_jpeg_dev sets it up for DECODE_TO_RGB_CS: chroma upsampled from 4:2:0 / 4:2:2
  YccToRgbaParams& p = img->rgba;
  p.y = (const uint8_t*)img->sdr.v.p[0];
  p.cb = (const uint8_t*)img->sdr.v.p[1];
  p.cr = (const uint8_t*)img->sdr.v.p[2];
  p.src_stride = img->sdr.v.stride[0];
  p.c_stride = img->sdr.v.stride[1];
  p.hs = sdr.v.fmt == F_YUV444 ? 1 : 2;
  p.vs = sdr.v.fmt == F_YUV420 ? 2 : 1;
  p.cw = (sdr.v.w + p.hs - 1) / p.hs;
  p.ch = (sdr.v.h + p.vs - 1) / p.vs;
  return ws.sync();   // resident on return; the codec's scratch (coefficients, decoded planes) is free again
}
}  // namespace

extern "C" {

UHDR_API int uhdr_b200_image_open_dev(const void* data, size_t size, int k, uhdr_b200_image_t** out) {
  if (!out) return fail(E_INVALID_PARAM, "received nullptr for the image handle");
  *out = nullptr;
  if (!data) return fail(E_INVALID_PARAM, "received nullptr for compressed img->data field");
  if (k != 1 && k != 2 && k != 4 && k != 8) return fail(E_INVALID_PARAM, "scale denominator %d, expects 1, 2, 4 or 8", k);
  DecodedInfo info;
  int rc = JpegRCodec().probe((const uint8_t*)data, size, &info);  // host only
  if (rc) return rc;
  JpegRCodec* c = nullptr;
  if ((rc = dev_codec(&c))) return rc;
  DevImage sdr, map;
  uhdr_gainmap_metadata_t md;
  if ((rc = c->decode_images((const uint8_t*)data, size, info, k, &sdr, &map, &md))) return rc;
  if (sdr.v.fmt != F_YUV420 && sdr.v.fmt != F_YUV422 && sdr.v.fmt != F_YUV444) {
    c->ws().sync();
    return fail(E_UNSUPPORTED, "a resident image needs a 4:2:0, 4:2:2 or 4:4:4 primary image, received format %d",
                sdr.v.fmt);
  }
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  uhdr_b200_image* img = new uhdr_b200_image();
  img->dev = dev;
  img->w = sdr.v.w;
  img->h = sdr.v.h;
  img->gm_w = map.v.w;
  img->gm_h = map.v.h;
  img->luts = c->ws().luts();
  img->md = md;
  rc = make_resident(*c, sdr, map, img);
  if (rc) {
    c->ws().sync();   // the copies may still read the codec's scratch or write the object's memory
    delete img;
    return rc;
  }
  *out = img;
  return E_OK;
}

UHDR_API int uhdr_b200_image_info(const uhdr_b200_image_t* img, unsigned* w, unsigned* h, unsigned* gm_w, unsigned* gm_h,
                                  uhdr_gainmap_metadata_t* md, size_t* device_bytes) {
  if (!img) return fail(E_INVALID_PARAM, "received nullptr for the image handle");
  if (w) *w = img->w;
  if (h) *h = img->h;
  if (gm_w) *gm_w = img->gm_w;
  if (gm_h) *gm_h = img->gm_h;
  if (md) *md = img->md;
  if (device_bytes) *device_bytes = img->dmem.reserved();
  return E_OK;
}

UHDR_API int uhdr_b200_image_render_dev(uhdr_b200_image_t* img, int out_ct, float max_display_boost, unsigned x,
                                        unsigned y, uhdr_raw_image_t* dest, void* stream) {
  // every check before anything is enqueued: a failing call writes nothing
  if (!img) return fail(E_INVALID_PARAM, "received nullptr for the image handle");
  if (!dest) return fail(E_INVALID_PARAM, "received nullptr for destination image");
  if (!std::isfinite(max_display_boost) || max_display_boost < 1.0f)
    return fail(E_INVALID_PARAM, "invalid display boost %f, expects to be >= 1.0f}", max_display_boost);
  const int fmt = dest->fmt;
  if ((fmt == UHDR_IMG_FMT_32bppRGBA1010102 && out_ct != UHDR_CT_HLG && out_ct != UHDR_CT_PQ) ||
      (fmt == UHDR_IMG_FMT_64bppRGBAHalfFloat && out_ct != UHDR_CT_LINEAR) ||
      (fmt == UHDR_IMG_FMT_32bppRGBA8888 && out_ct != UHDR_CT_SRGB) ||
      (fmt != UHDR_IMG_FMT_32bppRGBA1010102 && fmt != UHDR_IMG_FMT_64bppRGBAHalfFloat && fmt != UHDR_IMG_FMT_32bppRGBA8888))
    return fail(E_INVALID_PARAM, "unsupported output pixel format and output color transfer pair");
  if (dest->w == 0 || dest->h == 0 || (unsigned long long)x + dest->w > (unsigned long long)img->w ||
      (unsigned long long)y + dest->h > (unsigned long long)img->h)
    return fail(E_INVALID_PARAM, "region %ux%u at (%u, %u) is empty or outside the %dx%d image", dest->w, dest->h, x, y,
                img->w, img->h);
  int rc = check_dev_planes(*dest, "destination");
  if (rc) return rc;
  DeviceScope scope(img->dev);
  if ((rc = check_dev_memory(*dest, "destination"))) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  const int slot = img->next;
  if (img->used[slot] && cudaEventQuery(img->done[slot]) != cudaSuccess) {
    cudaGetLastError();   // cudaErrorNotReady: the render that used this slot is still in flight
    CUDA_TRY(cudaEventSynchronize(img->done[slot]));
  }
  const ApplyRegion region{(int)x, (int)y, (int)dest->w, (int)dest->h};
  int cg;
  if (out_ct == UHDR_CT_SRGB) {  // the base image alone, as decode_dev's colour conversion
    YccToRgbaParams p = img->rgba;
    p.w = region.w;
    p.h = region.h;
    p.ox = region.ox;
    p.oy = region.oy;
    p.dst = (uint8_t*)dest->planes[0];
    p.dst_stride = dest->stride[0];
    CUDA_TRY(launch_ycc_to_rgba(p, st));
    cg = img->sdr.cg;
  } else {
    DevImage dst;
    memset(&dst, 0, sizeof dst);
    dst.v.fmt = fmt;
    dst.v.w = region.w;
    dst.v.h = region.h;
    dst.v.p[0] = dest->planes[0];
    dst.v.stride[0] = dest->stride[0];
    dst.cg = dst.ct = dst.range = -1;
    rc = apply_gainmap_region(nullptr, st, img->luts, img->sdr, img->map, img->md, out_ct, max_display_boost, &dst,
                              &region, img->h_tab[slot], img->d_tab[slot]);
    if (rc) {
      // a table upload may have been enqueued before the failure: the slot waits for it
      if (cudaEventRecord(img->done[slot], st) == cudaSuccess) img->used[slot] = true;
      return rc;
    }
    cg = dst.cg;
  }
  // the slot (its staging table) and, for release, the object's planes are in use until here
  CUDA_TRY(cudaEventRecord(img->done[slot], st));
  img->used[slot] = true;
  img->next = (slot + 1) % uhdr_b200_image::kSlots;
  dest->cg = (uhdr_color_gamut_t)cg;
  dest->ct = out_ct == UHDR_CT_SRGB ? UHDR_CT_UNSPECIFIED : (uhdr_color_transfer_t)out_ct;
  dest->range = UHDR_CR_FULL_RANGE;
  return E_OK;
}

UHDR_API int uhdr_b200_image_release(uhdr_b200_image_t* img) {
  if (!img) return fail(E_INVALID_PARAM, "received nullptr for the image handle");
  DeviceScope scope(img->dev);
  delete img;   // waits for the outstanding renders, then parks the memory
  return E_OK;
}

}  // extern "C"
