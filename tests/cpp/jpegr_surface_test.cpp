// Source-compatibility and behaviour check of the ultrahdr::JpegR C++ surface.
//
// This ONE translation unit is compiled twice, unmodified:
//   (a) against the reference's own headers and objects (/root/reference/lib/include, oracle/_ref/obj_turbo):
//       tools/make_surface_golden.py does that in the build container, runs it on the CPU and stores the
//       digests it prints in tests/golden/jpegr_surface_ref.txt;
//   (b) against include/ and libuhdr_b200.so (tests/test_cpp_surface.py, on the GPU box).
// Both builds must print the same lines.  The calls follow the reference's own integration tests
// (tests/jpegr_test.cpp:1564-2329): the deprecated jr_* overloads of encode API-0..4 with the stride
// variants the reference exercises, decode to every output format, getJPEGRInfo, and the current
// uhdr_*_t overloads.
//
//   usage: jpegr_surface_test <raw_p010_image.p010> <raw_yuv420_image.yuv420>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <memory>
#include <vector>

#include "ultrahdr_api.h"
#include "ultrahdr/jpegr.h"
#include "ultrahdr/ultrahdrcommon.h"

using namespace ultrahdr;

static const int kW = 1280, kH = 720, kQuality = 90;

static uint64_t fnv(const void* p, size_t n) {
  const uint8_t* b = (const uint8_t*)p;
  uint64_t h = 1469598103934665603ull;
  for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 1099511628211ull;
  return h;
}
static std::vector<uint8_t> slurp(const char* path, size_t want) {
  std::vector<uint8_t> v(want);
  FILE* f = fopen(path, "rb");
  if (!f || fread(v.data(), 1, want, f) != want) { fprintf(stderr, "cannot read %s\n", path); exit(2); }
  fclose(f);
  return v;
}
#define CHECK(cond) do { if (!(cond)) { printf("FAILED %s:%d %s\n", __FILE__, __LINE__, #cond); return 1; } } while (0)

// P010 with explicit strides (jpegr_test.cpp's UhdrUnCompressedStructWrapper::setImageStride)
struct P010 {
  std::vector<uint16_t> luma, chroma;
  jpegr_uncompressed_struct d;
  P010(const std::vector<uint8_t>& tight, unsigned ls, unsigned cs, bool separate_chroma) {
    const uint16_t* src = (const uint16_t*)tight.data();
    const unsigned lstride = ls ? ls : kW, cstride = cs ? cs : lstride;
    if (!separate_chroma && !cs) {  // one buffer, chroma right behind luma with the luma stride
      luma.assign((size_t)lstride * kH * 3 / 2, 0);
      for (int y = 0; y < kH; y++) memcpy(&luma[(size_t)y * lstride], src + (size_t)y * kW, kW * 2);
      for (int y = 0; y < kH / 2; y++) memcpy(&luma[(size_t)lstride * kH + (size_t)y * lstride], src + (size_t)kW * kH + (size_t)y * kW, kW * 2);
      d.chroma_data = nullptr;
      d.chroma_stride = 0;
    } else {
      luma.assign((size_t)lstride * kH, 0);
      chroma.assign((size_t)cstride * kH / 2, 0);
      for (int y = 0; y < kH; y++) memcpy(&luma[(size_t)y * lstride], src + (size_t)y * kW, kW * 2);
      for (int y = 0; y < kH / 2; y++) memcpy(&chroma[(size_t)y * cstride], src + (size_t)kW * kH + (size_t)y * kW, kW * 2);
      d.chroma_data = chroma.data();
      d.chroma_stride = cstride;
    }
    d.data = luma.data();
    d.width = kW;
    d.height = kH;
    d.colorGamut = ULTRAHDR_COLORGAMUT_BT2100;
    d.luma_stride = ls;
    d.pixelFormat = UHDR_IMG_FMT_24bppYCbCrP010;
    d.colorRange = UHDR_CR_LIMITED_RANGE;
  }
};

static jpegr_compressed_struct out_buf(std::vector<uint8_t>& v) {
  v.assign((size_t)kW * kH * 3 * 2, 0);
  jpegr_compressed_struct c;
  c.data = v.data();
  c.length = 0;
  c.maxLength = v.size();
  c.colorGamut = ULTRAHDR_COLORGAMUT_UNSPECIFIED;
  return c;
}

int main(int argc, char** argv) {
  if (argc < 3) { fprintf(stderr, "usage: %s p010 yuv420\n", argv[0]); return 2; }
  const std::vector<uint8_t> p010 = slurp(argv[1], (size_t)kW * kH * 3), yuv = slurp(argv[2], (size_t)kW * kH * 3 / 2);

  JpegR jr;  // the reference's C++ defaults: scale 4, quality 85, single channel, REALTIME
  // ---- API-0, deprecated overload, stride variants must not change the file -----------------------
  std::vector<uint8_t> b0;
  jpegr_compressed_struct j0 = out_buf(b0);
  {
    P010 in(p010, 0, 0, false);
    CHECK(jr.encodeJPEGR(&in.d, ULTRAHDR_TF_HLG, &j0, kQuality, nullptr) == JPEGR_NO_ERROR);
    printf("api0 %zu %016llx\n", j0.length, (unsigned long long)fnv(j0.data, j0.length));
    const unsigned variants[4][2] = {{kW + 18, 0}, {kW + 18, kW + 28}, {0, kW + 34}, {kW, kW + 38}};
    for (int v = 0; v < 4; v++) {
      P010 in2(p010, variants[v][0], variants[v][1], variants[v][1] != 0 && v != 3);
      std::vector<uint8_t> b;
      jpegr_compressed_struct j = out_buf(b);
      CHECK(jr.encodeJPEGR(&in2.d, ULTRAHDR_TF_HLG, &j, kQuality, nullptr) == JPEGR_NO_ERROR);
      CHECK(j.length == j0.length && !memcmp(j.data, j0.data, j.length));
    }
    // argument checks of the deprecated path
    P010 bad(p010, 0, 0, false);
    bad.d.colorGamut = ULTRAHDR_COLORGAMUT_UNSPECIFIED;
    std::vector<uint8_t> b;
    jpegr_compressed_struct j = out_buf(b);
    CHECK(jr.encodeJPEGR(&bad.d, ULTRAHDR_TF_HLG, &j, kQuality, nullptr) == ERROR_JPEGR_INVALID_COLORGAMUT);
    CHECK(jr.encodeJPEGR(&in.d, ULTRAHDR_TF_SRGB, &j, kQuality, nullptr) == ERROR_JPEGR_INVALID_TRANS_FUNC);
    CHECK(jr.encodeJPEGR(&in.d, ULTRAHDR_TF_HLG, &j, 101, nullptr) == ERROR_JPEGR_INVALID_QUALITY_FACTOR);
    CHECK(jr.encodeJPEGR(&in.d, ULTRAHDR_TF_HLG, nullptr, kQuality, nullptr) == ERROR_JPEGR_BAD_PTR);
  }
  // ---- API-1 ----------------------------------------------------------------------------------------
  std::vector<uint8_t> yuvbuf = yuv;
  jpegr_uncompressed_struct sdr;
  sdr.data = yuvbuf.data();
  sdr.width = kW;
  sdr.height = kH;
  sdr.colorGamut = ULTRAHDR_COLORGAMUT_BT709;
  sdr.pixelFormat = UHDR_IMG_FMT_12bppYCbCr420;
  sdr.colorRange = UHDR_CR_FULL_RANGE;
  std::vector<uint8_t> b1;
  jpegr_compressed_struct j1 = out_buf(b1);
  P010 hdr(p010, 0, 0, false);
  CHECK(jr.encodeJPEGR(&hdr.d, &sdr, ULTRAHDR_TF_HLG, &j1, kQuality, nullptr) == JPEGR_NO_ERROR);
  printf("api1 %zu %016llx\n", j1.length, (unsigned long long)fnv(j1.data, j1.length));
  {
    jpegr_uncompressed_struct small = sdr;
    small.width = kW - 2;
    std::vector<uint8_t> b;
    jpegr_compressed_struct j = out_buf(b);
    CHECK(jr.encodeJPEGR(&hdr.d, &small, ULTRAHDR_TF_HLG, &j, kQuality, nullptr) == ERROR_JPEGR_RESOLUTION_MISMATCH);
  }
  // ---- a compressed sdr intent through JpegEncoderHelper, then API-2 and API-3 -------------------------
  JpegEncoderHelper enc;
  {
    const uint8_t* planes[3] = {yuvbuf.data(), yuvbuf.data() + (size_t)kW * kH, yuvbuf.data() + (size_t)kW * kH * 5 / 4};
    const unsigned strides[3] = {(unsigned)kW, (unsigned)kW / 2, (unsigned)kW / 2};
    uhdr_error_info_t st = enc.compressImage(planes, strides, kW, kH, UHDR_IMG_FMT_12bppYCbCr420, kQuality, nullptr, 0);
    CHECK(st.error_code == UHDR_CODEC_OK);
    printf("sdrjpg %zu %016llx\n", enc.getCompressedImageSize(), (unsigned long long)fnv(enc.getCompressedImagePtr(), enc.getCompressedImageSize()));
  }
  // widths that are not a multiple of 8: the helper's edge padding for tight strides (0 / 128 columns, rows below the
  // image repeated from the previous iMCU row) and for wide ones (the caller's bytes up to the aligned width)
  for (int wide = 0; wide < 2; wide++) {
    const int w = 246, h = 26;
    std::vector<uint8_t> tight((size_t)w * h + 2 * (size_t)(w / 2) * (h / 2));
    for (int y = 0; y < h; y++) memcpy(tight.data() + (size_t)y * w, yuvbuf.data() + (size_t)y * kW, w);
    for (int c = 0; c < 2; c++)
      for (int y = 0; y < h / 2; y++)
        memcpy(tight.data() + (size_t)w * h + (size_t)c * (w / 2) * (h / 2) + (size_t)y * (w / 2),
               yuvbuf.data() + (size_t)kW * kH + (size_t)c * (kW / 2) * (kH / 2) + (size_t)y * (kW / 2), w / 2);
    const uint8_t* planes[3] = {tight.data(), tight.data() + (size_t)w * h, tight.data() + (size_t)w * h + (size_t)(w / 2) * (h / 2)};
    const unsigned strides[3] = {(unsigned)w, (unsigned)w / 2, (unsigned)w / 2};
    const uint8_t* wplanes[3] = {yuvbuf.data(), yuvbuf.data() + (size_t)kW * kH, yuvbuf.data() + (size_t)kW * kH * 5 / 4};
    const unsigned wstrides[3] = {(unsigned)kW, (unsigned)kW / 2, (unsigned)kW / 2};
    for (int fmt = 0; fmt < 2; fmt++) {
      JpegEncoderHelper e;
      uhdr_error_info_t st = e.compressImage(wide ? wplanes : planes, wide ? wstrides : strides, w - (fmt ? 1 : 0), h - (fmt ? 5 : 0),
                                             fmt ? UHDR_IMG_FMT_8bppYCbCr400 : UHDR_IMG_FMT_12bppYCbCr420, kQuality, nullptr, 0);
      CHECK(st.error_code == UHDR_CODEC_OK);
      printf("ragged %s %s %zu %016llx\n", wide ? "wide" : "tight", fmt ? "y400" : "420", e.getCompressedImageSize(),
             (unsigned long long)fnv(e.getCompressedImagePtr(), e.getCompressedImageSize()));
    }
  }
  jpegr_compressed_struct sdrjpg;
  sdrjpg.data = enc.getCompressedImagePtr();
  sdrjpg.length = sdrjpg.maxLength = enc.getCompressedImageSize();
  sdrjpg.colorGamut = ULTRAHDR_COLORGAMUT_BT709;
  std::vector<uint8_t> b2, b3;
  jpegr_compressed_struct j2 = out_buf(b2), j3 = out_buf(b3);
  CHECK(jr.encodeJPEGR(&hdr.d, &sdr, &sdrjpg, ULTRAHDR_TF_HLG, &j2) == JPEGR_NO_ERROR);
  printf("api2 %zu %016llx\n", j2.length, (unsigned long long)fnv(j2.data, j2.length));
  CHECK(jr.encodeJPEGR(&hdr.d, &sdrjpg, ULTRAHDR_TF_HLG, &j3) == JPEGR_NO_ERROR);
  printf("api3 %zu %016llx\n", j3.length, (unsigned long long)fnv(j3.data, j3.length));
  // ---- getJPEGRInfo + decode (deprecated overload) to every output format ---------------------------
  jpeg_info_struct pinfo, ginfo;
  jpegr_info_struct info;
  info.primaryImgInfo = &pinfo;
  info.gainmapImgInfo = &ginfo;
  CHECK(jr.getJPEGRInfo(&j1, &info) == JPEGR_NO_ERROR);
  printf("info %u %u gm %u %u comps %u icc %zu iso %zu\n", info.width, info.height, ginfo.width, ginfo.height, ginfo.numComponents,
         pinfo.iccData.size(), ginfo.isoData.size());
  ultrahdr_metadata_struct md;
  const ultrahdr_output_format fmts[4] = {ULTRAHDR_OUTPUT_SDR, ULTRAHDR_OUTPUT_HDR_LINEAR, ULTRAHDR_OUTPUT_HDR_PQ, ULTRAHDR_OUTPUT_HDR_HLG};
  for (int f = 0; f < 4; f++) {
    std::vector<uint8_t> px((size_t)kW * kH * 8, 0);
    jpegr_uncompressed_struct dst;
    dst.data = px.data();
    dst.width = dst.height = 0;
    dst.colorGamut = ULTRAHDR_COLORGAMUT_UNSPECIFIED;
    // (the reference parses the gain-map image only when HDR output or the gain-map image is asked for:
    //  metadata with plain SDR output is an error there, and here)
    if (fmts[f] == ULTRAHDR_OUTPUT_SDR) CHECK(jr.decodeJPEGR(&j1, &dst, 4.0f, nullptr, fmts[f], nullptr, &md) == JPEGR_UNKNOWN_ERROR);
    CHECK(jr.decodeJPEGR(&j1, &dst, 4.0f, nullptr, fmts[f], nullptr, fmts[f] == ULTRAHDR_OUTPUT_SDR ? nullptr : &md) == JPEGR_NO_ERROR);
    const size_t bpp = fmts[f] == ULTRAHDR_OUTPUT_HDR_LINEAR ? 8 : 4;
    printf("decode fmt %d -> %ux%u pix %d gamut %d %016llx\n", (int)fmts[f], dst.width, dst.height, (int)dst.pixelFormat,
           (int)dst.colorGamut, (unsigned long long)fnv(px.data(), (size_t)kW * kH * bpp));
  }
  printf("metadata %s max %.9g min %.9g gamma %.9g offs %.9g %.9g cap %.9g %.9g\n", md.version.c_str(), md.maxContentBoost,
         md.minContentBoost, md.gamma, md.offsetSdr, md.offsetHdr, md.hdrCapacityMin, md.hdrCapacityMax);
  {
    std::vector<uint8_t> px((size_t)kW * kH * 8, 0);
    jpegr_uncompressed_struct dst;
    dst.data = px.data();
    CHECK(jr.decodeJPEGR(&j1, &dst, 0.5f) == ERROR_JPEGR_INVALID_DISPLAY_BOOST);
  }
  // ---- API-4 from the pieces of the API-1 file ----------------------------------------------------------
  {
    jpegr_compressed_struct base, gm;
    base.data = pinfo.imgData.data();
    base.length = base.maxLength = pinfo.imgData.size();
    base.colorGamut = ULTRAHDR_COLORGAMUT_BT709;
    gm.data = ginfo.imgData.data();
    gm.length = gm.maxLength = ginfo.imgData.size();
    gm.colorGamut = ULTRAHDR_COLORGAMUT_UNSPECIFIED;
    std::vector<uint8_t> b4;
    jpegr_compressed_struct j4 = out_buf(b4);
    CHECK(jr.encodeJPEGR(&base, &gm, &md, &j4) == JPEGR_NO_ERROR);
    printf("api4 %zu %016llx\n", j4.length, (unsigned long long)fnv(j4.data, j4.length));
  }
  // ---- current overloads: library defaults (scale 1, q95, multichannel, BEST_QUALITY) ------------------
  {
    JpegR lib(nullptr, kMapDimensionScaleFactorDefault, kMapCompressQualityDefault, kUseMultiChannelGainMapDefault,
              kGainMapGammaDefault, kEncSpeedPresetDefault);
    uhdr_raw_image_t h{}, s{};
    h.fmt = UHDR_IMG_FMT_24bppYCbCrP010; h.cg = UHDR_CG_BT_2100; h.ct = UHDR_CT_PQ; h.range = UHDR_CR_LIMITED_RANGE;
    h.w = kW; h.h = kH;
    std::vector<uint8_t> hb = p010;
    h.planes[UHDR_PLANE_Y] = hb.data(); h.stride[UHDR_PLANE_Y] = kW;
    h.planes[UHDR_PLANE_UV] = hb.data() + (size_t)kW * kH * 2; h.stride[UHDR_PLANE_UV] = kW;
    s.fmt = UHDR_IMG_FMT_12bppYCbCr420; s.cg = UHDR_CG_DISPLAY_P3; s.ct = UHDR_CT_SRGB; s.range = UHDR_CR_FULL_RANGE;
    s.w = kW; s.h = kH;
    s.planes[UHDR_PLANE_Y] = yuvbuf.data(); s.stride[UHDR_PLANE_Y] = kW;
    s.planes[UHDR_PLANE_U] = yuvbuf.data() + (size_t)kW * kH; s.stride[UHDR_PLANE_U] = kW / 2;
    s.planes[UHDR_PLANE_V] = yuvbuf.data() + (size_t)kW * kH * 5 / 4; s.stride[UHDR_PLANE_V] = kW / 2;
    uhdr_compressed_image_ext_t out(UHDR_CG_UNSPECIFIED, UHDR_CT_UNSPECIFIED, UHDR_CR_UNSPECIFIED, (size_t)kW * kH * 6);
    uhdr_error_info_t st = lib.encodeJPEGR(&h, &s, &out, 95, nullptr);
    CHECK(st.error_code == UHDR_CODEC_OK);
    printf("new api1 %zu %016llx\n", out.data_sz, (unsigned long long)fnv(out.data, out.data_sz));
    // stage members
    uhdr_gainmap_metadata_ext_t gmd(kJpegrVersion);
    std::unique_ptr<uhdr_raw_image_ext_t> gmap;
    st = lib.generateGainMap(&s, &h, &gmd, gmap);
    CHECK(st.error_code == UHDR_CODEC_OK && gmap);
    uint64_t hh = 1469598103934665603ull;
    for (unsigned y = 0; y < gmap->h; y++) hh ^= fnv((uint8_t*)gmap->planes[0] + (size_t)y * gmap->stride[0] * 3, (size_t)gmap->w * 3) * (y + 1);
    printf("generateGainMap %ux%u fmt %d stride %u %016llx max %.9g\n", gmap->w, gmap->h, (int)gmap->fmt, gmap->stride[0],
           (unsigned long long)hh, gmd.max_content_boost[0]);
    uhdr_raw_image_ext_t dst(UHDR_IMG_FMT_64bppRGBAHalfFloat, UHDR_CG_UNSPECIFIED, UHDR_CT_LINEAR, UHDR_CR_FULL_RANGE, kW, kH, 1);
    st = lib.applyGainMap(&s, gmap.get(), &gmd, UHDR_CT_LINEAR, UHDR_IMG_FMT_64bppRGBAHalfFloat, FLT_MAX, &dst);
    CHECK(st.error_code == UHDR_CODEC_OK);
    printf("applyGainMap gamut %d %016llx\n", (int)dst.cg, (unsigned long long)fnv(dst.planes[0], (size_t)kW * kH * 8));
    // metadata that uhdr_validate_gainmap_metadata_descriptor refuses: one case per rule, and non-finite fields
    for (int k = 0; k < 9; k++) {
      uhdr_gainmap_metadata_ext_t bad = gmd;
      switch (k) {
        case 0: bad.max_content_boost[1] = bad.min_content_boost[1] * 0.5f; break;
        case 1: bad.min_content_boost[0] = 0.0f; break;
        case 2: bad.gamma[2] = 0.0f; break;
        case 3: bad.offset_sdr[1] = -1e-3f; break;
        case 4: bad.offset_hdr[0] = -1e-7f; break;
        case 5: bad.hdr_capacity_max = bad.hdr_capacity_min; break;
        case 6: bad.hdr_capacity_min = 0.5f; break;
        case 7: bad.max_content_boost[0] = std::numeric_limits<float>::quiet_NaN(); break;
        default: bad.gamma[0] = std::numeric_limits<float>::infinity(); break;
      }
      st = lib.applyGainMap(&s, gmap.get(), &bad, UHDR_CT_LINEAR, UHDR_IMG_FMT_64bppRGBAHalfFloat, FLT_MAX, &dst);
      printf("applyGainMap invalid metadata %d: error %d\n", k, (int)st.error_code);
    }
    uhdr_raw_image_ext_t tm(UHDR_IMG_FMT_12bppYCbCr420, UHDR_CG_UNSPECIFIED, UHDR_CT_UNSPECIFIED, UHDR_CR_UNSPECIFIED, kW, kH, 1);
    st = lib.toneMap(&h, &tm);
    CHECK(st.error_code == UHDR_CODEC_OK);
    printf("toneMap gamut %d %016llx\n", (int)tm.cg, (unsigned long long)fnv(tm.planes[0], (size_t)kW * kH * 3 / 2));
    // decode through the current overload with a gain-map image and metadata
    uhdr_compressed_image_t in = out;
    uhdr_raw_image_ext_t px(UHDR_IMG_FMT_32bppRGBA1010102, UHDR_CG_UNSPECIFIED, UHDR_CT_HLG, UHDR_CR_FULL_RANGE, kW, kH, 1);
    uhdr_raw_image_ext_t gpx(UHDR_IMG_FMT_32bppRGBA8888, UHDR_CG_UNSPECIFIED, UHDR_CT_UNSPECIFIED, UHDR_CR_FULL_RANGE, kW, kH, 1);
    uhdr_gainmap_metadata_t gmd2;
    st = lib.decodeJPEGR(&in, &px, FLT_MAX, UHDR_CT_HLG, UHDR_IMG_FMT_32bppRGBA1010102, &gpx, &gmd2);
    CHECK(st.error_code == UHDR_CODEC_OK);
    printf("new decode hlg %016llx map %016llx max %.9g %.9g %.9g\n", (unsigned long long)fnv(px.planes[0], (size_t)kW * kH * 4),
           (unsigned long long)fnv(gpx.planes[0], (size_t)kW * kH * 4), gmd2.max_content_boost[0], gmd2.max_content_boost[1],
           gmd2.max_content_boost[2]);
  }
  printf("surface test done\n");
  return 0;
}
