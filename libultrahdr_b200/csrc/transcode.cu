// JPEG/R -> JPEG/R transcoding (uhdr_b200_transcode): both JPEGs decoded at 1/k on the device, re-encoded by the block
// stage and the device entropy coder, assembled by the container layer.  No pixel crosses PCIe.
#include <cstring>

#include "codec.h"

namespace uhdr_b200 {

namespace {

// libjpeg's compression input stage for a 4:2:0 frame from full-size YCbCr scanlines (jcprepct.c, jcsample.c), written
// as the block stage reads a 4:2:0 image: luma lw x lh samples, chroma cw x ch, every row the block stage loads.
//  * luma: row / column past the image = the last one (expand_right_edge, expand_bottom_edge)
//  * chroma: h2v2_downsample of the edge-expanded rows, (a + b + c + d + bias) >> 2 with bias 1, 2, 1, 2, ... along an
//    output row; an odd last input row pairs with itself; rows past ceil(h / 2) repeat the last downsampled row
// One thread per chroma sample, which also writes the 2x2 luma samples above it.
struct Ycc420Params {
  const uint8_t *y, *cb, *cr;
  int src_stride, w, h;
  uint8_t *dy, *dcb, *dcr;
  int dy_stride, dc_stride, lw, lh, cw, ch;
};

__global__ void k_ycc444_to_420(const Ycc420Params p) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= p.cw || i >= p.ch) return;
#pragma unroll
  for (int dy = 0; dy < 2; dy++) {
    const int yy = 2 * i + dy;
    if (yy >= p.lh) break;
    const size_t srow = (size_t)min(yy, p.h - 1) * p.src_stride;
#pragma unroll
    for (int dx = 0; dx < 2; dx++) {
      const int xx = 2 * j + dx;
      if (xx < p.lw) p.dy[(size_t)yy * p.dy_stride + xx] = __ldg(p.y + srow + min(xx, p.w - 1));
    }
  }
  const int ii = min(i, (p.h + 1) / 2 - 1);
  const size_t r0 = (size_t)(2 * ii) * p.src_stride, r1 = (size_t)min(2 * ii + 1, p.h - 1) * p.src_stride;
  const int c0 = min(2 * j, p.w - 1), c1 = min(2 * j + 1, p.w - 1), bias = 1 + (j & 1);
  const size_t o = (size_t)i * p.dc_stride + j;
  p.dcb[o] = (uint8_t)((__ldg(p.cb + r0 + c0) + __ldg(p.cb + r0 + c1) + __ldg(p.cb + r1 + c0) + __ldg(p.cb + r1 + c1) + bias) >> 2);
  p.dcr[o] = (uint8_t)((__ldg(p.cr + r0 + c0) + __ldg(p.cr + r0 + c1) + __ldg(p.cr + r1 + c0) + __ldg(p.cr + r1 + c1) + bias) >> 2);
}

cudaError_t launch_ycc444_to_420(const Ycc420Params& p, cudaStream_t s) {
  count_launches(1);
  const dim3 block(32, 8), grid((p.cw + 31) / 32, (p.ch + 7) / 8);
  k_ycc444_to_420<<<grid, block, 0, s>>>(p);
  return cudaGetLastError();
}

// `src` (YUV444, one stride for all planes) as the 4:2:0 block-stage input libjpeg makes of it; rows[c]: the rows of
// plane c the block stage reads from memory
int ycc444_to_420_dev(Workspace& ws, const DevImage& src, DevImage* out, int rows[3]) {
  int rc = alloc_dev_image(ws, F_YUV420, src.v.w, src.v.h, 64, out);
  if (rc) return rc;
  JpegFrame f;
  if ((rc = jpeg_frame_init(&f, F_YUV420, src.v.w, src.v.h, 75))) return rc;
  Ycc420Params p;
  p.y = (const uint8_t*)src.v.p[0];
  p.cb = (const uint8_t*)src.v.p[1];
  p.cr = (const uint8_t*)src.v.p[2];
  p.src_stride = src.v.stride[0];
  p.w = src.v.w;
  p.h = src.v.h;
  p.dy = (uint8_t*)out->v.p[0];
  p.dcb = (uint8_t*)out->v.p[1];
  p.dcr = (uint8_t*)out->v.p[2];
  p.dy_stride = out->v.stride[0];
  p.dc_stride = out->v.stride[1];
  p.lw = f.comp[0].wblocks * 8;
  p.lh = f.comp[0].hblocks * 8;
  p.cw = f.comp[1].wblocks * 8;
  p.ch = f.comp[1].hblocks * 8;
  rows[0] = p.lh;
  rows[1] = rows[2] = p.ch;
  TIMED(ws, "ycc444_to_420", launch_ycc444_to_420(p, ws.stream()));
  return E_OK;
}

// a decoded image (decoder scratch, its own strides) as JpegEncoderHelper takes it with strides equal to the plane
// widths: a 64-pixel-stride workspace copy with the helper's padding
int stage_tight(Workspace& ws, const DevImage& src, DevImage* out, int rows[3]) {
  rows[0] = rows[1] = rows[2] = 0;
  uhdr_raw_image_t v;
  memset(&v, 0, sizeof v);
  v.fmt = (uhdr_img_fmt_t)src.v.fmt;
  v.w = src.v.w;
  v.h = src.v.h;
  v.cg = UHDR_CG_UNSPECIFIED;
  v.ct = UHDR_CT_UNSPECIFIED;
  v.range = UHDR_CR_FULL_RANGE;
  for (int i = 0; i < fmt_planes(src.v.fmt); i++) {
    v.planes[i] = const_cast<void*>(src.v.p[i]);
    v.stride[i] = src.v.stride[i];
  }
  int rc = upload_image(ws, v, out, cudaMemcpyDeviceToDevice);
  if (rc) return rc;
  for (int i = 0; i < fmt_planes(src.v.fmt); i++) {
    int pw, ph, esz;
    fmt_plane_geom(src.v.fmt, src.v.w, src.v.h, i, &pw, &ph, &esz);
    v.stride[i] = pw;
  }
  return helper_padding(ws, v, cudaMemcpyDeviceToDevice, *out, rows);
}

}  // namespace

int JpegRCodec::transcode(const uint8_t* data, size_t size, const DecodedInfo& probed, const uhdr_b200_transcode_config_t& cfg,
                          uint8_t* out, size_t cap, size_t* out_size) {
  (void)size;
  int rc = settle();
  if (rc) return rc;
  PhaseTrace tr;
  ws_.rewind();
  map_pending_ = false;
  DevImage sdr, map;
  JpegHeader ph, gh;
  // DECODE_TO_YCBCR_CS for both: raw planes, a 3-channel map as YCbCr
  rc = decode_pair(data, probed.base_off, probed.base_len, probed.gainmap_off, probed.gainmap_len, 0, nullptr, true, cfg.k,
                   &sdr, &map, &ph, &gh, tr, /*map_mode=*/0);
  DevImage base_in, map_in;
  int base_rows[3], map_rows[3];
  JpegEncodeJob base_jpeg, gm_jpeg;
  if (!rc) {
    if (cfg.base_420 && sdr.v.fmt == F_YUV422)
      rc = fail(E_UNSUPPORTED, "a 4:2:0 base image is written from 4:4:4 or 4:2:0 input, the base image is 4:2:2");
    else if (cfg.base_420 && sdr.v.fmt == F_YUV444)
      rc = ycc444_to_420_dev(ws_, sdr, &base_in, base_rows);
    else
      rc = stage_tight(ws_, sdr, &base_in, base_rows);
  }
  if (!rc) rc = stage_tight(ws_, map, &map_in, map_rows);
  if (!rc) rc = jpeg_forward_dev(ws_, base_in, cfg.base_quality, &base_jpeg, /*zigzag=*/true, base_rows);
  if (!rc) rc = jpeg_entropy_dev(ws_, &base_jpeg);
  if (!rc) rc = jpeg_forward_dev(ws_, map_in, cfg.gainmap_quality, &gm_jpeg, /*zigzag=*/true, map_rows);
  if (!rc) rc = jpeg_entropy_dev(ws_, &gm_jpeg);
  if (!rc) tr.mark("encodes enqueued");
  if (!rc) rc = ws_.sync();   // the two scan sizes
  if (!rc) rc = jpeg_entropy_fetch(ws_, &base_jpeg);
  if (!rc) rc = jpeg_entropy_fetch(ws_, &gm_jpeg);
  if (!rc) rc = ws_.sync();
  if (rc) {
    mark_in_flight();   // as decode(): kernels of both JPEGs may still run
    return rc;
  }
  tr.mark("scans on the host");
  const uint8_t* pd = data + probed.base_off;
  const uint8_t* gd = data + probed.gainmap_off;
  const ByteView base_icc = find_marker(pd, ph, 0xE2, "ICC_PROFILE", 12), gm_icc = find_marker(gd, gh, 0xE2, "ICC_PROFILE", 12);
  const uhdr_gainmap_metadata_t& md = probed.metadata;
  // API-4's checks (encode_from_compressed) on the new pair
  if (!md.use_base_cg && gm_icc.empty())
    return fail(E_UNSUPPORTED, "For gainmap application space to be alternate image space, gainmap image is expected to "
                "contain alternate image color space in the form of ICC. The ICC marker in gainmap jpeg is missing.");
  const uint8_t* add_icc = nullptr;
  size_t add_icc_n = 0;
  if (base_icc.empty()) {
    if (sdr.cg <= UHDR_CG_UNSPECIFIED || sdr.cg > UHDR_CG_BT_2100) return fail(E_INVALID_PARAM, "Unrecognized 420 color gamut %d", sdr.cg);
    add_icc = icc_profile(UHDR_CT_SRGB, sdr.cg, &add_icc_n);
  }
  const char* base_com = base_in.v.fmt == F_Y400 ? jpeg_gainmap_comment() : nullptr;
  const char* gm_com = map_in.v.fmt == F_Y400 ? jpeg_gainmap_comment() : nullptr;
  JpegPieces pb, pg;
  const size_t base_cap = jpeg_head_capacity(base_icc.size, base_com), gm_cap = jpeg_head_capacity(gm_icc.size, gm_com);
  uint8_t* base_head = (uint8_t*)ws_.halloc(base_cap);
  uint8_t* gm_head = (uint8_t*)ws_.halloc(gm_cap);
  if (!base_head || !gm_head) return E_MEM;
  rc = jpeg_stream_pieces(base_jpeg, base_icc.data, base_icc.size, base_com, base_head, base_cap, &pb.head_len, &pb.scan, &pb.scan_len);
  if (rc) return rc;
  rc = jpeg_stream_pieces(gm_jpeg, gm_icc.data, gm_icc.size, gm_com, gm_head, gm_cap, &pg.head_len, &pg.scan, &pg.scan_len);
  if (rc) return rc;
  pb.head = base_head;
  pg.head = gm_head;
  // keep_exif: the reference moves an EXIF segment of the base image into the container right after JFIF
  // (jpegr.cpp:1173-1217), which is where appendGainMap writes an EXIF block handed to it
  const ByteView exif = cfg.keep_exif ? probed.exif : ByteView();
  // assembled into the workspace first: on failure `out` stays untouched, and a short `cap` learns the size needed
  const size_t bound = pb.total() + pg.total() + exif.size + add_icc_n + 1024;
  uint8_t* file = (uint8_t*)ws_.halloc(bound);
  if (!file) return E_MEM;
  size_t n = 0;
  rc = assemble_jpegr(pb, pg, exif.data, exif.size, md, file, bound, &n, add_icc, add_icc_n);
  if (rc) return rc;
  *out_size = n;
  if (n > cap) return fail(E_MEM, "output buffer of %zu bytes is too small for the encoded stream of %zu bytes", cap, n);
  memcpy(out, file, n);
  tr.mark("file assembled");
  return E_OK;
}

}  // namespace uhdr_b200
