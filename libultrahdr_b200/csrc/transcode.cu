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

// chroma sample (j, i), j < cw, i < ch: that sample of both chroma planes and the 2x2 luma samples above it
__device__ __forceinline__ void ycc444_to_420_at(const Ycc420Params& p, const int j, const int i) {
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

__global__ void k_ycc444_to_420(const Ycc420Params p) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y * blockDim.y + threadIdx.y;
  if (j >= p.cw || i >= p.ch) return;
  ycc444_to_420_at(p, j, i);
}

// One image plane (or, with `ycc420`, one 4:2:0 input image) of k_stage_batch: the bytes the block stage reads.
//  * plane: stage_tight + helper_padding of a decoded plane pw x ph (src, src_stride) into dst (dst_stride): columns
//    [pw, aw) hold `fill` (0 luma, 128 chroma), and when pw < aw the rows [ph, rows) are the helper's scratch rows --
//    the row one iMCU (imcu rows) above, or inside the first iMCU 0 up to pw and `fill` after it.  width = aw.
//  * ycc420: libjpeg's 4:2:0 input stage of a 4:4:4 image, k_ycc444_to_420's bytes; width = cw, one thread per chroma
//    sample.
struct StageJob {
  Ycc420Params p;
  const uint8_t* src;
  uint8_t* dst;
  int src_stride, dst_stride, pw, ph, aw, rows, fill, imcu;
  int ycc420, width;
};

// every plane of a group in one launch: 256 work items (bytes; chroma samples of a ycc420 job) per CTA, the job found
// by a binary search over the jobs' cumulative CTA counts
__global__ void __launch_bounds__(256) k_stage_batch(const StageJob* __restrict__ jobs, const unsigned* __restrict__ cta_end,
                                                     unsigned njobs) {
  const unsigned ji = batch_find(cta_end, njobs, blockIdx.x);
  const StageJob& J = jobs[ji];
  const unsigned idx = (blockIdx.x - (ji ? cta_end[ji - 1] : 0u)) * 256u + threadIdx.x;
  const int y = (int)(idx / (unsigned)J.width), x = (int)(idx - (unsigned)y * J.width);
  if (J.ycc420) {
    if (y < J.p.ch) ycc444_to_420_at(J.p, x, y);
    return;
  }
  if (y >= J.rows) return;
  int sy = y;
  while (sy >= J.ph && sy >= J.imcu) sy -= J.imcu;   // helper_padding copies the row one iMCU up
  uint8_t v = (uint8_t)J.fill;
  if (x < J.pw) v = sy < J.ph ? __ldg(J.src + (size_t)sy * J.src_stride + x) : (uint8_t)0;
  J.dst[(size_t)y * J.dst_stride + x] = v;
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
      rc = fail_base_422();
    else if (cfg.base_420 && sdr.v.fmt == F_YUV444)
      rc = ycc444_to_420_dev(ws_, sdr, &base_in, base_rows);
    else
      rc = stage_tight(ws_, sdr, &base_in, base_rows);
  }
  if (!rc) rc = stage_tight(ws_, map, &map_in, map_rows);
  if (!rc) rc = jpeg_encode_dev(ws_, base_in, cfg.base_quality, &base_jpeg, base_rows);
  if (!rc) rc = jpeg_encode_dev(ws_, map_in, cfg.gainmap_quality, &gm_jpeg, map_rows);
  if (!rc) tr.mark("encodes enqueued");
  JpegEncodeJob* jobs[] = {&base_jpeg, &gm_jpeg};   // the base's overflow is the one reported
  if (!rc) rc = jpeg_entropy_collect(ws_, jobs, 2);
  if (rc) {
    mark_in_flight();   // as decode(): kernels of both JPEGs may still run
    return rc;
  }
  tr.mark("scans on the host");
  rc = transcode_finish(data, probed, ph, gh, base_jpeg, gm_jpeg, cfg, out, cap, out_size);
  if (!rc) tr.mark("file assembled");
  return rc;
}

int JpegRCodec::fail_base_422() {
  return fail(E_UNSUPPORTED, "a 4:2:0 base image is written from 4:4:4 or 4:2:0 input, the base image is 4:2:2");
}

int JpegRCodec::transcode_finish(const uint8_t* data, const DecodedInfo& probed, const JpegHeader& ph, const JpegHeader& gh,
                                 const JpegEncodeJob& base_jpeg, const JpegEncodeJob& gm_jpeg,
                                 const uhdr_b200_transcode_config_t& cfg, uint8_t* out, size_t cap, size_t* out_size) {
  const uint8_t* pd = data + probed.base_off;
  const uint8_t* gd = data + probed.gainmap_off;
  const ByteView base_icc = find_marker(pd, ph, 0xE2, "ICC_PROFILE", 12), gm_icc = find_marker(gd, gh, 0xE2, "ICC_PROFILE", 12);
  const uhdr_gainmap_metadata_t& md = probed.metadata;
  // API-4's rules on the new pair; the decode gives a primary image without ICC no gamut
  const uint8_t* add_icc;
  size_t add_icc_n;
  int rc = api4_icc(base_icc, !gm_icc.empty(), UHDR_CG_UNSPECIFIED, md, &add_icc, &add_icc_n);
  if (rc) return rc;
  JpegPieces pb, pg;
  if ((rc = jpeg_stream_pieces(ws_, base_jpeg, base_icc.data, base_icc.size, &pb)) ||
      (rc = jpeg_stream_pieces(ws_, gm_jpeg, gm_icc.data, gm_icc.size, &pg)))
    return rc;
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
  return E_OK;
}

namespace {

// a workspace plane of aw x rows bytes for the block stage
int stage_plane(Workspace& ws, int aw, int rows, uint8_t** out) {
  *out = (uint8_t*)ws.dalloc((size_t)aw * rows);
  return *out ? E_OK : E_MEM;
}

// stage_tight's (and helper_padding's) bytes of `src` as k_stage_batch jobs into a new image *out; rows[c] as there
int plan_stage_tight(Workspace& ws, const DevImage& src, StageJob* jobs, int* nj, DevImage* out, int rows[3]) {
  memset(out, 0, sizeof *out);
  out->v = src.v;
  for (int i = 0; i < fmt_planes(src.v.fmt); i++) {
    int pw, ph, esz;
    fmt_plane_geom(src.v.fmt, src.v.w, src.v.h, i, &pw, &ph, &esz);
    const int aw = (pw + 7) / 8 * 8;
    StageJob& J = jobs[(*nj)++];
    memset(&J, 0, sizeof J);
    J.src = (const uint8_t*)src.v.p[i];
    J.src_stride = src.v.stride[i];
    J.pw = pw;
    J.ph = ph;
    J.aw = J.width = aw;
    J.rows = rows[i] = pw == aw ? ph : (ph + 7) / 8 * 8;
    J.fill = i == 0 ? 0 : 128;
    J.imcu = (src.v.fmt == F_YUV420 && i == 0) ? 16 : 8;
    J.dst_stride = aw;
    int rc = stage_plane(ws, aw, J.rows, &J.dst);
    if (rc) return rc;
    out->v.p[i] = J.dst;
    out->v.stride[i] = aw;
  }
  return E_OK;
}

// ycc444_to_420_dev's bytes as one k_stage_batch job
int plan_ycc444_to_420(Workspace& ws, const DevImage& src, StageJob* jobs, int* nj, DevImage* out, int rows[3]) {
  JpegFrame f;
  int rc = jpeg_frame_init(&f, F_YUV420, src.v.w, src.v.h, 75);
  if (rc) return rc;
  StageJob& J = jobs[(*nj)++];
  memset(&J, 0, sizeof J);
  Ycc420Params& p = J.p;
  p.y = (const uint8_t*)src.v.p[0];
  p.cb = (const uint8_t*)src.v.p[1];
  p.cr = (const uint8_t*)src.v.p[2];
  p.src_stride = src.v.stride[0];
  p.w = src.v.w;
  p.h = src.v.h;
  p.lw = f.comp[0].wblocks * 8;
  p.lh = f.comp[0].hblocks * 8;
  p.cw = f.comp[1].wblocks * 8;
  p.ch = f.comp[1].hblocks * 8;
  p.dy_stride = p.lw;
  p.dc_stride = p.cw;
  uint8_t* planes[3];
  if ((rc = stage_plane(ws, p.lw, p.lh, &planes[0])) || (rc = stage_plane(ws, p.cw, p.ch, &planes[1])) ||
      (rc = stage_plane(ws, p.cw, p.ch, &planes[2])))
    return rc;
  p.dy = planes[0];
  p.dcb = planes[1];
  p.dcr = planes[2];
  J.ycc420 = 1;
  J.width = p.cw;
  rows[0] = p.lh;
  rows[1] = rows[2] = p.ch;
  memset(out, 0, sizeof *out);
  out->v.fmt = F_YUV420;
  out->v.w = src.v.w;
  out->v.h = src.v.h;
  out->v.full_range = 1;
  for (int c = 0; c < 3; c++) {
    out->v.p[c] = planes[c];
    out->v.stride[c] = c ? p.cw : p.lw;
  }
  return E_OK;
}

// one H2D copy of a host plan array into workspace device memory
template <class T>
int upload_plan(Workspace& ws, const T* h, size_t n, T** d) {
  *d = (T*)ws.dalloc(sizeof(T) * n);
  if (!*d) return E_MEM;
  CUDA_TRY(cudaMemcpyAsync(*d, h, sizeof(T) * n, cudaMemcpyHostToDevice, ws.stream()));
  return E_OK;
}

}  // namespace

size_t JpegRCodec::encode_bytes(const DecodedInfo& in, int k) {
  const size_t w = (in.width + k - 1) / k, h = (in.height + k - 1) / k, gw = (in.gm_width + k - 1) / k,
               gh = (in.gm_height + k - 1) / k;
  size_t enc = 0;
  for (int j = 0; j < 2; j++) {   // per JPEG: staged planes, 256 B of code-word entries and 16 B of meta per block, the scan
    const size_t pw = j ? gw : w, ph = j ? gh : h, blocks = 3 * ((pw + 15) / 8) * ((ph + 15) / 8);
    enc += 3 * (pw + 8) * (ph + 16) + blocks * (256 + 16) + pw * ph * 6 + 8192;
  }
  return enc;
}

size_t JpegRCodec::batch_decode_bytes(int w, int h, int gw, int gh, int k, size_t size) {
  // coefficients (128 B per 8x8 block, at most 3 components at full size) and their DC terms, planes, coded bits
  const size_t px = (size_t)w * k * h * k + (size_t)gw * k * gh * k;
  return px * 7 + (size_t)(w * h + gw * gh) * 16 + 2 * size;
}

int JpegRCodec::transcode_batch(TranscodeBatchItem* items, int n, const uhdr_b200_transcode_config_t& cfg, size_t group_bytes) {
  int rc = settle();
  if (rc) return rc;
  map_pending_ = false;
  const int k = cfg.k;
  auto cost = [&](int i, size_t* coded) {
    const DecodedInfo& in = items[i].info;
    *coded = items[i].size;
    const int w = (in.width + k - 1) / k, h = (in.height + k - 1) / k, gw = (in.gm_width + k - 1) / k,
              gh = (in.gm_height + k - 1) / k;
    return batch_decode_bytes(w, h, gw, gh, k, items[i].size) + encode_bytes(in, k);
  };
  rc = for_each_group(n, group_bytes, cost, [&](int g0, int g1) { return transcode_batch_group(items + g0, g1 - g0, cfg); });
  if (rc) mark_in_flight();   // as transcode(): kernels of the group may still run
  return rc;
}

int JpegRCodec::transcode_batch_group(TranscodeBatchItem* items, int n, const uhdr_b200_transcode_config_t& cfg) {
  // 1-3. both JPEGs of every item decoded as transcode() decodes them: raw planes, a 3-channel map as YCbCr
  int rc = decode_batch_files(items, n, cfg.k, 0, false, 0);
  if (rc) return rc;
  for (int i = 0; i < n; i++) items[i].cfg = cfg;
  return transcode_encode(items, n);
}

int JpegRCodec::transcode_ladders(LadderFile* files, int n, TranscodeBatchItem* rungs, size_t group_bytes) {
  int rc = settle();
  if (rc) return rc;
  map_pending_ = false;
  // a file's scratch: its coefficients and full-size planes once, its planes at every other k, each rung's encode
  auto cost = [&](int i, size_t* coded) {
    const LadderFile& F = files[i];
    *coded = 0;
    if (F.rc) return size_t(0);
    const DecodedInfo& in = F.info;
    const size_t size = in.base_len + in.gainmap_len;
    *coded = size;
    size_t b = batch_decode_bytes(in.width, in.height, in.gm_width, in.gm_height, 1, size);
    bool seen[9] = {false};
    for (int j = 0; j < F.nr; j++) {
      const TranscodeBatchItem& r = rungs[F.r0 + j];
      if (r.rc) continue;
      const int k = r.cfg.k;
      if (k != 1 && !seen[k]) {
        const size_t w = (in.width + k - 1) / k, h = (in.height + k - 1) / k, gw = (in.gm_width + k - 1) / k,
                     gh = (in.gm_height + k - 1) / k;
        b += 3 * (w * h + gw * gh);
      }
      seen[k] = true;
      b += encode_bytes(in, k);
    }
    return b;
  };
  // the distinct quality pairs of the group being formed, at most kLadderMaxRungs
  int pairs[kLadderMaxRungs][2], npairs = 0;
  auto admit = [&](int i, bool fresh) {
    if (fresh) npairs = 0;
    int m = npairs;
    for (int j = 0; j < files[i].nr && !files[i].rc; j++) {
      const TranscodeBatchItem& r = rungs[files[i].r0 + j];
      if (r.rc) continue;
      int p = 0;
      while (p < m && (pairs[p][0] != r.cfg.base_quality || pairs[p][1] != r.cfg.gainmap_quality)) p++;
      if (p < m) continue;
      if (m == kLadderMaxRungs) return false;   // a file alone has at most kLadderMaxRungs rungs: never when fresh
      pairs[m][0] = r.cfg.base_quality;
      pairs[m++][1] = r.cfg.gainmap_quality;
    }
    npairs = m;
    return true;
  };
  rc = for_each_group(n, group_bytes, cost, [&](int g0, int g1) {
    // the group's rungs follow each other in `rungs`; a group of files with argument errors alone has none
    const int r0 = files[g0].r0, r1 = files[g1 - 1].r0 + files[g1 - 1].nr;
    int r = decode_ladders(files + g0, g1 - g0, rungs);
    return r || r1 == r0 ? r : transcode_encode(rungs + r0, r1 - r0);
  }, admit);
  if (rc) mark_in_flight();   // as transcode(): kernels of the group may still run
  return rc;
}

int JpegRCodec::transcode_encode(TranscodeBatchItem* items, int n) {
  if ((int)batch_enc_.size() < 2 * n) batch_enc_.resize(2 * n);
  // 4. the staging jobs and the block stage's planes of both JPEGs of every item; per quality pair, base quantisers
  // 0 / 1, map's 2 / 3
  StageJob* h_stage = (StageJob*)ws_.halloc(sizeof(StageJob) * 6 * n);
  unsigned* h_stage_end = (unsigned*)ws_.halloc(sizeof(unsigned) * 6 * n);
  Fdct8Plane* h_pl = (Fdct8Plane*)ws_.halloc(sizeof(Fdct8Plane) * 6 * n);
  int* h_pair = (int*)ws_.halloc(sizeof(int) * 6 * n);
  Fdct8Plane* h_sub = (Fdct8Plane*)ws_.halloc(sizeof(Fdct8Plane) * 6 * n);
  unsigned* h_sub_end = (unsigned*)ws_.halloc(sizeof(unsigned) * 6 * n);
  if (!h_stage || !h_stage_end || !h_pl || !h_pair || !h_sub || !h_sub_end) return E_MEM;
  int pairs[kLadderMaxRungs][2], npairs = 0;
  uint16_t q[kLadderMaxRungs][4][64];
  int rc = E_OK, nst = 0, npl = 0, nenc = 0;
  JpegEncodeJob** enc = batch_enc_.data();
  for (int i = 0; i < n; i++) {
    TranscodeBatchItem& it = items[i];
    if (it.rc) continue;
    const uhdr_b200_transcode_config_t& cfg = it.cfg;
    if (cfg.base_420 && it.sdr.v.fmt == F_YUV422) {   // after every map error, as in transcode()
      batch_fail(it, fail_base_422(), last_error());
      continue;
    }
    DevImage base_in, map_in;
    int base_rows[3], map_rows[3];
    const int nst0 = nst;
    int r = cfg.base_420 && it.sdr.v.fmt == F_YUV444 ? plan_ycc444_to_420(ws_, it.sdr, h_stage, &nst, &base_in, base_rows)
                                                     : plan_stage_tight(ws_, it.sdr, h_stage, &nst, &base_in, base_rows);
    if (!r) r = plan_stage_tight(ws_, it.map, h_stage, &nst, &map_in, map_rows);
    Fdct8Params P[2];
    if (!r) r = jpeg_forward_plan(ws_, base_in, cfg.base_quality, &it.base_jpeg, /*zigzag=*/true, base_rows, &P[0]);
    if (!r) r = jpeg_forward_plan(ws_, map_in, cfg.gainmap_quality, &it.gm_jpeg, /*zigzag=*/true, map_rows, &P[1]);
    if (r == E_MEM) return r;
    if (r) {
      nst = nst0;
      batch_fail(it, r, last_error());
      continue;
    }
    int pi = 0;
    while (pi < npairs && (pairs[pi][0] != cfg.base_quality || pairs[pi][1] != cfg.gainmap_quality)) pi++;
    if (pi == npairs) {
      if (npairs == kLadderMaxRungs) return fail(E_ERROR, "internal: more than %d quality pairs in one call", kLadderMaxRungs);
      pairs[pi][0] = cfg.base_quality;
      pairs[pi][1] = cfg.gainmap_quality;
      for (int j = 0; j < 2; j++) memcpy(q[pi][2 * j], P[j].q, sizeof P[j].q);
      npairs++;
    }
    for (int j = 0; j < 2; j++) {
      for (int c = 0; c < P[j].nplanes; c++) {
        h_pl[npl] = P[j].plane[c];
        h_pl[npl].tq[0] += 2 * j;
        h_pair[npl++] = pi;
      }
    }
    enc[nenc++] = &it.base_jpeg;
    enc[nenc++] = &it.gm_jpeg;
  }
  if (!nenc) return E_OK;
  unsigned ctas = 0;
  for (int j = 0; j < nst; j++) {
    const StageJob& J = h_stage[j];
    ctas += (unsigned)(((size_t)J.width * (J.ycc420 ? J.p.ch : J.rows) + 255) / 256);
    h_stage_end[j] = ctas;
  }
  // 5. one staging launch, one block-stage launch per quality pair, one entropy-coding launch for every item
  StageJob* d_stage;
  unsigned* d_stage_end;
  if ((rc = upload_plan(ws_, h_stage, nst, &d_stage)) || (rc = upload_plan(ws_, h_stage_end, nst, &d_stage_end))) return rc;
  count_launches(1);
  ws_.t_begin("stage_batch");
  k_stage_batch<<<ctas, 256, 0, ws_.stream()>>>(d_stage, d_stage_end, (unsigned)nst);
  ws_.t_end();
  CUDA_TRY(cudaGetLastError());
  for (int pi = 0, off = 0; pi < npairs; pi++) {
    int ns = 0;
    unsigned items_total = 0;
    for (int j = 0; j < npl; j++) {
      if (h_pair[j] != pi) continue;
      h_sub[off + ns] = h_pl[j];
      items_total += (unsigned)(h_pl[j].wblocks * h_pl[j].hblocks + 31) / 32;
      h_sub_end[off + ns++] = items_total;
    }
    Fdct8Plane* d_pl;
    unsigned* d_pl_end;
    if ((rc = upload_plan(ws_, h_sub + off, ns, &d_pl)) || (rc = upload_plan(ws_, h_sub_end + off, ns, &d_pl_end))) return rc;
    TIMED(ws_, "fdct_code_batch", launch_fdct8_code_batch(d_pl, d_pl_end, (unsigned)ns, items_total, q[pi], ws_.stream()));
    off += ns;
  }
  if ((rc = jpeg_entropy_batch_dev(ws_, enc, nenc))) return rc;
  // 6. two host waits: every scan's size, then every scan's bytes
  if ((rc = ws_.sync())) return rc;
  if ((rc = jpeg_entropy_batch_fetch(ws_, enc, nenc))) return rc;
  if ((rc = ws_.sync())) return rc;
  // 7. per item, the file
  for (int i = 0; i < n; i++) {
    TranscodeBatchItem& it = items[i];
    if (it.rc) continue;
    int r = jpeg_scan_check(it.base_jpeg);   // in transcode()'s order
    if (!r) r = jpeg_scan_check(it.gm_jpeg);
    if (!r) r = transcode_finish(it.data, it.info, it.ph, it.gh, it.base_jpeg, it.gm_jpeg, it.cfg, it.out, it.cap, &it.out_size);
    if (r) batch_fail(it, r, last_error());
  }
  return E_OK;
}

}  // namespace uhdr_b200
