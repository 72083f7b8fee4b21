// Device orchestration of the JPEG block stage (see jpeg.h).
#include <atomic>
#include <cmath>
#include <cstring>

#include "jpeg.h"

namespace uhdr_b200 {

int jpeg_forward_dev(Workspace& ws, const DevImage& img, int quality, JpegEncodeJob* job, bool zigzag, const int* rows) {
  Fdct8Params P;
  const int rc = jpeg_forward_plan(ws, img, quality, job, zigzag, rows, &P);
  if (rc) return rc;
  TIMED(ws, "fdct_quant", launch_fdct8(P, ws.stream()));
  return E_OK;
}

int jpeg_encode_dev(Workspace& ws, const DevImage& img, int quality, JpegEncodeJob* job, const int* rows) {
  int rc = jpeg_forward_dev(ws, img, quality, job, /*zigzag=*/true, rows);
  if (rc) return rc;
  return jpeg_entropy_dev(ws, job);
}

int jpeg_stream_pieces(Workspace& ws, const JpegEncodeJob& job, const void* icc, size_t icc_size, JpegPieces* out) {
  const size_t cap = kJpegHeadBytes + icc_size;
  uint8_t* head = (uint8_t*)ws.halloc(cap);
  if (!head) return E_MEM;
  ByteSink o(head, cap);
  jpeg_write_headers(job, icc, icc_size, o);
  if (!o.ok()) return fail(E_ERROR, "JPEG header of %zu bytes exceeds its bound of %zu", o.size(), cap);
  *out = JpegPieces{head, o.size(), job.h_scan, job.h_scan_bytes[3]};
  return E_OK;
}

int jpeg_forward_plan(Workspace& ws, const DevImage& img, int quality, JpegEncodeJob* job, bool zigzag, const int* rows,
                      Fdct8Params* out) {
  int rc = jpeg_frame_init(&job->frame, img.v.fmt, img.v.w, img.v.h, quality);
  if (rc) return rc;
  const JpegFrame& f = job->frame;
  job->zigzag = zigzag;
  job->gainmap_comment = img.v.fmt == F_RGB888 || img.v.fmt == F_Y400;
  Fdct8Params& P = *out;
  memset(&P, 0, sizeof P);
  P.zigzag = zigzag ? 1 : 0;
  memcpy(P.q[0], f.qt[0], sizeof P.q[0]);
  memcpy(P.q[1], f.qt[1], sizeof P.q[1]);
  for (int c = 0; c < f.ncomp; c++) {
    // natural order: 64 coefficients per block; device entropy path: 64 code-word entries of 4 bytes
    // per block (only the entries of non-zero coefficients are ever written or read)
    job->d_coefs[c] = (int16_t*)ws.dalloc(f.blocks(c) * (zigzag ? 256 : 128));
    if (!job->d_coefs[c]) return E_MEM;
    job->d_meta[c] = nullptr;
    if (zigzag) {  // side information for the device entropy coder
      job->d_meta[c] = (uint4*)ws.dalloc(f.blocks(c) * sizeof(uint4));
      if (!job->d_meta[c]) return E_MEM;
    }
  }
  if (img.v.fmt == F_RGB888) {
    // jpeg_write_scanlines path: jccolor.c conversion, edges replicated (jcsample.c/jcprepct.c);
    // the three components come out of one pass over the pixels
    Fdct8Plane& pl = P.plane[0];
    P.nplanes = 1;
    pl.src = (const uint8_t*)img.v.p[0];
    pl.stride = img.v.stride[0];
    pl.w = img.v.w;
    pl.h = img.v.h;
    pl.wblocks = f.comp[0].wblocks;
    pl.hblocks = f.comp[0].hblocks;
    pl.rgb = 1;
    for (int c = 0; c < 3; c++) {
      pl.tq[c] = f.comp[c].tq;
      pl.coefs[c] = job->d_coefs[c];
      pl.meta[c] = job->d_meta[c];
      pl.hsel[c] = c == 0 ? 0 : 1;
    }
  } else {
    // raw_data_in path (jpegencoderhelper.cpp:246-309): whole blocks are read from the plane
    // (device strides are >= wblocks*8 and the bytes past the width are defined, see
    // alloc_dev_image / upload); rows past the plane height come from the helper's pad row:
    // 0 for luma, 128 for chroma.
    P.nplanes = f.ncomp;
    for (int c = 0; c < f.ncomp; c++) {
      const JpegComp& k = f.comp[c];
      if (img.v.stride[c] < k.wblocks * 8)
        return fail(E_ERROR, "internal: device plane stride %d < padded width %d", img.v.stride[c], k.wblocks * 8);
      if (((size_t)img.v.p[c] & 7) || (img.v.stride[c] & 7))
        return fail(E_ERROR, "internal: device plane %d not 8-byte aligned", c);
      Fdct8Plane& pl = P.plane[c];
      pl.src = (const uint8_t*)img.v.p[c];
      pl.stride = img.v.stride[c];
      pl.w = k.wblocks * 8;
      pl.h = rows && rows[c] > 0 ? rows[c] : k.height;
      pl.wblocks = k.wblocks;
      pl.hblocks = k.hblocks;
      pl.fill = c == 0 ? 0 : 128;
      pl.tq[0] = k.tq;
      pl.coefs[0] = job->d_coefs[c];
      pl.meta[0] = job->d_meta[c];
      pl.hsel[0] = c == 0 ? 0 : 1;
    }
  }
  return E_OK;
}

int jpeg_idct_dev(Workspace& ws, const JpegHeader& h, int16_t* const d_coefs[3], uint8_t* d_planes[3], int plane_stride[3]) {
  const JpegFrame& f = h.frame;
  for (int c = 0; c < f.ncomp; c++) {
    const JpegComp& k = f.comp[c];
    IdctPlaneParams p;
    memset(&p, 0, sizeof p);
    p.coefs = d_coefs[c];
    memcpy(p.q, f.qt[k.tq], sizeof p.q);
    p.wblocks = k.wblocks;
    p.hblocks = k.hblocks;
    p.dst = d_planes[c];
    p.dst_stride = plane_stride[c];
    p.dst_w = k.wblocks * 8 < plane_stride[c] ? k.wblocks * 8 : plane_stride[c];
    p.dst_h = k.hblocks * 8;
    TIMED(ws, "idct_dequant", launch_idct_dequant(p, ws.stream()));
  }
  return E_OK;
}

int jpeg_inverse_dev(Workspace& ws, const JpegHeader& h, int16_t* const h_coefs[3], uint8_t* d_planes[3],
                     int plane_stride[3]) {
  const JpegFrame& f = h.frame;
  int16_t* d_coefs[3] = {nullptr, nullptr, nullptr};
  for (int c = 0; c < f.ncomp; c++) {
    d_coefs[c] = (int16_t*)ws.dalloc(f.blocks(c) * 128);
    if (!d_coefs[c]) return E_MEM;
    CUDA_TRY(cudaMemcpyAsync(d_coefs[c], h_coefs[c], f.blocks(c) * 128, cudaMemcpyHostToDevice, ws.stream()));
  }
  return jpeg_idct_dev(ws, h, d_coefs, d_planes, plane_stride);
}

int jpeg_idct_scaled_dev(Workspace& ws, const JpegHeader& h, const JpegScaled& g, int16_t* const d_coefs[3],
                         uint8_t* d_planes[3], int plane_stride[3]) {
  const JpegFrame& f = h.frame;
  for (int c = 0; c < f.ncomp; c++) {
    if (g.s[c] != 8) continue;
    const JpegComp& k = f.comp[c];
    IdctPlaneParams p;
    memset(&p, 0, sizeof p);
    p.coefs = d_coefs[c];
    memcpy(p.q, f.qt[k.tq], sizeof p.q);
    p.wblocks = k.wblocks;
    p.hblocks = k.hblocks;
    p.dst = d_planes[c];
    p.dst_stride = plane_stride[c];
    p.dst_w = k.wblocks * 8 < plane_stride[c] ? k.wblocks * 8 : plane_stride[c];
    p.dst_h = k.hblocks * 8;
    TIMED(ws, "idct_dequant", launch_idct_dequant(p, ws.stream()));
  }
  for (int size = 4; size >= 1; size /= 2) {
    IdctScaledParams p;
    memset(&p, 0, sizeof p);
    int blocks = 0;
    for (int c = 0; c < f.ncomp; c++) {
      if (g.s[c] != size) continue;
      const JpegComp& k = f.comp[c];
      IdctScaledParams::Plane& pl = p.plane[p.nplanes];
      pl.coefs = d_coefs[c];
      memcpy(pl.q, f.qt[k.tq], sizeof pl.q);
      pl.wblocks = k.wblocks;
      pl.dst = d_planes[c];
      pl.dst_stride = plane_stride[c];
      pl.dst_w = k.wblocks * size;
      pl.dst_h = k.hblocks * size;
      blocks += k.wblocks * k.hblocks;
      p.block_end[p.nplanes++] = blocks;
    }
    if (p.nplanes) TIMED(ws, "idct_scaled", launch_idct_scaled(p, size, ws.stream()));
  }
  return E_OK;
}

int jpeg_inverse_scaled_dev(Workspace& ws, const JpegHeader& h, const JpegScaled& g, int16_t* const h_coefs[3],
                            uint8_t* d_planes[3], int plane_stride[3]) {
  const JpegFrame& f = h.frame;
  int16_t* d_coefs[3] = {nullptr, nullptr, nullptr};
  for (int c = 0; c < f.ncomp; c++) {
    d_coefs[c] = (int16_t*)ws.dalloc(f.blocks(c) * 128);
    if (!d_coefs[c]) return E_MEM;
    CUDA_TRY(cudaMemcpyAsync(d_coefs[c], h_coefs[c], f.blocks(c) * 128, cudaMemcpyHostToDevice, ws.stream()));
  }
  return jpeg_idct_scaled_dev(ws, h, g, d_coefs, d_planes, plane_stride);
}

int jpeg_idct_batch_dev(Workspace& ws, const JpegIdctJob* jobs, int n) {
  const size_t cap = 3 * (size_t)n;
  for (int size = 8; size >= 1; size /= 2) {
    IdctBatchPlane* h_pl = (IdctBatchPlane*)ws.halloc(sizeof(IdctBatchPlane) * cap);
    unsigned* h_end = (unsigned*)ws.halloc(sizeof(unsigned) * cap);
    if (!h_pl || !h_end) return E_MEM;
    unsigned np = 0, ctas = 0;
    for (int i = 0; i < n; i++) {
      const JpegFrame& f = jobs[i].h->frame;
      for (int c = 0; c < f.ncomp; c++) {
        if ((jobs[i].g ? jobs[i].g->s[c] : 8) != size) continue;
        const JpegComp& k = f.comp[c];
        IdctBatchPlane& p = h_pl[np];
        p.coefs = jobs[i].d_coefs[c];
        memcpy(p.q, f.qt[k.tq], sizeof p.q);
        p.wblocks = k.wblocks;
        p.blocks = k.wblocks * k.hblocks;
        p.dst = jobs[i].planes[c];
        p.dst_stride = jobs[i].strides[c];
        p.dst_w = size == 8 ? (k.wblocks * 8 < p.dst_stride ? k.wblocks * 8 : p.dst_stride) : k.wblocks * size;
        p.dst_h = k.hblocks * size;
        ctas += (unsigned)(p.blocks + 127) / 128;
        h_end[np++] = ctas;
      }
    }
    if (!np) continue;
    IdctBatchPlane* d_pl = (IdctBatchPlane*)ws.dalloc(sizeof(IdctBatchPlane) * np);
    unsigned* d_end = (unsigned*)ws.dalloc(sizeof(unsigned) * np);
    if (!d_pl || !d_end) return E_MEM;
    CUDA_TRY(cudaMemcpyAsync(d_pl, h_pl, sizeof(IdctBatchPlane) * np, cudaMemcpyHostToDevice, ws.stream()));
    CUDA_TRY(cudaMemcpyAsync(d_end, h_end, sizeof(unsigned) * np, cudaMemcpyHostToDevice, ws.stream()));
    if (size == 8) TIMED(ws, "idct_dequant_batch", launch_idct_dequant_batch(d_pl, d_end, np, ctas, ws.stream()));
    else TIMED(ws, "idct_scaled_batch", launch_idct_scaled_batch(d_pl, d_end, np, ctas, size, ws.stream()));
  }
  return E_OK;
}

int jpeg_idct_multi_dev(Workspace& ws, const IdctMultiPlane* planes, int n) {
  unsigned* h_end = (unsigned*)ws.halloc(sizeof(unsigned) * n);
  if (!h_end) return E_MEM;
  unsigned ctas = 0;
  for (int i = 0; i < n; i++) {
    ctas += (unsigned)(planes[i].blocks + 127) / 128;
    h_end[i] = ctas;
  }
  IdctMultiPlane* d_pl = (IdctMultiPlane*)ws.dalloc(sizeof(IdctMultiPlane) * n);
  unsigned* d_end = (unsigned*)ws.dalloc(sizeof(unsigned) * n);
  if (!d_pl || !d_end) return E_MEM;
  CUDA_TRY(cudaMemcpyAsync(d_pl, planes, sizeof(IdctMultiPlane) * n, cudaMemcpyHostToDevice, ws.stream()));
  CUDA_TRY(cudaMemcpyAsync(d_end, h_end, sizeof(unsigned) * n, cudaMemcpyHostToDevice, ws.stream()));
  TIMED(ws, "idct_multi", launch_idct_multi(d_pl, d_end, (unsigned)n, ctas, ws.stream()));
  return E_OK;
}

namespace {
std::atomic<int> g_entropy_decoder{0};
}
void jpeg_set_entropy_decoder(int mode) { g_entropy_decoder.store(mode < 0 || mode > 2 ? 0 : mode); }
int jpeg_get_entropy_decoder() { return g_entropy_decoder.load(); }

}  // namespace uhdr_b200
