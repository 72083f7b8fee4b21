// Device orchestration of the JPEG block stage (see jpeg.h).
#include <algorithm>
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

IdctPlane* jpeg_idct_stage(Workspace& ws, int n) {
  return (IdctPlane*)ws.halloc((sizeof(IdctPlane) + sizeof(unsigned)) * n);
}

void jpeg_idct_plane(IdctPlane* p, const JpegFrame& f, int c, const int16_t* coefs, int s, uint8_t* dst, int stride) {
  const JpegComp& k = f.comp[c];
  if (!p->nout) {
    p->coefs = coefs;
    memcpy(p->q, f.qt[k.tq], sizeof p->q);
    p->wblocks = k.wblocks;
    p->blocks = k.wblocks * k.hblocks;
  }
  IdctPlane::Out& o = p->out[p->nout++];
  o.dst = dst;
  o.s = s;
  o.dst_stride = stride;
  o.dst_w = s == 8 ? std::min(k.wblocks * 8, stride) : k.wblocks * s;
  o.dst_h = k.hblocks * s;
}

namespace {
// planes[0, n) of a jpeg_idct_stage and the CTA ends after them, end[n] (each run of planes launched together counts
// from 0), to the device with one copy
int idct_upload(Workspace& ws, const IdctPlane* planes, int n, IdctPlane** d_pl, unsigned** d_end) {
  const size_t bytes = (sizeof(IdctPlane) + sizeof(unsigned)) * n;
  *d_pl = (IdctPlane*)ws.dalloc(bytes);
  if (!*d_pl) return E_MEM;
  *d_end = (unsigned*)(*d_pl + n);
  CUDA_TRY(cudaMemcpyAsync(*d_pl, planes, bytes, cudaMemcpyHostToDevice, ws.stream()));
  return E_OK;
}
}  // namespace

int jpeg_idct_dev(Workspace& ws, const JpegIdctJob* jobs, int n) {
  int np = 0;
  for (int i = 0; i < n; i++) np += jobs[i].h->frame.ncomp;
  IdctPlane* h_pl = jpeg_idct_stage(ws, np);
  if (!h_pl) return E_MEM;
  unsigned* h_end = (unsigned*)(h_pl + np);
  // the planes by size, 8 first: run r (size 8 >> r) is planes [first[r], first[r + 1]), ctas[r] CTAs
  int first[5], m = 0;
  unsigned ctas[4];
  for (int r = 0; r < 4; r++) {
    first[r] = m;
    ctas[r] = 0;
    for (int i = 0; i < n; i++) {
      const JpegFrame& f = jobs[i].h->frame;
      for (int c = 0; c < f.ncomp; c++) {
        const int s = jobs[i].g ? jobs[i].g->s[c] : 8;
        if (s != 8 >> r) continue;
        IdctPlane& p = h_pl[m];
        p.nout = 0;
        jpeg_idct_plane(&p, f, c, jobs[i].d_coefs[c], s, jobs[i].planes[c], jobs[i].strides[c]);
        ctas[r] += (unsigned)(p.blocks + 127) / 128;
        h_end[m++] = ctas[r];
      }
    }
  }
  first[4] = m;
  IdctPlane* d_pl;
  unsigned* d_end;
  if (int rc = idct_upload(ws, h_pl, np, &d_pl, &d_end)) return rc;
  for (int r = 0; r < 4; r++) {
    const unsigned k = (unsigned)(first[r + 1] - first[r]);
    if (k)
      TIMED(ws, r ? "idct_scaled" : "idct_dequant", launch_idct(8 >> r, d_pl + first[r], d_end + first[r], k, ctas[r], ws.stream()));
  }
  return E_OK;
}

int jpeg_idct_multi_dev(Workspace& ws, IdctPlane* planes, int n) {
  unsigned* h_end = (unsigned*)(planes + n);
  unsigned ctas = 0;
  for (int i = 0; i < n; i++) {
    ctas += (unsigned)(planes[i].blocks + 127) / 128;
    h_end[i] = ctas;
  }
  IdctPlane* d_pl;
  unsigned* d_end;
  if (int rc = idct_upload(ws, planes, n, &d_pl, &d_end)) return rc;
  TIMED(ws, "idct_multi", launch_idct(0, d_pl, d_end, (unsigned)n, ctas, ws.stream()));
  return E_OK;
}

namespace {
std::atomic<int> g_entropy_decoder{0};
}
void jpeg_set_entropy_decoder(int mode) { g_entropy_decoder.store(mode < 0 || mode > 2 ? 0 : mode); }
int jpeg_get_entropy_decoder() { return g_entropy_decoder.load(); }

}  // namespace uhdr_b200
