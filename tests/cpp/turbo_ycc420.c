/*
 * turbo_ycc420.c -- TEST INFRASTRUCTURE ONLY: the checker of uhdr_b200_transcode's 4:2:0 base image.
 *
 * A thin harness over the real libjpeg-turbo (the binary oracle/_ref/libuhdr_ref_turbo.so links, declared by
 * oracle/ref_turbo/jpeglib.h).  tests/transcode_testlib.py compiles it into a temporary directory.
 */
#include <setjmp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "jpeglib.h"

/* exported by every libjpeg-turbo build, not declared by the hand-written header */
extern void jpeg_mem_dest(j_compress_ptr cinfo, unsigned char** outbuffer, unsigned long* outsize);

typedef struct {
  struct jpeg_error_mgr pub;
  jmp_buf jb;
} tyc_err_t;

static void tyc_error_exit(j_common_ptr cinfo) { longjmp(((tyc_err_t*)cinfo->err)->jb, 1); }
static void tyc_quiet(j_common_ptr cinfo, int level) {
  (void)cinfo;
  (void)level;
}

/* The 4:2:0 JPEG libjpeg-turbo writes from full-size YCbCr planes (each w x h, stride w) through jpeg_write_scanlines:
 * jpeg_set_defaults, jpeg_set_quality(quality, TRUE), sampling 2x2 / 1x1 / 1x1, JDCT_ISLOW, and the APP2 marker `icc`
 * (whole payload, none for icc_size 0) written right after jpeg_start_compress, as JpegEncoderHelper writes it.  The
 * chroma goes through libjpeg's own downsampler (jcsample.c h2v2_downsample) and edge replication (jcprepct.c).
 * Returns 0, 1 on a libjpeg error, 2 if cap is too small (*size is then the size needed). */
int tyc_encode_ycc420(const uint8_t* y, const uint8_t* cb, const uint8_t* cr, int w, int h, int quality, const uint8_t* icc,
                      size_t icc_size, uint8_t* out, size_t cap, size_t* size) {
  struct jpeg_compress_struct cinfo;
  tyc_err_t err;
  unsigned char* volatile mem = NULL;
  unsigned long mem_size = 0;
  uint8_t* volatile row = NULL;
  memset(&cinfo, 0, sizeof cinfo);
  cinfo.err = jpeg_std_error(&err.pub);
  err.pub.error_exit = tyc_error_exit;
  err.pub.emit_message = tyc_quiet;
  if (setjmp(err.jb)) {
    jpeg_destroy_compress(&cinfo);
    free(mem);
    free(row);
    return 1;
  }
  jpeg_create_compress(&cinfo);
  jpeg_mem_dest(&cinfo, (unsigned char**)&mem, &mem_size);
  cinfo.image_width = (JDIMENSION)w;
  cinfo.image_height = (JDIMENSION)h;
  cinfo.input_components = 3;
  cinfo.in_color_space = JCS_YCbCr;
  jpeg_set_defaults(&cinfo);
  jpeg_set_quality(&cinfo, quality, TRUE);
  cinfo.comp_info[0].h_samp_factor = 2;
  cinfo.comp_info[0].v_samp_factor = 2;
  for (int c = 1; c < 3; c++) cinfo.comp_info[c].h_samp_factor = cinfo.comp_info[c].v_samp_factor = 1;
  cinfo.dct_method = JDCT_ISLOW;
  jpeg_start_compress(&cinfo, TRUE);
  if (icc && icc_size) jpeg_write_marker(&cinfo, JPEG_APP0 + 2, icc, (unsigned)icc_size);
  row = (uint8_t*)malloc((size_t)w * 3);
  while (cinfo.next_scanline < cinfo.image_height) {
    const size_t o = (size_t)cinfo.next_scanline * w;
    for (int x = 0; x < w; x++) {
      row[3 * x] = y[o + x];
      row[3 * x + 1] = cb[o + x];
      row[3 * x + 2] = cr[o + x];
    }
    JSAMPROW r = row;
    jpeg_write_scanlines(&cinfo, &r, 1);
  }
  jpeg_finish_compress(&cinfo);
  jpeg_destroy_compress(&cinfo);
  free(row);
  *size = mem_size;
  const int rc = mem_size > cap ? 2 : 0;
  if (!rc) memcpy(out, mem, mem_size);
  free(mem);
  return rc;
}
