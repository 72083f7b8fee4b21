/*
 * jpeg_scaled_ref.c -- TEST INFRASTRUCTURE ONLY.
 *
 * A thin harness over the real libjpeg-turbo (the binary _ref/libuhdr_ref_turbo.so links, declared by
 * ref_turbo/jpeglib.h) that decodes a baseline JPEG with scale_num = 1, scale_denom = k: what libjpeg-turbo
 * users (TurboJPEG, Pillow's draft()) get as a reduced-size decode.  It is the checker of the scaled decoder:
 *   jsr_decode(..., mode 0) raw_data_out planes, as JpegDecoderHelper decodes the primary image;
 *   jsr_decode(..., mode 1) JCS_EXT_RGBA scanlines, as it decodes a 3-channel gain map.
 * Built by oracle/scaled.mk into _ref/libjpeg_scaled_ref.so.
 */
#include <setjmp.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "jpeglib.h"

/* exported by every libjpeg-turbo build, not declared by the hand-written header */
extern void jpeg_mem_src(j_decompress_ptr cinfo, const unsigned char* inbuffer, unsigned long insize);

typedef struct {
  struct jpeg_error_mgr pub;
  jmp_buf jb;
} jsr_err_t;

static void jsr_error_exit(j_common_ptr cinfo) { longjmp(((jsr_err_t*)cinfo->err)->jb, 1); }
/* prints nothing, but counts warnings (level -1: corrupt data that libjpeg decodes anyway) like the default does */
static void jsr_quiet(j_common_ptr cinfo, int level) {
  if (level < 0) cinfo->err->num_warnings++;
}

/* info (16 ints): [0] output_width, [1] output_height, [2] num_components, [3] min_DCT_scaled_size, then per
 * component c < 3: [4 + 3c] DCT_scaled_size, [5 + 3c] downsampled_width, [6 + 3c] downsampled_height; [15] the
 * warnings libjpeg raised (after a decode; 0 for out == NULL).
 * mode 0: planes back to back, plane c downsampled_width x downsampled_height, tightly packed.
 * mode 1: output_width x output_height RGBA pixels.
 * out == NULL: header and geometry only.  Returns 0, 1 on a libjpeg error, 2 if cap is too small. */
int jsr_decode(const uint8_t* data, size_t size, int k, int mode, uint8_t* out, size_t cap, int info[16]) {
  struct jpeg_decompress_struct cinfo;
  jsr_err_t err;
  uint8_t* volatile tmp = NULL;    /* volatile: still valid after the longjmp of an error */
  JSAMPROW* volatile rows = NULL;
  volatile int rc = 1;
  memset(&cinfo, 0, sizeof cinfo);
  cinfo.err = jpeg_std_error(&err.pub);
  err.pub.error_exit = jsr_error_exit;
  err.pub.emit_message = jsr_quiet;
  if (setjmp(err.jb)) {
    free(tmp);
    free(rows);
    jpeg_destroy_decompress(&cinfo);
    return rc;
  }
  jpeg_create_decompress(&cinfo);
  jpeg_mem_src(&cinfo, data, (unsigned long)size);
  jpeg_read_header(&cinfo, TRUE);
  cinfo.scale_num = 1;
  cinfo.scale_denom = (unsigned)k;
  cinfo.dct_method = JDCT_ISLOW;
  if (mode == 0) {
    cinfo.raw_data_out = TRUE;
  } else {
    cinfo.out_color_space = JCS_EXT_RGBA;
  }
  jpeg_start_decompress(&cinfo);
  memset(info, 0, 16 * sizeof(int));
  info[0] = (int)cinfo.output_width;
  info[1] = (int)cinfo.output_height;
  info[2] = cinfo.num_components;
  info[3] = cinfo.min_DCT_scaled_size;
  size_t need = 0;
  for (int c = 0; c < cinfo.num_components; c++) {
    const jpeg_component_info* ci = &cinfo.comp_info[c];
    if (c < 3) {
      info[4 + 3 * c] = ci->DCT_scaled_size;
      info[5 + 3 * c] = (int)ci->downsampled_width;
      info[6 + 3 * c] = (int)ci->downsampled_height;
    }
    need += (size_t)ci->downsampled_width * ci->downsampled_height;
  }
  if (mode == 1) need = (size_t)cinfo.output_width * cinfo.output_height * 4;
  if (!out) {
    jpeg_abort_decompress(&cinfo);
    jpeg_destroy_decompress(&cinfo);
    return 0;
  }
  rc = 2;
  if (need > cap) longjmp(err.jb, 1);
  rc = 1;
  if (mode == 1) {
    rows = (JSAMPROW*)malloc(sizeof(JSAMPROW));
    while (cinfo.output_scanline < cinfo.output_height) {
      rows[0] = out + (size_t)cinfo.output_scanline * cinfo.output_width * 4;
      jpeg_read_scanlines(&cinfo, rows, 1);
    }
  } else {
    /* jpeg_read_raw_data hands out one iMCU row per call: v_samp * DCT_scaled_size rows of whole blocks per
     * component; the planes are collected padded to whole iMCU rows and blocks, then cropped */
    const int nc = cinfo.num_components;
    const int lines = cinfo.max_v_samp_factor * cinfo.min_DCT_scaled_size;
    size_t pw[4], ph[4], off[4], total = 0;
    int per_call[4];
    for (int c = 0; c < nc; c++) {
      const jpeg_component_info* ci = &cinfo.comp_info[c];
      pw[c] = (size_t)cinfo.MCUs_per_row * ci->MCU_width * ci->DCT_scaled_size;
      if (nc == 1) pw[c] = (size_t)ci->width_in_blocks * ci->DCT_scaled_size;
      per_call[c] = ci->v_samp_factor * ci->DCT_scaled_size;
      ph[c] = (size_t)cinfo.total_iMCU_rows * per_call[c];
      off[c] = total;
      total += pw[c] * ph[c];
    }
    tmp = (uint8_t*)calloc(total ? total : 1, 1);
    int max_rows = 0;
    for (int c = 0; c < nc; c++) max_rows += per_call[c];
    rows = (JSAMPROW*)malloc(sizeof(JSAMPROW) * (size_t)max_rows);
    JSAMPARRAY arr[4];
    for (unsigned r = 0; r < cinfo.total_iMCU_rows; r++) {
      JSAMPROW* p = rows;
      for (int c = 0; c < nc; c++) {
        arr[c] = p;
        for (int i = 0; i < per_call[c]; i++) *p++ = tmp + off[c] + ((size_t)r * per_call[c] + i) * pw[c];
      }
      jpeg_read_raw_data(&cinfo, arr, (JDIMENSION)lines);
    }
    uint8_t* o = out;
    for (int c = 0; c < nc; c++) {
      const jpeg_component_info* ci = &cinfo.comp_info[c];
      for (unsigned y = 0; y < ci->downsampled_height; y++, o += ci->downsampled_width)
        memcpy(o, tmp + off[c] + y * pw[c], ci->downsampled_width);
    }
  }
  jpeg_finish_decompress(&cinfo);
  info[15] = (int)err.pub.num_warnings;
  jpeg_destroy_decompress(&cinfo);
  free(tmp);
  free(rows);
  return 0;
}
