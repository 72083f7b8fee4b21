/* Heap-call probe of the editor effects (uhdr_add_effect_*): alloc_probe.c's counting malloc, driven through
 *
 *   alloc_probe_effects W H   on a GPU: reset + set_raw_image x2 + five effects + uhdr_encode (API-1, P010 + 4:2:0),
 *                             then reset + set_image + five effects + uhdr_decode + both images fetched, on warmed handles
 *
 * prints "ours=<n> cuda=<n> other=<n>" per phase; exit status 0 iff ours == 0 everywhere.
 */
#define main alloc_probe_main
#include "alloc_probe.c"
#undef main

static void add_chain(uhdr_codec_private_t* h, int w, int hgt) {
  CHECK(uhdr_add_effect_crop(h, 2, w - 6, 4, hgt - 2));
  CHECK(uhdr_add_effect_rotate(h, 90));
  CHECK(uhdr_add_effect_mirror(h, UHDR_MIRROR_HORIZONTAL));
  CHECK(uhdr_add_effect_resize(h, hgt / 2, w / 2));
  CHECK(uhdr_add_effect_rotate(h, 180));
}

static int run_effects(int w, int h) {
  const size_t npx = (size_t)w * h;
  uint16_t* p010 = (uint16_t*)__libc_malloc(npx * 3);
  uint8_t* yuv = (uint8_t*)__libc_malloc(npx * 3 / 2);
  uint32_t s = 777;
  for (size_t i = 0; i < npx * 3 / 2; i++) {
    s = s * 1664525u + 1013904223u;
    p010[i] = (uint16_t)((64 + (s >> 22) % 876) << 6);
    yuv[i] = (uint8_t)(s >> 24);
  }
  uhdr_raw_image_t hdr, sdr;
  memset(&hdr, 0, sizeof hdr);
  memset(&sdr, 0, sizeof sdr);
  hdr.fmt = UHDR_IMG_FMT_24bppYCbCrP010; hdr.cg = UHDR_CG_BT_2100; hdr.ct = UHDR_CT_HLG; hdr.range = UHDR_CR_LIMITED_RANGE;
  hdr.w = w; hdr.h = h; hdr.planes[0] = p010; hdr.planes[1] = p010 + npx; hdr.stride[0] = w; hdr.stride[1] = w;
  sdr.fmt = UHDR_IMG_FMT_12bppYCbCr420; sdr.cg = UHDR_CG_BT_709; sdr.ct = UHDR_CT_SRGB; sdr.range = UHDR_CR_FULL_RANGE;
  sdr.w = w; sdr.h = h; sdr.planes[0] = yuv; sdr.planes[1] = yuv + npx; sdr.planes[2] = yuv + npx + npx / 4;
  sdr.stride[0] = w; sdr.stride[1] = sdr.stride[2] = w / 2;
  int bad = 0;
  uhdr_codec_private_t* enc = uhdr_create_encoder();
  for (int it = 0; it < 6; it++) {
    armed = it >= 3 || count_warmup;
    uhdr_reset_encoder(enc);
    CHECK(uhdr_enc_set_raw_image(enc, &hdr, UHDR_HDR_IMG));
    CHECK(uhdr_enc_set_raw_image(enc, &sdr, UHDR_SDR_IMG));
    add_chain(enc, w, h);
    CHECK(uhdr_encode(enc));
    if (!uhdr_get_encoded_stream(enc)) exit(2);
    armed = 0;
  }
  bad |= report("api-1 reset + set_raw_image x2 + 5 effects + encode");
  /* decode a file without effects, so that the decoder's chain starts from the full size */
  uhdr_reset_encoder(enc);
  CHECK(uhdr_enc_set_raw_image(enc, &hdr, UHDR_HDR_IMG));
  CHECK(uhdr_enc_set_raw_image(enc, &sdr, UHDR_SDR_IMG));
  CHECK(uhdr_encode(enc));
  uhdr_compressed_image_t* out = uhdr_get_encoded_stream(enc);
  uhdr_codec_private_t* dec = uhdr_create_decoder();
  for (int it = 0; it < 6; it++) {
    armed = it >= 3 || count_warmup;
    uhdr_reset_decoder(dec);
    CHECK(uhdr_dec_set_image(dec, out));
    add_chain(dec, w, h);
    CHECK(uhdr_decode(dec));
    if (!uhdr_get_decoded_image(dec) || !uhdr_get_decoded_gainmap_image(dec)) exit(2);
    armed = 0;
  }
  bad |= report("reset + set_image + 5 effects + uhdr_decode");
  uhdr_release_decoder(dec);
  uhdr_release_encoder(enc);
  return bad;
}

int main(int argc, char** argv) {
  void* warm[4];
  count_warmup = getenv("ALLOC_PROBE_COUNT_WARMUP") != NULL;
  backtrace(warm, 4);
  if (argc != 3) { fprintf(stderr, "usage: alloc_probe_effects W H\n"); return 2; }
  uhdr_codec_private_t* tmp = uhdr_create_decoder();
  uhdr_release_decoder(tmp);
  dl_iterate_phdr(phdr_cb, NULL);
  const int bad = run_effects(atoi(argv[1]), atoi(argv[2]));
  if (!ours_hi) { fprintf(stderr, "libuhdr_b200.so not found among the loaded objects\n"); return 2; }
  return bad ? 1 : 0;
}
