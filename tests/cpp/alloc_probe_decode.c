/* Heap-call probe for uhdr_decode of a JPEG/R file (alloc_probe.c's interposed malloc and counting, one more mode).
 *
 *   alloc_probe_decode FILE     on a GPU: reset + set_image + uhdr_decode of FILE on a warmed decoder, then the
 *                               entropy decoder's scan counts over the counted iterations
 * prints "ours=<n> cuda=<n> other=<n>" and "device_scans=<n> handed_back=<n>"; exit status 0 iff ours == 0.
 */
#define main alloc_probe_main
#include "alloc_probe.c"
#undef main

int main(int argc, char** argv) {
  void* warm[4];
  backtrace(warm, 4);
  if (argc != 2) { fprintf(stderr, "usage: alloc_probe_decode file.jpg\n"); return 2; }
  uhdr_codec_private_t* dec = uhdr_create_decoder();
  dl_iterate_phdr(phdr_cb, NULL);
  if (!ours_hi) { fprintf(stderr, "libuhdr_b200.so not found among the loaded objects\n"); return 2; }
  size_t n;
  unsigned char* data = slurp(argv[1], &n);
  uhdr_compressed_image_t in = {data, n, n, UHDR_CG_UNSPECIFIED, UHDR_CT_UNSPECIFIED, UHDR_CR_UNSPECIFIED};
  unsigned long long s0[3], s1[3];
  for (int it = 0; it < 6; it++) {   /* three warm-up iterations, three counted */
    if (it == 3) uhdr_b200_entropy_decoder_stats(s0);
    armed = it >= 3;
    uhdr_reset_decoder(dec);
    CHECK(uhdr_dec_set_image(dec, &in));
    CHECK(uhdr_decode(dec));
    if (!uhdr_get_decoded_image(dec)) exit(2);
    armed = 0;
  }
  uhdr_b200_entropy_decoder_stats(s1);
  const int bad = report("reset + set_image + uhdr_decode (file)");
  printf("device_scans=%llu handed_back=%llu\n", s1[0] - s0[0], s1[1] - s0[1]);
  uhdr_release_decoder(dec);
  return bad;
}
