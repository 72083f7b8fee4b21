/* Heap-call probe for uhdr_b200_transcode_batch (alloc_probe.c's interposed malloc and counting, one more mode).
 *
 *   alloc_probe_transcode_batch FILE     on a GPU: 8 copies of FILE transcoded at 1/2 in one call, three warm-up calls,
 *                                        then three counted ones
 * prints "ours=<n> cuda=<n> other=<n>"; exit status 0 iff ours == 0.
 */
#define main alloc_probe_main
#include "alloc_probe.c"
#undef main

#define N 8

int main(int argc, char** argv) {
  void* warm[4];
  backtrace(warm, 4);
  if (argc != 2) { fprintf(stderr, "usage: alloc_probe_transcode_batch file.jpg\n"); return 2; }
  dl_iterate_phdr(phdr_cb, NULL);
  if (!ours_hi) { fprintf(stderr, "libuhdr_b200.so not found among the loaded objects\n"); return 2; }
  size_t n;
  unsigned char* data = slurp(argv[1], &n);
  const size_t cap = 2 * n + (1 << 20);
  uhdr_b200_transcode_item_t items[N];
  static unsigned char out[N][4 << 20];
  if (cap > sizeof out[0]) { fprintf(stderr, "file too large for the probe\n"); return 2; }
  uhdr_b200_transcode_config_t cfg = {2, 80, 70, 1, 1};
  for (int i = 0; i < N; i++) {
    items[i].data = data; items[i].size = n;
    items[i].out = out[i]; items[i].cap = cap;
  }
  for (int it = 0; it < 6; it++) {   /* three warm-up iterations, three counted */
    armed = it >= 3;
    const int rc = uhdr_b200_transcode_batch(items, N, &cfg);
    armed = 0;
    if (rc) { fprintf(stderr, "transcode_batch failed: %s\n", uhdr_b200_last_error()); return 2; }
  }
  return report("uhdr_b200_transcode_batch, 8 files at 1/2");
}
