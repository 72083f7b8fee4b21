/* Heap-call probe for uhdr_b200_transcode_ladder (alloc_probe.c's interposed malloc and counting, one more mode).
 *
 *   alloc_probe_transcode_ladder FILE    on a GPU: FILE transcoded into a five-rung ladder (k = 1 at two qualities,
 *                                        2, 4 and 8), three warm-up calls, then three counted ones, the last of them
 *                                        with a smaller ladder (the first three rungs)
 * prints "ours=<n> cuda=<n> other=<n>"; exit status 0 iff ours == 0.
 */
#define main alloc_probe_main
#include "alloc_probe.c"
#undef main

#define N 5

int main(int argc, char** argv) {
  void* warm[4];
  backtrace(warm, 4);
  if (argc != 2) { fprintf(stderr, "usage: alloc_probe_transcode_ladder file.jpg\n"); return 2; }
  dl_iterate_phdr(phdr_cb, NULL);
  if (!ours_hi) { fprintf(stderr, "libuhdr_b200.so not found among the loaded objects\n"); return 2; }
  size_t n;
  unsigned char* data = slurp(argv[1], &n);
  const size_t cap = 2 * n + (1 << 20);
  static unsigned char out[N][4 << 20];
  if (cap > sizeof out[0]) { fprintf(stderr, "file too large for the probe\n"); return 2; }
  const uhdr_b200_transcode_config_t cfgs[N] = {{1, 85, 85, 0, 1}, {1, 60, 90, 1, 0}, {2, 80, 70, 1, 1}, {4, 80, 70, 1, 1},
                                                {8, 80, 70, 0, 0}};
  uhdr_b200_transcode_rung_t rungs[N];
  for (int i = 0; i < N; i++) {
    rungs[i].cfg = cfgs[i];
    rungs[i].out = out[i];
    rungs[i].cap = cap;
  }
  for (int it = 0; it < 6; it++) {   /* three warm-up iterations, three counted */
    armed = it >= 3;
    const int rc = uhdr_b200_transcode_ladder(data, n, rungs, it == 5 ? 3 : N);
    armed = 0;
    if (rc) { fprintf(stderr, "transcode_ladder failed: %s\n", uhdr_b200_last_error()); return 2; }
  }
  return report("uhdr_b200_transcode_ladder, five rungs, then three");
}
