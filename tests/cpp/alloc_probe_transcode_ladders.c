/* Heap-call probe for uhdr_b200_transcode_ladders (alloc_probe.c's interposed malloc and counting, one more mode).
 *
 *   alloc_probe_transcode_ladders A B    on a GPU: four files (A, B, A, B), each with its own ladder of up to five rungs
 *                                        (k = 1 at two qualities, 2, 4 and 8), three warm-up calls, then three counted
 *                                        ones, the last of them with a smaller shape (three files, three rungs each)
 * prints "ours=<n> cuda=<n> other=<n>"; exit status 0 iff ours == 0.
 */
#define main alloc_probe_main
#include "alloc_probe.c"
#undef main

#define F 4
#define N 5

int main(int argc, char** argv) {
  void* warm[4];
  backtrace(warm, 4);
  if (argc != 3) { fprintf(stderr, "usage: alloc_probe_transcode_ladders a.jpg b.jpg\n"); return 2; }
  dl_iterate_phdr(phdr_cb, NULL);
  if (!ours_hi) { fprintf(stderr, "libuhdr_b200.so not found among the loaded objects\n"); return 2; }
  size_t sz[2];
  unsigned char* data[2] = {slurp(argv[1], &sz[0]), slurp(argv[2], &sz[1])};
  static unsigned char out[F][N][4 << 20];
  const uhdr_b200_transcode_config_t cfgs[N] = {{1, 85, 85, 0, 1}, {1, 60, 90, 1, 0}, {2, 80, 70, 1, 1}, {4, 80, 70, 1, 1},
                                                {8, 80, 70, 0, 0}};
  uhdr_b200_transcode_rung_t rungs[F][N];
  uhdr_b200_transcode_file_t files[F];
  for (int f = 0; f < F; f++) {
    const size_t cap = 2 * sz[f & 1] + (1 << 20);
    if (cap > sizeof out[0][0]) { fprintf(stderr, "file too large for the probe\n"); return 2; }
    for (int i = 0; i < N; i++) {
      rungs[f][i].cfg = cfgs[(i + f) % N];   /* every file its own ladder */
      rungs[f][i].out = out[f][i];
      rungs[f][i].cap = cap;
    }
    files[f].data = data[f & 1];
    files[f].size = sz[f & 1];
    files[f].rungs = rungs[f];
  }
  for (int it = 0; it < 6; it++) {   /* three warm-up iterations, three counted */
    for (int f = 0; f < F; f++) files[f].n = it == 5 ? 3 : N - (f & 1);
    armed = it >= 3;
    const int rc = uhdr_b200_transcode_ladders(files, it == 5 ? 3 : F);
    armed = 0;
    if (rc) { fprintf(stderr, "transcode_ladders failed: %s\n", uhdr_b200_last_error()); return 2; }
  }
  return report("uhdr_b200_transcode_ladders, four files of five and four rungs, then three of three");
}
