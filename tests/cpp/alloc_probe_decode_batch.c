/* Heap-call probe for uhdr_b200_decode_batch_dev (alloc_probe.c's interposed malloc and counting, one more mode).
 *
 *   alloc_probe_decode_batch FILE     on a GPU: 8 copies of FILE decoded at 1/2 into device planes in one call, three
 *                                     warm-up calls, then three counted ones
 * prints "ours=<n> cuda=<n> other=<n>"; exit status 0 iff ours == 0.
 */
#define main alloc_probe_main
#include "alloc_probe.c"
#undef main

#include <cuda_runtime_api.h>

#define N 8

int main(int argc, char** argv) {
  void* warm[4];
  backtrace(warm, 4);
  if (argc != 2) { fprintf(stderr, "usage: alloc_probe_decode_batch file.jpg\n"); return 2; }
  dl_iterate_phdr(phdr_cb, NULL);
  if (!ours_hi) { fprintf(stderr, "libuhdr_b200.so not found among the loaded objects\n"); return 2; }
  size_t n;
  unsigned char* data = slurp(argv[1], &n);
  unsigned w, h, gw, gh;
  if (uhdr_b200_scaled_dims(data, n, 2, &w, &h, &gw, &gh)) { fprintf(stderr, "scaled_dims failed\n"); return 2; }
  uhdr_raw_image_t dest[N], map[N];
  uhdr_gainmap_metadata_t md[N];
  uhdr_b200_decode_item_t items[N];
  for (int i = 0; i < N; i++) {
    memset(&dest[i], 0, sizeof dest[i]);
    memset(&map[i], 0, sizeof map[i]);
    dest[i].fmt = UHDR_IMG_FMT_64bppRGBAHalfFloat;
    dest[i].w = w; dest[i].h = h; dest[i].stride[0] = w;
    map[i].w = gw; map[i].h = gh; map[i].stride[0] = gw;
    if (cudaMalloc(&dest[i].planes[0], (size_t)w * h * 8) || cudaMalloc(&map[i].planes[0], (size_t)gw * gh * 4)) return 2;
    items[i].data = data; items[i].size = n;
    items[i].dest_dev = &dest[i]; items[i].gainmap_dev = &map[i]; items[i].metadata_out = &md[i];
  }
  for (int it = 0; it < 6; it++) {   /* three warm-up iterations, three counted */
    armed = it >= 3;
    const int rc = uhdr_b200_decode_batch_dev(items, N, 2, UHDR_CT_LINEAR, 4.0f, NULL);
    armed = 0;
    if (rc) { fprintf(stderr, "decode_batch_dev failed: %s\n", uhdr_b200_last_error()); return 2; }
    cudaDeviceSynchronize();
  }
  return report("uhdr_b200_decode_batch_dev, 8 files at 1/2");
}
