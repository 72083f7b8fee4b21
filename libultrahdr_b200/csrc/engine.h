// Host orchestration of the device stages: the CUDA counterpart of the reference's
// UltraHdr::{generateGainMap, applyGainMap, toneMap, convertYuv} members
// (lib/include/ultrahdr/ultrahdrcommon.h:471-546, bodies in lib/src/jpegr.cpp).  All functions
// enqueue on the workspace stream and return without synchronising unless stated.
#pragma once
#include "../../include/uhdr_b200.h"
#include "kernels.cuh"
#include "runtime.h"
#include "tables.h"

namespace uhdr_b200 {

struct DevImage {  // a uhdr_raw_image_t whose planes live in device memory
  ImgView v;
  int cg, ct, range;
};

int fmt_planes(int fmt);
inline bool fmt_is_rgb_host(int f) { return f == F_RGBAF16 || f == F_RGBA8888 || f == F_RGBA1010102; }
// elements per row (w or chroma width), rows and element size of plane `i`
void fmt_plane_geom(int fmt, int w, int h, int i, int* pw, int* ph, int* esz);

int alloc_dev_image(Workspace& ws, int fmt, int w, int h, int stride_align, DevImage* out);
// a copy of `src` in workspace memory: strides aligned to 64 pixels, the bytes past each row's width zero.
// kind = cudaMemcpyDeviceToDevice stages a caller's device image the same way.
int upload_image(Workspace& ws, const uhdr_raw_image_t& src, DevImage* out,
                 cudaMemcpyKind kind = cudaMemcpyHostToDevice);
int download_image(Workspace& ws, const DevImage& src, uhdr_raw_image_t* dst);

struct GainmapJob {      // state between enqueue and metadata finish
  DevImage map{};        // RGB888 / Y400 in device memory, stride = map_w aligned to `map_align`; planes preset by the caller = destination
  int nch = 0, onepass = 0;
  float hdr_white_nits = 0, gamma = 1;
  float target_nits = -1;
  int use_base_cg = 1;
  float* h_minmax = nullptr;  // pinned, 6 floats (two-pass)
  unsigned* exact_word = nullptr;      // pinned; k_affine_q: values that took the fp64 log2 (null: other kernels ran)
  unsigned long long values = 0;       // map_w * map_h * channels of that run
};
// map_align: stride alignment of the produced map in pixels (reference allocates with 64)
int generate_gainmap_dev(Workspace& ws, const DevImage& sdr, const DevImage& hdr,
                         const uhdr_b200_gm_config_t& cfg, int map_align, GainmapJob* job);
// after the stream has been synchronised: fill the metadata (jpegr.cpp:724-734, 1031-1048)
void finish_gainmap_metadata(const GainmapJob& job, uhdr_gainmap_metadata_t* md);
// two-pass fast path since process start: [0] gain values quantised by k_affine_q, [1] of those through the fp64 log2
void gainmap_affine_stats(unsigned long long out[2]);

int apply_gainmap_dev(Workspace& ws, const DevImage& sdr, const DevImage& map,
                      const uhdr_gainmap_metadata_t& md, int out_ct, float max_display_boost,
                      DevImage* dst /* allocated by caller, fmt F16 / 1010102 */);
// A rectangle of the image: dst->v.w x dst->v.h pixels starting at (ox, oy), w / h being the same.
struct ApplyRegion { int ox, oy, w, h; };
// apply_gainmap_dev on `stream`, with the LUT blob `luts`, of `region` (null: the whole image).  h_tab / d_tab: pinned
// and device blocks of apply_table_floats(sdr, map) floats for the per-call tables, or null to take them from *ws.  ws
// null: nothing is timed, and a map whose aspect ratio differs from sdr's is an error (resize it first).
int apply_gainmap_region(Workspace* ws, cudaStream_t stream, const float* luts, const DevImage& sdr,
                         const DevImage& map, const uhdr_gainmap_metadata_t& md, int out_ct,
                         float max_display_boost, DevImage* dst, const ApplyRegion* region, float* h_tab,
                         float* d_tab);
size_t apply_table_floats(const DevImage& sdr, const DevImage& map);
// applyGainMap's aspect-ratio check (jpegr.cpp:1652-1671): the map is resized to w x h first
bool map_needs_resize(int w, int h, int map_w, int map_h);
// resize_image of the map to w x h into rs (rs->v.p[0] null: allocated from ws, stride aligned to 64), on ws.stream()
int resize_map_dev(Workspace& ws, const DevImage& map, int w, int h, DevImage* rs);
// apply_gainmap_dev launches since process start: [0] k_apply_lin1, [1] k_apply_fast, [2] k_apply_gainmap, [3] k_resize_map
void apply_route_stats(unsigned long long out[4]);
int tonemap_dev(Workspace& ws, const DevImage& hdr, DevImage* sdr /* allocated by caller */);
// in_place = false: the result goes to workspace scratch and *img is redirected to it (the source stays intact)
int convert_yuv_dev(Workspace& ws, DevImage* img, int src_cg, int dst_cg, bool in_place = true);
// convert_raw_input_to_ycbcr for RGBA8888 / RGB888 (gainmapmath.cpp:1440-1467): new YCbCr 4:4:4 device image
int rgb_to_ycbcr_dev(Workspace& ws, const DevImage& rgb, DevImage* out);

}  // namespace uhdr_b200
