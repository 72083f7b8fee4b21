// Image effects of the editor API: host planning of a chain (effects.h) and k_effect_gather, the one pass per plane
// that carries it out.
#include "effects.h"

#include <algorithm>
#include <cstring>

#include "../../include/ultrahdr_api.h"

namespace uhdr_b200 {

// ---- kernel ----------------------------------------------------------------------------------------------------
// One CTA covers a 32 x 32 tile of the destination with 32 x 8 threads.
//  * no swap: a warp walks a destination row, so stores are coalesced; a source row is read along cols[], which is a
//    contiguous (crop), reversed (mirror) or strided (resize) run.
//  * swap: destination columns come from source rows.  The tile is read along source rows into shared memory and
//    written along destination rows, so both sides are coalesced; the 33-element pitch keeps the transposed read free
//    of bank conflicts for every element size.
template <typename T, bool SWAP>
__global__ void __launch_bounds__(256) k_effect_gather(const T* __restrict__ src, int ss, T* __restrict__ dst, int ds,
                                                       int w, int h, const int* __restrict__ cols,
                                                       const int* __restrict__ rows) {
  const int x0 = blockIdx.x * 32, y0 = blockIdx.y * 32, tx = threadIdx.x, ty = threadIdx.y;
  if (!SWAP) {
    const int x = x0 + tx;
    if (x >= w) return;
    const int c = cols[x];
    for (int r = ty; r < 32; r += 8) {
      const int y = y0 + r;
      if (y < h) dst[(size_t)y * ds + x] = src[(size_t)rows[y] * ss + c];
    }
  } else {
    __shared__ T tile[32][33];
    for (int i = ty; i < 32; i += 8) {   // tile[i][j]: destination (x0 + i, y0 + j) = source row cols[x], column rows[y]
      const int x = x0 + i, y = y0 + tx;
      if (x < w && y < h) tile[i][tx] = src[(size_t)cols[x] * ss + rows[y]];
    }
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
      const int x = x0 + tx, y = y0 + j;
      if (x < w && y < h) dst[(size_t)y * ds + x] = tile[tx][j];
    }
  }
}

template <typename T>
static cudaError_t launch_gather_t(const void* src, int ss, void* dst, int ds, int w, int h, const int* cols,
                                   const int* rows, bool swap, cudaStream_t s) {
  const dim3 grid((w + 31) / 32, (h + 31) / 32), block(32, 8);
  if (swap)
    k_effect_gather<T, true><<<grid, block, 0, s>>>((const T*)src, ss, (T*)dst, ds, w, h, cols, rows);
  else
    k_effect_gather<T, false><<<grid, block, 0, s>>>((const T*)src, ss, (T*)dst, ds, w, h, cols, rows);
  return cudaGetLastError();
}

// ---- one plane's chain ----------------------------------------------------------------------------------------
// cols / rows are v_[c_] / v_[1 - c_]: a rotation exchanges their roles without moving a vector, so the same chain
// planned again reuses the same capacities
void GatherPlan::reset(int w, int h) {
  w_ = w;
  h_ = h;
  c_ = 0;
  swap_ = false;
  v_[0].resize(w);
  v_[1].resize(h);
  for (int i = 0; i < w; i++) v_[0][i] = i;
  for (int i = 0; i < h; i++) v_[1][i] = i;
}

// rotate_buffer_clockwise / mirror_buffer (editorhelper.cpp:20-65), in destination coordinates
void GatherPlan::mirror(int direction) {
  std::vector<int>& t = direction == UHDR_MIRROR_VERTICAL ? rows() : cols();
  std::reverse(t.begin(), t.end());
}

void GatherPlan::rotate(int degrees) {
  if (degrees == 180) {
    std::reverse(cols().begin(), cols().end());
    std::reverse(rows().begin(), rows().end());
  } else {
    // 90: dst[i][j] = src[h - 1 - j][i]; 270: dst[i][j] = src[j][w - 1 - i]
    c_ = 1 - c_;
    swap_ = !swap_;
    std::swap(w_, h_);
    std::vector<int>& t = degrees == 90 ? cols() : rows();
    std::reverse(t.begin(), t.end());
  }
}

void GatherPlan::crop(int left, int top, int wd, int ht) {
  std::vector<int>& c = cols();
  std::vector<int>& r = rows();
  std::copy(c.begin() + left, c.begin() + left + wd, c.begin());
  std::copy(r.begin() + top, r.begin() + top + ht, r.begin());
  c.resize(wd);
  r.resize(ht);
  w_ = wd;
  h_ = ht;
}

// resize_buffer: dst[i][j] = src[i * (src_h / dst_h)][j * (src_w / dst_w)], integer ratios (0 when enlarging)
void GatherPlan::resize(int dw, int dh) {
  auto one = [this](std::vector<int>& t, int n, int dn) {
    const int ratio = n / dn;
    tmp_.resize(dn);
    for (int i = 0; i < dn; i++) tmp_[i] = t[(size_t)i * ratio];
    t.assign(tmp_.begin(), tmp_.end());
  };
  one(cols(), w_, dw);
  one(rows(), h_, dh);
  w_ = dw;
  h_ = dh;
}

int GatherPlan::launch(Workspace& ws, const void* src, int src_stride, int esz, void* dst, int dst_stride) const {
  const size_t n = (size_t)w_ + h_;
  int* h_tab = (int*)ws.halloc(n * sizeof(int));
  int* d_tab = (int*)ws.dalloc(n * sizeof(int));
  if (!h_tab || !d_tab) return E_MEM;
  memcpy(h_tab, cols().data(), (size_t)w_ * sizeof(int));
  memcpy(h_tab + w_, rows().data(), (size_t)h_ * sizeof(int));
  CUDA_TRY(cudaMemcpyAsync(d_tab, h_tab, n * sizeof(int), cudaMemcpyHostToDevice, ws.stream()));
  const int* c = d_tab;
  const int* r = d_tab + w_;
  cudaStream_t s = ws.stream();
  count_launches(1);
  switch (esz) {
    case 1: TIMED(ws, "effect_gather", (launch_gather_t<uint8_t>(src, src_stride, dst, dst_stride, w_, h_, c, r, swap_, s))); break;
    case 2: TIMED(ws, "effect_gather", (launch_gather_t<uint16_t>(src, src_stride, dst, dst_stride, w_, h_, c, r, swap_, s))); break;
    case 4: TIMED(ws, "effect_gather", (launch_gather_t<uint32_t>(src, src_stride, dst, dst_stride, w_, h_, c, r, swap_, s))); break;
    case 8: TIMED(ws, "effect_gather", (launch_gather_t<uint64_t>(src, src_stride, dst, dst_stride, w_, h_, c, r, swap_, s))); break;
    default: return fail(E_UNSUPPORTED, "no gather for %d-byte elements", esz);
  }
  return E_OK;
}

int gather_image(Workspace& ws, const DevImage& src, const GatherPlan& full, const GatherPlan* half, DevImage* out) {
  int rc = alloc_dev_image(ws, src.v.fmt, full.w(), full.h(), 64, out);
  if (rc) return rc;
  out->cg = src.cg;
  out->ct = src.ct;
  out->range = src.range;
  out->v.full_range = src.v.full_range;
  const int np = fmt_planes(src.v.fmt);
  for (int i = 0; i < np; i++) {
    int pw, ph, esz;
    fmt_plane_geom(src.v.fmt, src.v.w, src.v.h, i, &pw, &ph, &esz);
    int ss = src.v.stride[i], ds = out->v.stride[i];
    const bool sub = i > 0 && (src.v.fmt == F_P010 || src.v.fmt == F_YUV420);
    if (sub && !half) return fail(E_UNKNOWN, "no chroma plan for a subsampled image");
    if (src.v.fmt == F_P010 && i == 1) {  // interleaved U, V moved as one 4-byte element (apply_* use uint32_t)
      esz = 4;
      ss /= 2;
      ds /= 2;
    }
    const GatherPlan& p = sub ? *half : full;
    if (p.w() == 0 || p.h() == 0) continue;
    rc = p.launch(ws, src.v.p[i], ss, esz, (void*)out->v.p[i], ds);
    if (rc) return rc;
  }
  return E_OK;
}

// ---- the reference's checks ------------------------------------------------------------------------------------
void DecodeEffects::plan(const std::vector<Effect>& fx, int w, int h, int map_w, int map_h) {
  image.reset(w, h);
  map.reset(map_w, map_h);
  rc = E_OK;
  detail[0] = 0;
  auto bad = [this](const char* fmt, auto... v) {
    rc = E_INVALID_PARAM;
    snprintf(detail, sizeof detail, fmt, v...);
  };
  for (const Effect& e : fx) {
    if (e.kind == FX_ROTATE) {
      image.rotate(e.a);
      map.rotate(e.a);
    } else if (e.kind == FX_MIRROR) {
      image.mirror(e.a);
      map.mirror(e.a);
    } else if (e.kind == FX_CROP) {   // ultrahdr_api.cpp:326-387
      const int left = std::max(0, e.a), right = std::min(image.w(), e.b);
      if (right <= left)
        return bad("unexpected crop dimensions. crop right is <= crop left, after crop image width is %d", right - left);
      const int top = std::max(0, e.c), bottom = std::min(image.h(), e.d);
      if (bottom <= top)
        return bad("unexpected crop dimensions. crop bottom is <= crop top, after crop image height is %d", bottom - top);
      const float wd_ratio = (float)image.w() / map.w(), ht_ratio = (float)image.h() / map.h();
      const int gm_left = (int)(left / wd_ratio), gm_right = (int)(right / wd_ratio);
      if (gm_right <= gm_left)
        return bad("unexpected crop dimensions. crop right is <= crop left for gainmap image, after crop gainmap image "
                   "width is %d", gm_right - gm_left);
      const int gm_top = (int)(top / ht_ratio), gm_bottom = (int)(bottom / ht_ratio);
      if (gm_bottom <= gm_top)
        return bad("unexpected crop dimensions. crop bottom is <= crop top for gainmap image, after crop gainmap image "
                   "height is %d", gm_bottom - gm_top);
      image.crop(left, top, right - left, bottom - top);
      map.crop(gm_left, gm_top, gm_right - gm_left, gm_bottom - gm_top);
    } else {   // resize, :388-415
      const int dst_w = e.a, dst_h = e.b;
      const float wd_ratio = (float)image.w() / map.w(), ht_ratio = (float)image.h() / map.h();
      const int dst_gm_w = (int)(dst_w / wd_ratio), dst_gm_h = (int)(dst_h / ht_ratio);
      if (dst_w <= 0 || dst_h <= 0 || dst_gm_w <= 0 || dst_gm_h <= 0 || dst_w > 8192 || dst_h > 8192 ||
          dst_gm_w > 8192 || dst_gm_h > 8192)
        return bad("destination dimension must be in range (0, %d] x (0, %d]. dest image width is %d, dest image height "
                   "is %d, dest gainmap width is %d, dest gainmap height is %d", 8192, 8192, dst_w, dst_h, dst_gm_w,
                   dst_gm_h);
      image.resize(dst_w, dst_h);
      map.resize(dst_gm_w, dst_gm_h);
    }
  }
}

int EncodeEffects::plan(const std::vector<Effect>& fx, int w, int h, int hdr_fmt, int sdr_fmt) {
  const bool p010 = hdr_fmt == F_P010, yuv420 = sdr_fmt == F_YUV420;
  has_half = p010 || yuv420;
  full.reset(w, h);
  if (has_half) half.reset(w / 2, h / 2);   // P010 / YUV420 intents have even sizes: uhdr_enc_set_raw_image and the checks below
  for (const Effect& e : fx) {
    if (e.kind == FX_ROTATE) {
      full.rotate(e.a);
      if (has_half) half.rotate(e.a);
    } else if (e.kind == FX_MIRROR) {
      full.mirror(e.a);
      if (has_half) half.mirror(e.a);
    } else if (e.kind == FX_CROP) {   // ultrahdr_api.cpp:150-224
      const int left = std::max(0, e.a), right = std::min(full.w(), e.b), crop_width = right - left;
      if (crop_width <= 0)
        return fail(E_INVALID_PARAM, "unexpected crop dimensions. crop width is expected to be > 0, crop width is %d",
                    crop_width);
      if (crop_width % 2 != 0 && p010)
        return fail(E_INVALID_PARAM, "unexpected crop dimensions. crop width is expected to even for format "
                    "{UHDR_IMG_FMT_24bppYCbCrP010}, crop width is %d", crop_width);
      const int top = std::max(0, e.c), bottom = std::min(full.h(), e.d), crop_height = bottom - top;
      if (crop_height <= 0)
        return fail(E_INVALID_PARAM, "unexpected crop dimensions. crop height is expected to be > 0, crop height is %d",
                    crop_height);
      if (crop_height % 2 != 0 && p010)
        return fail(E_INVALID_PARAM, "unexpected crop dimensions. crop height is expected to even for format "
                    "{UHDR_IMG_FMT_24bppYCbCrP010}. crop height is %d", crop_height);
      if (crop_width % 2 != 0 && yuv420)
        return fail(E_INVALID_PARAM, "unexpected crop dimensions. crop width is expected to even for format "
                    "{UHDR_IMG_FMT_12bppYCbCr420}, crop width is %d", crop_width);
      if (crop_height % 2 != 0 && yuv420)
        return fail(E_INVALID_PARAM, "unexpected crop dimensions. crop height is expected to even for format "
                    "{UHDR_IMG_FMT_12bppYCbCr420}. crop height is %d", crop_height);
      full.crop(left, top, crop_width, crop_height);
      if (has_half) half.crop(left / 2, top / 2, crop_width / 2, crop_height / 2);
    } else {   // resize, :225-264
      const int dst_w = e.a, dst_h = e.b;
      if (dst_w <= 0 || dst_h <= 0 || dst_w > 8192 || dst_h > 8192)
        return fail(E_INVALID_PARAM, "destination dimensions must be in range (0, %d] x (0, %d]. dest image width is %d, "
                    "dest image height is %d", 8192, 8192, dst_w, dst_h);
      if ((dst_w % 2 != 0 || dst_h % 2 != 0) && p010)
        return fail(E_INVALID_PARAM, "destination dimensions cannot be odd for format {UHDR_IMG_FMT_24bppYCbCrP010}. "
                    "dest image width is %d, dest image height is %d", dst_w, dst_h);
      if ((dst_w % 2 != 0 || dst_h % 2 != 0) && yuv420)
        return fail(E_INVALID_PARAM, "destination dimensions cannot be odd for format {UHDR_IMG_FMT_12bppYCbCr420}. "
                    "dest image width is %d, dest image height is %d", dst_w, dst_h);
      full.resize(dst_w, dst_h);
      if (has_half) half.resize(dst_w / 2, dst_h / 2);
    }
  }
  return E_OK;
}

}  // namespace uhdr_b200
