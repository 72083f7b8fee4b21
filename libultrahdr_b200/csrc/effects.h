// The editor API's image effects (uhdr_add_effect_*, reference lib/src/editorhelper.cpp) as one index gather per
// plane.  Every effect is a pure index map: mirror and rotate permute pixels, crop takes a sub-rectangle and resize is
// nearest neighbour with an integer ratio (resize_buffer, editorhelper.cpp:78-86).  A chain therefore composes, on the
// host, into one axis-swap bit and two int32 tables: destination column x reads source axis value cols[x], destination
// row y reads rows[y]; without the swap those are a source column and a source row, with it a source row and a source
// column.  k_effect_gather (effects.cu) then moves each plane once, whatever the chain's length.
#pragma once
#include <vector>

#include "engine.h"

namespace uhdr_b200 {

enum : int { FX_MIRROR = 0, FX_ROTATE = 1, FX_CROP = 2, FX_RESIZE = 3 };

struct Effect {   // one uhdr_add_effect_* call, its arguments as given
  int kind;
  int a, b, c, d;   // mirror: a = direction; rotate: a = degrees; crop: left, right, top, bottom; resize: width, height
};

// One plane's composed chain.  The vectors keep their capacity across reset(), so a handle planning the same chain
// again does not touch the heap.
class GatherPlan {
 public:
  void reset(int w, int h);          // identity on a w x h plane
  int w() const { return w_; }
  int h() const { return h_; }
  void mirror(int direction);        // UHDR_MIRROR_VERTICAL / UHDR_MIRROR_HORIZONTAL
  void rotate(int degrees);          // clockwise, 90 / 180 / 270
  void crop(int left, int top, int wd, int ht);   // inside the current plane (the caller has clamped it)
  void resize(int dw, int dh);       // dw, dh > 0
  // enqueue the gather of `src` (elements of esz = 1, 2, 4 or 8 bytes, strides in elements) into dst, which holds
  // w() x h() elements; the tables go through the workspace's pinned and device arenas
  int launch(Workspace& ws, const void* src, int src_stride, int esz, void* dst, int dst_stride) const;

 private:
  std::vector<int>& cols() { return v_[c_]; }
  std::vector<int>& rows() { return v_[1 - c_]; }
  const std::vector<int>& cols() const { return v_[c_]; }
  const std::vector<int>& rows() const { return v_[1 - c_]; }
  std::vector<int> v_[2], tmp_;
  int c_ = 0, w_ = 0, h_ = 0;
  bool swap_ = false;
};

// An image through a plan: a new workspace image of the plan's size in the layout upload_image gives (strides aligned
// to 64 pixels, zero tails where the JPEG block stage reads them).  `half` plans the 2x2-subsampled chroma planes of
// P010 / YUV420 (the reference's apply_* run the same effect on w / 2 x h / 2 planes).
int gather_image(Workspace& ws, const DevImage& src, const GatherPlan& full, const GatherPlan* half, DevImage* out);

// uhdr_decode's chain over the output image and the decoded gain map (ultrahdr_api.cpp:289-429): sizes, checks and
// error details of the reference, planned before anything is decoded.  rc != E_OK: the code uhdr_decode returns once
// the decode itself succeeded, with `detail`.
struct DecodeEffects {
  GatherPlan image, map;
  int rc = 0;
  char detail[256] = {0};
  void plan(const std::vector<Effect>& fx, int w, int h, int map_w, int map_h);
};

// uhdr_encode's chain over the raw intents (ultrahdr_api.cpp:131-283): `full` for the full-size planes, `half` for
// the 4:2:0 chroma planes when an intent is P010 or YUV420.  Returns the code, the error detail set with fail().
struct EncodeEffects {
  GatherPlan full, half;
  bool has_half = false;
  int plan(const std::vector<Effect>& fx, int w, int h, int hdr_fmt, int sdr_fmt /* -1: no raw SDR intent */);
};

}  // namespace uhdr_b200
