// Test-only host wrapper around the OpenPose overlay's span generator (tokenhmr_b200/csrc/keypoints.cuh), so that the
// CPU suite can hold the very code the raster kernel runs against live cv2 without a GPU.
#include <stdint.h>

#include "../../tokenhmr_b200/csrc/keypoints.cuh"

namespace {
struct MaskEmit {
  uint8_t* mask;
  int W;
  void operator()(int y, int x0, int x1) const {
    for (int x = x0; x <= x1; ++x) mask[static_cast<long long>(y) * W + x] = 1;
  }
};
}  // namespace

// kind 0: cv2.line(p0, p1, thickness 2);  kind 1 / 2: cv2.circle(p0, radius 1, thickness kind).  Sets mask[y * W + x]
// (uint8 [H, W], caller-zeroed) to 1 on every pixel painted.  Returns 0, or -1 for a bad kind or size.
extern "C" __attribute__((visibility("default"))) int probe_pose_draw(int kind, long long x0, long long y0,
                                                                      long long x1, long long y1, int W, int H,
                                                                      uint8_t* mask) {
  if (!mask || W < 1 || H < 1) return -1;
  MaskEmit emit{mask, W};
  if (kind == 0)
    thmr::cv_line(W, H, x0, y0, x1, y1, emit);
  else if (kind == 1 || kind == 2)
    thmr::cv_circle(W, H, x0, y0, kind, emit);
  else
    return -1;
  return 0;
}
