// OpenPose skeleton overlays and the prediction grid behind tokenhmr_b200.render.MeshRenderer (the reference's
// MeshRenderer.visualize_tensorboard, tokenhmr/lib/utils/mesh_renderer.py:70-107, drawing with
// lib/utils/render_openpose.py).  Contract: DESIGN.md §2 "Rendering".
//
// The overlay is bit for bit what render_openpose paints with OpenCV 4.x on 255 * crop, divided by 255.  Below about
// 11 700 px of width its thickness formula always gives lines of thickness 2 and circles of radius 1, so three cv2
// primitives are enough, each restated here as the scanline spans it paints (span generator, __host__ __device__ so
// that the test probe can hold it against live cv2 on the CPU):
//   cv_line       cv2.line(.., 2, LINE_8): clipLine to the image grown by 2 px, then ThickLine -- a convex quad in
//                 16-bit fixed point (FillConvexPoly over its Line2 outline) plus a filled radius-1 Circle at each end
//   cv_circle(2)  cv2.circle(.., 1, .., 2): EllipseEx -- a 5-point polyline of thickness-2 ThickLines
//   cv_circle(1)  cv2.circle(.., 1, .., 1): the midpoint Circle, unfilled
//
// Stages, all stream-ordered, no host synchronisation and no allocation (CUDA-graph capturable):
//   keys     cudaMemsetAsync to 0
//   raster   one thread per (sample, keypoint set, primitive): the image's setup (scaling, keypoint_matches,
//            validity, rectangle, circle thickness) in the reference's float32 arithmetic, then every pixel of the
//            primitive's spans does atomicMax(key, primitive + 1).  Limbs come first in pair order, joints after, so
//            the largest key is the primitive cv2 drew last: "last drawn wins" whatever the scheduling.
//   grid     one thread per grid pixel: the make_grid layout (pad 0), the crop, the two mesh tiles, and the skeleton
//            tiles: the winning primitive's colour / 255 or the background fl32(fl32(255 x) / 255).
#pragma once
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace thmr {

constexpr int kPoseKeypoints = 44;   // pred_keypoints_2d / keypoints_2d: 25 OpenPose body + 19 extra joints
constexpr int kPoseBody = 25;
constexpr int kPoseExtra = 19;
constexpr int kPoseLimbs = 24;
constexpr int kPosePrims = kPoseLimbs + kPoseBody;   // draw order: limbs, then joints
constexpr int kPoseMaxWidth = 11718;  // widest image whose thickness formula still yields line 2 / radius 1
constexpr int kXYShift = 16;
constexpr int64_t kXYOne = int64_t(1) << kXYShift;

__host__ __device__ __forceinline__ int64_t cv_round(double x) {   // cvRound: round half to even
#ifdef __CUDA_ARCH__
  return __double2ll_rn(x);
#else
  return static_cast<int64_t>(nearbyint(x));
#endif
}
// products, sums and quotients exactly as OpenCV's compiled code rounds them (no contraction into FMA)
__host__ __device__ __forceinline__ double dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

// clipLine(Size2l(W, H), p1, p2): false when the segment misses [0, W) x [0, H).
__host__ __device__ inline bool cv_clip_line(int64_t W, int64_t H, int64_t& x1, int64_t& y1, int64_t& x2,
                                             int64_t& y2) {
  const int64_t right = W - 1, bottom = H - 1;
  int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
  int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
  if ((c1 & c2) == 0 && (c1 | c2) != 0) {
    int64_t a;
    if (c1 & 12) {
      a = c1 < 8 ? 0 : bottom;
      x1 += static_cast<int64_t>(dmul(static_cast<double>(a - y1), static_cast<double>(x2 - x1)) /
                                 static_cast<double>(y2 - y1));
      y1 = a;
      c1 = (x1 < 0) + (x1 > right) * 2;
    }
    if (c2 & 12) {
      a = c2 < 8 ? 0 : bottom;
      x2 += static_cast<int64_t>(dmul(static_cast<double>(a - y2), static_cast<double>(x2 - x1)) /
                                 static_cast<double>(y2 - y1));
      y2 = a;
      c2 = (x2 < 0) + (x2 > right) * 2;
    }
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
      if (c1) {
        a = c1 == 1 ? 0 : right;
        y1 += static_cast<int64_t>(dmul(static_cast<double>(a - x1), static_cast<double>(y2 - y1)) /
                                   static_cast<double>(x2 - x1));
        x1 = a;
        c1 = 0;
      }
      if (c2) {
        a = c2 == 1 ? 0 : right;
        y2 += static_cast<int64_t>(dmul(static_cast<double>(a - x2), static_cast<double>(y2 - y1)) /
                                   static_cast<double>(x2 - x1));
        x2 = a;
        c2 = 0;
      }
    }
  }
  return (c1 | c2) == 0;
}

// Line2: the 8-connected outline of one fixed-point polygon edge, both ends included, clipped to the image.
template <class Emit>
__host__ __device__ void cv_line2(int W, int H, int64_t x1, int64_t y1, int64_t x2, int64_t y2, Emit& emit) {
  if (!cv_clip_line(static_cast<int64_t>(W) << kXYShift, static_cast<int64_t>(H) << kXYShift, x1, y1, x2, y2)) return;
  int64_t dx = x2 - x1, dy = y2 - y1;
  const int64_t ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
  int64_t step = 0;
  int64_t ecount;
  const bool xmajor = ax > ay;
  if (xmajor) {
    if (dx < 0) { int64_t t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dy = -dy; }
    step = dy * kXYOne / (ax | 1);
    ecount = (x2 - x1) >> kXYShift;
  } else {
    if (dy < 0) { int64_t t = x1; x1 = x2; x2 = t; t = y1; y1 = y2; y2 = t; dx = -dx; }
    step = dx * kXYOne / (ay | 1);
    ecount = (y2 - y1) >> kXYShift;
  }
  x1 += kXYOne >> 1;
  y1 += kXYOne >> 1;
  auto put = [&](int64_t x, int64_t y) {
    if (x >= 0 && x < W && y >= 0 && y < H) emit(static_cast<int>(y), static_cast<int>(x), static_cast<int>(x));
  };
  put((x2 + (kXYOne >> 1)) >> kXYShift, (y2 + (kXYOne >> 1)) >> kXYShift);
  if (xmajor) {
    x1 >>= kXYShift;
    for (; ecount >= 0; --ecount, ++x1, y1 += step) put(x1, y1 >> kXYShift);
  } else {
    y1 >>= kXYShift;
    for (; ecount >= 0; --ecount, ++y1, x1 += step) put(x1 >> kXYShift, y1);
  }
}

// FillConvexPoly(.., LINE_8, XY_SHIFT) of a fixed-point quad: the outline, then one span per scanline.  Rows above
// the image are skipped in one step per edge (x advances by exactly dx per row), which paints what cv2's row-by-row
// walk paints.
template <class Emit>
__host__ __device__ void cv_fill_quad(int W, int H, const int64_t (&vx)[4], const int64_t (&vy)[4], Emit& emit) {
  constexpr int n = 4;
  const int64_t delta = kXYOne >> 1;
  int64_t xmin = vx[0], xmax = vx[0], ymin = vy[0], ymax = vy[0];
  int imin = 0;
  for (int i = 0, j = n - 1; i < n; j = i++) {
    if (vy[i] < ymin) { ymin = vy[i]; imin = i; }
    ymax = vy[i] > ymax ? vy[i] : ymax;
    xmax = vx[i] > xmax ? vx[i] : xmax;
    xmin = vx[i] < xmin ? vx[i] : xmin;
    cv_line2(W, H, vx[j], vy[j], vx[i], vy[i], emit);
  }
  xmin = (xmin + delta) >> kXYShift; xmax = (xmax + delta) >> kXYShift;
  ymin = (ymin + delta) >> kXYShift; ymax = (ymax + delta) >> kXYShift;
  if (xmax < 0 || ymax < 0 || xmin >= W || ymin >= H) return;
  if (ymax > H - 1) ymax = H - 1;
  int eidx[2] = {imin, imin}, edi[2] = {1, n - 1};
  int64_t ex[2] = {-kXYOne, -kXYOne}, edx[2] = {0, 0}, eye[2] = {ymin, ymin};
  int edges = n;
  int64_t y = ymin;
  for (;;) {
    for (int i = 0; i < 2; ++i) {
      if (y < eye[i]) continue;
      int idx0 = eidx[i], idx = idx0 + edi[i];
      if (idx >= n) idx -= n;
      for (; edges-- > 0;) {
        const int64_t ty = (vy[idx] + delta) >> kXYShift;
        if (ty > y) {
          eye[i] = ty;
          edx[i] = ((vx[idx] - vx[idx0]) * 2 + (ty - y)) / (2 * (ty - y));
          ex[i] = vx[idx0];
          eidx[i] = idx;
          break;
        }
        idx0 = idx;
        idx += edi[i];
        if (idx >= n) idx -= n;
      }
    }
    if (edges < 0) break;
    if (y < 0) {   // jump to the next edge change or row 0, whichever comes first
      int64_t next = eye[0] < eye[1] ? eye[0] : eye[1];
      if (next > 0 || next <= y) next = 0;
      const int64_t k = next - y;
      ex[0] += edx[0] * k; ex[1] += edx[1] * k;
      y = next;
      if (y > ymax) break;
      continue;
    }
    const int l = ex[0] > ex[1] ? 1 : 0;
    const int64_t xx1 = (ex[l] + delta) >> kXYShift, xx2 = (ex[1 - l] + delta) >> kXYShift;
    if (xx2 >= 0 && xx1 < W)
      emit(static_cast<int>(y), static_cast<int>(xx1 < 0 ? 0 : xx1), static_cast<int>(xx2 >= W ? W - 1 : xx2));
    ex[0] += edx[0]; ex[1] += edx[1];
    if (++y > ymax) break;
  }
}

// Circle(img, c, 1, color, fill): the plus sign (filled) or its four arms (unfilled), clipped.
template <class Emit>
__host__ __device__ void cv_circle_r1(int W, int H, int64_t cx, int64_t cy, bool fill, Emit& emit) {
  if (cy >= 0 && cy < H) {
    if (fill) {
      const int64_t a = cx - 1 < 0 ? 0 : cx - 1, b = cx + 1 > W - 1 ? W - 1 : cx + 1;
      if (a <= b) emit(static_cast<int>(cy), static_cast<int>(a), static_cast<int>(b));
    } else {
      if (cx - 1 >= 0 && cx - 1 < W) emit(static_cast<int>(cy), static_cast<int>(cx - 1), static_cast<int>(cx - 1));
      if (cx + 1 >= 0 && cx + 1 < W) emit(static_cast<int>(cy), static_cast<int>(cx + 1), static_cast<int>(cx + 1));
    }
  }
  if (cx >= 0 && cx < W) {
    if (cy - 1 >= 0 && cy - 1 < H) emit(static_cast<int>(cy - 1), static_cast<int>(cx), static_cast<int>(cx));
    if (cy + 1 >= 0 && cy + 1 < H) emit(static_cast<int>(cy + 1), static_cast<int>(cx), static_cast<int>(cx));
  }
}

// ThickLine(.., thickness 2, LINE_8, flags, XY_SHIFT) between fixed-point points; flags bit 0 / 1 draw the cap at
// the first / second end.
template <class Emit>
__host__ __device__ void cv_thick_line(int W, int H, int64_t x0, int64_t y0, int64_t x1, int64_t y1, int flags,
                                       Emit& emit) {
  const double inv_one = 1.0 / static_cast<double>(kXYOne);
  const double dx = dmul(static_cast<double>(x0 - x1), inv_one), dy = dmul(static_cast<double>(y1 - y0), inv_one);
  double r = dadd(dmul(dx, dx), dmul(dy, dy));
  if (fabs(r) > 2.220446049250313e-16) {   // DBL_EPSILON
    r = static_cast<double>(kXYOne) / sqrt(r);   // (thickness 2 << 15) / |d|
    const int64_t dpx = cv_round(dmul(dy, r)), dpy = cv_round(dmul(dx, r));
    const int64_t qx[4] = {x0 + dpx, x0 - dpx, x1 - dpx, x1 + dpx};
    const int64_t qy[4] = {y0 + dpy, y0 - dpy, y1 - dpy, y1 + dpy};
    cv_fill_quad(W, H, qx, qy, emit);
  }
  if (flags & 1) cv_circle_r1(W, H, (x0 + (kXYOne >> 1)) >> kXYShift, (y0 + (kXYOne >> 1)) >> kXYShift, true, emit);
  if (flags & 2) cv_circle_r1(W, H, (x1 + (kXYOne >> 1)) >> kXYShift, (y1 + (kXYOne >> 1)) >> kXYShift, true, emit);
}

// cv2.line(img, p0, p1, color, 2, LINE_8, 0).  cv2.line first clips the segment, in whole pixels, to the image grown
// by the thickness on every side (clipLine on Rect(-2, -2, W + 4, H + 4)) and draws nothing when it misses it.
template <class Emit>
__host__ __device__ void cv_line(int W, int H, int64_t x0, int64_t y0, int64_t x1, int64_t y1, Emit& emit) {
  x0 += 2; y0 += 2; x1 += 2; y1 += 2;
  if (!cv_clip_line(static_cast<int64_t>(W) + 4, static_cast<int64_t>(H) + 4, x0, y0, x1, y1)) return;
  cv_thick_line(W, H, (x0 - 2) * kXYOne, (y0 - 2) * kXYOne, (x1 - 2) * kXYOne, (y1 - 2) * kXYOne, 3, emit);
}

// cv2.circle(img, c, 1, color, thickness, LINE_8, 0), thickness 1 or 2.  Thickness 2 goes through EllipseEx, whose
// ellipse2Poly points at 0, 90, 180, 270 and 360 degrees are exact: a closed diamond of four thick segments.
template <class Emit>
__host__ __device__ void cv_circle(int W, int H, int64_t cx, int64_t cy, int thickness, Emit& emit) {
  if (thickness == 1) {
    cv_circle_r1(W, H, cx, cy, false, emit);
    return;
  }
  const int64_t X = cx * kXYOne, Y = cy * kXYOne;
  const int64_t px[5] = {X + kXYOne, X, X - kXYOne, X, X + kXYOne};
  const int64_t py[5] = {Y, Y + kXYOne, Y, Y - kXYOne, Y};
  for (int k = 1; k < 5; ++k) cv_thick_line(W, H, px[k - 1], py[k - 1], px[k], py[k], k == 1 ? 3 : 2, emit);
}

// ------------------------------------------------------------------------------------------ the overlay's setup
// render_body_keypoints' pairs and colours (render_openpose.py:107-134); limb k takes the colour of its second joint.
__constant__ int8_t kPosePairs[2 * kPoseLimbs] = {1, 8, 1, 2, 1, 5, 2, 3, 3, 4, 5, 6, 6, 7, 8, 9, 9, 10, 10, 11, 8, 12,
                                                  12, 13, 13, 14, 1, 0, 0, 15, 15, 17, 0, 16, 16, 18, 14, 19, 19, 20,
                                                  14, 21, 11, 22, 22, 23, 11, 24};
__constant__ uint8_t kPoseColors[3 * kPoseBody] = {255, 0, 85, 255, 0, 0, 255, 85, 0, 255, 170, 0, 255, 255, 0, 170,
                                                   255, 0, 85, 255, 0, 0, 255, 0, 255, 0, 0, 0, 255, 85, 0, 255, 170, 0,
                                                   255, 255, 0, 170, 255, 0, 85, 255, 0, 0, 255, 255, 0, 170, 170, 0,
                                                   255, 255, 0, 255, 85, 0, 255, 0, 0, 255, 0, 0, 255, 0, 0, 255, 0, 255,
                                                   255, 0, 255, 255, 0, 255, 255};
// keypoint_matches (mesh_renderer.py:80): body joint <- extra joint
__constant__ int8_t kPoseMatch[28] = {1, 12, 2, 8, 3, 7, 4, 6, 5, 9, 6, 10, 7, 11, 8, 14, 9, 2, 10, 1, 11, 0, 12, 3, 13,
                                      4, 14, 5};
__device__ __forceinline__ int pose_pair(int limb, int end) { return kPosePairs[2 * limb + end]; }
__device__ __forceinline__ float pose_color(int joint, int c) { return static_cast<float>(kPoseColors[3 * joint + c]); }
__device__ __forceinline__ int pose_match(int k, int end) { return kPoseMatch[2 * k + end]; }

struct PoseGridParams {
  int n, H, W;
  const float* images;   // [n, 3, H, W]
  const float* front;    // [n, H, W, 3]
  const float* side;     // [n, H, W, 4]
  const float* kp[2];    // [n, 44, 2] predictions, [n, 44, 3] GT (either may be null)
  int n_sets, set_of[2]; // keypoint sets present, and which of kp[] each one reads
  float img_res;
  int tiles, xmaps, padding;   // tiles per sample, grid columns, padding
  int grid_h, grid_w;
  float* out;
  long long out_sc, out_sy;    // channel and row strides of out (elements)
  uint32_t* keys;              // [n, n_sets, H, W] workspace
};

// The body keypoints of sample b of keypoint set `gt` in pixels, after the scaling and the keypoint_matches
// substitution, in the reference's float32 arithmetic (mesh_renderer.py:75-97).
__device__ inline void pose_body(const float* kp_all, bool gt, int b, float img_res, float (&x)[kPoseBody],
                                 float (&y)[kPoseBody], float (&conf)[kPoseBody]) {
  const int dims = gt ? 3 : 2;
  const float* kp = kp_all + static_cast<long long>(b) * kPoseKeypoints * dims;
  auto scaled = [&](int j, float& px, float& py, float& pc) {
    px = __fmul_rn(img_res, __fadd_rn(kp[j * dims], 0.5f));
    py = __fmul_rn(img_res, __fadd_rn(kp[j * dims + 1], 0.5f));
    // predictions get a confidence column of ones, scaled with the rest (:76-77); GT keeps its own (:79)
    pc = gt ? kp[j * dims + 2] : __fmul_rn(img_res, 1.5f);
  };
  for (int j = 0; j < kPoseBody; ++j) scaled(j, x[j], y[j], conf[j]);
  for (int k = 0; k < 14; ++k) {
    const int i = pose_match(k, 0), e = kPoseKeypoints - kPoseExtra + pose_match(k, 1);
    float ex, ey, ec;
    scaled(e, ex, ey, ec);
    if (!gt || (ec > 0.f && conf[i] == 0.f)) { x[i] = ex; y[i] = ey; conf[i] = ec; }
  }
}

// astype(int) of a float32 pixel coordinate: truncation toward zero.  Outside int32 (and NaN) cv2 refuses the point,
// so the reference raises; such a primitive is not drawn.
__device__ __forceinline__ bool pose_coord(float v, int64_t& out) {
  if (!(v >= -2147483648.f && v < 2147483648.f)) return false;
  out = static_cast<int64_t>(truncf(v));
  return true;
}

struct PoseKeyEmit {
  uint32_t* keys;
  int W;
  uint32_t key;
  __device__ void operator()(int y, int x0, int x1) const {
    uint32_t* row = keys + static_cast<long long>(y) * W;
    for (int x = x0; x <= x1; ++x) atomicMax(row + x, key);
  }
};

__global__ void pose_raster_kernel(const __grid_constant__ PoseGridParams p) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(p.n) * p.n_sets * kPosePrims) return;
  const int prim = static_cast<int>(idx % kPosePrims);
  const int img = static_cast<int>(idx / kPosePrims);   // (sample, set)
  const int b = img / p.n_sets, s = p.set_of[img % p.n_sets];
  float x[kPoseBody], y[kPoseBody], conf[kPoseBody];
  pose_body(p.kp[s], s == 1, b, p.img_res, x, y, conf);
  // get_keypoints_rectangle(.., 0.1) and the thicknesses (render_openpose.py:10-31, 56-69); the image's width is
  // shape[1] == W and its "height" shape[2] == 3
  float mnx = 0.f, mxx = 0.f, mny = 0.f, mxy = 0.f;
  bool any = false;
  for (int j = 0; j < kPoseBody; ++j) {
    if (!(conf[j] > 0.1f)) continue;
    if (!any) { mnx = mxx = x[j]; mny = mxy = y[j]; any = true; continue; }
    mnx = fminf(mnx, x[j]); mxx = fmaxf(mxx, x[j]); mny = fminf(mny, y[j]); mxy = fmaxf(mxy, y[j]);
  }
  if (!any) return;
  const float pw = __fsub_rn(mxx, mnx), ph = __fsub_rn(mxy, mny);
  if (!(__fmul_rn(pw, ph) > 0.f)) return;   // person_area > 0: nothing is drawn otherwise
  const float rw = __fdiv_rn(pw, static_cast<float>(p.W)), rh = __fdiv_rn(ph, 3.f);
  const float mx = rh > rw ? rh : rw;                 // max(pw / width, ph / height)
  const bool thick = !(mx < 1.f) || mx > 0.05f;       // min(1, .) > 0.05, compared in float32
  PoseKeyEmit emit{p.keys + static_cast<long long>(img) * p.H * p.W, p.W, static_cast<uint32_t>(prim + 1)};
  int64_t x0, y0, x1, y1;
  if (prim < kPoseLimbs) {
    const int i1 = pose_pair(prim, 0), i2 = pose_pair(prim, 1);
    if (!(conf[i1] > 0.1f && conf[i2] > 0.1f)) return;
    if (!(pose_coord(x[i1], x0) && pose_coord(y[i1], y0) && pose_coord(x[i2], x1) && pose_coord(y[i2], y1))) return;
    cv_line(p.W, p.H, x0, y0, x1, y1, emit);
  } else {
    const int j = prim - kPoseLimbs;
    if (!(conf[j] > 0.1f)) return;
    if (!(pose_coord(x[j], x0) && pose_coord(y[j], y0))) return;
    cv_circle(p.W, p.H, x0, y0, thick ? 2 : 1, emit);
  }
}

// The colour of primitive key - 1 (limbs take their second joint's colour), or 0 for none.
__device__ __forceinline__ int pose_color_joint(uint32_t key) {
  const int prim = static_cast<int>(key) - 1;
  return prim < kPoseLimbs ? pose_pair(prim, 1) : prim - kPoseLimbs;
}

__global__ void pose_grid_kernel(const __grid_constant__ PoseGridParams p) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(p.grid_h) * p.grid_w) return;
  const int gy = static_cast<int>(idx / p.grid_w), gx = static_cast<int>(idx - static_cast<long long>(gy) * p.grid_w);
  float v[3] = {0.f, 0.f, 0.f};   // make_grid's pad_value
  const int th = p.H + p.padding, tw = p.W + p.padding;
  const int ry = gy - p.padding, rx = gx - p.padding;
  if (ry >= 0 && rx >= 0) {
    const int ty = ry / th, tx = rx / tw, py = ry - ty * th, px = rx - tx * tw;
    const long long tile = static_cast<long long>(ty) * p.xmaps + tx;
    if (py < p.H && px < p.W && tile < static_cast<long long>(p.n) * p.tiles) {
      const int b = static_cast<int>(tile / p.tiles), slot = static_cast<int>(tile - static_cast<long long>(b) * p.tiles);
      const long long hw = static_cast<long long>(p.H) * p.W, pix = static_cast<long long>(py) * p.W + px;
      const long long bp = static_cast<long long>(b) * hw + pix;
      if (slot == 1) {
        for (int c = 0; c < 3; ++c) v[c] = p.front[bp * 3 + c];
      } else if (slot == 2) {
        for (int c = 0; c < 3; ++c) v[c] = p.side[bp * 4 + c];
      } else {
        for (int c = 0; c < 3; ++c) v[c] = p.images[(b * 3LL + c) * hw + pix];
        if (slot >= 3) {   // skeleton: render_openpose(255 * crop) / 255
          const uint32_t key = p.keys[(static_cast<long long>(b) * p.n_sets + slot - 3) * hw + pix];
          if (key) {
            const int j = pose_color_joint(key);
            for (int c = 0; c < 3; ++c) v[c] = __fdiv_rn(pose_color(j, c), 255.f);
          } else {
            for (int c = 0; c < 3; ++c) v[c] = __fdiv_rn(__fmul_rn(255.f, v[c]), 255.f);
          }
        }
      }
    }
  }
  for (int c = 0; c < 3; ++c) p.out[c * p.out_sc + gy * p.out_sy + gx] = v[c];
}

inline size_t pose_grid_carve(void* base, int n, int n_sets, int W, int H, PoseGridParams* p) {
  Bump bp(base);
  uint32_t* keys = bp.take<uint32_t>(static_cast<size_t>(n) * (n_sets > 0 ? n_sets : 1) * W * H);
  if (p) p->keys = keys;
  return bp.off;
}

}  // namespace thmr
