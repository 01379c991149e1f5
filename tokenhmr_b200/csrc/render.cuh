// Mesh rasterizer behind tokenhmr_b200.render.Renderer (the reference's pyrender Renderer,
// tokenhmr/lib/utils/renderer.py:137-359).  Contract: DESIGN.md §2 "Rendering".
//
// Frame: the model's camera frame q (x right, y down, z forward), in which the reference's whole camera chain
// (x flip of the translation, 180° about x, IntrinsicsCamera at (W/2, H/2)) reduces to perspective_projection of
// q = R v + t (crop view) or q = R (v + t) (render_rgba_multiple).  Lights arrive in the same frame.
//
// Stages, all stream-ordered, no host synchronisation and no allocation (CUDA-graph capturable):
//   keys    cudaMemsetAsync to ~0 (empty)
//   vertex  one thread per (mesh, vertex): q, screen (x, y)
//   normal  one thread per (mesh, vertex): sum of the cross products of the vertex's faces, gathered in CSR order
//           (bit-stable), normalised
//   raster  one thread per (mesh, face); faces whose pixel box exceeds kRasterWarpArea are walked by the whole warp.
//           Each covered pixel does a 64-bit atomicMin of (float_bits(z) << 32 | global face id): positive floats order
//           like their bits, so the nearest z wins and the lower face id breaks ties, whatever the scheduling.
//   resolve one thread per pixel: decode, perspective-correct barycentrics, shade, quantise, composite.
// Bound: atomics and launch count, not FLOPs (an SMPL face covers a few pixels at 256 x 256).
#pragma once
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace thmr {

constexpr int kRenderMaxLights = THMR_RENDER_MAX_LIGHTS;
constexpr int kRenderMaxMeshes = THMR_RENDER_MAX_MESHES;
constexpr int kRasterWarpArea = 64;   // pixel boxes larger than this are rasterized by a whole warp
constexpr unsigned long long kEmptyKey = ~0ull;

struct RenderLight {
  int type;
  float x, y, z, intensity;
};

// Passed by value: the launch copies it, so a captured graph keeps the values of the capturing call.
struct RenderParams {
  const float* verts;   // [n, V, 3]
  const float* trans;   // [n, 3]
  const int32_t* faces; // [F, 3]
  const int32_t* vf_off;  // [V + 1]
  const int32_t* vf_face; // [3F]
  int n, V, F, W, H, n_images;
  float R[9];
  int rotate_translation;
  float focal, cx, cy, znear;
  float base[3], bg[3];
  float ambient;
  int n_lights;
  RenderLight lights[kRenderMaxLights];
  int bg_layout;
  const float* bg_image;
  float mean[3], std[3];
  float* rgba;
  float* composite;
  int32_t* face_id;
  float* depth;
  // workspace
  float4* q;            // [n*V] camera-frame position
  float2* scr;          // [n*V] screen position (pixels, rows down)
  float4* nrm;          // [n*V] unit smooth normal
  unsigned long long* keys; // [n_images, H, W]
  uint16_t mesh_image[kRenderMaxMeshes];
};

__global__ void render_vertex_kernel(const __grid_constant__ RenderParams p) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(p.n) * p.V) return;
  const int m = static_cast<int>(idx / p.V);
  const float* v = p.verts + idx * 3;
  const float* t = p.trans + m * 3;
  float a0 = v[0], a1 = v[1], a2 = v[2];
  if (p.rotate_translation) { a0 += t[0]; a1 += t[1]; a2 += t[2]; }
  float qx = p.R[0] * a0 + p.R[1] * a1 + p.R[2] * a2;
  float qy = p.R[3] * a0 + p.R[4] * a1 + p.R[5] * a2;
  float qz = p.R[6] * a0 + p.R[7] * a1 + p.R[8] * a2;
  if (!p.rotate_translation) { qx += t[0]; qy += t[1]; qz += t[2]; }
  p.q[idx] = make_float4(qx, qy, qz, 0.f);
  // perspective_projection (geometry.py:115-124): divide by z, then apply K
  p.scr[idx] = make_float2(fmaf(p.focal, qx / qz, p.cx), fmaf(p.focal, qy / qz, p.cy));
}

__device__ __forceinline__ float3 f3sub(float4 a, float4 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }

__global__ void render_normal_kernel(const __grid_constant__ RenderParams p) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<long long>(p.n) * p.V) return;
  const int m = static_cast<int>(idx / p.V);
  const int i = static_cast<int>(idx - static_cast<long long>(m) * p.V);
  const float4* q = p.q + static_cast<long long>(m) * p.V;
  float nx = 0.f, ny = 0.f, nz = 0.f;
  for (int k = p.vf_off[i]; k < p.vf_off[i + 1]; ++k) {   // fixed order: bitwise-stable sums
    const int f = p.vf_face[k];
    const float4 q0 = q[p.faces[3 * f]], q1 = q[p.faces[3 * f + 1]], q2 = q[p.faces[3 * f + 2]];
    const float3 e1 = f3sub(q1, q0), e2 = f3sub(q2, q0);
    nx += e1.y * e2.z - e1.z * e2.y;   // |cross| = twice the area: area-weighted
    ny += e1.z * e2.x - e1.x * e2.z;
    nz += e1.x * e2.y - e1.y * e2.x;
  }
  const float len = sqrtf(nx * nx + ny * ny + nz * nz);
  const float s = len > 0.f ? 1.f / len : 0.f;
  p.nrm[idx] = make_float4(nx * s, ny * s, nz * s, 0.f);
}

// Edge function of the directed edge a -> b at point (px, py), evaluated in fp64 on the fp32 screen positions.  Both
// triangles that share an edge evaluate it in one canonical direction (lower vertex id first) and negate, so their
// values are exact negatives of each other and the fill rule gives every pixel centre on the edge to exactly one.
struct Edge {
  double ax, ay, dx, dy, sgn;   // canonical origin and direction, sign of the directed edge relative to it
  bool tl;                      // directed edge is top or left (decided after orienting the triangle)
};

__device__ __forceinline__ Edge make_edge(int ia, int ib, float2 a, float2 b) {
  Edge e;
  const bool swap = ib < ia;
  const float2 o = swap ? b : a, d = swap ? a : b;
  e.ax = o.x; e.ay = o.y;
  e.dx = static_cast<double>(d.x) - o.x;
  e.dy = static_cast<double>(d.y) - o.y;
  e.sgn = swap ? -1.0 : 1.0;
  e.tl = false;
  return e;
}
__device__ __forceinline__ double edge_eval(const Edge& e, double px, double py) {
  return e.sgn * (e.dx * (py - e.ay) - e.dy * (px - e.ax));
}
// With the triangle oriented so that its inside is positive (rows point down): top edge = horizontal with dx > 0,
// left edge = dy < 0.  The reversed edge gets the opposite answer, so a shared edge has exactly one owner.
__device__ __forceinline__ bool edge_top_left(const Edge& e, double orient) {
  const double dx = e.sgn * orient * e.dx, dy = e.sgn * orient * e.dy;
  return dy < 0.0 || (dy == 0.0 && dx > 0.0);
}

struct Tri {
  Edge e[3];
  double orient, inv_area;   // inside: orient * E > 0 (or == 0 on a top-left edge)
  float iz[3];               // 1 / z of the vertices
  int x0, x1, y0, y1;        // pixel box, clipped to the viewport
  unsigned long long* keys;
  unsigned int fid;
};

// Sets up face f of mesh m; returns false if it is dropped (vertex nearer than znear, non-finite, zero area, or no
// pixel in its box).
__device__ bool tri_setup(const RenderParams& p, int m, int f, Tri& T) {
  const long long base = static_cast<long long>(m) * p.V;
  const int i0 = p.faces[3 * f], i1 = p.faces[3 * f + 1], i2 = p.faces[3 * f + 2];
  const float z0 = p.q[base + i0].z, z1 = p.q[base + i1].z, z2 = p.q[base + i2].z;
  if (!(z0 >= p.znear && z1 >= p.znear && z2 >= p.znear)) return false;   // dropped, not clipped (NaN too)
  const float2 s0 = p.scr[base + i0], s1 = p.scr[base + i1], s2 = p.scr[base + i2];
  if (!(isfinite(s0.x) && isfinite(s0.y) && isfinite(s1.x) && isfinite(s1.y) && isfinite(s2.x) && isfinite(s2.y)))
    return false;
  T.e[0] = make_edge(i1, i2, s1, s2);   // e[k] is the edge opposite vertex k: its value at vertex k is the area
  T.e[1] = make_edge(i2, i0, s2, s0);
  T.e[2] = make_edge(i0, i1, s0, s1);
  const double area = edge_eval(T.e[2], s2.x, s2.y);
  if (area == 0.0) return false;
  T.orient = area > 0.0 ? 1.0 : -1.0;
  T.inv_area = 1.0 / fabs(area);
  for (int k = 0; k < 3; ++k) T.e[k].tl = edge_top_left(T.e[k], T.orient);
  T.iz[0] = 1.f / z0; T.iz[1] = 1.f / z1; T.iz[2] = 1.f / z2;
  // centre (c + 0.5) inside [min, max]  <=>  c in [min - 0.5, max - 0.5]; one pixel of slack, the edge test decides
  const float mnx = fminf(s0.x, fminf(s1.x, s2.x)), mxx = fmaxf(s0.x, fmaxf(s1.x, s2.x));
  const float mny = fminf(s0.y, fminf(s1.y, s2.y)), mxy = fmaxf(s0.y, fmaxf(s1.y, s2.y));
  T.x0 = static_cast<int>(fmaxf(floorf(mnx - 0.5f), 0.f));
  T.y0 = static_cast<int>(fmaxf(floorf(mny - 0.5f), 0.f));
  T.x1 = static_cast<int>(fminf(ceilf(mxx - 0.5f), static_cast<float>(p.W - 1)));
  T.y1 = static_cast<int>(fminf(ceilf(mxy - 0.5f), static_cast<float>(p.H - 1)));
  if (T.x0 > T.x1 || T.y0 > T.y1) return false;
  T.keys = p.keys + static_cast<long long>(p.mesh_image[m]) * p.W * p.H;
  T.fid = static_cast<unsigned int>(m) * static_cast<unsigned int>(p.F) + static_cast<unsigned int>(f);
  return true;
}

// Screen-space barycentrics of pixel (x, y) if its centre is covered; the fill rule decides ties.
__device__ __forceinline__ bool tri_cover(const Tri& T, int x, int y, double w[3]) {
  const double px = x + 0.5, py = y + 0.5;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double e = T.orient * edge_eval(T.e[k], px, py);
    if (e < 0.0 || (e == 0.0 && !T.e[k].tl)) return false;
    w[k] = e * T.inv_area;
  }
  return true;
}

__device__ __forceinline__ void tri_pixel(const Tri& T, int W, int x, int y) {
  double w[3];
  if (!tri_cover(T, x, y, w)) return;
  // perspective-correct depth: 1/z is affine in screen space
  const double iz = w[0] * T.iz[0] + w[1] * T.iz[1] + w[2] * T.iz[2];
  const float z = static_cast<float>(1.0 / iz);
  const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(z)) << 32) | T.fid;
  atomicMin(T.keys + static_cast<long long>(y) * W + x, key);
}

__global__ void __launch_bounds__(128) render_raster_kernel(const __grid_constant__ RenderParams p) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const int lane = threadIdx.x & 31;
  Tri T;
  bool live = false;
  if (idx < static_cast<long long>(p.n) * p.F) {
    const int m = static_cast<int>(idx / p.F);
    live = tri_setup(p, m, static_cast<int>(idx - static_cast<long long>(m) * p.F), T);
  }
  const int bw = live ? T.x1 - T.x0 + 1 : 0, bh = live ? T.y1 - T.y0 + 1 : 0;
  const bool big = live && static_cast<long long>(bw) * bh > kRasterWarpArea;
  if (live && !big)
    for (int y = T.y0; y <= T.y1; ++y)
      for (int x = T.x0; x <= T.x1; ++x) tri_pixel(T, p.W, x, y);
  // large faces: the warp takes them one at a time, each lane striding the pixel box
  unsigned int todo = __ballot_sync(0xffffffffu, big);
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    Tri S;
    const int* ti = reinterpret_cast<const int*>(&T);
    int* si = reinterpret_cast<int*>(&S);
#pragma unroll
    for (int k = 0; k < static_cast<int>(sizeof(Tri) / sizeof(int)); ++k) si[k] = __shfl_sync(0xffffffffu, ti[k], src);
    const int sw = S.x1 - S.x0 + 1;
    const long long total = static_cast<long long>(sw) * (S.y1 - S.y0 + 1);
    for (long long k = lane; k < total; k += 32)
      tri_pixel(S, p.W, S.x0 + static_cast<int>(k % sw), S.y0 + static_cast<int>(k / sw));
  }
}

__device__ __forceinline__ float quant8(float c) { return rintf(c * 255.f) / 255.f; }   // uint8 framebuffer / 255

__global__ void render_resolve_kernel(const __grid_constant__ RenderParams p) {
  const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long hw = static_cast<long long>(p.W) * p.H;
  if (idx >= p.n_images * hw) return;
  const int img = static_cast<int>(idx / hw);
  const long long pix = idx - img * hw;
  const int y = static_cast<int>(pix / p.W), x = static_cast<int>(pix - static_cast<long long>(y) * p.W);
  const unsigned long long key = p.keys[idx];
  float col[3], alpha = 0.f, depth = 0.f;
  int fid = -1;
  if (key == kEmptyKey) {
    for (int c = 0; c < 3; ++c) col[c] = quant8(p.bg[c]);
  } else {
    fid = static_cast<int>(key & 0xffffffffu);
    depth = __uint_as_float(static_cast<unsigned int>(key >> 32));
    const int m = fid / p.F, f = fid - m * p.F;
    Tri T;
    tri_setup(p, m, f, T);   // same fp64 edge values as the raster stage
    double w[3];
    w[0] = T.orient * edge_eval(T.e[0], x + 0.5, y + 0.5) * T.inv_area;
    w[1] = T.orient * edge_eval(T.e[1], x + 0.5, y + 0.5) * T.inv_area;
    w[2] = T.orient * edge_eval(T.e[2], x + 0.5, y + 0.5) * T.inv_area;
    // perspective-correct barycentrics
    const double b0 = w[0] * T.iz[0], b1 = w[1] * T.iz[1], b2 = w[2] * T.iz[2];
    const double bs = 1.0 / (b0 + b1 + b2);
    const float c0 = static_cast<float>(b0 * bs), c1 = static_cast<float>(b1 * bs), c2 = static_cast<float>(b2 * bs);
    const long long base = static_cast<long long>(m) * p.V;
    const int i0 = p.faces[3 * f], i1 = p.faces[3 * f + 1], i2 = p.faces[3 * f + 2];
    const float4 n0 = p.nrm[base + i0], n1 = p.nrm[base + i1], n2 = p.nrm[base + i2];
    float nx = c0 * n0.x + c1 * n1.x + c2 * n2.x;
    float ny = c0 * n0.y + c1 * n1.y + c2 * n2.y;
    float nz = c0 * n0.z + c1 * n1.z + c2 * n2.z;
    const float nl = sqrtf(nx * nx + ny * ny + nz * nz);
    const float s = nl > 0.f ? 1.f / nl : 0.f;
    nx *= s; ny *= s; nz *= s;
    const float4 q0 = p.q[base + i0], q1 = p.q[base + i1], q2 = p.q[base + i2];
    const float px = c0 * q0.x + c1 * q1.x + c2 * q2.x;
    const float py = c0 * q0.y + c1 * q1.y + c2 * q2.y;
    const float pz = c0 * q0.z + c1 * q1.z + c2 * q2.z;
    float light = p.ambient;
    for (int l = 0; l < p.n_lights; ++l) {
      const RenderLight L = p.lights[l];
      if (L.type == THMR_LIGHT_DIRECTIONAL) {
        light += L.intensity * fmaxf(0.f, nx * L.x + ny * L.y + nz * L.z);
      } else {
        const float dx = L.x - px, dy = L.y - py, dz = L.z - pz;
        const float d2 = dx * dx + dy * dy + dz * dz;
        const float inv = rsqrtf(d2);
        light += L.intensity * fmaxf(0.f, (nx * dx + ny * dy + nz * dz) * inv) / d2;
      }
    }
    light = fminf(fmaxf(light, 0.f), 1.f);
    for (int c = 0; c < 3; ++c) col[c] = quant8(p.base[c] * light);
    alpha = 1.f;
  }
  if (p.rgba) {
    float4 o = make_float4(col[0], col[1], col[2], alpha);
    reinterpret_cast<float4*>(p.rgba)[idx] = o;
  }
  if (p.composite) {
    float bgc[3];
    if (p.bg_layout == THMR_BG_HWC) {
      for (int c = 0; c < 3; ++c) bgc[c] = p.bg_image[idx * 3 + c];
    } else {   // normalised CHW crop: img * std + mean (renderer.py:177-178), unfused like torch
      for (int c = 0; c < 3; ++c)
        bgc[c] = __fadd_rn(__fmul_rn(p.bg_image[(img * 3LL + c) * hw + pix], p.std[c]), p.mean[c]);
    }
    // color * a + (1 - a) * image (renderer.py:224-226), in numpy's operation order
    for (int c = 0; c < 3; ++c)
      p.composite[idx * 3 + c] = __fadd_rn(__fmul_rn(col[c], alpha), __fmul_rn(__fsub_rn(1.f, alpha), bgc[c]));
  }
  if (p.face_id) p.face_id[idx] = fid;
  if (p.depth) p.depth[idx] = depth;
}

// Workspace layout of one call (base == nullptr only measures); fills p's workspace pointers when p != nullptr.
inline size_t render_carve(void* base, int V, int n, int n_images, int W, int H, RenderParams* p) {
  Bump bp(base);
  const size_t nv = static_cast<size_t>(n) * V;
  float4* q = bp.take<float4>(nv);
  float2* scr = bp.take<float2>(nv);
  float4* nrm = bp.take<float4>(nv);
  unsigned long long* keys = bp.take<unsigned long long>(static_cast<size_t>(n_images) * W * H);
  if (p) { p->q = q; p->scr = scr; p->nrm = nrm; p->keys = keys; }
  return bp.off;
}

}  // namespace thmr

struct thmr_render_topology {
  int F = 0, V = 0;
  int32_t* faces = nullptr;    // [F, 3]
  int32_t* vf_off = nullptr;   // [V + 1]
  int32_t* vf_face = nullptr;  // [3F], ascending face id per vertex
};
