// SMPL linear blend skinning (smplx.lbs.lbs, pose2rot both ways) + the TokenHMR SMPL wrapper
// (tokenhmr/lib/models/smpl_wrapper.py:27-41) as four kernels:
//
//   smpl_pose_kernel    per pose: (Rodrigues) -> joint locations -> 24-joint kinematic chain -> relative
//                       transforms A (3x4), posed joints, and the blend feature [R - I (207) | betas (10) | 1] split
//                       into fp16 hi/lo operands for the tensor-core blend GEMM
//   [wgmma GEMM]        v_posed = feature (B x 218) * [posedirs ; shapedirs ; v_template] (218 x 3V): the shape blend
//                       and the template ride in the same contraction as the pose blend (blend_shapes + pose offsets
//                       of smplx.lbs in one pass); split-fp16 (hi*hi + lo*hi + hi*lo, operands pre-scaled by 2^10)
//                       gives ~2^-21 relative error with fp32 accumulation
//   smpl_skin_kernel    per (vertex, pose): T = sum_k w_k A_jk (sparse skinning weights, ELL); vertex = T [v_posed;1]
//   smpl_joints_kernel  per pose: 45 smplx joints -> 25 OpenPose joints (joint_map) + 19 regressed extra
//                       joints (sparse CSR regressor) ; optional camera translation + perspective projection
//                       (tokenhmr.py:165-187, geometry.py:86-124)
//
// All skinning math is fp32 (tolerance: 1e-4 relative to the fp32 reference).
#pragma once
#include "common.cuh"

namespace thmr {

constexpr int kSmplJ = 24;
constexpr int kSmplPF = 207;        // (24-1)*9 pose-blend features
constexpr int kSmplFeatBeta = 207;  // feature columns [207, 217): betas;  217: the constant 1 (template)
constexpr int kSmplFeatOne = 217;
constexpr int kSmplPFPad = 224;     // feature row: 207 + 10 + 1, padded to a multiple of 16 (fp16 pitch, UMMA K step)
constexpr float kSplitScale = 1024.0f;

struct SmplModel {
  int V = 0, nb = 10;
  // device buffers (owned)
  float* v_template = nullptr;    // [V,3]
  float* shapedirs = nullptr;     // [V,3,nb]
  float* J_template = nullptr;    // [24,3]      = J_regressor . v_template
  float* J_shapedirs = nullptr;   // [24,3,nb]   = J_regressor . shapedirs
  __half* posedirsT = nullptr;    // [3V, 3*224] fp16: [hi | hi | lo] of 1024 * [posedirs^T | shapedirs | v_template]
  int ell = 0;                    // max non-zeros per vertex of lbs_weights
  int* w_idx = nullptr;           // [V, ell]
  float* w_val = nullptr;         // [V, ell]
  int* jx_ptr = nullptr;          // CSR of joint_regressor_extra [19, V]
  int* jx_idx = nullptr;
  float* jx_val = nullptr;
  int n_extra = 0;
  int* extra_vid = nullptr;       // [21] VertexJointSelector ids
  int* joint_map = nullptr;       // [25]
  int parents[kSmplJ];
  // backward only (smpl_grad.cuh)
  float* basis32 = nullptr;       // [207 + nb, off_pitch] fp32 [posedirs ; shapedirs^T], pad columns zero
  int* bw_ptr = nullptr;          // [nvb*24 + 1] per (256-vertex block, joint): list of the block's vertices ...
  int* bw_lv = nullptr;           // ... (local index) skinned to that joint ...
  float* bw_val = nullptr;        // ... and their weights, vertices in increasing order
  int* cx_ptr = nullptr;          // [V + 1] per vertex: the grad_joints rows that read it (CSC of the joint map's
  int* cx_row = nullptr;          //         extra-vertex picks, weight 1, then of joint_regressor_extra)
  float* cx_val = nullptr;
};

// ---- init-time: J_template / J_shapedirs (one block per output scalar) ---------------------------------
__global__ void smpl_jreg_kernel(const float* __restrict__ Jreg, const float* __restrict__ v_template,
                                 const float* __restrict__ shapedirs, float* __restrict__ J_template,
                                 float* __restrict__ J_shapedirs, int V, int nb) {
  // blockIdx.x = j*3*(nb+1) + c*(nb+1) + l   (l == nb -> template)
  const int l = blockIdx.x % (nb + 1);
  const int c = (blockIdx.x / (nb + 1)) % 3;
  const int j = blockIdx.x / (3 * (nb + 1));
  float s = 0.f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const float w = Jreg[static_cast<size_t>(j) * V + v];
    if (w != 0.f) s += w * (l == nb ? v_template[v * 3 + c] : shapedirs[(static_cast<size_t>(v) * 3 + c) * nb + l]);
  }
  __shared__ float red[32];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (blockDim.x >> 5); ++i) t += red[i];
    if (l == nb) J_template[j * 3 + c] = t;
    else J_shapedirs[(j * 3 + c) * nb + l] = t;
  }
}

// ---- init-time: blend basis -> transposed split fp16 [3V, 3*224]: row n = (vertex, coordinate), columns
//      [posedirs(207, n) | shapedirs(n, 0..nb) | v_template(n) | 0]
__global__ void smpl_pack_posedirs_kernel(const float* __restrict__ posedirs, const float* __restrict__ shapedirs,
                                          const float* __restrict__ v_template, int nb, __half* __restrict__ out, int V3) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long>(V3) * kSmplPFPad) return;
  const int k = i % kSmplPFPad;
  const int n = i / kSmplPFPad;
  float v = 0.f;
  if (k < kSmplPF) v = posedirs[static_cast<size_t>(k) * V3 + n];
  else if (k < kSmplFeatBeta + nb) v = shapedirs[static_cast<size_t>(n) * nb + (k - kSmplFeatBeta)];
  else if (k == kSmplFeatOne) v = v_template[n];
  v *= kSplitScale;
  const __half hi = __float2half_rn(v);
  const __half lo = __float2half_rn(v - __half2float(hi));
  __half* o = out + static_cast<size_t>(n) * (3 * kSmplPFPad);
  o[k] = hi;
  o[kSmplPFPad + k] = hi;
  o[2 * kSmplPFPad + k] = lo;
}

// ---- per pose: rotations, joints, kinematic chain -------------------------------------------------------
//   pose: pose2rot ? (B,24,3) axis-angle : (B,24,3,3) rotation matrices
//   A (B,24,12) row-major 3x4: [ R_world | t_world - R_world J ];  Jposed (B,24,3);  pf16 (B, 3*208) split feature
__global__ void __launch_bounds__(32)
smpl_pose_kernel(const float* __restrict__ pose, int pose2rot, const float* __restrict__ betas,
                 const float* __restrict__ J_template, const float* __restrict__ J_shapedirs, int nb,
                 const int* __restrict__ parents_dev, float* __restrict__ A, float* __restrict__ Jposed,
                 __half* __restrict__ pf16, int B) {
  __shared__ float R[kSmplJ][9];
  __shared__ float Jl[kSmplJ][3];
  __shared__ float G[kSmplJ][12];
  const int b = blockIdx.x;
  const int j = threadIdx.x;
  if (j < kSmplJ) {
    float r[9];
    if (pose2rot) {
      // smplx.lbs.batch_rodrigues: angle = ||r + 1e-8||, dir = r / angle
      const float* a = pose + (static_cast<size_t>(b) * kSmplJ + j) * 3;
      const float x = a[0], y = a[1], z = a[2];
      const float ex = x + 1e-8f, ey = y + 1e-8f, ez = z + 1e-8f;
      const float angle = sqrtf(ex * ex + ey * ey + ez * ez);
      const float dx = x / angle, dy = y / angle, dz = z / angle;
      float s, c;
      sincosf(angle, &s, &c);
      const float oc = 1.f - c;
      // R = I + s K + (1-c) K K,  K = skew(d)
      r[0] = 1.f + oc * (-(dy * dy) - dz * dz); r[1] = -s * dz + oc * dx * dy;          r[2] = s * dy + oc * dx * dz;
      r[3] = s * dz + oc * dx * dy;             r[4] = 1.f + oc * (-(dx * dx) - dz * dz); r[5] = -s * dx + oc * dy * dz;
      r[6] = -s * dy + oc * dx * dz;            r[7] = s * dx + oc * dy * dz;           r[8] = 1.f + oc * (-(dx * dx) - dy * dy);
    } else {
      const float* a = pose + (static_cast<size_t>(b) * kSmplJ + j) * 9;
#pragma unroll
      for (int e = 0; e < 9; ++e) r[e] = a[e];
    }
#pragma unroll
    for (int e = 0; e < 9; ++e) R[j][e] = r[e];
    // joint location of the shaped template
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = J_template[j * 3 + c];
      for (int l = 0; l < nb; ++l) v += J_shapedirs[(j * 3 + c) * nb + l] * betas[static_cast<size_t>(b) * nb + l];
      Jl[j][c] = v;
    }
    // pose-blend feature (R - I) for joints 1..23, split hi/lo, scaled by 2^10
    if (j >= 1) {
      __half* o = pf16 + static_cast<size_t>(b) * (3 * kSmplPFPad) + (j - 1) * 9;
#pragma unroll
      for (int e = 0; e < 9; ++e) {
        const float v = (r[e] - ((e == 0 || e == 4 || e == 8) ? 1.f : 0.f)) * kSplitScale;
        const __half hi = __float2half_rn(v);
        const __half lo = __float2half_rn(v - __half2float(hi));
        o[e] = hi;
        o[kSmplPFPad + e] = lo;
        o[2 * kSmplPFPad + e] = hi;
      }
    } else {
      // shape-blend features: betas (columns 207..216), the constant 1 that multiplies v_template (217), zero padding
      __half* o = pf16 + static_cast<size_t>(b) * (3 * kSmplPFPad);
      for (int k = kSmplFeatBeta; k < kSmplPFPad; ++k) {
        float v = 0.f;
        if (k < kSmplFeatBeta + nb) v = betas[static_cast<size_t>(b) * nb + (k - kSmplFeatBeta)];
        else if (k == kSmplFeatOne) v = 1.f;
        v *= kSplitScale;
        const __half hi = __float2half_rn(v);
        const __half lo = __float2half_rn(v - __half2float(hi));
        o[k] = hi;
        o[kSmplPFPad + k] = lo;
        o[2 * kSmplPFPad + k] = hi;
      }
    }
  }
  __syncwarp();
  // kinematic chain (batch_rigid_transform): G_0 = [R_0 | J_0], G_i = G_parent * [R_i | J_i - J_parent]
  for (int i = 0; i < kSmplJ; ++i) {
    if (j == i) {
      const int par = parents_dev[i];
      if (par < 0) {
#pragma unroll
        for (int rr = 0; rr < 3; ++rr) {
          G[i][rr * 4 + 0] = R[i][rr * 3 + 0]; G[i][rr * 4 + 1] = R[i][rr * 3 + 1]; G[i][rr * 4 + 2] = R[i][rr * 3 + 2];
          G[i][rr * 4 + 3] = Jl[i][rr];
        }
      } else {
        const float tx = Jl[i][0] - Jl[par][0], ty = Jl[i][1] - Jl[par][1], tz = Jl[i][2] - Jl[par][2];
#pragma unroll
        for (int rr = 0; rr < 3; ++rr) {
          const float g0 = G[par][rr * 4 + 0], g1 = G[par][rr * 4 + 1], g2 = G[par][rr * 4 + 2], g3 = G[par][rr * 4 + 3];
          G[i][rr * 4 + 0] = g0 * R[i][0] + g1 * R[i][3] + g2 * R[i][6];
          G[i][rr * 4 + 1] = g0 * R[i][1] + g1 * R[i][4] + g2 * R[i][7];
          G[i][rr * 4 + 2] = g0 * R[i][2] + g1 * R[i][5] + g2 * R[i][8];
          G[i][rr * 4 + 3] = g0 * tx + g1 * ty + g2 * tz + g3;
        }
      }
    }
    __syncwarp();
  }
  if (j < kSmplJ) {
    float* a = A + (static_cast<size_t>(b) * kSmplJ + j) * 12;
    float* jp = Jposed + (static_cast<size_t>(b) * kSmplJ + j) * 3;
#pragma unroll
    for (int rr = 0; rr < 3; ++rr) {
      const float g0 = G[j][rr * 4 + 0], g1 = G[j][rr * 4 + 1], g2 = G[j][rr * 4 + 2], g3 = G[j][rr * 4 + 3];
      a[rr * 4 + 0] = g0; a[rr * 4 + 1] = g1; a[rr * 4 + 2] = g2;
      a[rr * 4 + 3] = g3 - (g0 * Jl[j][0] + g1 * Jl[j][1] + g2 * Jl[j][2]);
      jp[rr] = g3;
    }
  }
}

// ---- skinning: thread = vertex, block = 128 vertices x SKIN_POSES poses ---------------------------------
// v_posed comes out of the blend GEMM (L2-resident chunk); the next pose's three coordinates are loaded while the current
// pose is skinned.  The 24 relative transforms of each pose sit in shared memory (odd joint stride: distinct joints
// hit distinct banks, equal joints broadcast).
// Launch shape: 256 vertices per block by default.  V = 6890 then gives 27 x ceil(B / 16) blocks, and a 512-pose chunk
// (864 blocks) is resident all at once (8 blocks of 20 KB / 256 threads per SM = 1184 slots); with 128 vertices per block the
// same chunk is 1728 blocks on 1628 slots, i.e. a second wave of 100 blocks during which most SMs idle
// (THMR_SKIN_THREADS=128 selects that shape).
constexpr int kSkinPoses = 16;
constexpr int kSkinAStride = 13;   // floats per joint in smem (12 used)
constexpr int kSkinThreadsDefault = 256;

// kEllReg: skinning weights held in registers (4 for SMPL's 4 influences per vertex: 40 registers per thread, so that six
// 256-thread blocks = 888 block slots fit an SM and the 864 blocks of a chunk form ONE wave; 8 otherwise).
template <int kSkinThreads, int kEllReg>
__global__ void __launch_bounds__(kSkinThreads, (kSkinThreads == 256) ? (kEllReg == 4 ? 6 : 4) : 10)
smpl_skin_kernel(const int* __restrict__ w_idx, const float* __restrict__ w_val, int ell, const float* __restrict__ A,
                 const float* __restrict__ vposed, long off_pitch, float* __restrict__ verts,
                 long vert_pitch /* floats between poses */, int V, int B) {
  __shared__ float sA[kSkinPoses][kSmplJ * kSkinAStride];
  const int p0 = blockIdx.y * kSkinPoses;
  const int np = (B - p0) < kSkinPoses ? (B - p0) : kSkinPoses;
  for (int i = threadIdx.x; i < np * kSmplJ * 12; i += kSkinThreads) {
    const int r = i % (kSmplJ * 12);
    sA[i / (kSmplJ * 12)][(r / 12) * kSkinAStride + r % 12] = A[static_cast<size_t>(p0) * kSmplJ * 12 + i];
  }
  __syncthreads();
  const int v = blockIdx.x * kSkinThreads + threadIdx.x;
  if (v >= V) return;
  // skinning weights of this vertex: registers when the ELL width is small (real SMPL: 4), else re-read
  int wi[kEllReg];
  float wv[kEllReg];
#pragma unroll
  for (int k = 0; k < kEllReg; ++k) {
    wi[k] = (k < ell) ? w_idx[static_cast<size_t>(v) * ell + k] * kSkinAStride : 0;
    wv[k] = (k < ell) ? w_val[static_cast<size_t>(v) * ell + k] : 0.f;
  }
  const float* src = vposed + static_cast<size_t>(p0) * off_pitch + v * 3;
  float nx0 = src[0], nx1 = src[1], nx2 = src[2];
  for (int pp = 0; pp < np; ++pp) {
    const float x0 = nx0, x1 = nx1, x2 = nx2;
    if (pp + 1 < np) {
      const float* nsrc = src + static_cast<size_t>(pp + 1) * off_pitch;
      nx0 = nsrc[0]; nx1 = nsrc[1]; nx2 = nsrc[2];
    }
    float T[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) T[e] = 0.f;
    if (ell <= kEllReg) {
#pragma unroll
      for (int k = 0; k < kEllReg; ++k) {
        if (k < ell) {
          const float w = wv[k];
          const float* a = &sA[pp][wi[k]];
#pragma unroll
          for (int e = 0; e < 12; ++e) T[e] = fmaf(w, a[e], T[e]);
        }
      }
    } else {
      for (int k = 0; k < ell; ++k) {
        const float w = w_val[static_cast<size_t>(v) * ell + k];
        const float* a = &sA[pp][w_idx[static_cast<size_t>(v) * ell + k] * kSkinAStride];
#pragma unroll
        for (int e = 0; e < 12; ++e) T[e] = fmaf(w, a[e], T[e]);
      }
    }
    float* o = verts + static_cast<size_t>(p0 + pp) * vert_pitch + v * 3;
#pragma unroll
    for (int rr = 0; rr < 3; ++rr) o[rr] = T[rr * 4 + 0] * x0 + T[rr * 4 + 1] * x1 + T[rr * 4 + 2] * x2 + T[rr * 4 + 3];
  }
}

// ---- joints: 25 mapped + n_extra regressed, optional camera / projection --------------------------------
// The camera tail of forward_step, shared with camera_tail_kernel (losses.cuh) so both give the same numbers.
// tokenhmr.py:166-168: the depth of pred_cam_t from the scale s of pred_cam = (s, tx, ty)
__device__ __forceinline__ float cam_depth(float s, float focal, float image_size) {
  return 2.f * focal / (image_size * s + 1e-9f);
}
// perspective_projection with rotation I, camera centre 0, focal = focal/image_size (geometry.py:110-124)
__device__ __forceinline__ float2 project_point(const float x[3], const float t[3], float focal, float image_size) {
  const float px = x[0] + t[0], py = x[1] + t[1], pz = x[2] + t[2];
  const float f = focal / image_size;
  return make_float2(f * (px / pz), f * (py / pz));
}

__global__ void __launch_bounds__(64)
smpl_joints_kernel(const float* __restrict__ Jposed, const float* __restrict__ verts, long vert_pitch,
                   const int* __restrict__ joint_map, const int* __restrict__ extra_vid,
                   const int* __restrict__ jx_ptr, const int* __restrict__ jx_idx, const float* __restrict__ jx_val,
                   int n_extra, float* __restrict__ joints /* (B, 25+n_extra, 3) */, const float* __restrict__ pred_cam,
                   float focal, float image_size, float* __restrict__ cam_t, float* __restrict__ focal_out,
                   float* __restrict__ kp2d) {
  const int b = blockIdx.x;
  const int nj = 25 + n_extra;
  const float* vb = verts + static_cast<size_t>(b) * vert_pitch;
  float t[3] = {0.f, 0.f, 0.f};
  if (pred_cam) {
    const float s = pred_cam[b * 3 + 0];
    t[0] = pred_cam[b * 3 + 1];
    t[1] = pred_cam[b * 3 + 2];
    t[2] = cam_depth(s, focal, image_size);
    if (threadIdx.x == 0) {
      cam_t[b * 3 + 0] = t[0]; cam_t[b * 3 + 1] = t[1]; cam_t[b * 3 + 2] = t[2];
      focal_out[b * 2 + 0] = focal; focal_out[b * 2 + 1] = focal;
    }
  }
  for (int k = threadIdx.x; k < nj; k += blockDim.x) {
    float x[3];
    if (k < 25) {
      const int src = joint_map[k];
      const float* s = (src < kSmplJ) ? (Jposed + (static_cast<size_t>(b) * kSmplJ + src) * 3)
                                      : (vb + static_cast<size_t>(extra_vid[src - kSmplJ]) * 3);
      x[0] = s[0]; x[1] = s[1]; x[2] = s[2];
    } else {
      const int r = k - 25;
      x[0] = x[1] = x[2] = 0.f;
      for (int e = jx_ptr[r]; e < jx_ptr[r + 1]; ++e) {
        const float w = jx_val[e];
        const float* s = vb + static_cast<size_t>(jx_idx[e]) * 3;
        x[0] += w * s[0]; x[1] += w * s[1]; x[2] += w * s[2];
      }
    }
    float* o = joints + (static_cast<size_t>(b) * nj + k) * 3;
    o[0] = x[0]; o[1] = x[1]; o[2] = x[2];
    if (pred_cam) {
      const float2 u = project_point(x, t, focal, image_size);
      kp2d[(static_cast<size_t>(b) * nj + k) * 2 + 0] = u.x;
      kp2d[(static_cast<size_t>(b) * nj + k) * 2 + 1] = u.y;
    }
  }
}

}  // namespace thmr
