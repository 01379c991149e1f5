// Backward (vector-Jacobian product) of the SMPL stage: thmr_smpl_forward without the camera tail, and thmr_lbs.
//
// Stateless: the backward takes the forward's inputs and the output cotangents, and recomputes what it needs with the
// forward's own kernels and chunking (smpl_pose_kernel for A and the posed joints, the split-fp16 blend GEMM for
// v_posed, kSmplChunk poses at a time), so the gradients are those of the function the forward computes.  Per chunk:
//
//   smpl_skin_bwd_kernel   thread = vertex, block = 256 vertices x kBwdPoses poses.  Effective vertex cotangent
//                          g_v = grad_verts_v + the grad_joints rows that reach vertex v (OpenPose joints taken from
//                          extra_vertex_ids, weight 1, and the regressed extra joints: a CSC copy of the regressor, so
//                          each vertex gathers its terms in a fixed order); vposed_bar_v = T_v,R^T g_v; and the partial
//                          sums of A_bar_j = sum_v,k: j_k = j  w_vk g_v [v_posed_v; 1]^T over the block's vertices, in a
//                          per-block per-joint list order fixed at create (no atomics)
//   smpl_blend_bwd_kernel  feat_bar (n x (207 + nb)) = vposed_bar (n x 3V) . basis^T in fp32 on the CUDA cores
//                          against an fp32 copy of [posedirs ; shapedirs] packed at create; split-K partials
//   smpl_chain_bwd_kernel  warp = pose: sums the A_bar and feat_bar partials in a fixed order, then the reverse
//                          kinematic-chain sweep (children before parents), the joint-location and shape terms, and
//                          for pose2rot the Rodrigues VJP (smplx's angle = ||r + 1e-8||, so a zero vector has a finite
//                          gradient)
//
// Every reduction runs in a fixed order: two calls give bitwise-equal gradients.
#pragma once
#include "engine.cuh"

namespace thmr {

constexpr int kBwdVerts = 256;      // vertices per skinning-backward block (and per A_bar partial)
constexpr int kBwdPoses = 16;       // poses per skinning-backward block
constexpr int kBwdAStride = 13;     // floats per joint of A in smem (12 used), as smpl_skin_kernel
constexpr int kBwdCStride = 13;     // floats per vertex of g [v_posed; 1]^T in smem (12 used)
constexpr int kBlendBwdTile = 64;   // poses x features per blend-backward block
constexpr int kBlendBwdK = 32;      // k step of the blend-backward block
constexpr int kBlendBwdSplit = 32;  // split-K slices of the blend backward

// Backward workspace, carved after the forward's SmplWs.
struct SmplBwdWs {
  SmplWs fwd;
  float* vbar;       // [min(B,kSmplChunk), off_pitch]        vposed_bar of a chunk
  float* apart;      // [nvb, min(B,kSmplChunk), 24*12]        A_bar partial sums per vertex block
  float* fpart;      // [kBlendBwdSplit, min(B,kSmplChunk), 224]  feat_bar partial sums per K slice
};
inline void smpl_bwd_carve(Bump& bp, const SmplModel& m, int B, SmplBwdWs* ws) {
  smpl_carve(bp, m, B, &ws->fwd);
  const size_t nc = static_cast<size_t>(B < kSmplChunk ? B : kSmplChunk);
  const size_t nvb = (m.V + kBwdVerts - 1) / kBwdVerts;
  ws->vbar = bp.take<float>(nc * ws->fwd.off_pitch);
  ws->apart = bp.take<float>(nvb * nc * kSmplJ * 12);
  ws->fpart = bp.take<float>(static_cast<size_t>(kBlendBwdSplit) * nc * kSmplPFPad);
}

// ---- create-time: fp32 blend basis [posedirs (207 rows) ; shapedirs^T (nb rows)] at the offsets pitch -----------
__global__ void smpl_pack_basis32_kernel(const float* __restrict__ posedirs, const float* __restrict__ shapedirs,
                                         int nb, float* __restrict__ out, int V3, long pitch) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long>(kSmplFeatBeta + nb) * pitch) return;
  const int k = static_cast<int>(i / pitch);
  const int c = static_cast<int>(i % pitch);
  float v = 0.f;
  if (c < V3) v = k < kSmplPF ? posedirs[static_cast<size_t>(k) * V3 + c]
                              : shapedirs[static_cast<size_t>(c) * nb + (k - kSmplFeatBeta)];
  out[i] = v;
}

// ---- skinning backward ------------------------------------------------------------------------------------
//   gj_rows: rows of grad_joints per pose (25 + n_extra), or 0 when there is no joint cotangent for vertices
//   cx_ptr/cx_row/cx_val: per vertex, the grad_joints rows that read it and their weights (CSC, fixed order)
//   bw_ptr [nvb*24 + 1], bw_lv, bw_val: per (vertex block, joint), the block's vertices skinned to that joint (local
//   index) and their weights, in increasing vertex order
__global__ void __launch_bounds__(kBwdVerts)
smpl_skin_bwd_kernel(const int* __restrict__ w_idx, const float* __restrict__ w_val, int ell,
                     const int* __restrict__ bw_ptr, const int* __restrict__ bw_lv, const float* __restrict__ bw_val,
                     const int* __restrict__ cx_ptr, const int* __restrict__ cx_row, const float* __restrict__ cx_val,
                     const float* __restrict__ A, const float* __restrict__ vposed, long off_pitch,
                     const float* __restrict__ grad_verts, const float* __restrict__ grad_joints, int gj_rows,
                     float* __restrict__ vbar, float* __restrict__ apart, int V, int n) {
  __shared__ float sA[kBwdPoses][kSmplJ * kBwdAStride];
  __shared__ float sC[kBwdVerts * kBwdCStride];
  const int vb = blockIdx.x;
  const int p0 = blockIdx.y * kBwdPoses;
  const int np = (n - p0) < kBwdPoses ? (n - p0) : kBwdPoses;
  for (int i = threadIdx.x; i < np * kSmplJ * 12; i += kBwdVerts) {
    const int r = i % (kSmplJ * 12);
    sA[i / (kSmplJ * 12)][(r / 12) * kBwdAStride + r % 12] = A[static_cast<size_t>(p0) * kSmplJ * 12 + i];
  }
  const int v = vb * kBwdVerts + threadIdx.x;
  const bool live = v < V;
  const int c0 = live && gj_rows ? cx_ptr[v] : 0, c1 = live && gj_rows ? cx_ptr[v + 1] : 0;
  __syncthreads();
  for (int pp = 0; pp < np; ++pp) {
    const int p = p0 + pp;
    if (live) {
      float g[3] = {0.f, 0.f, 0.f};
      if (grad_verts) {
        const float* s = grad_verts + (static_cast<size_t>(p) * V + v) * 3;
        g[0] = s[0]; g[1] = s[1]; g[2] = s[2];
      }
      for (int e = c0; e < c1; ++e) {
        const float w = cx_val[e];
        const float* s = grad_joints + (static_cast<size_t>(p) * gj_rows + cx_row[e]) * 3;
        g[0] = fmaf(w, s[0], g[0]); g[1] = fmaf(w, s[1], g[1]); g[2] = fmaf(w, s[2], g[2]);
      }
      float T[12];
#pragma unroll
      for (int e = 0; e < 12; ++e) T[e] = 0.f;
      for (int k = 0; k < ell; ++k) {
        const float w = w_val[static_cast<size_t>(v) * ell + k];
        const float* a = &sA[pp][w_idx[static_cast<size_t>(v) * ell + k] * kBwdAStride];
#pragma unroll
        for (int e = 0; e < 12; ++e) T[e] = fmaf(w, a[e], T[e]);
      }
      const float* x = vposed + static_cast<size_t>(p) * off_pitch + v * 3;
      const float x0 = x[0], x1 = x[1], x2 = x[2];
      float* o = vbar + static_cast<size_t>(p) * off_pitch + v * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = T[0 * 4 + c] * g[0] + T[1 * 4 + c] * g[1] + T[2 * 4 + c] * g[2];
      float* cs = sC + threadIdx.x * kBwdCStride;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        cs[r * 4 + 0] = g[r] * x0; cs[r * 4 + 1] = g[r] * x1; cs[r * 4 + 2] = g[r] * x2; cs[r * 4 + 3] = g[r];
      }
    }
    __syncthreads();
    // A_bar partials of this vertex block: output (j, e) sums its joint's list in order
    for (int q = threadIdx.x; q < kSmplJ * 12; q += kBwdVerts) {
      const int j = q / 12, e = q % 12;
      float s = 0.f;
      for (int i = bw_ptr[vb * kSmplJ + j]; i < bw_ptr[vb * kSmplJ + j + 1]; ++i)
        s = fmaf(bw_val[i], sC[bw_lv[i] * kBwdCStride + e], s);
      apart[(static_cast<size_t>(vb) * n + p) * (kSmplJ * 12) + q] = s;
    }
    __syncthreads();
  }
}

// ---- blend backward: fpart[s, p, k] = sum_{n in slice s} vbar[p, n] basis32[k, n] --------------------------------
//   block = 64 poses x 64 features of one K slice, 256 threads x (4 x 4) outputs; k beyond 3V reads as zero
__global__ void __launch_bounds__(256)
smpl_blend_bwd_kernel(const float* __restrict__ vbar, long ldv, const float* __restrict__ basis32, long ldb,
                      int nfeat, int K3, int kslice, float* __restrict__ fpart, int n) {
  __shared__ float sV[kBlendBwdK][kBlendBwdTile + 4];
  __shared__ float sB[kBlendBwdK][kBlendBwdTile + 4];
  const int f0 = blockIdx.x * kBlendBwdTile, p0 = blockIdx.y * kBlendBwdTile, s = blockIdx.z;
  const int kb = s * kslice, ke = min(K3, kb + kslice);
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;   // features tx*4.., poses ty*4..
  float acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
  for (int k0 = kb; k0 < ke; k0 += kBlendBwdK) {
    // 64 rows x 32 k of each operand: 2048 values, 8 per thread, k fastest (coalesced rows)
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int i = it * 256 + threadIdx.x;
      const int row = i / kBlendBwdK, kk = i % kBlendBwdK, k = k0 + kk;
      const bool kin = k < ke;
      sV[kk][row] = (kin && p0 + row < n) ? vbar[static_cast<size_t>(p0 + row) * ldv + k] : 0.f;
      sB[kk][row] = (kin && f0 + row < nfeat) ? basis32[static_cast<size_t>(f0 + row) * ldb + k] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < kBlendBwdK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) { a[q] = sV[kk][ty * 4 + q]; b[q] = sB[kk][tx * 4 + q]; }
#pragma unroll
      for (int x = 0; x < 4; ++x)
#pragma unroll
        for (int y = 0; y < 4; ++y) acc[x][y] = fmaf(a[x], b[y], acc[x][y]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int x = 0; x < 4; ++x) {
    const int p = p0 + ty * 4 + x;
    if (p >= n) continue;
#pragma unroll
    for (int y = 0; y < 4; ++y) {
      const int f = f0 + tx * 4 + y;
      if (f < nfeat) fpart[(static_cast<size_t>(s) * n + p) * kSmplPFPad + f] = acc[x][y];
    }
  }
}

// ---- chain backward: warp = pose ---------------------------------------------------------------------------------
//   pose: the forward's input (axis-angle or rotation matrices); A: smpl_pose_kernel's relative transforms
//   joints_mode: 0 = grad_joints is [B, 25+n_extra, 3] over the wrapper's joints (joint_map routes rows < 25 to the
//   posed joints), 1 = grad_joints is [B, 24, 3] over J_transformed (thmr_lbs)
//   grad_pose: [B,24,3] (pose2rot) or [B,24,3,3]
__global__ void __launch_bounds__(32)
smpl_chain_bwd_kernel(const float* __restrict__ pose, int pose2rot, const float* __restrict__ betas,
                      const float* __restrict__ J_template, const float* __restrict__ J_shapedirs, int nb,
                      const int* __restrict__ parents_dev, const int* __restrict__ joint_map,
                      const float* __restrict__ A, const float* __restrict__ grad_joints, int gj_rows, int joints_mode,
                      const float* __restrict__ apart, int nvb, const float* __restrict__ fpart, int nsplit,
                      float* __restrict__ grad_pose, float* __restrict__ grad_betas, int p0, int n) {
  __shared__ float R[kSmplJ][9], Jl[kSmplJ][3], GR[kSmplJ][9];
  __shared__ float GbR[kSmplJ][9], Gbt[kSmplJ][3], Rb[kSmplJ][9], Jlb[kSmplJ][3];
  __shared__ float fb[kSmplPFPad];
  const int pl = blockIdx.x;          // pose within the chunk
  const int b = p0 + pl;              // pose within the batch
  const int j = threadIdx.x;
  const int nfeat = kSmplFeatBeta + nb;
  // feat_bar: fixed-order sum of the split-K partials
  for (int k = j; k < nfeat; k += 32) {
    float s = 0.f;
    for (int q = 0; q < nsplit; ++q) s += fpart[(static_cast<size_t>(q) * n + pl) * kSmplPFPad + k];
    fb[k] = s;
  }
  __syncwarp();
  float ax = 0.f, ay = 0.f, az = 0.f;   // axis-angle of joint j (pose2rot)
  if (j < kSmplJ) {
    // R and the joint location, as smpl_pose_kernel computes them
    float r[9];
    if (pose2rot) {
      const float* a = pose + (static_cast<size_t>(b) * kSmplJ + j) * 3;
      ax = a[0]; ay = a[1]; az = a[2];
      const float ex = ax + 1e-8f, ey = ay + 1e-8f, ez = az + 1e-8f;
      const float angle = sqrtf(ex * ex + ey * ey + ez * ez);
      const float dx = ax / angle, dy = ay / angle, dz = az / angle;
      float s, c;
      sincosf(angle, &s, &c);
      const float oc = 1.f - c;
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
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float v = J_template[j * 3 + c];
      for (int l = 0; l < nb; ++l) v += J_shapedirs[(j * 3 + c) * nb + l] * betas[static_cast<size_t>(b) * nb + l];
      Jl[j][c] = v;
    }
    // A_bar_j: fixed-order sum over the vertex blocks
    float ab[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) ab[e] = 0.f;
    for (int q = 0; q < nvb; ++q) {
      const float* s = apart + (static_cast<size_t>(q) * n + pl) * (kSmplJ * 12) + j * 12;
#pragma unroll
      for (int e = 0; e < 12; ++e) ab[e] += s[e];
    }
    // posed-joint cotangent
    float jb[3] = {0.f, 0.f, 0.f};
    if (grad_joints) {
      if (joints_mode == 1) {
        const float* s = grad_joints + (static_cast<size_t>(b) * kSmplJ + j) * 3;
        jb[0] = s[0]; jb[1] = s[1]; jb[2] = s[2];
      } else {
        for (int k = 0; k < 25; ++k) {
          if (joint_map[k] != j) continue;
          const float* s = grad_joints + (static_cast<size_t>(b) * gj_rows + k) * 3;
          jb[0] += s[0]; jb[1] += s[1]; jb[2] += s[2];
        }
      }
    }
    const float* a = A + (static_cast<size_t>(b) * kSmplJ + j) * 12;
#pragma unroll
    for (int rr = 0; rr < 3; ++rr)
#pragma unroll
      for (int c = 0; c < 3; ++c) GR[j][rr * 3 + c] = a[rr * 4 + c];
    // A_j = [G_R | G_t - G_R Jl]:  G_R_bar = A_R_bar - A_t_bar Jl^T,  G_t_bar = A_t_bar + Jposed_bar,
    // Jl_bar = -G_R^T A_t_bar
#pragma unroll
    for (int rr = 0; rr < 3; ++rr) {
#pragma unroll
      for (int c = 0; c < 3; ++c) GbR[j][rr * 3 + c] = ab[rr * 4 + c] - ab[rr * 4 + 3] * Jl[j][c];
      Gbt[j][rr] = ab[rr * 4 + 3] + jb[rr];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      Jlb[j][c] = -(a[0 * 4 + c] * ab[0 * 4 + 3] + a[1 * 4 + c] * ab[1 * 4 + 3] + a[2 * 4 + c] * ab[2 * 4 + 3]);
      // R_bar from the blend feature (R - I) of joints 1..23
#pragma unroll
      for (int e = 0; e < 3; ++e) Rb[j][c * 3 + e] = j >= 1 ? fb[(j - 1) * 9 + c * 3 + e] : 0.f;
    }
  }
  __syncwarp();
  // reverse sweep through G_i = G_p [R_i | Jl_i - Jl_p]; children have larger indices than their parents
  for (int i = kSmplJ - 1; i >= 1; --i) {
    if (j == i) {
      const int p = parents_dev[i];
      const float t[3] = {Jl[i][0] - Jl[p][0], Jl[i][1] - Jl[p][1], Jl[i][2] - Jl[p][2]};
      // R_bar_i += G_R,p^T G_R_bar_i ;  t_bar = G_R,p^T G_t_bar_i
      float tb[3];
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
          Rb[i][rr * 3 + c] += GR[p][0 * 3 + rr] * GbR[i][0 * 3 + c] + GR[p][1 * 3 + rr] * GbR[i][1 * 3 + c] +
                               GR[p][2 * 3 + rr] * GbR[i][2 * 3 + c];
        tb[rr] = GR[p][0 * 3 + rr] * Gbt[i][0] + GR[p][1 * 3 + rr] * Gbt[i][1] + GR[p][2 * 3 + rr] * Gbt[i][2];
      }
      // G_R_bar_p += G_R_bar_i R_i^T + G_t_bar_i t^T ;  G_t_bar_p += G_t_bar_i
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
          GbR[p][rr * 3 + c] += GbR[i][rr * 3 + 0] * R[i][c * 3 + 0] + GbR[i][rr * 3 + 1] * R[i][c * 3 + 1] +
                                GbR[i][rr * 3 + 2] * R[i][c * 3 + 2] + Gbt[i][rr] * t[c];
        Gbt[p][rr] += Gbt[i][rr];
        Jlb[i][rr] += tb[rr];
        Jlb[p][rr] -= tb[rr];
      }
    }
    __syncwarp();
  }
  if (j == 0) {
    // G_0 = [R_0 | Jl_0]
#pragma unroll
    for (int e = 0; e < 9; ++e) Rb[0][e] += GbR[0][e];
#pragma unroll
    for (int c = 0; c < 3; ++c) Jlb[0][c] += Gbt[0][c];
  }
  __syncwarp();
  // betas: the blend feature's shape columns + J_shapedirs^T Jl_bar
  if (j < nb) {
    float s = fb[kSmplFeatBeta + j];
    for (int jj = 0; jj < kSmplJ; ++jj)
#pragma unroll
      for (int c = 0; c < 3; ++c) s = fmaf(J_shapedirs[(jj * 3 + c) * nb + j], Jlb[jj][c], s);
    grad_betas[static_cast<size_t>(b) * nb + j] = s;
  }
  if (j < kSmplJ) {
    if (!pose2rot) {
      float* o = grad_pose + (static_cast<size_t>(b) * kSmplJ + j) * 9;
#pragma unroll
      for (int e = 0; e < 9; ++e) o[e] = Rb[j][e];
    } else {
      // Rodrigues VJP: R = I + s K + (1 - c) K K,  K = skew(d),  d = r / angle,  angle = ||r + 1e-8||
      const float ex = ax + 1e-8f, ey = ay + 1e-8f, ez = az + 1e-8f;
      const float angle = sqrtf(ex * ex + ey * ey + ez * ez);
      const float d[3] = {ax / angle, ay / angle, az / angle};
      float s, c;
      sincosf(angle, &s, &c);
      const float oc = 1.f - c;
      const float K[9] = {0.f, -d[2], d[1], d[2], 0.f, -d[0], -d[1], d[0], 0.f};
      float KK[9];
#pragma unroll
      for (int rr = 0; rr < 3; ++rr)
#pragma unroll
        for (int cc = 0; cc < 3; ++cc)
          KK[rr * 3 + cc] = K[rr * 3 + 0] * K[0 * 3 + cc] + K[rr * 3 + 1] * K[1 * 3 + cc] + K[rr * 3 + 2] * K[2 * 3 + cc];
      const float* G = Rb[j];
      float sb = 0.f, ocb = 0.f;
#pragma unroll
      for (int e = 0; e < 9; ++e) { sb = fmaf(G[e], K[e], sb); ocb = fmaf(G[e], KK[e], ocb); }
      // K_bar = s G + oc (G K^T + K^T G)
      float Kb[9];
#pragma unroll
      for (int rr = 0; rr < 3; ++rr)
#pragma unroll
        for (int cc = 0; cc < 3; ++cc) {
          float gkt = 0.f, ktg = 0.f;
#pragma unroll
          for (int m = 0; m < 3; ++m) { gkt += G[rr * 3 + m] * K[cc * 3 + m]; ktg += K[m * 3 + rr] * G[m * 3 + cc]; }
          Kb[rr * 3 + cc] = s * G[rr * 3 + cc] + oc * (gkt + ktg);
        }
      const float db[3] = {Kb[7] - Kb[5], Kb[2] - Kb[6], Kb[3] - Kb[1]};
      // angle_bar = s_bar cos + oc_bar sin - (d_bar . d) / angle
      const float angb = sb * c + ocb * s - (db[0] * d[0] + db[1] * d[1] + db[2] * d[2]) / angle;
      float* o = grad_pose + (static_cast<size_t>(b) * kSmplJ + j) * 3;
      o[0] = db[0] / angle + angb * ex / angle;
      o[1] = db[1] / angle + angb * ey / angle;
      o[2] = db[2] / angle + angb * ez / angle;
    }
  }
}

// grad_joints: [B, 25+n_extra, 3] (joints_mode 0) or [B, 24, 3] (joints_mode 1), nullable; grad_verts nullable
inline int smpl_backward_run(const thmr_smpl* sm, const float* pose, int pose2rot, const float* betas, int B,
                             const float* grad_verts, const float* grad_joints, int joints_mode, float* grad_pose,
                             float* grad_betas, const SmplBwdWs& ws, cudaStream_t st) {
  const SmplModel& m = sm->m;
  const SmplWs& fw = ws.fwd;
  smpl_pose_kernel<<<B, 32, 0, st>>>(pose, pose2rot, betas, m.J_template, m.J_shapedirs, m.nb, sm->parents_dev, fw.A,
                                     fw.Jposed, fw.pf16, B);
  THMR_CUDA(cudaGetLastError());
  const int nvb = (m.V + kBwdVerts - 1) / kBwdVerts;
  const int gj_rows = (grad_joints && joints_mode == 0) ? 25 + m.n_extra : 0;
  const int nfeat = kSmplFeatBeta + m.nb;
  const int K3 = 3 * m.V;
  const int kslice = ((K3 + kBlendBwdSplit - 1) / kBlendBwdSplit + kBlendBwdK - 1) / kBlendBwdK * kBlendBwdK;
  const int nsplit = (K3 + kslice - 1) / kslice;
  for (int p0 = 0; p0 < B; p0 += kSmplChunk) {
    const int n = (B - p0) < kSmplChunk ? (B - p0) : kSmplChunk;
    GemmPlan plan;
    THMR_TRY(smpl_blend_plan(m, fw, p0, n, &plan));
    THMR_TRY(gemm_launch(plan, st));
    const float* Ac = fw.A + static_cast<size_t>(p0) * kSmplJ * 12;
    const float* gv = grad_verts ? grad_verts + static_cast<size_t>(p0) * m.V * 3 : nullptr;
    const float* gj = gj_rows ? grad_joints + static_cast<size_t>(p0) * gj_rows * 3 : nullptr;
    smpl_skin_bwd_kernel<<<dim3(nvb, (n + kBwdPoses - 1) / kBwdPoses), kBwdVerts, 0, st>>>(
        m.w_idx, m.w_val, m.ell, m.bw_ptr, m.bw_lv, m.bw_val, m.cx_ptr, m.cx_row, m.cx_val, Ac, fw.offsets,
        fw.off_pitch, gv, gj, gj_rows, ws.vbar, ws.apart, m.V, n);
    THMR_CUDA(cudaGetLastError());
    smpl_blend_bwd_kernel<<<dim3((nfeat + kBlendBwdTile - 1) / kBlendBwdTile, (n + kBlendBwdTile - 1) / kBlendBwdTile,
                                 nsplit), 256, 0, st>>>(ws.vbar, fw.off_pitch, m.basis32, fw.off_pitch, nfeat, K3, kslice,
                                                        ws.fpart, n);
    THMR_CUDA(cudaGetLastError());
    smpl_chain_bwd_kernel<<<n, 32, 0, st>>>(pose, pose2rot, betas, m.J_template, m.J_shapedirs, m.nb, sm->parents_dev,
                                            m.joint_map, fw.A, grad_joints, 25 + m.n_extra, joints_mode,
                                            ws.apart, nvb, ws.fpart, nsplit, grad_pose, grad_betas, p0, n);
    THMR_CUDA(cudaGetLastError());
  }
  return THMR_OK;
}

}  // namespace thmr
