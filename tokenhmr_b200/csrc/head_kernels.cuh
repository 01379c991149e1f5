// Small per-image kernels of the SMPL heads: one-query cross-attention and the read-out assembly.
#pragma once
#include "common.cuh"
#include "elementwise.cuh"

namespace thmr {

// CrossAttention core for a single query token (pose_transformer.py:111-124):
//   dots = (q . k_j) * dim_head^-0.5 over the T context tokens, softmax, out = sum_j p_j v_j.
// q (B, H*64) fp32; K/V fp16 rows of the batched to_kv GEMM output: kv[(b*T + j) * ld + koff + h*64 + d],
// V at +voff.  One block per (image, head) so that B*H blocks cover the chip; thread j scores key j
// (one 128-byte row read per thread), then 64 threads accumulate the 64 output dims over all keys
// (coalesced 128-byte reads per key).  dim_head = 64 fixed.  out (B, H*64) fp16.
template <int T>
__global__ void __launch_bounds__(T)
dec_cross_attn_kernel(const float* __restrict__ q, const __half* __restrict__ kv, int ld, int koff, int voff,
                      float scale, __half* __restrict__ out, int heads) {
  __shared__ float sq[64];
  __shared__ float sp[T];
  __shared__ float red[T / 32];
  __shared__ float so[T / 64][64];
  const int b = blockIdx.x / heads;
  const int h = blockIdx.x % heads;
  const int j = threadIdx.x;
  const int lane = j & 31, w = j >> 5;
  const int inner = heads * 64;
  if (j < 64) sq[j] = q[static_cast<size_t>(b) * inner + h * 64 + j];
  __syncthreads();
  const __half* kr = kv + (static_cast<size_t>(b) * T + j) * ld + koff + h * 64;
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < 64; c += 8) {
    const uint4 pk = *reinterpret_cast<const uint4*>(kr + c);
    const __half2* h2 = reinterpret_cast<const __half2*>(&pk);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(h2[e]);
      s += sq[c + 2 * e] * f.x + sq[c + 2 * e + 1] * f.y;
    }
  }
  s *= scale;
  float m = warp_max(s);
  if (lane == 0) red[w] = m;
  __syncthreads();
  m = red[0];
#pragma unroll
  for (int i = 1; i < T / 32; ++i) m = fmaxf(m, red[i]);
  const float e = expf(s - m);
  float sum = warp_sum(e);
  __syncthreads();
  if (lane == 0) red[w] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < T / 32; ++i) sum += red[i];
  sp[j] = e / sum;
  __syncthreads();
  // out[d] = sum_j p_j v[j][d]: T/64 key groups x 64 dims, then a final reduction over the groups
  const int d = j & 63, g = j >> 6;
  const __half* vb = kv + static_cast<size_t>(b) * T * ld + voff + h * 64 + d;
  float o = 0.f;
  for (int k = g; k < T; k += T / 64) o += sp[k] * __half2float(vb[static_cast<size_t>(k) * ld]);
  so[g][d] = o;
  __syncthreads();
  if (j < 64) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < T / 64; ++i) t += so[i][j];
    out[static_cast<size_t>(b) * inner + h * 64 + j] = __float2half_rn(t);
  }
}

// rot6d_to_rotmat (geometry.py:64-84) of one 6D vector: x.reshape(2,3).permute -> a1 = x[0:3], a2 = x[3:6];
// F.normalize eps = 1e-12; R rows b1, b2, b3 = b1 x b2.  The one copy of this arithmetic: the read-out assembly of
// both heads and the stand-alone operator call it.
__device__ __forceinline__ void rot6d_to_rotmat_one(const float* x, float* R) {
  const float n1 = fmaxf(sqrtf(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]), 1e-12f);
  const float b1x = x[0] / n1, b1y = x[1] / n1, b1z = x[2] / n1;
  const float dp = b1x * x[3] + b1y * x[4] + b1z * x[5];
  const float ux = x[3] - dp * b1x, uy = x[4] - dp * b1y, uz = x[5] - dp * b1z;
  const float n2 = fmaxf(sqrtf(ux * ux + uy * uy + uz * uz), 1e-12f);
  const float b2x = ux / n2, b2y = uy / n2, b2z = uz / n2;
  R[0] = b1x; R[1] = b1y; R[2] = b1z;
  R[3] = b2x; R[4] = b2y; R[5] = b2z;
  R[6] = b1y * b2z - b1z * b2y;
  R[7] = b1z * b2x - b1x * b2z;
  R[8] = b1x * b2y - b1y * b2x;
}

// Read-out assembly + rot6d_to_rotmat, for both SMPL heads.
//   token head (bpose != NULL; token_head.py:99-105,123-128):
//     readout (B, ld_r) fp32 = [grot(6) | hands(12) | betas(10) | cam(3)] linear outputs (bias included)
//     bpose   rows (b*pitch + lo + j), 6 floats each: tokenizer decoder output for the 21 body joints
//     pose6d = cat[grot, bpose(126), hands] + init_pose
//   regression head (bpose == NULL; smpl_head.py:82-84,89-105):
//     readout (B, ld_r) fp32 = [pose(144) | betas(10) | cam(3)];  pose6d = pose + init_pose
//   both: betas += init_betas;  cam += init_cam
// One thread per (image, joint).
__global__ void head_assemble_kernel(const float* __restrict__ readout, int ld_r, const float* __restrict__ bpose,
                                     int ld_b, int pitch, int lo, const float* __restrict__ init_pose,
                                     const float* __restrict__ init_betas, const float* __restrict__ init_cam,
                                     float* __restrict__ rotmats, float* __restrict__ betas, float* __restrict__ cam,
                                     float* __restrict__ pose6d_out, int B, int nb) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * 24) return;
  const int b = t / 24, j = t % 24;
  const float* r = readout + static_cast<size_t>(b) * ld_r;
  float x[6];
  if (!bpose) {
#pragma unroll
    for (int e = 0; e < 6; ++e) x[e] = r[j * 6 + e];
  } else if (j == 0) {
#pragma unroll
    for (int e = 0; e < 6; ++e) x[e] = r[e];
  } else if (j <= 21) {
    const float* s = bpose + (static_cast<size_t>(b) * pitch + lo + (j - 1)) * ld_b;
#pragma unroll
    for (int e = 0; e < 6; ++e) x[e] = s[e];
  } else {
#pragma unroll
    for (int e = 0; e < 6; ++e) x[e] = r[6 + (j - 22) * 6 + e];
  }
#pragma unroll
  for (int e = 0; e < 6; ++e) x[e] += init_pose[j * 6 + e];
  if (pose6d_out) {
#pragma unroll
    for (int e = 0; e < 6; ++e) pose6d_out[static_cast<size_t>(b) * 144 + j * 6 + e] = x[e];
  }
  rot6d_to_rotmat_one(x, rotmats + static_cast<size_t>(t) * 9);
  if (j == 0) {
    const int rb = bpose ? 18 : 144;   // first betas column of the read-out
    for (int l = 0; l < nb; ++l) betas[static_cast<size_t>(b) * nb + l] = r[rb + l] + init_betas[l];
    for (int e = 0; e < 3; ++e) cam[b * 3 + e] = r[rb + 10 + e] + init_cam[e];
  }
}

// Stand-alone rot6d_to_rotmat (geometry.py:64-84): x (N,6) -> R (N,3,3), rows b1, b2, b3.
__global__ void rot6d_kernel(const float* __restrict__ x6, float* __restrict__ rot, long N) {
  const long t = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (t >= N) return;
  rot6d_to_rotmat_one(x6 + t * 6, rot + t * 9);
}

}  // namespace thmr
