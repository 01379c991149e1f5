// HBM-bound row kernels: patch im2col, LayerNorm, softmax, gathers.  Warp-shuffle reductions, fp32 math,
// vectorised coalesced loads; outputs are written in the operand format of the consuming wgmma GEMM (fp16).
#pragma once
#include <stdlib.h>

#include "common.cuh"
#include "ptx.cuh"

namespace thmr {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------------
// Patch im2col (vit.py:341-343 crop + PatchEmbed conv as a GEMM, vit.py:168-175)
//   img  (B,3,S,S) fp32 NCHW, cropped to columns [x0, x0+Wc)
//   out  (B*gh*gw, 3*P*P) fp16, k = c*P*P + dy*P + dx, zero outside the cropped image (padding `pad`).
// One thread per (row, c, dy): writes P consecutive fp16 (32 B for P=16).
// ------------------------------------------------------------------------------------------------
__global__ void im2col_patch_kernel(const float* __restrict__ img, __half* __restrict__ out, int B, int S, int x0,
                                    int Wc, int P, int pad, int gh, int gw, unsigned long long* stamp) {
  stamp_start(stamp);
  const long total = static_cast<long>(B) * gh * gw * 3 * P;
  const long t = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (t >= total) return;
  const int dy = t % P;
  const int c = (t / P) % 3;
  const long row = t / (3 * P);
  const int j = row % gw;
  const int i = (row / gw) % gh;
  const int b = row / (static_cast<long>(gw) * gh);
  const int y = i * P - pad + dy;
  __half* o = out + row * (3 * P * P) + c * P * P + dy * P;
  const float* src = img + ((static_cast<long>(b) * 3 + c) * S + y) * S + x0;
  for (int dx = 0; dx < P; ++dx) {
    const int x = j * P - pad + dx;
    float v = 0.f;
    if (y >= 0 && y < S && x >= 0 && x < Wc) v = src[x];
    o[dx] = __float2half_rn(v);
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over the last dimension (nn.LayerNorm: biased variance, eps inside the sqrt).
//   x (R,C) fp32 -> y16 (fp16, nullable) and/or y32 (fp32, nullable); optional ReLU (FCBlock, modules.py:15-19).
//   One warp per row; the row lives in registers (C <= 32*4*VEC4 elements), two-pass statistics.
//   out_t > 0: outputs (fp16 and fp32) written transposed inside groups of out_t rows:
//       y16[(r / T) * C * T + c * T + (r % T)]   (MixerLayer token mixing, modules.py:56-59)
//   Row pitch of the fp16 output is ld16 (elements) when not transposed.
// ------------------------------------------------------------------------------------------------
// PLAIN16: the ViT's case (fp16 output only, no ReLU, not transposed, C == 128 * VEC4 exactly), compiled without the other
// output modes' branches and without the per-chunk column guards.
template <int VEC4, bool PREFETCH, bool PLAIN16 = false>  // float4 loads per lane; PREFETCH: the next row's loads are issued before this row's math
__global__ void __launch_bounds__(256, VEC4 > 10 ? (PREFETCH ? 1 : 2) : (PREFETCH ? 2 : 4))
layernorm_reg_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                     __half* __restrict__ y16, int ld16, float* __restrict__ y32_, int R, int C_, float eps, int relu_,
                     int out_t_, unsigned long long* stamp) {
  const int C = PLAIN16 ? VEC4 * 128 : C_;
  float* const y32 = PLAIN16 ? nullptr : y32_;
  const int relu = PLAIN16 ? 0 : relu_;
  const int out_t = PLAIN16 ? 0 : out_t_;
  stamp_start(stamp);
  // gamma/beta staged in shared memory once per (persistent) block: read from global inside the output loop they
  // were the largest stall of the kernel (an L2-latency load per 4 outputs, after the reductions)
  extern __shared__ float4 s_gb[];   // [2][C/4]
  float4* sg = s_gb;
  float4* sb = s_gb + C / 4;
  pdl_launch_dependents();
  for (int c = threadIdx.x; c < C / 4; c += blockDim.x) {
    sg[c] = reinterpret_cast<const float4*>(gamma)[c];
    sb[c] = reinterpret_cast<const float4*>(beta)[c];
  }
  __syncthreads();
  pdl_wait();       // gamma / beta are weights; x is the predecessor's output
  const int lane = threadIdx.x & 31;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  auto load_row = [&](float4 (&v)[VEC4], int row) {
    const float* xr = x + static_cast<size_t>(row) * C;
#pragma unroll
    for (int i = 0; i < VEC4; ++i) {
      const int c = (i * 32 + lane) * 4;
      v[i] = (PLAIN16 || c < C) ? *reinterpret_cast<const float4*>(xr + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  // persistent warps: the grid is sized to the resident capacity and every warp walks rows with a grid stride
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  float4 v[VEC4];
  if (PREFETCH && warp < R) load_row(v, warp);
  for (; warp < R; warp += warps_total) {
    float4 nx[VEC4];
    if (PREFETCH) {
      if (warp + warps_total < R) load_row(nx, warp + warps_total);
    } else {
      load_row(v, warp);
    }
    // Two partial sums per lane (even / odd columns) for the mean and the variance.
    // Rows shorter than the register tile hold zeros beyond C (they add 0 to the sum; the variance pass masks them).
    float s_lo = 0.f, s_hi = 0.f;
#pragma unroll
    for (int i = 0; i < VEC4; ++i) {
      s_lo += v[i].x; s_hi += v[i].y;
      s_lo += v[i].z; s_hi += v[i].w;
    }
    const float mean = warp_sum(s_lo + s_hi) / C;
    float q_lo = 0.f, q_hi = 0.f;
#pragma unroll
    for (int i = 0; i < VEC4; ++i) {
      const int c = (i * 32 + lane) * 4;
      if (PLAIN16 || c < C) {
        const float d0 = v[i].x - mean, d1 = v[i].y - mean, d2 = v[i].z - mean, d3 = v[i].w - mean;
        q_lo = fmaf(d0, d0, q_lo); q_hi = fmaf(d1, d1, q_hi);
        q_lo = fmaf(d2, d2, q_lo); q_hi = fmaf(d3, d3, q_hi);
      }
    }
    const float rstd = rsqrtf(warp_sum(q_lo + q_hi) / C + eps);
#pragma unroll
    for (int i = 0; i < VEC4; ++i) {
      const int c = (i * 32 + lane) * 4;
      if (PLAIN16 || c < C) {
        const float4 g = sg[c >> 2];
        const float4 bb = sb[c >> 2];
        // ((x - mean) * rstd) * g + b, the reference's order of operations
        float4 o;
        o.x = fmaf((v[i].x - mean) * rstd, g.x, bb.x);
        o.y = fmaf((v[i].y - mean) * rstd, g.y, bb.y);
        o.z = fmaf((v[i].z - mean) * rstd, g.z, bb.z);
        o.w = fmaf((v[i].w - mean) * rstd, g.w, bb.w);
        if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
        if (y32) {
          if (out_t > 0) {   // transposed inside groups of out_t rows, like the fp16 output (strict mode operand)
            float* base = y32 + static_cast<size_t>(warp / out_t) * C * out_t + (warp % out_t);
            base[static_cast<size_t>(c) * out_t] = o.x;
            base[static_cast<size_t>(c + 1) * out_t] = o.y;
            base[static_cast<size_t>(c + 2) * out_t] = o.z;
            base[static_cast<size_t>(c + 3) * out_t] = o.w;
          } else {
            *reinterpret_cast<float4*>(y32 + static_cast<size_t>(warp) * C + c) = o;
          }
        }
        if (y16) {
          if (out_t > 0) {
            __half* base = y16 + static_cast<size_t>(warp / out_t) * C * out_t + (warp % out_t);
            base[static_cast<size_t>(c) * out_t] = __float2half_rn(o.x);
            base[static_cast<size_t>(c + 1) * out_t] = __float2half_rn(o.y);
            base[static_cast<size_t>(c + 2) * out_t] = __float2half_rn(o.z);
            base[static_cast<size_t>(c + 3) * out_t] = __float2half_rn(o.w);
          } else {
            __half2 h0 = __floats2half2_rn(o.x, o.y), h1 = __floats2half2_rn(o.z, o.w);
            uint2 pk;
            pk.x = *reinterpret_cast<uint32_t*>(&h0);
            pk.y = *reinterpret_cast<uint32_t*>(&h1);
            *reinterpret_cast<uint2*>(y16 + static_cast<size_t>(warp) * ld16 + c) = pk;
          }
        }
      }
    }
    if (PREFETCH) {
#pragma unroll
      for (int i = 0; i < VEC4; ++i) v[i] = nx[i];
    }
  }
}

// Wide rows (C up to 64K, e.g. the 10240-wide FCBlock norm): one block per row, three passes over L1/L2.
__global__ void __launch_bounds__(256)
layernorm_wide_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                      __half* __restrict__ y16, int ld16, float* __restrict__ y32, int R, int C, float eps, int relu,
                      unsigned long long* stamp) {
  stamp_start(stamp);
  __shared__ float red[8];
  __shared__ float bcast;
  const int row = blockIdx.x;
  const float* xr = x + static_cast<size_t>(row) * C;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  auto block_sum = [&](float v) -> float {
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int i = 0; i < 8; ++i) t += red[i];
      bcast = t;
    }
    __syncthreads();
    return bcast;
  };
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += 256) s += xr[c];
  const float mean = block_sum(s) / C;
  float q = 0.f;
  for (int c = threadIdx.x; c < C; c += 256) { const float d = xr[c] - mean; q += d * d; }
  const float rstd = rsqrtf(block_sum(q) / C + eps);
  for (int c = threadIdx.x; c < C; c += 256) {
    float o = (xr[c] - mean) * rstd * gamma[c] + beta[c];
    if (relu) o = fmaxf(o, 0.f);
    if (y32) y32[static_cast<size_t>(row) * C + c] = o;
    if (y16) y16[static_cast<size_t>(row) * ld16 + c] = __float2half_rn(o);
  }
}

inline int layernorm_launch(const float* x, const float* gamma, const float* beta, __half* y16, int ld16, float* y32,
                            int R, int C, float eps, int relu, int out_t, cudaStream_t st,
                            unsigned long long* stamp = nullptr) {
  THMR_CHECK(C % 4 == 0, "layernorm: C=%d not a multiple of 4", C);
  if (ld16 == 0) ld16 = C;
  if (C <= 2048) {
    static const int prefetch = [] { const char* e = getenv("THMR_LN_PREFETCH"); return e ? atoi(e) : 0; }();
    static const int env_shape = [] { const char* e = getenv("THMR_LN_SHAPE"); return e ? atoi(e) : 0; }();
    // Persistent warps walk the rows with a grid stride, so the launch shape decides how evenly the rows divide.
    // THMR_LN_SHAPE=1 picks, among fully resident shapes, the one with the fewest idle warp-rounds; the fixed 256 x 4
    // shape is the default.
    int threads = 256, bps = prefetch ? 2 : 4;
    if (env_shape && !prefetch) {
      double best = -1.0;
      const int cand[8][2] = {{256, 4}, {256, 3}, {128, 8}, {128, 7}, {128, 6}, {128, 5}, {256, 2}, {128, 4}};
      for (const auto& cnd : cand) {
        const long W = static_cast<long>(num_sms()) * cnd[1] * (cnd[0] / 32);
        const long rounds = (R + W - 1) / W;
        // efficiency of the last round, discounted a little for low occupancy (latency hiding)
        const double eff = static_cast<double>(R) / (rounds * W) * (W >= 24L * num_sms() ? 1.0 : 0.97);
        if (eff > best + 1e-3) { best = eff; threads = cnd[0]; bps = cnd[1]; }
      }
    }
    const int rows_per_block = threads / 32;
    int grid = (R + rows_per_block - 1) / rows_per_block;
    const int resident = num_sms() * bps;
    if (grid > resident) grid = resident;
    THMR_CHECK(C % 4 == 0, "layernorm: C must be a multiple of 4");
    const size_t smem = 2 * static_cast<size_t>(C) * sizeof(float);
    const int vec4 = (C / 4 + 31) / 32;
    const bool plain16 = y16 && !y32 && !relu && out_t == 0 && C == 128 * vec4 && !prefetch;
#define THMR_LN_LAUNCH(V)                                                                                           \
  do {                                                                                                             \
    if (prefetch) THMR_CUDA(launch_pdl(layernorm_reg_kernel<V, true>, grid, threads, smem, st, x, gamma, beta, y16, \
                                       ld16, y32, R, C, eps, relu, out_t, stamp));                                 \
    else if (plain16 && V == vec4) THMR_CUDA(launch_pdl(layernorm_reg_kernel<V, false, true>, grid, threads, smem,  \
                                       st, x, gamma, beta, y16, ld16, y32, R, C, eps, relu, out_t, stamp));        \
    else THMR_CUDA(launch_pdl(layernorm_reg_kernel<V, false>, grid, threads, smem, st, x, gamma, beta, y16, ld16,   \
                              y32, R, C, eps, relu, out_t, stamp));                                                \
  } while (0)
    if (vec4 <= 1) THMR_LN_LAUNCH(1);
    else if (vec4 <= 8) THMR_LN_LAUNCH(8);
    else if (vec4 <= 10) THMR_LN_LAUNCH(10);
    else THMR_LN_LAUNCH(16);
#undef THMR_LN_LAUNCH
  } else {
    THMR_CHECK(out_t == 0, "layernorm: transposed output needs C <= 2048");
    layernorm_wide_kernel<<<R, 256, 0, st>>>(x, gamma, beta, y16, ld16, y32, R, C, eps, relu, stamp);
  }
  THMR_CUDA(cudaGetLastError());
  return THMR_OK;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm with an e4m3 output: the FP8 A operand of the ViT's QKV and fc1 GEMMs.  Same two-pass fp32 statistics and
// output expression as layernorm_reg_kernel; C = 128 * VEC4, so the lane's float4 i of the row lies in 128-column group
// i.  Per (row, group): s = the smallest power of two with amax / s <= 448, codes = cvt.rn.satfinite(y / s), scales to
// ys[group * lds + row] (the k-block-major layout of GemmParams::a_scale).  y32 (nullable) receives the fp32 values
// before quantisation.
template <int VEC4>
__global__ void __launch_bounds__(256)
layernorm_e4m3_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                      uint8_t* __restrict__ y8, float* __restrict__ ys, int lds, float* __restrict__ y32, int R,
                      float eps, unsigned long long* stamp) {
  constexpr int C = VEC4 * 128;
  stamp_start(stamp);
  extern __shared__ float4 s_gb[];   // [2][C/4]
  float4* sg = s_gb;
  float4* sb = s_gb + C / 4;
  for (int c = threadIdx.x; c < C / 4; c += blockDim.x) {
    sg[c] = reinterpret_cast<const float4*>(gamma)[c];
    sb[c] = reinterpret_cast<const float4*>(beta)[c];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warps_total = (gridDim.x * blockDim.x) >> 5;
  for (int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; warp < R; warp += warps_total) {
    const float* xr = x + static_cast<size_t>(warp) * C;
    float4 v[VEC4];
#pragma unroll
    for (int i = 0; i < VEC4; ++i) v[i] = *reinterpret_cast<const float4*>(xr + (i * 32 + lane) * 4);
    float s_lo = 0.f, s_hi = 0.f;
#pragma unroll
    for (int i = 0; i < VEC4; ++i) {
      s_lo += v[i].x; s_hi += v[i].y;
      s_lo += v[i].z; s_hi += v[i].w;
    }
    const float mean = warp_sum(s_lo + s_hi) / C;
    float q_lo = 0.f, q_hi = 0.f;
#pragma unroll
    for (int i = 0; i < VEC4; ++i) {
      const float d0 = v[i].x - mean, d1 = v[i].y - mean, d2 = v[i].z - mean, d3 = v[i].w - mean;
      q_lo = fmaf(d0, d0, q_lo); q_hi = fmaf(d1, d1, q_hi);
      q_lo = fmaf(d2, d2, q_lo); q_hi = fmaf(d3, d3, q_hi);
    }
    const float rstd = rsqrtf(warp_sum(q_lo + q_hi) / C + eps);
#pragma unroll
    for (int i = 0; i < VEC4; ++i) {
      const int c = (i * 32 + lane) * 4;
      const float4 g = sg[c >> 2];
      const float4 bb = sb[c >> 2];
      float4 o;
      o.x = fmaf((v[i].x - mean) * rstd, g.x, bb.x);
      o.y = fmaf((v[i].y - mean) * rstd, g.y, bb.y);
      o.z = fmaf((v[i].z - mean) * rstd, g.z, bb.z);
      o.w = fmaf((v[i].w - mean) * rstd, g.w, bb.w);
      if (y32) *reinterpret_cast<float4*>(y32 + static_cast<size_t>(warp) * C + c) = o;
      const float s = e4m3_scale(warp_max(fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w)))));
      const float inv = 1.0f / s;
      const uint32_t q = cvt_e4m3x2(o.x * inv, o.y * inv) | (static_cast<uint32_t>(cvt_e4m3x2(o.z * inv, o.w * inv)) << 16);
      *reinterpret_cast<uint32_t*>(y8 + static_cast<size_t>(warp) * C + c) = q;
      if (lane == 0) ys[static_cast<size_t>(i) * lds + warp] = s;
    }
  }
}

inline int layernorm_e4m3_launch(const float* x, const float* gamma, const float* beta, uint8_t* y8, float* ys, int lds,
                                 float* y32, int R, int C, float eps, cudaStream_t st,
                                 unsigned long long* stamp = nullptr) {
  THMR_CHECK(C == 1280 || C == 1024 || C == 128, "layernorm e4m3: C=%d (128, 1024 or 1280)", C);
  THMR_CHECK(lds >= R, "layernorm e4m3: scale pitch %d < rows %d", lds, R);
  int grid = (R + 7) / 8;
  if (grid > num_sms() * 4) grid = num_sms() * 4;
  const size_t smem = 2 * static_cast<size_t>(C) * sizeof(float);
  if (C == 1280) layernorm_e4m3_kernel<10><<<grid, 256, smem, st>>>(x, gamma, beta, y8, ys, lds, y32, R, eps, stamp);
  else if (C == 1024) layernorm_e4m3_kernel<8><<<grid, 256, smem, st>>>(x, gamma, beta, y8, ys, lds, y32, R, eps, stamp);
  else layernorm_e4m3_kernel<1><<<grid, 256, smem, st>>>(x, gamma, beta, y8, ys, lds, y32, R, eps, stamp);
  THMR_CUDA(cudaGetLastError());
  return THMR_OK;
}

// ------------------------------------------------------------------------------------------------
// Row softmax over C = 32*4*VEC4 classes (token_classifier.py:104): logits fp32 -> probs fp32 (the
// cls_logits_softmax output) + an fp16 copy laid out for the soft-codebook GEMM (quantize_cnn.py:92-93),
// whose rows live in zero-padded sequences: row r = b*T + t  ->  p16 row b*pitch + lo + t.
// ------------------------------------------------------------------------------------------------
template <int VEC4>
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ logits, float* __restrict__ p32, __half* __restrict__ p16, int R, int C,
                    int T, int pitch, int lo) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= R) return;
  const float* xr = logits + static_cast<size_t>(warp) * C;
  float4 v[VEC4];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < VEC4; ++i) {
    const int c = (i * 32 + lane) * 4;
    v[i] = (c < C) ? *reinterpret_cast<const float4*>(xr + c) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    m = fmaxf(m, fmaxf(fmaxf(v[i].x, v[i].y), fmaxf(v[i].z, v[i].w)));
  }
  m = warp_max(m);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VEC4; ++i) {
    v[i].x = expf(v[i].x - m); v[i].y = expf(v[i].y - m); v[i].z = expf(v[i].z - m); v[i].w = expf(v[i].w - m);
    s += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  const float inv = 1.0f / warp_sum(s);
  const size_t prow = (T > 0) ? (static_cast<size_t>(warp / T) * pitch + lo + warp % T) : warp;
#pragma unroll
  for (int i = 0; i < VEC4; ++i) {
    const int c = (i * 32 + lane) * 4;
    if (c < C) {
      float4 o = make_float4(v[i].x * inv, v[i].y * inv, v[i].z * inv, v[i].w * inv);
      if (p32) *reinterpret_cast<float4*>(p32 + static_cast<size_t>(warp) * C + c) = o;
      if (p16) {
        __half2 h0 = __floats2half2_rn(o.x, o.y), h1 = __floats2half2_rn(o.z, o.w);
        uint2 pk;
        pk.x = *reinterpret_cast<uint32_t*>(&h0);
        pk.y = *reinterpret_cast<uint32_t*>(&h1);
        *reinterpret_cast<uint2*>(p16 + prow * C + c) = pk;
      }
    }
  }
}

inline int softmax_rows_launch(const float* logits, float* p32, __half* p16, int R, int C, int T, int pitch, int lo,
                               cudaStream_t st) {
  THMR_CHECK(C % 4 == 0 && C <= 2048, "softmax: C=%d unsupported", C);
  const int grid = (R + 7) / 8;
  softmax_rows_kernel<16><<<grid, 256, 0, st>>>(logits, p32, p16, R, C, T, pitch, lo);
  THMR_CUDA(cudaGetLastError());
  return THMR_OK;
}

// ------------------------------------------------------------------------------------------------
// nn.Upsample(size) nearest on zero-padded channels-last sequences (vanilla_pose_vqvae.py:139-141):
//   dst (B, Lout + 2*pad, C) <- src (B, Lin + 2*pad, C),   dst[b, pad + j] = src[b, pad + idx[j]]
// idx[j] = floor(j * (Lin/Lout)) computed in fp32 like ATen's legacy 'nearest'.  Pad rows are zeroed.
// ------------------------------------------------------------------------------------------------
__global__ void upsample_rows_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int B, int Lin, int Lout,
                                     int pad, int C8 /* C/8 */) {
  const long total = static_cast<long>(B) * (Lout + 2 * pad) * C8;
  const long t = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (t >= total) return;
  const int c8 = t % C8;
  const long row = t / C8;
  const int r = row % (Lout + 2 * pad);
  const int b = row / (Lout + 2 * pad);
  uint4 v = make_uint4(0, 0, 0, 0);
  if (r >= pad && r < pad + Lout) {
    const float scale = static_cast<float>(Lin) / static_cast<float>(Lout);
    int si = static_cast<int>(floorf(static_cast<float>(r - pad) * scale));
    si = si < Lin - 1 ? si : Lin - 1;
    v = reinterpret_cast<const uint4*>(src)[(static_cast<long>(b) * (Lin + 2 * pad) + pad + si) * C8 + c8];
  }
  reinterpret_cast<uint4*>(dst)[row * C8 + c8] = v;
}

// Mixer glue (modules.py:55-63):  out = x + y^T (+ z), where yT (B, H, T) fp32 is the token-mix MLP output
// in its transposed layout and z (B*T, H) fp32 the channel-mix output.  x, out: (B*T, H).
__global__ void mixer_add_kernel(const float* __restrict__ x, const float* __restrict__ yT, const float* __restrict__ z,
                                 float* __restrict__ out, int B, int T, int H) {
  const long total = static_cast<long>(B) * T * H;
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= total) return;
  const int h = i % H;
  const int t = (i / H) % T;
  const int b = i / (static_cast<long>(H) * T);
  float v = x[i] + yT[(static_cast<long>(b) * H + h) * T + t];
  if (z) v += z[i];
  out[i] = v;
}

// fp32 -> fp16 cast (GEMM operand format), 4 elements per thread.
__global__ void cast_f16_kernel(const float* __restrict__ in, __half* __restrict__ out, long n4) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i >= n4) return;
  const float4 v = reinterpret_cast<const float4*>(in)[i];
  __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
  uint2 pk;
  pk.x = *reinterpret_cast<uint32_t*>(&h0);
  pk.y = *reinterpret_cast<uint32_t*>(&h1);
  reinterpret_cast<uint2*>(out)[i] = pk;
}

// Broadcast one fp32 row to R rows (the constant decoder query token, pose_transformer.py:350,354).
__global__ void broadcast_row_kernel(const float* __restrict__ row, float* __restrict__ out, int R, int C) {
  const long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x;
  if (i < static_cast<long>(R) * C) out[i] = row[i % C];
}

}  // namespace thmr
