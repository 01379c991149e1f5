// Training HMR 2.0's regression head (SMPLTransformerDecoderHead, heads/smpl_head.py:52-105 with IEF_ITERS 1,
// TRANSFORMER_INPUT 'zero', JOINT_REP '6d'): an fp32 forward that keeps what the backward needs, and the backward to
// every parameter (thmr_reg_head_train_forward / thmr_reg_head_backward).  No gradient for the features.
//
// The query length is 1, so the cross-attention never needs K or V.  For layer l, head h, image b, with query q (64)
// and context X_b (192 x 1280, read channel-first from the backbone's (B,1280,16,12) features):
//   forward   kq = W_k,h^T q;  s = scale X_b kq;  P = softmax(s);  c = X_b^T P;  o = W_v,h c
//   backward  d~ = W_v,h^T dO;  dP = X_b d~;  dS = P (dP - delta), delta = dO . o (= d~ . c);  u = X_b^T dS
//             dq = scale W_k,h u;  dW_k,h = scale sum_b q (x) u;  dW_v,h = sum_b dO (x) c
// One pass over X_b per layer and direction: each image's 192 positions are split over kRhChunks CTAs, which stage
// their 1280 x 16 slice in shared memory, take the per-position dot products, and write a partial (flash-decoding:
// local max and sum in the forward); a combine kernel merges the chunks in a fixed order.
//
// The token-side linears (M = B rows) and every weight gradient (K = B) go through one tiled fp32 kernel
// (hl_gemm_kernel) in three operand orientations: x W^T, dY W and dY^T X.  Small grids split K and reduce the
// partials in a fixed order, so a step uses no float atomics, is deterministic, and a graph replay equals eager.
//
// The decoder part (rh_layout_decoder, rh_decoder_forward, rh_decoder_backward) is shared with the token head
// (token_head_train.cuh), which has the same TransformerDecoder under the same transformer.* names.
#pragma once
#include <math.h>

#include "common.cuh"
#include "head_kernels.cuh"
#include "strict.cuh"

namespace thmr {

constexpr int kRhDim = 1024;       // decoder width (smpl_head.py:26 dim=1024)
constexpr int kRhDimHead = 64;     // TRANSFORMER_DECODER.dim_head
constexpr int kRhCtx = 1280;       // context_dim: the ViT-H width
constexpr int kRhTokens = 192;     // 16 x 12 positions
constexpr int kRhMaxHeads = 8;
constexpr int kRhPose = 144, kRhBetas = 10, kRhCam = 3, kRhReadLd = 160;
constexpr int kRhChunk = 16;                               // positions per CTA
constexpr int kRhChunks = kRhTokens / kRhChunk;           // 12
constexpr int kRhPitch = kRhChunk + 4;                    // padded smem row: conflict-free float4 reads
constexpr float kRhLnEps = 1e-5f;

// ------------------------------------------------------------------------------------------------ parameter layout
// The one list of the head's parameters, in SMPLTransformerDecoderHead.named_parameters() order, with their
// state_dict names.  Every parameter starts on a 64-float boundary of the flat buffer.
struct RhParam {
  char name[96];
  int ndim;
  long long shape[3];
  long long offset, numel;
};

enum RhLayerSlot {
  kL0g, kL0b, kQkv, kSaOw, kSaOb, kL1g, kL1b, kKv, kQ, kCaOw, kCaOb, kL2g, kL2b, kF1w, kF1b, kF2w, kF2b, kLayerSlots
};
enum RhTopSlot { kPos, kTokW, kTokB };
constexpr int kRhTop = 3, kRhTail = 6;   // pos/token embedding first, then the three read-outs' weight and bias

inline int rh_num_params(int depth) { return kRhTop + depth * kLayerSlots + kRhTail; }
inline int rh_decoder_params(int depth) { return kRhTop + depth * kLayerSlots; }

// One layout entry: name, shape and the next 64-float boundary at or after off.
inline void rh_set_param(RhParam* q, const char* name, int nd, long long a, long long b, long long c, long long* off) {
  *q = RhParam{};
  snprintf(q->name, sizeof(q->name), "%s", name);
  q->ndim = nd;
  q->shape[0] = a; q->shape[1] = b; q->shape[2] = c;
  q->numel = a * (nd > 1 ? b : 1) * (nd > 2 ? c : 1);
  q->offset = *off;
  *off += (q->numel + 63) / 64 * 64;
}

// The decoder's parameters (the transformer.* names both SMPL heads share), out[0 .. rh_decoder_params(depth)).
// Returns the offset after the last one.
inline long long rh_layout_decoder(int depth, int heads, int mlp, RhParam* out) {
  const long long E = kRhDim, I = static_cast<long long>(heads) * kRhDimHead, C = kRhCtx, M = mlp;
  long long off = 0;
  rh_set_param(&out[kPos], "transformer.pos_embedding", 3, 1, 1, E, &off);
  rh_set_param(&out[kTokW], "transformer.to_token_embedding.weight", 2, E, 1, 0, &off);
  rh_set_param(&out[kTokB], "transformer.to_token_embedding.bias", 1, E, 0, 0, &off);
  static const char* const sfx[kLayerSlots] = {
      "0.norm.weight", "0.norm.bias", "0.fn.to_qkv.weight", "0.fn.to_out.0.weight", "0.fn.to_out.0.bias",
      "1.norm.weight", "1.norm.bias", "1.fn.to_kv.weight", "1.fn.to_q.weight", "1.fn.to_out.0.weight",
      "1.fn.to_out.0.bias", "2.norm.weight", "2.norm.bias", "2.fn.net.0.weight", "2.fn.net.0.bias",
      "2.fn.net.3.weight", "2.fn.net.3.bias"};
  const long long r2[kLayerSlots][2] = {{E, 0}, {E, 0}, {3 * I, E}, {E, I}, {E, 0}, {E, 0}, {E, 0}, {2 * I, C},
                                        {I, E}, {E, I}, {E, 0}, {E, 0}, {E, 0}, {M, E}, {M, 0}, {E, M}, {E, 0}};
  char nm[96];
  for (int l = 0; l < depth; ++l)
    for (int s = 0; s < kLayerSlots; ++s) {
      snprintf(nm, sizeof(nm), "transformer.transformer.layers.%d.%s", l, sfx[s]);
      rh_set_param(&out[kRhTop + l * kLayerSlots + s], nm, r2[s][1] ? 2 : 1, r2[s][0], r2[s][1], 0, &off);
    }
  return off;
}

// Fills out[0 .. rh_num_params(depth)) in one pass: the decoder, then the three read-outs.
inline void rh_layout(int depth, int heads, int mlp, RhParam* out) {
  long long off = rh_layout_decoder(depth, heads, mlp, out);
  static const char* const names[kRhTail] = {"decpose.weight", "decpose.bias", "decshape.weight", "decshape.bias",
                                             "deccam.weight", "deccam.bias"};
  const long long rows[3] = {kRhPose, kRhBetas, kRhCam};
  for (int t = 0; t < kRhTail; ++t) {
    RhParam* q = &out[rh_decoder_params(depth) + t];
    if (t % 2 == 0) rh_set_param(q, names[t], 2, rows[t / 2], kRhDim, 0, &off);
    else rh_set_param(q, names[t], 1, rows[t / 2], 0, 0, &off);
  }
}

constexpr int kRhMaxParams = kRhTop + 64 * kLayerSlots + kRhTail;

// Fills p for parameter i; returns false when i is out of range.
inline bool rh_param(int depth, int heads, int mlp, int i, RhParam* p) {
  if (i < 0 || i >= rh_num_params(depth)) return false;
  static thread_local RhParam all[kRhMaxParams];
  rh_layout(depth, heads, mlp, all);
  *p = all[i];
  return true;
}

inline long long rh_param_floats(int depth, int heads, int mlp) {
  RhParam p;
  rh_param(depth, heads, mlp, rh_num_params(depth) - 1, &p);
  return p.offset + (p.numel + 63) / 64 * 64;
}

// Device pointers of one parameter set (weights or their gradients) in the flat layout.
struct RhLayerPtr {
  float* p[kLayerSlots];
};
struct RhPtrs {
  float *pos, *tok_w, *tok_b;
  RhLayerPtr layer[64];
  float *pose_w, *pose_b, *betas_w, *betas_b, *cam_w, *cam_b;
};

// The decoder's pointers from a filled layout (rh_layout_decoder's entries come first in both heads' layouts).
inline void rh_decoder_pointers(float* base, const RhParam* all, int depth, RhPtrs* out) {
  auto at = [&](int i) { return base + all[i].offset; };
  out->pos = at(kPos);
  out->tok_w = at(kTokW);
  out->tok_b = at(kTokB);
  for (int l = 0; l < depth; ++l)
    for (int s = 0; s < kLayerSlots; ++s) out->layer[l].p[s] = at(kRhTop + l * kLayerSlots + s);
}

inline void rh_pointers(float* base, int depth, int heads, int mlp, RhPtrs* out) {
  static thread_local RhParam all[kRhMaxParams];
  rh_layout(depth, heads, mlp, all);
  rh_decoder_pointers(base, all, depth, out);
  auto at = [&](int i) { return base + all[i].offset; };
  const int t = rh_decoder_params(depth);
  out->pose_w = at(t); out->pose_b = at(t + 1);
  out->betas_w = at(t + 2); out->betas_b = at(t + 3);
  out->cam_w = at(t + 4); out->cam_b = at(t + 5);
}

// ------------------------------------------------------------------------------------------------ small device functions
__device__ __forceinline__ float block_sum_256(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) t += red[w];
  return t;
}

// LayerNorm over kRhDim (eps 1e-5), one 256-thread block per row; keeps mean and 1/std for the backward.
__global__ void __launch_bounds__(256) rh_ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                        const float* __restrict__ b, float* __restrict__ y,
                                                        float* __restrict__ mean, float* __restrict__ rstd) {
  __shared__ float red[8];
  const int r = blockIdx.x, t = threadIdx.x;
  const float4 v = reinterpret_cast<const float4*>(x + static_cast<size_t>(r) * kRhDim)[t];
  const float mu = block_sum_256(v.x + v.y + v.z + v.w, red) * (1.f / kRhDim);
  const float d0 = v.x - mu, d1 = v.y - mu, d2 = v.z - mu, d3 = v.w - mu;
  const float var = block_sum_256(d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3, red) * (1.f / kRhDim);
  const float rs = rsqrtf(var + kRhLnEps);
  const float4 gg = reinterpret_cast<const float4*>(g)[t], bb = reinterpret_cast<const float4*>(b)[t];
  reinterpret_cast<float4*>(y + static_cast<size_t>(r) * kRhDim)[t] =
      make_float4(d0 * rs * gg.x + bb.x, d1 * rs * gg.y + bb.y, d2 * rs * gg.z + bb.z, d3 * rs * gg.w + bb.w);
  if (t == 0) {
    mean[r] = mu;
    rstd[r] = rs;
  }
}

// LayerNorm backward to the input, added into dx: dx += rstd (g dy - mean(g dy) - xhat mean(g dy xhat)).
__global__ void __launch_bounds__(256) rh_ln_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                        const float* __restrict__ mean, const float* __restrict__ rstd,
                                                        const float* __restrict__ dy, float* __restrict__ dx) {
  __shared__ float red[8];
  const int r = blockIdx.x, t = threadIdx.x;
  const size_t o = static_cast<size_t>(r) * kRhDim;
  const float4 v = reinterpret_cast<const float4*>(x + o)[t];
  const float4 d = reinterpret_cast<const float4*>(dy + o)[t];
  const float4 gg = reinterpret_cast<const float4*>(g)[t];
  const float mu = mean[r], rs = rstd[r];
  const float h[4] = {(v.x - mu) * rs, (v.y - mu) * rs, (v.z - mu) * rs, (v.w - mu) * rs};
  const float gd[4] = {d.x * gg.x, d.y * gg.y, d.z * gg.z, d.w * gg.w};
  const float m1 = block_sum_256(gd[0] + gd[1] + gd[2] + gd[3], red) * (1.f / kRhDim);
  const float m2 = block_sum_256(gd[0] * h[0] + gd[1] * h[1] + gd[2] * h[2] + gd[3] * h[3], red) * (1.f / kRhDim);
  float4 a = reinterpret_cast<float4*>(dx + o)[t];
  a.x += rs * (gd[0] - m1 - h[0] * m2);
  a.y += rs * (gd[1] - m1 - h[1] * m2);
  a.z += rs * (gd[2] - m1 - h[2] * m2);
  a.w += rs * (gd[3] - m1 - h[3] * m2);
  reinterpret_cast<float4*>(dx + o)[t] = a;
}

// Column sums over the batch in row order (bias, LayerNorm and embedding gradients): out[n] = sum_b dy[b,n] and, with
// x / mean / rstd, out_g[n] = sum_b dy[b,n] xhat[b,n].  out2 (optional) receives a copy of out.
__global__ void rh_colsum_kernel(const float* __restrict__ dy, int ld, int B, int N, float* __restrict__ out,
                                 float* __restrict__ out2, const float* __restrict__ x, const float* __restrict__ mean,
                                 const float* __restrict__ rstd, float* __restrict__ out_g) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float s = 0.f, sg = 0.f;
  for (int b = 0; b < B; ++b) {
    const float d = dy[static_cast<size_t>(b) * ld + n];
    s += d;
    if (out_g) sg += d * (x[static_cast<size_t>(b) * ld + n] - mean[b]) * rstd[b];
  }
  out[n] = s;
  if (out2) out2[n] = s;
  if (out_g) out_g[n] = sg;
}

// x0[b] = to_token_embedding.bias + pos_embedding (the token embedding of a zero input, pose_transformer.py:350,354)
__global__ void rh_token0_kernel(const float* __restrict__ tok_b, const float* __restrict__ pos, float* __restrict__ x,
                                 int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B * kRhDim) x[i] = tok_b[i % kRhDim] + pos[i % kRhDim];
}

// d(read-out) (B, kRhReadLd) = [d pose6d (rot6d backward + direct) | d betas | d cam], one thread per (image, joint)
__global__ void rh_readout_bwd_kernel(const float* __restrict__ pose6d, const float* __restrict__ g_rot,
                                      const float* __restrict__ g_pose6d, const float* __restrict__ g_betas,
                                      const float* __restrict__ g_cam, float* __restrict__ dread, int B) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= B * 24) return;
  const int b = t / 24, j = t % 24;
  float gx[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (g_rot) rot6d_to_rotmat_backward_one(pose6d + static_cast<size_t>(t) * 6, g_rot + static_cast<size_t>(t) * 9, gx);
  float* d = dread + static_cast<size_t>(b) * kRhReadLd;
#pragma unroll
  for (int e = 0; e < 6; ++e) d[j * 6 + e] = gx[e] + (g_pose6d ? g_pose6d[static_cast<size_t>(t) * 6 + e] : 0.f);
  if (j == 0) {
    for (int l = 0; l < kRhBetas; ++l) d[kRhPose + l] = g_betas ? g_betas[b * kRhBetas + l] : 0.f;
    for (int e = 0; e < kRhCam; ++e) d[kRhPose + kRhBetas + e] = g_cam ? g_cam[b * kRhCam + e] : 0.f;
    for (int e = kRhPose + kRhBetas + kRhCam; e < kRhReadLd; ++e) d[e] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------------ tiled fp32 GEMM
// C[z] (M x N) = epilogue(alpha * sum_k A(m,k) B(k,n)) for z < batch, with A(m,k) = A[z*sAz + m*sAm + k*sAk] and
// B(k,n) = Bm[z*sBz + k*sBk + n*sBn].  The three orientations of a linear layer y = x W^T:
//   x W^T   (forward, dq):      A k-contiguous, B(k,n) = W[n,k]  k-contiguous
//   dY W    (input gradient):   A k-contiguous, B(k,n) = W[k,n]  n-contiguous
//   dY^T X  (weight gradient):  A(m,k) = dY[k,m] m-contiguous, B(k,n) = X[k,n] n-contiguous
// Epilogue, in order: + bias[n];  * gelu'(dgelu[m,n]);  + C (accumulate);  store;  gelu_out = gelu(stored value).
struct HlGemm {
  const float* A;
  long long sAm, sAk, sAz;
  const float* Bm;
  long long sBk, sBn, sBz;
  float* C;
  long long ldc, sCz;
  int M, N, K, batch;
  float alpha;
  const float* bias;
  const float* dgelu;
  float* gelu_out;
  int accumulate;
  float* partial;   // split-K partial sums [splits][batch][M][N]
  int splits;
};

constexpr int kGBM = 64, kGBN = 64, kGBK = 16;

__device__ __forceinline__ void hl_epilogue(const HlGemm& p, int z, int m, int n, float acc) {
  const size_t o = static_cast<size_t>(z) * p.sCz + static_cast<size_t>(m) * p.ldc + n;
  float v = p.alpha * acc;
  if (p.bias) v += p.bias[n];
  if (p.dgelu) v *= gelu_exact_grad(p.dgelu[o]);
  if (p.accumulate) v += p.C[o];
  p.C[o] = v;
  if (p.gelu_out) p.gelu_out[o] = gelu_exact(v);
}

template <bool kAKContig, bool kBKContig>
__global__ void __launch_bounds__(256) hl_gemm_kernel(const HlGemm p) {
  __shared__ __align__(16) float As[kGBK][kGBM + 4];
  __shared__ __align__(16) float Bs[kGBK][kGBN + 4];
  const int t = threadIdx.x, tx = t % 16, ty = t / 16;
  const int n0 = blockIdx.x * kGBN, m0 = blockIdx.y * kGBM;
  const int z = blockIdx.z % p.batch, split = blockIdx.z / p.batch;
  const int kper = (p.K + p.splits - 1) / p.splits;
  const int kbeg = split * kper, kend = min(p.K, kbeg + kper);
  const float* A = p.A + static_cast<size_t>(z) * p.sAz;
  const float* Bm = p.Bm + static_cast<size_t>(z) * p.sBz;
  float acc[4][4] = {};
  for (int k0 = kbeg; k0 < kend; k0 += kGBK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = t + 256 * i;
      const int kk = kAKContig ? e % kGBK : e / kGBM, mm = kAKContig ? e / kGBK : e % kGBM;
      const int m = m0 + mm, k = k0 + kk;
      As[kk][mm] = (m < p.M && k < kend) ? A[static_cast<size_t>(m) * p.sAm + static_cast<size_t>(k) * p.sAk] : 0.f;
      const int kb = kBKContig ? e % kGBK : e / kGBN, nn = kBKContig ? e / kGBK : e % kGBN;
      const int n = n0 + nn, k2 = k0 + kb;
      Bs[kb][nn] = (n < p.N && k2 < kend) ? Bm[static_cast<size_t>(k2) * p.sBk + static_cast<size_t>(n) * p.sBn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kGBK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= p.N) continue;
      if (p.splits > 1)
        p.partial[((static_cast<size_t>(split) * p.batch + z) * p.M + m) * p.N + n] = acc[i][j];
      else
        hl_epilogue(p, z, m, n, acc[i][j]);
    }
  }
}

// Sums the split-K partials in split order, then the epilogue.
__global__ void hl_gemm_reduce_kernel(const HlGemm p) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long per = static_cast<long long>(p.M) * p.N, total = per * p.batch;
  if (i >= total) return;
  float s = 0.f;
  for (int k = 0; k < p.splits; ++k) s += p.partial[k * total + i];
  const int z = static_cast<int>(i / per), m = static_cast<int>((i % per) / p.N), n = static_cast<int>(i % p.N);
  hl_epilogue(p, z, m, n, s);
}

// Split-K partial buffer: splits * tiles <= kSplitTarget, so the partials never exceed this many floats.
constexpr int kSplitTarget = 2 * 132;
constexpr long long kSplitFloats = static_cast<long long>(kSplitTarget) * kGBM * kGBN;

enum HlOrient { kXWt, kDyW, kDytX };

// Split-K count of one GEMM: 1 without a split buffer or when the grid already has kSplitTarget / 2 tiles, else as
// many splits as fill kSplitTarget CTAs, keeping at least 4 k-blocks per split.
inline int hl_split_count(const HlGemm& p) {
  const int tn = (p.N + kGBN - 1) / kGBN, tm = (p.M + kGBM - 1) / kGBM;
  const int tiles = tn * tm * p.batch;
  int splits = 1;
  if (p.partial && tiles < kSplitTarget / 2) {
    splits = kSplitTarget / tiles;
    splits = splits < p.K / (4 * kGBK) ? splits : p.K / (4 * kGBK);   // at least 4 k-blocks per split
    if (splits < 1) splits = 1;
  }
  return splits;
}

inline void hl_gemm(HlGemm p, HlOrient o, cudaStream_t st) {
  const int tn = (p.N + kGBN - 1) / kGBN, tm = (p.M + kGBM - 1) / kGBM;
  const int splits = hl_split_count(p);
  p.splits = splits;
  dim3 grid(tn, tm, p.batch * splits);
  if (o == kXWt) hl_gemm_kernel<true, true><<<grid, 256, 0, st>>>(p);
  else if (o == kDyW) hl_gemm_kernel<true, false><<<grid, 256, 0, st>>>(p);
  else hl_gemm_kernel<false, false><<<grid, 256, 0, st>>>(p);
  if (splits > 1) {
    const long long total = static_cast<long long>(p.M) * p.N * p.batch;
    hl_gemm_reduce_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(p);
  }
}

inline HlGemm hl_make(int M, int N, int K, float* partial) {
  HlGemm p{};
  p.M = M; p.N = N; p.K = K; p.batch = 1; p.alpha = 1.f; p.partial = partial; p.splits = 1;
  return p;
}

// y (B x N, ld ldy) [+]= x (B x K, ld ldx) W^T (W: N x K) + bias
inline void hl_linear(const float* x, int ldx, const float* W, const float* bias, float* y, int ldy, int B, int N,
                      int K, bool accumulate, float* gelu_out, float* partial, cudaStream_t st) {
  HlGemm p = hl_make(B, N, K, partial);
  p.A = x; p.sAm = ldx; p.sAk = 1;
  p.Bm = W; p.sBk = 1; p.sBn = K;
  p.C = y; p.ldc = ldy;
  p.bias = bias; p.accumulate = accumulate; p.gelu_out = gelu_out;
  hl_gemm(p, kXWt, st);
}

// dx (B x K, ld ldx) [+]= dy (B x N, ld ldy) W (W: N x K); dgelu: multiply by gelu'(dgelu) (ld ldx)
inline void hl_linear_dx(const float* dy, int ldy, const float* W, float* dx, int ldx, int B, int N, int K,
                         bool accumulate, const float* dgelu, float* partial, cudaStream_t st) {
  HlGemm p = hl_make(B, K, N, partial);
  p.A = dy; p.sAm = ldy; p.sAk = 1;
  p.Bm = W; p.sBk = K; p.sBn = 1;
  p.C = dx; p.ldc = ldx;
  p.accumulate = accumulate; p.dgelu = dgelu;
  hl_gemm(p, kDyW, st);
}

// dW (N x K) = alpha dy^T (B x N, ld ldy) x (B x K, ld ldx)
inline void hl_linear_dw(const float* dy, int ldy, const float* x, int ldx, float* dW, int B, int N, int K, float alpha,
                         cudaStream_t st) {
  HlGemm p = hl_make(N, K, B, nullptr);
  p.A = dy; p.sAm = 1; p.sAk = ldy;
  p.Bm = x; p.sBk = ldx; p.sBn = 1;
  p.C = dW; p.ldc = K;
  p.alpha = alpha;
  hl_gemm(p, kDytX, st);
}

// ------------------------------------------------------------------------------------------------ factorised attention
// One CTA per (chunk of kRhChunk positions, image); warp h < H handles head h in the per-position phase.
//   forward  (vec = kq, B x H x C):   s = scale X^T kq -> s_out;  p = exp(s - m_loc);  part = sum_j p_j X[:,j],
//            stat = (m_loc, sum_j p_j)
//   backward (vec = d~):              dP = X^T d~;  P = exp(s - lse);  dS = P (dP - delta), delta = dO . o;
//            part = sum_j dS_j X[:,j]
template <bool kBwd>
__global__ void __launch_bounds__(256) rh_attn_chunk_kernel(const float* __restrict__ X, const float* __restrict__ vec,
                                                            int H, float scale, float* __restrict__ s_io,
                                                            const float* __restrict__ lse, const float* __restrict__ dO,
                                                            const float* __restrict__ o, float* __restrict__ stat,
                                                            float* __restrict__ part) {
  extern __shared__ __align__(16) float xs[];              // [kRhCtx][kRhPitch]
  __shared__ float w[kRhMaxHeads][kRhChunk];
  const int chunk = blockIdx.x, b = blockIdx.y, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int n0 = chunk * kRhChunk, I = H * kRhDimHead;
  const float* Xb = X + static_cast<size_t>(b) * kRhCtx * kRhTokens + n0;
  for (int e = t; e < kRhCtx * (kRhChunk / 4); e += 256) {
    const int c = e / (kRhChunk / 4), q = e % (kRhChunk / 4);
    *reinterpret_cast<float4*>(&xs[c * kRhPitch + q * 4]) =
        *reinterpret_cast<const float4*>(Xb + static_cast<size_t>(c) * kRhTokens + q * 4);
  }
  __syncthreads();
  if (warp < H) {
    const int h = warp;
    const float* v = vec + (static_cast<size_t>(b) * H + h) * kRhCtx;
    float acc[kRhChunk];
#pragma unroll
    for (int j = 0; j < kRhChunk; ++j) acc[j] = 0.f;
    for (int c = lane; c < kRhCtx; c += 32) {
      const float vc = v[c];
#pragma unroll
      for (int q = 0; q < kRhChunk / 4; ++q) {
        const float4 x4 = *reinterpret_cast<const float4*>(&xs[c * kRhPitch + q * 4]);
        acc[q * 4 + 0] = fmaf(vc, x4.x, acc[q * 4 + 0]);
        acc[q * 4 + 1] = fmaf(vc, x4.y, acc[q * 4 + 1]);
        acc[q * 4 + 2] = fmaf(vc, x4.z, acc[q * 4 + 2]);
        acc[q * 4 + 3] = fmaf(vc, x4.w, acc[q * 4 + 3]);
      }
    }
    float mine = 0.f;    // lane j < kRhChunk keeps position j's dot product
#pragma unroll
    for (int j = 0; j < kRhChunk; ++j) {
      float a = acc[j];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
      if (lane == j) mine = a;
    }
    float* srow = s_io + (static_cast<size_t>(b) * H + h) * kRhTokens + n0;
    if (!kBwd) {
      const float s = scale * mine;
      float m = lane < kRhChunk ? s : -INFINITY;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
      const float pj = lane < kRhChunk ? expf(s - m) : 0.f;
      float l = pj;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) l += __shfl_xor_sync(0xffffffffu, l, off);
      if (lane < kRhChunk) {
        srow[lane] = s;
        w[h][lane] = pj;
      }
      if (lane == 0) {
        float* st = stat + ((static_cast<size_t>(b) * kRhChunks + chunk) * H + h) * 2;
        st[0] = m;
        st[1] = l;
      }
    } else {
      const float* dob = dO + static_cast<size_t>(b) * I + h * kRhDimHead;
      const float* ob = o + static_cast<size_t>(b) * I + h * kRhDimHead;
      float delta = dob[lane] * ob[lane] + dob[lane + 32] * ob[lane + 32];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) delta += __shfl_xor_sync(0xffffffffu, delta, off);
      if (lane < kRhChunk) {
        const float P = expf(srow[lane] - lse[static_cast<size_t>(b) * H + h]);
        w[h][lane] = P * (mine - delta);
      }
    }
  }
  __syncthreads();
  for (int c = t; c < kRhCtx; c += 256) {
    float x[kRhChunk];
#pragma unroll
    for (int q = 0; q < kRhChunk / 4; ++q) {
      const float4 x4 = *reinterpret_cast<const float4*>(&xs[c * kRhPitch + q * 4]);
      x[q * 4 + 0] = x4.x; x[q * 4 + 1] = x4.y; x[q * 4 + 2] = x4.z; x[q * 4 + 3] = x4.w;
    }
    for (int h = 0; h < H; ++h) {
      float a = 0.f;
#pragma unroll
      for (int j = 0; j < kRhChunk; ++j) a = fmaf(w[h][j], x[j], a);
      part[((static_cast<size_t>(b) * kRhChunks + chunk) * H + h) * kRhCtx + c] = a;
    }
  }
}

// Merges the chunks of one (image, head) in chunk order.  forward: c = sum_k e^(m_k - m) part_k / L and
// lse = m + log L;  backward (stat == NULL): u = sum_k part_k.
__global__ void __launch_bounds__(256) rh_attn_combine_kernel(const float* __restrict__ part,
                                                              const float* __restrict__ stat, int H,
                                                              float* __restrict__ out, float* __restrict__ lse) {
  const int bh = blockIdx.x, b = bh / H, h = bh % H;
  float wk[kRhChunks];
  float m = -INFINITY, L = 0.f;
  if (stat) {
#pragma unroll
    for (int k = 0; k < kRhChunks; ++k) m = fmaxf(m, stat[((static_cast<size_t>(b) * kRhChunks + k) * H + h) * 2]);
#pragma unroll
    for (int k = 0; k < kRhChunks; ++k) {
      const float* st = stat + ((static_cast<size_t>(b) * kRhChunks + k) * H + h) * 2;
      wk[k] = expf(st[0] - m);
      L += wk[k] * st[1];
    }
#pragma unroll
    for (int k = 0; k < kRhChunks; ++k) wk[k] /= L;
    if (threadIdx.x == 0) lse[bh] = m + logf(L);
  } else {
#pragma unroll
    for (int k = 0; k < kRhChunks; ++k) wk[k] = 1.f;
  }
  for (int c = threadIdx.x; c < kRhCtx; c += 256) {
    float a = 0.f;
#pragma unroll
    for (int k = 0; k < kRhChunks; ++k)
      a = fmaf(wk[k], part[((static_cast<size_t>(b) * kRhChunks + k) * H + h) * kRhCtx + c], a);
    out[static_cast<size_t>(bh) * kRhCtx + c] = a;
  }
}

constexpr size_t kRhAttSmem = static_cast<size_t>(kRhCtx) * kRhPitch * sizeof(float);

inline int rh_configure() {
  static bool done = false;
  if (!done) {
    THMR_CUDA(cudaFuncSetAttribute(rh_attn_chunk_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRhAttSmem));
    THMR_CUDA(cudaFuncSetAttribute(rh_attn_chunk_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRhAttSmem));
    done = true;
  }
  return THMR_OK;
}

// ------------------------------------------------------------------------------------------------ workspace
// Activations the forward keeps for the backward, then scratch.  All in floats, each array 64-float aligned.
struct RhLayerAct {
  float *x0, *x1, *x2;              // sub-layer inputs (B x E)
  float *y0, *y1, *y2;              // LayerNorm outputs
  float *mean, *rstd;               // [3][B]
  float *v, *q, *o;                 // B x I: self-attention value, cross-attention query and output
  float *s, *lse;                   // B x H x 192 scaled scores, B x H log-sum-exp
  float *c;                         // B x H x C context summaries
  float *u, *h;                     // B x mlp: pre-GELU and GELU
};
struct RhWs {
  RhLayerAct act[64];
  float *tok, *read, *pose6d;       // B x E output token, B x 160 read-out, B x 144 6D pose
  // scratch
  float *kq, *part, *stat, *split;
  float *dx, *dy, *dI, *dI2, *dU, *dtil, *uatt, *dread;
  size_t floats;
};

inline void rh_carve(float* base, int B, int depth, int H, int mlp, RhWs* w) {
  size_t off = 0;
  auto take = [&](size_t n) {
    float* p = base ? base + off : nullptr;
    off += (n + 63) / 64 * 64;
    return p;
  };
  const size_t E = kRhDim, I = static_cast<size_t>(H) * kRhDimHead;
  for (int l = 0; l < depth; ++l) {
    RhLayerAct& a = w->act[l];
    a.x0 = take(B * E); a.x1 = take(B * E); a.x2 = take(B * E);
    a.y0 = take(B * E); a.y1 = take(B * E); a.y2 = take(B * E);
    a.mean = take(3 * B); a.rstd = take(3 * B);
    a.v = take(B * I); a.q = take(B * I); a.o = take(B * I);
    a.s = take(static_cast<size_t>(B) * H * kRhTokens); a.lse = take(static_cast<size_t>(B) * H);
    a.c = take(static_cast<size_t>(B) * H * kRhCtx);
    a.u = take(static_cast<size_t>(B) * mlp); a.h = take(static_cast<size_t>(B) * mlp);
  }
  w->tok = take(B * E);
  w->read = take(static_cast<size_t>(B) * kRhReadLd);
  w->pose6d = take(static_cast<size_t>(B) * kRhPose);
  w->kq = take(static_cast<size_t>(B) * H * kRhCtx);
  w->part = take(static_cast<size_t>(B) * kRhChunks * H * kRhCtx);
  w->stat = take(static_cast<size_t>(B) * kRhChunks * H * 2);
  w->split = take(kSplitFloats);
  w->dx = take(B * E); w->dy = take(B * E);
  w->dI = take(B * I); w->dI2 = take(B * I);
  w->dU = take(static_cast<size_t>(B) * mlp);
  w->dtil = take(static_cast<size_t>(B) * H * kRhCtx);
  w->uatt = take(static_cast<size_t>(B) * H * kRhCtx);
  w->dread = take(static_cast<size_t>(B) * kRhReadLd);
  w->floats = off;
}

inline size_t rh_workspace_bytes(int B, int depth, int H, int mlp) {
  RhWs w;
  rh_carve(nullptr, B, depth, H, mlp, &w);
  return w.floats * sizeof(float);
}

// ------------------------------------------------------------------------------------------------ forward
// The decoder's layer loop (both SMPL heads): P's decoder pointers, the channel-first features -> w.tok (B x E), with
// every layer's activations kept in w.act.
inline int rh_decoder_forward(const RhPtrs& P, const float* feats, int B, int depth, int H, int mlp, RhWs& w,
                              cudaStream_t st) {
  const int E = kRhDim, I = H * kRhDimHead, C = kRhCtx;
  const float scale = 1.f / sqrtf(static_cast<float>(kRhDimHead));
  THMR_TRY(rh_configure());
  rh_token0_kernel<<<(B * E + 255) / 256, 256, 0, st>>>(P.tok_b, P.pos, w.act[0].x0, B);
  for (int l = 0; l < depth; ++l) {
    RhLayerAct& a = w.act[l];
    float* const* L = P.layer[l].p;
    float* xout = l + 1 < depth ? w.act[l + 1].x0 : w.tok;
    // self-attention over one key: x1 = x0 + to_out(W_v LN0(x0))
    rh_ln_fwd_kernel<<<B, 256, 0, st>>>(a.x0, L[kL0g], L[kL0b], a.y0, a.mean, a.rstd);
    hl_linear(a.y0, E, L[kQkv] + static_cast<size_t>(2) * I * E, nullptr, a.v, I, B, I, E, false, nullptr, w.split, st);
    THMR_CUDA(cudaMemcpyAsync(a.x1, a.x0, sizeof(float) * B * E, cudaMemcpyDeviceToDevice, st));
    hl_linear(a.v, I, L[kSaOw], L[kSaOb], a.x1, E, B, E, I, true, nullptr, w.split, st);
    // cross-attention, factorised: kq = W_k,h^T q per head; one pass over X; o = W_v,h c per head
    rh_ln_fwd_kernel<<<B, 256, 0, st>>>(a.x1, L[kL1g], L[kL1b], a.y1, a.mean + B, a.rstd + B);
    hl_linear(a.y1, E, L[kQ], nullptr, a.q, I, B, I, E, false, nullptr, w.split, st);
    {
      HlGemm p = hl_make(B, C, kRhDimHead, w.split);     // kq[b,h,:] = q[b,h,:] W_k[h]   (dY W orientation)
      p.batch = H;
      p.A = a.q; p.sAm = I; p.sAk = 1; p.sAz = kRhDimHead;
      p.Bm = L[kKv]; p.sBk = C; p.sBn = 1; p.sBz = static_cast<long long>(kRhDimHead) * C;
      p.C = w.kq; p.ldc = static_cast<long long>(H) * C; p.sCz = C;
      hl_gemm(p, kDyW, st);
    }
    rh_attn_chunk_kernel<false><<<dim3(kRhChunks, B), 256, kRhAttSmem, st>>>(feats, w.kq, H, scale, a.s, nullptr,
                                                                            nullptr, nullptr, w.stat, w.part);
    rh_attn_combine_kernel<<<B * H, 256, 0, st>>>(w.part, w.stat, H, a.c, a.lse);
    {
      HlGemm p = hl_make(B, kRhDimHead, C, w.split);     // o[b,h,:] = W_v[h] c[b,h,:]   (x W^T orientation)
      p.batch = H;
      p.A = a.c; p.sAm = static_cast<long long>(H) * C; p.sAk = 1; p.sAz = C;
      p.Bm = L[kKv] + static_cast<size_t>(I) * C; p.sBk = 1; p.sBn = C; p.sBz = static_cast<long long>(kRhDimHead) * C;
      p.C = a.o; p.ldc = I; p.sCz = kRhDimHead;
      hl_gemm(p, kXWt, st);
    }
    THMR_CUDA(cudaMemcpyAsync(a.x2, a.x1, sizeof(float) * B * E, cudaMemcpyDeviceToDevice, st));
    hl_linear(a.o, I, L[kCaOw], L[kCaOb], a.x2, E, B, E, I, true, nullptr, w.split, st);
    // feed-forward: xout = x2 + W2 gelu(W1 LN2(x2) + b1) + b2
    rh_ln_fwd_kernel<<<B, 256, 0, st>>>(a.x2, L[kL2g], L[kL2b], a.y2, a.mean + 2 * B, a.rstd + 2 * B);
    hl_linear(a.y2, E, L[kF1w], L[kF1b], a.u, mlp, B, mlp, E, false, a.h, w.split, st);
    THMR_CUDA(cudaMemcpyAsync(xout, a.x2, sizeof(float) * B * E, cudaMemcpyDeviceToDevice, st));
    hl_linear(a.h, mlp, L[kF2w], L[kF2b], xout, E, B, E, mlp, true, nullptr, w.split, st);
  }
  return THMR_OK;
}

inline int rh_forward(const thmr_reg_head_desc& d, RhWs& w, cudaStream_t st) {
  const int B = d.B, E = kRhDim;
  RhPtrs P;
  rh_pointers(const_cast<float*>(d.params), d.depth, d.heads, d.mlp_dim, &P);
  THMR_TRY(rh_decoder_forward(P, d.feats, B, d.depth, d.heads, d.mlp_dim, w, st));
  // read-outs (smpl_head.py:82-84) into [pose | betas | cam], then + init_* and rot6d_to_rotmat (:89-99)
  hl_linear(w.tok, E, P.pose_w, P.pose_b, w.read, kRhReadLd, B, kRhPose, E, false, nullptr, w.split, st);
  hl_linear(w.tok, E, P.betas_w, P.betas_b, w.read + kRhPose, kRhReadLd, B, kRhBetas, E, false, nullptr, w.split, st);
  hl_linear(w.tok, E, P.cam_w, P.cam_b, w.read + kRhPose + kRhBetas, kRhReadLd, B, kRhCam, E, false, nullptr, w.split,
            st);
  head_assemble_kernel<<<(B * 24 + 127) / 128, 128, 0, st>>>(w.read, kRhReadLd, nullptr, 0, 0, 0, d.init_body_pose,
                                                             d.init_betas, d.init_cam, d.rotmats, d.betas, d.cam,
                                                             w.pose6d, B, kRhBetas);
  THMR_CUDA(cudaGetLastError());
  if (d.pose6d)
    THMR_CUDA(cudaMemcpyAsync(d.pose6d, w.pose6d, sizeof(float) * B * kRhPose, cudaMemcpyDeviceToDevice, st));
  return THMR_OK;
}

// ------------------------------------------------------------------------------------------------ backward
// The decoder's layer loop backward (both SMPL heads): from d tok in w.dx to the gradient of every decoder parameter
// (G's decoder pointers), reading the activations rh_decoder_forward kept.
inline int rh_decoder_backward(const RhPtrs& P, const RhPtrs& G, const float* feats, int B, int depth, int H, int mlp,
                               RhWs& w, cudaStream_t st) {
  const int E = kRhDim, I = H * kRhDimHead, C = kRhCtx;
  const float scale = 1.f / sqrtf(static_cast<float>(kRhDimHead));
  THMR_TRY(rh_configure());
  const unsigned colE = (E + 127) / 128;
  for (int l = depth - 1; l >= 0; --l) {
    RhLayerAct& a = w.act[l];
    float* const* L = P.layer[l].p;
    float* const* Lg = G.layer[l].p;
    // feed-forward
    rh_colsum_kernel<<<colE, 128, 0, st>>>(w.dx, E, B, E, Lg[kF2b], nullptr, nullptr, nullptr, nullptr, nullptr);
    hl_linear_dw(w.dx, E, a.h, mlp, Lg[kF2w], B, E, mlp, 1.f, st);
    hl_linear_dx(w.dx, E, L[kF2w], w.dU, mlp, B, E, mlp, false, a.u, w.split, st);
    rh_colsum_kernel<<<(mlp + 127) / 128, 128, 0, st>>>(w.dU, mlp, B, mlp, Lg[kF1b], nullptr, nullptr, nullptr,
                                                         nullptr, nullptr);
    hl_linear_dw(w.dU, mlp, a.y2, E, Lg[kF1w], B, mlp, E, 1.f, st);
    hl_linear_dx(w.dU, mlp, L[kF1w], w.dy, E, B, mlp, E, false, nullptr, w.split, st);
    rh_colsum_kernel<<<colE, 128, 0, st>>>(w.dy, E, B, E, Lg[kL2b], nullptr, a.x2, a.mean + 2 * B, a.rstd + 2 * B,
                                           Lg[kL2g]);
    rh_ln_bwd_kernel<<<B, 256, 0, st>>>(a.x2, L[kL2g], a.mean + 2 * B, a.rstd + 2 * B, w.dy, w.dx);
    // cross-attention
    rh_colsum_kernel<<<colE, 128, 0, st>>>(w.dx, E, B, E, Lg[kCaOb], nullptr, nullptr, nullptr, nullptr, nullptr);
    hl_linear_dw(w.dx, E, a.o, I, Lg[kCaOw], B, E, I, 1.f, st);
    hl_linear_dx(w.dx, E, L[kCaOw], w.dI, I, B, E, I, false, nullptr, w.split, st);   // dO
    {
      HlGemm p = hl_make(B, C, kRhDimHead, w.split);     // d~[b,h,:] = dO[b,h,:] W_v[h]
      p.batch = H;
      p.A = w.dI; p.sAm = I; p.sAk = 1; p.sAz = kRhDimHead;
      p.Bm = L[kKv] + static_cast<size_t>(I) * C; p.sBk = C; p.sBn = 1; p.sBz = static_cast<long long>(kRhDimHead) * C;
      p.C = w.dtil; p.ldc = static_cast<long long>(H) * C; p.sCz = C;
      hl_gemm(p, kDyW, st);
    }
    {
      HlGemm p = hl_make(kRhDimHead, C, B, nullptr);     // dW_v[h] = sum_b dO[b,h,:] (x) c[b,h,:]
      p.batch = H;
      p.A = w.dI; p.sAm = 1; p.sAk = I; p.sAz = kRhDimHead;
      p.Bm = a.c; p.sBk = static_cast<long long>(H) * C; p.sBn = 1; p.sBz = C;
      p.C = Lg[kKv] + static_cast<size_t>(I) * C; p.ldc = C; p.sCz = static_cast<long long>(kRhDimHead) * C;
      hl_gemm(p, kDytX, st);
    }
    rh_attn_chunk_kernel<true><<<dim3(kRhChunks, B), 256, kRhAttSmem, st>>>(feats, w.dtil, H, scale, a.s, a.lse,
                                                                           w.dI, a.o, nullptr, w.part);
    rh_attn_combine_kernel<<<B * H, 256, 0, st>>>(w.part, nullptr, H, w.uatt, nullptr);
    {
      HlGemm p = hl_make(kRhDimHead, C, B, nullptr);     // dW_k[h] = scale sum_b q[b,h,:] (x) u[b,h,:]
      p.batch = H;
      p.alpha = scale;
      p.A = a.q; p.sAm = 1; p.sAk = I; p.sAz = kRhDimHead;
      p.Bm = w.uatt; p.sBk = static_cast<long long>(H) * C; p.sBn = 1; p.sBz = C;
      p.C = Lg[kKv]; p.ldc = C; p.sCz = static_cast<long long>(kRhDimHead) * C;
      hl_gemm(p, kDytX, st);
    }
    {
      HlGemm p = hl_make(B, kRhDimHead, C, w.split);     // dq[b,h,:] = scale W_k[h] u[b,h,:]
      p.batch = H;
      p.alpha = scale;
      p.A = w.uatt; p.sAm = static_cast<long long>(H) * C; p.sAk = 1; p.sAz = C;
      p.Bm = L[kKv]; p.sBk = 1; p.sBn = C; p.sBz = static_cast<long long>(kRhDimHead) * C;
      p.C = w.dI2; p.ldc = I; p.sCz = kRhDimHead;
      hl_gemm(p, kXWt, st);
    }
    hl_linear_dw(w.dI2, I, a.y1, E, Lg[kQ], B, I, E, 1.f, st);
    hl_linear_dx(w.dI2, I, L[kQ], w.dy, E, B, I, E, false, nullptr, w.split, st);
    rh_colsum_kernel<<<colE, 128, 0, st>>>(w.dy, E, B, E, Lg[kL1b], nullptr, a.x1, a.mean + B, a.rstd + B, Lg[kL1g]);
    rh_ln_bwd_kernel<<<B, 256, 0, st>>>(a.x1, L[kL1g], a.mean + B, a.rstd + B, w.dy, w.dx);
    // self-attention: the Q and K thirds of to_qkv see no gradient (softmax over one key)
    rh_colsum_kernel<<<colE, 128, 0, st>>>(w.dx, E, B, E, Lg[kSaOb], nullptr, nullptr, nullptr, nullptr, nullptr);
    hl_linear_dw(w.dx, E, a.v, I, Lg[kSaOw], B, E, I, 1.f, st);
    hl_linear_dx(w.dx, E, L[kSaOw], w.dI, I, B, E, I, false, nullptr, w.split, st);   // dv
    THMR_CUDA(cudaMemsetAsync(Lg[kQkv], 0, sizeof(float) * 2 * I * E, st));
    hl_linear_dw(w.dI, I, a.y0, E, Lg[kQkv] + static_cast<size_t>(2) * I * E, B, I, E, 1.f, st);
    hl_linear_dx(w.dI, I, L[kQkv] + static_cast<size_t>(2) * I * E, w.dy, E, B, I, E, false, nullptr, w.split, st);
    rh_colsum_kernel<<<colE, 128, 0, st>>>(w.dy, E, B, E, Lg[kL0b], nullptr, a.x0, a.mean, a.rstd, Lg[kL0g]);
    rh_ln_bwd_kernel<<<B, 256, 0, st>>>(a.x0, L[kL0g], a.mean, a.rstd, w.dy, w.dx);
  }
  // x0 = to_token_embedding(0) + pos_embedding: both the bias and pos_embedding receive sum_b dx0; the weight
  // multiplies a zero input
  rh_colsum_kernel<<<colE, 128, 0, st>>>(w.dx, E, B, E, G.tok_b, G.pos, nullptr, nullptr, nullptr, nullptr);
  THMR_CUDA(cudaMemsetAsync(G.tok_w, 0, sizeof(float) * E, st));
  return THMR_OK;
}

inline int rh_backward(const thmr_reg_head_desc& d, RhWs& w, cudaStream_t st) {
  const int B = d.B, H = d.heads, mlp = d.mlp_dim, E = kRhDim;
  RhPtrs P, G;
  rh_pointers(const_cast<float*>(d.params), d.depth, H, mlp, &P);
  rh_pointers(d.grads, d.depth, H, mlp, &G);
  // read-outs
  rh_readout_bwd_kernel<<<(B * 24 + 127) / 128, 128, 0, st>>>(w.pose6d, d.grad_rotmats, d.grad_pose6d, d.grad_betas,
                                                              d.grad_cam, w.dread, B);
  const int rows[3] = {kRhPose, kRhBetas, kRhCam}, col[3] = {0, kRhPose, kRhPose + kRhBetas};
  float* const rw[3] = {P.pose_w, P.betas_w, P.cam_w};
  float* const gw[3] = {G.pose_w, G.betas_w, G.cam_w};
  float* const gb[3] = {G.pose_b, G.betas_b, G.cam_b};
  for (int r = 0; r < 3; ++r) {
    hl_linear_dw(w.dread + col[r], kRhReadLd, w.tok, E, gw[r], B, rows[r], E, 1.f, st);
    rh_colsum_kernel<<<1, 256, 0, st>>>(w.dread + col[r], kRhReadLd, B, rows[r], gb[r], nullptr, nullptr, nullptr,
                                        nullptr, nullptr);
    hl_linear_dx(w.dread + col[r], kRhReadLd, rw[r], w.dx, E, B, rows[r], E, r > 0, nullptr, w.split, st);
  }
  THMR_TRY(rh_decoder_backward(P, G, d.feats, B, d.depth, H, mlp, w, st));
  THMR_CUDA(cudaGetLastError());
  return THMR_OK;
}

}  // namespace thmr
