// Training TokenHMR's token head (SMPLTokenDecoderHead, heads/token_head.py:65-128 with IEF_ITERS 1, TRANSFORMER_INPUT
// 'zero', JOINT_REP '6d'): an fp32 forward that keeps what the backward needs, and the backward to every trainable
// parameter (thmr_tok_head_train_forward / thmr_tok_head_backward).  No gradient for the features, none for the
// tokenizer, which the reference reaches through a Proxy and never trains.
//
// The decoder is the regression head's (rh_decoder_forward / rh_decoder_backward in head_train.cuh).  After its
// output token tok (B x 1024):
//   read-outs   decpose_grot (6), decpose_hands (12), decshape (10), deccam (3): linears on tok
//   classifier  mixer_trans = ReLU(LN(Linear 1024 -> 10240)) as (B, 160, 64); 4 MixerLayers (token MLP 160 -> 64 -> 160
//               and channel MLP 64 -> 256 -> 64, GELU, two LayerNorms over 64); mixer_norm_layer = ReLU(LN(Linear 64 ->
//               64)); class_pred_layer 64 -> 2048; softmax -> P (B, 160, 2048) = cls_logits_softmax
//   tokenizer   Z = P codebook (B, 160, 256); Conv1d 256 -> 512 k3, ReLU; 4 x [nearest resize to 125, 90, 55, 21;
//               Conv1d k3; ReLU]; 2 ResNet1D blocks (dilation 3, 1); Conv1d k3; Conv1d 512 -> 6 k3 -> (B, 21, 6)
// Every activation is channel-last: rows (image, position), columns channels.  A convolution is an im2col (column
// c * taps + j, the order of the Conv1d weight's (Cin, k) dims, so the weight is used as stored) feeding hl_gemm; the
// nearest resize and the ReLU on the conv's input are folded into the im2col's read.  Its backward to the input is
// dY W followed by a gather: one thread per input element sums its taps, and through the resize its source
// positions, in a fixed order.  The tokenizer's weights are constants: the backward takes no gradient for them.
// The large contractions (soft lookup, class_pred_layer, mixer_trans, convolutions) and every weight gradient go
// through hl_gemm; bias and LayerNorm gradients are column sums in a fixed row order.  No float atomics anywhere.
#pragma once
#include <algorithm>
#include <utility>

#include "elementwise.cuh"
#include "head_train.cuh"

namespace thmr {

constexpr int kTkT = 160, kTkHid = 64, kTkTokInter = 64, kTkChInter = 256, kTkBlocks = 4, kTkClasses = 2048;
constexpr int kTkMix = kTkT * kTkHid;                       // 10240: mixer_trans width
constexpr int kTkCode = 256, kTkWidth = 512, kTkJoints = 21, kTkUps = 4, kTkResBlocks = 2;
constexpr int kTkUpLen[kTkUps] = {125, 90, 55, 21};          // PoseSPDecoderV1's nn.Upsample sizes
constexpr int kTkResDil[kTkResBlocks] = {3, 1};              // Resnet1D(reverse_dilation=True), stored order
constexpr int kTkColRows = 160;                              // rows per partial of the two-stage column sums

// ------------------------------------------------------------------------------------------------ parameter layouts
// Trainable: the decoder (rh_layout_decoder), then the tail below, in SMPLTokenDecoderHead.named_parameters() order.
enum TkTail {
  kTgW, kTgB, kTsW, kTsB, kTcW, kTcB, kThW, kThB,     // decpose_grot, decshape, deccam, decpose_hands
  kTmtW, kTmtB, kTmtG, kTmtBeta,                      // mixer_trans.ff.0 (Linear), ff.1 (LayerNorm)
  kTmix,                                              // + 12 per MixerLayer, slots below
  kTmnW = kTmix + 12 * kTkBlocks, kTmnB, kTmnG, kTmnBeta, kTclsW, kTclsB, kTkTail
};
enum TkMixSlot { kM1g, kM1b, kMt1w, kMt1b, kMt2w, kMt2b, kM2g, kM2b, kMc1w, kMc1b, kMc2w, kMc2b };

inline int tk_num_params(int depth) { return rh_decoder_params(depth) + kTkTail; }
constexpr int kTkMaxParams = kRhTop + 64 * kLayerSlots + kTkTail;

inline void tk_layout(int depth, int heads, int mlp, RhParam* out) {
  long long off = rh_layout_decoder(depth, heads, mlp, out);
  RhParam* q = out + rh_decoder_params(depth);
  const long long E = kRhDim;
  auto lin = [&](const char* name, long long o, long long i) {
    char nm[96];
    snprintf(nm, sizeof(nm), "%s.weight", name);
    rh_set_param(q++, nm, 2, o, i, 0, &off);
    snprintf(nm, sizeof(nm), "%s.bias", name);
    rh_set_param(q++, nm, 1, o, 0, 0, &off);
  };
  auto ln = [&](const char* name, long long n) {   // LayerNorm: weight and bias, both (n,)
    char nm[96];
    snprintf(nm, sizeof(nm), "%s.weight", name);
    rh_set_param(q++, nm, 1, n, 0, 0, &off);
    snprintf(nm, sizeof(nm), "%s.bias", name);
    rh_set_param(q++, nm, 1, n, 0, 0, &off);
  };
  lin("decpose_grot", 6, E);
  lin("decshape", kRhBetas, E);
  lin("deccam", kRhCam, E);
  lin("decpose_hands", 12, E);
  lin("decpose.mixer_trans.ff.0", kTkMix, E);
  ln("decpose.mixer_trans.ff.1", kTkMix);
  char nm[96];
  for (int i = 0; i < kTkBlocks; ++i) {
    auto sub = [&](const char* s) { snprintf(nm, sizeof(nm), "decpose.mixer_head.%d.%s", i, s); return nm; };
    ln(sub("layernorm1"), kTkHid);
    lin(sub("MLP_token.ff.0"), kTkTokInter, kTkT);
    lin(sub("MLP_token.ff.3"), kTkT, kTkTokInter);
    ln(sub("layernorm2"), kTkHid);
    lin(sub("MLP_channel.ff.0"), kTkChInter, kTkHid);
    lin(sub("MLP_channel.ff.3"), kTkHid, kTkChInter);
  }
  lin("decpose.mixer_norm_layer.ff.0", kTkHid, kTkHid);
  ln("decpose.mixer_norm_layer.ff.1", kTkHid);
  lin("decpose.class_pred_layer", kTkClasses, kTkHid);
}
inline bool tk_param(int depth, int heads, int mlp, int i, RhParam* p) {
  if (i < 0 || i >= tk_num_params(depth)) return false;
  static thread_local RhParam all[kTkMaxParams];
  tk_layout(depth, heads, mlp, all);
  *p = all[i];
  return true;
}

inline long long tk_param_floats(int depth, int heads, int mlp) {
  RhParam p;
  tk_param(depth, heads, mlp, tk_num_params(depth) - 1, &p);
  return p.offset + (p.numel + 63) / 64 * 64;
}

struct TkPtrs {
  RhPtrs dec;
  float* t[kTkTail];
  float* mix(int i, int s) const { return t[kTmix + 12 * i + s]; }
};

inline void tk_pointers(float* base, int depth, int heads, int mlp, TkPtrs* out) {
  static thread_local RhParam all[kTkMaxParams];
  tk_layout(depth, heads, mlp, all);
  rh_decoder_pointers(base, all, depth, &out->dec);
  for (int k = 0; k < kTkTail; ++k) out->t[k] = base + all[rh_decoder_params(depth) + k].offset;
}

// Frozen: the tokenizer decoder's tensors and the codebook, under their checkpoint names (PoseSPDecoderV1's Sequential
// indices as saved: conv 0, the four resize convs 3 6 9 12, the ResNet1D 14.0, conv 14.1, the output conv 15).
enum TkTokSlot {
  kK0w, kK0b, kKup, kKres = kKup + 2 * kTkUps, kKpostW = kKres + 4 * kTkResBlocks, kKpostB, kKoutW, kKoutB, kKcb,
  kTkTokTensors
};

inline void tk_tokenizer_layout(RhParam* out) {
  long long off = 0;
  const char* t = "tokenizer.decoder.decoder";
  const long long W = kTkWidth;
  char nm[128];
  auto conv = [&](int slot, const char* name, long long o, long long i, long long k) {
    snprintf(nm, sizeof(nm), "%s.%s.weight", t, name);
    rh_set_param(&out[slot], nm, 3, o, i, k, &off);
    snprintf(nm, sizeof(nm), "%s.%s.bias", t, name);
    rh_set_param(&out[slot + 1], nm, 1, o, 0, 0, &off);
  };
  conv(kK0w, "0", W, kTkCode, 3);
  char sub[64];
  for (int u = 0; u < kTkUps; ++u) {
    snprintf(sub, sizeof(sub), "%d", 3 + 3 * u);
    conv(kKup + 2 * u, sub, W, W, 3);
  }
  const int r = 2 + 3 * kTkUps;   // 14
  for (int d = 0; d < kTkResBlocks; ++d) {
    snprintf(sub, sizeof(sub), "%d.0.model.%d.conv1", r, d);
    conv(kKres + 4 * d, sub, W, W, 3);
    snprintf(sub, sizeof(sub), "%d.0.model.%d.conv2", r, d);
    conv(kKres + 4 * d + 2, sub, W, W, 1);
  }
  snprintf(sub, sizeof(sub), "%d.1", r);
  conv(kKpostW, sub, W, W, 3);
  snprintf(sub, sizeof(sub), "%d", r + 1);
  conv(kKoutW, sub, 6, W, 3);
  rh_set_param(&out[kKcb], "tokenizer.quantizer.codebook", 2, kTkClasses, kTkCode, 0, &off);
}

inline bool tk_tokenizer_param(int i, RhParam* p) {
  if (i < 0 || i >= kTkTokTensors) return false;
  static thread_local RhParam all[kTkTokTensors];
  tk_tokenizer_layout(all);
  *p = all[i];
  return true;
}

inline long long tk_tokenizer_floats() {
  RhParam p;
  tk_tokenizer_param(kTkTokTensors - 1, &p);
  return p.offset + (p.numel + 63) / 64 * 64;
}

struct TkTok {
  const float* t[kTkTokTensors];
};

inline void tk_tokenizer_pointers(const float* base, TkTok* out) {
  RhParam all[kTkTokTensors];
  tk_tokenizer_layout(all);
  for (int k = 0; k < kTkTokTensors; ++k) out->t[k] = base + all[k].offset;
}

// ------------------------------------------------------------------------------------------------ sequence maps
// The positions a conv reads: src[p] for p < lout is the input position of (resized) position p, lo[s] .. lo[s+1] the
// positions that read input s (the resize is monotone).  Identity when lin == lout.  nn.Upsample(size), mode
// 'nearest': src = floor(p * (lin / lout)), the scale rounded to fp32 and the product taken in fp32, as ATen does.
// Passed to the kernels by value, built on the host once per call.
struct TkSeqMap {
  int lin, lout;
  short src[kTkT];
  short lo[kTkT + 1];
};

inline TkSeqMap tk_seq_map(int lin, int lout) {
  TkSeqMap m{};
  m.lin = lin;
  m.lout = lout;
  const float scale = static_cast<float>(static_cast<double>(lin) / lout);
  for (int p = 0; p < lout; ++p) {
    const int s = static_cast<int>(floorf(static_cast<float>(p) * scale));
    m.src[p] = static_cast<short>(s < lin - 1 ? s : lin - 1);
  }
  int p = 0;
  for (int s = 0; s <= lin; ++s) {
    while (p < lout && m.src[p] < s) ++p;
    m.lo[s] = static_cast<short>(p);
  }
  return m;
}

// ------------------------------------------------------------------------------------------------ kernels
// col[(b, l), c * taps + j] = act(X[b, src[l + (j - taps/2) dil], c]), zero outside [0, lout); act = ReLU or identity
__global__ void tk_im2col_kernel(const float* __restrict__ X, int Cin, const TkSeqMap m, int taps, int dil, int relu,
                                 float* __restrict__ col, int B) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  const long long K = static_cast<long long>(Cin) * taps;
  if (i >= static_cast<long long>(B) * m.lout * K) return;
  const long long row = i / K;
  const int e = static_cast<int>(i % K), c = e / taps, j = e % taps;
  const int b = static_cast<int>(row / m.lout), l = static_cast<int>(row % m.lout);
  const int p = l + (j - taps / 2) * dil;
  float v = 0.f;
  if (p >= 0 && p < m.lout) {
    v = X[(static_cast<size_t>(b) * m.lin + m.src[p]) * Cin + c];
    if (relu) v = fmaxf(v, 0.f);
  }
  col[i] = v;
}

// The conv's backward to its input, as a gather: dX[b, s, c] = sum over the positions p that read s (in order) and the
// taps j (in order) of dcol[(b, p - (j - taps/2) dil), c * taps + j];  then * [mask > 0], + resid, * [mask_out > 0]
// (each optional).
__global__ void tk_col2im_kernel(const float* __restrict__ dcol, int Cin, const TkSeqMap m, int taps, int dil,
                                 const float* __restrict__ mask, const float* __restrict__ resid,
                                 const float* __restrict__ mask_out, float* __restrict__ dX, int B) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long long>(B) * m.lin * Cin) return;
  const int c = static_cast<int>(i % Cin);
  const long long row = i / Cin;
  const int b = static_cast<int>(row / m.lin), s = static_cast<int>(row % m.lin);
  const size_t K = static_cast<size_t>(Cin) * taps;
  float v = 0.f;
  for (int p = m.lo[s]; p < m.lo[s + 1]; ++p)
    for (int j = 0; j < taps; ++j) {
      const int l = p - (j - taps / 2) * dil;
      if (l >= 0 && l < m.lout) v += dcol[(static_cast<size_t>(b) * m.lout + l) * K + static_cast<size_t>(c) * taps + j];
    }
  if (mask && !(mask[i] > 0.f)) v = 0.f;
  if (resid) v += resid[i];
  if (mask_out && !(mask_out[i] > 0.f)) v = 0.f;
  dX[i] = v;
}

// out (n floats) = max(in, 0)
__global__ void tk_relu_copy_kernel(const float* __restrict__ in, float* __restrict__ out, long long n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = fmaxf(in[i], 0.f);
}

// out[b] (C x R) = in[b]^T (in[b]: R x C) [+ add[b]], through a 32 x 33 shared tile
__global__ void __launch_bounds__(256) tk_transpose_kernel(const float* __restrict__ in, int R, int C,
                                                           const float* __restrict__ add, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const size_t base = static_cast<size_t>(blockIdx.z) * R * C;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32, tx = threadIdx.x, ty = threadIdx.y;
  for (int k = ty; k < 32; k += 8) {
    const int r = r0 + k, c = c0 + tx;
    if (r < R && c < C) tile[k][tx] = in[base + static_cast<size_t>(r) * C + c];
  }
  __syncthreads();
  for (int k = ty; k < 32; k += 8) {
    const int c = c0 + k, r = r0 + tx;
    if (r < R && c < C) {
      const size_t o = base + static_cast<size_t>(c) * R + r;
      out[o] = tile[tx][k] + (add ? add[o] : 0.f);
    }
  }
}

// LayerNorm over kTkMix columns (mixer_trans.ff.1, eps 1e-5) then ReLU; one 256-thread block per row.
__global__ void __launch_bounds__(256) tk_ln_wide_fwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                             const float* __restrict__ b, float* __restrict__ y,
                                                             float* __restrict__ mean, float* __restrict__ rstd) {
  constexpr int V = kTkMix / 1024;
  __shared__ float red[8];
  const int r = blockIdx.x, t = threadIdx.x;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(r) * kTkMix);
  float4 v[V];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = xr[t + 256 * i];
    s += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  const float mu = block_sum_256(s, red) * (1.f / kTkMix);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float d0 = v[i].x - mu, d1 = v[i].y - mu, d2 = v[i].z - mu, d3 = v[i].w - mu;
    q += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
  }
  const float rs = rsqrtf(block_sum_256(q, red) * (1.f / kTkMix) + kRhLnEps);
  float4* yr = reinterpret_cast<float4*>(y + static_cast<size_t>(r) * kTkMix);
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float4 gg = reinterpret_cast<const float4*>(g)[t + 256 * i], bb = reinterpret_cast<const float4*>(b)[t + 256 * i];
    yr[t + 256 * i] = make_float4(fmaxf((v[i].x - mu) * rs * gg.x + bb.x, 0.f), fmaxf((v[i].y - mu) * rs * gg.y + bb.y, 0.f),
                                  fmaxf((v[i].z - mu) * rs * gg.z + bb.z, 0.f), fmaxf((v[i].w - mu) * rs * gg.w + bb.w, 0.f));
  }
  if (t == 0) {
    mean[r] = mu;
    rstd[r] = rs;
  }
}

// Its backward: dy (the gradient at the ReLU's output) is masked in place by [y > 0], then dx = rstd (g dy - mean(g dy)
// - xhat mean(g dy xhat)) (overwritten).
__global__ void __launch_bounds__(256) tk_ln_wide_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                             const float* __restrict__ mean,
                                                             const float* __restrict__ rstd, const float* __restrict__ y,
                                                             float* __restrict__ dy, float* __restrict__ dx) {
  constexpr int V = kTkMix / 1024;
  __shared__ float red[8];
  const int r = blockIdx.x, t = threadIdx.x;
  const size_t o = static_cast<size_t>(r) * kTkMix;
  const float mu = mean[r], rs = rstd[r];
  float h[V][4], gd[V][4];
  float s1 = 0.f, s2 = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const int k = t + 256 * i;
    const float4 xv = reinterpret_cast<const float4*>(x + o)[k], yv = reinterpret_cast<const float4*>(y + o)[k];
    float4 d = reinterpret_cast<float4*>(dy + o)[k];
    const float4 gg = reinterpret_cast<const float4*>(g)[k];
    d.x = yv.x > 0.f ? d.x : 0.f; d.y = yv.y > 0.f ? d.y : 0.f; d.z = yv.z > 0.f ? d.z : 0.f; d.w = yv.w > 0.f ? d.w : 0.f;
    reinterpret_cast<float4*>(dy + o)[k] = d;
    h[i][0] = (xv.x - mu) * rs; h[i][1] = (xv.y - mu) * rs; h[i][2] = (xv.z - mu) * rs; h[i][3] = (xv.w - mu) * rs;
    gd[i][0] = d.x * gg.x; gd[i][1] = d.y * gg.y; gd[i][2] = d.z * gg.z; gd[i][3] = d.w * gg.w;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      s1 += gd[i][e];
      s2 += gd[i][e] * h[i][e];
    }
  }
  const float m1 = block_sum_256(s1, red) * (1.f / kTkMix), m2 = block_sum_256(s2, red) * (1.f / kTkMix);
#pragma unroll
  for (int i = 0; i < V; ++i)
    reinterpret_cast<float4*>(dx + o)[t + 256 * i] =
        make_float4(rs * (gd[i][0] - m1 - h[i][0] * m2), rs * (gd[i][1] - m1 - h[i][1] * m2),
                    rs * (gd[i][2] - m1 - h[i][2] * m2), rs * (gd[i][3] - m1 - h[i][3] * m2));
}

// LayerNorm over kTkHid = 64 columns (eps 1e-5), optionally then ReLU; one warp per row, eight rows per block.
__global__ void __launch_bounds__(256) tk_ln64_fwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                          const float* __restrict__ b, float* __restrict__ y,
                                                          float* __restrict__ mean, float* __restrict__ rstd, int rows,
                                                          int relu) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* xr = x + static_cast<size_t>(r) * kTkHid;
  const float a = xr[lane], c = xr[lane + 32];
  const float mu = warp_sum(a + c) * (1.f / kTkHid);
  const float da = a - mu, dc = c - mu;
  const float rs = rsqrtf(warp_sum(da * da + dc * dc) * (1.f / kTkHid) + kRhLnEps);
  float ya = da * rs * g[lane] + b[lane], yc = dc * rs * g[lane + 32] + b[lane + 32];
  if (relu) {
    ya = fmaxf(ya, 0.f);
    yc = fmaxf(yc, 0.f);
  }
  y[static_cast<size_t>(r) * kTkHid + lane] = ya;
  y[static_cast<size_t>(r) * kTkHid + lane + 32] = yc;
  if (lane == 0) {
    mean[r] = mu;
    rstd[r] = rs;
  }
}

// Its backward: with y (the ReLU's output) dy is first masked in place by [y > 0]; dx (+)= rstd (g dy - mean(g dy) -
// xhat mean(g dy xhat)).
__global__ void __launch_bounds__(256) tk_ln64_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                          const float* __restrict__ mean, const float* __restrict__ rstd,
                                                          const float* __restrict__ y, float* __restrict__ dy,
                                                          float* __restrict__ dx, int rows, int accumulate) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const size_t o = static_cast<size_t>(r) * kTkHid;
  float da = dy[o + lane], dc = dy[o + lane + 32];
  if (y) {
    da = y[o + lane] > 0.f ? da : 0.f;
    dc = y[o + lane + 32] > 0.f ? dc : 0.f;
    dy[o + lane] = da;
    dy[o + lane + 32] = dc;
  }
  const float mu = mean[r], rs = rstd[r];
  const float ha = (x[o + lane] - mu) * rs, hc = (x[o + lane + 32] - mu) * rs;
  const float ga = da * g[lane], gc = dc * g[lane + 32];
  const float m1 = warp_sum(ga + gc) * (1.f / kTkHid), m2 = warp_sum(ga * ha + gc * hc) * (1.f / kTkHid);
  const float va = rs * (ga - m1 - ha * m2), vc = rs * (gc - m1 - hc * m2);
  dx[o + lane] = accumulate ? dx[o + lane] + va : va;
  dx[o + lane + 32] = accumulate ? dx[o + lane + 32] + vc : vc;
}

// Row softmax over 2048 classes, in place (token_classifier.py:104): one warp per row loads the row into registers,
// then overwrites it.  One pointer, so the in-place use is well defined.
__global__ void __launch_bounds__(256) tk_softmax_fwd_kernel(float* x, int rows) {
  constexpr int V = kTkClasses / 128;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  float4* xr = reinterpret_cast<float4*>(x + static_cast<size_t>(r) * kTkClasses);
  float4 v[V];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = xr[i * 32 + lane];
    m = fmaxf(m, fmaxf(fmaxf(v[i].x, v[i].y), fmaxf(v[i].z, v[i].w)));
  }
  m = warp_max(m);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = make_float4(expf(v[i].x - m), expf(v[i].y - m), expf(v[i].z - m), expf(v[i].w - m));
    s += v[i].x + v[i].y + v[i].z + v[i].w;
  }
  const float inv = 1.0f / warp_sum(s);
#pragma unroll
  for (int i = 0; i < V; ++i) xr[i * 32 + lane] = make_float4(v[i].x * inv, v[i].y * inv, v[i].z * inv, v[i].w * inv);
}

// Softmax backward over 2048 classes, in place: dP <- P (dP - sum_c P dP); one warp per row.
__global__ void __launch_bounds__(256) tk_softmax_bwd_kernel(const float* __restrict__ P, float* __restrict__ dP,
                                                             int rows) {
  constexpr int V = kTkClasses / 128;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float4* pr = reinterpret_cast<const float4*>(P + static_cast<size_t>(r) * kTkClasses);
  float4* dr = reinterpret_cast<float4*>(dP + static_cast<size_t>(r) * kTkClasses);
  float4 p[V], d[V];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    p[i] = pr[i * 32 + lane];
    d[i] = dr[i * 32 + lane];
    s += p[i].x * d[i].x + p[i].y * d[i].y + p[i].z * d[i].z + p[i].w * d[i].w;
  }
  s = warp_sum(s);
#pragma unroll
  for (int i = 0; i < V; ++i)
    dr[i * 32 + lane] = make_float4(p[i].x * (d[i].x - s), p[i].y * (d[i].y - s), p[i].z * (d[i].z - s),
                                    p[i].w * (d[i].w - s));
}

// Two-stage column sums over many rows, in a fixed order: part[k, n] = sum of rows [k kTkColRows, (k+1) kTkColRows) of
// dy[:, n] (and, with x / mean / rstd, of dy xhat), then out[n] = sum_k part[k, n] in k order.
__global__ void tk_colsum_part_kernel(const float* __restrict__ dy, int ld, int rows, int N,
                                      const float* __restrict__ x, const float* __restrict__ mean,
                                      const float* __restrict__ rstd, float* __restrict__ part,
                                      float* __restrict__ part_g) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x, k = blockIdx.y;
  if (n >= N) return;
  const int r1 = min(rows, (k + 1) * kTkColRows);
  float s = 0.f, sg = 0.f;
  for (int r = k * kTkColRows; r < r1; ++r) {
    const float d = dy[static_cast<size_t>(r) * ld + n];
    s += d;
    if (x) sg += d * (x[static_cast<size_t>(r) * ld + n] - mean[r]) * rstd[r];
  }
  part[static_cast<size_t>(k) * N + n] = s;
  if (x) part_g[static_cast<size_t>(k) * N + n] = sg;
}

__global__ void tk_colsum_reduce_kernel(const float* __restrict__ part, const float* __restrict__ part_g, int chunks,
                                        int N, float* __restrict__ out, float* __restrict__ out_g) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float s = 0.f, sg = 0.f;
  for (int k = 0; k < chunks; ++k) {
    s += part[static_cast<size_t>(k) * N + n];
    if (out_g) sg += part_g[static_cast<size_t>(k) * N + n];
  }
  out[n] = s;
  if (out_g) out_g[n] = sg;
}

// ------------------------------------------------------------------------------------------------ workspace
struct TkBlockAct {
  float *y1t;                 // LN1 output, transposed: (B, 64, 160)
  float *m1, *r1, *m2, *r2;   // LN statistics, B*160 each
  float *u1, *h1;             // token MLP pre-GELU and GELU: (B*64, 64)
  float *s;                   // x + token MLP output: (B*160, 64)
  float *y2;                  // LN2 output
  float *u2, *h2;             // channel MLP pre-GELU and GELU: (B*160, 256)
};
struct TkWs {
  RhWs dec;                   // the decoder's activations and scratch; read / pose6d / dread are the read-outs'
  float *f0, *mt_mean, *mt_rstd;
  float* X[kTkBlocks + 1];    // mixer inputs; X[0] = ReLU(LN(f0)), X[kTkBlocks] the last block's output
  TkBlockAct blk[kTkBlocks];
  float *u3, *m3, *r3, *x4;   // mixer_norm_layer: pre-LN, stats, post-ReLU
  float* Y[kTkUps + 1];       // conv outputs before their ReLU: 160, 125, 90, 55, 21 positions x 512
  float *hh[kTkResBlocks], *x1, *x2, *Y5, *Y6;   // ResNet1D conv1 outputs, block outputs, post conv, (B*21, 6)
  // scratch
  float *col, *dcol, *gA, *gB, *gx, *gy, *gz, *gU, *dP, *part, *part_g;
  size_t floats;
};

inline void tk_carve(float* base, int B, int depth, int H, int mlp, TkWs* w) {
  rh_carve(base, B, depth, H, mlp, &w->dec);
  size_t off = w->dec.floats;
  auto take = [&](size_t n) {
    float* p = base ? base + off : nullptr;
    off += (n + 63) / 64 * 64;
    return p;
  };
  const size_t b = B, rows = b * kTkT;
  w->f0 = take(b * kTkMix); w->mt_mean = take(b); w->mt_rstd = take(b);
  for (int i = 0; i <= kTkBlocks; ++i) w->X[i] = take(rows * kTkHid);
  for (int i = 0; i < kTkBlocks; ++i) {
    TkBlockAct& a = w->blk[i];
    a.y1t = take(rows * kTkHid);
    a.m1 = take(rows); a.r1 = take(rows); a.m2 = take(rows); a.r2 = take(rows);
    a.u1 = take(b * kTkHid * kTkTokInter); a.h1 = take(b * kTkHid * kTkTokInter);
    a.s = take(rows * kTkHid); a.y2 = take(rows * kTkHid);
    a.u2 = take(rows * kTkChInter); a.h2 = take(rows * kTkChInter);
  }
  w->u3 = take(rows * kTkHid); w->m3 = take(rows); w->r3 = take(rows); w->x4 = take(rows * kTkHid);
  w->Y[0] = take(rows * kTkWidth);
  for (int u = 0; u < kTkUps; ++u) w->Y[u + 1] = take(b * kTkUpLen[u] * kTkWidth);
  const size_t j = b * kTkJoints * kTkWidth;
  for (int d = 0; d < kTkResBlocks; ++d) w->hh[d] = take(j);
  w->x1 = take(j); w->x2 = take(j); w->Y5 = take(j); w->Y6 = take(b * kTkJoints * 6);
  size_t colf = rows * kTkCode * 3;
  for (int u = 0; u < kTkUps; ++u) colf = std::max(colf, b * kTkUpLen[u] * kTkWidth * 3);
  w->col = take(colf); w->dcol = take(colf);
  w->gA = take(rows * kTkWidth); w->gB = take(rows * kTkWidth);
  w->gx = take(rows * kTkHid); w->gy = take(rows * kTkHid); w->gz = take(rows * kTkHid);
  w->gU = take(rows * kTkChInter);
  w->dP = take(rows * kTkClasses);
  // the widest column sums: 2048 columns over B*160 rows, and 10240 columns over B rows
  auto chunks = [](size_t r) { return (r + kTkColRows - 1) / kTkColRows; };
  const size_t pf = std::max(chunks(rows) * kTkClasses, chunks(b) * kTkMix);
  w->part = take(pf); w->part_g = take(pf);
  w->floats = off;
}

inline size_t tk_workspace_bytes(int B, int depth, int H, int mlp) {
  TkWs w;
  tk_carve(nullptr, B, depth, H, mlp, &w);
  return w.floats * sizeof(float);
}

// ------------------------------------------------------------------------------------------------ launch helpers
inline unsigned tk_blocks(long long n, int t = 256) { return static_cast<unsigned>((n + t - 1) / t); }

// out = sum over rows of dy (N columns, leading dim ld); with x / mean / rstd also out_g = sum of dy xhat
inline void tk_colsum(const float* dy, int ld, int rows, int N, float* out, const float* x, const float* mean,
                      const float* rstd, float* out_g, TkWs& w, cudaStream_t st) {
  const int chunks = (rows + kTkColRows - 1) / kTkColRows;
  tk_colsum_part_kernel<<<dim3((N + 127) / 128, chunks), 128, 0, st>>>(dy, ld, rows, N, x, mean, rstd, w.part,
                                                                       w.part_g);
  tk_colsum_reduce_kernel<<<(N + 127) / 128, 128, 0, st>>>(w.part, w.part_g, chunks, N, out, x ? out_g : nullptr);
}

// dW (N x K) = dy^T (rows x N, ld ldy) x (rows x K, ld ldx), split over the rows when the grid is small
inline void tk_linear_dw(const float* dy, int ldy, const float* x, int ldx, float* dW, int rows, int N, int K,
                         float* partial, cudaStream_t st) {
  HlGemm p = hl_make(N, K, rows, partial);
  p.A = dy; p.sAm = 1; p.sAk = ldy;
  p.Bm = x; p.sBk = ldx; p.sBn = 1;
  p.C = dW; p.ldc = K;
  hl_gemm(p, kDytX, st);
}

// Y (B*lout x Cout) = conv(act(X)) through im2col; X is (B*lin x Cin)
inline void tk_conv(const float* X, int Cin, const TkSeqMap& m, int taps, int dil, int relu, const float* W,
                    const float* bias, int Cout, float* Y, bool accumulate, int B, TkWs& w, cudaStream_t st) {
  const int K = Cin * taps, rows = B * m.lout;
  tk_im2col_kernel<<<tk_blocks(static_cast<long long>(rows) * K), 256, 0, st>>>(X, Cin, m, taps, dil, relu, w.col, B);
  hl_linear(w.col, K, W, bias, Y, Cout, rows, Cout, K, accumulate, nullptr, w.dec.split, st);
}

// the conv's backward to its input, from dcol = dY W already in w.dcol
inline void tk_col2im(int Cin, const TkSeqMap& m, int taps, int dil, const float* mask, const float* resid,
                      const float* mask_out, float* dX, int B, TkWs& w, cudaStream_t st) {
  tk_col2im_kernel<<<tk_blocks(static_cast<long long>(B) * m.lin * Cin), 256, 0, st>>>(w.dcol, Cin, m, taps, dil, mask,
                                                                                       resid, mask_out, dX, B);
}

inline void tk_conv_bwd(const float* dY, int Cout, const float* W, int Cin, const TkSeqMap& m, int taps, int dil,
                        const float* mask, const float* resid, const float* mask_out, float* dX, int B, TkWs& w,
                        cudaStream_t st) {
  const int K = Cin * taps, rows = B * m.lout;
  hl_linear_dx(dY, Cout, W, w.dcol, K, rows, Cout, K, false, nullptr, w.dec.split, st);
  tk_col2im(Cin, m, taps, dil, mask, resid, mask_out, dX, B, w, st);
}

inline void tk_transpose(const float* in, int R, int C, const float* add, float* out, int B, cudaStream_t st) {
  tk_transpose_kernel<<<dim3((C + 31) / 32, (R + 31) / 32, B), dim3(32, 8), 0, st>>>(in, R, C, add, out);
}

// ------------------------------------------------------------------------------------------------ forward
inline int tk_forward(const thmr_tok_head_desc& d, TkWs& w, cudaStream_t st) {
  const int B = d.B, E = kRhDim, rows = B * kTkT;
  TkPtrs P;
  TkTok K;
  tk_pointers(const_cast<float*>(d.params), d.depth, d.heads, d.mlp_dim, &P);
  tk_tokenizer_pointers(d.tokenizer, &K);
  THMR_TRY(rh_decoder_forward(P.dec, d.feats, B, d.depth, d.heads, d.mlp_dim, w.dec, st));
  float* const* T = P.t;
  float* split = w.dec.split;
  // read-outs (token_head.py:99-105) into [grot | hands | betas | cam], head_assemble_kernel's token layout
  float* rd = w.dec.read;
  hl_linear(w.dec.tok, E, T[kTgW], T[kTgB], rd, kRhReadLd, B, 6, E, false, nullptr, split, st);
  hl_linear(w.dec.tok, E, T[kThW], T[kThB], rd + 6, kRhReadLd, B, 12, E, false, nullptr, split, st);
  hl_linear(w.dec.tok, E, T[kTsW], T[kTsB], rd + 18, kRhReadLd, B, kRhBetas, E, false, nullptr, split, st);
  hl_linear(w.dec.tok, E, T[kTcW], T[kTcB], rd + 28, kRhReadLd, B, kRhCam, E, false, nullptr, split, st);
  // classifier (token_classifier.py:89-104, modules.py:11-63)
  hl_linear(w.dec.tok, E, T[kTmtW], T[kTmtB], w.f0, kTkMix, B, kTkMix, E, false, nullptr, split, st);
  tk_ln_wide_fwd_kernel<<<B, 256, 0, st>>>(w.f0, T[kTmtG], T[kTmtBeta], w.X[0], w.mt_mean, w.mt_rstd);
  const unsigned lnb = (rows + 7) / 8;
  for (int i = 0; i < kTkBlocks; ++i) {
    TkBlockAct& a = w.blk[i];
    float* X = w.X[i];
    tk_ln64_fwd_kernel<<<lnb, 256, 0, st>>>(X, P.mix(i, kM1g), P.mix(i, kM1b), w.gx, a.m1, a.r1, rows, 0);
    tk_transpose(w.gx, kTkT, kTkHid, nullptr, a.y1t, B, st);
    hl_linear(a.y1t, kTkT, P.mix(i, kMt1w), P.mix(i, kMt1b), a.u1, kTkTokInter, B * kTkHid, kTkTokInter, kTkT, false,
              a.h1, split, st);
    hl_linear(a.h1, kTkTokInter, P.mix(i, kMt2w), P.mix(i, kMt2b), w.gy, kTkT, B * kTkHid, kTkT, kTkTokInter, false,
              nullptr, split, st);
    tk_transpose(w.gy, kTkHid, kTkT, X, a.s, B, st);                          // s = x + token MLP output
    tk_ln64_fwd_kernel<<<lnb, 256, 0, st>>>(a.s, P.mix(i, kM2g), P.mix(i, kM2b), a.y2, a.m2, a.r2, rows, 0);
    hl_linear(a.y2, kTkHid, P.mix(i, kMc1w), P.mix(i, kMc1b), a.u2, kTkChInter, rows, kTkChInter, kTkHid, false, a.h2,
              split, st);
    THMR_CUDA(cudaMemcpyAsync(w.X[i + 1], a.s, sizeof(float) * rows * kTkHid, cudaMemcpyDeviceToDevice, st));
    hl_linear(a.h2, kTkChInter, P.mix(i, kMc2w), P.mix(i, kMc2b), w.X[i + 1], kTkHid, rows, kTkHid, kTkChInter, true,
              nullptr, split, st);
  }
  hl_linear(w.X[kTkBlocks], kTkHid, T[kTmnW], T[kTmnB], w.u3, kTkHid, rows, kTkHid, kTkHid, false, nullptr, split, st);
  tk_ln64_fwd_kernel<<<lnb, 256, 0, st>>>(w.u3, T[kTmnG], T[kTmnBeta], w.x4, w.m3, w.r3, rows, 1);
  // the logits go straight into the cls_logits_softmax output, which the softmax overwrites in place; the backward
  // reads P from there, so no second (B, 160, 2048) buffer exists
  float* const probs = d.cls_probs;
  hl_linear(w.x4, kTkHid, T[kTclsW], T[kTclsB], probs, kTkClasses, rows, kTkClasses, kTkHid, false, nullptr, split, st);
  tk_softmax_fwd_kernel<<<(rows + 7) / 8, 256, 0, st>>>(probs, rows);
                                                                                      // row before it writes it
  // tokenizer decoder (vanilla_pose_vqvae.py:135-154, 294-297): Z = P codebook, then the convolutions
  hl_linear_dx(probs, kTkClasses, K.t[kKcb], w.gA, kTkCode, rows, kTkClasses, kTkCode, false, nullptr, split, st);
  tk_conv(w.gA, kTkCode, tk_seq_map(kTkT, kTkT), 3, 1, 0, K.t[kK0w], K.t[kK0b], kTkWidth, w.Y[0], false, B, w, st);
  int len = kTkT;
  for (int u = 0; u < kTkUps; ++u) {
    tk_conv(w.Y[u], kTkWidth, tk_seq_map(len, kTkUpLen[u]), 3, 1, 1, K.t[kKup + 2 * u], K.t[kKup + 2 * u + 1],
            kTkWidth, w.Y[u + 1], false, B, w, st);
    len = kTkUpLen[u];
  }
  const TkSeqMap id = tk_seq_map(kTkJoints, kTkJoints);
  const long long nj = static_cast<long long>(B) * kTkJoints * kTkWidth;
  // ResNet1D (resnet.py:51-82): x += conv2(relu(conv1(relu(x)))); its input is relu(Y4)
  tk_relu_copy_kernel<<<tk_blocks(nj), 256, 0, st>>>(w.Y[kTkUps], w.x1, nj);
  const float* xin[kTkResBlocks] = {w.Y[kTkUps], w.x1};
  float* xout[kTkResBlocks] = {w.x1, w.x2};
  for (int r = 0; r < kTkResBlocks; ++r) {
    const float* const* c = &K.t[kKres + 4 * r];
    tk_conv(xin[r], kTkWidth, id, 3, kTkResDil[r], 1, c[0], c[1], kTkWidth, w.hh[r], false, B, w, st);
    if (r > 0) THMR_CUDA(cudaMemcpyAsync(xout[r], xout[r - 1], sizeof(float) * nj, cudaMemcpyDeviceToDevice, st));
    tk_conv(w.hh[r], kTkWidth, id, 1, 1, 1, c[2], c[3], kTkWidth, xout[r], true, B, w, st);
  }
  tk_conv(w.x2, kTkWidth, id, 3, 1, 0, K.t[kKpostW], K.t[kKpostB], kTkWidth, w.Y5, false, B, w, st);
  tk_conv(w.Y5, kTkWidth, id, 3, 1, 0, K.t[kKoutW], K.t[kKoutB], 6, w.Y6, false, B, w, st);
  // assembly: cat[grot, body, hands] + init_body_pose, rot6d_to_rotmat; betas / cam + init_*
  head_assemble_kernel<<<(B * 24 + 127) / 128, 128, 0, st>>>(rd, kRhReadLd, w.Y6, 6, kTkJoints, 0, d.init_body_pose,
                                                             d.init_betas, d.init_cam, d.rotmats, d.betas, d.cam,
                                                             w.dec.pose6d, B, kRhBetas);
  THMR_CUDA(cudaGetLastError());
  if (d.pose6d)
    THMR_CUDA(cudaMemcpyAsync(d.pose6d, w.dec.pose6d, sizeof(float) * B * kRhPose, cudaMemcpyDeviceToDevice, st));
  return THMR_OK;
}

// ------------------------------------------------------------------------------------------------ backward
inline int tk_backward(const thmr_tok_head_desc& d, TkWs& w, cudaStream_t st) {
  const int B = d.B, E = kRhDim, rows = B * kTkT;
  TkPtrs P, G;
  TkTok K;
  tk_pointers(const_cast<float*>(d.params), d.depth, d.heads, d.mlp_dim, &P);
  tk_pointers(d.grads, d.depth, d.heads, d.mlp_dim, &G);
  tk_tokenizer_pointers(d.tokenizer, &K);
  float* const* T = P.t;
  float* const* Tg = G.t;
  float* split = w.dec.split;
  // read-outs: dread = [d pose6d (144) | d betas | d cam]; pose6d = [grot (6) | body (126) | hands (12)]
  float* dr = w.dec.dread;
  rh_readout_bwd_kernel<<<(B * 24 + 127) / 128, 128, 0, st>>>(w.dec.pose6d, d.grad_rotmats, d.grad_pose6d,
                                                              d.grad_betas, d.grad_cam, dr, B);
  const int rn[4] = {6, 12, kRhBetas, kRhCam}, col[4] = {0, 132, kRhPose, kRhPose + kRhBetas};
  const int wi[4] = {kTgW, kThW, kTsW, kTcW};
  for (int r = 0; r < 4; ++r) {
    hl_linear_dw(dr + col[r], kRhReadLd, w.dec.tok, E, Tg[wi[r]], B, rn[r], E, 1.f, st);
    rh_colsum_kernel<<<1, 256, 0, st>>>(dr + col[r], kRhReadLd, B, rn[r], Tg[wi[r] + 1], nullptr, nullptr, nullptr,
                                        nullptr, nullptr);
    hl_linear_dx(dr + col[r], kRhReadLd, T[wi[r]], w.dec.dx, E, B, rn[r], E, r > 0, nullptr, split, st);
  }
  // tokenizer decoder, to its input: conv_out's dY is the body columns of dread, (B, 21, 6) at row stride 160
  const TkSeqMap id = tk_seq_map(kTkJoints, kTkJoints);
  {
    HlGemm p = hl_make(kTkJoints, 3 * kTkWidth, 6, split);
    p.batch = B;
    p.A = dr + 6; p.sAm = 6; p.sAk = 1; p.sAz = kRhReadLd;
    p.Bm = K.t[kKoutW]; p.sBk = 3 * kTkWidth; p.sBn = 1;
    p.C = w.dcol; p.ldc = 3 * kTkWidth; p.sCz = static_cast<long long>(kTkJoints) * 3 * kTkWidth;
    hl_gemm(p, kDyW, st);
  }
  tk_col2im(kTkWidth, id, 3, 1, nullptr, nullptr, nullptr, w.gA, B, w, st);                         // d Y5
  tk_conv_bwd(w.gA, kTkWidth, K.t[kKpostW], kTkWidth, id, 3, 1, nullptr, nullptr, nullptr, w.gB, B, w, st);   // d x2
  // ResNet1D blocks, last first: x_out = x_in + conv2(relu(hh)), hh = conv1(relu(x_in))
  {
    const float* const* c = &K.t[kKres + 4];
    tk_conv_bwd(w.gB, kTkWidth, c[2], kTkWidth, id, 1, 1, w.hh[1], nullptr, nullptr, w.gA, B, w, st);     // d hh1
    tk_conv_bwd(w.gA, kTkWidth, c[0], kTkWidth, id, 3, kTkResDil[1], w.x1, w.gB, nullptr, w.gA, B, w, st);   // d x1
    c = &K.t[kKres];
    tk_conv_bwd(w.gA, kTkWidth, c[2], kTkWidth, id, 1, 1, w.hh[0], nullptr, nullptr, w.gB, B, w, st);     // d hh0
    // x1 = relu(Y4) + ..., hh0 = conv1(relu(Y4)): d Y4 = [Y4 > 0] (d x1 + conv1's backward)
    tk_conv_bwd(w.gB, kTkWidth, c[0], kTkWidth, id, 3, kTkResDil[0], nullptr, w.gA, w.Y[kTkUps], w.gB, B, w, st);
  }
  float *gcur = w.gB, *gnext = w.gA;
  for (int u = kTkUps - 1; u >= 0; --u) {
    const int lin = u == 0 ? kTkT : kTkUpLen[u - 1];
    tk_conv_bwd(gcur, kTkWidth, K.t[kKup + 2 * u], kTkWidth, tk_seq_map(lin, kTkUpLen[u]), 3, 1, w.Y[u], nullptr,
                nullptr, gnext, B, w, st);   // d Y_u: through the resize and Y_u's ReLU
    std::swap(gcur, gnext);
  }
  tk_conv_bwd(gcur, kTkWidth, K.t[kK0w], kTkCode, tk_seq_map(kTkT, kTkT), 3, 1, nullptr, nullptr, nullptr, gnext, B, w,
              st);   // d Z (B*160, 256)
  // soft lookup: dP = dZ codebook^T (+ the cls_logits_softmax gradient), then the softmax's backward
  if (d.grad_cls_probs)
    THMR_CUDA(cudaMemcpyAsync(w.dP, d.grad_cls_probs, sizeof(float) * rows * kTkClasses, cudaMemcpyDeviceToDevice, st));
  hl_linear(gnext, kTkCode, K.t[kKcb], nullptr, w.dP, kTkClasses, rows, kTkClasses, kTkCode, d.grad_cls_probs != nullptr,
            nullptr, split, st);
  tk_softmax_bwd_kernel<<<(rows + 7) / 8, 256, 0, st>>>(d.cls_probs, w.dP, rows);
  // class_pred_layer
  tk_colsum(w.dP, kTkClasses, rows, kTkClasses, Tg[kTclsB], nullptr, nullptr, nullptr, nullptr, w, st);
  tk_linear_dw(w.dP, kTkClasses, w.x4, kTkHid, Tg[kTclsW], rows, kTkClasses, kTkHid, split, st);
  hl_linear_dx(w.dP, kTkClasses, T[kTclsW], w.gy, kTkHid, rows, kTkClasses, kTkHid, false, nullptr, split, st);
  // mixer_norm_layer: x4 = relu(LN(u3)), u3 = Linear(X[4])
  const unsigned lnb = (rows + 7) / 8;
  tk_ln64_bwd_kernel<<<lnb, 256, 0, st>>>(w.u3, T[kTmnG], w.m3, w.r3, w.x4, w.gy, w.gz, rows, 0);
  tk_colsum(w.gy, kTkHid, rows, kTkHid, Tg[kTmnBeta], w.u3, w.m3, w.r3, Tg[kTmnG], w, st);
  tk_colsum(w.gz, kTkHid, rows, kTkHid, Tg[kTmnB], nullptr, nullptr, nullptr, nullptr, w, st);
  tk_linear_dw(w.gz, kTkHid, w.X[kTkBlocks], kTkHid, Tg[kTmnW], rows, kTkHid, kTkHid, split, st);
  hl_linear_dx(w.gz, kTkHid, T[kTmnW], w.gx, kTkHid, rows, kTkHid, kTkHid, false, nullptr, split, st);
  // mixer layers, last first; w.gx carries d(layer output) -> d(layer input)
  for (int i = kTkBlocks - 1; i >= 0; --i) {
    TkBlockAct& a = w.blk[i];
    // channel MLP: out = s + W2 gelu(W1 LN2(s) + b1) + b2
    tk_colsum(w.gx, kTkHid, rows, kTkHid, G.mix(i, kMc2b), nullptr, nullptr, nullptr, nullptr, w, st);
    tk_linear_dw(w.gx, kTkHid, a.h2, kTkChInter, G.mix(i, kMc2w), rows, kTkHid, kTkChInter, split, st);
    hl_linear_dx(w.gx, kTkHid, P.mix(i, kMc2w), w.gU, kTkChInter, rows, kTkHid, kTkChInter, false, a.u2, split, st);
    tk_colsum(w.gU, kTkChInter, rows, kTkChInter, G.mix(i, kMc1b), nullptr, nullptr, nullptr, nullptr, w, st);
    tk_linear_dw(w.gU, kTkChInter, a.y2, kTkHid, G.mix(i, kMc1w), rows, kTkChInter, kTkHid, split, st);
    hl_linear_dx(w.gU, kTkChInter, P.mix(i, kMc1w), w.gy, kTkHid, rows, kTkChInter, kTkHid, false, nullptr, split, st);
    tk_colsum(w.gy, kTkHid, rows, kTkHid, G.mix(i, kM2b), a.s, a.m2, a.r2, G.mix(i, kM2g), w, st);
    tk_ln64_bwd_kernel<<<lnb, 256, 0, st>>>(a.s, P.mix(i, kM2g), a.m2, a.r2, nullptr, w.gy, w.gx, rows, 1);   // d s
    // token MLP, on the transposed (B, 64, 160) rows: s = x + (W2 gelu(W1 LN1(x)^T + b1) + b2)^T
    tk_transpose(w.gx, kTkT, kTkHid, nullptr, w.gz, B, st);
    tk_colsum(w.gz, kTkT, B * kTkHid, kTkT, G.mix(i, kMt2b), nullptr, nullptr, nullptr, nullptr, w, st);
    tk_linear_dw(w.gz, kTkT, a.h1, kTkTokInter, G.mix(i, kMt2w), B * kTkHid, kTkT, kTkTokInter, split, st);
    hl_linear_dx(w.gz, kTkT, P.mix(i, kMt2w), w.gU, kTkTokInter, B * kTkHid, kTkT, kTkTokInter, false, a.u1, split,
                 st);
    tk_colsum(w.gU, kTkTokInter, B * kTkHid, kTkTokInter, G.mix(i, kMt1b), nullptr, nullptr, nullptr, nullptr, w, st);
    tk_linear_dw(w.gU, kTkTokInter, a.y1t, kTkT, G.mix(i, kMt1w), B * kTkHid, kTkTokInter, kTkT, split, st);
    hl_linear_dx(w.gU, kTkTokInter, P.mix(i, kMt1w), w.gz, kTkT, B * kTkHid, kTkTokInter, kTkT, false, nullptr, split,
                 st);
    tk_transpose(w.gz, kTkHid, kTkT, nullptr, w.gy, B, st);                                                // d LN1 out
    tk_colsum(w.gy, kTkHid, rows, kTkHid, G.mix(i, kM1b), w.X[i], a.m1, a.r1, G.mix(i, kM1g), w, st);
    tk_ln64_bwd_kernel<<<lnb, 256, 0, st>>>(w.X[i], P.mix(i, kM1g), a.m1, a.r1, nullptr, w.gy, w.gx, rows, 1);  // d x
  }
  // mixer_trans: X[0] = relu(LN(f0)), f0 = Linear(tok); w.gx is d X[0] as (B, 10240)
  tk_ln_wide_bwd_kernel<<<B, 256, 0, st>>>(w.f0, T[kTmtG], w.mt_mean, w.mt_rstd, w.X[0], w.gx, w.gz);
  tk_colsum(w.gx, kTkMix, B, kTkMix, Tg[kTmtBeta], w.f0, w.mt_mean, w.mt_rstd, Tg[kTmtG], w, st);
  tk_colsum(w.gz, kTkMix, B, kTkMix, Tg[kTmtB], nullptr, nullptr, nullptr, nullptr, w, st);
  hl_linear_dw(w.gz, kTkMix, w.dec.tok, E, Tg[kTmtW], B, kTkMix, E, 1.f, st);
  hl_linear_dx(w.gz, kTkMix, T[kTmtW], w.dec.dx, E, B, kTkMix, E, true, nullptr, split, st);
  THMR_TRY(rh_decoder_backward(P.dec, G.dec, d.feats, B, d.depth, d.heads, d.mlp_dim, w.dec, st));
  THMR_CUDA(cudaGetLastError());
  return THMR_OK;
}

}  // namespace thmr
