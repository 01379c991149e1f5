// Test-only probe of the two heads' training kernels (tests/libthmr_head_train_probe.so): thin extern "C" wrappers
// around what rh_forward / rh_backward in tokenhmr_b200/csrc/head_train.cuh and tk_forward / tk_backward in
// tokenhmr_b200/csrc/token_head_train.cuh launch, each with the engine's grid, block and shared-memory sizes.
//   regression head: hl_gemm through its own planner, the cross-attention chunk and combine kernels, LayerNorm forward
//                    and backward, the column sums, token 0 and the read-out backward;
//   token head:      im2col and its gather backward through a resize map, ReLU copy, the batched transpose, LayerNorm
//                    at widths 10240 and 64, the softmax, the two-stage column sums, the conv composites, and the
//                    host-side resize map itself.
// Used by tests/test_gpu_head_train_kernels.py and tests/test_gpu_token_head_train_kernels.py; ctypes twin:
// tests/head_train_probe.py.  The product never loads this library.
#include <stdint.h>

#include "../../tokenhmr_b200/csrc/common.cuh"
#include "../../tokenhmr_b200/csrc/head_train.cuh"
#include "../../tokenhmr_b200/csrc/token_head_train.cuh"

using namespace thmr;

#define HEAD_PROBE_API extern "C" __attribute__((visibility("default")))

static cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }

#define PROBE_LAUNCHED()           \
  do {                             \
    THMR_CUDA(cudaGetLastError()); \
    return THMR_OK;                \
  } while (0)

HEAD_PROBE_API const char* head_probe_last_error(void) { return last_error_buf(); }

// Reads and clears this library's own device status words (its copies of g_pipeline_timeout and g_strict_overflow).
// Returns bit 0 = pipeline timeout, bit 1 = split-precision overflow, or -1 on a CUDA error.
HEAD_PROBE_API int head_probe_check_device_flags(void) {
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  unsigned int t = 0, o = 0, zero = 0;
  if (cudaMemcpyFromSymbol(&t, g_pipeline_timeout, sizeof(t)) != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(&o, g_strict_overflow, sizeof(o)) != cudaSuccess) return -1;
  if (cudaMemcpyToSymbol(g_pipeline_timeout, &zero, sizeof(zero)) != cudaSuccess) return -1;
  if (cudaMemcpyToSymbol(g_strict_overflow, &zero, sizeof(zero)) != cudaSuccess) return -1;
  return (t ? 1 : 0) | (o ? 2 : 0);
}

HEAD_PROBE_API size_t head_probe_hl_gemm_desc_size(void) { return sizeof(HlGemm); }
HEAD_PROBE_API long long head_probe_hl_split_floats(void) { return kSplitFloats; }

// hl_gemm as the engine calls it, in orientation orient (kXWt / kDyW / kDytX); g->splits is ignored (the planner sets
// it).  Returns the split count it launched with, or a negative status.
HEAD_PROBE_API int head_probe_hl_gemm(const HlGemm* g, int orient, void* stream) {
  THMR_CHECK(g && g->A && g->Bm && g->C && orient >= kXWt && orient <= kDytX, "head_probe_hl_gemm: bad argument");
  hl_gemm(*g, static_cast<HlOrient>(orient), as_stream(stream));
  THMR_CUDA(cudaGetLastError());
  return hl_split_count(*g);
}

// rh_forward's cross-attention: chunk kernel <false> on (kRhChunks, B), then the combine -> s [B,H,192],
// stat [B,12,H,2], part [B,12,H,1280], c [B,H,1280], lse [B,H]
HEAD_PROBE_API int head_probe_rh_attn_fwd(const float* X, const float* kq, int H, float scale, int B, float* s,
                                          float* stat, float* part, float* c, float* lse, void* stream) {
  THMR_TRY(rh_configure());
  cudaStream_t st = as_stream(stream);
  rh_attn_chunk_kernel<false><<<dim3(kRhChunks, B), 256, kRhAttSmem, st>>>(X, kq, H, scale, s, nullptr, nullptr,
                                                                          nullptr, stat, part);
  rh_attn_combine_kernel<<<B * H, 256, 0, st>>>(part, stat, H, c, lse);
  PROBE_LAUNCHED();
}

// rh_backward's: chunk kernel <true> (dtil [B,H,1280], s, lse, dO / o [B, 64 H]), then the combine without stat -> u
HEAD_PROBE_API int head_probe_rh_attn_bwd(const float* X, const float* dtil, int H, float scale, int B, const float* s,
                                          const float* lse, const float* dO, const float* o, float* part, float* u,
                                          void* stream) {
  THMR_TRY(rh_configure());
  cudaStream_t st = as_stream(stream);
  rh_attn_chunk_kernel<true><<<dim3(kRhChunks, B), 256, kRhAttSmem, st>>>(X, dtil, H, scale, const_cast<float*>(s),
                                                                         lse, dO, o, nullptr, part);
  rh_attn_combine_kernel<<<B * H, 256, 0, st>>>(part, nullptr, H, u, nullptr);
  PROBE_LAUNCHED();
}

HEAD_PROBE_API int head_probe_rh_ln_fwd(const float* x, const float* g, const float* b, float* y, float* mean,
                                        float* rstd, int B, void* stream) {
  rh_ln_fwd_kernel<<<B, 256, 0, as_stream(stream)>>>(x, g, b, y, mean, rstd);
  PROBE_LAUNCHED();
}

HEAD_PROBE_API int head_probe_rh_ln_bwd(const float* x, const float* g, const float* mean, const float* rstd,
                                        const float* dy, float* dx, int B, void* stream) {
  rh_ln_bwd_kernel<<<B, 256, 0, as_stream(stream)>>>(x, g, mean, rstd, dy, dx);
  PROBE_LAUNCHED();
}

// threads 256: the read-outs' <<<1, 256>>> (N <= 256); 128: the <<<ceil(N / 128), 128>>> of every other column sum
HEAD_PROBE_API int head_probe_rh_colsum(int threads, const float* dy, int ld, int B, int N, float* out, float* out2,
                                        const float* x, const float* mean, const float* rstd, float* out_g,
                                        void* stream) {
  THMR_CHECK((threads == 256 && N <= 256) || threads == 128, "head_probe_rh_colsum: threads %d N %d", threads, N);
  const unsigned grid = threads == 256 ? 1u : static_cast<unsigned>((N + 127) / 128);
  rh_colsum_kernel<<<grid, threads, 0, as_stream(stream)>>>(dy, ld, B, N, out, out2, x, mean, rstd, out_g);
  PROBE_LAUNCHED();
}

HEAD_PROBE_API int head_probe_rh_token0(const float* tok_b, const float* pos, float* x, int B, void* stream) {
  rh_token0_kernel<<<(B * kRhDim + 255) / 256, 256, 0, as_stream(stream)>>>(tok_b, pos, x, B);
  PROBE_LAUNCHED();
}

// Any of g_rot, g_pose6d, g_betas and g_cam may be null.  dread [B, 160]
HEAD_PROBE_API int head_probe_rh_readout_bwd(const float* pose6d, const float* g_rot, const float* g_pose6d,
                                             const float* g_betas, const float* g_cam, float* dread, int B,
                                             void* stream) {
  rh_readout_bwd_kernel<<<(B * 24 + 127) / 128, 128, 0, as_stream(stream)>>>(pose6d, g_rot, g_pose6d, g_betas, g_cam,
                                                                           dread, B);
  PROBE_LAUNCHED();
}

// ------------------------------------------------------------------------------------------------ token head
#define TK_MAP_CHECK(lin, lout)                                                                            \
  THMR_CHECK((lin) >= 1 && (lin) <= kTkT && (lout) >= 1 && (lout) <= kTkT, "tk_seq_map: lin %d lout %d outside 1..%d", \
             (lin), (lout), kTkT)

// The resize map on the host: src[0 .. lout) and lo[0 .. lin] (tk_seq_map's arrays, as the kernels receive them).
HEAD_PROBE_API int head_probe_tk_seq_map(int lin, int lout, short* src, short* lo) {
  TK_MAP_CHECK(lin, lout);
  THMR_CHECK(src && lo, "head_probe_tk_seq_map: null output");
  const TkSeqMap m = tk_seq_map(lin, lout);
  for (int p = 0; p < lout; ++p) src[p] = m.src[p];
  for (int s = 0; s <= lin; ++s) lo[s] = m.lo[s];
  return THMR_OK;
}

// col (B*lout x Cin*taps) from X (B*lin x Cin), as tk_conv launches it
HEAD_PROBE_API int head_probe_tk_im2col(const float* X, int Cin, int lin, int lout, int taps, int dil, int relu,
                                        float* col, int B, void* stream) {
  TK_MAP_CHECK(lin, lout);
  const long long n = static_cast<long long>(B) * lout * Cin * taps;
  tk_im2col_kernel<<<tk_blocks(n), 256, 0, as_stream(stream)>>>(X, Cin, tk_seq_map(lin, lout), taps, dil, relu, col, B);
  PROBE_LAUNCHED();
}

// dX (B*lin x Cin) from dcol (B*lout x Cin*taps); mask, resid and mask_out may be null
HEAD_PROBE_API int head_probe_tk_col2im(const float* dcol, int Cin, int lin, int lout, int taps, int dil,
                                        const float* mask, const float* resid, const float* mask_out, float* dX, int B,
                                        void* stream) {
  TK_MAP_CHECK(lin, lout);
  TkWs w{};
  w.dcol = const_cast<float*>(dcol);
  tk_col2im(Cin, tk_seq_map(lin, lout), taps, dil, mask, resid, mask_out, dX, B, w, as_stream(stream));
  PROBE_LAUNCHED();
}

HEAD_PROBE_API int head_probe_tk_relu_copy(const float* in, float* out, long long n, void* stream) {
  tk_relu_copy_kernel<<<tk_blocks(n), 256, 0, as_stream(stream)>>>(in, out, n);
  PROBE_LAUNCHED();
}

// out[b] (C x R) = in[b]^T (+ add[b]); add may be null
HEAD_PROBE_API int head_probe_tk_transpose(const float* in, int R, int C, const float* add, float* out, int B,
                                           void* stream) {
  tk_transpose(in, R, C, add, out, B, as_stream(stream));
  PROBE_LAUNCHED();
}

HEAD_PROBE_API int head_probe_tk_ln_wide_fwd(const float* x, const float* g, const float* b, float* y, float* mean,
                                             float* rstd, int B, void* stream) {
  tk_ln_wide_fwd_kernel<<<B, 256, 0, as_stream(stream)>>>(x, g, b, y, mean, rstd);
  PROBE_LAUNCHED();
}

// dy is masked in place by [y > 0]; dx is overwritten
HEAD_PROBE_API int head_probe_tk_ln_wide_bwd(const float* x, const float* g, const float* mean, const float* rstd,
                                             const float* y, float* dy, float* dx, int B, void* stream) {
  tk_ln_wide_bwd_kernel<<<B, 256, 0, as_stream(stream)>>>(x, g, mean, rstd, y, dy, dx);
  PROBE_LAUNCHED();
}

HEAD_PROBE_API int head_probe_tk_ln64_fwd(const float* x, const float* g, const float* b, float* y, float* mean,
                                          float* rstd, int rows, int relu, void* stream) {
  tk_ln64_fwd_kernel<<<(rows + 7) / 8, 256, 0, as_stream(stream)>>>(x, g, b, y, mean, rstd, rows, relu);
  PROBE_LAUNCHED();
}

// y may be null (no ReLU mask; dy untouched); accumulate: dx += instead of dx =
HEAD_PROBE_API int head_probe_tk_ln64_bwd(const float* x, const float* g, const float* mean, const float* rstd,
                                          const float* y, float* dy, float* dx, int rows, int accumulate,
                                          void* stream) {
  tk_ln64_bwd_kernel<<<(rows + 7) / 8, 256, 0, as_stream(stream)>>>(x, g, mean, rstd, y, dy, dx, rows, accumulate);
  PROBE_LAUNCHED();
}

// in place: x (rows x 2048) <- softmax(x)
HEAD_PROBE_API int head_probe_tk_softmax_fwd(float* x, int rows, void* stream) {
  tk_softmax_fwd_kernel<<<(rows + 7) / 8, 256, 0, as_stream(stream)>>>(x, rows);
  PROBE_LAUNCHED();
}

// in place: dP <- P (dP - sum_c P dP)
HEAD_PROBE_API int head_probe_tk_softmax_bwd(const float* P, float* dP, int rows, void* stream) {
  tk_softmax_bwd_kernel<<<(rows + 7) / 8, 256, 0, as_stream(stream)>>>(P, dP, rows);
  PROBE_LAUNCHED();
}

// tk_colsum's two launches with caller-provided partials (ceil(rows / 160) x N floats each); x / mean / rstd / out_g
// null for the plain sum
HEAD_PROBE_API int head_probe_tk_colsum(const float* dy, int ld, int rows, int N, float* out, const float* x,
                                        const float* mean, const float* rstd, float* out_g, float* part,
                                        float* part_g, void* stream) {
  TkWs w{};
  w.part = part;
  w.part_g = part_g;
  tk_colsum(dy, ld, rows, N, out, x, mean, rstd, out_g, w, as_stream(stream));
  PROBE_LAUNCHED();
}

HEAD_PROBE_API int head_probe_tk_colsum_chunks(int rows) { return (rows + kTkColRows - 1) / kTkColRows; }

// tk_conv: Y (B*lout x Cout) [+]= conv(act(X)); col (B*lout x Cin*taps) and split (kSplitFloats) are its scratch
HEAD_PROBE_API int head_probe_tk_conv(const float* X, int Cin, int lin, int lout, int taps, int dil, int relu,
                                      const float* W, const float* bias, int Cout, float* Y, int accumulate, int B,
                                      float* col, float* split, void* stream) {
  TK_MAP_CHECK(lin, lout);
  TkWs w{};
  w.col = col;
  w.dec.split = split;
  tk_conv(X, Cin, tk_seq_map(lin, lout), taps, dil, relu, W, bias, Cout, Y, accumulate != 0, B, w, as_stream(stream));
  PROBE_LAUNCHED();
}

// tk_conv_bwd: dX (B*lin x Cin) from dY (B*lout x Cout); dcol (B*lout x Cin*taps) and split are its scratch
HEAD_PROBE_API int head_probe_tk_conv_bwd(const float* dY, int Cout, const float* W, int Cin, int lin, int lout,
                                          int taps, int dil, const float* mask, const float* resid,
                                          const float* mask_out, float* dX, int B, float* dcol, float* split,
                                          void* stream) {
  TK_MAP_CHECK(lin, lout);
  TkWs w{};
  w.dcol = dcol;
  w.dec.split = split;
  tk_conv_bwd(dY, Cout, W, Cin, tk_seq_map(lin, lout), taps, dil, mask, resid, mask_out, dX, B, w, as_stream(stream));
  PROBE_LAUNCHED();
}
