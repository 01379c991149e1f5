// Test-only probe of the regression head's training kernels (tests/libthmr_head_train_probe.so): thin extern "C"
// wrappers around what rh_forward / rh_backward in tokenhmr_b200/csrc/head_train.cuh launch, each with the engine's
// grid, block and shared-memory sizes: hl_gemm through its own planner, the cross-attention chunk and combine kernels,
// LayerNorm forward and backward, the column sums, token 0 and the read-out backward.  Used by
// tests/test_gpu_head_train_kernels.py; ctypes twin: tests/head_train_probe.py.  The product never loads this library.
#include <stdint.h>

#include "../../tokenhmr_b200/csrc/common.cuh"
#include "../../tokenhmr_b200/csrc/head_train.cuh"

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
