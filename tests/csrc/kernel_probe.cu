// Test-only probe library (tests/libthmr_probe.so): thin extern "C" wrappers around the launchers of
// tokenhmr_b200/csrc that the engine dispatches but the product ABI does not expose (GEMM epilogue options, the
// split-precision operand builder, the strict-mode fp32 kernels, the head and tokenizer glue kernels, every LayerNorm
// dispatch variant).  Each wrapper launches exactly what the engine launches, with the engine's grid shapes, so that
// tests/test_gpu_kernels.py and tests/test_gpu_strict_kernels.py can compare one stage at a time against fp64.
// The product never loads this library.
#include "../../tokenhmr_b200/csrc/attention_mma.cuh"
#include "../../tokenhmr_b200/csrc/common.cuh"
#include "../../tokenhmr_b200/csrc/elementwise.cuh"
#include "../../tokenhmr_b200/csrc/gemm_host.cuh"
#include "../../tokenhmr_b200/csrc/head_kernels.cuh"
#include "../../tokenhmr_b200/csrc/strict.cuh"

using namespace thmr;

#define PROBE_API extern "C" __attribute__((visibility("default")))

// Mirrors the GemmDesc fields the engine sets for a plain (non-arg-min) GEMM; ctypes twin in tests/probe.py.
struct probe_gemm_desc {
  const void* A; int lda; long long a_rows;
  const void* B; int ldb;
  int M, N, K;
  const float* bias;
  const float* resid; int ldr; int resid_mod;
  int act; int act32;
  float* out32; int ld32;
  void* out16; int ld16;
  int taps, cin, tap_row0, tap_stride;
  int seq_pitch, seq_lo, seq_hi;
  float alpha;
  int force_bn;
};

static cudaStream_t as_stream(void* s) { return static_cast<cudaStream_t>(s); }

#define PROBE_LAUNCHED()        \
  do {                          \
    THMR_CUDA(cudaGetLastError()); \
    return THMR_OK;             \
  } while (0)

PROBE_API const char* probe_last_error(void) { return last_error_buf(); }

PROBE_API size_t probe_gemm_desc_size(void) { return sizeof(probe_gemm_desc); }

// Reads and clears this library's own device status words (its copies of g_pipeline_timeout and g_strict_overflow).
// Returns bit 0 = pipeline timeout, bit 1 = split-precision overflow, or -1 on a CUDA error.
PROBE_API int probe_check_device_flags(void) {
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  unsigned int t = 0, o = 0, zero = 0;
  if (cudaMemcpyFromSymbol(&t, g_pipeline_timeout, sizeof(t)) != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(&o, g_strict_overflow, sizeof(o)) != cudaSuccess) return -1;
  if (cudaMemcpyToSymbol(g_pipeline_timeout, &zero, sizeof(zero)) != cudaSuccess) return -1;
  if (cudaMemcpyToSymbol(g_strict_overflow, &zero, sizeof(zero)) != cudaSuccess) return -1;
  return (t ? 1 : 0) | (o ? 2 : 0);
}

PROBE_API int probe_gemm(const probe_gemm_desc* g, void* stream) {
  THMR_CHECK(g && g->A && g->B, "probe_gemm: null argument");
  GemmDesc d;
  d.A = static_cast<const __half*>(g->A); d.lda = g->lda; d.a_rows = g->a_rows;
  d.B = static_cast<const __half*>(g->B); d.ldb = g->ldb;
  d.M = g->M; d.N = g->N; d.K = g->K;
  d.bias = g->bias; d.resid = g->resid; d.ldr = g->ldr; d.resid_mod = g->resid_mod;
  d.act = g->act; d.act32 = g->act32;
  d.out32 = g->out32; d.ld32 = g->ld32; d.out16 = static_cast<__half*>(g->out16); d.ld16 = g->ld16;
  d.taps = g->taps; d.cin = g->cin; d.tap_row0 = g->tap_row0; d.tap_stride = g->tap_stride;
  d.seq_pitch = g->seq_pitch; d.seq_lo = g->seq_lo; d.seq_hi = g->seq_hi;
  d.alpha = g->alpha;
  d.force_bn = g->force_bn;
  GemmPlan plan;
  THMR_TRY(gemm_make_plan(d, &plan));
  return gemm_launch(plan, as_stream(stream));
}

PROBE_API int probe_split_rows(const float* src, long lds, void* dst, long R, int C, int act, int T, int pitch, int lo,
                               void* stream) {
  return split_rows_launch(src, lds, static_cast<__half*>(dst), R, C, act, T, pitch, lo, as_stream(stream));
}

PROBE_API int probe_layernorm(const float* x, const float* gamma, const float* beta, void* y16, int ld16, float* y32,
                              int R, int C, float eps, int relu, int out_t, void* stream) {
  return layernorm_launch(x, gamma, beta, static_cast<__half*>(y16), ld16, y32, R, C, eps, relu, out_t,
                          as_stream(stream));
}

PROBE_API int probe_softmax_rows(const float* logits, float* p32, void* p16, int R, int C, int T, int pitch, int lo,
                                 void* stream) {
  return softmax_rows_launch(logits, p32, static_cast<__half*>(p16), R, C, T, pitch, lo, as_stream(stream));
}

PROBE_API int probe_vit_attention(const void* qkv, int B, int heads, void* out, void* stream) {
  AttnPlan plan;
  THMR_TRY(attention_make_plan(static_cast<const __half*>(qkv), 3 * heads * kAttHeadDim, B, heads,
                               static_cast<__half*>(out), heads * kAttHeadDim, nullptr, &plan));
  return attention_dispatch(plan, as_stream(stream));
}

PROBE_API int probe_attention_f32(const float* qkv, int ld, int B, int H, float* out, int ldo, float scale,
                                  void* stream) {
  return attention_f32_launch(qkv, ld, B, H, out, ldo, scale, as_stream(stream));
}

PROBE_API int probe_dec_cross_attn(const float* q, const void* kv, int ld, int koff, int voff, float scale, void* out,
                                   int B, int heads, void* stream) {
  dec_cross_attn_kernel<192><<<B * heads, 192, 0, as_stream(stream)>>>(q, static_cast<const __half*>(kv), ld, koff, voff,
                                                                       scale, static_cast<__half*>(out), heads);
  PROBE_LAUNCHED();
}

PROBE_API int probe_dec_cross_attn_f32(const float* q, const float* kv, int ld, int koff, int voff, float scale,
                                       float* out, int B, int heads, void* stream) {
  dec_cross_attn_f32_kernel<192><<<B * heads, 192, 0, as_stream(stream)>>>(q, kv, ld, koff, voff, scale, out, heads);
  PROBE_LAUNCHED();
}

PROBE_API int probe_im2col_patch(const float* img, void* out, int B, int S, int x0, int Wc, int P, int pad, int gh,
                                 int gw, void* stream) {
  const long total = static_cast<long>(B) * gh * gw * 3 * P;
  im2col_patch_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, as_stream(stream)>>>(
      img, static_cast<__half*>(out), B, S, x0, Wc, P, pad, gh, gw, nullptr);
  PROBE_LAUNCHED();
}

PROBE_API int probe_im2col_patch_f32(const float* img, float* out, int B, int S, int x0, int Wc, int P, int pad, int gh,
                                     int gw, void* stream) {
  const long total = static_cast<long>(B) * gh * gw * 3 * P;
  im2col_patch_f32_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, as_stream(stream)>>>(
      img, out, B, S, x0, Wc, P, pad, gh, gw);
  PROBE_LAUNCHED();
}

PROBE_API int probe_relu_inplace(float* x, long n4, void* stream) {
  relu_inplace_kernel<<<static_cast<unsigned>((n4 + 255) / 256), 256, 0, as_stream(stream)>>>(x, n4);
  PROBE_LAUNCHED();
}

// c8 = row width in 16-byte units: C / 8 for fp16 rows, C / 4 for the fp32 rows of strict mode and the tokenizer encoder
PROBE_API int probe_upsample_rows(const void* src, void* dst, int B, int Lin, int Lout, int pad, int c8, void* stream) {
  const long n = static_cast<long>(B) * (Lout + 2 * pad) * c8;
  upsample_rows_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, as_stream(stream)>>>(
      static_cast<const __half*>(src), static_cast<__half*>(dst), B, Lin, Lout, pad, c8);
  PROBE_LAUNCHED();
}

PROBE_API int probe_mixer_add(const float* x, const float* yT, const float* z, float* out, int B, int T, int H,
                              void* stream) {
  const long n = static_cast<long>(B) * T * H;
  mixer_add_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, as_stream(stream)>>>(x, yT, z, out, B, T, H);
  PROBE_LAUNCHED();
}

PROBE_API int probe_cast_f16(const float* in, void* out, long n4, void* stream) {
  cast_f16_kernel<<<static_cast<unsigned>((n4 + 255) / 256), 256, 0, as_stream(stream)>>>(in, static_cast<__half*>(out),
                                                                                        n4);
  PROBE_LAUNCHED();
}

PROBE_API int probe_head_assemble(const float* readout, int ld_r, const float* bpose, int ld_b, int pitch, int lo,
                                  const float* init_pose, const float* init_betas, const float* init_cam, float* rotmats,
                                  float* betas, float* cam, float* pose6d, int B, int nb, void* stream) {
  head_assemble_kernel<<<(B * 24 + 127) / 128, 128, 0, as_stream(stream)>>>(readout, ld_r, bpose, ld_b, pitch, lo,
                                                                           init_pose, init_betas, init_cam, rotmats,
                                                                           betas, cam, pose6d, B, nb);
  PROBE_LAUNCHED();
}
