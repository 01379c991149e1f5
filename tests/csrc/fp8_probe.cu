// Test-only probe library of the FP8 mode (tests/libthmr_fp8_probe.so): thin extern "C" wrappers around the launchers
// the fp8 engine dispatches but the product ABI does not expose (the block-scaled e4m3 GEMM with its epilogue options,
// including the e4m3 output, and the LayerNorm with e4m3 output).  Each wrapper launches exactly what the engine
// launches, so that tests/test_gpu_fp8.py can compare one stage at a time against the quantisation definition and
// fp64.  ctypes twin: tests/fp8_probe.py.  The product never loads this library.
#include "../../tokenhmr_b200/csrc/common.cuh"
#include "../../tokenhmr_b200/csrc/elementwise.cuh"
#include "../../tokenhmr_b200/csrc/gemm_host.cuh"

using namespace thmr;

#define FP8_PROBE_API extern "C" __attribute__((visibility("default")))

// The GemmDesc fields of an FP8 GEMM (gemm_make_plan_fp8): A, B e4m3 codes; the block scales and the e4m3 output as
// GemmDesc documents them.
struct fp8_probe_gemm_desc {
  const void* A; int lda; long long a_rows;
  const void* B; int ldb;
  int M, N, K;
  const float* bias;
  const float* resid; int ldr;
  int act;
  float* out32; int ld32;
  void* out16; int ld16;
  float alpha;
  int force_bn;
  const float* a_scale; int ld_as;
  const float* w_scale;
  void* out8; int ld8; float* out8_scale; int ld8s;
};

FP8_PROBE_API const char* fp8_probe_last_error(void) { return last_error_buf(); }

FP8_PROBE_API size_t fp8_probe_gemm_desc_size(void) { return sizeof(fp8_probe_gemm_desc); }

// Reads and clears this library's own copy of g_pipeline_timeout: 1 = a pipeline wait expired, 0 = none, -1 = CUDA error.
FP8_PROBE_API int fp8_probe_check_device_flags(void) {
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  unsigned int t = 0, zero = 0;
  if (cudaMemcpyFromSymbol(&t, g_pipeline_timeout, sizeof(t)) != cudaSuccess) return -1;
  if (cudaMemcpyToSymbol(g_pipeline_timeout, &zero, sizeof(zero)) != cudaSuccess) return -1;
  return t ? 1 : 0;
}

FP8_PROBE_API int fp8_probe_gemm(const fp8_probe_gemm_desc* g, void* stream) {
  THMR_CHECK(g && g->A && g->B, "fp8_probe_gemm: null argument");
  GemmDesc d;
  d.fp8 = 1;
  d.A = static_cast<const __half*>(g->A); d.lda = g->lda; d.a_rows = g->a_rows;
  d.B = static_cast<const __half*>(g->B); d.ldb = g->ldb;
  d.M = g->M; d.N = g->N; d.K = g->K;
  d.bias = g->bias; d.resid = g->resid; d.ldr = g->ldr;
  d.act = g->act;
  d.out32 = g->out32; d.ld32 = g->ld32; d.out16 = static_cast<__half*>(g->out16); d.ld16 = g->ld16;
  d.alpha = g->alpha;
  d.force_bn = g->force_bn;
  d.a_scale = g->a_scale; d.ld_as = g->ld_as; d.w_scale = g->w_scale;
  d.out8 = static_cast<uint8_t*>(g->out8); d.ld8 = g->ld8; d.out8_scale = g->out8_scale; d.ld8s = g->ld8s;
  GemmPlan plan;
  THMR_TRY(gemm_make_plan(d, &plan));
  return gemm_launch(plan, static_cast<cudaStream_t>(stream));
}

FP8_PROBE_API int fp8_probe_layernorm_e4m3(const float* x, const float* gamma, const float* beta, void* y8, float* ys,
                                           int lds, float* y32, int R, int C, float eps, void* stream) {
  return layernorm_e4m3_launch(x, gamma, beta, static_cast<uint8_t*>(y8), ys, lds, y32, R, C, eps,
                               static_cast<cudaStream_t>(stream));
}
