// Test-only GEMM plan probe (tests/libthmr_gemm_probe.so): the fp16 GEMM of tokenhmr_b200/csrc/gemm_host.cuh with a
// forced epilogue kind (GemmDesc::force_epi), the plan gemm_make_plan makes (block_n, epilogue kind, grid), and the
// per-tile timeline kernels (gemm_f16_tn_kernel<..., TIMELINE = true>), which only this library instantiates.  Used by
// tests/test_gpu_gemm_epilogue_kinds.py and scripts/gemm_anatomy.py; ctypes twin: tests/gemm_probe.py.  The product
// never loads this library.
#include <stdint.h>

#include "../../tokenhmr_b200/csrc/common.cuh"
#include "../../tokenhmr_b200/csrc/gemm_host.cuh"

using namespace thmr;

#define GEMM_PROBE_API extern "C" __attribute__((visibility("default")))

// The GemmDesc fields of a plain fp16 GEMM; ctypes twin in tests/gemm_probe.py.
struct gemm_probe_desc {
  const void* A; int lda; long long a_rows;
  const void* B; int ldb;
  int M, N, K;
  const float* bias;
  const float* resid; int ldr; int resid_mod;
  int act; int act32;
  float* out32; int ld32;
  void* out16; int ld16;
  int seq_pitch, seq_lo, seq_hi;
  float alpha;
  int force_bn;
  int force_epi;   // GemmDesc::force_epi: 0 = the plan's epilogue kind, 1 + kEpi* = that kind
};

GEMM_PROBE_API const char* gemm_probe_last_error(void) { return last_error_buf(); }

GEMM_PROBE_API size_t gemm_probe_desc_size(void) { return sizeof(gemm_probe_desc); }

// Reads and clears this library's own pipeline-timeout flag: 1 if a wait timed out, 0 if not, -1 on a CUDA error.
GEMM_PROBE_API int gemm_probe_check_device_flags(void) {
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  unsigned int t = 0, zero = 0;
  if (cudaMemcpyFromSymbol(&t, g_pipeline_timeout, sizeof(t)) != cudaSuccess) return -1;
  if (cudaMemcpyToSymbol(g_pipeline_timeout, &zero, sizeof(zero)) != cudaSuccess) return -1;
  return t ? 1 : 0;
}

static int make_plan(const gemm_probe_desc* g, GemmPlan* plan) {
  THMR_CHECK(g && g->A && g->B, "gemm_probe: null argument");
  GemmDesc d;
  d.A = static_cast<const __half*>(g->A); d.lda = g->lda; d.a_rows = g->a_rows;
  d.B = static_cast<const __half*>(g->B); d.ldb = g->ldb;
  d.M = g->M; d.N = g->N; d.K = g->K;
  d.bias = g->bias; d.resid = g->resid; d.ldr = g->ldr; d.resid_mod = g->resid_mod;
  d.act = g->act; d.act32 = g->act32;
  d.out32 = g->out32; d.ld32 = g->ld32; d.out16 = static_cast<__half*>(g->out16); d.ld16 = g->ld16;
  d.seq_pitch = g->seq_pitch; d.seq_lo = g->seq_lo; d.seq_hi = g->seq_hi;
  d.alpha = g->alpha;
  d.force_bn = g->force_bn;
  d.force_epi = g->force_epi;
  return gemm_make_plan(d, plan);
}

GEMM_PROBE_API int gemm_probe_run(const gemm_probe_desc* g, void* stream) {
  GemmPlan plan;
  THMR_TRY(make_plan(g, &plan));
  return gemm_launch(plan, static_cast<cudaStream_t>(stream));
}

// The plan gemm_make_plan makes for *g, without launching: block_n, epilogue kind (kEpi*) and grid.
GEMM_PROBE_API int gemm_probe_plan(const gemm_probe_desc* g, int* bn, int* epi, int* grid) {
  THMR_CHECK(bn && epi && grid, "gemm_probe_plan: null output");
  GemmPlan plan;
  THMR_TRY(make_plan(g, &plan));
  *bn = plan.bn;
  *epi = plan.epi;
  *grid = plan.grid;
  return THMR_OK;
}

// gemm_probe_run with the per-tile timeline (GemmParams::timeline): timeline u64 [grid][slots][2][4] and sm int32
// [grid], caller-initialised; fp16 block_n 128 / 256 plans only.
GEMM_PROBE_API int gemm_probe_timeline(const gemm_probe_desc* g, unsigned long long* timeline, int slots, int* sm,
                                       void* stream) {
  THMR_CHECK(timeline && sm && slots > 0, "gemm_probe_timeline: null buffer");
  GemmPlan plan;
  THMR_TRY(make_plan(g, &plan));
  plan.p.timeline = timeline;
  plan.p.timeline_slots = slots;
  plan.p.timeline_sm = sm;
  return gemm_launch<true>(plan, static_cast<cudaStream_t>(stream));
}
