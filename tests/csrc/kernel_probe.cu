// Test-only probe library (tests/libthmr_probe.so): thin extern "C" wrappers around the launchers of
// tokenhmr_b200/csrc that the engine dispatches but the product ABI does not expose (GEMM epilogue options, the
// split-precision operand builder, the strict-mode fp32 kernels, the head and tokenizer glue kernels, every LayerNorm
// dispatch variant, the SMPL stage's kernels, the FP8 mode's block-scaled e4m3 GEMM and e4m3 LayerNorm, and the fused
// SMPLify-inverse's loss and Adam kernels), plus the OpenPose overlay's span generator run on the host.  Each wrapper
// launches exactly what the engine launches, with the engine's grid shapes, so that tests/test_gpu_kernels.py,
// tests/test_gpu_strict_kernels.py, tests/test_gpu_smpl_kernels.py, tests/test_gpu_fp8.py and
// tests/test_gpu_smplify_fused.py can compare one stage at a time against fp64, and
// tests/test_mesh_renderer_oracle.py can hold the span generator against live cv2 without a GPU.
// ctypes twin: tests/probe.py.  The product never loads this library.
#include <stdint.h>

#include "../../tokenhmr_b200/csrc/attention_mma.cuh"
#include "../../tokenhmr_b200/csrc/common.cuh"
#include "../../tokenhmr_b200/csrc/elementwise.cuh"
#include "../../tokenhmr_b200/csrc/engine.cuh"
#include "../../tokenhmr_b200/csrc/gemm_host.cuh"
#include "../../tokenhmr_b200/csrc/head_kernels.cuh"
#include "../../tokenhmr_b200/csrc/keypoints.cuh"
#include "../../tokenhmr_b200/csrc/smpl_lbs.cuh"
#include "../../tokenhmr_b200/csrc/smplify.cuh"
#include "../../tokenhmr_b200/csrc/strict.cuh"

using namespace thmr;

#define PROBE_API extern "C" __attribute__((visibility("default")))

// Mirrors the GemmDesc fields the engine sets for a plain (non-arg-min) GEMM, fp16 or, with fp8 set, block-scaled e4m3
// (A, B e4m3 codes; the block scales and the e4m3 output as GemmDesc documents them); ctypes twin in tests/probe.py.
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
  int fp8;
  const float* a_scale; int ld_as;
  const float* w_scale;
  void* out8; int ld8; float* out8_scale; int ld8s;
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
  d.fp8 = g->fp8;
  d.a_scale = g->a_scale; d.ld_as = g->ld_as; d.w_scale = g->w_scale;
  d.out8 = static_cast<uint8_t*>(g->out8); d.ld8 = g->ld8; d.out8_scale = g->out8_scale; d.ld8s = g->ld8s;
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

PROBE_API int probe_layernorm_e4m3(const float* x, const float* gamma, const float* beta, void* y8, float* ys, int lds,
                                   float* y32, int R, int C, float eps, void* stream) {
  return layernorm_e4m3_launch(x, gamma, beta, static_cast<uint8_t*>(y8), ys, lds, y32, R, C, eps, as_stream(stream));
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

// ---- SMPL stage (smpl_lbs.cuh; launched by thmr_smpl_create and smpl_run in engine.cuh) --------------------------
// thmr_smpl_create: J_template / J_shapedirs, one block per output scalar
PROBE_API int probe_smpl_jreg(const float* Jreg, const float* v_template, const float* shapedirs, float* J_template,
                              float* J_shapedirs, int V, int nb, void* stream) {
  smpl_jreg_kernel<<<kSmplJ * 3 * (nb + 1), 256, 0, as_stream(stream)>>>(Jreg, v_template, shapedirs, J_template,
                                                                         J_shapedirs, V, nb);
  PROBE_LAUNCHED();
}

// thmr_smpl_create: zero the basis including its pad rows (3V rounded up to 4), then pack [3V, 3*224]
PROBE_API int probe_smpl_pack_posedirs(const float* posedirs, const float* shapedirs, const float* v_template, int nb,
                                       void* out, int V, void* stream) {
  const size_t rows_pad = (static_cast<size_t>(3) * V + 3) / 4 * 4;
  THMR_CUDA(cudaMemsetAsync(out, 0, rows_pad * 3 * kSmplPFPad * sizeof(__half), as_stream(stream)));
  const long n = static_cast<long>(3) * V * kSmplPFPad;
  smpl_pack_posedirs_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, as_stream(stream)>>>(
      posedirs, shapedirs, v_template, nb, static_cast<__half*>(out), 3 * V);
  PROBE_LAUNCHED();
}

PROBE_API int probe_smpl_pose(const float* pose, int pose2rot, const float* betas, const float* J_template,
                              const float* J_shapedirs, int nb, const int* parents_dev, float* A, float* Jposed,
                              void* pf16, int B, void* stream) {
  smpl_pose_kernel<<<B, 32, 0, as_stream(stream)>>>(pose, pose2rot, betas, J_template, J_shapedirs, nb, parents_dev, A,
                                                    Jposed, static_cast<__half*>(pf16), B);
  PROBE_LAUNCHED();
}

// The blend GEMM of one chunk of n poses starting at pose p0, planned by smpl_blend_plan as smpl_run does:
// pf16 [>= p0 + n, 3*224], posedirsT [off_pitch, 3*224], offsets [n, off_pitch] with off_pitch = 3V rounded up to 4.
PROBE_API int probe_smpl_blend(const void* pf16, const void* posedirsT, int V, int p0, int n, float* offsets,
                               void* stream) {
  SmplModel m;
  m.V = V;
  m.posedirsT = static_cast<__half*>(const_cast<void*>(posedirsT));
  SmplWs ws{};
  ws.pf16 = static_cast<__half*>(const_cast<void*>(pf16));
  ws.offsets = offsets;
  ws.off_pitch = (3L * V + 3) / 4 * 4;   // smpl_carve
  GemmPlan plan;
  THMR_TRY(smpl_blend_plan(m, ws, p0, n, &plan));
  return gemm_launch(plan, as_stream(stream));
}

// smpl_run's skinning launch; threads (256 | 128) and ell_reg (4 | 8) pick the instantiation
PROBE_API int probe_smpl_skin(int threads, int ell_reg, const int* w_idx, const float* w_val, int ell, const float* A,
                              const float* vposed, long off_pitch, float* verts, long vert_pitch, int V, int B,
                              void* stream) {
  THMR_CHECK((threads == 256 || threads == 128) && (ell_reg == 4 || ell_reg == 8), "probe_smpl_skin: threads %d ell_reg %d",
             threads, ell_reg);
  const dim3 grid((V + threads - 1) / threads, (B + kSkinPoses - 1) / kSkinPoses);
  cudaStream_t st = as_stream(stream);
  if (threads == 256 && ell_reg == 4)
    smpl_skin_kernel<256, 4><<<grid, 256, 0, st>>>(w_idx, w_val, ell, A, vposed, off_pitch, verts, vert_pitch, V, B);
  else if (threads == 256)
    smpl_skin_kernel<256, 8><<<grid, 256, 0, st>>>(w_idx, w_val, ell, A, vposed, off_pitch, verts, vert_pitch, V, B);
  else if (ell_reg == 4)
    smpl_skin_kernel<128, 4><<<grid, 128, 0, st>>>(w_idx, w_val, ell, A, vposed, off_pitch, verts, vert_pitch, V, B);
  else
    smpl_skin_kernel<128, 8><<<grid, 128, 0, st>>>(w_idx, w_val, ell, A, vposed, off_pitch, verts, vert_pitch, V, B);
  PROBE_LAUNCHED();
}

PROBE_API int probe_smpl_joints(const float* Jposed, const float* verts, long vert_pitch, const int* joint_map,
                                const int* extra_vid, const int* jx_ptr, const int* jx_idx, const float* jx_val,
                                int n_extra, float* joints, const float* pred_cam, float focal, float image_size,
                                float* cam_t, float* focal_out, float* kp2d, int B, void* stream) {
  smpl_joints_kernel<<<B, 64, 0, as_stream(stream)>>>(Jposed, verts, vert_pitch, joint_map, extra_vid, jx_ptr, jx_idx,
                                                      jx_val, n_extra, joints, pred_cam, focal, image_size, cam_t,
                                                      focal_out, kp2d);
  PROBE_LAUNCHED();
}

// ---- fused SMPLify-inverse (smplify.cuh; launched by thmr_smplify_inv) ----------------------------------------------
// smplify_loss_kernel as an iteration launches it (grad_joints / grad_cam non-null) or as the final forward does
// (both null, pj2d non-null); no done flag
PROBE_API int probe_smplify_loss(const float* joints, const float* cam, const float* focal, const float* kp2d,
                                 const float* kp3d, int J, int B, float* grad_joints, float* grad_cam, float* part,
                                 float* pj2d, void* stream) {
  return smplify_loss_launch(joints, cam, focal, kp2d, kp3d, J, B, grad_joints, grad_cam, part, pj2d, nullptr,
                             as_stream(stream));
}

// smplify_adam_kernel for Adam step `step` (1-based) at learning rate lr over n flat elements; no done flag
PROBE_API int probe_smplify_adam(float* p, float* m, float* v, const float* g, long n, int step, double lr,
                                 void* stream) {
  return smplify_adam_launch(p, m, v, g, n, step, lr, nullptr, as_stream(stream));
}

// ---- OpenPose overlay span generator (keypoints.cuh), run on the host ----------------------------------------------
namespace {
struct MaskEmit {
  uint8_t* mask;
  int W;
  void operator()(int y, int x0, int x1) const {
    for (int x = x0; x <= x1; ++x) mask[static_cast<long long>(y) * W + x] = 1;
  }
};
}  // namespace

// kind 0: cv2.line(p0, p1, thickness 2);  kind 1 / 2: cv2.circle(p0, radius 1, thickness kind).  Sets mask[y * W + x]
// (uint8 [H, W], caller-zeroed) to 1 on every pixel painted.  Returns 0, or -1 for a bad kind or size.
PROBE_API int probe_pose_draw(int kind, long long x0, long long y0, long long x1, long long y1, int W, int H,
                              uint8_t* mask) {
  if (!mask || W < 1 || H < 1) return -1;
  MaskEmit emit{mask, W};
  if (kind == 0)
    cv_line(W, H, x0, y0, x1, y1, emit);
  else if (kind == 1 || kind == 2)
    cv_circle(W, H, x0, y0, kind, emit);
  else
    return -1;
  return 0;
}
