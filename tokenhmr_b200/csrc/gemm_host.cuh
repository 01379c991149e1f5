// Host side of the wgmma GEMM: plan construction (TMA descriptors, tile choice) and launch.
#pragma once
#include "common.cuh"

#include "gemm_wgmma.cuh"

namespace thmr {

struct GemmPlan {
  CUtensorMap tmA, tmB;
  // TMA-stored kinds, SWIZZLE_128B (zero for the other plans): out16, box 64 x 64 (fp16 kinds), or out32 = the
  // residual, box 64 rows x 32 fp32 (residual kind: its loads and its stores)
  CUtensorMap tmC;
  GemmParams p;
  int bn;
  int grid;
  int cluster;   // 2: CTA pairs sharing the B tile (gemm_wgmma.cuh)
  int fp8;       // e4m3 operands (gemm_make_plan_fp8)
  int epi;       // epilogue kind (kEpi*, gemm_wgmma.cuh)
};

struct GemmDesc {
  const __half* A; int lda; long long a_rows;  // a_rows: rows addressable through the A descriptor
  const __half* B; int ldb;
  int M, N, K;
  const float* bias = nullptr;
  const float* resid = nullptr; int ldr = 0; int resid_mod = 0;
  int act = kActNone; int act32 = 0;
  float* out32 = nullptr; int ld32 = 0;
  __half* out16 = nullptr; int ld16 = 0;
  // implicit conv1d (taps > 1): K = taps * cin, tap t reads A rows (m + tap_row0 + t*tap_stride), cols [0,cin)
  int taps = 1; int cin = 0; int tap_row0 = 0; int tap_stride = 0;
  int seq_pitch = 0, seq_lo = 0, seq_hi = 0;
  float alpha = 1.0f;
  long long* argmin_out = nullptr; const float* row_sq = nullptr; const float* col_sq = nullptr;
  // screened arg-min (GemmParams): pass 1 queues uncertain rows, the exact pass takes its row count from the device
  int* screen_rows = nullptr; int* screen_count = nullptr; const float* screen_cmax2 = nullptr;
  float screen_rel = 0.f, screen_abs = 0.f; int screen_row0 = 0;
  const int* row_map = nullptr; const int* m_dev = nullptr; int m_dev_off = 0;
  int force_bn = 0;   // 32 / 64 / 128 / 256, or 512 = a CTA pair (2-CTA cluster) on a 256 x 256 tile
  int force_epi = 0;  // 0: the plan picks the epilogue kind; 1 + kEpi*: that kind (a specialised one only where it fits)
  unsigned long long* stamp = nullptr;   // in-graph start stamp slot (nullable)
  // FP8 (GemmParams): A and B point to e4m3 bytes (lda / ldb in elements = bytes), K a multiple of 128; block_n 64 or
  // 128, 128 with out8.  a_scale [K / 128][ld_as] must hold the tile-padded rows (ld_as >= M rounded up to 128).
  int fp8 = 0;
  const float* a_scale = nullptr; int ld_as = 0;
  const float* w_scale = nullptr;
  uint8_t* out8 = nullptr; int ld8 = 0; float* out8_scale = nullptr; int ld8s = 0;
};

// Tile width: wide tiles move fewer operand bytes per MAC (every k-block moves (128 + BN) * 128 bytes for
// 128 * BN * 64 MACs), so they win unless they leave SMs idle or their epilogue dominates.  Cost model per tile in
// cycles on an H100 SM: per k-block max(MMA at 2048 fp16 MAC/clk, operand feed at ~32 B/clk from L2) plus a fixed
// overhead, plus the epilogue.  The epilogue terms are fitted to the ViT GEMMs (M = 12288) on an H100 80GB HBM3 (700 W
// power limit; scripts/gemm_anatomy.py, per-tile timeline), so that the model picks the measured-faster width at all
// five of them.  Of the specialised epilogue kinds (block_n 128 / 256 only), the TMA-stored fp16 ones hold the
// consumers 0.8-2.3 us per 128 columns (~2500 cycles), the fp32 residual one ~5 us at block_n 256 (~9000 cycles: its
// reductions of every SM drain through L2 at once) and ~3 us at 128; 256 wins at all five either way.  The general epilogue costs ~30 us per 128 x 256 tile (eight
// 32-column chunks) against ~7 us per 128 x 128 tile; the narrower tiles are scaled from 128.  The row arg-min
// epilogue (VQ) is not staged and is not charged.
inline int pick_bn(int M, int N, int K, bool staged_epilogue, int epi_kind, int force) {
  if (force) return force;
  const int sms = num_sms();
  const int tm = (M + kGemmBM - 1) / kGemmBM;
  const int num_kb = (K + kGemmBK - 1) / kGemmBK;
  int best = 256;
  double best_cost = -1;
  const int cands[4] = {256, 128, 64, 32};
  for (int i = 0; i < 4; ++i) {
    const int bn = cands[i];
    const long tiles = static_cast<long>(tm) * ((N + bn - 1) / bn);
    const long waves = (tiles + sms - 1) / sms;
    const double mma = 4.0 * bn;
    const double feed = (128.0 + bn) * 128.0 / 32.0;
    const double epilogue = !staged_epilogue                                 ? 0.0
                            : bn >= 128 && gemm_epi_tma_store(epi_kind)       ? 2500.0 * bn / 128
                            : bn >= 128 && epi_kind == kEpiBiasResidF32       ? 9000.0 * bn / 128
                            : bn == 256                                       ? 55000.0
                                                                              : 7000.0 * bn / 128;
    const double cost = waves * (num_kb * ((mma > feed ? mma : feed) + 40.0) + epilogue);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = bn; }
  }
  return best;
}

// FP8 tile width, the same model at FP8 rates: a 128-element k-block moves the bytes of an fp16 64-element one and
// takes the same MMA time (4096 e4m3 MAC/clk), so per K there are half the k-blocks; each k-block adds the promotion
// (BN / 2 FMAs per consumer thread, ~BN cycles per SM).  Two accumulator sets leave 64 and 128 only.
inline int pick_bn_fp8(int M, int N, int K) {
  const int sms = num_sms();
  const int tm = (M + kGemmBM - 1) / kGemmBM;
  const int num_kb = (K + 127) / 128;
  int best = 128;
  double best_cost = -1;
  const int cands[2] = {128, 64};
  for (int i = 0; i < 2; ++i) {
    const int bn = cands[i];
    const long tiles = static_cast<long>(tm) * ((N + bn - 1) / bn);
    const long waves = (tiles + sms - 1) / sms;
    const double mma = 4.0 * bn;
    const double feed = (128.0 + bn) * 128.0 / 32.0;
    const double cost = waves * (num_kb * ((mma > feed ? mma : feed) + bn + 40.0) + 7000.0 * bn / 128);
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = bn; }
  }
  return best;
}

// Epilogue kind of a plain fp16 GEMM: a specialised kind where the descriptor asks for exactly its operations and every
// base and pitch it touches allows 16-byte row vectors (the TMA kinds need that of their tensor maps), else kEpiGeneral.
// The residual kind also needs the residual to alias out32 (resid == out32, ldr == ld32), as at every call site of the
// engine: one tensor map then serves its loads and its stores.  Only the 128- and 256-wide tiles, where the ViT's GEMMs
// run, have the specialised kernels.
inline int gemm_pick_epi(const GemmDesc& d, int bn, int cluster) {
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if ((bn != 128 && bn != 256) || cluster != 1 || d.argmin_out || d.resid_mod || d.seq_pitch || d.act32 || !al16(d.bias))
    return kEpiGeneral;
  if (d.out16 && !d.out32 && !d.resid && d.ld16 % 8 == 0 && al16(d.out16)) {
    if (d.act == kActNone) return d.bias ? kEpiBiasF16 : kEpiF16;
    if (d.act == kActGelu && d.bias) return kEpiBiasGeluF16;
  }
  if (d.out32 && !d.out16 && d.resid == d.out32 && d.ldr == d.ld32 && d.bias && d.act == kActNone &&
      d.ld32 % 4 == 0 && al16(d.out32))
    return kEpiBiasResidF32;
  return kEpiGeneral;
}

inline int make_tmap_2d_e4m3(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                             uint32_t box_rows, uint32_t box_cols) {
  return make_tmap_2d(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, base, rows, cols, ld, box_rows, box_cols,
                      CU_TENSOR_MAP_SWIZZLE_128B);
}

inline int gemm_make_plan_fp8(const GemmDesc& d, GemmPlan* plan) {
  THMR_CHECK(d.M > 0 && d.N > 0 && d.K > 0 && d.K % 128 == 0, "gemm fp8: bad shape %dx%dx%d (K %% 128 != 0)", d.M, d.N,
             d.K);
  THMR_CHECK(d.out32 || d.out16 || d.out8, "gemm fp8: no output");
  THMR_CHECK(d.a_scale && d.w_scale, "gemm fp8: missing block scales");
  THMR_CHECK(!d.argmin_out && d.taps == 1 && !d.m_dev && !d.row_map, "gemm fp8: plain GEMMs only");
  const long m_pad = (d.M + kGemmBM - 1) / kGemmBM * kGemmBM;
  THMR_CHECK(d.ld_as >= m_pad && d.ld_as % 4 == 0 && (reinterpret_cast<uintptr_t>(d.a_scale) & 15) == 0,
             "gemm fp8: activation scales need a 16-byte aligned [K/128][>= %ld] layout (ld_as %d)", m_pad, d.ld_as);
  int bn = d.force_bn ? d.force_bn : d.out8 ? 128 : pick_bn_fp8(d.M, d.N, d.K);
  THMR_CHECK(bn == 64 || bn == 128, "gemm fp8: block_n %d (64 or 128)", bn);
  THMR_CHECK(!d.out8 || (bn == 128 && d.out8_scale && d.ld8s >= d.M && !d.resid && !d.act32 && !d.seq_pitch),
             "gemm fp8: e4m3 output needs block_n 128, its scale array and no residual / mask / act32");
  GemmParams& p = plan->p;
  memset(&p, 0, sizeof(p));
  p.M = d.M; p.N = d.N; p.K = d.K;
  p.out32 = d.out32; p.ld32 = d.ld32; p.out16 = d.out16; p.ld16 = d.ld16;
  p.bias = d.bias; p.resid = d.resid; p.ldr = d.ldr; p.resid_mod = d.resid_mod; p.act = d.act; p.act32 = d.act32;
  p.seq_pitch = d.seq_pitch; p.seq_lo = d.seq_lo; p.seq_hi = d.seq_hi;
  p.alpha = d.alpha;
  p.stamp = d.stamp;
  p.kblocks_per_tap = d.K / 128;
  p.a_scale = d.a_scale; p.ld_as = d.ld_as; p.w_scale = d.w_scale;
  p.out8 = d.out8; p.ld8 = d.ld8; p.out8_scale = d.out8_scale; p.ld8s = d.ld8s;
  THMR_TRY(make_tmap_2d_e4m3(&plan->tmA, d.A, d.a_rows, d.K, d.lda, kGemmBM, 128));
  THMR_TRY(make_tmap_2d_e4m3(&plan->tmB, d.B, d.N, d.K, d.ldb, bn, 128));
  memset(&plan->tmC, 0, sizeof(plan->tmC));
  THMR_CHECK(d.force_epi == 0 || d.force_epi == 1 + kEpiGeneral, "gemm fp8: general epilogue only");
  plan->bn = bn;
  plan->cluster = 1;
  plan->fp8 = 1;
  plan->epi = kEpiGeneral;
  const long tiles_m = (d.M + kGemmBM - 1) / kGemmBM;
  const long tiles = tiles_m * ((d.N + bn - 1) / bn);
  p.m_fast = (tiles_m > 1 && d.M < d.N) ? 1 : 0;
  const long slots = num_sms();
  plan->grid = static_cast<int>(tiles < slots ? tiles : slots);
  return THMR_OK;
}

inline int gemm_make_plan(const GemmDesc& d, GemmPlan* plan) {
  if (d.fp8) return gemm_make_plan_fp8(d, plan);
  THMR_CHECK(d.M > 0 && d.N > 0 && d.K > 0, "gemm: bad shape %dx%dx%d", d.M, d.N, d.K);
  THMR_CHECK(d.out32 || d.out16 || d.argmin_out, "gemm: no output");
  const int cluster = d.force_bn == 512 ? 2 : 1;
  THMR_CHECK(cluster == 1 || !d.argmin_out, "gemm: block_n 512 (CTA pair) does not support the arg-min modes");
  const int kind = gemm_pick_epi(d, 256, cluster);   // the kind does not depend on the width
  const int bn = cluster == 2 ? 256 : pick_bn(d.M, d.N, d.K, d.argmin_out == nullptr, kind, d.force_bn);
  THMR_CHECK(bn == 32 || bn == 64 || bn == 128 || bn == 256, "gemm: bad block_n %d", bn);
  GemmParams& p = plan->p;
  memset(&p, 0, sizeof(p));
  p.M = d.M; p.N = d.N; p.K = d.K;
  p.out32 = d.out32; p.ld32 = d.ld32; p.out16 = d.out16; p.ld16 = d.ld16;
  p.bias = d.bias; p.resid = d.resid; p.ldr = d.ldr; p.resid_mod = d.resid_mod; p.act = d.act; p.act32 = d.act32;
  p.seq_pitch = d.seq_pitch; p.seq_lo = d.seq_lo; p.seq_hi = d.seq_hi;
  p.alpha = d.alpha; p.argmin_out = d.argmin_out; p.row_sq = d.row_sq; p.col_sq = d.col_sq;
  THMR_CHECK(!d.screen_rows || (d.argmin_out && d.screen_count && d.screen_cmax2),
             "gemm: screened arg-min needs its queue");
  THMR_CHECK((!d.m_dev && !d.row_map) || d.argmin_out, "gemm: device row count / row map are arg-min options");
  p.screen_rows = d.screen_rows; p.screen_count = d.screen_count; p.screen_cmax2 = d.screen_cmax2;
  p.screen_rel = d.screen_rel; p.screen_abs = d.screen_abs; p.screen_row0 = d.screen_row0;
  p.row_map = d.row_map; p.m_dev = d.m_dev; p.m_dev_off = d.m_dev_off;
  p.stamp = d.stamp;
  const int num_kb = (d.K + kGemmBK - 1) / kGemmBK;
  uint64_t a_cols = d.K;
  if (d.taps > 1) {
    THMR_CHECK(d.cin % kGemmBK == 0 && d.K == d.taps * d.cin, "gemm conv: cin %d taps %d K %d", d.cin, d.taps, d.K);
    p.kblocks_per_tap = d.cin / kGemmBK;
    p.tap_row0 = d.tap_row0; p.tap_stride = d.tap_stride;
    a_cols = d.cin;
  } else {
    p.kblocks_per_tap = num_kb;
  }
  THMR_TRY(make_tmap_2d_f16(&plan->tmA, d.A, d.a_rows, a_cols, d.lda, kGemmBM, kGemmBK, CU_TENSOR_MAP_SWIZZLE_128B));
  THMR_TRY(make_tmap_2d_f16(&plan->tmB, d.B, d.N, d.K, d.ldb, bn / cluster, kGemmBK, CU_TENSOR_MAP_SWIZZLE_128B));
  plan->bn = bn;
  plan->cluster = cluster;
  plan->fp8 = 0;
  plan->epi = gemm_pick_epi(d, bn, cluster);
  THMR_CHECK(d.force_epi == 0 || d.force_epi - 1 == kEpiGeneral || d.force_epi - 1 == plan->epi,
             "gemm: epilogue kind %d does not fit this GEMM (its kind is %d)", d.force_epi - 1, plan->epi);
  if (d.force_epi) plan->epi = d.force_epi - 1;
  memset(&plan->tmC, 0, sizeof(plan->tmC));
  // gemm_pick_epi checked the 16-byte base and pitch TMA needs
  if (gemm_epi_tma_store(plan->epi))
    THMR_TRY(make_tmap_2d_f16(&plan->tmC, d.out16, d.M, d.N, d.ld16, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B));
  if (plan->epi == kEpiBiasResidF32)
    THMR_TRY(make_tmap_2d(&plan->tmC, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, d.out32, d.M, d.N, d.ld32, 64, 32,
                          CU_TENSOR_MAP_SWIZZLE_128B));
  const long tiles_m = (d.M + kGemmBM * cluster - 1) / (kGemmBM * cluster);
  const long tiles = d.argmin_out ? tiles_m : tiles_m * ((d.N + bn - 1) / bn);
  // the CTAs of a wave should share tiles of the larger operand (TileIter)
  p.m_fast = (!d.argmin_out && tiles_m > 1 && d.M < d.N) ? 1 : 0;
  const long slots = num_sms() / cluster;   // CTAs (clusters) resident at once
  plan->grid = cluster * static_cast<int>(tiles < slots ? tiles : slots);
  return THMR_OK;
}

template <int BN, int STAGES, int CLUSTER = 1, bool FP8 = false, int EPI = kEpiGeneral, bool TIMELINE = false>
inline int gemm_launch_t(const GemmPlan& plan, cudaStream_t stream) {
  using S = GemmSmem<BN, STAGES, FP8, EPI>;
  static_assert(S::kTotal <= kGemmSmemLimit, "GEMM shared memory exceeds 227 KB");
  static bool configured = false;
  if (!configured) {
    THMR_CUDA(cudaFuncSetAttribute(gemm_f16_tn_kernel<BN, STAGES, CLUSTER, FP8, EPI, TIMELINE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   S::kTotal));
    configured = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(plan.grid);
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = S::kTotal;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CLUSTER;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  THMR_CUDA(cudaLaunchKernelEx(&cfg, gemm_f16_tn_kernel<BN, STAGES, CLUSTER, FP8, EPI, TIMELINE>, plan.tmA, plan.tmB,
                               plan.tmC, plan.p));
  return THMR_OK;
}

// Operand ring depth of the 128- and 256-wide fp16 kernels; the residual kind's ring (GemmSmem::kResidBufs) takes
// what is left.  At block_n 128 the residual kind gives up one stage so that its ring holds the whole tile (4 boxes per
// warpgroup instead of 2); at 256 it keeps all 4 stages (2 boxes): one stage fewer (5 boxes) slowed the main loop more
// than it shortened the epilogue.  DESIGN.md §6 has the timelines this was chosen from.
template <int BN, int EPI>
constexpr int gemm_stages() {
  return BN == 256 ? 4 : EPI == kEpiBiasResidF32 ? 5 : 6;
}

template <int BN, bool TIMELINE>
inline int gemm_launch_epi(const GemmPlan& plan, cudaStream_t stream) {
  switch (plan.epi) {
    case kEpiGeneral: return gemm_launch_t<BN, gemm_stages<BN, kEpiGeneral>(), 1, false, kEpiGeneral, TIMELINE>(plan, stream);
    case kEpiF16: return gemm_launch_t<BN, gemm_stages<BN, kEpiF16>(), 1, false, kEpiF16, TIMELINE>(plan, stream);
    case kEpiBiasF16: return gemm_launch_t<BN, gemm_stages<BN, kEpiBiasF16>(), 1, false, kEpiBiasF16, TIMELINE>(plan, stream);
    case kEpiBiasGeluF16:
      return gemm_launch_t<BN, gemm_stages<BN, kEpiBiasGeluF16>(), 1, false, kEpiBiasGeluF16, TIMELINE>(plan, stream);
    case kEpiBiasResidF32:
      return gemm_launch_t<BN, gemm_stages<BN, kEpiBiasResidF32>(), 1, false, kEpiBiasResidF32, TIMELINE>(plan, stream);
  }
  return fail(THMR_ERR_INVALID, "gemm: unsupported epilogue kind %d", plan.epi);
}

// Launches a plan made by gemm_make_plan / gemm_make_plan_fp8.
inline int gemm_launch_plain(const GemmPlan& plan, cudaStream_t stream) {
  if (plan.fp8) {
    // the stage ring also carries 512 bytes of activation scales per stage, and the epilogue the row scales
    if (plan.bn == 128) return gemm_launch_t<128, 5, 1, true>(plan, stream);
    if (plan.bn == 64) return gemm_launch_t<64, 7, 1, true>(plan, stream);
    return fail(THMR_ERR_INVALID, "gemm fp8: unsupported block_n %d", plan.bn);
  }
  if (plan.cluster == 2) return gemm_launch_t<256, 4, 2>(plan, stream);
  switch (plan.bn) {
    case 256: return gemm_launch_epi<256, false>(plan, stream);
    case 128: return gemm_launch_epi<128, false>(plan, stream);
    case 64: return gemm_launch_t<64, 8>(plan, stream);
    case 32: return gemm_launch_t<32, 8>(plan, stream);
  }
  return fail(THMR_ERR_INVALID, "gemm: unsupported block_n %d", plan.bn);
}

// gemm_launch<true>: the per-tile timeline kernels (GemmParams::timeline, test probe only), fp16 single-CTA plans at
// block_n 128 / 256
template <bool TIMELINE = false>
inline int gemm_launch(const GemmPlan& plan, cudaStream_t stream) {
  if constexpr (TIMELINE) {
    THMR_CHECK(!plan.fp8 && plan.cluster == 1 && (plan.bn == 128 || plan.bn == 256),
               "gemm timeline: fp16 block_n 128 / 256 only (block_n %d)", plan.bn);
    return plan.bn == 256 ? gemm_launch_epi<256, true>(plan, stream) : gemm_launch_epi<128, true>(plan, stream);
  } else {
    THMR_CHECK(plan.epi == kEpiGeneral || (plan.bn >= 128 && plan.cluster == 1 && !plan.fp8),
               "gemm: epilogue kind %d at block_n %d", plan.epi, plan.bn);
    return gemm_launch_plain(plan, stream);
  }
}

}  // namespace thmr
