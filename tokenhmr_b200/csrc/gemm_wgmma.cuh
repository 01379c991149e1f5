// Persistent warp-specialised wgmma GEMM:  C[M,N] = epilogue(alpha * A[M,K] * B[N,K]^T)
//   A (activations) and B (nn.Linear / conv weight, stored [out, in]) are both K-major fp16,
//   accumulation is fp32 in the registers of two consumer warpgroups.
//
//   warps 0-3 : consumer warpgroup 0, rows 0..63 of the 128-row tile    wgmma m64nBNk16, then the epilogue
//   warps 4-7 : consumer warpgroup 1, rows 64..127
//   warps 8-11: producer warpgroup; one thread issues the TMA loads  global -> 128B-swizzled smem ring of STAGES k-blocks
//               (residual kind: one thread each of warps 9 and 10 issues the TMA reductions of consumer
//               warpgroup 0 / 1)
//
// setmaxnreg moves registers from the producer warpgroup (40 per thread) to the consumers (232), so that a 64 x 256
// fp32 accumulator tile (128 registers per thread) and the epilogue fit without spilling.
//
// CLUSTER = 2 (block_n 512 on the C ABI): the two CTAs of a cluster compute one 256 x BN tile, 128 rows each, and share
// its B operand: each producer loads half of the B rows and multicasts them into both CTAs' shared memory, so every
// k-block moves 128 x 128 + BN / 2 x 128 bytes per CTA from L2 instead of 128 x 128 + BN x 128.  A stage is free again
// once the consumers of BOTH CTAs have released it (the empty barrier counts the consumer warps of the cluster).
//
// The producer runs ahead into the next tile while the consumers store the current one, so the epilogue overlaps the
// operand loads of the next tile.  The element-wise epilogue stages the accumulators through shared memory and stores
// whole row segments (gemm_epilogue_rows); it handles alpha scale, bias, a residual (may alias out32: same element,
// same thread), residual tables, padded-sequence masking, activations, fp32 and / or fp16 outputs.  The fp16-output
// epilogue kinds instead hand their finished tiles to TMA stores and go straight on to the next tile
// (gemm_epilogue_f16_tma); so does the in-place fp32 residual kind, whose alpha * acc + bias two more producer threads
// add into the residual with TMA reductions (gemm_resid_thread, gemm_epilogue_resid_tma).  The
// row-argmin modes of the VQ nearest-code search work straight from the accumulator registers.
//
// The same kernel runs the implicit-GEMM Conv1d (k=3, dilated) of the pose-token decoder: k-blocks are
// grouped in "taps", each tap reads the A rows shifted by a row offset (TMA zero-fills out-of-range rows).
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace thmr {

enum : int { kActNone = 0, kActGelu = 1, kActRelu = 2 };

// Epilogue kinds (GemmPlan::epi, a template parameter of the kernel).  kEpiGeneral (gemm_epilogue_rows) compiles every
// option of GemmParams in; the others compile only what the ViT's call sites use:
//   kEpiF16           alpha * acc -> fp16                          decoder to_kv   (gemm_epilogue_f16_tma)
//   kEpiBiasF16       alpha * acc + bias -> fp16                   QKV             (gemm_epilogue_f16_tma)
//   kEpiBiasGeluF16   GELU(alpha * acc + bias) -> fp16             fc1             (gemm_epilogue_f16_tma)
//   kEpiBiasResidF32  alpha * acc + bias + resid -> fp32           proj, fc2 (resid aliases out32; gemm_epilogue_resid_tma)
enum : int { kEpiGeneral = 0, kEpiF16 = 1, kEpiBiasF16 = 2, kEpiBiasGeluF16 = 3, kEpiBiasResidF32 = 4 };

// The fp16-output kinds store their tiles with TMA through GemmPlan::tmC; the residual kind adds into x through it.
constexpr bool gemm_epi_tma_store(int epi) { return epi == kEpiF16 || epi == kEpiBiasF16 || epi == kEpiBiasGeluF16; }

struct GemmParams {
  int M, N, K;
  float* out32;   // acc + bias + resid, fp32 (nullable)
  int ld32;
  __half* out16;  // act(acc + bias + resid) rounded to fp16 (nullable)
  int ld16;
  const float* bias;   // [N] (nullable)
  const float* resid;  // fp32 [*, N] (nullable); may alias out32 (same element, same thread)
  int ldr;
  int resid_mod;  // > 0: residual row = row % resid_mod (position-embedding table)
  int act;
  int act32;  // apply the activation to the fp32 output as well (conv + ReLU feeding a residual)
  // implicit conv: tap t = kb / kblocks_per_tap reads A rows (m + tap_row0 + t * tap_stride)
  int kblocks_per_tap;
  int tap_row0, tap_stride;
  // padded sequences: rows with (row % seq_pitch) outside [seq_lo, seq_hi) are stored as zero
  int seq_pitch, seq_lo, seq_hi;
  float alpha;  // accumulator scale (split-precision operands are pre-scaled by powers of two)
  // row-argmin mode (VQ nearest code, quantize_cnn.py:80-86): the CTA walks all column tiles of one row
  // block and keeps a running first-minimum of  d = (row_sq[row] - 2*alpha*acc) + col_sq[col]
  long long* argmin_out;   // [M] int64 (nullable = normal GEMM)
  const float* row_sq;     // [M]
  const float* col_sq;     // [N]
  // screened row-argmin (vq.cuh, two-pass hard quantise).  Pass 1 (screen_rows != nullptr) runs single-product fp16
  // operands, keeps the best AND the second-best of  e = col_sq - 2*alpha*acc  per row, always stores the best index
  // and appends the row to screen_rows when (second - best) does not exceed the rigorous error margin
  //   tau = screen_rel * sqrt(row_sq * cmax2) + screen_abs * (row_sq + cmax2) + 1e-12   (cmax2 = max col_sq);
  // such rows are re-done by the exact split-precision pass.  The exact pass reads its row count from device memory
  // (m_dev, minus m_dev_off, clamped to [0, M]) and scatters through row_map.
  int* screen_rows;            // [>= M rows of capacity overall] global row ids of the rows to re-do (nullable)
  int* screen_count;           // device counter (appended with one atomicAdd per warp)
  const float* screen_cmax2;   // device scalar: max over col_sq
  float screen_rel, screen_abs;
  int screen_row0;             // global id of row 0 of this launch (pass 1 runs in L2-sized chunks)
  const int* row_map;          // exact pass: argmin_out[row_map[row]] (nullable = identity)
  const int* m_dev;            // device row count (nullable = M)
  int m_dev_off;
  unsigned long long* stamp;   // in-graph start stamp (common.cuh stamp_start), nullable
  int m_fast;     // row tile fastest in the tile order (see TileIter)
  // FP8 operands (gemm_f16_tn_kernel<..., FP8 = true>): A and B are e4m3 with power-of-two block scales, a k-block is
  // 128 elements.  Each k-block's products accumulate in a fresh register tile that is then promoted into the fp32
  // accumulator:  acc += tile * (a_scale[kb][row] * w_scale[n / 128][kb]).
  const float* a_scale;  // [K / 128][ld_as] per (row, k-block), k-block-major: one 512-byte run per 128-row tile
  int ld_as;             // >= the tile-padded row count, a multiple of 4
  const float* w_scale;  // [ceil(N / 128)][K / 128] per 128 x 128 block of B
  // e4m3 output (FP8 only, block_n 128): act(alpha * acc + bias) as codes of one power-of-two scale per (row, 128
  // columns), i.e. per tile row; the scales go to out8_scale[n / 128][row], the layout a_scale expects
  uint8_t* out8;   // nullable
  int ld8;
  float* out8_scale;
  int ld8s;
  // per-tile phase timeline (gemm_f16_tn_kernel<..., TIMELINE = true>, test probe only): lane 0 of each consumer
  // warpgroup writes four %globaltimer stamps per tile into timeline[cta][slot][wg][4] (tile start, first full barrier
  // passed, last wgmma retired, epilogue done -- for the TMA-stored kinds: the tile's stores issued, not completed)
  // for the CTA's first timeline_slots tiles, and %smid into timeline_sm[cta]
  unsigned long long* timeline;
  int timeline_slots;
  int* timeline_sm;
};

// Tile order shared by the producer and the consumers.  Normal mode: tiles round-robin over CTAs, column tile
// fastest -- or row tile fastest (GemmParams::m_fast, chosen by the host when M < N): the CTAs of a wave then share the
// tiles of the LARGER operand, which is streamed from HBM once instead of once per wave (SMPL blend GEMM: 256 poses x
// 20672 basis rows).  Row-argmin mode: row blocks round-robin over CTAs, all column tiles of a row block in sequence.
struct TileIter {
  int tiles_m, tiles_n, m_blk, n_blk, tile, num_tiles;
  bool m_stationary, m_fast;
  int stride;   // tiles (or row blocks) advance by the number of CTAs (clusters) of the grid
  __device__ TileIter(int tm, int tn, bool ms, bool mf, int start, int step)
      : tiles_m(tm), tiles_n(tn), m_stationary(ms), m_fast(mf), stride(step) {
    num_tiles = tm * tn;
    tile = start;
    m_blk = start;
    n_blk = 0;
  }
  __device__ bool valid() const { return m_stationary ? (m_blk < tiles_m) : (tile < num_tiles); }
  __device__ int m0(int bm) const { return (m_stationary ? m_blk : (m_fast ? tile % tiles_m : tile / tiles_n)) * bm; }
  __device__ int n0(int bn) const { return (m_stationary ? n_blk : (m_fast ? tile / tiles_m : tile % tiles_n)) * bn; }
  __device__ bool last_n() const { return n_blk == tiles_n - 1; }
  __device__ void next() {
    if (m_stationary) {
      if (++n_blk == tiles_n) { n_blk = 0; m_blk += stride; }
    } else {
      tile += stride;
    }
  }
};

constexpr int kGemmBM = 128;
constexpr int kGemmBK = 64;
constexpr int kGemmConsumerWarps = 8;
constexpr int kGemmThreads = 32 * kGemmConsumerWarps + 128;  // two consumer warpgroups + the producer warpgroup
constexpr int kWarpTma = kGemmConsumerWarps;

// Columns of one epilogue chunk: each consumer warpgroup stages 64 rows x gemm_chunk fp32 accumulators in shared
// memory.  At BN = 256 the accumulators still held for the later chunks leave registers for the residuals of 32
// columns only (64 spill); narrower tiles take 64.
template <int BN>
constexpr int gemm_chunk() { return BN == 64 || BN == 128 ? 64 : 32; }

// Elements per k-block: one 128-byte swizzle row, 64 fp16 or 128 e4m3.  Both have the same byte geometry.
template <bool FP8>
constexpr int gemm_bk() { return FP8 ? 128 : kGemmBK; }

// Largest dynamic shared memory of one CTA on sm_90 (227 KB).
constexpr uint32_t kGemmSmemLimit = 232448;
// One box of the residual kind's ring (gemm_epilogue_resid_tma): 64 rows x 32 fp32 columns, one 128-byte swizzle row each.
constexpr uint32_t kResidBoxBytes = 64 * 32 * 4;

template <int BN, int STAGES, bool FP8 = false, int EPI = kEpiGeneral>
struct GemmSmem {
  static constexpr uint32_t kABytes = kGemmBM * kGemmBK * 2;
  static constexpr uint32_t kBBytes = BN * kGemmBK * 2;
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;   // multiple of 1024: every operand tile stays swizzle-aligned
  static constexpr uint32_t kEpiOffset = STAGES * kStageBytes;
  // residual kind: per warpgroup a ring of kResidBufs 64 x 32 fp32 boxes, as many as fit next to the operand ring (at
  // most one tile's worth); they hold alpha * acc + bias until the TMA reductions have read it
  static constexpr int kResidFit = static_cast<int>((kGemmSmemLimit - kEpiOffset - 256 - 1024) / (2 * kResidBoxBytes));
  static constexpr int kResidBufs = EPI != kEpiBiasResidF32 ? 0 : kResidFit < BN / 32 ? kResidFit : BN / 32;
  static_assert(EPI != kEpiBiasResidF32 || kResidBufs >= 2, "residual ring needs two boxes per warpgroup");
  // otherwise epilogue staging, 16 KB per warpgroup: a 64 x gemm_chunk block of fp32 accumulators (general epilogue) or
  // a 64 x 128 fp16 output tile, two 128B-swizzled TMA store boxes (fp16 kinds).  Either way 1024-byte aligned.
  static constexpr uint32_t kEpiWgBytes = EPI == kEpiBiasResidF32 ? kResidBufs * kResidBoxBytes : 64 * 128 * 2;
  static_assert(EPI == kEpiBiasResidF32 || 64 * gemm_chunk<BN>() * 4 <= kEpiWgBytes,
                "fp32 staging chunk exceeds the warpgroup's block");
  static constexpr uint32_t kEpiBytes = 2 * kEpiWgBytes;
  // FP8: the 128 activation scales of each stage's k-block ride the same ring, outside the swizzled operand tiles
  static constexpr uint32_t kScaleOffset = kEpiOffset + kEpiBytes;
  static constexpr uint32_t kScaleBytes = FP8 ? STAGES * kGemmBM * 4 : 0;
  // mbarriers: full / empty per stage, then (residual kind) free / done per ring box of each warpgroup
  static constexpr uint32_t kBarOffset = kScaleOffset + kScaleBytes;
  static_assert((2 * STAGES + 4 * kResidBufs) * 8 <= 256, "mbarriers exceed their 256 bytes");
  static constexpr uint32_t kRowScaleOffset = kBarOffset + 256;   // FP8 e4m3 output: 1 / scale of each tile row
  static constexpr uint32_t kRowScaleBytes = FP8 ? kGemmBM * 4 : 0;
  static constexpr uint32_t kTotal = kRowScaleOffset + kRowScaleBytes + 1024;  // alignment slack
};

// Exact-erf GELU (nn.GELU default, vit.py:73).  The epilogue evaluates 63 M of these per MLP layer, so erf uses
// Abramowitz-Stegun 7.1.28  erf(a) = 1 - (1 + c1 a + ... + c6 a^6)^-16  (|err| < 2e-6 in fp32, i.e. GELU within
// 9e-7 absolute of the libm path; the result is rounded to fp16 afterwards): 7 FMA + 4 MUL + 1 MUFU.RCP, no branches.
__device__ __forceinline__ float gelu_erf(float x) {
  const float a = fabsf(x) * 0.70710678118654752f;
  float p = fmaf(0.0000430638f, a, 0.0002765672f);
  p = fmaf(p, a, 0.0001520143f);
  p = fmaf(p, a, 0.0092705272f);
  p = fmaf(p, a, 0.0422820123f);
  p = fmaf(p, a, 0.0705230784f);
  p = fmaf(p, a, 1.0f);
  p *= p; p *= p; p *= p; p *= p;
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(p));   // 1 ulp-class MUFU reciprocal (p >= 1; p = inf -> 0)
  const float e = 1.0f - r;                       // erf(|x| / sqrt(2))
  // 0.5 x (1 + sign(x) e) as fma(x, 0.5, (0.5 |x|) e), spelled out so that every epilogue kind rounds it alike
  return fmaf(x, 0.5f, __fmul_rn(__fmul_rn(fabsf(x), 0.5f), e));
}

template <int BN>
__device__ __forceinline__ void wgmma_tile_k16(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BN == 32) wgmma_m64n32k16(acc, da, db, scale_d);
  else if constexpr (BN == 64) wgmma_m64n64k16(acc, da, db, scale_d);
  else if constexpr (BN == 128) wgmma_m64n128k16(acc, da, db, scale_d);
  else wgmma_m64n256k16(acc, da, db, scale_d);
}

template <int BN>
__device__ __forceinline__ void wgmma_tile_k32_e4m3(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BN == 64) wgmma_m64n64k32_e4m3(acc, da, db, scale_d);
  else wgmma_m64n128k32_e4m3(acc, da, db, scale_d);
}

__device__ __forceinline__ float gemm_act(int act, float v) {
  return act == kActGelu ? gelu_erf(v) : act == kActRelu ? fmaxf(v, 0.f) : v;
}

__device__ __forceinline__ bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

// Fragment -> staging block: the accumulators of chunk c (columns c * CH ..) of the thread's rows fr, fr + 8 of the
// warpgroup's 64, in the swizzled staging layout of gemm_epilogue_rows.  c must be a compile-time constant after
// unrolling, so that acc is indexed by constants and stays in registers.
template <int BN>
__device__ __forceinline__ void gemm_stage_chunk(const float (&acc)[BN / 2], int c, uint32_t stage, int fr, int fswz,
                                                 int lane) {
  constexpr int CH = gemm_chunk<BN>();
  constexpr int OCT = CH / 8;
#pragma unroll
  for (int j = 0; j < OCT; ++j) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int u = 2 * j + ((lane & 3) >> 1);
      const int a = 4 * (c * OCT + j) + 2 * i;
      sts_f32x2(stage + 4 * ((fr + 8 * i) * CH + (((u & ~7) | ((u ^ fswz) & 7)) << 2) + 2 * (lane & 1)), acc[a],
                acc[a + 1]);
    }
  }
}

// Element-wise epilogue of one consumer warpgroup: its 64 rows x BN columns of accumulators, rows m0w.. of the output.
// The accumulator fragment (two rows x two columns per 8-column group and thread) goes to a shared-memory chunk of
// 64 x CH fp32; the warpgroup then walks the chunk row-major, each thread owning 8 consecutive columns ("octets") of
// two rows, so that every global access is a 16-byte vector of one row (scalar when base, pitch or N forbid it).  All
// residual loads of a chunk are issued before any of its stores: one memory round trip per chunk instead of one per
// accumulator pair.  A residual aliasing out32 is safe: each element is read and written by the same thread.
// Staging layout: row r of the chunk holds CH / 4 16-byte units; unit u sits at u ^ swz(r) (low three bits), which keeps
// both the fragment writes (four rows x 32 bytes per half-warp) and the row reads (eight rows of one unit per
// quarter-warp) free of bank conflicts.
// FP8 e4m3 output (p.out8): the accumulators already hold act(alpha * acc + bias) (gemm_row_scales_e4m3), so the
// values are only stored: fp32 / fp16 copies as they are, and the codes of v / s with 1 / s read from row_inv.
template <int BN, bool FP8 = false>
__device__ __forceinline__ void gemm_epilogue_rows(const GemmParams& p, const float (&acc)[BN / 2], uint32_t stage,
                                                   int m0w, int n0, int M_eff, uint32_t bar_id, bool vec_r, bool vec32,
                                                   bool vec16, uint32_t row_inv = 0) {
  const bool final_vals = FP8 && p.out8 != nullptr;
  constexpr int CH = gemm_chunk<BN>();
  constexpr int OCT = CH / 8;          // octets per chunk row
  constexpr int ITEMS = OCT / 2;       // (row, octet) items per thread and chunk: 64 * OCT / 128
  const int lane = threadIdx.x & 31;
  const int w4 = (threadIdx.x >> 5) & 3;
  // fragment side: rows (16 w4 + lane / 4 + 8 i), columns 8 j + 2 (lane % 4) + {0, 1}
  const int fr = w4 * 16 + (lane >> 2);
  const int fswz = (((lane >> 2) & 3) << 1) | ((lane >> 4) & 1);   // swz(fr), fr % 8 = lane / 4
  // row side: item k is row (8 (w4 + 4 (k % 2)) + lane % 8), octet (4 (k / 2) + lane / 8) of the chunk
  const int rswz = ((lane & 3) << 1) | ((lane >> 2) & 1);          // swz(row), row % 8 = lane % 8
  // row terms, once per tile: the thread's two rows, whether they exist, the padded-sequence mask, the residual row
  int rows[2];
  bool live[2], keep[2];
  const float* rres[2];
#pragma unroll
  for (int ri = 0; ri < 2; ++ri) {
    const int row = m0w + 8 * (w4 + 4 * ri) + (lane & 7);
    rows[ri] = row;
    live[ri] = row < M_eff;
    keep[ri] = true;
    if (p.seq_pitch > 0) {
      const int rr = row % p.seq_pitch;
      keep[ri] = rr >= p.seq_lo && rr < p.seq_hi;
    }
    // a masked row is stored as zero whatever its residual, so the residual is not read
    rres[ri] = (p.resid && live[ri] && keep[ri])
                   ? p.resid + static_cast<size_t>(p.resid_mod > 0 ? row % p.resid_mod : row) * p.ldr
                   : nullptr;
  }

#pragma unroll
  for (int c = 0; c < BN / CH; ++c) {
    gemm_stage_chunk<BN>(acc, c, stage, fr, fswz, lane);
    named_barrier_sync(bar_id, 128);

    const int ccol = n0 + c * CH + 8 * (lane >> 3);   // first column of octet 0 of this thread in the chunk
    float bias[ITEMS / 2][8];
    float res[ITEMS][8];
#pragma unroll
    for (int ob = 0; ob < ITEMS / 2; ++ob)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int col = ccol + 32 * ob + e;
        bias[ob][e] = (p.bias && col < p.N) ? __ldg(p.bias + col) : 0.f;
      }
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const int col = ccol + 32 * (k >> 1);
      const float* r = rres[k & 1];
#pragma unroll
      for (int e = 0; e < 8; ++e) res[k][e] = 0.f;
      if (r != nullptr && col < p.N) {
        if (vec_r && col + 8 <= p.N) {
          const float4 x0 = *reinterpret_cast<const float4*>(r + col);
          const float4 x1 = *reinterpret_cast<const float4*>(r + col + 4);
          res[k][0] = x0.x; res[k][1] = x0.y; res[k][2] = x0.z; res[k][3] = x0.w;
          res[k][4] = x1.x; res[k][5] = x1.y; res[k][6] = x1.z; res[k][7] = x1.w;
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (col + e < p.N) res[k][e] = r[col + e];
        }
      }
    }
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
      const int ri = k & 1;
      const int lr = 8 * (w4 + 4 * ri) + (lane & 7);
      const int oct = 4 * (k >> 1) + (lane >> 3);
      const int col = ccol + 32 * (k >> 1);
      const int row = rows[ri];
      if (!live[ri] || col >= p.N) continue;
      float v[8];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int u = 2 * oct + h;
        const float4 s = lds_f32x4(stage + 4 * (lr * CH + (((u & ~7) | ((u ^ rswz) & 7)) << 2)));
        v[4 * h] = s.x; v[4 * h + 1] = s.y; v[4 * h + 2] = s.z; v[4 * h + 3] = s.w;
      }
      // alpha * acc + bias + resid, mask, activation: the operation order of the reference epilogue, element for element
      // (rounded step by step, never contracted: gemm_epilogue_kind computes the same values)
      if (!final_vals) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          v[e] = __fmul_rn(v[e], p.alpha);
          if (p.bias) v[e] = __fadd_rn(v[e], bias[k >> 1][e]);
          if (p.resid) v[e] = __fadd_rn(v[e], res[k][e]);
          if (!keep[ri]) v[e] = 0.f;
          if (p.act32) v[e] = gemm_act(p.act, v[e]);
        }
      }
      const bool full = col + 8 <= p.N;
      if (p.out32) {
        float* o = p.out32 + static_cast<size_t>(row) * p.ld32 + col;
        if (full && vec32) {
          reinterpret_cast<float4*>(o)[0] = make_float4(v[0], v[1], v[2], v[3]);
          reinterpret_cast<float4*>(o)[1] = make_float4(v[4], v[5], v[6], v[7]);
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (col + e < p.N) o[e] = v[e];
        }
      }
      if constexpr (FP8) {
        if (p.out8) {
          const float inv = lds_f32(row_inv + 4 * lr);
          uint8_t* o = p.out8 + static_cast<size_t>(row) * p.ld8 + col;
          uint16_t q[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) q[e] = cvt_e4m3x2(v[2 * e] * inv, v[2 * e + 1] * inv);
          if (full && p.ld8 % 8 == 0 && (reinterpret_cast<uintptr_t>(p.out8) & 7) == 0) {
            *reinterpret_cast<uint2*>(o) = make_uint2(q[0] | (static_cast<uint32_t>(q[1]) << 16),
                                                      q[2] | (static_cast<uint32_t>(q[3]) << 16));
          } else {
#pragma unroll
            for (int e = 0; e < 8; ++e)
              if (col + e < p.N) o[e] = static_cast<uint8_t>(q[e >> 1] >> (8 * (e & 1)));
          }
        }
      }
      if (p.out16) {
        if (!p.act32 && !final_vals) {
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = gemm_act(p.act, v[e]);
        }
        __half* o = p.out16 + static_cast<size_t>(row) * p.ld16 + col;
        if (full && vec16) {
          uint4 q;
          __half2* h2 = reinterpret_cast<__half2*>(&q);
#pragma unroll
          for (int e = 0; e < 4; ++e) h2[e] = __floats2half2_rn(v[2 * e], v[2 * e + 1]);
          *reinterpret_cast<uint4*>(o) = q;
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (col + e < p.N) o[e] = __float2half_rn(v[e]);
        }
      }
    }
    // the next chunk (or tile) overwrites the staging block
    named_barrier_sync(bar_id, 128);
  }
}

// Ring position of a warpgroup's residual boxes (kEpiBiasResidF32): the reduction thread and the consumers walk the
// same sequence of boxes, so each side keeps its own copy.
struct RingPos {
  int slot = 0;
  uint32_t phase = 0;
  template <int NB>
  __device__ __forceinline__ void next() {
    if (++slot == NB) { slot = 0; phase ^= 1; }
  }
};

// The boxes of one consumer warpgroup in the order its residual epilogue takes them: per tile, one 64 x 32 box of rows
// m0w .. m0w + 63 per 32 columns.  Boxes past N are skipped, and so are the tiles in which the warpgroup has no rows
// (m0w >= M); TMA clips the reductions past [M, N].
template <int BN>
struct ResidBoxIter {
  TileIter it;
  int row_off, M, N, c = 0;
  __device__ ResidBoxIter(const TileIter& t, int ro, int m, int n) : it(t), row_off(ro), M(m), N(n) { skip(); }
  __device__ bool valid() const { return it.valid(); }
  __device__ int m0w() const { return it.m0(kGemmBM) + row_off; }
  __device__ int col() const { return it.n0(BN) + 32 * c; }
  __device__ void skip() {
    while (it.valid() && m0w() >= M) it.next();
  }
  __device__ void next() {
    if (++c == BN / 32 || col() >= N) {
      c = 0;
      it.next();
      skip();
    }
  }
};

// Reduction thread of one consumer warpgroup (kEpiBiasResidF32; one thread of the producer warpgroup each).  It owns the
// TMA side of the warpgroup's ring of NB boxes: for each box in turn it waits until the consumers have written
// alpha * acc + bias into it, adds the box into x with a TMA reduction (x += box, in L2), and hands the previous box
// back to the consumers as soon as its reduction has read it.  The residual is never loaded into the SM, and the waits
// on the reductions are this thread's alone, so the consumers only wait for a free box.
template <int BN, int NB>
__device__ __forceinline__ void gemm_resid_thread(const CUtensorMap* tm, uint32_t ring, uint64_t* free_bar,
                                                  uint64_t* done, ResidBoxIter<BN> it) {
  for (int s = 0; s < NB; ++s) mbar_arrive(&free_bar[s]);
  RingPos rp;
  int prev = -1;
  for (; it.valid(); it.next()) {
    mbar_wait(&done[rp.slot], rp.phase);
    tma_reduce_add_2d(tm, ring + rp.slot * kResidBoxBytes, it.col(), it.m0w());
    tma_store_commit();
    if (prev >= 0) {
      tma_store_wait_read<1>();
      mbar_arrive(&free_bar[prev]);
    }
    prev = rp.slot;
    rp.next<NB>();
  }
  // the reductions complete (and stop reading the ring) before the CTA exits
  tma_store_wait<0>();
}

// Epilogue of one consumer warpgroup for kEpiBiasResidF32, x = alpha * acc + bias + x in place (out32 aliases the
// residual; GemmPlan::tmC maps it): its 64 rows x BN columns, rows m0w.. of the output, one 64 x 32 box of the ring
// per 32 columns.  Each thread writes alpha * acc + bias, rounded step by step as gemm_epilogue_rows does, from the
// accumulator fragment into a free box (SWIZZLE_128B: row r is 128 bytes, 16-byte unit u at u ^ (r % 8)); each warp
// then hands the box to gemm_resid_thread, whose TMA reduction adds it into x, and goes on without waiting.  fp32
// addition is commutative, so x + v equals the general epilogue's v + x bit for bit, except that the reduction
// flushes a subnormal x, v or sum (|.| < 2^-126) to zero.
// The fragment's rows r and r ^ 1 hit the same two units of a column group, so odd rows take the column groups in the
// order 2, 3, 0, 1: the sixteen 64-bit stores of a half-warp (four rows x 32 bytes) then fall on distinct banks.
template <int BN, int NB>
__device__ __forceinline__ void gemm_epilogue_resid_tma(const GemmParams& p, const float (&acc)[BN / 2], uint32_t ring,
                                                        uint64_t* free_bar, uint64_t* done, RingPos& rp, int n0) {
  const int lane = threadIdx.x & 31;
  // fragment: rows fr, fr + 8 of the warpgroup (both = lane / 4 mod 8), columns 8 j + c0 + {0, 1}
  const int fr = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  const int c0 = 2 * (lane & 3);
  const int swz = (lane >> 2) & 7;
  const int jx = (lane & 4) ? 2 : 0;   // odd rows: column group jj ^ 2
#pragma unroll 1
  for (int c = 0; c < BN / 32; ++c) {
    const int nc = n0 + 32 * c;
    if (nc >= p.N) break;
    mbar_wait(&free_bar[rp.slot], rp.phase);
    const uint32_t box = ring + rp.slot * kResidBoxBytes;
#pragma unroll
    for (int cc = 0; cc < BN / 32; ++cc) {
      if (cc != c) continue;   // a uniform branch: the fragment is indexed by constants
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int jj = t ^ jx;
        const int col = nc + 8 * jj + c0;
        // columns past N are clipped by the reduction, so their bias may be any value
        const float b0 = __ldg(p.bias + min(col, p.N - 1));
        const float b1 = __ldg(p.bias + min(col + 1, p.N - 1));
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int a = 4 * (4 * cc + t) + 2 * i, a2 = 4 * (4 * cc + (t ^ 2)) + 2 * i;
          const float v0 = jx ? acc[a2] : acc[a];
          const float v1 = jx ? acc[a2 + 1] : acc[a + 1];
          sts_f32x2(box + (fr + 8 * i) * 128 + (((2 * jj + (c0 >> 2)) ^ swz) << 4) + 4 * (c0 & 3),
                    __fadd_rn(__fmul_rn(v0, p.alpha), b0), __fadd_rn(__fmul_rn(v1, p.alpha), b1));
        }
      }
    }
    // the values become visible to the TMA unit (async proxy) before the reduction thread hands them to it
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) mbar_arrive(&done[rp.slot]);
    rp.next<NB>();
  }
}

// Epilogue of one consumer warpgroup for the fp16-output kinds (kEpiF16, kEpiBiasF16, kEpiBiasGeluF16): its 64 rows x
// BN columns, rows m0w.. of the output.  The values are computed in the accumulator fragment with the rounding steps of
// gemm_epilogue_rows (so they equal the general epilogue's bit for bit), rounded to fp16 and written into the
// warpgroup's staging tile of 64 rows x 128 columns: two 64 x 64 boxes of out16's tensor map (GemmPlan::tmC), each in
// the SWIZZLE_128B layout (row r: 128 bytes, 16-byte unit u at u ^ (r % 8)), so the fragment writes (eight rows of one
// unit per warp store) are free of bank conflicts.  One thread then issues the TMA stores and the warpgroup goes on to
// the next tile without waiting for them; TMA clips the boxes at [M, N], so partial tiles need no scalar tail.  BN = 256
// takes two passes through the staging tile.  Before the tile is overwritten, the issuing thread waits until the
// previous stores have read it.
template <int BN, int EPI>
__device__ __forceinline__ void gemm_epilogue_f16_tma(const GemmParams& p, const float (&acc)[BN / 2],
                                                      const CUtensorMap* tm, uint32_t stage, int m0w, int n0,
                                                      int M_eff, uint32_t bar_id) {
  static_assert(gemm_epi_tma_store(EPI) && BN % 128 == 0, "fp16 TMA-store kinds, 128-column passes");
  const int lane = threadIdx.x & 31;
  const bool issuer = (threadIdx.x & 127) == 0;
  // fragment: rows fr, fr + 8 of the warpgroup (both = lane / 4 mod 8), columns 8 j + c0 + {0, 1}
  const int fr = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  const int c0 = 2 * (lane & 3);
  const int swz = lane >> 2;
#pragma unroll
  for (int q = 0; q < BN / 128; ++q) {
    const int nq = n0 + 128 * q;
    if (nq >= p.N) break;
    if (issuer) tma_store_wait_read<0>();
    named_barrier_sync(bar_id, 128);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = nq + 8 * j + c0;
      float b[2] = {0.f, 0.f};
      if constexpr (EPI != kEpiF16) {
        // columns past N are clipped by the store, so their bias may be any value
        b[0] = __ldg(p.bias + min(col, p.N - 1));
        b[1] = __ldg(p.bias + min(col + 1, p.N - 1));
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float v[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          v[c] = __fmul_rn(acc[64 * q + 4 * j + 2 * i + c], p.alpha);
          if constexpr (EPI != kEpiF16) v[c] = __fadd_rn(v[c], b[c]);
          if constexpr (EPI == kEpiBiasGeluF16) v[c] = gelu_erf(v[c]);
        }
        const __half2 h = __floats2half2_rn(v[0], v[1]);
        sts_u32(stage + (j >> 3) * 8192 + (fr + 8 * i) * 128 + (((j & 7) ^ swz) << 4) + 2 * c0,
                *reinterpret_cast<const uint32_t*>(&h));
      }
    }
    // the staging writes become visible to the TMA unit (async proxy) before it reads them
    fence_proxy_async_smem();
    named_barrier_sync(bar_id, 128);
    if (issuer && m0w < M_eff) {
      tma_store_2d(tm, stage, nq, m0w);
      if (nq + 64 < p.N) tma_store_2d(tm, stage + 8192, nq + 64, m0w);
      tma_store_commit();
    }
  }
}

// e4m3 output, before the element-wise epilogue: replaces the thread's accumulators by v = act(alpha * acc + bias) and
// derives each tile row's scale from the amax of all its BN = 128 columns (the four lanes of a quad hold one row), so
// that no code of a row is written before its whole 128-column group has been seen.  The scale goes to out8_scale,
// its reciprocal (exact: a power of two) to row_inv for the epilogue.
template <int BN>
__device__ __forceinline__ void gemm_row_scales_e4m3(const GemmParams& p, float (&acc)[BN / 2], int m0, int n0,
                                                     int r0, int c0, int wg, int M_eff, uint32_t row_inv) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int col = n0 + 8 * j + c0 + c;
        float v = acc[4 * j + 2 * i + c] * p.alpha;
        if (p.bias && col < p.N) v += __ldg(p.bias + col);
        v = gemm_act(p.act, v);
        acc[4 * j + 2 * i + c] = v;
        if (col < p.N) amax = fmaxf(amax, fabsf(v));
      }
    }
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    const float s = e4m3_scale(amax);
    const int r = r0 + 8 * i;   // row of the tile
    if ((threadIdx.x & 3) == 0) {
      sts_f32(row_inv + 4 * (r - wg * 64), 1.0f / s);
      if (m0 + r < M_eff) p.out8_scale[static_cast<size_t>(n0 / 128) * p.ld8s + m0 + r] = s;
    }
  }
}

template <int BN, int STAGES, int CLUSTER, bool FP8 = false, int EPI = kEpiGeneral, bool TIMELINE = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_f16_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
  using S = GemmSmem<BN, STAGES, FP8, EPI>;
  constexpr int BK = gemm_bk<FP8>();
  constexpr int NB = S::kResidBufs;
  static_assert(BN == 32 || BN == 64 || BN == 128 || BN == 256, "BN must be a power of two in [32,256]");
  static_assert(CLUSTER == 1 || (CLUSTER == 2 && BN >= 128), "cluster pairs split B in two halves of >= 64 rows");
  static_assert(!FP8 || (CLUSTER == 1 && (BN == 64 || BN == 128)), "FP8: two accumulator sets fit at BN <= 128");
  static_assert(EPI == kEpiGeneral || (!FP8 && CLUSTER == 1 && BN >= 128), "epilogue kinds: fp16 BN 128 / 256 only");
  static_assert(!TIMELINE || (!FP8 && CLUSTER == 1), "timeline: fp16 single-CTA kernels only");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  // residual kind: the ring boxes' free (reduction has read it) and done (values written) barriers, NB per warpgroup
  uint64_t* rfree_bar = empty_bar + STAGES;
  uint64_t* rdone_bar = rfree_bar + 2 * NB;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // rows of this launch: p.M, or (exact pass of the screened arg-min) a count a previous kernel left in device memory.
  // Every thread reads the same word, so the producer and the consumers walk identical tile sequences.
  int M_eff = p.M;
  if (p.m_dev != nullptr) {
    const int m = __ldg(p.m_dev) - p.m_dev_off;
    M_eff = m < 0 ? 0 : (m < p.M ? m : p.M);
  }
  constexpr int kRows = kGemmBM * CLUSTER;   // rows of one tile of the CTA (cluster)
  const int tiles_m = (M_eff + kRows - 1) / kRows;
  const int tiles_n = (p.N + BN - 1) / BN;
  const int num_kb = (p.K + BK - 1) / BK;
  const bool m_stationary = p.argmin_out != nullptr;   // (the host never combines arg-min with CLUSTER = 2)
  const int rank = CLUSTER == 2 ? static_cast<int>(cluster_ctarank()) : 0;
  const int tile0 = static_cast<int>(blockIdx.x) / CLUSTER, tile_step = static_cast<int>(gridDim.x) / CLUSTER;

  stamp_start(p.stamp);
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kGemmConsumerWarps * CLUSTER);   // one arrive per consumer warp of the cluster
    }
    for (int b = 0; b < 2 * NB; ++b) {
      mbar_init(&rfree_bar[b], 1);   // the reduction thread's arrive
      mbar_init(&rdone_bar[b], 4);   // one arrive per warp of the consumer warpgroup
    }
    fence_mbar_init();
  }
  if (warp == kWarpTma && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (gemm_epi_tma_store(EPI) || EPI == kEpiBiasResidF32) tma_prefetch_desc(&tmC);
  }
  if constexpr (CLUSTER == 2) cluster_sync_all();   // the peer's barriers are initialised before any multicast or arrive
  else __syncthreads();

  if (warp >= kWarpTma) {
    // ------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == kWarpTma && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (TileIter it(tiles_m, tiles_n, m_stationary, p.m_fast != 0, tile0, tile_step); it.valid(); it.next()) {
        const int m0 = it.m0(kRows) + rank * kGemmBM;
        const int n0 = it.n0(BN);
        for (int kb = 0; kb < num_kb; ++kb) {
          if constexpr (CLUSTER == 2) mbar_wait_cluster(&empty_bar[stage], phase ^ 1);
          else mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * S::kStageBytes;
          uint8_t* sb = sa + S::kABytes;
          const int tap = kb / p.kblocks_per_tap;
          const int kk = kb - tap * p.kblocks_per_tap;
          // the whole stage lands here: own A rows, own half of B and (CLUSTER = 2) the peer's half of B
          mbar_arrive_expect_tx(&full_bar[stage], S::kStageBytes + (FP8 ? kGemmBM * 4 : 0));
          tma_load_2d(sa, &tmA, &full_bar[stage], kk * BK, m0 + p.tap_row0 + tap * p.tap_stride);
          if constexpr (CLUSTER == 2)
            tma_load_2d_mcast(sb + rank * (BN / 2) * 128, &tmB, &full_bar[stage], kb * BK, n0 + rank * (BN / 2), 3);
          else
            tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, n0);
          if constexpr (FP8)
            bulk_load_1d(smem + S::kScaleOffset + stage * kGemmBM * 4, p.a_scale + static_cast<size_t>(kb) * p.ld_as + m0,
                         kGemmBM * 4, &full_bar[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    if constexpr (EPI == kEpiBiasResidF32) {
      // warps kWarpTma + 1 and + 2: the reduction threads of consumer warpgroups 0 and 1
      const int rw = warp - kWarpTma - 1;
      if ((rw == 0 || rw == 1) && lane == 0)
        gemm_resid_thread<BN, NB>(
            &tmC, smem_u32(smem + S::kEpiOffset + rw * S::kEpiWgBytes), rfree_bar + rw * NB, rdone_bar + rw * NB,
            ResidBoxIter<BN>(TileIter(tiles_m, tiles_n, false, p.m_fast != 0, tile0, tile_step), 64 * rw, M_eff, p.N));
    }
    if constexpr (CLUSTER == 2) cluster_sync_all();
    return;
  }

  // -------------------------------------------------------------- consumers: main loop + epilogue
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = warp >> 2;
  const uint32_t smem_base = smem_u32(smem);
  // 16-byte vectors of one row: the base and the pitch keep every 8-column group 16-byte aligned
  const bool vec_r = p.resid && p.ldr % 4 == 0 && aligned16(p.resid);
  const bool vec32 = p.out32 && p.ld32 % 4 == 0 && aligned16(p.out32);
  const bool vec16 = p.out16 && p.ld16 % 8 == 0 && aligned16(p.out16);
  const uint32_t epi_stage = smem_base + S::kEpiOffset + wg * S::kEpiWgBytes;
  const bool screen = p.argmin_out != nullptr && p.screen_rows != nullptr;
  const float m2a = -2.0f * p.alpha;
  // accumulator fragment of this thread: rows r0, r0 + 8 of the tile, columns 8 j + c0 + {0, 1}
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c0 = 2 * (lane & 3);
  float best[2] = {INFINITY, INFINITY}, second[2] = {INFINITY, INFINITY};
  int best_idx[2] = {0, 0};
  int stage = 0;
  uint32_t phase = 0;
  float acc[BN / 2];
  float tile[FP8 ? BN / 2 : 1];   // FP8: the current k-block's products
  RingPos rp;   // residual kind: this warpgroup's position in its ring

  // a consumed stage is released to the producers of every CTA of the cluster
  auto release = [&](int s) {
    __syncwarp();
    if (lane == 0) {
      if constexpr (CLUSTER == 2) {
        mbar_arrive_cluster(&empty_bar[s], 0);
        mbar_arrive_cluster(&empty_bar[s], 1);
      } else {
        mbar_arrive(&empty_bar[s]);
      }
    }
  };
  // timeline (TIMELINE only): lane 0 of each warpgroup stores stamp k of a recorded tile as it takes it, and the slot is
  // derived from the tile index, so that the timeline holds no register across the tile (the 256-wide kinds have none)
  auto stamp = [&](const TileIter& it, int k) {
    if (TIMELINE && p.timeline != nullptr && (threadIdx.x & 127) == 0) {
      const int slot = (it.tile - tile0) / tile_step;
      if (slot < p.timeline_slots)
        p.timeline[((static_cast<size_t>(blockIdx.x) * p.timeline_slots + slot) * 2 + wg) * 4 + k] = globaltimer();
    }
  };
  if (TIMELINE && p.timeline != nullptr && threadIdx.x == 0) p.timeline_sm[blockIdx.x] = static_cast<int>(smid());
  for (TileIter it(tiles_m, tiles_n, m_stationary, p.m_fast != 0, tile0, tile_step); it.valid(); it.next()) {
    const int m0 = it.m0(kRows) + rank * kGemmBM;
    const int n0 = it.n0(BN);
    int prev = -1;
    if constexpr (TIMELINE) stamp(it, 0);
    if constexpr (FP8) {
      // per k-block: four k32 MMAs into a fresh tile, then the promotion  acc += tile * (s_a[row] * s_w).  The tile is
      // reused by the next k-block, so each warpgroup waits for its MMAs; the other warpgroup's keep the tensor core busy.
      const int r0l = r0 - wg * 64;
      const float* wsc = p.w_scale + static_cast<size_t>(n0 / 128) * num_kb;
#pragma unroll
      for (int a = 0; a < BN / 2; ++a) acc[a] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_base + stage * S::kStageBytes + wg * (64 * 128);
        const uint32_t sb = smem_base + stage * S::kStageBytes + S::kABytes;
        wgmma_fence_operand(tile);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 32; ++k)
          wgmma_tile_k32_e4m3<BN>(tile, make_wgmma_desc_sw128(sa + k * 32), make_wgmma_desc_sw128(sb + k * 32),
                                  k != 0 ? 1u : 0u);
        wgmma_commit();
        const float sw = __ldg(wsc + kb);
        const uint32_t ss = smem_base + S::kScaleOffset + stage * kGemmBM * 4 + (wg * 64 + r0l) * 4;
        const float s0 = lds_f32(ss) * sw, s1 = lds_f32(ss + 32) * sw;   // rows r0, r0 + 8: exact products
        wgmma_wait<0>();
        wgmma_fence_operand(tile);
        release(stage);
#pragma unroll
        for (int a = 0; a < BN / 2; ++a) acc[a] = fmaf(tile[a], (a & 2) ? s1 : s0, acc[a]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    } else {
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if constexpr (TIMELINE) if (kb == 0) stamp(it, 1);
        const uint32_t sa = smem_base + stage * S::kStageBytes + wg * (64 * 128);
        const uint32_t sb = smem_base + stage * S::kStageBytes + S::kABytes;
        wgmma_fence_operand(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kGemmBK / 16; ++k)
          wgmma_tile_k16<BN>(acc, make_wgmma_desc_sw128(sa + k * 32), make_wgmma_desc_sw128(sb + k * 32),
                             (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        // the previous k-block's MMAs have retired once at most one group is pending: its smem slot is free
        wgmma_wait<1>();
        wgmma_fence_operand(acc);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      if constexpr (TIMELINE) stamp(it, 2);
      if (prev >= 0) release(prev);
    }

    if (p.argmin_out) {
      // ---- row arg-min: running (best, index[, second]) of the thread's two rows over its columns, in column order
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int row = m0 + r0 + 8 * i;
        const float x2 = row < M_eff ? __ldg(p.row_sq + row) : 0.f;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int col = n0 + 8 * j + c0 + c;
            if (col < p.N) {
              const float a = acc[4 * j + 2 * i + c];
              const float c2 = __ldg(p.col_sq + col);
              // pass 1 of the screened arg-min: the row norm is common to every column; ties and near-ties are settled
              // by the exact pass, so only the margin matters.  Exact mode: the reference's expression order,
              // (sum x^2 - 2 x.c) + sum c^2
              const float d = screen ? fmaf(m2a, a, c2) : (x2 - 2.0f * (p.alpha * a)) + c2;
              second[i] = fminf(second[i], fmaxf(d, best[i]));
              if (d < best[i]) { best[i] = d; best_idx[i] = col; }
            }
          }
        }
      }
      if (it.last_n()) {
        const float cm2 = screen ? __ldg(p.screen_cmax2) : 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          // merge the four lanes of a row: smaller distance wins, equal distances -> smaller index
          // (== first minimum over the whole row, as torch.min returns)
#pragma unroll
          for (int off = 1; off <= 2; off <<= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best[i], off);
            const int oi = __shfl_xor_sync(0xffffffffu, best_idx[i], off);
            const float os = __shfl_xor_sync(0xffffffffu, second[i], off);
            // second best of the merged set: the smaller of the two seconds and the larger of the two bests
            second[i] = fminf(fminf(second[i], os), fmaxf(best[i], ob));
            if (ob < best[i] || (ob == best[i] && oi < best_idx[i])) { best[i] = ob; best_idx[i] = oi; }
          }
          const int row = m0 + r0 + 8 * i;
          const bool row_ok = row < M_eff;
          if ((lane & 3) == 0 && row_ok) p.argmin_out[p.row_map ? __ldg(p.row_map + row) : row] = best_idx[i];
          if (screen) {
            // rows whose margin does not clear the error bound of the single-product pass are queued for the exact pass
            // (NaNs fail the comparison and are queued too); one atomicAdd per warp
            const float x2 = row_ok ? __ldg(p.row_sq + row) : 0.f;
            const float tau = p.screen_rel * sqrtf(x2 * cm2) + p.screen_abs * (x2 + cm2) + 1e-12f;
            const bool redo = (lane & 3) == 0 && row_ok && !(second[i] - best[i] > tau);
            const unsigned mask = __ballot_sync(0xffffffffu, redo);
            if (mask != 0u) {
              const int leader = __ffs(mask) - 1;
              int base = 0;
              if (lane == leader) base = atomicAdd(p.screen_count, __popc(mask));
              base = __shfl_sync(0xffffffffu, base, leader);
              if (redo) p.screen_rows[base + __popc(mask & ((1u << lane) - 1u))] = p.screen_row0 + row;
            }
          }
          best[i] = INFINITY;
          second[i] = INFINITY;
          best_idx[i] = 0;
        }
      }
    } else if constexpr (FP8) {
      const uint32_t row_inv = smem_base + S::kRowScaleOffset + wg * 64 * 4;
      if (p.out8) gemm_row_scales_e4m3<BN>(p, acc, m0, n0, r0, c0, wg, M_eff, row_inv);
      gemm_epilogue_rows<BN, true>(p, acc, epi_stage, m0 + wg * 64, n0, M_eff, 1 + wg, vec_r, vec32, vec16, row_inv);
    } else if constexpr (EPI == kEpiBiasResidF32) {
      if (m0 + wg * 64 < M_eff)
        gemm_epilogue_resid_tma<BN, NB>(p, acc, epi_stage, rfree_bar + wg * NB, rdone_bar + wg * NB, rp, n0);
    } else if constexpr (EPI != kEpiGeneral) {
      gemm_epilogue_f16_tma<BN, EPI>(p, acc, &tmC, epi_stage, m0 + wg * 64, n0, M_eff, 1 + wg);
    } else {
      gemm_epilogue_rows<BN>(p, acc, epi_stage, m0 + wg * 64, n0, M_eff, 1 + wg, vec_r, vec32, vec16);
    }
    if constexpr (TIMELINE) stamp(it, 3);
  }
  // the last tile's TMA stores complete (and stop reading the staging tile) before the CTA exits
  if constexpr (gemm_epi_tma_store(EPI))
    if ((threadIdx.x & 127) == 0) tma_store_wait<0>();
  // the peer may still arrive on this CTA's barriers: neither CTA leaves before both are done
  if constexpr (CLUSTER == 2) cluster_sync_all();
}

}  // namespace thmr
