// Several linear layers of an encoder layer in ONE persistent launch (wgmma, 128 x 256 tiles per CTA).
//
// Why.  Launched one by one (gemm2.cu), every linear layer pays its own tile quantisation and a kernel boundary (the
// tail imbalance of the last round + the prologue + the first TMA round trip).  Here the tiles of out-proj, FFN1, FFN2
// and the NEXT layer's QKV projection (or the output head) form one list of 256 x 256 tiles walked in order by CTA pairs
// (CTA 2 c + r of pair c owns rows [128 r, 128 r + 128) of each of the pair's tiles); the smem ring and the warp roles
// simply keep running across phase boundaries.
//
// Dependencies.  Phase p + 1 reads, as its A operand, rows that phase p writes.  Tiles are ordered row-pair-major
// inside a phase; when a CTA's half of a tile is in memory it bumps a per-(phase, row-pair) counter, and the TMA
// producer of a consuming tile spins on that counter (acquire) before it issues the first load of the tile.
// All CTAs are co-resident (grid <= SM count, checked at start-up with the occupancy API), walk their tiles in increasing
// global index and publish every tile before they start the MMAs of the next one, and a tile only ever waits for tiles of
// LOWER index: no deadlock.  The producer (thread 0, also an MMA thread) therefore only ever blocks on a counter at the
// start of a tile; while the MMAs of a tile run it prefetches the next tile's operands only if their counter is ready.
//
//   all warps:      TMA stores -> cp.async.bulk.wait_group 0 (lane 0) -> CTA barrier
//   thread 0:       fence.proxy.async -> __threadfence -> atomicAdd(counter)
//   consumer TMA:   ld.acquire.gpu(counter) >= target -> fence.proxy.async -> cp.async.bulk.tensor loads
//   epilogue reads of activations written in this launch use ld.global.cg
//
// Epilogue.  Two warpgroups; warpgroup j holds the accumulator of the tile's columns [128 j, 128 j + 128) (two m64 halves,
// interleaved so that warp w owns rows 32 w .. 32 w + 31; k-block sums of the tensor cores added up in fp32 registers,
// see mma_kblock_promoted).  A tile of a phase with a residual (out-proj, FFN2)
// is cut into 32-column slices, four per warp: bias, the residual LayerNorm(v) re-derived from v's bf16 planes (coalesced
// loads transposed through the warp's 4 KB staging tile, the next slice's block prefetched into registers), partial row
// statistics, one store of both bf16 planes through 64-byte-swizzled boxes.  A tile of a planes-only phase (FFN1, QKV) is
// cut into 64-column pairs, two per warp: folded-LayerNorm scale / shift, bias, GELU (branch-free rational erf), hi plane
// then lo plane through 128-byte-swizzled boxes.  Per-column constants are loaded once per tile into registers and
// handed out by shuffle.  Shared memory: 2 operand stages x 96 KB (A and W, hi + lo), 8 x 4 KB staging tiles.
#include <type_traits>

#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "kernels.h"

namespace cmdi {

namespace {

constexpr int kBlockM = 128;  // per CTA; 256 per pair
constexpr int kBlockN = 256;
constexpr int kBlockK = 64;
constexpr int kNumEpiWarps = 8;  // two warpgroups; the slice / pair assignment below is written for two warps per row group
constexpr int kWarpsPerLaneGroup = kNumEpiWarps / 4;
constexpr int kNumThreads = kNumEpiWarps * 32;
constexpr int kStages = 2;
constexpr int kPlaneBytes = kBlockM * kBlockK * 2;   // one bf16 plane of a 128-row x 64-column operand block = 16 KB
constexpr int kWPlaneBytes = kBlockN * kBlockK * 2;  // one bf16 plane of the 256-row W block = 32 KB
constexpr int kStageBytes = 2 * (kPlaneBytes + kWPlaneBytes);
constexpr int kSlices = kBlockN / 32;                // 32-column slices per tile
constexpr int kPartN = kBlockN / 2;                  // columns per warpgroup

struct __align__(8) ChainBarriers {
  uint64_t full[kStages], empty[kStages];
};

constexpr int kSmemBytes = 1024 + kStages * kStageBytes + kNumEpiWarps * kEpiStageBytes + (int)sizeof(ChainBarriers) +
                           kMaxChainPhases * (int)sizeof(ChainPhaseInfo);
static_assert(kSmemBytes <= 232448, "shared memory budget");

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// Bounded like mbar_wait: a protocol bug must trap, not hang the GPU (and, like it, without a printf: see mbar_wait).
__device__ __forceinline__ void wait_counter(const int* ctr, int target) {
  if (ld_acquire_gpu(ctr) >= target) return;
  const long long t0 = clock64();
  while (ld_acquire_gpu(ctr) < target) {
    __nanosleep(32);
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}

// Partial LayerNorm statistics: every epilogue warp Chan-combines the (mean, M2) of its slices of a tile in registers and
// publishes ONE partial per row, so a 512-wide row has kRowPartials = (512 / 256) * kWarpsPerLaneGroup partials of
// 512 / kRowPartials columns each.
static_assert(kSlices % kWarpsPerLaneGroup == 0, "equal column counts per partial");
constexpr int kRowPartials = 2 * kWarpsPerLaneGroup;
constexpr int kPartialStride = 16;  // float2 per row in the statistics arrays (engine.cu allocates 16)

// (mean, rstd) of a 512-wide row from its partial statistics (Chan et al. parallel combination, equal counts; fp32)
__device__ __forceinline__ float2 combine_row_stats(const float2* partials_row) {
  float m[kRowPartials], q = 0.f, s = 0.f;
#pragma unroll
  for (int i = 0; i < kRowPartials / 2; ++i) {
    const uint4 a = ld_global_cg_v4(partials_row + 2 * i);
    m[2 * i] = __uint_as_float(a.x);
    m[2 * i + 1] = __uint_as_float(a.z);
    q += __uint_as_float(a.y) + __uint_as_float(a.w);
  }
#pragma unroll
  for (int i = 0; i < kRowPartials; ++i) s += m[i];
  const float mean = s * (1.0f / kRowPartials);
  float dev = 0.f;
#pragma unroll
  for (int i = 0; i < kRowPartials; ++i) {
    const float d = m[i] - mean;
    dev = fmaf(d, d, dev);
  }
  const float var = (q + (512.0f / kRowPartials) * dev) * (1.0f / 512.0f);
  return make_float2(mean, rsqrtf(var + 1e-5f));  // nn.LayerNorm default eps, as nn.TransformerEncoderLayer uses it
}

// hi and lo planes of a 32-row x 32-column block (thread `lane` holds row `lane` as 16 bf16x2 words per plane) through
// the warp's staging tile as two {64 B x 32 rows} boxes with the 64-byte swizzle (16-byte chunk c of row r sits at
// chunk c ^ ((r >> 1) & 3): conflict-free for a row-per-lane writer), one bulk tensor store each.
__device__ __forceinline__ void store_planes_tma(uint32_t stage, int lane, const uint32_t (&hw)[16], const uint32_t (&lw)[16],
                                                 const CUtensorMap* map_hi, const CUtensorMap* map_lo, bool with_lo, int col, int row) {
  if (lane == 0) tma_store_wait_read();
  __syncwarp();
  const uint32_t sw = (uint32_t)(lane >> 1) & 3u;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    st_shared_v4(stage + lane * 64 + ((c ^ sw) << 4), hw[c * 4], hw[c * 4 + 1], hw[c * 4 + 2], hw[c * 4 + 3]);
    if (with_lo) st_shared_v4(stage + 2048 + lane * 64 + ((c ^ sw) << 4), lw[c * 4], lw[c * 4 + 1], lw[c * 4 + 2], lw[c * 4 + 3]);
  }
  fence_proxy_async_smem();
  __syncwarp();
  if (lane == 0) {
    tma_store_2d(map_hi, stage, col, row);
    if (with_lo) tma_store_2d(map_lo, stage + 2048, col, row);
    tma_store_commit();
  }
}

// erf(x) as a rational function of the clamped argument (numerator degree 13, denominator degree 8 in x; max abs error
// 3.7e-7 over the real line, checked against math.erf in tests/test_host_logic.py): branch-free, 14 FMAs + one division.
// The FFN1 epilogue is issue-bound and CUDA's erff (two polynomial branches + exp) was its largest single item (8 % of
// the chain kernel's samples); |GELU error| <= 6.4e-7 against 2^-17 ~ 7.6e-6 relative of the bf16x3 products around it.
__device__ __forceinline__ float erf_rational(float x) {
  x = fminf(fmaxf(x, -4.0f), 4.0f);
  const float x2 = x * x;
  float p = -2.72614225801306e-10f;
  p = fmaf(p, x2, 2.77068142495902e-08f);
  p = fmaf(p, x2, -2.10102402082508e-06f);
  p = fmaf(p, x2, -5.69250639462346e-05f);
  p = fmaf(p, x2, -7.34990630326855e-04f);
  p = fmaf(p, x2, -2.95459980854025e-03f);
  p = fmaf(p, x2, -1.60960333262415e-02f);
  float q = -1.45660718464996e-05f;
  q = fmaf(q, x2, -2.13374055278905e-04f);
  q = fmaf(q, x2, -1.68282697438203e-03f);
  q = fmaf(q, x2, -7.37332916720468e-03f);
  q = fmaf(q, x2, -1.42647390514189e-02f);
  return __fdividef(x * p, q);
}
__device__ __forceinline__ float gelu_fast(float x) { return 0.5f * x * (1.0f + erf_rational(x * 0.70710678118654752440f)); }

constexpr int kSlicesPerWarp = (kSlices + kWarpsPerLaneGroup - 1) / kWarpsPerLaneGroup;  // of one tile

struct RowStats {   // per-tile cache of what this thread needs for its slices of the tile
  float2 fold, ln;                 // (mean, rstd) of its row: folded LayerNorm of the A operand / LayerNorm of the residual
  // Per-COLUMN constants (bias, folded-LN c, LayerNorm gamma / beta of the residual): lane l holds column l of the warp's
  // k-th slice of the tile, loaded with one coalesced request per vector before the tile's accumulator wait
  // (load_tile_constants) and handed out by shuffle.  History: fetched at the point of use they were ~15 % of this kernel's
  // stall samples (an L2 round trip costs 2-3 us under this load); loaded per tile but one predicated load at a time, 11 %.
  // (Per slice, one slice ahead, in 4 registers instead of 16: slower, 154.6 -> 161.6 us per launch.)
  float bias[kSlicesPerWarp], c[kSlicesPerWarp], g[kSlicesPerWarp], b[kSlicesPerWarp];
  float run_mean, run_m2;          // running statistics of this thread's output row over the warp's slices of the tile
};
__device__ __forceinline__ float pick(const float (&a)[kSlicesPerWarp], int k) {
  float v = a[0];
#pragma unroll
  for (int i = 1; i < kSlicesPerWarp; ++i) v = (k == i) ? a[i] : v;
  return v;
}

// Start of a tile for one epilogue warp: per-column constants of its four 32-column slices and the statistics of its row.
// Warp group j (= warp_in_group) owns the slices 4 j .. 4 j + 3 (in the `wide` phases: the 64-column pairs 2 j, 2 j + 1).
__device__ __forceinline__ int warp_slice(int k, int warp_in_group, bool /*wide*/) { return warp_in_group * kSlicesPerWarp + k; }
// The constants do not depend on anything computed in this launch: they are requested BEFORE the warp waits for the tile's
// accumulator, all loads of a vector in flight together (indices clamped instead of predicated; measured before: one
// predicated load at a time, each followed by the spill of its result, was 11 % of this kernel's stall samples).
__device__ __forceinline__ void load_tile_constants(const LinearParams& p, RowStats& rs, int n_blk, int warp_in_group, bool wide, int lane) {
  int idx[kSlicesPerWarp];
  bool ok[kSlicesPerWarp];
#pragma unroll
  for (int k = 0; k < kSlicesPerWarp; ++k) {
    const int sl = warp_slice(k, warp_in_group, wide);
    const int n = n_blk * kBlockN + sl * 32 + lane;
    ok[k] = sl < kSlices && n < p.N;
    idx[k] = ok[k] ? n : 0;
  }
  const bool ln = p.ln_src || p.ln_src_hi;
  float t[4][kSlicesPerWarp];
#pragma unroll
  for (int k = 0; k < kSlicesPerWarp; ++k) {
    t[0][k] = p.bias ? __ldg(p.bias + idx[k]) : 0.f;
    t[1][k] = p.fold_stats ? __ldg(p.fold_c + idx[k]) : 0.f;
    t[2][k] = ln ? __ldg(p.ln_gamma + idx[k]) : 0.f;
    t[3][k] = ln ? __ldg(p.ln_beta + idx[k]) : 0.f;
  }
#pragma unroll
  for (int k = 0; k < kSlicesPerWarp; ++k) {
    rs.bias[k] = ok[k] ? t[0][k] : 0.f;
    rs.c[k] = ok[k] ? t[1][k] : 0.f;
    rs.g[k] = ok[k] ? t[2][k] : 0.f;
    rs.b[k] = ok[k] ? t[3][k] : 0.f;
  }
}
// ... and, once the accumulator (hence the producer phase's statistics) is there, the statistics of the thread's row
__device__ __forceinline__ void load_row_statistics(const LinearParams& p, RowStats& rs, int row) {
  if (p.fold_stats) rs.fold = combine_row_stats(p.fold_stats + (size_t)row * kPartialStride);
  if (p.ln_partials) rs.ln = combine_row_stats(p.ln_partials + (size_t)row * kPartialStride);
  rs.run_mean = 0.f; rs.run_m2 = 0.f;
}

// A 64-column pair of slices of a phase that writes planes only (FFN1, QKV): one accumulator read, one pass of math over
// 64 values and two {128 B x 32 rows} plane stores -- half the per-slice synchronisation (accumulator transpose, staging-tile
// turn-around, proxy fence) per column of the 32-column path, which needs its registers for the residual instead.
__device__ __forceinline__ void epilogue_pair(const LinearParams& p, const ChainPhaseDesc& pd, const float (&acc0)[kPartN / 2],
                                              const float (&acc1)[kPartN / 2], int m_blk, int n_blk, int pair, int k2, int lane_group,
                                              int lane, uint32_t stage, const RowStats& rs) {
  const int n0 = n_blk * kBlockN + pair * 64;
  if (n0 >= p.N) return;  // warp-uniform
  const int warp_row0 = m_blk * kBlockM + lane_group * 32;
  if (lane == 0) tma_store_wait_read();  // the staging tile is about to be rewritten
  uint32_t v[64];
  acc_rows_to_lanes(acc0, acc1, k2 * 8, stage, lane, *reinterpret_cast<uint32_t(*)[32]>(&v[0]));
  acc_rows_to_lanes(acc0, acc1, k2 * 8 + 4, stage, lane, *reinterpret_cast<uint32_t(*)[32]>(&v[32]));
  float f[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) f[j] = __uint_as_float(v[j]);
  if (p.fold_stats) {
    const float nm = -rs.fold.x, c0 = pick(rs.c, 2 * k2), c1 = pick(rs.c, 2 * k2 + 1);
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      f[j] = __fmaf_rn(nm, __shfl_sync(0xffffffffu, c0, j), f[j]) * rs.fold.y;
      f[32 + j] = __fmaf_rn(nm, __shfl_sync(0xffffffffu, c1, j), f[32 + j]) * rs.fold.y;
    }
  }
  if (p.bias) {
    const float b0 = pick(rs.bias, 2 * k2), b1 = pick(rs.bias, 2 * k2 + 1);
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      f[j] += __shfl_sync(0xffffffffu, b0, j);
      f[32 + j] += __shfl_sync(0xffffffffu, b1, j);
    }
  }
  if (p.act == 1) {
#pragma unroll
    for (int j = 0; j < 64; ++j) f[j] = gelu_fast(f[j]);
  }
  // hi plane first, the remainders stay in f (same arithmetic as split_bf16x2, 96 instead of 128 live registers)
  uint32_t w[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
    w[j] = *reinterpret_cast<const uint32_t*>(&h);
    f[2 * j] -= __uint_as_float(w[j] << 16);
    f[2 * j + 1] -= __uint_as_float(w[j] & 0xffff0000u);
  }
  store_block_tma(stage, lane, w, &pd.o_hi, n0, warp_row0);
  if (p.nsplit_out == 3) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const __nv_bfloat162 l = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
      w[j] = *reinterpret_cast<const uint32_t*>(&l);
    }
    store_block_tma(stage, lane, w, &pd.o_lo, n0, warp_row0);
  }
}

// One 32-column slice of a 128-row accumulator: fragments -> row-per-thread registers -> [folded LayerNorm] -> bias -> [residual] ->
// [partial statistics] -> [GELU] -> fp32 rows and/or bf16 hi/lo planes.
__device__ __forceinline__ void epilogue_slice(const LinearParams& p, const ChainPhaseDesc& pd, const float (&acc0)[kPartN / 2],
                                               const float (&acc1)[kPartN / 2], int m_blk, int n_blk, int slice, int k_in_tile, int lane_group, int lane, uint32_t stage, RowStats& rs, uint4 (&rv)[8],
                                               bool& rv_ready, int next_slice, int warp_in_group, long long* dbg) {
  long long t0 = clock64(), t1;
#define CMDI_T(i) do { if (dbg) { t1 = clock64(); dbg[i] += t1 - t0; t0 = t1; } } while (0)
  const int warp_row0 = m_blk * kBlockM + lane_group * 32;
  const int row = warp_row0 + lane;
  const int n0 = n_blk * kBlockN + slice * 32;
  if (n0 >= p.N) return;  // warp-uniform: columns beyond the layer's width (output head)
  const float* res_src = p.residual ? p.residual : p.ln_src;
  const bool res_planes = p.ln_src_hi != nullptr;  // LayerNorm's input as bf16 hi / lo planes instead of fp32 rows
  const bool has_res = res_src || res_planes;
  // the staging tile is about to be rewritten (residual fetch or stores): the bulk store issued from it has been read out
  CMDI_T(8);   // row statistics
  if (lane == 0) tma_store_wait_read();
  __syncwarp();
  CMDI_T(9);   // staging free
  const long long res_ld = p.residual ? p.ld_res : p.ld_ln;
  // Residual block of 32 rows x 32 columns, fetched coalesced into rv: fp32 rows (8 x 16 B per thread, 4 complete 128 B
  // row segments per instruction) or the two bf16 planes (4 + 4 x 16 B, 8 complete 64 B segments per instruction).
  // Under this kernel's load an L2 round trip costs ~2 us, so the block of the warp's NEXT slice of the same tile is
  // requested while this one is processed (below); only a tile's first slice pays the latency here.
  auto fetch_residual = [&](int n) {
    if (res_planes) {
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const long long off = (long long)(warp_row0 + it * 8 + (lane >> 2)) * p.ld_ln + n + (lane & 3) * 8;
        rv[it] = ld_global_cg_v4(p.ln_src_hi + off);
        rv[4 + it] = ld_global_cg_v4(p.ln_src_lo + off);
      }
    } else {
#pragma unroll
      for (int it = 0; it < 8; ++it)
        rv[it] = ld_global_cg_v4(res_src + (long long)(warp_row0 + it * 4 + (lane >> 3)) * res_ld + n + (lane & 7) * 4);
    }
  };
  if (has_res && !rv_ready) fetch_residual(n0);
  rv_ready = false;
  uint32_t v[32];
  acc_rows_to_lanes(acc0, acc1, k_in_tile * 4, stage, lane, v);
  CMDI_T(10);  // residual loads issued + accumulator read
  float f[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(v[j]);
  if (p.fold_stats) {
    // acc = v (W.gamma)^T  ->  rstd * (acc - mean * c[n]);  the bias added next carries W beta + b
    const float nm = -rs.fold.x, ck = pick(rs.c, k_in_tile);
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = __fmaf_rn(nm, __shfl_sync(0xffffffffu, ck, j), f[j]) * rs.fold.y;
  }
  if (p.bias) {
    const float bk = pick(rs.bias, k_in_tile);
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] += __shfl_sync(0xffffffffu, bk, j);
  }
  if (has_res) {
    // transpose through the staging tile: every thread gets its own row
    if (res_planes) {
      // hi block at +0, lo block at +2048, 64 B rows, 16 B chunk c of row r at chunk c ^ ((r >> 1) & 3)
#pragma unroll
      for (int it = 0; it < 4; ++it) {
        const int rr = it * 8 + (lane >> 2);
        const uint32_t a = stage + rr * 64 + ((((uint32_t)lane & 3u) ^ (((uint32_t)rr >> 1) & 3u)) << 4);
        st_shared_v4(a, rv[it].x, rv[it].y, rv[it].z, rv[it].w);
        st_shared_v4(a + 2048, rv[4 + it].x, rv[4 + it].y, rv[4 + it].z, rv[4 + it].w);
      }
    } else {
      const int c = lane & 7;
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int rr = it * 4 + (lane >> 3);
        st_shared_v4(stage + rr * 128 + ((c ^ (rr & 7)) << 4), rv[it].x, rv[it].y, rv[it].z, rv[it].w);
      }
    }
    if (next_slice >= 0 && n_blk * kBlockN + next_slice * 32 < p.N) {
      // the registers are free again: request the residual block of this warp's next slice (same tile, same rows)
      fetch_residual(n_blk * kBlockN + next_slice * 32);
      rv_ready = true;
    }
    __syncwarp();
    const float gk = pick(rs.g, k_in_tile), btk = pick(rs.b, k_in_tile);
    if (res_planes) {
      const uint32_t sw = ((uint32_t)lane >> 1) & 3u;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const uint4 uh = ld_shared_v4(stage + lane * 64 + (((uint32_t)c ^ sw) << 4));
        const uint4 ul = ld_shared_v4(stage + 2048 + lane * 64 + (((uint32_t)c ^ sw) << 4));
        const uint32_t hw[4] = {uh.x, uh.y, uh.z, uh.w}, lw[4] = {ul.x, ul.y, ul.z, ul.w};
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          const int j = c * 8 + w * 2;
          const float x0 = __uint_as_float(hw[w] << 16) + __uint_as_float(lw[w] << 16);
          const float x1 = __uint_as_float(hw[w] & 0xffff0000u) + __uint_as_float(lw[w] & 0xffff0000u);
          f[j] += ln_apply(x0, rs.ln.x, rs.ln.y, __shfl_sync(0xffffffffu, gk, j), __shfl_sync(0xffffffffu, btk, j));
          f[j + 1] += ln_apply(x1, rs.ln.x, rs.ln.y, __shfl_sync(0xffffffffu, gk, j + 1), __shfl_sync(0xffffffffu, btk, j + 1));
        }
      }
    } else {
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const uint4 u = ld_shared_v4(stage + lane * 128 + ((g ^ (lane & 7)) << 4));
        if (p.ln_src) {
          // residual = LayerNorm(ln_src) re-derived from its fp32 input, the row statistics and gamma / beta
          f[g * 4 + 0] += ln_apply(__uint_as_float(u.x), rs.ln.x, rs.ln.y, __shfl_sync(0xffffffffu, gk, g * 4 + 0), __shfl_sync(0xffffffffu, btk, g * 4 + 0));
          f[g * 4 + 1] += ln_apply(__uint_as_float(u.y), rs.ln.x, rs.ln.y, __shfl_sync(0xffffffffu, gk, g * 4 + 1), __shfl_sync(0xffffffffu, btk, g * 4 + 1));
          f[g * 4 + 2] += ln_apply(__uint_as_float(u.z), rs.ln.x, rs.ln.y, __shfl_sync(0xffffffffu, gk, g * 4 + 2), __shfl_sync(0xffffffffu, btk, g * 4 + 2));
          f[g * 4 + 3] += ln_apply(__uint_as_float(u.w), rs.ln.x, rs.ln.y, __shfl_sync(0xffffffffu, gk, g * 4 + 3), __shfl_sync(0xffffffffu, btk, g * 4 + 3));
        } else {
          f[g * 4 + 0] += __uint_as_float(u.x); f[g * 4 + 1] += __uint_as_float(u.y);
          f[g * 4 + 2] += __uint_as_float(u.z); f[g * 4 + 3] += __uint_as_float(u.w);
        }
      }
    }
  }
  CMDI_T(11);  // fold + bias + residual
  if (p.stats_out) {
    // LayerNorm statistics of this thread's 32 output values (two-pass in registers), merged into the running pair of
    // the warp's earlier slices of this tile; the warp's last slice of the tile publishes the partial
    float sm = 0.f;
#pragma unroll
    for (int j = 0; j < 32; j += 4) sm += (f[j] + f[j + 1]) + (f[j + 2] + f[j + 3]);
    const float mean32 = sm * (1.0f / 32.0f);
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const float a = f[j] - mean32;
      q = fmaf(a, a, q);
    }
    // Chan's update with n_a = 32 k, n_b = 32: n_b / n_ab = 1 / (k + 1), n_a n_b / n_ab = 32 k / (k + 1)
    const float inv = k_in_tile == 0 ? 1.0f : k_in_tile == 1 ? 0.5f : k_in_tile == 2 ? (1.0f / 3.0f) : 0.25f;
    static_assert(kSlicesPerWarp <= 4, "reciprocal table");
    const float delta = mean32 - rs.run_mean;
    rs.run_mean += delta * inv;
    rs.run_m2 += q + delta * delta * (32.0f * (float)k_in_tile * inv);
    if (k_in_tile == kSlicesPerWarp - 1)
      p.stats_out[(size_t)row * kPartialStride + n_blk * kWarpsPerLaneGroup + warp_in_group] = make_float2(rs.run_mean, rs.run_m2);
  }
  if (p.act == 1) {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = gelu_fast(f[j]);
  }
  CMDI_T(12);  // statistics + activation
  if (p.out_f32) {
    uint32_t w[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) w[j] = __float_as_uint(f[j]);
    if (p.tma_store) {
      store_block_tma(stage, lane, w, &pd.o_f32, n0, warp_row0);
    } else {
      // row-mapped fp32 output (output head: sequence rows -> frame rows, token row dropped): masked coalesced stores
      RowSlots rows;
      rows.ok = 0;
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        int pos_unused;
        long long r;
        if (map_row(p, warp_row0 + it * 4 + (lane >> 3), r, pos_unused)) rows.ok |= 1u << it;
        rows.row[it] = (int)r;
      }
      store_block_coalesced(stage, lane, w, reinterpret_cast<char*>(p.out_f32 + n0), rows, (long long)p.ld_f32 * 4, (p.N - n0) / 4, 1, 0);
    }
  }
  CMDI_T(13);  // fp32 store
  if (p.out_hi) {
    uint32_t hw[16], lw[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) split_bf16x2(f[2 * j], f[2 * j + 1], hw[j], lw[j]);
    store_planes_tma(stage, lane, hw, lw, &pd.o_hi, &pd.o_lo, p.nsplit_out == 3, n0, warp_row0);
  }
  CMDI_T(14);  // plane stores
#undef CMDI_T
}

// The operand stream of one CTA (thread 0): k-block after k-block of its tiles, one ring stage each.
template <int NSPLIT>
struct ChainProducer {
  const ChainPhaseDesc* phases;
  const ChainPhaseInfo* info;
  uint8_t* ring;
  ChainBarriers* bars;
  int cluster_id, num_clusters, rank, my_tiles;
  int seq, kb, ph, stage;
  uint32_t phase;
  int issued;  // k-blocks issued so far

  // Issues the next k-block.  blocking = false: only if the tile's dependency counter (first k-block) is already
  // satisfied and both warpgroups have released the stage; returns false then without issuing, and the caller retries
  // later instead of waiting for the other warpgroup.
  __device__ bool issue_next(bool blocking) {
    if (seq >= my_tiles) return false;
    const int tile = cluster_id + seq * num_clusters;
    while (tile >= info[ph].tile_end) ++ph;
    const ChainPhaseInfo& pi = info[ph];
    const ChainPhaseDesc& pd = phases[ph];
    const int local = tile - pi.tile_begin;
    const int m_pair = local / pi.num_n_blocks;
    const int m_blk = 2 * m_pair + rank;
    const int n_blk = local % pi.num_n_blocks;
    if (kb == 0 && pi.wait_ctr) {
      // the A rows of this row pair are written by an earlier phase of this launch
      if (!blocking && ld_acquire_gpu(pi.wait_ctr + m_pair) < pi.wait_target) return false;
      wait_counter(pi.wait_ctr + m_pair, pi.wait_target);
      fence_proxy_async_all();
    }
    constexpr int nplanes = (NSPLIT == 3) ? 2 : 1;
    if (!blocking && !mbar_test_wait(&bars->empty[stage], phase ^ 1)) return false;
    mbar_wait(&bars->empty[stage], phase ^ 1);
    uint8_t* da = ring + (size_t)stage * kStageBytes;
    uint8_t* dw = da + 2 * kPlaneBytes;
    if (pi.p.debug & 4) {
      // bring-up decomposition (CMDI_DEBUG=4): no operand loads, only the pipeline bookkeeping
      mbar_arrive(&bars->full[stage]);
    } else {
      mbar_arrive_expect_tx(&bars->full[stage], nplanes * (kPlaneBytes + kWPlaneBytes));
      const int kc = kb * kBlockK;
      tma_load_2d(da, &pd.a_hi, &bars->full[stage], kc, m_blk * kBlockM);
      tma_load_2d(dw, &pd.w_hi, &bars->full[stage], kc, n_blk * kBlockN);
      tma_load_2d(dw + kWPlaneBytes / 2, &pd.w_hi, &bars->full[stage], kc, n_blk * kBlockN + kBlockN / 2);
      if constexpr (nplanes == 2) {
        tma_load_2d(da + kPlaneBytes, &pd.a_lo, &bars->full[stage], kc, m_blk * kBlockM);
        tma_load_2d(dw + kWPlaneBytes, &pd.w_lo, &bars->full[stage], kc, n_blk * kBlockN);
        tma_load_2d(dw + kWPlaneBytes + kWPlaneBytes / 2, &pd.w_lo, &bars->full[stage], kc, n_blk * kBlockN + kBlockN / 2);
      }
    }
    if (++stage == kStages) { stage = 0; phase ^= 1; }
    if (++kb == pi.num_k_blocks) { kb = 0; ++seq; }
    ++issued;
    return true;
  }
};

// NSPLIT (1 or 3: the bf16 products per MMA, as LinearParams::nsplit; every phase of a launch has the same) is a
// template parameter so that mma_kblock_promoted's term loop has a constant trip count: with a runtime count its early
// exit puts the wgmmas on a divergent path, and ptxas then serialises all of them (C7520).
template <int NSPLIT>
__global__ void __launch_bounds__(kNumThreads, 1)
linear_chain_kernel(const ChainPhaseDesc* __restrict__ phases, const int num_phases, const int total_tiles, long long* dbg) {
  // dbg (bring-up, CMDI_CHAIN_DBG=1): [gridDim.x][kMaxChainPhases][16] counters per CTA and phase, thread 0:
  //   0 tiles  1 dependency wait at the tile start  2 blocking refills inside the mainloop  3 operand wait (full barriers)
  //   4 MMA issue + promotion (the rest of the mainloop)  5 mainloop  6 epilogue  7 publish wait
  long long* dbg_me = dbg ? dbg + (size_t)blockIdx.x * kMaxChainPhases * 16 : nullptr;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* ring = smem;
  uint8_t* epi_stage = ring + kStages * kStageBytes;  // kNumEpiWarps x 4 KB store-staging tiles
  ChainBarriers* bars = reinterpret_cast<ChainBarriers*>(epi_stage + kNumEpiWarps * kEpiStageBytes);
  ChainPhaseInfo* info = reinterpret_cast<ChainPhaseInfo*>(bars + 1);

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int rank = (int)(blockIdx.x & 1);
  const int cluster_id = blockIdx.x >> 1;
  const int num_clusters = gridDim.x >> 1;
  const int my_tiles = (total_tiles - cluster_id + num_clusters - 1) / num_clusters;
  const bool is_producer = threadIdx.x == 0;

  // phase descriptors (all but the tensor maps) into shared memory: every role reads them per tile
  for (int i = threadIdx.x; i < num_phases * (int)(sizeof(ChainPhaseInfo) / 4); i += kNumThreads) {
    const int ph = i / (int)(sizeof(ChainPhaseInfo) / 4), w = i % (int)(sizeof(ChainPhaseInfo) / 4);
    reinterpret_cast<uint32_t*>(info + ph)[w] = reinterpret_cast<const uint32_t*>(&phases[ph].info)[w];
  }
  if (is_producer) {
    for (int ph = 0; ph < num_phases; ++ph) {
      tma_prefetch_desc(&phases[ph].a_hi);
      tma_prefetch_desc(&phases[ph].w_hi);
    }
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&bars->full[s], 1);
      mbar_init(&bars->empty[s], kNumEpiWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  ChainProducer<NSPLIT> prod{phases, info, ring, bars, cluster_id, num_clusters, rank, my_tiles, 0, 0, 0, 0, 0u, 0};

  const int j3 = warp_idx >> 2;          // warpgroup = column half of the tile
  const int lane_group = warp_idx & 3;   // rows 32 * lane_group .. + 31 of the CTA's 128
  const uint32_t epi_stage_addr = smem_u32(epi_stage + warp_idx * kEpiStageBytes);
  const uint32_t w_off = 2 * kPlaneBytes + j3 * kPartN * 128;  // this warpgroup's W rows in a stage
  float acc0[kPartN / 2], acc1[kPartN / 2];
  RowStats rs{};
  int ph = 0, stage = 0, consumed = 0;
  uint32_t phase = 0;
  for (int seq = 0; seq < my_tiles; ++seq) {
    long long c0 = clock64();
    const int tile = cluster_id + seq * num_clusters;
    while (tile >= info[ph].tile_end) ++ph;
    const ChainPhaseInfo& pi = info[ph];
    const int local = tile - pi.tile_begin;
    const int m_blk = 2 * (local / pi.num_n_blocks) + rank;
    const int n_blk = local % pi.num_n_blocks;
    const bool wide = pi.wide != 0;
    load_tile_constants(pi.p, rs, n_blk, j3, wide, lane);
    // ---- mainloop ----
    // Thread 0 refills stages without blocking: a stage the other warpgroup still reads is retried after the next
    // sub-chunk's promotion (mma_kblock_body), so neither warpgroup waits for the other inside the k-block loop; thread 0
    // blocks only for the k-block the MMAs need next.  Every k-block's wgmmas have retired at its end: carrying the
    // fragment ring across the k-block boundary, over the barrier waits and thread 0's producer branch, makes ptxas
    // serialise every wgmma of the kernel (C7518).
    long long dep_wait = 0, issue_wait = 0, operand_wait = 0;  // thread 0's cycles (CMDI_CHAIN_DBG)
    auto refill = [&] {
      if (is_producer && prod.issued < consumed + kStages) prod.issue_next(false);
    };
    // The k-block loop exists twice, with and without MMAs (CMDI_CHAIN_SKIP=2), chosen once per tile: the same loop with
    // the MMAs behind a runtime test inside it puts them on a divergent path, and ptxas serialises them (C7520).
    auto mainloop = [&](auto with_mma) {
      for (int kb = 0; kb < pi.num_k_blocks; ++kb) {
        if (is_producer) {
          // every earlier tile of this CTA is published: blocking on a dependency counter is safe here
          const long long d0 = clock64();
          while (prod.issued <= consumed) prod.issue_next(true);
          (kb > 0 ? issue_wait : dep_wait) += clock64() - d0;
        }
        const long long d1 = clock64();
        mbar_wait(&bars->full[stage], phase);
        operand_wait += clock64() - d1;
        const uint32_t sa = smem_u32(ring + (size_t)stage * kStageBytes);
        if constexpr (decltype(with_mma)::value) {
          float t0[32], t1[32];
          mma_subchunk_issue<NSPLIT, false>(t0, sa, sa + w_off, kPlaneBytes, kWPlaneBytes, 0, 0);
          mma_kblock_body<kPartN, NSPLIT, false>(acc0, acc1, t0, t1, sa, sa + w_off, kPlaneBytes, kWPlaneBytes, refill);
          wgmma_wait<0>();
          mma_subchunk_promote(acc1, t1, kPartN / 64 - 1);
        }
        // the tensor cores have read this stage: it may be refilled
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars->empty[stage]);
        ++consumed;
        refill();
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
    };
#pragma unroll
    for (int i = 0; i < kPartN / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    if (!(pi.p.debug & 2))
      mainloop(std::true_type{});
    else
      mainloop(std::false_type{});
    long long c1 = clock64();
    // ---- epilogue ----
    load_row_statistics(pi.p, rs, m_blk * kBlockM + lane_group * 32 + lane);
    long long* dbg_w = (dbg_me && warp_idx == 0 && lane == 0) ? dbg_me + ph * 16 : nullptr;
    if (wide) {
#pragma unroll
      for (int k2 = 0; k2 < kSlicesPerWarp / 2; ++k2)
        epilogue_pair(pi.p, phases[ph], acc0, acc1, m_blk, n_blk, 2 * j3 + k2, k2, lane_group, lane, epi_stage_addr, rs);
    } else {
      uint4 rv[8];  // residual block in flight for this warp's next slice (see epilogue_slice)
      bool rv_ready = false;
#pragma unroll
      for (int k = 0; k < kSlicesPerWarp; ++k) {
        const int slice = warp_slice(k, j3, false);
        const int next_slice = k + 1 < kSlicesPerWarp ? slice + 1 : -1;
        epilogue_slice(pi.p, phases[ph], acc0, acc1, m_blk, n_blk, slice, k, lane_group, lane, epi_stage_addr, rs, rv, rv_ready,
                       next_slice, j3, nullptr);
      }
    }
    long long c2 = clock64();
    refill();  // a stage the other warpgroup was still reading at the end of the mainloop
    // ---- publish: everything this CTA stored for the tile is in memory, then one counter bump ----
    __syncwarp();  // the other lanes' plain stores (row-mapped outputs, partial statistics) before lane 0's wait
    if (lane == 0) tma_store_wait_all();
    __syncthreads();
    if (is_producer && pi.done_ctr) {
      fence_proxy_async_all();
      __threadfence();
      atomicAdd(pi.done_ctr + (tile - pi.tile_begin) / pi.num_n_blocks, 1);
    }
    if (dbg_w) {
      dbg_w[0] += 1;
      dbg_w[1] += dep_wait;
      dbg_w[2] += issue_wait;
      dbg_w[3] += operand_wait;
      dbg_w[4] += (c1 - c0) - dep_wait - issue_wait - operand_wait;
      dbg_w[5] += c1 - c0; dbg_w[6] += c2 - c1; dbg_w[7] += clock64() - c2;
    }
  }
}

}  // namespace

cudaError_t configure_linear_chain_kernel() {
  cudaError_t e = cudaFuncSetAttribute(linear_chain_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(linear_chain_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
}

// how many CTA pairs of the nsplit instance can be resident at once on the current device (they spin on each other's
// counters: the launch must never exceed this)
int linear_chain_max_clusters(int num_sms, int nsplit) {
  int per_sm = 0;
  const cudaError_t e = nsplit == 3
      ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, linear_chain_kernel<3>, kNumThreads, kSmemBytes)
      : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, linear_chain_kernel<1>, kNumThreads, kSmemBytes);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return per_sm * num_sms / 2;
}

cudaError_t launch_linear_chain(const ChainPhaseDesc* phases_dev, int num_phases, int total_tiles, int nsplit, int num_sms,
                                cudaStream_t stream, long long* dbg) {
  if (num_phases < 1 || num_phases > kMaxChainPhases || total_tiles < 1 || (nsplit != 1 && nsplit != 3)) {
    set_last_error("launch_linear_chain: bad phase list (%d phases, %d tiles, nsplit %d)", num_phases, total_tiles, nsplit);
    return cudaErrorInvalidValue;
  }
  static int max_clusters[2] = {-1, -1};  // [nsplit == 3]
  int& max_c = max_clusters[nsplit == 3];
  if (max_c < 0) max_c = linear_chain_max_clusters(num_sms, nsplit);
  int clusters = num_sms / 2;
  if (clusters > total_tiles) clusters = total_tiles;
  if (clusters > max_c) {
    set_last_error("launch_linear_chain: %d co-resident CTA pairs needed, the device offers %d", clusters, max_c);
    return cudaErrorInvalidConfiguration;
  }
  return launch_kernel(nsplit == 3 ? linear_chain_kernel<3> : linear_chain_kernel<1>, dim3(2 * clusters), dim3(kNumThreads),
                       (size_t)kSmemBytes, stream, phases_dev, num_phases, total_tiles, dbg);
}

}  // namespace cmdi
