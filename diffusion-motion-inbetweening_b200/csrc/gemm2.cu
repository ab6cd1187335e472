// Linear layers (and the UNet's 1-D convolutions) on Hopper tensor cores: one CTA per 128 x BLOCK_N output tile,
// persistent over the tile list.
//
// The W operand is loaded as two {64, BLOCK_N / 2} boxes (the tensor maps the engine builds for this kernel).
// Operands are bf16 (one plane, or hi/lo planes with nsplit = 3) or, in the F16 instantiations, one fp16 plane each
// (CMDI_PRECISION_FP16: CUDA autocast's arithmetic, see gemm_epilogue.cuh).
#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "kernels.h"

namespace cmdi {

namespace {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kNumMmaWarps = 8;
constexpr int kNumThreads = kNumMmaWarps * 32;
constexpr int kMaxStages = 8;
constexpr int kSmemLimit = 232448;
constexpr int kABytes = kBlockM * kBlockK * 2;

struct __align__(8) GemmBarriers {
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
};

// The operand stream of one CTA: k-block after k-block of its tiles, one ring stage each.  Driven by thread 0 only.
template <int BLOCK_N>
struct Producer {
  const CUtensorMap *a_hi, *a_lo, *w_hi, *w_lo;
  const LinearParams* p;
  uint8_t* ring;
  GemmBarriers* bars;
  uint32_t stage_bytes;
  int num_stages, num_tiles, num_n_blocks, num_k_blocks, kb_per_tap;
  int tile, kb, stage;
  uint32_t phase;

  __device__ void issue_next() {
    if (tile >= num_tiles) return;
    constexpr int kHalfN = BLOCK_N / 2;
    constexpr int kBBytes = BLOCK_N * kBlockK * 2;
    const int nplanes = (p->nsplit == 3) ? 2 : 1;
    const int m_blk = tile / num_n_blocks, n_blk = tile % num_n_blocks;
    mbar_wait(&bars->empty[stage], phase ^ 1);
    uint8_t* sa = ring + (size_t)stage * stage_bytes;
    uint8_t* sb = sa + nplanes * kABytes;
    if (p->debug & 4) {
      mbar_arrive(&bars->full[stage]);
    } else {
      mbar_arrive_expect_tx(&bars->full[stage], stage_bytes);
      int a_col = kb * kBlockK, w_col = a_col, a_row = m_blk * kBlockM;
      if (p->num_taps > 0) {
        const int tap = kb / kb_per_tap, kc = (kb - tap * kb_per_tap) * kBlockK;
        a_col = p->tap_a_col[tap] + kc; w_col = p->tap_w_col[tap] + kc; a_row += p->tap_row[tap];
      }
      tma_load_2d(sa, a_hi, &bars->full[stage], a_col, a_row);
      tma_load_2d(sb, w_hi, &bars->full[stage], w_col, n_blk * BLOCK_N);
      tma_load_2d(sb + kHalfN * 128, w_hi, &bars->full[stage], w_col, n_blk * BLOCK_N + kHalfN);
      if (nplanes == 2) {
        tma_load_2d(sa + kABytes, a_lo, &bars->full[stage], a_col, a_row);
        tma_load_2d(sb + kBBytes, w_lo, &bars->full[stage], w_col, n_blk * BLOCK_N);
        tma_load_2d(sb + kBBytes + kHalfN * 128, w_lo, &bars->full[stage], w_col, n_blk * BLOCK_N + kHalfN);
      }
    }
    if (++stage == num_stages) { stage = 0; phase ^= 1; }
    if (++kb == num_k_blocks) { kb = 0; tile += gridDim.x; }
  }
};

template <int BLOCK_N, int PART_N, bool F16, bool SUM32>
__device__ __forceinline__ void mma_and_epilogue(const LinearParams& p, const EpiStoreMaps& maps, Producer<BLOCK_N>& prod, bool is_producer,
                                                 int col_part, int lane_group, int lane, uint32_t epi_stage_addr) {
  constexpr int kPart0 = epi_part0_cols<BLOCK_N>();
  const bool split = p.nsplit == 3;
  const uint32_t a_plane = kABytes, b_plane = BLOCK_N * kBlockK * 2;
  const uint32_t b_off = (split ? 2 : 1) * kABytes + (col_part ? kPart0 * 128 : 0);  // this warpgroup's W rows
  const int num_stages = prod.num_stages, num_k_blocks = prod.num_k_blocks, num_n_blocks = prod.num_n_blocks;
  GemmBarriers* bars = prod.bars;
  float acc0[PART_N / 2], acc1[PART_N / 2];
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < prod.num_tiles; tile += gridDim.x) {
    const int m_blk = tile / num_n_blocks;
    const int n_blk = tile % num_n_blocks;
#pragma unroll
    for (int i = 0; i < PART_N / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
    for (int kb = 0; kb < num_k_blocks; ++kb) {
      mbar_wait(&bars->full[stage], phase);
      const uint32_t sa = smem_u32(prod.ring + (size_t)stage * prod.stage_bytes);
      if (!(p.debug & 2)) mma_kblock_promoted<PART_N, F16>(acc0, acc1, sa, sa + b_off, a_plane, b_plane, split);
      // the tensor cores have read this stage: it may be refilled
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->empty[stage]);
      if (is_producer) prod.issue_next();
      if (++stage == num_stages) { stage = 0; phase ^= 1; }
    }
    epilogue_tile<BLOCK_N, PART_N, F16, SUM32>(p, maps, acc0, acc1, m_blk, n_blk, lane_group, col_part, lane, epi_stage_addr);
  }
}

// Warp roles (256 threads, two warpgroups, up to 255 registers per thread): warpgroup j computes the tile's column part j
// (epi_part0_cols) for all 128 rows with wgmma (mma_kblock_promoted: fp32 sums per k-block on the tensor cores, added up on
// the CUDA cores) -- two m64 halves over an interleaved A descriptor, so each warp ends up
// owning 32 consecutive rows -- and runs the epilogue on its registers.  Thread 0 also drives the TMA operand stream,
// `num_stages` k-blocks ahead of the MMAs and across tile boundaries (the next tile's operands arrive under the epilogue).
// Barriers: full[s] (1 arrival + the TMA transaction bytes), empty[s] (one arrival per warp once its wgmmas that read
// stage s have completed).
template <int BLOCK_N, bool F16, bool SUM32>
__device__ __forceinline__ void linear2_body(const CUtensorMap& map_a_hi, const CUtensorMap& map_a_lo, const CUtensorMap& map_w_hi,
                                             const CUtensorMap& map_w_lo, const CUtensorMap& map_o_hi, const CUtensorMap& map_o_lo,
                                             const CUtensorMap& map_o_f32, const LinearParams& p, const int num_stages,
                                             const int num_m_blocks, const int num_n_blocks) {
  static_assert(BLOCK_N == 128 || BLOCK_N == 192 || BLOCK_N == 256, "BLOCK_N");
  constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  constexpr int kPart0 = epi_part0_cols<BLOCK_N>();

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nplanes = (p.nsplit == 3) ? 2 : 1;
  const uint32_t stage_bytes = nplanes * (kABytes + kBBytes);
  uint8_t* ring = smem;
  uint8_t* epi_stage = ring + (size_t)num_stages * stage_bytes;  // kNumMmaWarps x 4 KB staging tiles
  GemmBarriers* bars = reinterpret_cast<GemmBarriers*>(epi_stage + kNumMmaWarps * kEpiStageBytes);

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_k_blocks = (p.K + kBlockK - 1) / kBlockK;
  Producer<BLOCK_N> prod{&map_a_hi, &map_a_lo, &map_w_hi, &map_w_lo, &p, ring, bars, stage_bytes, num_stages,
                         num_m_blocks * num_n_blocks, num_n_blocks, num_k_blocks,
                         p.num_taps > 0 ? p.k_per_tap / kBlockK : num_k_blocks,  // convolution taps: see LinearParams
                         (int)blockIdx.x, 0, 0, 0u};
  const bool is_producer = threadIdx.x == 0;

  if (is_producer) {
    tma_prefetch_desc(&map_a_hi);
    tma_prefetch_desc(&map_w_hi);
    for (int s = 0; s < num_stages; ++s) {
      mbar_init(&bars->full[s], 1);
      mbar_init(&bars->empty[s], kNumMmaWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (is_producer)
    for (int s = 0; s < num_stages; ++s) prod.issue_next();

  const int col_part = warp_idx >> 2;
  const int lane_group = warp_idx & 3;
  const uint32_t epi_stage_addr = smem_u32(epi_stage + warp_idx * kEpiStageBytes);
  const EpiStoreMaps epi_maps{&map_o_hi, &map_o_lo, &map_o_f32};
  if (col_part == 0)
    mma_and_epilogue<BLOCK_N, kPart0, F16, SUM32>(p, epi_maps, prod, is_producer, col_part, lane_group, lane, epi_stage_addr);
  else
    mma_and_epilogue<BLOCK_N, BLOCK_N - kPart0, F16, SUM32>(p, epi_maps, prod, false, col_part, lane_group, lane, epi_stage_addr);
  if (p.tma_store && lane == 0) tma_store_wait_all();
}

template <int BLOCK_N, bool F16>
__global__ void __launch_bounds__(kNumThreads, 1)
linear2_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
               const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
               const __grid_constant__ CUtensorMap map_o_hi, const __grid_constant__ CUtensorMap map_o_lo,
               const __grid_constant__ CUtensorMap map_o_f32,
               const LinearParams p, const int num_stages, const int num_m_blocks, const int num_n_blocks) {
  linear2_body<BLOCK_N, F16, false>(map_a_hi, map_a_lo, map_w_hi, map_w_lo, map_o_hi, map_o_lo, map_o_f32, p, num_stages, num_m_blocks,
                                    num_n_blocks);
}

// fp16 operands whose fp16-rounded sum gets an fp32 residual added without a second rounding (epilogue_tile, SUM32): the
// gradient sums of the UNet's input-VJP.  A kernel of its own, so that linear2_kernel's code is what it was.
template <int BLOCK_N>
__global__ void __launch_bounds__(kNumThreads, 1)
linear2_f16_sum32_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                         const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                         const __grid_constant__ CUtensorMap map_o_hi, const __grid_constant__ CUtensorMap map_o_lo,
                         const __grid_constant__ CUtensorMap map_o_f32,
                         const LinearParams p, const int num_stages, const int num_m_blocks, const int num_n_blocks) {
  linear2_body<BLOCK_N, true, true>(map_a_hi, map_a_lo, map_w_hi, map_w_lo, map_o_hi, map_o_lo, map_o_f32, p, num_stages, num_m_blocks,
                                    num_n_blocks);
}

template <int BLOCK_N, bool F16, bool SUM32 = false>
cudaError_t launch_impl2(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& w_hi, const CUtensorMap& w_lo,
                         const LinearParams& p_in, int num_sms, cudaStream_t stream, const LinearStoreMaps* st) {
  LinearParams p = p_in;
  p.tma_store = 0;
  CUtensorMap o_hi = a_hi, o_lo = a_hi, o_f32 = a_hi;  // placeholders when the STG epilogue is used
  if (st && (st->hi || st->f32) && p.rowmap == ROWMAP_IDENTITY && p.dup_row_offset == 0 &&
      (!p.out_hi || (st->hi && (p.nsplit_out != 3 || st->lo))) && (!p.out_f32 || st->f32)) {
    p.tma_store = 1;
    if (st->hi) o_hi = *st->hi;
    if (st->lo) o_lo = *st->lo;
    if (st->f32) o_f32 = *st->f32;
  }
  constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  const int nplanes = (p.nsplit == 3) ? 2 : 1;
  const int num_m_blocks = (p.M + kBlockM - 1) / kBlockM;
  const int num_n_blocks = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int num_tiles = num_m_blocks * num_n_blocks;
  int ctas = num_sms;
  if (ctas > num_tiles) ctas = num_tiles;
  const int fixed = 1024 + kNumMmaWarps * kEpiStageBytes + (int)sizeof(GemmBarriers);
  const int stage_bytes = nplanes * (kABytes + kBBytes);
  int num_stages = (kSmemLimit - fixed) / stage_bytes;
  if (num_stages > kMaxStages) num_stages = kMaxStages;
  const size_t smem = (size_t)fixed + (size_t)num_stages * stage_bytes;
  if constexpr (SUM32)
    return launch_kernel(linear2_f16_sum32_kernel<BLOCK_N>, dim3(ctas), dim3(kNumThreads), smem, stream, a_hi, a_lo, w_hi, w_lo,
                         o_hi, o_lo, o_f32, p, num_stages, num_m_blocks, num_n_blocks);
  return launch_kernel(linear2_kernel<BLOCK_N, F16>, dim3(ctas), dim3(kNumThreads), smem, stream, a_hi, a_lo, w_hi, w_lo,
                       o_hi, o_lo, o_f32, p, num_stages, num_m_blocks, num_n_blocks);
}

}  // namespace

cudaError_t configure_linear2_kernels() {
  cudaError_t e = cudaSuccess;
  auto set = [&](auto kernel) {
    if (e == cudaSuccess) e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
  };
  set(linear2_kernel<128, false>); set(linear2_kernel<192, false>); set(linear2_kernel<256, false>);
  set(linear2_kernel<128, true>); set(linear2_kernel<256, true>);
  set(linear2_f16_sum32_kernel<128>); set(linear2_f16_sum32_kernel<256>);
  return e;
}

// Tensor maps: A box {64, 128}; W box {64, block_n / 2}.
cudaError_t launch_linear_pair(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& w_hi, const CUtensorMap& w_lo,
                               const LinearParams& p, int block_n, int num_sms, cudaStream_t stream,
                               const LinearStoreMaps* st, bool f16, bool sum32) {
  if (p.N % 8 != 0 || (p.nsplit != 1 && p.nsplit != 3)) {
    set_last_error("launch_linear_pair: N must be a multiple of 8 and nsplit 1 or 3 (N=%d nsplit=%d)", p.N, p.nsplit);
    return cudaErrorInvalidValue;
  }
  if (sum32 && !f16) {
    set_last_error("launch_linear_pair: the fp32 residual sum exists for fp16 operands only");
    return cudaErrorInvalidValue;
  }
  if (f16) {
    if (p.nsplit != 1 || (block_n != 128 && block_n != 256)) {
      set_last_error("launch_linear_pair: fp16 operands take one plane (nsplit 1) and block_n 128 or 256 (nsplit=%d block_n=%d)",
                     p.nsplit, block_n);
      return cudaErrorInvalidValue;
    }
    if (sum32) {
      if (block_n == 256) return launch_impl2<256, true, true>(a_hi, a_lo, w_hi, w_lo, p, num_sms, stream, st);
      return launch_impl2<128, true, true>(a_hi, a_lo, w_hi, w_lo, p, num_sms, stream, st);
    }
    if (block_n == 256) return launch_impl2<256, true>(a_hi, a_lo, w_hi, w_lo, p, num_sms, stream, st);
    return launch_impl2<128, true>(a_hi, a_lo, w_hi, w_lo, p, num_sms, stream, st);
  }
  if (block_n == 256) return launch_impl2<256, false>(a_hi, a_lo, w_hi, w_lo, p, num_sms, stream, st);
  if (block_n == 192) return launch_impl2<192, false>(a_hi, a_lo, w_hi, w_lo, p, num_sms, stream, st);
  if (block_n == 128) return launch_impl2<128, false>(a_hi, a_lo, w_hi, w_lo, p, num_sms, stream, st);
  set_last_error("launch_linear_pair: unsupported block_n %d", block_n);
  return cudaErrorInvalidValue;
}

}  // namespace cmdi
