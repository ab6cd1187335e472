// Backward of the attention core on wgmma tensor cores (reconstruction guidance only: the denoiser's input-VJP,
// gaussian_diffusion.py:411-416 runs autograd through nn.MultiheadAttention here).
//
//   S = Q K^T / sqrt(128)   P = softmax_rows(S)   O = P V
//   dV = P^T dO    dP = dO V^T    delta_i = sum_j P_ij dP_ij    dS = P o (dP - delta) / sqrt(128)
//   dQ = dS K      dK = dS^T Q
//
// Two launches of one kernel, each CTA owning a 128-row tile of one (sequence, head), 64 rows per warpgroup:
//   mode 0 (rows = queries): X = Q_t K^T, Y = dO_t V^T; row statistics (max, sum, delta) by the four threads of a row (a
//           quad of the wgmma fragment); dS in registers -> bf16 hi/lo A fragments; dQ_t = dS K (K MN-major from the tile
//           that served X).  Writes lse2_i = max*c + log2(sum) and delta_i per query row for mode 1.
//   mode 1 (rows = keys):    X = K_t Q^T = S^T, Y = V_t dO^T = dP^T; P^T = exp2(c X - lse2_i) and dS^T with the
//           per-column statistics of mode 0; dV_t = P^T dO in two 64-column halves, dK_t = dS^T Q.
// Every product uses the bf16 hi/lo operand split (3 MMAs), fp32 accumulation in registers.
//
// Shared memory (220 KB, one CTA per SM):
//   R_A  64 KB: the 128-row tile operand of X (hi, lo), then of Y
//   R_B 104 KB: the 208-row operand of X (hi, lo); stays resident as the MN-major B operand of dQ / dK
//   R_C  52 KB: the 208-row operand of Y, streamed one 64-column block (hi + lo) at a time; in mode 1 the
//               same blocks are streamed a second time as the MN-major B operand of dV
#include "common.cuh"
#include "kernels.h"

namespace cmdi {

namespace {

constexpr int kHeadDim = 128;
constexpr int kTile = 128;
constexpr int kPad = kAttnKeyPad;             // 208 = 13 * 16
constexpr int kKeyBlocks = kPad / 16;
constexpr int kTBlk = kTile * 128;            // 16384: 64 head-dim columns of a 128-row tile
constexpr int kFBlk = kPad * 128;             // 26624: 64 head-dim columns of a 208-row operand
constexpr int kOffAHi = 0, kOffALo = 2 * kTBlk;
constexpr int kOffBHi = 4 * kTBlk, kOffBLo = kOffBHi + 2 * kFBlk;
constexpr int kOffCHi = kOffBLo + 2 * kFBlk, kOffCLo = kOffCHi + kFBlk;
constexpr int kSmemTiles = kOffCLo + kFBlk;   // 225280
constexpr int kThreads = 256;

struct __align__(8) BwdBarriers {
  uint64_t x_full, a2_full, c_full;
  float col_lse[kPad];
  float col_delta[kPad];
};

// bf16 hi / lo A fragments (m64k16, see common.cuh) of key block t from an accumulator-layout row fragment v
__device__ __forceinline__ void to_frags(const float (&v)[kPad / 2], uint32_t (&hi)[kKeyBlocks][4], uint32_t (&lo)[kKeyBlocks][4]) {
#pragma unroll
  for (int t = 0; t < kKeyBlocks; ++t)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = 8 * t + 4 * (q >> 1) + 2 * (q & 1);
      split_bf16x2(v[i], v[i + 1], hi[t][q], lo[t][q]);
    }
}

// D (+)= A[64 x 208] B^T with the A operand of this warpgroup at a_off (+ k-block kb) and B at b_off, three bf16 terms
__device__ __forceinline__ void mma_x(float (&d)[kPad / 2], uint32_t sbase, uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                      int kb0, int kb1, uint32_t a_blk, uint32_t b_blk, bool split, bool first) {
  const int nterms = split ? 3 : 1;
#pragma unroll
  for (int term = 0; term < 3; ++term) {
    if (term >= nterms) break;
    const uint32_t ao = (split && term == 0) ? a_lo : a_hi;
    const uint32_t bo = (split && term == 1) ? b_lo : b_hi;
    for (int kb = kb0; kb < kb1; ++kb) {
      const uint64_t da = make_desc_kmajor_sw128(sbase + ao + kb * a_blk);
      const uint64_t db = make_desc_kmajor_sw128(sbase + bo + kb * b_blk);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_m64n208k16_ss(d, desc_advance(da, kk * 32), desc_advance(db, kk * 32), (first && term == 0 && kb == kb0 && kk == 0) ? 0u : 1u);
    }
  }
}

// D = A[64 x 208 keys] (registers, hi / lo) * B[208 x N] (MN-major in shared memory), three bf16 terms
template <int N>
__device__ __forceinline__ void mma_rs(float (&d)[N / 2], const uint32_t (&ah)[kKeyBlocks][4], const uint32_t (&al)[kKeyBlocks][4],
                                       uint32_t b_hi, uint32_t b_lo, bool split) {
  const uint64_t dh = make_desc_mnmajor_sw128(b_hi, kFBlk);
  const uint64_t dl = make_desc_mnmajor_sw128(b_lo, kFBlk);
  wgmma_fence_operands(d);
  wgmma_fence();
#pragma unroll
  for (int t = 0; t < kKeyBlocks; ++t) {
    if constexpr (N == 128) {
      if (split) wgmma_m64n128k16_rs_tb(d, al[t], desc_advance(dh, t * 2048), t ? 1u : 0u);
      wgmma_m64n128k16_rs_tb(d, ah[t], desc_advance(dh, t * 2048), (split || t) ? 1u : 0u);
      if (split) wgmma_m64n128k16_rs_tb(d, ah[t], desc_advance(dl, t * 2048), 1u);
    } else {
      if (split) wgmma_m64n64k16_rs_tb(d, al[t], desc_advance(dh, t * 2048), t ? 1u : 0u);
      wgmma_m64n64k16_rs_tb(d, ah[t], desc_advance(dh, t * 2048), (split || t) ? 1u : 0u);
      if (split) wgmma_m64n64k16_rs_tb(d, ah[t], desc_advance(dl, t * 2048), 1u);
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_operands(d);
}

// rows r0 = 16 w + lane / 4 and r0 + 8 of the warpgroup's 64: fp32 accumulator columns -> bf16 hi / lo planes
template <int N>
__device__ __forceinline__ void store_rows(const AttnBwdParams& p, const float (&d)[N / 2], int tile_row0, int row0, int out_col, int lane) {
#pragma unroll
  for (int g = 0; g < 2; ++g) {
    const int r = tile_row0 + 8 * g;
    if (r >= p.seq_len) continue;
    const size_t off = (size_t)(row0 + r) * p.ld_dqkv + out_col + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      uint32_t hw, lw;
      split_bf16x2(d[4 * j + 2 * g], d[4 * j + 2 * g + 1], hw, lw);
      *reinterpret_cast<uint32_t*>(p.dqkv_hi + off + 8 * j) = hw;
      *reinterpret_cast<uint32_t*>(p.dqkv_lo + off + 8 * j) = lw;
    }
  }
}

__global__ void __launch_bounds__(kThreads, 1)
attention_bwd_tc_kernel(const __grid_constant__ CUtensorMap qkv_t_hi, const __grid_constant__ CUtensorMap qkv_t_lo,
                        const __grid_constant__ CUtensorMap qkv_f_hi, const __grid_constant__ CUtensorMap qkv_f_lo,
                        const __grid_constant__ CUtensorMap do_t_hi, const __grid_constant__ CUtensorMap do_t_lo,
                        const __grid_constant__ CUtensorMap do_f_hi, const __grid_constant__ CUtensorMap do_f_lo,
                        const AttnBwdParams p, const int mode) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  BwdBarriers* bars = reinterpret_cast<BwdBarriers*>(smem + kSmemTiles);
  const uint32_t sbase = smem_u32(smem);

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp_idx >> 2, w = warp_idx & 3;
  const int tile = blockIdx.x, head = blockIdx.y, seq = blockIdx.z;
  const int S = p.seq_len, H = p.num_heads;
  const bool split = (p.nsplit == 3);
  const int row0 = seq * S;
  const int q_col = head * kHeadDim, k_col = H * kHeadDim + head * kHeadDim, v_col = 2 * H * kHeadDim + head * kHeadDim;
  const int do_col = head * kHeadDim;
  // mode 0: A1 = Q tile, B1 = K, A2 = dO tile, B2 = V.   mode 1: A1 = K tile, B1 = Q, A2 = V tile, B2 = dO.
  const CUtensorMap* a2_hi = mode == 0 ? &do_t_hi : &qkv_t_hi;
  const CUtensorMap* a2_lo = mode == 0 ? &do_t_lo : &qkv_t_lo;
  const CUtensorMap* b2_hi = mode == 0 ? &qkv_f_hi : &do_f_hi;
  const CUtensorMap* b2_lo = mode == 0 ? &qkv_f_lo : &do_f_lo;
  const int a1_col = mode == 0 ? q_col : k_col, b1_col = mode == 0 ? k_col : q_col;
  const int a2_col = mode == 0 ? do_col : v_col, b2_col = mode == 0 ? v_col : do_col;
  const uint32_t planes = split ? 2 : 1;
  auto load_c = [&](int blk) {  // one 64-column block (hi + lo) of the 208-row Y operand
    mbar_arrive_expect_tx(&bars->c_full, planes * kFBlk);
    tma_load_2d(smem + kOffCHi, b2_hi, &bars->c_full, b2_col + blk * 64, row0);
    if (split) tma_load_2d(smem + kOffCLo, b2_lo, &bars->c_full, b2_col + blk * 64, row0);
  };

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&qkv_t_hi);
    tma_prefetch_desc(&qkv_f_hi);
    mbar_init(&bars->x_full, 1);
    mbar_init(&bars->a2_full, 1);
    mbar_init(&bars->c_full, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(&bars->x_full, planes * 2 * (kTBlk + kFBlk));
    for (int j = 0; j < 2; ++j) {
      tma_load_2d(smem + kOffAHi + j * kTBlk, &qkv_t_hi, &bars->x_full, a1_col + j * 64, row0 + tile * kTile);
      tma_load_2d(smem + kOffBHi + j * kFBlk, &qkv_f_hi, &bars->x_full, b1_col + j * 64, row0);
      if (split) {
        tma_load_2d(smem + kOffALo + j * kTBlk, &qkv_t_lo, &bars->x_full, a1_col + j * 64, row0 + tile * kTile);
        tma_load_2d(smem + kOffBLo + j * kFBlk, &qkv_f_lo, &bars->x_full, b1_col + j * 64, row0);
      }
    }
    load_c(0);
  }
  if (mode == 1) {
    // per-query statistics written by the mode-0 launch (lse2 = +inf for padded queries -> P = 0)
    for (int i = threadIdx.x; i < kPad; i += kThreads) {
      float2 st = make_float2(INFINITY, 0.f);
      if (i < S) st = p.stats[(long long)(row0 + i) * H + head];
      bars->col_lse[i] = st.x;
      bars->col_delta[i] = st.y;
    }
  }
  __syncthreads();

  const float c_exp = 0.08838834764831845f * 1.4426950408889634f;  // log2(e) / sqrt(128)
  const float c_scale = 0.08838834764831845f;
  const uint32_t a_wg = wg * 64 * 128;  // this warpgroup's rows of the tile operand
  const int cq = 2 * (lane & 3);
  const int tile_row0 = tile * kTile + wg * 64 + 16 * w + (lane >> 2);  // rows tile_row0 and tile_row0 + 8

  // ---------------- X = A1 B1^T ----------------
  float x[kPad / 2];
  mbar_wait(&bars->x_full, 0);
  wgmma_fence_operands(x);
  wgmma_fence();
  mma_x(x, sbase, kOffAHi + a_wg, kOffALo + a_wg, kOffBHi, kOffBLo, 0, 2, kTBlk, kFBlk, split, true);
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_operands(x);
  __syncthreads();  // R_A is free: the Y tile operand replaces it
  if (threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bars->a2_full, planes * 2 * kTBlk);
    for (int j = 0; j < 2; ++j) {
      tma_load_2d(smem + kOffAHi + j * kTBlk, a2_hi, &bars->a2_full, a2_col + j * 64, row0 + tile * kTile);
      if (split) tma_load_2d(smem + kOffALo + j * kTBlk, a2_lo, &bars->a2_full, a2_col + j * 64, row0 + tile * kTile);
    }
  }

  // ---------------- probabilities (unnormalised in mode 0) ----------------
  float mc0 = 0.f, mc1 = 0.f, sum0 = 0.f, sum1 = 0.f;
  if (mode == 0) {
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < kPad / 8; ++j) {
      if (8 * j + cq >= S) { x[4 * j] = -INFINITY; x[4 * j + 2] = -INFINITY; }  // padded keys
      if (8 * j + cq + 1 >= S) { x[4 * j + 1] = -INFINITY; x[4 * j + 3] = -INFINITY; }
      mx0 = fmaxf(mx0, fmaxf(x[4 * j], x[4 * j + 1]));
      mx1 = fmaxf(mx1, fmaxf(x[4 * j + 2], x[4 * j + 3]));
    }
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, o));
    }
    mc0 = mx0 * c_exp; mc1 = mx1 * c_exp;
#pragma unroll
    for (int i = 0; i < kPad / 2; ++i) {
      x[i] = fast_exp2(fmaf(x[i], c_exp, -((i & 2) ? mc1 : mc0)));
      if (i & 2) sum1 += x[i]; else sum0 += x[i];
    }
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      sum0 += __shfl_xor_sync(0xffffffffu, sum0, o);
      sum1 += __shfl_xor_sync(0xffffffffu, sum1, o);
    }
  } else {
#pragma unroll
    for (int i = 0; i < kPad / 2; ++i) x[i] = fast_exp2(fmaf(x[i], c_exp, -bars->col_lse[8 * (i >> 2) + cq + (i & 1)]));
  }

  // ---------------- Y = A2 B2^T, one 64-column block of the contraction at a time ----------------
  float y[kPad / 2];
  mbar_wait(&bars->a2_full, 0);
  for (int kb = 0; kb < 2; ++kb) {
    mbar_wait(&bars->c_full, kb & 1);
    wgmma_fence_operands(y);
    wgmma_fence();
    mma_x(y, sbase, kOffAHi + a_wg, kOffALo + a_wg, kOffCHi, kOffCLo, kb, kb + 1, kTBlk, 0, split, kb == 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(y);
    __syncthreads();  // R_C is free
    if (threadIdx.x == 0 && (kb == 0 || mode == 1)) load_c(kb ^ 1);  // mode 1: dO block 0 again, for dV
  }

  uint32_t ah[kKeyBlocks][4], al[kKeyBlocks][4];
  if (mode == 0) {
    // delta = sum_j P_ij dP_ij, dS = P (dP - delta) / sqrt(d)
    float d0 = 0.f, d1 = 0.f;
#pragma unroll
    for (int i = 0; i < kPad / 2; ++i) {
      if (i & 2) d1 = fmaf(x[i], y[i], d1); else d0 = fmaf(x[i], y[i], d0);
    }
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      d0 += __shfl_xor_sync(0xffffffffu, d0, o);
      d1 += __shfl_xor_sync(0xffffffffu, d1, o);
    }
    const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
    const float delta0 = d0 * inv0, delta1 = d1 * inv1;
    if ((lane & 3) == 0) {
      if (tile_row0 < S) p.stats[(long long)(row0 + tile_row0) * H + head] = make_float2(mc0 + log2f(sum0), delta0);
      if (tile_row0 + 8 < S) p.stats[(long long)(row0 + tile_row0 + 8) * H + head] = make_float2(mc1 + log2f(sum1), delta1);
    }
#pragma unroll
    for (int i = 0; i < kPad / 2; ++i) y[i] = x[i] * ((i & 2) ? inv1 : inv0) * (y[i] - ((i & 2) ? delta1 : delta0)) * c_scale;
    to_frags(y, ah, al);
    // dQ_t = dS K: B = the resident R_B operand, MN-major
    float acc[kHeadDim / 2];
    mma_rs<kHeadDim>(acc, ah, al, sbase + kOffBHi, sbase + kOffBLo, split);
    store_rows<kHeadDim>(p, acc, tile_row0, row0, q_col, lane);
  } else {
    // dS^T = P^T (dP^T - delta_i) / sqrt(d)
#pragma unroll
    for (int i = 0; i < kPad / 2; ++i) y[i] = x[i] * (y[i] - bars->col_delta[8 * (i >> 2) + cq + (i & 1)]) * c_scale;
    to_frags(x, ah, al);
    // dV_t = P^T dO, 64 head-dim columns at a time (R_C holds that block of dO as an MN-major B operand)
    for (int nb = 0; nb < 2; ++nb) {
      mbar_wait(&bars->c_full, nb & 1);  // third and fourth completion of c_full
      float acc[32];
      mma_rs<64>(acc, ah, al, sbase + kOffCHi, sbase + kOffCLo, split);
      __syncthreads();
      if (threadIdx.x == 0 && nb == 0) load_c(1);
      store_rows<64>(p, acc, tile_row0, row0, v_col + nb * 64, lane);
    }
    to_frags(y, ah, al);
    // dK_t = dS^T Q: B = the resident R_B operand, MN-major
    float acc[kHeadDim / 2];
    mma_rs<kHeadDim>(acc, ah, al, sbase + kOffBHi, sbase + kOffBLo, split);
    store_rows<kHeadDim>(p, acc, tile_row0, row0, k_col, lane);
  }
}

}  // namespace

cudaError_t configure_attention_bwd_tc_kernel() {
  return cudaFuncSetAttribute(attention_bwd_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)(1024 + kSmemTiles + sizeof(BwdBarriers)));
}

cudaError_t launch_attention_bwd_tc(const AttnBwdTcMaps& m, const AttnBwdParams& p, cudaStream_t stream) {
  if (p.seq_len > kPad || p.seq_len < 1 || (p.nsplit != 1 && p.nsplit != 3) || !p.stats) {
    set_last_error("launch_attention_bwd_tc: unsupported seq_len=%d nsplit=%d (or no statistics buffer)", p.seq_len, p.nsplit);
    return cudaErrorInvalidValue;
  }
  const size_t smem = 1024 + kSmemTiles + sizeof(BwdBarriers);
  dim3 grid((p.seq_len + kTile - 1) / kTile, p.num_heads, p.num_seqs);
  for (int mode = 0; mode < 2; ++mode) {
    attention_bwd_tc_kernel<<<grid, kThreads, smem, stream>>>(*m.qkv_t_hi, *m.qkv_t_lo, *m.qkv_f_hi, *m.qkv_f_lo, *m.do_t_hi,
                                                               *m.do_t_lo, *m.do_f_hi, *m.do_f_lo, p, mode);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace cmdi
