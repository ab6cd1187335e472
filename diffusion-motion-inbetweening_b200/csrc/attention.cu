// Self-attention core of nn.MultiheadAttention for the MDM encoder (reference: model/mdm.py:107-114, :284;
// no key-padding mask -- `src_key_padding_mask` is commented out there), head dim 128, S <= 208 keys:
//
//   O[s, :] = softmax_j( Q[s,:] . K[j,:] / sqrt(128) ) V[j, :]
//
// One CTA per (sequence, head, 128-query half), two warpgroups of 64 query rows each.  Both contractions run on wgmma:
//   S = Q K^T   : A = Q rows (smem, K-major), B = K (smem, K-major, all 208 padded keys), D = 64 x 208 fp32 per warpgroup
//   O = P V     : A = P (bf16 hi / lo, converted in registers from the S fragment), B = V (smem, MN-major), D = 64 x 128
// Q, K and V are read straight out of the QKV projection's [tokens, 3*H*128] bf16 planes with TMA
// (no head-split or transpose kernels).  With nsplit = 3 every product uses the hi/lo bf16 split
// (X_lo*Y_hi + X_hi*Y_lo + X_hi*Y_hi), P included, so the result is fp32-accurate.
//
// A query row lives in the four threads of a quad (the wgmma fragment layout): row max and row sum are two shuffles.
// Shared memory: Q 64 KB + K 104 KB + V_hi 52 KB; V_lo is loaded into Q's space once S is complete, under the softmax.
#include "common.cuh"
#include "gemm_epilogue.cuh"
#include "kernels.h"

namespace cmdi {

namespace {

constexpr int kHeadDim = 128;
constexpr int kQTile = 128;                     // query rows per CTA (two warpgroups of 64)
constexpr int kKeyPad = kAttnKeyPad;            // 208 = 13 * 16
constexpr int kKeyBlocks = kKeyPad / 16;
constexpr int kQBlockBytes = kQTile * 128;      // 64 dh-columns of 128 queries
constexpr int kKVBlockBytes = kKeyPad * 128;    // 64 dh-columns of 208 keys  (26 swizzle atoms)
constexpr int kQPlane = 2 * kQBlockBytes;       // 32768
constexpr int kKVPlane = 2 * kKVBlockBytes;     // 53248
constexpr int kOffQHi = 0, kOffQLo = kQPlane;
constexpr int kOffKHi = 2 * kQPlane, kOffKLo = kOffKHi + kKVPlane;
constexpr int kOffVHi = kOffKLo + kKVPlane;
constexpr int kOffVLo = 0;                      // over Q, once S is complete
constexpr int kSmemTiles = kOffVHi + kKVPlane;  // 225280
constexpr int kThreads = 256;
static_assert(kKVBlockBytes % 1024 == 0 && kKVPlane <= 2 * kQPlane, "operand tile layout");

struct __align__(8) AttnBarriers {
  uint64_t qkv_full, vlo_full;
};

__global__ void __launch_bounds__(kThreads, 1)
attention_kernel(const __grid_constant__ CUtensorMap map_q_hi, const __grid_constant__ CUtensorMap map_q_lo,
                 const __grid_constant__ CUtensorMap map_kv_hi, const __grid_constant__ CUtensorMap map_kv_lo, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  AttnBarriers* bars = reinterpret_cast<AttnBarriers*>(smem + kSmemTiles);
  const int S = p.seq_len;
  const bool split = (p.nsplit == 3);
  const int half = blockIdx.x & 1;
  const int item = blockIdx.x >> 1;
  const int head = item % p.num_heads, seq = item / p.num_heads;
  if (half * kQTile >= S) return;  // no query rows here (CTA-uniform)
  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp_idx >> 2, w = warp_idx & 3;
  const uint32_t sbase = smem_u32(smem);
  const int row0 = seq * S;
  const int kcol = p.num_heads * kHeadDim + head * kHeadDim, vcol = 2 * p.num_heads * kHeadDim + head * kHeadDim;
  const uint32_t planes = split ? 2 : 1;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&map_q_hi);
    tma_prefetch_desc(&map_kv_hi);
    mbar_init(&bars->qkv_full, 1);
    mbar_init(&bars->vlo_full, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx(&bars->qkv_full, planes * (kQPlane + kKVPlane) + kKVPlane);
    for (int j = 0; j < 2; ++j) {
      tma_load_2d(smem + kOffQHi + j * kQBlockBytes, &map_q_hi, &bars->qkv_full, head * kHeadDim + j * 64, row0 + half * kQTile);
      tma_load_2d(smem + kOffKHi + j * kKVBlockBytes, &map_kv_hi, &bars->qkv_full, kcol + j * 64, row0);
      tma_load_2d(smem + kOffVHi + j * kKVBlockBytes, &map_kv_hi, &bars->qkv_full, vcol + j * 64, row0);
      if (split) {
        tma_load_2d(smem + kOffQLo + j * kQBlockBytes, &map_q_lo, &bars->qkv_full, head * kHeadDim + j * 64, row0 + half * kQTile);
        tma_load_2d(smem + kOffKLo + j * kKVBlockBytes, &map_kv_lo, &bars->qkv_full, kcol + j * 64, row0);
      }
    }
  }
  __syncthreads();

  // ---------------- S = Q K^T (this warpgroup's 64 query rows) ----------------
  float s[kKeyPad / 2];
  mbar_wait(&bars->qkv_full, 0);
  wgmma_fence_operands(s);
  wgmma_fence();
  {
    const int nterms = split ? 3 : 1;
#pragma unroll
    for (int term = 0; term < 3; ++term) {
      if (term >= nterms) break;
      const uint32_t qo = (split && term == 0) ? kOffQLo : kOffQHi;
      const uint32_t ko = (split && term == 1) ? kOffKLo : kOffKHi;
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const uint64_t da = make_desc_kmajor_sw128(sbase + qo + j * kQBlockBytes + wg * 64 * 128);
        const uint64_t db = make_desc_kmajor_sw128(sbase + ko + j * kKVBlockBytes);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_m64n208k16_ss(s, desc_advance(da, kk * 32), desc_advance(db, kk * 32), (term | j | kk) ? 1u : 0u);
      }
    }
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_operands(s);
  __syncthreads();  // both warpgroups are done with Q: V_lo may overwrite it
  if (split && threadIdx.x == 0) {
    mbar_arrive_expect_tx(&bars->vlo_full, kKVPlane);
    for (int j = 0; j < 2; ++j)
      tma_load_2d(smem + kOffVLo + j * kKVBlockBytes, &map_kv_lo, &bars->vlo_full, vcol + j * 64, row0);
  }

  // ---------------- softmax over the keys (rows r0 = 16 w + lane / 4 and r0 + 8 of the warpgroup) ----------------
  const float c_scale = 0.08838834764831845f * 1.4426950408889634f;  // 1/sqrt(128) * log2(e)
  const int cq = 2 * (lane & 3);
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < kKeyPad / 8; ++j) {
    const bool ok0 = 8 * j + cq < S, ok1 = 8 * j + cq + 1 < S;  // padded keys: exp2 -> 0
    if (!ok0) { s[4 * j] = -INFINITY; s[4 * j + 2] = -INFINITY; }
    if (!ok1) { s[4 * j + 1] = -INFINITY; s[4 * j + 3] = -INFINITY; }
    mx0 = fmaxf(mx0, fmaxf(s[4 * j], s[4 * j + 1]));
    mx1 = fmaxf(mx1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, o));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, o));
  }
  const float mc0 = mx0 * c_scale, mc1 = mx1 * c_scale;
  float sum0 = 0.f, sum1 = 0.f;
  const bool trunc = p.trunc_split != 0;
  uint32_t ph[kKeyBlocks][4], pl[kKeyBlocks][4];
#pragma unroll
  for (int t = 0; t < kKeyBlocks; ++t) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {  // a[q]: rows r0 (q even) / r0 + 8 (q odd), keys 16 t + 8 (q / 2) + cq + {0, 1}
      const int i = 8 * t + 4 * (q >> 1) + 2 * (q & 1);
      const float mc = (q & 1) ? mc1 : mc0;
      const float p0 = fast_exp2(fmaf(s[i], c_scale, -mc));
      const float p1 = fast_exp2(fmaf(s[i + 1], c_scale, -mc));
      if (q & 1) sum1 += p0 + p1; else sum0 += p0 + p1;
      if (trunc) split_bf16x2_trunc(p0, p1, ph[t][q], pl[t][q]); else split_bf16x2(p0, p1, ph[t][q], pl[t][q]);
    }
  }
#pragma unroll
  for (int o = 1; o <= 2; o <<= 1) {
    sum0 += __shfl_xor_sync(0xffffffffu, sum0, o);
    sum1 += __shfl_xor_sync(0xffffffffu, sum1, o);
  }

  // ---------------- O = P V ----------------
  float o[kHeadDim / 2];
  const uint64_t dv_hi = make_desc_mnmajor_sw128(sbase + kOffVHi, kKVBlockBytes);
  wgmma_fence_operands(o);
  wgmma_fence();
  if (split) {
#pragma unroll
    for (int t = 0; t < kKeyBlocks; ++t) wgmma_m64n128k16_rs_tb(o, pl[t], desc_advance(dv_hi, t * 2048), t ? 1u : 0u);
  }
#pragma unroll
  for (int t = 0; t < kKeyBlocks; ++t) wgmma_m64n128k16_rs_tb(o, ph[t], desc_advance(dv_hi, t * 2048), (split || t) ? 1u : 0u);
  wgmma_commit();
  if (split) {
    mbar_wait(&bars->vlo_full, 0);
    const uint64_t dv_lo = make_desc_mnmajor_sw128(sbase + kOffVLo, kKVBlockBytes);
#pragma unroll
    for (int t = 0; t < kKeyBlocks; ++t) wgmma_m64n128k16_rs_tb(o, ph[t], desc_advance(dv_lo, t * 2048), 1u);
    wgmma_commit();
  }
  wgmma_wait<0>();
  wgmma_fence_operands(o);

  // ---------------- output: O / row sum -> bf16 hi / lo planes ----------------
  const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
  const int q0 = half * kQTile + wg * 64 + 16 * w + (lane >> 2);
#pragma unroll
  for (int g = 0; g < 2; ++g) {
    const int q = q0 + 8 * g;
    if (q >= S) continue;
    const float inv = g ? inv1 : inv0;
    const size_t off = (size_t)(row0 + q) * p.ld_out + head * kHeadDim + cq;
#pragma unroll
    for (int j = 0; j < kHeadDim / 8; ++j) {
      uint32_t hw, lw;
      if (trunc) split_bf16x2_trunc(o[4 * j + 2 * g] * inv, o[4 * j + 2 * g + 1] * inv, hw, lw);
      else split_bf16x2(o[4 * j + 2 * g] * inv, o[4 * j + 2 * g + 1] * inv, hw, lw);
      *reinterpret_cast<uint32_t*>(p.out_hi + off + 8 * j) = hw;
      if (p.nsplit_out == 3) *reinterpret_cast<uint32_t*>(p.out_lo + off + 8 * j) = lw;
    }
  }
}

}  // namespace

cudaError_t configure_attention_kernel() {
  return cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)(1024 + kSmemTiles + sizeof(AttnBarriers)));
}

cudaError_t launch_attention(const AttnMaps& m, const AttnParams& p, cudaStream_t stream) {
  if (p.seq_len > kKeyPad || p.seq_len < 1 || (p.nsplit != 1 && p.nsplit != 3)) {
    set_last_error("launch_attention: unsupported seq_len=%d nsplit=%d", p.seq_len, p.nsplit);
    return cudaErrorInvalidValue;
  }
  const int num_items = p.num_heads * p.num_seqs;
  const size_t smem = 1024 + kSmemTiles + sizeof(AttnBarriers);
  return launch_kernel(attention_kernel, dim3(2 * num_items), dim3(kThreads), smem, stream, *m.q_hi, *m.q_lo, *m.kv_hi, *m.kv_lo, p);
}

}  // namespace cmdi
