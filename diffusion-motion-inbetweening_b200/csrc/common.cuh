// Device-side primitives for the sm_90a kernels of the CondMDI sampling engine.
//
// Everything here is a thin wrapper over one PTX instruction: mbarrier, TMA (cp.async.bulk.tensor), wgmma
// (warpgroup MMA: fence / issue / commit / wait) and the shared-memory matrix descriptors the Hopper tensor cores
// consume.  Descriptor bit layouts follow the PTX ISA "matrix descriptor format" table for wgmma.
#pragma once

#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda.h>
#include <stdio.h>
#include <stdint.h>

namespace cmdi {

// ----------------------------------------------------------------------------------------------
// small helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

// 2^x on the SFU (ex2.approx.ftz: relative error ~2^-22, exp2(-inf) = 0)
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// bf16 split of an fp32 value: v ~= hi + lo with |v - hi - lo| <= 2^-17 |v|.
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

// Split two fp32 values at once: hi_word / lo_word hold {a (low half), b (high half)} as bf16x2.
// One packed cvt.rn.bf16x2.f32 per plane (half the conversion-pipe work of four scalar converts).
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi_word, uint32_t& lo_word) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  hi_word = *reinterpret_cast<const uint32_t*>(&h);
  const float ha = __uint_as_float(hi_word << 16), hb = __uint_as_float(hi_word & 0xffff0000u);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - ha, b - hb);
  lo_word = *reinterpret_cast<const uint32_t*>(&l);
}

// fp32 -> the nearest fp16 value, as fp32 (the rounding CUDA autocast applies to every conv / linear output)
__device__ __forceinline__ float round_f16(float v) { return __half2float(__float2half_rn(v)); }
// fp16 x 2 -> one 32-bit word {a (low half), b (high half)}
__device__ __forceinline__ uint32_t pack_f16x2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// y = (x - mean) * rstd * gamma + beta with a fixed operation order: the LayerNorm kernel and the epilogues that
// re-derive LayerNorm's output as a residual (from its fp32 input and the row statistics) must agree bit for bit.
__device__ __forceinline__ float ln_apply(float x, float mean, float rstd, float g, float b) {
  return __fmaf_rn(__fmul_rn(__fsub_rn(x, mean), rstd), g, b);
}

// Same split with the hi half taken by truncation (one PRMT instead of a conversion): v = hi + lo still holds to
// 2^-16 |v| (hi is exact in bf16, lo = RN(v - hi) with |v - hi| < 2^-7 |v|).  Halves the work on the conversion pipe
// where the values are produced at MUFU rate anyway (softmax probabilities, attention outputs).
__device__ __forceinline__ void split_bf16x2_trunc(float a, float b, uint32_t& hi_word, uint32_t& lo_word) {
  const uint32_t ua = __float_as_uint(a), ub = __float_as_uint(b);
  hi_word = __byte_perm(ua, ub, 0x7632);
  const __nv_bfloat162 l = __floats2bfloat162_rn(a - __uint_as_float(ua & 0xffff0000u), b - __uint_as_float(ub & 0xffff0000u));
  lo_word = *reinterpret_cast<const uint32_t*>(&l);
}

// ----------------------------------------------------------------------------------------------
// programmatic dependent launch: a kernel launched with programmaticStreamSerializationAllowed may start while its
// predecessor drains; it must not touch global memory before griddep_wait() (no-op for ordinary launches)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// make generic-proxy smem writes visible to the async proxy (TMA / UMMA reads of smem)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe: has the phase with this parity completed?
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a trapped kernel (an error the host sees),
// never as a hung GPU. ~4e9 cycles is seconds; every legitimate wait here is microseconds.
// No printf on the timeout path: it compiles to a call to vprintf, and ptxas serialises every wgmma of a kernel that
// contains a call (C7510), so one diagnostic line would cost every MMA kernel its tensor-core pipelining.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// 2D tiled load: box lands in smem (swizzled as the map says), completes `bytes` on the mbarrier.
// c0 = coordinate along the contiguous (inner) dimension, c1 = row coordinate.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int32_t c0,
                                            int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// L2 prefetch of a box (no shared-memory destination, no completion to wait for)
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0),
               "r"(c1)
               : "memory");
}

// 2D tiled store: the (128B-swizzled) smem box is written to global memory; completion is tracked by bulk async-groups.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t smem_src_addr, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_src_addr), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all committed bulk stores of this thread have finished READING their shared-memory source
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... and have completed their global writes
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }


// ----------------------------------------------------------------------------------------------
// wgmma: shared-memory matrix descriptors
// ----------------------------------------------------------------------------------------------
// 64-bit descriptor:
//   [0,14)  start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4   [49,52) base offset = 0 (tiles are 1024 B aligned)   [62,64) swizzle: 1 = 128 B
//
// K-major operand, 128 B swizzle (tile written by a TMA box of 64 bf16 x rows):
//   row r at byte r*128, 16 B chunks XOR-swizzled by (r & 7); 8-row groups SBO bytes apart (1024 for dense rows).
//   LBO is unused for swizzled K-major layouts (set to 1 like CUTLASS does).
// MN-major operand, 128 B swizzle (TMA box of 64 contiguous MN-elements x K rows):
//   K index k at byte k*128 inside a 64-wide MN group -> SBO = 1024 (8 K-rows),
//   next 64-wide MN group LBO bytes further (= rows_in_box * 128).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ uint64_t make_desc_kmajor_sw128(uint32_t smem_addr) {
  return make_smem_desc(smem_addr, 16, 1024);
}
// A 128-row K-major tile read as two m64 operands whose 8-row groups interleave: operand h (start + h * 1024) covers
// rows {16 g + 8 h + i : g < 8, i < 8}.  Warp w of the consuming warpgroup then holds accumulator rows 32 w .. 32 w + 31
// of the tile (fragment rows 16 w + i -> 32 w + 8 h + i, 16 w + 8 + i -> 32 w + 16 + 8 h + i): the same rows a warp
// owns in the epilogue's row-per-thread layout (see acc_rows_to_lanes).
__device__ __forceinline__ uint64_t make_desc_kmajor_sw128_interleaved(uint32_t smem_addr) {
  return make_smem_desc(smem_addr, 16, 2048);
}
__device__ __forceinline__ uint64_t make_desc_mnmajor_sw128(uint32_t smem_addr, uint32_t mn_group_stride_bytes) {
  return make_smem_desc(smem_addr, mn_group_stride_bytes, 1024);
}
// advance a descriptor's start address by `bytes` (must keep the result inside the 14-bit field)
__device__ __forceinline__ uint64_t desc_advance(uint64_t desc, uint32_t bytes) { return desc + (uint64_t)(bytes >> 4); }

// ----------------------------------------------------------------------------------------------
// wgmma: issue / commit / wait (warpgroup-collective)
// ----------------------------------------------------------------------------------------------
// Accumulator fragment of an m64nN tile, thread t of the warpgroup (warp w = t / 32, lane l):
//   d[4 j + 0, 1] = (row 16 w + l / 4,     columns 8 j + 2 (l % 4) + {0, 1})
//   d[4 j + 2, 3] = (row 16 w + 8 + l / 4, the same columns)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// register budget of a warpgroup role (setmaxnreg: producer warps give registers to the MMA / epilogue warpgroups)
template <int N>
__device__ __forceinline__ void warpgroup_reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void warpgroup_reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ void named_barrier_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// D (+)= A * B with both operands in shared memory, K-major (scale_d = 0: D = A * B)
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
// the same MMA on fp16 operands (autocast precision: one fp16 plane per operand)
__device__ __forceinline__ void wgmma_m64n64k16_ss_f16(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_m64n128k16_ss(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_m64n208k16_ss(float (&d)[104], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %106, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n208k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103}, %104, %105, p, 1, 1, 0, 0;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103])
      : "l"(da), "l"(db), "r"(scale_d));
}
// A from registers (a[0..3]: the m64k16 bf16 fragment), B MN-major in shared memory
__device__ __forceinline__ void wgmma_m64n128k16_rs_tb(float (&d)[64], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
// A from registers (a[0..3]: the m64k16 bf16 fragment), B MN-major in shared memory
__device__ __forceinline__ void wgmma_m64n64k16_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

// One 64-deep k-block of a 128-row x PART_N tile for one warpgroup (A: interleaved 128-row K-major tile, B: PART_N
// K-major rows; a_plane / b_plane: offsets of the lo planes), with nterms = split ? 3 : 1 bf16 products (lo*hi, hi*lo,
// hi*hi).  The tensor cores accumulate each 64-column chunk of the k-block in a fresh register fragment, which is then
// added into acc0 / acc1 with fp32 adds on the CUDA cores.  The tensor cores' own fp32 accumulation rounds toward zero:
// carried over a whole K = 1024 reduction, that is a bias of -3.5e-6 relative on positive data.  Added up once per k-block
// instead, the bias stays at the level of a 64-long sum.
// F16: the operands are single fp16 planes (CMDI_PRECISION_FP16; `split` must be false), same descriptors and swizzle.
//
// Pipelined: each 64-column chunk c is cut into its two m64 halves h, the sub-chunks (c, h), each summed in a fresh
// 32-register fragment; two fragments form a ring, so the tensor cores work on one sub-chunk (a commit group of
// 4 x nterms MMAs) while the CUDA cores add the previous one into the accumulator (wgmma.wait_group 1).  Every fragment
// receives the same MMAs in the same order as a chunk's half did before (term 0 for k = 0..3, then term 1, then term 2),
// and is added once per k-block: the sums are the same bit for bit.
// The term count is a template parameter: with a runtime count the term loop's early exit leaves ptxas unable to tell
// which commit group a fragment belongs to, and it then waits for every group before the fragment is read (C7517,
// C7518) or serialises every wgmma (C7520).  mma_kblock_promoted dispatches a runtime `split` once per k-block.
//
// One sub-chunk: issue its MMAs into a fresh fragment (the first one with scale-d = 0: D = A * B, which is what ptxas
// makes of an MMA onto a zeroed fragment anyway), commit them as one group.
template <int NTERMS, bool F16>
__device__ __forceinline__ void mma_subchunk_issue(float (&t)[32], uint32_t sa, uint32_t sb, uint32_t a_plane, uint32_t b_plane,
                                                   int c, int h) {
  static_assert(NTERMS == 1 || (NTERMS == 3 && !F16), "1 or 3 bf16 products, fp16 operands: 1");
  constexpr bool split = NTERMS == 3;
  wgmma_fence();
#pragma unroll
  for (int term = 0; term < NTERMS; ++term) {
    const uint64_t da = make_desc_kmajor_sw128_interleaved(sa + ((split && term == 0) ? a_plane : 0u));
    const uint64_t db = make_desc_kmajor_sw128(sb + ((split && term == 1) ? b_plane : 0u) + c * 64 * 128);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t scale_d = (term == 0 && k == 0) ? 0u : 1u;
      if constexpr (F16)
        wgmma_m64n64k16_ss_f16(t, desc_advance(da, h * 1024 + k * 32), desc_advance(db, k * 32), scale_d);
      else
        wgmma_m64n64k16_ss(t, desc_advance(da, h * 1024 + k * 32), desc_advance(db, k * 32), scale_d);
    }
  }
  wgmma_commit();
}
// ... and, once its group has retired, its promotion into columns [32 c, 32 c + 32) of the accumulator of half h
template <int R>
__device__ __forceinline__ void mma_subchunk_promote(float (&acc)[R], float (&t)[32], int c) {
  wgmma_fence_operands(t);
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[32 * c + i] += t[i];
}

// The sub-chunks of a k-block in ring order: (c, 0) in t0, (c, 1) in t1, then c + 1.  Expects sub-chunk (0, 0) issued
// into t0 already; issues the rest, promotes all but the last, and returns with the last, (PART_N / 64 - 1, 1) in t1,
// still in flight (its commit group is the newest), so that a caller can issue its next k-block's first sub-chunk before
// it waits for it.  `between()` runs after every promotion (the chained kernel's TMA thread retries a refill there).
template <int PART_N, int NTERMS, bool F16, class Between>
__device__ __forceinline__ void mma_kblock_body(float (&acc0)[PART_N / 2], float (&acc1)[PART_N / 2], float (&t0)[32], float (&t1)[32],
                                                uint32_t sa, uint32_t sb, uint32_t a_plane, uint32_t b_plane, Between&& between) {
  static_assert(PART_N % 64 == 0, "64-column chunks");
#pragma unroll
  for (int c = 0; c < PART_N / 64; ++c) {
    mma_subchunk_issue<NTERMS, F16>(t1, sa, sb, a_plane, b_plane, c, 1);
    wgmma_wait<1>();
    mma_subchunk_promote(acc0, t0, c);
    between();
    if (c + 1 < PART_N / 64) {
      mma_subchunk_issue<NTERMS, F16>(t0, sa, sb, a_plane, b_plane, c + 1, 0);
      wgmma_wait<1>();
      mma_subchunk_promote(acc1, t1, c);
      between();
    }
  }
}

template <int PART_N, int NTERMS, bool F16>
__device__ __forceinline__ void mma_kblock_pipelined(float (&acc0)[PART_N / 2], float (&acc1)[PART_N / 2], uint32_t sa, uint32_t sb,
                                                     uint32_t a_plane, uint32_t b_plane) {
  float t0[32], t1[32];
  mma_subchunk_issue<NTERMS, F16>(t0, sa, sb, a_plane, b_plane, 0, 0);
  mma_kblock_body<PART_N, NTERMS, F16>(acc0, acc1, t0, t1, sa, sb, a_plane, b_plane, [] {});
  wgmma_wait<0>();
  mma_subchunk_promote(acc1, t1, PART_N / 64 - 1);
}

template <int PART_N, bool F16 = false>
__device__ __forceinline__ void mma_kblock_promoted(float (&acc0)[PART_N / 2], float (&acc1)[PART_N / 2], uint32_t sa, uint32_t sb,
                                                    uint32_t a_plane, uint32_t b_plane, bool split) {
  if constexpr (F16) {
    mma_kblock_pipelined<PART_N, 1, true>(acc0, acc1, sa, sb, a_plane, b_plane);
  } else {
    if (split)
      mma_kblock_pipelined<PART_N, 3, false>(acc0, acc1, sa, sb, a_plane, b_plane);
    else
      mma_kblock_pipelined<PART_N, 1, false>(acc0, acc1, sa, sb, a_plane, b_plane);
  }
}

// The 32 accumulator values of one warp for 32 columns [8 j0, 8 j0 + 32) of an interleaved 128-row tile (acc0 / acc1: the
// two m64 halves, see make_desc_kmajor_sw128_interleaved) -> row-per-lane layout: lane i receives row 32 w + i,
// v[c] = column c.  Through the warp's 4 KB staging tile (16-byte chunks XOR-swizzled by row & 7).
template <int R>
__device__ __forceinline__ void acc_rows_to_lanes(const float (&acc0)[R], const float (&acc1)[R], int j0, uint32_t stage, int lane,
                                                  uint32_t (&v)[32]) {
  __syncwarp();
  const int q = lane >> 2, c2 = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float(&a)[R] = h ? acc1 : acc0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        const int r = 16 * g + 8 * h + q, c = 8 * j + c2;
        const uint32_t addr = stage + r * 128 + ((((uint32_t)c >> 2) ^ ((uint32_t)r & 7u)) << 4) + (c & 3) * 4;
        asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a[4 * (j0 + j) + 2 * g]), "f"(a[4 * (j0 + j) + 2 * g + 1])
                     : "memory");
      }
    }
  }
  __syncwarp();
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    uint32_t x, y, z, w;
    asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w)
                 : "r"(stage + lane * 128 + (((uint32_t)k ^ ((uint32_t)lane & 7u)) << 4)) : "memory");
    v[4 * k] = x; v[4 * k + 1] = y; v[4 * k + 2] = z; v[4 * k + 3] = w;
  }
  __syncwarp();
}

// ----------------------------------------------------------------------------------------------
// vector global stores / loads
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_global_v4(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_global_v4f(float* p, float a, float b, float c, float d) {
  asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

}  // namespace cmdi
