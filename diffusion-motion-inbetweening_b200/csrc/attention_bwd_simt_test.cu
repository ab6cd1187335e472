// TEST-ONLY translation unit: the fp32 CUDA-core attention backward of round 1.
//
// The engine never launches it (the sampling path uses attention_bwd_tc.cu); it is the INDEPENDENT implementation
// `cmdi_test_attention_bwd` (capi_test.cu, CMDI_TEST_ATTN_BWD_SIMT=1) runs so that tests/test_gpu_kernels.py can hold the
// wgmma kernel against a second, structurally different device implementation as well as against torch autograd.
#include "common.cuh"
#include "kernels.h"

namespace cmdi {

namespace {

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float bf16_pair_to_f32(const __nv_bfloat16* hi, const __nv_bfloat16* lo, size_t i) {
  return __bfloat162float(hi[i]) + (lo ? __bfloat162float(lo[i]) : 0.f);
}


// ---------------------------------------------------------------------------------------------
// attention backward, fp32 on CUDA cores.  One CTA per (sequence, head); 8 warps; two passes that share one routine:
//   pass 1 (outer = query i, inner = key j):  X = K, Y = V, a = q_i, b = dO_i
//       s_j = a . X_j ; t_j = b . Y_j ; p = softmax_j(s * scale) ; delta_i = sum_j p_j t_j
//       ds_j = p_j (t_j - delta_i) * scale ;  dQ_i = sum_j ds_j X_j            (+ stats m_i, l_i, delta_i saved)
//   pass 2 (outer = key j, inner = query i):  X = Q, Y = dO, a = k_j, b = v_j
//       s_i, t_i as above ; p_i = exp(s_i * scale - m_i) / l_i ; ds_i = p_i (t_i - delta_i) * scale
//       dK_j = sum_i ds_i X_i ;  dV_j = sum_i p_i Y_i
// X and Y ([S][128] fp32, row stride 132) live in shared memory; each warp handles R = 4 outer rows at a time so
// every shared-memory operand is reused 4 times.
// ---------------------------------------------------------------------------------------------
constexpr int kHD = 128;
constexpr int kStride = 132;       // floats; 16-byte aligned rows, conflict-free 128-bit column reads
constexpr int kR = 4;              // outer rows per warp iteration
constexpr int kMaxS = 197;         // guidance supports the HumanML3D length (196 frames + 1 token)
constexpr int kInnerPerLane = (kMaxS + 31) / 32;  // 7

struct AttnBwdSmem {
  float X[kMaxS * kStride];
  float Y[kMaxS * kStride];
  float stat_m[kMaxS], stat_l[kMaxS], stat_d[kMaxS];
};

template <bool kPass2>
__device__ __forceinline__ void attn_bwd_pass(AttnBwdSmem& sm, const AttnBwdParams& p, int seq, int head, int warp, int lane) {
  const int S = p.seq_len;
  const int row0 = seq * S;
  const int ld = 3 * p.num_heads * kHD;
  const float scale = 0.08838834764831845f;  // 1/sqrt(128)
  // column offsets inside the [tokens, 3*H*128] QKV layout
  const int qc = head * kHD, kc = p.num_heads * kHD + head * kHD, vc = 2 * p.num_heads * kHD + head * kHD;
  const int xcol = kPass2 ? qc : kc;            // X: K (pass 1) / Q (pass 2)
  // ---- stage X and Y ----
  for (int idx = threadIdx.x; idx < S * (kHD / 4); idx += blockDim.x) {
    const int r = idx / (kHD / 4), c4 = (idx % (kHD / 4)) * 4;
    float4 xv, yv;
    const size_t gx = (size_t)(row0 + r) * ld + xcol + c4;
    xv.x = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gx); xv.y = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gx + 1);
    xv.z = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gx + 2); xv.w = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gx + 3);
    if (kPass2) {
      const size_t gy = (size_t)(row0 + r) * p.ld_do + head * kHD + c4;  // Y = dO
      yv.x = bf16_pair_to_f32(p.do_hi, p.do_lo, gy); yv.y = bf16_pair_to_f32(p.do_hi, p.do_lo, gy + 1);
      yv.z = bf16_pair_to_f32(p.do_hi, p.do_lo, gy + 2); yv.w = bf16_pair_to_f32(p.do_hi, p.do_lo, gy + 3);
    } else {
      const size_t gy = (size_t)(row0 + r) * ld + vc + c4;               // Y = V
      yv.x = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gy); yv.y = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gy + 1);
      yv.z = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gy + 2); yv.w = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gy + 3);
    }
    *reinterpret_cast<float4*>(&sm.X[r * kStride + c4]) = xv;
    *reinterpret_cast<float4*>(&sm.Y[r * kStride + c4]) = yv;
  }
  __syncthreads();

  for (int o0 = warp * kR; o0 < S; o0 += 8 * kR) {
    // ---- a, b vectors of the R outer rows: lane l keeps dims 4l..4l+3 in registers (broadcast by shuffle) ----
    float4 areg[kR], breg[kR];
#pragma unroll
    for (int r = 0; r < kR; ++r) {
      const int o = o0 + r;
      float4 av = make_float4(0.f, 0.f, 0.f, 0.f), bv = av;
      if (o < S) {
        const size_t ga = (size_t)(row0 + o) * ld + (kPass2 ? kc : qc) + lane * 4;
        av.x = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, ga); av.y = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, ga + 1);
        av.z = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, ga + 2); av.w = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, ga + 3);
        if (kPass2) {
          const size_t gb = (size_t)(row0 + o) * ld + vc + lane * 4;  // b = v_j
          bv.x = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gb); bv.y = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gb + 1);
          bv.z = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gb + 2); bv.w = bf16_pair_to_f32(p.qkv_hi, p.qkv_lo, gb + 3);
        } else {
          const size_t gb = (size_t)(row0 + o) * p.ld_do + head * kHD + lane * 4;  // b = dO_i
          bv.x = bf16_pair_to_f32(p.do_hi, p.do_lo, gb); bv.y = bf16_pair_to_f32(p.do_hi, p.do_lo, gb + 1);
          bv.z = bf16_pair_to_f32(p.do_hi, p.do_lo, gb + 2); bv.w = bf16_pair_to_f32(p.do_hi, p.do_lo, gb + 3);
        }
      }
      areg[r] = av;
      breg[r] = bv;
    }

    // ---- s = a . X_c, t = b . Y_c for this lane's inner indices c = lane + 32 k ----
    float s[kR][kInnerPerLane], t[kR][kInnerPerLane];
#pragma unroll
    for (int r = 0; r < kR; ++r)
#pragma unroll
      for (int k = 0; k < kInnerPerLane; ++k) s[r][k] = t[r][k] = 0.f;
#pragma unroll 2
    for (int d = 0; d < kHD; d += 4) {
      float4 av[kR], bv[kR];
#pragma unroll
      for (int r = 0; r < kR; ++r) {
        const int src = d >> 2;
        av[r].x = __shfl_sync(0xffffffffu, areg[r].x, src); av[r].y = __shfl_sync(0xffffffffu, areg[r].y, src);
        av[r].z = __shfl_sync(0xffffffffu, areg[r].z, src); av[r].w = __shfl_sync(0xffffffffu, areg[r].w, src);
        bv[r].x = __shfl_sync(0xffffffffu, breg[r].x, src); bv[r].y = __shfl_sync(0xffffffffu, breg[r].y, src);
        bv[r].z = __shfl_sync(0xffffffffu, breg[r].z, src); bv[r].w = __shfl_sync(0xffffffffu, breg[r].w, src);
      }
#pragma unroll
      for (int k = 0; k < kInnerPerLane; ++k) {
        const int c = lane + 32 * k;
        if (c < S) {
          const float4 xv = *reinterpret_cast<const float4*>(&sm.X[c * kStride + d]);
          const float4 yv = *reinterpret_cast<const float4*>(&sm.Y[c * kStride + d]);
#pragma unroll
          for (int r = 0; r < kR; ++r) {
            s[r][k] = fmaf(av[r].x, xv.x, fmaf(av[r].y, xv.y, fmaf(av[r].z, xv.z, fmaf(av[r].w, xv.w, s[r][k]))));
            t[r][k] = fmaf(bv[r].x, yv.x, fmaf(bv[r].y, yv.y, fmaf(bv[r].z, yv.z, fmaf(bv[r].w, yv.w, t[r][k]))));
          }
        }
      }
    }

    // ---- probabilities and dS (overwrites s with p and t with ds) ----
#pragma unroll
    for (int r = 0; r < kR; ++r) {
      const int o = o0 + r;
      if (!kPass2) {
        float mx = -INFINITY;
#pragma unroll
        for (int k = 0; k < kInnerPerLane; ++k)
          if (lane + 32 * k < S) mx = fmaxf(mx, s[r][k] * scale);
        mx = warp_max_f(mx);
        float l = 0.f;
#pragma unroll
        for (int k = 0; k < kInnerPerLane; ++k) {
          s[r][k] = (lane + 32 * k < S) ? __expf(s[r][k] * scale - mx) : 0.f;
          l += s[r][k];
        }
        l = warp_sum_f(l);
        const float inv = 1.0f / l;
        float dl = 0.f;
#pragma unroll
        for (int k = 0; k < kInnerPerLane; ++k) {
          s[r][k] *= inv;
          dl += s[r][k] * t[r][k];
        }
        dl = warp_sum_f(dl);
#pragma unroll
        for (int k = 0; k < kInnerPerLane; ++k) t[r][k] = s[r][k] * (t[r][k] - dl) * scale;
        if (lane == 0 && o < S) {
          sm.stat_m[o] = mx;
          sm.stat_l[o] = l;
          sm.stat_d[o] = dl;
        }
      } else {
#pragma unroll
        for (int k = 0; k < kInnerPerLane; ++k) {
          const int c = lane + 32 * k;
          if (c < S) {
            const float pv = __expf(s[r][k] * scale - sm.stat_m[c]) / sm.stat_l[c];
            t[r][k] = pv * (t[r][k] - sm.stat_d[c]) * scale;
            s[r][k] = pv;
          } else {
            s[r][k] = t[r][k] = 0.f;
          }
        }
      }
    }

    // ---- out1 = sum_c ds_c X_c ; out2 = sum_c p_c Y_c (pass 2 only); lane l owns dims 4l..4l+3 ----
    float4 o1[kR], o2[kR];
#pragma unroll
    for (int r = 0; r < kR; ++r) o1[r] = o2[r] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < kInnerPerLane; ++k) {
      const int cbase = 32 * k;
      const int cnt = min(32, S - cbase);
      for (int src = 0; src < cnt; ++src) {
        const int c = cbase + src;
        const float4 xv = *reinterpret_cast<const float4*>(&sm.X[c * kStride + lane * 4]);
        float4 yv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (kPass2) yv = *reinterpret_cast<const float4*>(&sm.Y[c * kStride + lane * 4]);
#pragma unroll
        for (int r = 0; r < kR; ++r) {
          const float dsv = __shfl_sync(0xffffffffu, t[r][k], src);
          o1[r].x = fmaf(dsv, xv.x, o1[r].x); o1[r].y = fmaf(dsv, xv.y, o1[r].y);
          o1[r].z = fmaf(dsv, xv.z, o1[r].z); o1[r].w = fmaf(dsv, xv.w, o1[r].w);
          if (kPass2) {
            const float pv = __shfl_sync(0xffffffffu, s[r][k], src);
            o2[r].x = fmaf(pv, yv.x, o2[r].x); o2[r].y = fmaf(pv, yv.y, o2[r].y);
            o2[r].z = fmaf(pv, yv.z, o2[r].z); o2[r].w = fmaf(pv, yv.w, o2[r].w);
          }
        }
      }
    }
    // ---- store: pass 1 -> dQ ; pass 2 -> dK, dV   (bf16 hi/lo planes in the QKV layout) ----
#pragma unroll
    for (int r = 0; r < kR; ++r) {
      const int o = o0 + r;
      if (o >= S) continue;
      uint32_t h0, l0, h1, l1;
      const size_t g1 = (size_t)(row0 + o) * ld + (kPass2 ? kc : qc) + lane * 4;
      split_bf16x2(o1[r].x, o1[r].y, h0, l0);
      split_bf16x2(o1[r].z, o1[r].w, h1, l1);
      *reinterpret_cast<uint2*>(p.dqkv_hi + g1) = make_uint2(h0, h1);
      if (p.dqkv_lo) *reinterpret_cast<uint2*>(p.dqkv_lo + g1) = make_uint2(l0, l1);
      if (kPass2) {
        const size_t g2 = (size_t)(row0 + o) * ld + vc + lane * 4;
        split_bf16x2(o2[r].x, o2[r].y, h0, l0);
        split_bf16x2(o2[r].z, o2[r].w, h1, l1);
        *reinterpret_cast<uint2*>(p.dqkv_hi + g2) = make_uint2(h0, h1);
        if (p.dqkv_lo) *reinterpret_cast<uint2*>(p.dqkv_lo + g2) = make_uint2(l0, l1);
      }
    }
    __syncwarp();
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256, 1) attention_bwd_kernel(const AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  AttnBwdSmem& sm = *reinterpret_cast<AttnBwdSmem*>((reinterpret_cast<uintptr_t>(smem_raw) + 15) & ~uintptr_t(15));
  const int head = blockIdx.x, seq = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  attn_bwd_pass<false>(sm, p, seq, head, warp, lane);
  attn_bwd_pass<true>(sm, p, seq, head, warp, lane);
}


}  // namespace

cudaError_t configure_attention_bwd_kernel() {
  return cudaFuncSetAttribute(attention_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(AttnBwdSmem) + 16);
}

cudaError_t launch_attention_bwd(const AttnBwdParams& p, cudaStream_t stream) {
  if (p.seq_len > kMaxS || p.seq_len < 1) {
    set_last_error("launch_attention_bwd: unsupported seq_len %d", p.seq_len);
    return cudaErrorInvalidValue;
  }
  dim3 grid(p.num_heads, p.num_seqs);
  attention_bwd_kernel<<<grid, 256, sizeof(AttnBwdSmem) + 16, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace cmdi
