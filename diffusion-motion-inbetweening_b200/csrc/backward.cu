// Input-VJP pieces of the denoiser for reconstruction guidance (reference: diffusion/gaussian_diffusion.py:405-425,
//   g = d/dz sum((x_obs - x0_hat(z))^2 * M) -- a backward pass through ClassifierFreeSampleModel(MDM) w.r.t. its input).
//
// Only dX is needed (no weight gradients).  The matrix products of the backward pass (dX = dY W for every linear)
// run on the same wgmma linear kernels as the forward pass, against transposed weight planes; this file holds
// the rest:
//   guidance_seed_kernel   dL/dx0_hat = -2 (x_obs - x0_hat) * M, split over the CFG cond / uncond outputs
//   layernorm512_bwd       dX of LayerNorm from the stashed pre-norm input
//   transpose_split        W[R,C] fp32 -> W^T bf16 hi/lo planes (once per weight load)
//
// The attention backward itself runs on the tensor cores (attention_bwd_tc.cu).
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
// guidance seed on the frame-major layout [B*L (x2 when cfg), D_pad]
// ---------------------------------------------------------------------------------------------
template <bool F16>
__global__ void __launch_bounds__(256) guidance_seed_kernel(const GuidanceSeedParams p) {
  const size_t n = (size_t)p.B * p.L * p.D_pad;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % p.D_pad);
    const int b = (int)(i / ((size_t)p.L * p.D_pad));
    float gc = 0.f, gu = 0.f;
    if (c < p.D) {
      float hat = p.model_out[i];
      float s = 1.f;
      if (p.cfg) {
        const float u = p.model_out[i + n];
        s = p.text_scale[b];
        hat = __fadd_rn(u, __fmul_rn(s, __fsub_rn(hat, u)));  // x0_hat = u + s (c - u)   (cfg_sampler.py:35)
      }
      const float m = p.obs_mask[i] ? 1.f : 0.f;
      const float G = -2.f * (p.x_obs[i] - hat) * m;  // d/dx0_hat of ((x_obs - x0_hat)^2 * M)
      gc = p.cfg ? s * G : G;
      gu = F16 ? __fsub_rn(G, __fmul_rn(G, s)) : (1.f - s) * G;
    }
    if constexpr (F16) {
      const int l = (int)((i / p.D_pad) % p.L);
      __half* seed = reinterpret_cast<__half*>(p.seed_hi);
      seed[((size_t)b * p.row_period + p.row_lo + l) * p.D_pad + c] = __float2half_rn(gc);
      if (p.cfg) seed[((size_t)(b + p.B) * p.row_period + p.row_lo + l) * p.D_pad + c] = __float2half_rn(gu);
      continue;
    }
    __nv_bfloat16 h, l;
    split_bf16(gc, h, l);
    p.seed_hi[i] = h;
    if (p.seed_lo) p.seed_lo[i] = l;
    if (p.cfg) {
      split_bf16(gu, h, l);
      p.seed_hi[i + n] = h;
      if (p.seed_lo) p.seed_lo[i + n] = l;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm backward (dX only): y = (v - mean) * rstd * gamma + beta
//   g = dY * gamma ;  dV = rstd * (g - mean(g) - xhat * mean(g * xhat))
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) layernorm512_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ v,
                                                               const float* __restrict__ gamma, float eps, int rows,
                                                               float* __restrict__ dv, __nv_bfloat16* __restrict__ dv_hi,
                                                               __nv_bfloat16* __restrict__ dv_lo) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float4* vs = reinterpret_cast<const float4*>(v + (size_t)row * 512);
  const float4* ds = reinterpret_cast<const float4*>(dy + (size_t)row * 512);
  float4 x[4], g[4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    x[i] = vs[i * 32 + lane];
    s += (x[i].x + x[i].y) + (x[i].z + x[i].w);
  }
  const float mean = warp_sum_f(s) * (1.0f / 512.0f);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    x[i].x -= mean; x[i].y -= mean; x[i].z -= mean; x[i].w -= mean;
    q += (x[i].x * x[i].x + x[i].y * x[i].y) + (x[i].z * x[i].z + x[i].w * x[i].w);
  }
  const float rstd = rsqrtf(warp_sum_f(q) * (1.0f / 512.0f) + eps);
  float m1 = 0.f, m2 = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int col = (i * 32 + lane) * 4;
    const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma + col));
    const float4 d = ds[i * 32 + lane];
    x[i].x *= rstd; x[i].y *= rstd; x[i].z *= rstd; x[i].w *= rstd;  // xhat
    g[i].x = d.x * gm.x; g[i].y = d.y * gm.y; g[i].z = d.z * gm.z; g[i].w = d.w * gm.w;
    m1 += (g[i].x + g[i].y) + (g[i].z + g[i].w);
    m2 += (g[i].x * x[i].x + g[i].y * x[i].y) + (g[i].z * x[i].z + g[i].w * x[i].w);
  }
  m1 = warp_sum_f(m1) * (1.0f / 512.0f);
  m2 = warp_sum_f(m2) * (1.0f / 512.0f);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int col = (i * 32 + lane) * 4;
    float4 o;
    o.x = rstd * (g[i].x - m1 - x[i].x * m2);
    o.y = rstd * (g[i].y - m1 - x[i].y * m2);
    o.z = rstd * (g[i].z - m1 - x[i].z * m2);
    o.w = rstd * (g[i].w - m1 - x[i].w * m2);
    reinterpret_cast<float4*>(dv + (size_t)row * 512)[i * 32 + lane] = o;
    uint32_t h0, l0, h1, l1;
    split_bf16x2(o.x, o.y, h0, l0);
    split_bf16x2(o.z, o.w, h1, l1);
    *reinterpret_cast<uint2*>(dv_hi + (size_t)row * 512 + col) = make_uint2(h0, h1);
    if (dv_lo) *reinterpret_cast<uint2*>(dv_lo + (size_t)row * 512 + col) = make_uint2(l0, l1);
  }
}

// ---------------------------------------------------------------------------------------------
// W[R, C] fp32 -> (W^T)[C, R] bf16 hi/lo planes with row pitch ld_out (zero padded)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) transpose_split_kernel(const float* __restrict__ w, int R, int C,
                                                              __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                                              int ld_out) {
  __shared__ float tile[32][33];
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty + i * 8, c = c0 + tx;
    tile[ty + i * 8][tx] = (r < R && c < C) ? w[(size_t)r * C + c] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + i * 8, r = r0 + tx;  // output row = c, output column = r
    if (c < C && r < ld_out) {
      __nv_bfloat16 h, l;
      split_bf16(r < R ? tile[tx][ty + i * 8] : 0.f, h, l);
      hi[(size_t)c * ld_out + r] = h;
      lo[(size_t)c * ld_out + r] = l;
    }
  }
}

}  // namespace

cudaError_t launch_guidance_seed(const GuidanceSeedParams& p, cudaStream_t stream) {
  const size_t n = (size_t)p.B * p.L * p.D_pad;
  size_t grid = (n + 255) / 256;
  if (grid > 132 * 16) grid = 132 * 16;
  if (p.f16) guidance_seed_kernel<true><<<(unsigned)grid, 256, 0, stream>>>(p);
  else guidance_seed_kernel<false><<<(unsigned)grid, 256, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_layernorm512_bwd(const float* dy, const float* v, const float* gamma, float eps, int rows, float* dv,
                                    __nv_bfloat16* dv_hi, __nv_bfloat16* dv_lo, cudaStream_t stream) {
  layernorm512_bwd_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(dy, v, gamma, eps, rows, dv, dv_hi, dv_lo);
  return cudaGetLastError();
}


cudaError_t launch_transpose_split(const float* w, int R, int C, __nv_bfloat16* hi, __nv_bfloat16* lo, int ld_out,
                                   cudaStream_t stream) {
  dim3 grid((C + 31) / 32, (ld_out + 31) / 32), block(32, 8);
  transpose_split_kernel<<<grid, block, 0, stream>>>(w, R, C, hi, lo, ld_out);
  return cudaGetLastError();
}

}  // namespace cmdi
