// Row / elementwise kernels of the MDM_UNET denoiser (reference: model/mdm_unet.py; SURVEY.md 8f-4, 8f-1).
//
// Activations are channel-last [rows, C] with a HALO layout: sequence b of a level with L positions occupies rows
// b * Lp .. b * Lp + Lp - 1 with Lp = 256 >> level (L = 224 >> level), position l at row b * Lp + 2 + l; the rows before
// and after a sequence's positions are zero.  A Conv1d(k = 5, padding = 2) is then a GEMM whose reduction walks five
// row-shifted views of the same matrix (gemm2.cu, LinearParams::num_taps), the zero rows are the convolution's padding,
// and with Lp halving per level the stride-2 convolutions become stride-1 over row PAIRS (engine_unet.cu).
//
//   unet_input_kernel        x <- obs_x0 * M + x * ~M ; cat([x, M])      mdm_unet.py:778-783 (+ the 224-frame padding :817)
//   unet_emb_kernel          emb = time_embed(pe[t]) (+ embed_text(cond))  mdm_unet.py:794-803
//   groupnorm_mish_kernel    GroupNorm(8) -> [AdaGN scale/shift] -> Mish -> [+ residual]   mdm_unet.py:33-100, :159-218
//   conv / conv-transpose weight re-layouts (once per weight load)
//
// Each kernel also has an F16 instantiation for CMDI_PRECISION_FP16, the arithmetic of CUDA autocast (fp16 planes in, fp16
// planes out, GroupNorm / AdaGN / Mish in fp32 between them; DESIGN.md section 3).
#include "common.cuh"
#include "kernels.h"

namespace cmdi {

namespace {

__device__ __forceinline__ float mish_dev(float x) { return x * tanhf(x > 20.0f ? x : log1pf(expf(x))); }

// ---------------------------------------------------------------------------------------------
// network input: planes [rows0, ld] (hi, lo), channels [0, D) = keyframe-blended x_t, [D, 2D) = mask (keyframe-
// conditioned models), zero elsewhere.  One thread per (sequence copy, frame, channel pair).
// ---------------------------------------------------------------------------------------------
template <bool F16>
__global__ void __launch_bounds__(256) unet_input_kernel(const UnetInputParams p) {
  const int pairs = p.ld / 2;
  const size_t total = (size_t)p.B * p.L * pairs;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int cp = (int)(i % pairs);
    const size_t fl = i / pairs;
    const int l = (int)(fl % p.L), b = (int)(fl / p.L);
    float v[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int c = cp * 2 + j;
      float val = 0.f;
      const size_t src = ((size_t)b * p.L + l) * p.D_pad;
      if (c < p.D) {
        val = p.x_t[src + c];
        if (p.obs_mask && p.obs_mask[src + c]) val = p.obs[src + c];
      } else if (p.obs_mask && c < 2 * p.D) {
        val = p.obs_mask[src + c - p.D] ? 1.0f : 0.0f;
      }
      v[j] = val;
    }
    uint32_t hw, lw = 0;
    if constexpr (F16) hw = pack_f16x2(v[0], v[1]);  // the blend is fp32; the first conv casts its input to fp16
    else split_bf16x2(v[0], v[1], hw, lw);
    for (int copy = 0; copy < p.copies; ++copy) {
      const size_t row = (size_t)(b + copy * p.B) * p.row_period + p.row_lo + l;
      *reinterpret_cast<uint32_t*>(p.out_hi + row * p.ld + cp * 2) = hw;
      if (!F16 && p.out_lo) *reinterpret_cast<uint32_t*>(p.out_lo + row * p.ld + cp * 2) = lw;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// emb[seq, :] = temb_table[tmap[t], :] + (cond_proj[seq % B] if seq < n_cond else uncond_proj)   -> bf16 planes [rows, 512]
// ---------------------------------------------------------------------------------------------
template <bool F16>
__global__ void __launch_bounds__(128) unet_emb_kernel(const TokenParams p) {
  const int seq = blockIdx.x;
  int t = *p.step_ptr;
  if (p.timestep_map) t = p.timestep_map[t];
  const int col = threadIdx.x * 4;
  float4 e = *reinterpret_cast<const float4*>(p.temb_table + (size_t)t * 512 + col);
  if (p.cond_proj) {
    const float* c = (seq < p.n_cond_seqs) ? p.cond_proj + (size_t)(seq % p.seq_len) * 512 : p.uncond_proj;  // seq_len carries B here
    const float4 cv = *reinterpret_cast<const float4*>(c + col);
    if constexpr (F16) {
      // fp16 + fp16 -> fp16; the unconditional row is embed_text(0) = the bias, cast to fp16
      e.x = round_f16(e.x + round_f16(cv.x)); e.y = round_f16(e.y + round_f16(cv.y));
      e.z = round_f16(e.z + round_f16(cv.z)); e.w = round_f16(e.w + round_f16(cv.w));
    } else {
      e.x += cv.x; e.y += cv.y; e.z += cv.z; e.w += cv.w;
    }
  }
  if constexpr (F16) {
    *reinterpret_cast<uint2*>(p.x_hi + (size_t)seq * 512 + col) = make_uint2(pack_f16x2(e.x, e.y), pack_f16x2(e.z, e.w));
    return;
  }
  uint32_t h01, l01, h23, l23;
  split_bf16x2(e.x, e.y, h01, l01);
  split_bf16x2(e.z, e.w, h23, l23);
  *reinterpret_cast<uint2*>(p.x_hi + (size_t)seq * 512 + col) = make_uint2(h01, h23);
  if (p.x_lo) *reinterpret_cast<uint2*>(p.x_lo + (size_t)seq * 512 + col) = make_uint2(l01, l23);
}

// ---------------------------------------------------------------------------------------------
// GroupNorm(groups of Cg channels over the L positions of one sequence) + optional AdaGN + Mish + optional residual.
// One CTA per (group, sequence): the [L, Cg] fp32 slab is staged in shared memory (<= 224 x 128 x 4 = 112 KB), the
// statistics are two-pass over that copy (mean, then centred squares: torch's group_norm numerics to fp32 rounding).
// ---------------------------------------------------------------------------------------------
template <bool F16>
__global__ void __launch_bounds__(512) groupnorm_mish_kernel(const GroupNormParams p) {
  extern __shared__ float slab[];  // [L][Cg]
  __shared__ float red[16];
  __shared__ float s_mean, s_rstd;
  const int g = blockIdx.x, b = blockIdx.y;
  const int Cg = p.C / p.groups, L = p.L;
  const int c0 = g * Cg;
  const size_t row0 = (size_t)b * p.row_period + p.row_lo;
  const int vec = Cg / 4;  // float4 per row
  const int n4 = L * vec;
  float sum = 0.f;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    const int l = i / vec, q = i - l * vec;
    const float4 v = *reinterpret_cast<const float4*>(p.y + (row0 + l) * p.ld_y + c0 + q * 4);
    reinterpret_cast<float4*>(slab)[i] = v;
    sum += (v.x + v.y) + (v.z + v.w);
  }
  auto block_sum = [&](float v) -> float {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    return t;
  };
  const float inv_n = 1.0f / (float)(L * Cg);
  const float mean = block_sum(sum) * inv_n;
  float sq = 0.f;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    const float4 v = reinterpret_cast<float4*>(slab)[i];
    const float a = v.x - mean, bb = v.y - mean, c = v.z - mean, d = v.w - mean;
    sq += (a * a + bb * bb) + (c * c + d * d);
  }
  const float rstd = rsqrtf(block_sum(sq) * inv_n + p.eps);
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    const int l = i / vec, q = i - l * vec;
    const int c = c0 + q * 4;
    const float4 v = reinterpret_cast<float4*>(slab)[i];
    const float4 gm = *reinterpret_cast<const float4*>(p.gamma + c);
    const float4 bt = *reinterpret_cast<const float4*>(p.beta + c);
    float o[4] = {(v.x - mean) * rstd * gm.x + bt.x, (v.y - mean) * rstd * gm.y + bt.y, (v.z - mean) * rstd * gm.z + bt.z,
                  (v.w - mean) * rstd * gm.w + bt.w};
    if (p.ada) {
      // cond = time_mlp(t) as [scale | shift] (mdm_unet.py:95-99): x * (1 + scale) + shift
      const float4 sc = *reinterpret_cast<const float4*>(p.ada + (size_t)b * p.ld_ada + c);
      const float4 sh = *reinterpret_cast<const float4*>(p.ada + (size_t)b * p.ld_ada + p.C + c);
      if constexpr (F16) {
        // scale / shift are fp16: `1 + scale` is an fp16 op, the product and sum with the fp32 GroupNorm output are fp32
        o[0] = __fadd_rn(__fmul_rn(o[0], round_f16(1.0f + sc.x)), sh.x); o[1] = __fadd_rn(__fmul_rn(o[1], round_f16(1.0f + sc.y)), sh.y);
        o[2] = __fadd_rn(__fmul_rn(o[2], round_f16(1.0f + sc.z)), sh.z); o[3] = __fadd_rn(__fmul_rn(o[3], round_f16(1.0f + sc.w)), sh.w);
      } else {
        o[0] = o[0] * (1.0f + sc.x) + sh.x; o[1] = o[1] * (1.0f + sc.y) + sh.y;
        o[2] = o[2] * (1.0f + sc.z) + sh.z; o[3] = o[3] * (1.0f + sc.w) + sh.w;
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = mish_dev(o[j]);
    const size_t row = row0 + l;
    if (p.res_f32) {
      const float4 r = *reinterpret_cast<const float4*>(p.res_f32 + row * p.ld_res + c);
      if constexpr (F16) {
        o[0] = __fadd_rn(o[0], r.x); o[1] = __fadd_rn(o[1], r.y); o[2] = __fadd_rn(o[2], r.z); o[3] = __fadd_rn(o[3], r.w);
      } else {
        o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
      }
    } else if (F16 && p.res_hi) {
      // an fp16 identity residual (a Downsample1d output): exact in fp32
      const uint2 rh = *reinterpret_cast<const uint2*>(p.res_hi + row * p.ld_res + c);
      const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&rh.x));
      const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&rh.y));
      o[0] = __fadd_rn(o[0], a.x); o[1] = __fadd_rn(o[1], a.y); o[2] = __fadd_rn(o[2], b.x); o[3] = __fadd_rn(o[3], b.y);
    } else if (p.res_hi) {
      const uint2 rh = *reinterpret_cast<const uint2*>(p.res_hi + row * p.ld_res + c);
      const uint2 rl = *reinterpret_cast<const uint2*>(p.res_lo + row * p.ld_res + c);
      o[0] += __uint_as_float(rh.x << 16) + __uint_as_float(rl.x << 16);
      o[1] += __uint_as_float(rh.x & 0xffff0000u) + __uint_as_float(rl.x & 0xffff0000u);
      o[2] += __uint_as_float(rh.y << 16) + __uint_as_float(rl.y << 16);
      o[3] += __uint_as_float(rh.y & 0xffff0000u) + __uint_as_float(rl.y & 0xffff0000u);
    }
    if constexpr (F16) {
      *reinterpret_cast<uint2*>(p.out_hi + row * p.ld_out + c) = make_uint2(pack_f16x2(o[0], o[1]), pack_f16x2(o[2], o[3]));
      if (p.out_f32) *reinterpret_cast<float4*>(p.out_f32 + row * p.ld_out_f32 + c) = make_float4(o[0], o[1], o[2], o[3]);
      continue;
    }
    uint32_t h01, l01, h23, l23;
    split_bf16x2(o[0], o[1], h01, l01);
    split_bf16x2(o[2], o[3], h23, l23);
    *reinterpret_cast<uint2*>(p.out_hi + row * p.ld_out + c) = make_uint2(h01, h23);
    if (p.out_lo) *reinterpret_cast<uint2*>(p.out_lo + row * p.ld_out + c) = make_uint2(l01, l23);
  }
}

// Conv1d weight [Co, Ci, k] fp32 -> tap-major planes [Co, k * Cp] (Cp >= Ci, zero padded):  W2[o, j * Cp + c] = W[o, c, j]
template <bool F16>
__global__ void conv_weight_planes_kernel(const float* __restrict__ w, int Co, int Ci, int k, int Cp, __nv_bfloat16* hi,
                                          __nv_bfloat16* lo, int ld) {
  const size_t total = (size_t)Co * k * Cp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cp);
    const int j = (int)((i / Cp) % k);
    const int o = (int)(i / ((size_t)Cp * k));
    const float v = c < Ci ? w[((size_t)o * Ci + c) * k + j] : 0.f;
    if constexpr (F16) {
      reinterpret_cast<__half*>(hi)[(size_t)o * ld + (size_t)j * Cp + c] = __float2half_rn(v);
      continue;
    }
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[(size_t)o * ld + (size_t)j * Cp + c] = h;
    lo[(size_t)o * ld + (size_t)j * Cp + c] = l;
  }
}

// ConvTranspose1d(k = 4, s = 2, p = 1) weight [Ci, Co, 4] -> planes [2 Co, 3 Ci]: even outputs (rows [0, Co)) use
// in[m - 1] W[..3] + in[m] W[..1], odd outputs (rows [Co, 2 Co)) use in[m] W[..2] + in[m + 1] W[..0]; tap blocks are
// ordered (m - 1, m, m + 1) and the two unused blocks are zero.
template <bool F16>
__global__ void convt_weight_planes_kernel(const float* __restrict__ w, int Ci, int Co, __nv_bfloat16* hi, __nv_bfloat16* lo, int ld) {
  const size_t total = (size_t)2 * Co * 3 * Ci;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % Ci);
    const int tap = (int)((i / Ci) % 3);
    const int n = (int)(i / ((size_t)3 * Ci));
    const int o = n % Co, odd = n / Co;
    int j = -1;
    if (!odd) j = tap == 0 ? 3 : (tap == 1 ? 1 : -1);
    else j = tap == 1 ? 2 : (tap == 2 ? 0 : -1);
    const float v = j >= 0 ? w[((size_t)c * Co + o) * 4 + j] : 0.f;
    if constexpr (F16) {
      reinterpret_cast<__half*>(hi)[(size_t)n * ld + (size_t)tap * Ci + c] = __float2half_rn(v);
      continue;
    }
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[(size_t)n * ld + (size_t)tap * Ci + c] = h;
    lo[(size_t)n * ld + (size_t)tap * Ci + c] = l;
  }
}

// autocast Linear on CUDA cores (embed_text, once per call): one warp per output element, K split across lanes
__global__ void __launch_bounds__(256) small_linear_f16_kernel(const float* __restrict__ in, const float* __restrict__ W,
                                                               const float* __restrict__ bias, float* __restrict__ out, int rows,
                                                               int N, int K) {
  const long long w = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= (long long)rows * N) return;
  const int r = (int)(w / N), n = (int)(w % N);
  const float* a = in + (size_t)r * K;
  const float* b = W + (size_t)n * K;
  float s = 0.f;
  for (int k = lane; k < K; k += 32) s = fmaf(round_f16(a[k]), round_f16(b[k]), s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[(size_t)r * N + n] = round_f16(s + (bias ? round_f16(bias[n]) : 0.f));
}

// ---------------------------------------------------------------------------------------------
// Input-VJP (CMDI_PRECISION_FP16 reconstruction guidance): the backward of one groupnorm_mish launch.  Same CTA shape as
// the forward: the stashed [L, Cg] slab in shared memory, the same two-pass statistics, then with
//   xhat = (y - mean) rstd,  a = xhat gamma + beta,  b = a fp16(1 + scale) + shift (AdaGN) or a,  o = Mish(b):
//   g = dO Mish'(b) [fp16(1 + scale)] gamma,  dY = rstd (g - mean(g) - xhat mean(g xhat))     (fp32; dY rounded to fp16)
// Mish' as PyTorch's mish_backward: tanh(softplus(b)) + b sigmoid(b) (1 - tanh(softplus(b))^2).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float mish_grad_dev(float x) {
  const float sg = 1.0f / (1.0f + expf(-x));
  const float ts = tanhf(log1pf(expf(x)));
  return ts + x * sg * (1.0f - ts * ts);
}

__global__ void __launch_bounds__(512) groupnorm_mish_bwd_kernel(const GroupNormBwdParams p) {
  extern __shared__ float slab[];  // [L][Cg]
  __shared__ float red[16];
  const int g = blockIdx.x, b = blockIdx.y;
  const int Cg = p.C / p.groups, L = p.L;
  const int c0 = g * Cg;
  const size_t seq0 = (size_t)b * p.row_period;
  const size_t row0 = seq0 + p.row_lo;
  const int vec = Cg / 4;
  const int n4 = L * vec;
  auto ld_h4 = [](const __nv_bfloat16* base, size_t off) -> float4 {
    const uint2 h = *reinterpret_cast<const uint2*>(base + off);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&h.x));
    const float2 c = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
    return make_float4(a.x, a.y, c.x, c.y);
  };
  float sum = 0.f;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    const int l = i / vec, q = i - l * vec;
    const float4 v = ld_h4(p.y, (row0 + l) * p.ld_y + c0 + q * 4);
    reinterpret_cast<float4*>(slab)[i] = v;
    sum += (v.x + v.y) + (v.z + v.w);
  }
  auto block_sum = [&](float v) -> float {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    return t;
  };
  const float inv_n = 1.0f / (float)(L * Cg);
  const float mean = block_sum(sum) * inv_n;
  float sq = 0.f;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    const float4 v = reinterpret_cast<float4*>(slab)[i];
    const float a = v.x - mean, bb = v.y - mean, c = v.z - mean, d = v.w - mean;
    sq += (a * a + bb * bb) + (c * c + d * d);
  }
  const float rstd = rsqrtf(block_sum(sq) * inv_n + p.eps);
  // g and xhat of element j of slab entry i (pass 1 also folds dout_add into dout)
  auto grad_of = [&](int i, bool first, float (&gg)[4], float (&xh)[4]) {
    const int l = i / vec, q = i - l * vec;
    const int c = c0 + q * 4;
    const size_t row = row0 + l;
    const float4 v = reinterpret_cast<float4*>(slab)[i];
    const float4 gm = *reinterpret_cast<const float4*>(p.gamma + c);
    const float4 bt = *reinterpret_cast<const float4*>(p.beta + c);
    float4 d4;
    if (p.dout_h) {
      d4 = ld_h4(p.dout_h, row * p.ld_dout + c);
    } else {
      d4 = *reinterpret_cast<const float4*>(p.dout + row * p.ld_dout + c);
      if (first && p.dout_add) {
        const float4 a4 = *reinterpret_cast<const float4*>(p.dout_add + row * p.ld_add + c);
        d4 = make_float4(__fadd_rn(d4.x, a4.x), __fadd_rn(d4.y, a4.y), __fadd_rn(d4.z, a4.z), __fadd_rn(d4.w, a4.w));
        *reinterpret_cast<float4*>(p.dout + row * p.ld_dout + c) = d4;
      }
    }
    const float vv[4] = {v.x, v.y, v.z, v.w}, gmv[4] = {gm.x, gm.y, gm.z, gm.w}, btv[4] = {bt.x, bt.y, bt.z, bt.w};
    const float dv[4] = {d4.x, d4.y, d4.z, d4.w};
    float s1[4] = {1.f, 1.f, 1.f, 1.f}, sh[4] = {0.f, 0.f, 0.f, 0.f};
    if (p.ada) {
      const float4 sc = *reinterpret_cast<const float4*>(p.ada + (size_t)b * p.ld_ada + c);
      const float4 sf = *reinterpret_cast<const float4*>(p.ada + (size_t)b * p.ld_ada + p.C + c);
      s1[0] = round_f16(1.0f + sc.x); s1[1] = round_f16(1.0f + sc.y); s1[2] = round_f16(1.0f + sc.z); s1[3] = round_f16(1.0f + sc.w);
      sh[0] = sf.x; sh[1] = sf.y; sh[2] = sf.z; sh[3] = sf.w;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      xh[j] = (vv[j] - mean) * rstd;
      const float a = (vv[j] - mean) * rstd * gmv[j] + btv[j];  // the forward's expression
      const float bv = p.ada ? __fadd_rn(__fmul_rn(a, s1[j]), sh[j]) : a;
      float t = dv[j] * mish_grad_dev(bv);
      if (p.ada) t = t * s1[j];
      gg[j] = t * gmv[j];
    }
  };
  float m1 = 0.f, m2 = 0.f;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    float gg[4], xh[4];
    grad_of(i, true, gg, xh);
    m1 += (gg[0] + gg[1]) + (gg[2] + gg[3]);
    m2 += (gg[0] * xh[0] + gg[1] * xh[1]) + (gg[2] * xh[2] + gg[3] * xh[3]);
  }
  m1 = block_sum(m1) * inv_n;  // (block_sum's barriers also order pass 1's dout write-back before pass 2's reads)
  m2 = block_sum(m2) * inv_n;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    float gg[4], xh[4];
    grad_of(i, false, gg, xh);
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = rstd * (gg[j] - m1 - xh[j] * m2);
    const int l = i / vec, q = i - l * vec;
    *reinterpret_cast<uint2*>(p.dy + (row0 + l) * p.ld_dy + c0 + q * 4) = make_uint2(pack_f16x2(o[0], o[1]), pack_f16x2(o[2], o[3]));
  }
  // the halo rows of this sequence (the next convolution's zero padding)
  const int halo = (p.row_period - L) * vec;
  for (int i = threadIdx.x; i < halo; i += blockDim.x) {
    const int h = i / vec, q = i - h * vec;
    const int r = h < p.row_lo ? h : L + h;
    *reinterpret_cast<uint2*>(p.dy + (seq0 + r) * p.ld_dy + c0 + q * 4) = make_uint2(0u, 0u);
  }
}

__global__ void dgrad_weight_planes_kernel(const DgradWeightParams p) {
  const size_t total = (size_t)p.N * p.taps * p.Kp;
  const __half* src = reinterpret_cast<const __half*>(p.src);
  __half* dst = reinterpret_cast<__half*>(p.dst);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % p.Kp);
    const int t = (int)((i / p.Kp) % p.taps);
    const int n = (int)(i / ((size_t)p.Kp * p.taps));
    __half v = __float2half_rn(0.f);
    if (p.kind == 0) {
      if (n < p.Ci && k < p.Co) v = src[(size_t)k * p.ld_src + (size_t)t * p.Cp_src + n];
    } else if (p.kind == 1) {
      const int C = p.Ci, ci = n % C, odd = n / C;
      // even input positions 2q: W1^T dOut[q]; odd 2q + 1: W2^T dOut[q] + W0^T dOut[q + 1]
      const int j = odd ? (t == 0 ? 2 : 0) : (t == 0 ? 1 : -1);
      if (j >= 0 && k < C) v = src[(size_t)k * p.ld_src + (size_t)j * p.Cp_src + ci];
    } else {
      // the forward's phase planes hold W[c, o, 3], W[c, o, 1] in row o (taps 0, 1) and W[c, o, 2], W[c, o, 0] in row C + o
      // (taps 1, 2)
      const int C = p.Ci, c = n, o = k;
      if (c < C && o < C) {
        const size_t even = (size_t)o * p.ld_src, odd = (size_t)(C + o) * p.ld_src;
        const size_t at[4] = {odd + 2 * (size_t)C + c, even + (size_t)C + c, odd + (size_t)C + c, even + c};
        v = src[at[t]];
      }
    }
    dst[(size_t)n * p.ld_dst + (size_t)t * p.Kp + k] = v;
  }
}

__global__ void __launch_bounds__(256) unet_input_grad_kernel(const float* __restrict__ xg, int ld, int num_seqs, int B, int L, int D,
                                                              int D_pad, int row_period, int row_lo, const uint8_t* __restrict__ obs_mask,
                                                              float* __restrict__ out) {
  const size_t total = (size_t)num_seqs * L * D_pad;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % D_pad);
    const size_t fl = i / D_pad;
    const int l = (int)(fl % L), q = (int)(fl / L);
    float v = 0.f;
    if (c < D) {
      v = xg[((size_t)q * row_period + row_lo + l) * ld + c];
      if (obs_mask && obs_mask[((size_t)(q % B) * L + l) * D_pad + c]) v = 0.f;  // x = obs_x0 M + x ~M (mdm_unet.py:781)
    }
    out[i] = v;
  }
}

inline dim3 grid_1d(size_t n, int block) {
  size_t g = (n + block - 1) / block;
  if (g > 132 * 32) g = 132 * 32;
  if (g < 1) g = 1;
  return dim3((unsigned)g);
}

}  // namespace

cudaError_t launch_unet_input(const UnetInputParams& p, cudaStream_t stream) {
  if (p.f16) unet_input_kernel<true><<<grid_1d((size_t)p.B * p.L * (p.ld / 2), 256), 256, 0, stream>>>(p);
  else unet_input_kernel<false><<<grid_1d((size_t)p.B * p.L * (p.ld / 2), 256), 256, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_unet_emb(const TokenParams& p, cudaStream_t stream, bool f16) {
  if (f16) unet_emb_kernel<true><<<p.num_seqs, 128, 0, stream>>>(p);
  else unet_emb_kernel<false><<<p.num_seqs, 128, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t configure_groupnorm_kernel() {
  const cudaError_t e = cudaFuncSetAttribute(groupnorm_mish_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 256 * 4);
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(groupnorm_mish_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 256 * 4);
}

cudaError_t launch_groupnorm_mish(const GroupNormParams& p, int num_seqs, cudaStream_t stream) {
  const int Cg = p.C / p.groups;
  if (p.C % p.groups || Cg % 4 || (size_t)p.L * Cg * 4 > 224 * 256 * 4) {
    set_last_error("launch_groupnorm_mish: unsupported shape C=%d groups=%d L=%d", p.C, p.groups, p.L);
    return cudaErrorInvalidValue;
  }
  if (p.f16) groupnorm_mish_kernel<true><<<dim3(p.groups, num_seqs), 512, (size_t)p.L * Cg * 4, stream>>>(p);
  else groupnorm_mish_kernel<false><<<dim3(p.groups, num_seqs), 512, (size_t)p.L * Cg * 4, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_conv_weight_planes(const float* w, int Co, int Ci, int k, int Cp, __nv_bfloat16* hi, __nv_bfloat16* lo, int ld,
                                      cudaStream_t stream, bool f16) {
  if (f16) conv_weight_planes_kernel<true><<<grid_1d((size_t)Co * k * Cp, 256), 256, 0, stream>>>(w, Co, Ci, k, Cp, hi, lo, ld);
  else conv_weight_planes_kernel<false><<<grid_1d((size_t)Co * k * Cp, 256), 256, 0, stream>>>(w, Co, Ci, k, Cp, hi, lo, ld);
  return cudaGetLastError();
}

cudaError_t launch_convt_weight_planes(const float* w, int Ci, int Co, __nv_bfloat16* hi, __nv_bfloat16* lo, int ld, cudaStream_t stream,
                                       bool f16) {
  if (f16) convt_weight_planes_kernel<true><<<grid_1d((size_t)2 * Co * 3 * Ci, 256), 256, 0, stream>>>(w, Ci, Co, hi, lo, ld);
  else convt_weight_planes_kernel<false><<<grid_1d((size_t)2 * Co * 3 * Ci, 256), 256, 0, stream>>>(w, Ci, Co, hi, lo, ld);
  return cudaGetLastError();
}

cudaError_t launch_small_linear_f16(const float* in, const float* W, const float* bias, float* out, int rows, int N, int K,
                                    cudaStream_t stream) {
  const long long warps = (long long)rows * N;
  small_linear_f16_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(in, W, bias, out, rows, N, K);
  return cudaGetLastError();
}

cudaError_t configure_groupnorm_bwd_kernel() {
  return cudaFuncSetAttribute(groupnorm_mish_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 256 * 4);
}

cudaError_t launch_groupnorm_mish_bwd(const GroupNormBwdParams& p, int num_seqs, cudaStream_t stream) {
  const int Cg = p.C / p.groups;
  if (p.C % p.groups || Cg % 4 || (size_t)p.L * Cg * 4 > 224 * 256 * 4 || (p.dout == nullptr) == (p.dout_h == nullptr) ||
      (p.dout_add && !p.dout)) {
    set_last_error("launch_groupnorm_mish_bwd: unsupported shape C=%d groups=%d L=%d or gradient inputs", p.C, p.groups, p.L);
    return cudaErrorInvalidValue;
  }
  groupnorm_mish_bwd_kernel<<<dim3(p.groups, num_seqs), 512, (size_t)p.L * Cg * 4, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_dgrad_weight_planes(const DgradWeightParams& p, cudaStream_t stream) {
  dgrad_weight_planes_kernel<<<grid_1d((size_t)p.N * p.taps * p.Kp, 256), 256, 0, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_unet_input_grad(const float* xg, int ld, int num_seqs, int B, int L, int D, int D_pad, int row_period, int row_lo,
                                   const uint8_t* obs_mask, float* out, cudaStream_t stream) {
  unet_input_grad_kernel<<<grid_1d((size_t)num_seqs * L * D_pad, 256), 256, 0, stream>>>(xg, ld, num_seqs, B, L, D, D_pad, row_period,
                                                                                        row_lo, obs_mask, out);
  return cudaGetLastError();
}

}  // namespace cmdi
