// Row-wise and elementwise kernels of the sampling path (HBM/L2-bound; coalesced, vectorised).
//
//   layernorm512           nn.TransformerEncoderLayer norm1/norm2 (post-norm)      mdm.py:107-114
//   token_rows             timestep(+text) token + PE[0]                           mdm.py:245-251,279-280
//   small_linear           TimestepEmbedder MLP / embed_text, once per loop        mdm.py:345-353,248-251
//   diffusion_step         p_mean_variance tail + p_sample / ddim_sample           gaussian_diffusion.py:352-534,656-713,1358-1416
//                          + ClassifierFreeSampleModel combine                     cfg_sampler.py:25-35
//                          + keyframe imputation blend                             gaussian_diffusion.py:427-435
//   layout converters      reference [B,D,1,L] <-> frame-major [B*L, D_pad]
//
// The step kernel uses explicit non-contracted fp32 intrinsics (__fmul_rn/__fadd_rn) in the
// reference's operation order so that, given the same denoiser output, it is bit-identical to
// the PyTorch CPU reference.
#include <curand_kernel.h>

#include "common.cuh"
#include "kernels.h"

namespace cmdi {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------
// LayerNorm over rows of 512 fp32: one warp per row, 16 values per lane (4 x float4, coalesced)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) layernorm512_kernel(const float* __restrict__ v, const float* __restrict__ gamma,
                                                           const float* __restrict__ beta, float eps, int rows,
                                                           float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_hi,
                                                           __nv_bfloat16* __restrict__ out_lo, float2* __restrict__ stats_out) {
  griddep_launch_dependents();
  griddep_wait();
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float4* src = reinterpret_cast<const float4*>(v + (size_t)row * 512);
  float4 x[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) x[i] = src[i * 32 + lane];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) s += (x[i].x + x[i].y) + (x[i].z + x[i].w);
  const float mean = warp_sum(s) * (1.0f / 512.0f);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float a = x[i].x - mean, b = x[i].y - mean, c = x[i].z - mean, d = x[i].w - mean;
    q += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(q) * (1.0f / 512.0f) + eps);
  if (stats_out && lane == 0) stats_out[row] = make_float2(mean, rstd);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int col = (i * 32 + lane) * 4;
    const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + col));
    const float4 bb = __ldg(reinterpret_cast<const float4*>(beta + col));
    float4 y;
    y.x = ln_apply(x[i].x, mean, rstd, g.x, bb.x);
    y.y = ln_apply(x[i].y, mean, rstd, g.y, bb.y);
    y.z = ln_apply(x[i].z, mean, rstd, g.z, bb.z);
    y.w = ln_apply(x[i].w, mean, rstd, g.w, bb.w);
    if (out_f32) reinterpret_cast<float4*>(out_f32 + (size_t)row * 512)[i * 32 + lane] = y;
    if (out_hi) {
      __nv_bfloat16 h0, l0, h1, l1, h2, l2, h3, l3;
      split_bf16(y.x, h0, l0); split_bf16(y.y, h1, l1); split_bf16(y.z, h2, l2); split_bf16(y.w, h3, l3);
      uint2 hw = make_uint2(pack_bf16x2(h0, h1), pack_bf16x2(h2, h3));
      *reinterpret_cast<uint2*>(out_hi + (size_t)row * 512 + col) = hw;
      if (out_lo) {
        uint2 lw = make_uint2(pack_bf16x2(l0, l1), pack_bf16x2(l2, l3));
        *reinterpret_cast<uint2*>(out_lo + (size_t)row * 512 + col) = lw;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// fp32 linear on CUDA cores: one warp per output element, K split across lanes
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) small_linear_kernel(const float* __restrict__ in, const float* __restrict__ W,
                                                           const float* __restrict__ bias, float* __restrict__ out, int rows,
                                                           int N, int K, int act) {
  const long long w = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (w >= (long long)rows * N) return;
  const int r = (int)(w / N), n = (int)(w % N);
  const float* a = in + (size_t)r * K;
  const float* b = W + (size_t)n * K;
  float s = 0.f;
  for (int k = lane; k < K; k += 32) s = fmaf(a[k], b[k], s);
  s = warp_sum(s);
  if (lane == 0) {
    if (bias) s += bias[n];
    if (act == 2) s = s / (1.0f + expf(-s));  // SiLU
    out[(size_t)r * N + n] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// conditioning token rows
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) token_rows_kernel(const TokenParams p) {
  griddep_launch_dependents();
  griddep_wait();
  const int seq = blockIdx.x;
  int t = *p.step_ptr;
  if (p.timestep_map) t = p.timestep_map[t];
  const int col = threadIdx.x * 4;
  float4 e = *reinterpret_cast<const float4*>(p.temb_table + (size_t)t * 512 + col);
  if (p.cond_proj) {
    // emb += embed_text(mask_cond(enc_text))   (mdm.py:250; uncond -> embed_text(0) = bias)
    const float* c = (seq < p.n_cond_seqs) ? p.cond_proj + (size_t)seq * 512 : p.uncond_proj;
    const float4 cv = *reinterpret_cast<const float4*>(c + col);
    e.x += cv.x; e.y += cv.y; e.z += cv.z; e.w += cv.w;
  }
  const float4 pe = *reinterpret_cast<const float4*>(p.pe0 + col);
  e.x += pe.x; e.y += pe.y; e.z += pe.z; e.w += pe.w;
  const size_t row = (size_t)seq * p.seq_len;
  *reinterpret_cast<float4*>(p.x_f32 + row * 512 + col) = e;
  __nv_bfloat16 h0, l0, h1, l1, h2, l2, h3, l3;
  split_bf16(e.x, h0, l0); split_bf16(e.y, h1, l1); split_bf16(e.z, h2, l2); split_bf16(e.w, h3, l3);
  *reinterpret_cast<uint2*>(p.x_hi + row * 512 + col) = make_uint2(pack_bf16x2(h0, h1), pack_bf16x2(h2, h3));
  if (p.x_lo) *reinterpret_cast<uint2*>(p.x_lo + row * 512 + col) = make_uint2(pack_bf16x2(l0, l1), pack_bf16x2(l2, l3));
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al. 2011) + Box-Muller: counter = (element index / 4, sample, stream, 0)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}
__device__ __forceinline__ float u01(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }
// four standard normals for the flat element indices 4*q .. 4*q+3 of sample `sample` on stream `stream_id`
__device__ __forceinline__ void philox_normal4(unsigned long long seed, unsigned long long stream_id, unsigned long long sample,
                                               unsigned long long q, float (&out)[4]) {
  const uint4 ctr = make_uint4((uint32_t)q, (uint32_t)sample, (uint32_t)stream_id,
                               (uint32_t)((q >> 32) | ((sample >> 32) << 8) | ((stream_id >> 32) << 20)));
  const uint4 r = philox4x32_10(ctr, make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const float rad0 = sqrtf(-2.0f * logf(u01(r.x))), rad1 = sqrtf(-2.0f * logf(u01(r.z)));
  float s0, c0, s1, c1;
  sincospif(2.0f * u01(r.y), &s0, &c0);
  sincospif(2.0f * u01(r.w), &s1, &c1);
  out[0] = rad0 * c0; out[1] = rad0 * s0; out[2] = rad1 * c1; out[3] = rad1 * s1;
}
// standard normal for flat element index `idx` (element idx & 3 of its quad)
__device__ __forceinline__ float philox_normal(unsigned long long seed, unsigned long long stream_id,
                                               unsigned long long sample, unsigned long long idx) {
  float v[4];
  philox_normal4(seed, stream_id, sample, idx >> 2, v);
  return v[idx & 3];
}

// ---------------------------------------------------------------------------------------------
// torch.randn-compatible stream.  ATen's normal_ kernel (aten/src/ATen/native/cuda/DistributionTemplates.h) runs
// G = 256 * grid threads; thread i initialises Philox4x32-10 with (seed, subsequence i, offset) and its j-th
// curand_normal4 call fills elements i + G * (4j + {0,1,2,3}).  So element e is component (e / G) & 3 of call
// (e / G) >> 2 of thread e % G: counter = (offset / 4 + call, thread), Box-Muller exactly as curand_normal4
// (the toolkit's own device functions are used so the bits match).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float aten_normal(unsigned long long seed, unsigned long long offset, unsigned int threads,
                                             unsigned long long e) {
  const unsigned long long thread = e % threads, r = e / threads;
  const unsigned long long blk = (offset >> 2) + (r >> 2);
  const uint4 ctr = make_uint4((uint32_t)blk, (uint32_t)(blk >> 32), (uint32_t)thread, (uint32_t)(thread >> 32));
  const uint4 x = curand_Philox4x32_10(ctr, make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const int comp = (int)(r & 3);
  const float2 n = comp < 2 ? _curand_box_muller(x.x, x.y) : _curand_box_muller(x.z, x.w);
  return (comp & 1) ? n.y : n.x;
}
__global__ void fill_normal_aten_kernel(float* out, size_t numel, unsigned long long seed, unsigned long long offset,
                                        unsigned int threads) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += (size_t)gridDim.x * blockDim.x)
    out[i] = aten_normal(seed, offset, threads, i);
}
__global__ void set_rng_kernel(RngState* dst, const RngState value) { *dst = value; }

__global__ void fill_normal_ref_kernel(float* out, int B, size_t per_sample, unsigned long long seed,
                                       unsigned long long stream_id, unsigned long long sample_offset) {
  const size_t quads = (per_sample + 3) / 4;
  const size_t total = (size_t)B * quads;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t b = i / quads, q = i - b * quads;
    float v[4];
    philox_normal4(seed, stream_id, sample_offset + b, q, v);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (q * 4 + j < per_sample) out[b * per_sample + q * 4 + j] = v[j];
  }
}

// ---------------------------------------------------------------------------------------------
// diffusion step. grid: (ceil(L/32), ceil(D_pad/32), B); block 32x8. Each block owns a 32(l) x 32(c)
// tile: frame-major operands are read/written with c fastest, the reference-layout noise tape with
// l fastest, through a padded smem tile.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) diffusion_step_kernel(const StepParams p) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ float s_noise[32][33];
  const int b = blockIdx.z;
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int t = *p.step_ptr;
  // first step index of the running call: a kernel argument, or (step graphs shared by every skip_timesteps) device memory
  const int tape_t0 = p.tape_t0 >= 0 ? p.tape_t0 : p.step_ptr[2];

  // ---- noise tile (reference layout [b][c][l], l contiguous) ----
  const bool want_noise = p.sampler != 2;  // the reference draws noise at every step, including t == 0
  if (want_noise) {
    RngState rng{};
    if (!p.noise_ref && p.rng) rng = *p.rng;
    if (!p.noise_ref && rng.mode == 1) {
      // torch.randn_like stream: draw number (tape_t0 - t) of this loop, element index in the (B, D, 1, L) layout
      const unsigned long long off = rng.aten_offset + (unsigned long long)(tape_t0 - t) * rng.aten_increment;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = c0 + ty + i * 8, l = l0 + tx;
        float nz = 0.f;
        if (c < p.D && l < p.L) nz = aten_normal(rng.seed, off, rng.aten_threads, ((size_t)b * p.D + c) * p.L + l);
        s_noise[ty + i * 8][tx] = nz;
      }
    } else if (!p.noise_ref && (p.L & 3) == 0) {
      // engine generator: one Philox call yields the 4 consecutive frames of a quad (l0 and L are multiples of 4)
      const int q = ty * 32 + tx;          // 256 quads = 32 features x 8 frame-quads
      const int cl = q >> 3, lq = (q & 7) * 4;
      const int c = c0 + cl, l = l0 + lq;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (c < p.D && l < p.L) philox_normal4(rng.seed, (unsigned long long)(t + 1), rng.sample_offset + b, ((size_t)c * p.L + l) >> 2, v);
#pragma unroll
      for (int j = 0; j < 4; ++j) s_noise[cl][lq + j] = v[j];
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = c0 + ty + i * 8, l = l0 + tx;
        float nz = 0.f;
        if (c < p.D && l < p.L) {
          const size_t e = (size_t)c * p.L + l;
          nz = p.noise_ref ? p.noise_ref[((size_t)(tape_t0 - t) * p.B + b) * p.D * p.L + e]
                           : philox_normal(rng.seed, (unsigned long long)(t + 1), rng.sample_offset + b, e);
        }
        s_noise[ty + i * 8][tx] = nz;
      }
    }
  }
  __syncthreads();

  // ---- per-step scalars (fp32, gathered exactly like _extract_into_tensor(...).float()) ----
  // (sampler 2 = plain denoiser evaluation: no schedule is needed, and none may be set)
  const float coef1 = p.sampler == 0 ? p.tab.post_coef1[t] : 0.f, coef2 = p.sampler == 0 ? p.tab.post_coef2[t] : 0.f;
  const float logvar = p.sampler == 0 ? p.tab.post_logvar[t] : 0.f;
  const float nonzero = (t != 0) ? 1.0f : 0.0f;
  const float text_scale = p.cfg ? p.text_scale[b] : 0.f;
  const bool do_impute = p.impute && (t >= p.stop_imputation_at);

  // one thread = 4 consecutive features of one frame (16-byte accesses; D_pad is a multiple of 8)
  {
    const int tid = ty * 32 + tx;
    const int ll = tid >> 3, cq = (tid & 7) * 4;
    const int l = l0 + ll, c = c0 + cq;
    if (l < p.L && c < p.D_pad) {
      const size_t idx = ((size_t)b * p.L + l) * p.D_pad + c;
      const size_t uoff = (size_t)p.B * p.L * p.D_pad;  // uncond half of the batch-doubled pass
      const float4 mo4 = *reinterpret_cast<const float4*>(p.model_out + idx);
      const float4 mu4 = p.cfg ? *reinterpret_cast<const float4*>(p.model_out + idx + uoff) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 xt4 = *reinterpret_cast<const float4*>(p.x_t + idx);
      const bool need_obs = p.guided || do_impute;
      const float4 ob4 = need_obs ? *reinterpret_cast<const float4*>(p.x_obs + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
      const uchar4 mk4 = need_obs ? *reinterpret_cast<const uchar4*>(p.obs_mask + idx) : make_uchar4(0, 0, 0, 0);
      float4 gg4 = make_float4(0.f, 0.f, 0.f, 0.f), gu4 = gg4;
      if (p.guided) {
        gg4 = *reinterpret_cast<const float4*>(p.guide_grad + idx);
        if (p.cfg) gu4 = *reinterpret_cast<const float4*>(p.guide_grad + idx + uoff);
      }
      const float mo[4] = {mo4.x, mo4.y, mo4.z, mo4.w}, mu[4] = {mu4.x, mu4.y, mu4.z, mu4.w};
      const float xtv[4] = {xt4.x, xt4.y, xt4.z, xt4.w}, ob[4] = {ob4.x, ob4.y, ob4.z, ob4.w};
      const unsigned char mk[4] = {mk4.x, mk4.y, mk4.z, mk4.w};
      const float gg[4] = {gg4.x, gg4.y, gg4.z, gg4.w}, gu[4] = {gu4.x, gu4.y, gu4.z, gu4.w};
      const float guide_c = p.guided ? p.guide_coef[t] : 0.f;
      float xn4[4], x04[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float xn = 0.f, x0 = 0.f;
        if (c + j < p.D) {
          // model output (+ classifier-free guidance: out_uncond + scale * (out - out_uncond), cfg_sampler.py:35)
          float out = mo[j];
          if (p.cfg) out = __fadd_rn(mu[j], __fmul_rn(text_scale, __fsub_rn(out, mu[j])));
          if (p.guided) {
            // reconstruction guidance (:416-425): cond_grad = grad * ~M ; tilde = hat - (w_r sqrt(abar) / 2) cond_grad ;
            // output = tilde * ~M + (imputing ? x_obs : hat) * M
            const float m = mk[j] ? 1.0f : 0.0f;
            float g = gg[j];
            if (p.cfg) g = __fadd_rn(g, gu[j]);
            g = __fmul_rn(g, 1.0f - m);
            const float tilde = __fsub_rn(out, __fmul_rn(guide_c, g));
            out = __fadd_rn(__fmul_rn(tilde, 1.0f - m), __fmul_rn(do_impute ? ob[j] : out, m));
          } else if (do_impute) {
            // imputation: (hat_x * ~M) + (x_obs * M)   (gaussian_diffusion.py:435)
            const float m = mk[j] ? 1.0f : 0.0f;
            out = __fadd_rn(__fmul_rn(out, 1.0f - m), __fmul_rn(ob[j], m));
          }
          x0 = out;  // START_X, no clipping (:513-515)
          const float xt = xtv[j];
          const float noise = s_noise[cq + j][ll];
          if (p.sampler == 2) {
            xn = 0.f;
          } else if (p.sampler == 0) {
            // mean = coef1*x0 + coef2*x_t (:338-342); sample = mean + nonzero*exp(0.5*logvar)*noise (:710-711)
            const float mean = __fadd_rn(__fmul_rn(coef1, x0), __fmul_rn(coef2, xt));
            const float sd = expf(__fmul_rn(0.5f, logvar));
            xn = __fadd_rn(mean, __fmul_rn(__fmul_rn(nonzero, sd), noise));
          } else {
            // ddim_sample_with_grad (:1397-1412)
            const float r1 = p.tab.sqrt_recip_acp[t], r2 = p.tab.sqrt_recipm1_acp[t];
            const float ab = p.tab.acp[t], abp = p.tab.acp_prev[t];
            const float eps = __fdiv_rn(__fsub_rn(__fmul_rn(r1, xt), x0), r2);
            const float sigma = __fmul_rn(__fmul_rn(p.eta, sqrtf(__fdiv_rn(1.0f - abp, 1.0f - ab))),
                                          sqrtf(__fsub_rn(1.0f, __fdiv_rn(ab, abp))));
            const float mean_pred = __fadd_rn(__fmul_rn(x0, sqrtf(abp)),
                                              __fmul_rn(sqrtf(__fsub_rn(__fsub_rn(1.0f, abp), __fmul_rn(sigma, sigma))), eps));
            xn = __fadd_rn(mean_pred, __fmul_rn(__fmul_rn(nonzero, sigma), noise));
          }
        }
        xn4[j] = xn;
        x04[j] = x0;
      }
      if (p.x_next) {
        *reinterpret_cast<float4*>(p.x_next + idx) = make_float4(xn4[0], xn4[1], xn4[2], xn4[3]);
        uint32_t h01, l01, h23, l23;
        split_bf16x2(xn4[0], xn4[1], h01, l01);
        split_bf16x2(xn4[2], xn4[3], h23, l23);
        *reinterpret_cast<uint2*>(p.x_next_hi + idx) = make_uint2(h01, h23);
        if (p.x_next_lo) *reinterpret_cast<uint2*>(p.x_next_lo + idx) = make_uint2(l01, l23);
      }
      if (p.pred_xstart) *reinterpret_cast<float4*>(p.pred_xstart + idx) = make_float4(x04[0], x04[1], x04[2], x04[3]);
    }
  }

  // ---- advance the device-side step counter once every block has read it ----
  if (p.advance) {
    __shared__ bool is_last;
    __threadfence();
    __syncthreads();
    if (tx == 0 && ty == 0) {
      const unsigned int total = gridDim.x * gridDim.y * gridDim.z;
      unsigned int* counter = reinterpret_cast<unsigned int*>(p.step_ptr + 1);
      const unsigned int prev = atomicAdd(counter, 1u);
      is_last = (prev == total - 1);
      if (is_last) {
        *counter = 0;
        *p.step_ptr = t - 1;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// layout converters (32x32 smem tile transposes)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ref_to_frames_kernel(const float* __restrict__ ref, int B, int D, int L, int D_pad,
                                                            float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_hi,
                                                            __nv_bfloat16* __restrict__ out_lo) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + i * 8, l = l0 + tx;
    tile[ty + i * 8][tx] = (c < D && l < L) ? ref[((size_t)b * D + c) * L + l] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int l = l0 + ty + i * 8, c = c0 + tx;
    if (l >= L || c >= D_pad) continue;
    const float v = tile[tx][ty + i * 8];
    const size_t idx = ((size_t)b * L + l) * D_pad + c;
    if (out_f32) out_f32[idx] = v;
    if (out_hi) {
      __nv_bfloat16 h, lo;
      split_bf16(v, h, lo);
      out_hi[idx] = h;
      if (out_lo) out_lo[idx] = lo;
    }
  }
}

__global__ void __launch_bounds__(256) frames_to_ref_kernel(const float* __restrict__ frames, int B, int D, int L, int D_pad,
                                                            float* __restrict__ ref) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int l = l0 + ty + i * 8, c = c0 + tx;
    tile[ty + i * 8][tx] = (l < L && c < D) ? frames[((size_t)b * L + l) * D_pad + c] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + i * 8, l = l0 + tx;
    if (c < D && l < L) ref[((size_t)b * D + c) * L + l] = tile[tx][ty + i * 8];
  }
}

__global__ void __launch_bounds__(256) mask_to_frames_kernel(const uint8_t* __restrict__ ref_mask,
                                                             const uint8_t* __restrict__ y_mask, int B, int D, int L,
                                                             int D_pad, uint8_t* __restrict__ out) {
  __shared__ uint8_t tile[32][33];
  const int b = blockIdx.z, l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + i * 8, l = l0 + tx;
    uint8_t m = 0;
    if (c < D && l < L) {
      // (inpainting_mask * y.mask.float()).bool()   (gaussian_diffusion.py:406-409, :432-433)
      m = ref_mask[((size_t)b * D + c) * L + l] != 0;
      if (y_mask) m = m && (y_mask[(size_t)b * L + l] != 0);
    }
    tile[ty + i * 8][tx] = m;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int l = l0 + ty + i * 8, c = c0 + tx;
    if (l < L && c < D_pad) out[((size_t)b * L + l) * D_pad + c] = tile[tx][ty + i * 8];
  }
}

__global__ void axpby_kernel(const float* __restrict__ x, const float* __restrict__ y, float a, float b, float* __restrict__ out,
                             size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = __fadd_rn(__fmul_rn(a, x[i]), __fmul_rn(b, y[i]));
}

__global__ void set_int_kernel(int* p, int v) {
  p[0] = v;
  p[1] = 0;  // block-arrival counter used by diffusion_step_kernel
}

// LayerNorm folded into the linear layer that consumes it: Wf[n,k] = W[n,k] * gamma[k] (fp32, split into planes by
// the caller), c[n] = sum_k Wf[n,k], d[n] = sum_k W[n,k] * beta[k] + bias[n].  One warp per output row, fp64 sums.
__global__ void __launch_bounds__(256) fold_ln_kernel(const float* __restrict__ W, int N, int K, const float* __restrict__ gamma,
                                                      const float* __restrict__ beta, const float* __restrict__ bias,
                                                      float* __restrict__ Wf, float* __restrict__ c, float* __restrict__ d) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  double cs = 0.0, ds = 0.0;
  for (int k = lane; k < K; k += 32) {
    const float w = W[(size_t)n * K + k];
    const float wf = w * gamma[k];
    Wf[(size_t)n * K + k] = wf;
    cs += (double)wf;
    ds += (double)w * (double)beta[k];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cs += __shfl_xor_sync(0xffffffffu, cs, o);
    ds += __shfl_xor_sync(0xffffffffu, ds, o);
  }
  if (lane == 0) {
    c[n] = (float)cs;
    d[n] = (float)(ds + (bias ? (double)bias[n] : 0.0));
  }
}

// out = a + b (fp32): LayerNorm beta + the bias of the layer whose epilogue re-derives that LayerNorm as its residual
__global__ void add_vectors_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + b[i];
}

__global__ void split_planes_kernel(const float* __restrict__ in, int rows, int cols, int ld_in, __nv_bfloat16* __restrict__ hi,
                                    __nv_bfloat16* __restrict__ lo, int ld_out) {
  const size_t total = (size_t)rows * ld_out;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / ld_out;
    const int c = (int)(i - r * ld_out);
    const float v = (c < cols) ? in[r * ld_in + c] : 0.f;
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    hi[i] = h;
    if (lo) lo[i] = l;
  }
}


// ---------------------------------------------------------------------------------------------
// HumanML3D vector -> joint positions (data_loaders/humanml/scripts/motion_process.py:402-441 recover_root_rot_pos,
// :474-489 recover_from_ric), optionally fused with the dataset de-normalisation x * std + mean
// (data_loaders/humanml/data/dataset.py:378-382) and the layout permutes sample/synthesize.py:153-157 does on the
// CPU.  One block per sequence; the two prefix sums over frames run sequentially on one thread, in the order
// torch.cumsum uses on the CPU, everything else is per (frame, joint).
// ---------------------------------------------------------------------------------------------
struct RicParams {
  const float* data;
  long long sb, sf, sc;      // input strides (elements): sequence, frame, feature
  const float* mean;         // [nfeats] or null
  const float* stdv;
  int B, L, joints, abs_3d;
  float* out;
  long long ob, of, oj, oc;  // output strides: sequence, frame, joint, coordinate
};
__global__ void __launch_bounds__(256) recover_from_ric_kernel(const RicParams p) {
  extern __shared__ float ric_smem[];
  float* ang = ric_smem;            // root heading per frame
  float* px = ang + p.L;            // root x, y, z per frame
  float* py = px + p.L;
  float* pz = py + p.L;
  float* vx = pz + p.L;             // (abs_3d == 0) de-normalised planar velocity
  float* vz = vx + p.L;
  const float* d = p.data + (long long)blockIdx.x * p.sb;
  auto feat = [&](int f, int c) -> float {
    const float v = d[f * p.sf + c * p.sc];
    return p.mean ? __fadd_rn(__fmul_rn(v, p.stdv[c]), p.mean[c]) : v;
  };
  for (int f = threadIdx.x; f < p.L; f += blockDim.x) {
    ang[f] = feat(f, 0);
    vx[f] = feat(f, 1);
    vz[f] = feat(f, 2);
    py[f] = feat(f, 3);
  }
  __syncthreads();
  if (!p.abs_3d) {
    if (threadIdx.x == 0) {  // r_rot_ang = cumsum([0, w_0, ..., w_{L-2}])
      float acc = 0.f, prev = ang[0];
      ang[0] = 0.f;
      for (int f = 1; f < p.L; ++f) {
        acc = __fadd_rn(acc, prev);
        prev = ang[f];
        ang[f] = acc;
      }
    }
    __syncthreads();
    // r_pos[f] = qrot(qinv(q_f), (vx[f-1], 0, vz[f-1])), q_f = (cos a, 0, sin a, 0); r_pos[0] = 0
    for (int f = threadIdx.x; f < p.L; f += blockDim.x) {
      float rx = 0.f, rz = 0.f;
      if (f > 0) {
        const float c = cosf(ang[f]), qy = -sinf(ang[f]);
        const float x = vx[f - 1], z = vz[f - 1];
        const float uv0 = __fmul_rn(qy, z), uv2 = -__fmul_rn(qy, x);
        const float uuv0 = __fmul_rn(qy, uv2), uuv2 = -__fmul_rn(qy, uv0);
        rx = __fadd_rn(x, __fmul_rn(2.f, __fadd_rn(__fmul_rn(c, uv0), uuv0)));
        rz = __fadd_rn(z, __fmul_rn(2.f, __fadd_rn(__fmul_rn(c, uv2), uuv2)));
      }
      px[f] = rx;
      pz[f] = rz;
    }
    __syncthreads();
    if (threadIdx.x < 2) {  // cumsum over frames, x on thread 0 and z on thread 1
      float* a = threadIdx.x == 0 ? px : pz;
      float acc = a[0];
      for (int f = 1; f < p.L; ++f) {
        acc = __fadd_rn(acc, a[f]);
        a[f] = acc;
      }
    }
    __syncthreads();
  } else {
    for (int f = threadIdx.x; f < p.L; f += blockDim.x) {
      px[f] = vx[f];
      pz[f] = vz[f];
    }
    __syncthreads();
  }
  float* o = p.out + (long long)blockIdx.x * p.ob;
  const int per_frame = p.joints;  // joint 0 = root, joints 1.. = rotation-invariant coordinates 4 + 3(j-1)
  for (int i = threadIdx.x; i < p.L * per_frame; i += blockDim.x) {
    const int f = i / per_frame, j = i - f * per_frame;
    float x, y, z;
    if (j == 0) {
      x = px[f]; y = py[f]; z = pz[f];
    } else {
      const float c = cosf(ang[f]), qy = -sinf(ang[f]);
      const float lx = feat(f, 4 + 3 * (j - 1)), ly = feat(f, 5 + 3 * (j - 1)), lz = feat(f, 6 + 3 * (j - 1));
      const float uv0 = __fmul_rn(qy, lz), uv2 = -__fmul_rn(qy, lx);
      const float uuv0 = __fmul_rn(qy, uv2), uuv2 = -__fmul_rn(qy, uv0);
      x = __fadd_rn(__fadd_rn(lx, __fmul_rn(2.f, __fadd_rn(__fmul_rn(c, uv0), uuv0))), px[f]);
      y = ly;
      z = __fadd_rn(__fadd_rn(lz, __fmul_rn(2.f, __fadd_rn(__fmul_rn(c, uv2), uuv2))), pz[f]);
    }
    float* dst = o + f * p.of + j * p.oj;
    dst[0] = x;
    dst[p.oc] = y;
    dst[2 * p.oc] = z;
  }
}

inline int grid_for(size_t n, int block) {
  size_t g = (n + block - 1) / block;
  if (g > 132 * 16) g = 132 * 16;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace

cudaError_t launch_layernorm512(const float* v, const float* gamma, const float* beta, float eps, int rows, float* out_f32,
                                __nv_bfloat16* out_hi, __nv_bfloat16* out_lo, cudaStream_t stream, float2* stats_out) {
  return launch_kernel(layernorm512_kernel, dim3((rows + 7) / 8), dim3(256), 0, stream, v, gamma, beta, eps,
                          rows, out_f32, out_hi, out_lo, stats_out);
}

cudaError_t launch_small_linear(const float* in, const float* W, const float* bias, float* out, int rows, int N, int K,
                                int act, cudaStream_t stream) {
  const long long warps = (long long)rows * N;
  small_linear_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(in, W, bias, out, rows, N, K, act);
  return cudaGetLastError();
}

cudaError_t launch_token_rows(const TokenParams& p, cudaStream_t stream) {
  return launch_kernel(token_rows_kernel, dim3(p.num_seqs), dim3(128), 0, stream, p);
}

cudaError_t launch_diffusion_step(const StepParams& p, cudaStream_t stream) {
  dim3 grid((p.L + 31) / 32, (p.D_pad + 31) / 32, p.B), block(32, 8);
  return launch_kernel(diffusion_step_kernel, grid, block, 0, stream, p);
}

cudaError_t launch_ref_to_frames(const float* ref, int B, int D, int L, int D_pad, float* out_f32, __nv_bfloat16* out_hi,
                                 __nv_bfloat16* out_lo, cudaStream_t stream) {
  dim3 grid((L + 31) / 32, (D_pad + 31) / 32, B), block(32, 8);
  ref_to_frames_kernel<<<grid, block, 0, stream>>>(ref, B, D, L, D_pad, out_f32, out_hi, out_lo);
  return cudaGetLastError();
}

cudaError_t launch_frames_to_ref(const float* frames, int B, int D, int L, int D_pad, float* ref, cudaStream_t stream) {
  dim3 grid((L + 31) / 32, (D + 31) / 32, B), block(32, 8);
  frames_to_ref_kernel<<<grid, block, 0, stream>>>(frames, B, D, L, D_pad, ref);
  return cudaGetLastError();
}

cudaError_t launch_mask_to_frames(const uint8_t* ref_mask, const uint8_t* y_mask, int B, int D, int L, int D_pad, uint8_t* out,
                                  cudaStream_t stream) {
  dim3 grid((L + 31) / 32, (D_pad + 31) / 32, B), block(32, 8);
  mask_to_frames_kernel<<<grid, block, 0, stream>>>(ref_mask, y_mask, B, D, L, D_pad, out);
  return cudaGetLastError();
}

cudaError_t launch_axpby(const float* x, const float* y, float a, float b, float* out, size_t n, cudaStream_t stream) {
  axpby_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, y, a, b, out, n);
  return cudaGetLastError();
}

cudaError_t launch_set_rng(RngState* dst, const RngState& value, cudaStream_t stream) {
  set_rng_kernel<<<1, 1, 0, stream>>>(dst, value);
  return cudaGetLastError();
}
cudaError_t launch_fill_normal_aten(float* out, size_t numel, unsigned long long seed, unsigned long long offset,
                                    unsigned int threads, cudaStream_t stream) {
  if (threads == 0 || (offset & 3)) return cudaErrorInvalidValue;
  fill_normal_aten_kernel<<<grid_for(numel, 256), 256, 0, stream>>>(out, numel, seed, offset, threads);
  return cudaGetLastError();
}
cudaError_t launch_fill_normal_ref(float* out, int B, size_t per_sample, unsigned long long seed, unsigned long long stream_id,
                                   unsigned long long sample_offset, cudaStream_t stream) {
  fill_normal_ref_kernel<<<grid_for((size_t)B * per_sample, 256), 256, 0, stream>>>(out, B, per_sample, seed, stream_id,
                                                                                  sample_offset);
  return cudaGetLastError();
}

cudaError_t launch_recover_from_ric(const float* data, long long sb, long long sf, long long sc, const float* mean,
                                    const float* stdv, int B, int L, int joints, int abs_3d, float* out, long long ob,
                                    long long of, long long oj, long long oc, cudaStream_t stream) {
  RicParams p{data, sb, sf, sc, mean, stdv, B, L, joints, abs_3d, out, ob, of, oj, oc};
  const size_t smem = (size_t)6 * L * sizeof(float);
  if (B <= 0) return cudaSuccess;
  if (smem > 48 * 1024) return cudaErrorInvalidValue;
  recover_from_ric_kernel<<<B, 256, smem, stream>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_set_int(int* p, int v, cudaStream_t stream) {
  set_int_kernel<<<1, 1, 0, stream>>>(p, v);
  return cudaGetLastError();
}

cudaError_t launch_fold_ln(const float* W, int N, int K, const float* gamma, const float* beta, const float* bias, float* Wf,
                           float* c, float* d, cudaStream_t stream) {
  fold_ln_kernel<<<(N + 7) / 8, 256, 0, stream>>>(W, N, K, gamma, beta, bias, Wf, c, d);
  return cudaGetLastError();
}

cudaError_t launch_add_vectors(const float* a, const float* b, float* out, int n, cudaStream_t stream) {
  add_vectors_kernel<<<(n + 255) / 256, 256, 0, stream>>>(a, b, out, n);
  return cudaGetLastError();
}

cudaError_t launch_split_planes(const float* in, int rows, int cols, int ld_in, __nv_bfloat16* hi, __nv_bfloat16* lo,
                                int ld_out, cudaStream_t stream) {
  split_planes_kernel<<<grid_for((size_t)rows * ld_out, 256), 256, 0, stream>>>(in, rows, cols, ld_in, hi, lo, ld_out);
  return cudaGetLastError();
}

}  // namespace cmdi
