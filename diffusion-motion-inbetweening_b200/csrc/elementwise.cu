// Row-wise and elementwise kernels of the sampling path (HBM/L2-bound; coalesced, vectorised).
//
//   layernorm512           nn.TransformerEncoderLayer norm1/norm2 (post-norm)      mdm.py:107-114
//   token_rows             timestep(+text) token + PE[0]                           mdm.py:245-251,279-280
//   small_linear           TimestepEmbedder MLP / embed_text, once per loop        mdm.py:345-353,248-251
//   diffusion_step         p_mean_variance tail + p_sample / ddim_sample           gaussian_diffusion.py:352-534,656-713,1358-1416
//                          + ClassifierFreeSampleModel combine                     cfg_sampler.py:25-35
//                          + keyframe imputation blend                             gaussian_diffusion.py:427-435
//   plms_step              plms_sample (pseudo linear multistep), same combine      gaussian_diffusion.py:1589-1687
//   ddim_reverse_step      ddim_reverse_sample (DDIM inversion, eta = 0), same combine  gaussian_diffusion.py:1418-1452
//   dpm_solver_step        DPM-Solver++ multistep (Lu et al. 2022), orders 1-3, same combine
//   unipc_step             UniPC predictor-corrector (Zhao et al. 2023), orders 1-3, same combine
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
// pred_xstart of one element (START_X, no clipping, :513-515): the model output (+ classifier-free guidance:
// out_uncond + scale * (out - out_uncond), cfg_sampler.py:35), then reconstruction guidance or the imputation blend
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float step_x0(float mo, float mu, float ob, unsigned char mk, float gg, float gu, int cfg, int guided,
                                         bool do_impute, float text_scale, float guide_c) {
  float out = mo;
  if (cfg) out = __fadd_rn(mu, __fmul_rn(text_scale, __fsub_rn(out, mu)));
  if (guided) {
    // reconstruction guidance (:416-425): cond_grad = grad * ~M ; tilde = hat - (w_r sqrt(abar) / 2) cond_grad ;
    // output = tilde * ~M + (imputing ? x_obs : hat) * M
    const float m = mk ? 1.0f : 0.0f;
    float g = gg;
    if (cfg) g = __fadd_rn(g, gu);
    g = __fmul_rn(g, 1.0f - m);
    const float tilde = __fsub_rn(out, __fmul_rn(guide_c, g));
    out = __fadd_rn(__fmul_rn(tilde, 1.0f - m), __fmul_rn(do_impute ? ob : out, m));
  } else if (do_impute) {
    // imputation: (hat_x * ~M) + (x_obs * M)   (gaussian_diffusion.py:435)
    const float m = mk ? 1.0f : 0.0f;
    out = __fadd_rn(__fmul_rn(out, 1.0f - m), __fmul_rn(ob, m));
  }
  return out;
}

// x0 (step_x0) of the 4 consecutive features at idx, the frame-major offset of feature c of a frame of row b, and
// x_t there when xt is given.  Operands are read with 16-byte loads, each under the predicate that makes it meaningful:
// an unguided, un-imputed step never touches x_obs / obs_mask / guide_grad, and only a CFG step reads the uncond half.
// Padding features (c + j >= D) get x0 = 0.
__device__ __forceinline__ void step_x0_at(const StepParams& p, size_t idx, int b, int c, bool do_impute, float guide_c,
                                           float x0[4], float* xt = nullptr) {
  const size_t uoff = (size_t)p.B * p.L * p.D_pad;  // uncond half of the batch-doubled pass
  const float text_scale = p.cfg ? p.text_scale[b] : 0.f;
  const bool need_obs = p.guided || do_impute;
  const float4 mo4 = *reinterpret_cast<const float4*>(p.model_out + idx);
  const float4 mu4 = p.cfg ? *reinterpret_cast<const float4*>(p.model_out + idx + uoff) : make_float4(0.f, 0.f, 0.f, 0.f);
  if (xt) {
    const float4 xt4 = *reinterpret_cast<const float4*>(p.x_t + idx);
    xt[0] = xt4.x; xt[1] = xt4.y; xt[2] = xt4.z; xt[3] = xt4.w;
  }
  const float4 ob4 = need_obs ? *reinterpret_cast<const float4*>(p.x_obs + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
  const uchar4 mk4 = need_obs ? *reinterpret_cast<const uchar4*>(p.obs_mask + idx) : make_uchar4(0, 0, 0, 0);
  float4 gg4 = make_float4(0.f, 0.f, 0.f, 0.f), gu4 = gg4;
  if (p.guided) {
    gg4 = *reinterpret_cast<const float4*>(p.guide_grad + idx);
    if (p.cfg) gu4 = *reinterpret_cast<const float4*>(p.guide_grad + idx + uoff);
  }
  const float mo[4] = {mo4.x, mo4.y, mo4.z, mo4.w}, mu[4] = {mu4.x, mu4.y, mu4.z, mu4.w};
  const float ob[4] = {ob4.x, ob4.y, ob4.z, ob4.w};
  const unsigned char mk[4] = {mk4.x, mk4.y, mk4.z, mk4.w};
  const float gg[4] = {gg4.x, gg4.y, gg4.z, gg4.w}, gu[4] = {gu4.x, gu4.y, gu4.z, gu4.w};
#pragma unroll
  for (int j = 0; j < 4; ++j)
    x0[j] = c + j < p.D ? step_x0(mo[j], mu[j], ob[j], mk[j], gg[j], gu[j], p.cfg, p.guided, do_impute, text_scale, guide_c) : 0.f;
}

// Overlapping windows: x0 of a global frame g that several windows cover becomes
//   (sum_k w_k(g) x0_k(g)) / sum_k w_k(g),   w_k(g) = 1 + min(g - f0(k), f0(k) + F - 1 - g),
// summed over the covering windows in ascending k with round-to-nearest fp32 products, sums and quotient.  Every
// covering window forms the same sum in the same order from the same inputs (each neighbour's x0 is recomputed from its
// own model output, guidance gradient and keyframes), so all of them store the same bits.  A frame covered by this
// window alone keeps its x0.  The weights are small integers, exact in fp32.
__device__ __forceinline__ void blend_window_x0(const StepParams& p, size_t idx, int b, int c, bool do_impute, float guide_c,
                                                float x0[4]) {
  const int K = p.win_K, F = p.L;
  const int k = b % K, row0 = b - k;
  const int g = p.win_f0[k] + (int)((idx / p.D_pad) % F);
  int lo = k, hi = k;
  while (lo > 0 && p.win_f0[lo - 1] + F > g) --lo;
  while (hi + 1 < K && p.win_f0[hi + 1] <= g) ++hi;
  if (lo == hi) return;
  float acc[4], wsum = 0.f;
  for (int kk = lo; kk <= hi; ++kk) {
    const int f0 = p.win_f0[kk];
    const float w = (float)(1 + min(g - f0, f0 + F - 1 - g));
    float v[4] = {x0[0], x0[1], x0[2], x0[3]};
    if (kk != k) step_x0_at(p, ((size_t)(row0 + kk) * F + (g - f0)) * p.D_pad + c, row0 + kk, c, do_impute, guide_c, v);
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = kk == lo ? __fmul_rn(w, v[j]) : __fadd_rn(acc[j], __fmul_rn(w, v[j]));
    wsum += w;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) x0[j] = __fdiv_rn(acc[j], wsum);
}

// x_t and x0 of the 4 consecutive features at idx (step_x0_at, then the window blend) for the evaluation at step index
// t_eval.  kWin: the step kernel instance for windowed calls (win_K > 1); the other instance has no blend code.
template <bool kWin = false>
__device__ __forceinline__ void load_step_x0(const StepParams& p, size_t idx, int b, int c, int t_eval, float xt[4], float x0[4]) {
  const bool do_impute = p.impute && (t_eval >= p.stop_imputation_at);
  const float guide_c = p.guided ? p.guide_coef[t_eval] : 0.f;
  step_x0_at(p, idx, b, c, do_impute, guide_c, x0, xt);
  if (kWin) blend_window_x0(p, idx, b, c, do_impute, guide_c, x0);
}

// Stores the state after a step for the 4 features at idx: x_next as fp32 and as bf16 planes (hi, and lo where the
// engine keeps split operands), and pred_xstart.  x_next is null for the pass-through evaluation (sampler 2).
__device__ __forceinline__ void store_step_state(const StepParams& p, size_t idx, const float xn[4], const float x0[4], bool write_pred) {
  if (p.x_next) {
    *reinterpret_cast<float4*>(p.x_next + idx) = make_float4(xn[0], xn[1], xn[2], xn[3]);
    uint32_t h01, l01, h23, l23;
    split_bf16x2(xn[0], xn[1], h01, l01);
    split_bf16x2(xn[2], xn[3], h23, l23);
    *reinterpret_cast<uint2*>(p.x_next_hi + idx) = make_uint2(h01, h23);
    if (p.x_next_lo) *reinterpret_cast<uint2*>(p.x_next_lo + idx) = make_uint2(l01, l23);
  }
  if (p.pred_xstart && write_pred) *reinterpret_cast<float4*>(p.pred_xstart + idx) = make_float4(x0[0], x0[1], x0[2], x0[3]);
}

// Bumps the block-arrival counter at step_ptr[1]; the last block to arrive stores `next` as the step index (every
// block has read the old one by then).
__device__ __forceinline__ void advance_step(int* step_ptr, int next) {
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0) {
    const unsigned int total = gridDim.x * gridDim.y * gridDim.z;
    unsigned int* counter = reinterpret_cast<unsigned int*>(step_ptr + 1);
    const unsigned int prev = atomicAdd(counter, 1u);
    is_last = (prev == total - 1);
    if (is_last) {
      *counter = 0;
      *step_ptr = next;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// PLMS step (plms_sample, gaussian_diffusion.py:1589-1687, cond_fn = None) on frame-major state [B*L, D_pad].  One
// thread = 4 consecutive features of one frame.  No noise is drawn.  The eps history lives in a ring of three
// [B*L, D_pad] buffers: eps of loop iteration k is at slot k % 3, with k = step_ptr[2] - t (step_ptr[2] holds the
// step index the history started at), so one kernel serves every Adams-Bashforth step.
//   phase 0  Adams-Bashforth step at t: one evaluation; advances t -> t - 1
//   phase 1  first step, after the evaluation at t: stores eps_0 and x_t, writes the second evaluation's input
//            m = x0 sqrt(abp) + sqrt(1 - abp) eps_0 (or, at t = 0, the sample x0); advances t -> t - 1
//   phase 2  first step, after the evaluation at t - 1 (= step_ptr[0]): the improved Euler sample from the kept x_t;
//            leaves the step index at t - 1
// ---------------------------------------------------------------------------------------------
template <bool kWin>
__global__ void __launch_bounds__(256) plms_step_kernel(const StepParams p, const PlmsParams q) {
  const int t_eval = *p.step_ptr;                    // step index of the evaluation in model_out
  const int t = q.phase == 2 ? t_eval + 1 : t_eval;  // step index of the PLMS step
  const int k = p.step_ptr[2] - t;                   // loop iteration since the history started
  const int cur_order = min(q.order, k + 1);
  const float r1e = p.tab.sqrt_recip_acp[t_eval], r2e = p.tab.sqrt_recipm1_acp[t_eval];
  const float r1 = p.tab.sqrt_recip_acp[t], r2 = p.tab.sqrt_recipm1_acp[t];
  const float abp = p.tab.acp_prev[t];
  const float sq_abp = sqrtf(abp), sq_1m_abp = sqrtf(__fsub_rn(1.0f, abp));
  const size_t n4 = (size_t)p.B * p.L * p.D_pad / 4;
  const size_t i4 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 < n4) {
    const size_t idx = i4 * 4;
    const int c = (int)(idx % p.D_pad);
    const int b = (int)(idx / ((size_t)p.L * p.D_pad));
    float* slot0 = q.eps_hist;
    float* cur = q.eps_hist + (size_t)(k % 3) * q.hist_stride;
    const float* h2 = q.eps_hist + (size_t)((k + 2) % 3) * q.hist_stride;  // iteration k - 1
    const float* h3 = q.eps_hist + (size_t)((k + 1) % 3) * q.hist_stride;  // k - 2
    const float* h4 = cur;                                                 // k - 3 (read before it is overwritten)
    float4 e2v = make_float4(0.f, 0.f, 0.f, 0.f), e3v = e2v, e4v = e2v, xkv = e2v;
    if (q.phase == 0) {
      if (cur_order >= 2) e2v = *reinterpret_cast<const float4*>(h2 + idx);
      if (cur_order >= 3) e3v = *reinterpret_cast<const float4*>(h3 + idx);
      if (cur_order >= 4) e4v = *reinterpret_cast<const float4*>(h4 + idx);
    } else if (q.phase == 2) {
      e2v = *reinterpret_cast<const float4*>(slot0 + idx);  // eps_0
      xkv = *reinterpret_cast<const float4*>(q.x_keep + idx);
    }
    const float e2[4] = {e2v.x, e2v.y, e2v.z, e2v.w}, e3[4] = {e3v.x, e3v.y, e3v.z, e3v.w}, e4[4] = {e4v.x, e4v.y, e4v.z, e4v.w};
    const float xk[4] = {xkv.x, xkv.y, xkv.z, xkv.w};
    float xtv[4], x04[4], xn4[4], ep4[4];
    load_step_x0<kWin>(p, idx, b, c, t_eval, xtv, x04);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float x0 = x04[j];
      float xn = 0.f, eps = 0.f;
      if (c + j < p.D) {
        // _predict_eps_from_xstart at the evaluation's (x, t) (:551-555)
        eps = __fdiv_rn(__fsub_rn(__fmul_rn(r1e, xtv[j]), x0), r2e);
        float ep, x;
        if (q.phase == 1) {
          // pseudo improved Euler, first half (:1647-1654): the input of the evaluation at t - 1
          xn = t != 0 ? __fadd_rn(__fmul_rn(x0, sq_abp), __fmul_rn(sq_1m_abp, eps)) : x0;
        } else {
          if (q.phase == 2) {
            ep = __fdiv_rn(__fadd_rn(e2[j], eps), 2.0f);  // (eps_0 + eps_2) / 2 (:1655)
            x = xk[j];
          } else {
            // Adams-Bashforth (:1660-1673), e_1 = eps the newest
            if (cur_order == 2) {
              ep = __fdiv_rn(__fsub_rn(__fmul_rn(3.0f, eps), e2[j]), 2.0f);
            } else if (cur_order == 3) {
              ep = __fdiv_rn(__fadd_rn(__fsub_rn(__fmul_rn(23.0f, eps), __fmul_rn(16.0f, e2[j])), __fmul_rn(5.0f, e3[j])), 12.0f);
            } else if (cur_order == 4) {
              ep = __fdiv_rn(__fsub_rn(__fadd_rn(__fsub_rn(__fmul_rn(55.0f, eps), __fmul_rn(59.0f, e2[j])), __fmul_rn(37.0f, e3[j])),
                                       __fmul_rn(9.0f, e4[j])), 24.0f);
            } else {
              ep = eps;
            }
            x = xtv[j];
          }
          // pred' = _predict_xstart_from_eps(x, t, eps') (:536-541); mean = pred' sqrt(abp) + sqrt(1 - abp) eps'
          const float pp = __fsub_rn(__fmul_rn(r1, x), __fmul_rn(r2, ep));
          const float mean = __fadd_rn(__fmul_rn(pp, sq_abp), __fmul_rn(sq_1m_abp, ep));
          xn = t != 0 ? mean : x0;  // :1679-1681
        }
      }
      xn4[j] = xn;
      ep4[j] = eps;
    }
    if (q.phase == 0) *reinterpret_cast<float4*>(cur + idx) = make_float4(ep4[0], ep4[1], ep4[2], ep4[3]);
    if (q.phase == 1) {
      *reinterpret_cast<float4*>(slot0 + idx) = make_float4(ep4[0], ep4[1], ep4[2], ep4[3]);
      *reinterpret_cast<float4*>(q.x_keep + idx) = make_float4(xtv[0], xtv[1], xtv[2], xtv[3]);
    }
    store_step_state(p, idx, xn4, x04, q.phase != 2);  // pred_xstart is the FIRST evaluation's x0 (:1685)
  }
  if (q.phase != 2) advance_step(p.step_ptr, t - 1);
}

// ---------------------------------------------------------------------------------------------
// DDIM reverse step (ddim_reverse_sample, gaussian_diffusion.py:1418-1452, eta = 0) on frame-major state [B*L, D_pad]:
// the deterministic encoder x_t -> x_{t+1}.  One thread = 4 consecutive features of one frame.  pred_xstart is the
// shared combine (p_mean_variance); no noise is drawn.  Advances t -> t + 1.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) ddim_reverse_step_kernel(const StepParams p) {
  const int t = *p.step_ptr;
  const float r1 = p.tab.sqrt_recip_acp[t], r2 = p.tab.sqrt_recipm1_acp[t];
  const float abn = p.tab.acp_next[t];  // _extract_into_tensor(alphas_cumprod_next, t).float() (:1445-1446)
  const float sq_abn = sqrtf(abn), sq_1m_abn = sqrtf(__fsub_rn(1.0f, abn));
  const size_t n4 = (size_t)p.B * p.L * p.D_pad / 4;
  const size_t i4 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 < n4) {
    const size_t idx = i4 * 4;
    const int c = (int)(idx % p.D_pad);
    const int b = (int)(idx / ((size_t)p.L * p.D_pad));
    float xtv[4], x04[4], xn4[4];
    load_step_x0(p, idx, b, c, t, xtv, x04);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float x0 = x04[j];
      float xn = 0.f;
      if (c + j < p.D) {
        // eps = (sqrt_recip_acp[t] x - x0) / sqrt_recipm1_acp[t] (:1442-1444);
        // mean_pred = x0 sqrt(ab_next) + sqrt(1 - ab_next) eps (:1449-1450)
        const float eps = __fdiv_rn(__fsub_rn(__fmul_rn(r1, xtv[j]), x0), r2);
        xn = __fadd_rn(__fmul_rn(x0, sq_abn), __fmul_rn(sq_1m_abn, eps));
      }
      xn4[j] = xn;
    }
    store_step_state(p, idx, xn4, x04, true);
  }
  advance_step(p.step_ptr, t + 1);
}

// ---------------------------------------------------------------------------------------------
// DPM-Solver++ multistep step (Lu et al. 2022, data prediction) on frame-major state [B*L, D_pad].  One thread = 4
// consecutive features of one frame.  m0 = x0 of the shared combine; the update is folded into four per-step
// coefficients (host-computed in float64 for the running history), x_{s-1} = A x_s + B0 m0 + B1 m1 + B2 m2, where m1 /
// m2 are the x0 of the previous two loop iterations.  The x0 history is a ring of three [B*L, D_pad] buffers: iteration
// k = step_ptr[2] - s at slot k % 3, so one kernel serves every step.  No noise is drawn.  Advances s -> s - 1.
// ---------------------------------------------------------------------------------------------
template <bool kWin>
__global__ void __launch_bounds__(256) dpm_solver_step_kernel(const StepParams p, const DpmParams q) {
  const int s = *p.step_ptr;
  const int k = p.step_ptr[2] - s;                      // loop iteration since the history started
  const int eff = min(min(q.order, k + 1), s + 1);      // effective order: lower while the history fills and at the end
  const float4 cf = *reinterpret_cast<const float4*>(q.coef + (size_t)s * 4);  // (A, B0, B1, B2)
  const size_t n4 = (size_t)p.B * p.L * p.D_pad / 4;
  const size_t i4 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 < n4) {
    const size_t idx = i4 * 4;
    const int c = (int)(idx % p.D_pad);
    const int b = (int)(idx / ((size_t)p.L * p.D_pad));
    float* cur = q.x0_hist + (size_t)(k % 3) * q.hist_stride;
    float4 m1v = make_float4(0.f, 0.f, 0.f, 0.f), m2v = m1v;
    if (eff >= 2) m1v = *reinterpret_cast<const float4*>(q.x0_hist + (size_t)((k + 2) % 3) * q.hist_stride + idx);  // k - 1
    if (eff >= 3) m2v = *reinterpret_cast<const float4*>(q.x0_hist + (size_t)((k + 1) % 3) * q.hist_stride + idx);  // k - 2
    const float m1[4] = {m1v.x, m1v.y, m1v.z, m1v.w}, m2[4] = {m2v.x, m2v.y, m2v.z, m2v.w};
    float xtv[4], x04[4], xn4[4];
    load_step_x0<kWin>(p, idx, b, c, s, xtv, x04);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float x0 = x04[j];
      float xn = 0.f;
      if (c + j < p.D) {
        xn = __fadd_rn(__fmul_rn(cf.x, xtv[j]), __fmul_rn(cf.y, x0));
        if (eff >= 2) xn = __fadd_rn(xn, __fmul_rn(cf.z, m1[j]));
        if (eff >= 3) xn = __fadd_rn(xn, __fmul_rn(cf.w, m2[j]));
        if (s == 0) xn = x0;  // the last step lands on abar = 1: the sample is x0 (A = 0, B0 = 1)
      }
      xn4[j] = xn;
    }
    *reinterpret_cast<float4*>(cur + idx) = make_float4(x04[0], x04[1], x04[2], x04[3]);
    store_step_state(p, idx, xn4, x04, true);
  }
  advance_step(p.step_ptr, s - 1);
}

// ---------------------------------------------------------------------------------------------
// UniPC step (Zhao et al. 2023, multistep, data prediction) on frame-major state [B*L, D_pad].  One thread = 4
// consecutive features of one frame.  The pass evaluated the uncorrected state x_s; m0 = its x0 (shared combine).  The
// kernel corrects (UniC) x_s^c = Ac x_{s+1}^c + C0 m0 + C1 m1 + C2 m2 + C3 m3 when a predictor step led into s, then
// predicts (UniP) x_{s-1} = A x_s^c + B0 m0 + B1 m1 + B2 m2; m_j is the x0 of iteration k - j.  The coefficients are
// host-computed in float64 for the running history, 12 per step index.  The x0 history is the ring of three buffers
// DPM-Solver++ uses: iteration k at slot k % 3, so m3 (iteration k - 3) sits in this step's own slot and is read before
// m0 overwrites it.  x_s^c replaces x_{s+1}^c in q.xc.  No noise is drawn.  Advances s -> s - 1.
// ---------------------------------------------------------------------------------------------
template <bool kWin>
__global__ void __launch_bounds__(256) unipc_step_kernel(const StepParams p, const UnipcParams q) {
  const int s = *p.step_ptr;
  const int k = p.step_ptr[2] - s;                                  // loop iteration since the history started
  const int pe = min(min(q.order, k + 1), s + 1);                   // predictor order of s -> s - 1
  const int ce = (q.corrector && k > 0 && s > 0) ? min(min(q.order, k), s + 2) : 0;  // order of the predictor into s
  const int nh = max(pe - 1, ce);                                   // history planes the two updates read
  const float4* row = reinterpret_cast<const float4*>(q.coef + (size_t)s * 12);
  const float4 cp = row[0];                                         // (A, B0, B1, B2)
  const float4 cc = ce ? row[1] : make_float4(0.f, 0.f, 0.f, 0.f);  // (Ac, C0, C1, C2)
  const float c3 = ce >= 3 ? row[2].x : 0.f;                        // C3
  const size_t n4 = (size_t)p.B * p.L * p.D_pad / 4;
  const size_t i4 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 < n4) {
    const size_t idx = i4 * 4;
    const int c = (int)(idx % p.D_pad);
    const int b = (int)(idx / ((size_t)p.L * p.D_pad));
    float* cur = q.x0_hist + (size_t)(k % 3) * q.hist_stride;
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 m1v = nh >= 1 ? *reinterpret_cast<const float4*>(q.x0_hist + (size_t)((k + 2) % 3) * q.hist_stride + idx) : z4;
    const float4 m2v = nh >= 2 ? *reinterpret_cast<const float4*>(q.x0_hist + (size_t)((k + 1) % 3) * q.hist_stride + idx) : z4;
    const float4 m3v = nh >= 3 ? *reinterpret_cast<const float4*>(cur + idx) : z4;  // k - 3, before m0 overwrites it
    const float4 xcv = ce ? *reinterpret_cast<const float4*>(q.xc + idx) : z4;
    const float m1[4] = {m1v.x, m1v.y, m1v.z, m1v.w}, m2[4] = {m2v.x, m2v.y, m2v.z, m2v.w};
    const float m3[4] = {m3v.x, m3v.y, m3v.z, m3v.w}, xcp[4] = {xcv.x, xcv.y, xcv.z, xcv.w};
    float xtv[4], x04[4], xn4[4], xc4[4];
    load_step_x0<kWin>(p, idx, b, c, s, xtv, x04);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float x0 = x04[j];
      float xn = 0.f, xc = 0.f;
      if (c + j < p.D) {
        xc = xtv[j];  // nothing to correct: x_s^c = x_s
        if (ce) {
          xc = __fadd_rn(__fadd_rn(__fmul_rn(cc.x, xcp[j]), __fmul_rn(cc.y, x0)), __fmul_rn(cc.z, m1[j]));
          if (ce >= 2) xc = __fadd_rn(xc, __fmul_rn(cc.w, m2[j]));
          if (ce >= 3) xc = __fadd_rn(xc, __fmul_rn(c3, m3[j]));
        }
        xn =__fadd_rn(__fmul_rn(cp.x, xc), __fmul_rn(cp.y, x0));
        if (pe >= 2) xn = __fadd_rn(xn, __fmul_rn(cp.z, m1[j]));
        if (pe >= 3) xn = __fadd_rn(xn, __fmul_rn(cp.w, m2[j]));
        if (s == 0) xn = x0;  // the last step lands on abar = 1: the sample is x0 (A = 0, B0 = 1)
      }
      xn4[j] = xn;
      xc4[j] = xc;
    }
    *reinterpret_cast<float4*>(cur + idx) = make_float4(x04[0], x04[1], x04[2], x04[3]);
    if (q.xc) *reinterpret_cast<float4*>(q.xc + idx) = make_float4(xc4[0], xc4[1], xc4[2], xc4[3]);
    store_step_state(p, idx, xn4, x04, true);
  }
  advance_step(p.step_ptr, s - 1);
}

// ---------------------------------------------------------------------------------------------
// The per-step noise of sample b at step index t for the 32(c) x 32(l) tile at (c0, l0), in the reference layout
// [b][c][l] (l contiguous), into s_noise[c - c0][l - l0]; block 32x8.  tape_t0 is the call's first step index, so
// (tape_t0 - t) numbers this step's draw within the call.  Three sources: the noise tape, the torch.randn_like stream
// (draw number (tape_t0 - t) after aten_offset) and the engine generator (stream t + 1, keyed by the global sample
// index).  With overlapping windows (win_K > 1) row b is window k of global sample s, and its frame l draws the noise
// of global frame f0(k) + l of sample s in the (B / win_K, D, 1, win_N) layout, from each of the three sources.  The
// caller synchronises the block before reading the tile.
// ---------------------------------------------------------------------------------------------
template <bool kWin = false>
__device__ __forceinline__ void fill_noise_tile(const StepParams& p, int t, int tape_t0, int b, int l0, int c0,
                                                float (&s_noise)[32][33]) {
  const int tx = threadIdx.x, ty = threadIdx.y;
  int gs = b, gf0 = 0, gL = p.L, gB = p.B;  // global sample, first global frame, global frames and samples
  if (kWin) {
    gs = b / p.win_K; gf0 = p.win_f0[b % p.win_K]; gL = p.win_N; gB = p.B / p.win_K;
  }
  RngState rng{};
  if (!p.noise_ref && p.rng) rng = *p.rng;
  if (!p.noise_ref && rng.mode == 1) {
    // torch.randn_like stream: draw number (tape_t0 - t) of this loop, element index in the (B, D, 1, L) layout
    const unsigned long long off = rng.aten_offset + (unsigned long long)(tape_t0 - t) * rng.aten_increment;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = c0 + ty + i * 8, l = l0 + tx;
      float nz = 0.f;
      if (c < p.D && l < p.L) nz = aten_normal(rng.seed, off, rng.aten_threads, ((size_t)gs * p.D + c) * gL + gf0 + l);
      s_noise[ty + i * 8][tx] = nz;
    }
  } else if (!p.noise_ref && (p.L & 3) == 0 && ((gf0 | gL) & 3) == 0) {
    // engine generator: one Philox call yields the 4 consecutive frames of a quad (l0, L and the global frame offset
    // and length are multiples of 4)
    const int q = ty * 32 + tx;          // 256 quads = 32 features x 8 frame-quads
    const int cl = q >> 3, lq = (q & 7) * 4;
    const int c = c0 + cl, l = l0 + lq;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (c < p.D && l < p.L)
      philox_normal4(rng.seed, (unsigned long long)(t + 1), rng.sample_offset + gs, ((size_t)c * gL + gf0 + l) >> 2, v);
#pragma unroll
    for (int j = 0; j < 4; ++j) s_noise[cl][lq + j] = v[j];
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = c0 + ty + i * 8, l = l0 + tx;
      float nz = 0.f;
      if (c < p.D && l < p.L) {
        const size_t e = (size_t)c * gL + gf0 + l;
        nz = p.noise_ref ? p.noise_ref[((size_t)(tape_t0 - t) * gB + gs) * p.D * gL + e]
                         : philox_normal(rng.seed, (unsigned long long)(t + 1), rng.sample_offset + gs, e);
      }
      s_noise[ty + i * 8][tx] = nz;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// SDE-DPM-Solver++ multistep step (Lu et al. 2022, "DPM-Solver++", the SDE solver in data prediction, midpoint form)
// on frame-major state [B*L, D_pad], with diffusion_step_kernel's grid, block and noise tile.  m0 = x0 of the shared
// combine; the update is folded into four per-step coefficients (host-computed in float64 for the running history),
// x_{s-1} = A x_s + B0 m0 + B1 m1 + Cn z, where m1 is the x0 of the previous loop iteration and z this step's draw.
// The x0 history is DPM-Solver++'s ring (iteration k = step_ptr[2] - s at slot k % 3).  The draw is numbered from the
// call's first step (step_ptr[3], or the tape_t0 argument), as p_sample_loop's draws are; the last step (s = 0)
// returns m0 and reads no noise.  Advances s -> s - 1.
// ---------------------------------------------------------------------------------------------
template <bool kWin>
__global__ void __launch_bounds__(256) dpm_solver_sde_step_kernel(const StepParams p, const DpmParams q) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ float s_noise[32][33];
  const int b = blockIdx.z;
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int s = *p.step_ptr;
  const int k = p.step_ptr[2] - s;                      // loop iteration since the history started
  const int call_t0 = p.tape_t0 >= 0 ? p.tape_t0 : p.step_ptr[3];
  const int eff = min(min(q.order, k + 1), s + 1);      // effective order: lower while the history fills and at the end
  if (s > 0) fill_noise_tile<kWin>(p, s, call_t0, b, l0, c0, s_noise);
  __syncthreads();
  const float4 cf = *reinterpret_cast<const float4*>(q.coef + (size_t)s * 4);  // (A, B0, B1, Cn)
  {
    const int tid = ty * 32 + tx;
    const int ll = tid >> 3, cq = (tid & 7) * 4;
    const int l = l0 + ll, c = c0 + cq;
    if (l < p.L && c < p.D_pad) {
      const size_t idx = ((size_t)b * p.L + l) * p.D_pad + c;
      float* cur = q.x0_hist + (size_t)(k % 3) * q.hist_stride;
      float4 m1v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (eff >= 2) m1v = *reinterpret_cast<const float4*>(q.x0_hist + (size_t)((k + 2) % 3) * q.hist_stride + idx);  // k - 1
      const float m1[4] = {m1v.x, m1v.y, m1v.z, m1v.w};
      float xtv[4], x04[4], xn4[4];
      load_step_x0<kWin>(p, idx, b, c, s, xtv, x04);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float x0 = x04[j];
        float xn = 0.f;
        if (c + j < p.D) {
          xn = __fadd_rn(__fmul_rn(cf.x, xtv[j]), __fmul_rn(cf.y, x0));
          if (eff >= 2) xn = __fadd_rn(xn, __fmul_rn(cf.z, m1[j]));
          xn = s != 0 ? __fadd_rn(xn, __fmul_rn(cf.w, s_noise[cq + j][ll])) : x0;  // s = 0 lands on abar = 1: x = m0
        }
        xn4[j] = xn;
      }
      *reinterpret_cast<float4*>(cur + idx) = make_float4(x04[0], x04[1], x04[2], x04[3]);
      store_step_state(p, idx, xn4, x04, true);
    }
  }
  advance_step(p.step_ptr, s - 1);
}

// ---------------------------------------------------------------------------------------------
// diffusion step. grid: (ceil(L/32), ceil(D_pad/32), B); block 32x8. Each block owns a 32(l) x 32(c)
// tile: frame-major operands are read/written with c fastest, the reference-layout noise tape with
// l fastest, through a padded smem tile.
// ---------------------------------------------------------------------------------------------
template <bool kWin>
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
  if (want_noise) fill_noise_tile<kWin>(p, t, tape_t0, b, l0, c0, s_noise);
  __syncthreads();

  // ---- per-step scalars (fp32, gathered exactly like _extract_into_tensor(...).float()) ----
  // (sampler 2 = plain denoiser evaluation: no schedule is needed, and none may be set)
  const float coef1 = p.sampler == 0 ? p.tab.post_coef1[t] : 0.f, coef2 = p.sampler == 0 ? p.tab.post_coef2[t] : 0.f;
  const float logvar = p.sampler == 0 ? p.tab.post_logvar[t] : 0.f;
  const float nonzero = (t != 0) ? 1.0f : 0.0f;

  // one thread = 4 consecutive features of one frame (16-byte accesses; D_pad is a multiple of 8)
  {
    const int tid = ty * 32 + tx;
    const int ll = tid >> 3, cq = (tid & 7) * 4;
    const int l = l0 + ll, c = c0 + cq;
    if (l < p.L && c < p.D_pad) {
      const size_t idx = ((size_t)b * p.L + l) * p.D_pad + c;
      float xtv[4], x04[4], xn4[4];
      load_step_x0<kWin>(p, idx, b, c, t, xtv, x04);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float x0 = x04[j];
        float xn = 0.f;
        if (c + j < p.D) {
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
      }
      store_step_state(p, idx, xn4, x04, true);
    }
  }

  if (p.advance) advance_step(p.step_ptr, t - 1);
}

// ---------------------------------------------------------------------------------------------
// RePaint resampling (Lugmayr et al. 2022, "time travel"): one op of the walk (engine.cu, repaint_walk) at the position
// s = step_ptr[0], on frame-major state [B*L, D_pad], with diffusion_step_kernel's grid, block and noise tile.
//   phase 0  denoise at s: p_sample at s with diffusion_step_kernel's DDPM arithmetic (x0 through load_step_x0, so
//            CFG, keyframe input, imputation and guidance as in DDPM; at s = 0 the sample is x0); s -> s - 1
//   phase 1  undo into u = s + 1: x <- a_u x + b_u z, one forward step of the spaced chain (non-contracted fp32,
//            multiply then add); pred_xstart is left as it is; s -> s + 1
// Every op takes one draw.  d = step_ptr[5] is the op's index in the walk started at t0 = step_ptr[2], and step_ptr[4]
// the index of the call's first op, so the draw is number d - step_ptr[4] of the call (tape slice, torch.randn_like
// stream).  The engine generator gives the first denoise op at s p_sample_loop's stream for step s (s + 1) and every
// other op the stream kWalkStream + 1 + d, which no step reaches.  The first visit of s is op (t0 - s) + 2 j (r - 1) n_s,
// n_s the number of jump points t >= s (t % j == 0, t + j <= t0).  fill_noise_tile numbers the draw (tape_t0 - t) and
// keys the stream t + 1, so it is called with t = key and tape_t0 = key + draw number.
// ---------------------------------------------------------------------------------------------
constexpr int kWalkStream = 1 << 30;

// advance_step for a walk op: the last block to arrive also moves the walk index step_ptr[5] to the next op.  (A copy,
// not an option of advance_step, so the six step kernels that use advance_step compile as before.)
__device__ __forceinline__ void advance_walk(int* step_ptr, int next) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0) {
    const unsigned int total = gridDim.x * gridDim.y * gridDim.z;
    unsigned int* counter = reinterpret_cast<unsigned int*>(step_ptr + 1);
    if (atomicAdd(counter, 1u) == total - 1) {
      *counter = 0;
      *step_ptr = next;
      step_ptr[5] += 1;
    }
  }
}

__global__ void __launch_bounds__(256) repaint_step_kernel(const StepParams p, const RepaintParams q) {
  griddep_launch_dependents();
  griddep_wait();
  __shared__ float s_noise[32][33];
  const int b = blockIdx.z;
  const int l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int s = *p.step_ptr;
  const int t0 = p.step_ptr[2], d = p.step_ptr[5];
  const int j = q.jump_length;
  const bool denoise = q.phase == 0;
  const bool first = denoise && d == t0 - s + 2 * j * (q.jump_n_sample - 1) * max(0, t0 / j - (s + j - 1) / j);
  const int key = first ? s : kWalkStream + d;
  fill_noise_tile(p, key, key + (d - p.step_ptr[4]), b, l0, c0, s_noise);
  __syncthreads();

  // per-op scalars: DDPM's (gathered like _extract_into_tensor(...).float()) or the undo row of s + 1
  float coef1 = 0.f, coef2 = 0.f, logvar = 0.f, ua = 0.f, ub = 0.f;
  if (denoise) {
    coef1 = p.tab.post_coef1[s]; coef2 = p.tab.post_coef2[s]; logvar = p.tab.post_logvar[s];
  } else {
    ua = q.undo_coef[(size_t)(s + 1) * 4]; ub = q.undo_coef[(size_t)(s + 1) * 4 + 1];
  }
  const float nonzero = (s != 0) ? 1.0f : 0.0f;
  {
    const int tid = ty * 32 + tx;
    const int ll = tid >> 3, cq = (tid & 7) * 4;
    const int l = l0 + ll, c = c0 + cq;
    if (l < p.L && c < p.D_pad) {
      const size_t idx = ((size_t)b * p.L + l) * p.D_pad + c;
      float xtv[4], x04[4] = {0.f, 0.f, 0.f, 0.f}, xn4[4];
      if (denoise) {
        load_step_x0(p, idx, b, c, s, xtv, x04);
      } else {
        const float4 xt4 = *reinterpret_cast<const float4*>(p.x_t + idx);
        xtv[0] = xt4.x; xtv[1] = xt4.y; xtv[2] = xt4.z; xtv[3] = xt4.w;
      }
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        float xn = 0.f;
        if (c + jj < p.D) {
          const float noise = s_noise[cq + jj][ll];
          if (denoise) {
            // diffusion_step_kernel's DDPM branch: mean = coef1*x0 + coef2*x_t; sample = mean + nonzero*exp(0.5*logvar)*z
            const float mean = __fadd_rn(__fmul_rn(coef1, x04[jj]), __fmul_rn(coef2, xtv[jj]));
            const float sd = expf(__fmul_rn(0.5f, logvar));
            xn = __fadd_rn(mean, __fmul_rn(__fmul_rn(nonzero, sd), noise));
          } else {
            xn = __fadd_rn(__fmul_rn(ua, xtv[jj]), __fmul_rn(ub, noise));
          }
        }
        xn4[jj] = xn;
      }
      store_step_state(p, idx, xn4, x04, denoise);
    }
  }
  advance_walk(p.step_ptr, denoise ? s - 1 : s + 1);
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

__global__ void __launch_bounds__(256) window_crop_kernel(const float* __restrict__ global, int Bg, int K, int D, int N, int F,
                                                          const int* __restrict__ f0, float* __restrict__ windows) {
  const size_t n = (size_t)Bg * K * D * F;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int l = (int)(i % F);
    const size_t r = i / F;
    const int c = (int)(r % D);
    const int row = (int)(r / D);
    windows[i] = global[((size_t)(row / K) * D + c) * N + f0[row % K] + l];
  }
}

__global__ void __launch_bounds__(256) window_gather_kernel(const float* __restrict__ frames, int Bg, int K, int D, int N, int F,
                                                            int D_pad, const int* __restrict__ f0, float* __restrict__ global) {
  const size_t n = (size_t)Bg * D * N;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int g = (int)(i % N);
    const size_t r = i / N;
    const int c = (int)(r % D);
    const int s = (int)(r / D);
    int k = 0;
    while (f0[k] + F <= g) ++k;  // the first window covering g (the last window ends at N)
    global[i] = frames[(((size_t)s * K + k) * F + (g - f0[k])) * D_pad + c];
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

__global__ void set_int_kernel(int* p, int v, int next) {
  p[0] = v;
  p[1] = next;  // after the step index: the block-arrival counter (0); after the history's first step: the call's
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
  const auto kernel = p.win_K > 1 ? diffusion_step_kernel<true> : diffusion_step_kernel<false>;
  return launch_kernel(kernel, grid, block, 0, stream, p);
}

cudaError_t launch_plms_step(const StepParams& p, const PlmsParams& q, cudaStream_t stream) {
  if (q.order < 2 || q.order > 4 || q.phase < 0 || q.phase > 2 || (p.D_pad & 3) || !p.x_next || !p.x_next_hi || !q.eps_hist ||
      !q.x_keep)
    return cudaErrorInvalidValue;
  const size_t n4 = (size_t)p.B * p.L * p.D_pad / 4;
  const auto kernel = p.win_K > 1 ? plms_step_kernel<true> : plms_step_kernel<false>;
  return launch_kernel(kernel, dim3((unsigned)((n4 + 255) / 256)), dim3(256), 0, stream, p, q);
}

cudaError_t launch_dpm_solver_step(const StepParams& p, const DpmParams& q, cudaStream_t stream) {
  if (q.order < 1 || q.order > 3 || (p.D_pad & 3) || !p.x_next || !p.x_next_hi || !q.x0_hist || !q.coef)
    return cudaErrorInvalidValue;
  const size_t n4 = (size_t)p.B * p.L * p.D_pad / 4;
  const auto kernel = p.win_K > 1 ? dpm_solver_step_kernel<true> : dpm_solver_step_kernel<false>;
  return launch_kernel(kernel, dim3((unsigned)((n4 + 255) / 256)), dim3(256), 0, stream, p, q);
}

cudaError_t launch_dpm_solver_sde_step(const StepParams& p, const DpmParams& q, cudaStream_t stream) {
  if (q.order < 1 || q.order > 2 || (p.D_pad & 3) || !p.x_next || !p.x_next_hi || !q.x0_hist || !q.coef)
    return cudaErrorInvalidValue;
  dim3 grid((p.L + 31) / 32, (p.D_pad + 31) / 32, p.B), block(32, 8);
  const auto kernel = p.win_K > 1 ? dpm_solver_sde_step_kernel<true> : dpm_solver_sde_step_kernel<false>;
  return launch_kernel(kernel, grid, block, 0, stream, p, q);
}

cudaError_t launch_repaint_step(const StepParams& p, const RepaintParams& q, cudaStream_t stream) {
  if (q.phase < 0 || q.phase > 1 || q.jump_length < 1 || q.jump_n_sample < 1 || (p.D_pad & 3) || !p.x_next ||
      !p.x_next_hi || !q.undo_coef)
    return cudaErrorInvalidValue;
  dim3 grid((p.L + 31) / 32, (p.D_pad + 31) / 32, p.B), block(32, 8);
  return launch_kernel(repaint_step_kernel, grid, block, 0, stream, p, q);
}

cudaError_t launch_unipc_step(const StepParams& p, const UnipcParams& q, cudaStream_t stream) {
  if (q.order < 1 || q.order > 3 || (q.corrector && !q.xc) || (p.D_pad & 3) || !p.x_next || !p.x_next_hi || !q.x0_hist || !q.coef)
    return cudaErrorInvalidValue;
  const size_t n4 = (size_t)p.B * p.L * p.D_pad / 4;
  const auto kernel = p.win_K > 1 ? unipc_step_kernel<true> : unipc_step_kernel<false>;
  return launch_kernel(kernel, dim3((unsigned)((n4 + 255) / 256)), dim3(256), 0, stream, p, q);
}

cudaError_t launch_ddim_reverse_step(const StepParams& p, cudaStream_t stream) {
  if ((p.D_pad & 3) || !p.x_next || !p.x_next_hi || !p.tab.acp_next) return cudaErrorInvalidValue;
  const size_t n4 = (size_t)p.B * p.L * p.D_pad / 4;
  return launch_kernel(ddim_reverse_step_kernel, dim3((unsigned)((n4 + 255) / 256)), dim3(256), 0, stream, p);
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

cudaError_t launch_window_crop(const float* global, int Bg, int K, int D, int N, int F, const int* f0, float* windows,
                               cudaStream_t stream) {
  window_crop_kernel<<<grid_for((size_t)Bg * K * D * F, 256), 256, 0, stream>>>(global, Bg, K, D, N, F, f0, windows);
  return cudaGetLastError();
}

cudaError_t launch_window_gather(const float* frames, int Bg, int K, int D, int N, int F, int D_pad, const int* f0,
                                 float* global, cudaStream_t stream) {
  window_gather_kernel<<<grid_for((size_t)Bg * D * N, 256), 256, 0, stream>>>(frames, Bg, K, D, N, F, D_pad, f0, global);
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

cudaError_t launch_set_int(int* p, int v, cudaStream_t stream, int next) {
  set_int_kernel<<<1, 1, 0, stream>>>(p, v, next);
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
