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
template <bool F16, bool JOINT>
__global__ void __launch_bounds__(256) guidance_seed_kernel(const GuidanceSeedParams p) {
  const size_t n = (size_t)p.B * p.L * p.D_pad;
  float cr = 0.f, cj = 0.f;
  if constexpr (JOINT) {
    const int t = *p.step_ptr;
    cr = p.seed_coef[2 * t];
    cj = p.seed_coef[2 * t + 1];
  }
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % p.D_pad);
    const int b = (int)(i / ((size_t)p.L * p.D_pad));
    const bool kf = F16 && p.keyframe_scale;
    float gc = 0.f, gu = 0.f, gn = 0.f;
    if (c < p.D) {
      float hat = p.model_out[i];
      float s = 1.f, w = 0.f;
      if (p.cfg) {
        const float u = p.model_out[i + n];
        s = p.text_scale[b];
        if (kf) {
          // x0_hat = (n + w_k (u - n)) + s (c - u)   (keyframe CFG)
          const float nf = p.model_out[i + 2 * n];
          w = p.keyframe_scale[b];
          hat = __fadd_rn(__fadd_rn(nf, __fmul_rn(w, __fsub_rn(u, nf))), __fmul_rn(s, __fsub_rn(hat, u)));
        } else {
          hat = __fadd_rn(u, __fmul_rn(s, __fsub_rn(hat, u)));  // x0_hat = u + s (c - u)   (cfg_sampler.py:35)
        }
      }
      const float m = p.obs_mask[i] ? 1.f : 0.f;
      float G = -2.f * (p.x_obs[i] - hat) * m;  // d/dx0_hat of ((x_obs - x0_hat)^2 * M)
      if constexpr (JOINT) G = __fadd_rn(__fmul_rn(cr, G), __fmul_rn(cj, p.joint_grad[i]));
      gc = p.cfg ? s * G : G;
      // the sums autograd forms: u receives w_k G from (u - n) and -(s G) from (c - u); n receives G and -(w_k G)
      if (kf) {
        gu = __fsub_rn(__fmul_rn(G, w), __fmul_rn(G, s));
        gn = __fsub_rn(G, __fmul_rn(G, w));
      } else {
        gu = F16 ? __fsub_rn(G, __fmul_rn(G, s)) : (1.f - s) * G;
      }
    }
    if constexpr (F16) {
      const int l = (int)((i / p.D_pad) % p.L);
      __half* seed = reinterpret_cast<__half*>(p.seed_hi);
      seed[((size_t)b * p.row_period + p.row_lo + l) * p.D_pad + c] = __float2half_rn(gc);
      if (p.cfg) seed[((size_t)(b + p.B) * p.row_period + p.row_lo + l) * p.D_pad + c] = __float2half_rn(gu);
      if (kf) seed[((size_t)(b + 2 * p.B) * p.row_period + p.row_lo + l) * p.D_pad + c] = __float2half_rn(gn);
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
// joint-position guidance seed (launch_joint_seed): recover_from_ric's forward and its VJP, one thread per frame
// ---------------------------------------------------------------------------------------------
// Inclusive prefix sum over the 256 threads of the block in thread order.  wsum: 8 floats of shared memory.
__device__ __forceinline__ float block_scan_256(float v, float* wsum) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v = __fadd_rn(v, u);
  }
  if (lane == 31) wsum[w] = v;
  __syncthreads();
  if (w == 0) {
    float t = lane < 8 ? wsum[lane] : 0.f;
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
      const float u = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t = __fadd_rn(t, u);
    }
    if (lane < 8) wsum[lane] = t;
  }
  __syncthreads();
  if (w > 0) v = __fadd_rn(v, wsum[w - 1]);
  __syncthreads();  // wsum may be reused
  return v;
}

// qrot(qinv(q), (x, 0, z)) for q = (cos a, 0, sin a, 0) in qrot's operation order (recover_from_ric_kernel's), i.e. the
// rotation by 2a about y: x' = C x - S z, z' = S x + C z with C = 1 - 2 sin^2 a, S = 2 sin a cos a
__device__ __forceinline__ void rot_y(float c, float sn, float x, float z, float& xo, float& zo) {
  const float qy = -sn;
  const float uv0 = __fmul_rn(qy, z), uv2 = -__fmul_rn(qy, x);
  const float uuv0 = __fmul_rn(qy, uv2), uuv2 = -__fmul_rn(qy, uv0);
  xo = __fadd_rn(x, __fmul_rn(2.f, __fadd_rn(__fmul_rn(c, uv0), uuv0)));
  zo = __fadd_rn(z, __fmul_rn(2.f, __fadd_rn(__fmul_rn(c, uv2), uuv2)));
}

// Foot-contact guidance's foot joints (7, 10, 8, 11) in label order: the index of joint j, or -1.
__device__ __forceinline__ int foot_index(int j) {
  return j == 7 ? 0 : j == 10 ? 1 : j == 8 ? 2 : j == 11 ? 3 : -1;
}

// The joint seed's body.  FC: foot-contact guidance (JointSeedParams::contact); OB: obstacle-avoidance guidance
// (JointSeedParams::obstacle).  The instance without either is the joint seed alone.
template <bool FC, bool OB>
__device__ __forceinline__ void joint_seed(const JointSeedParams& p) {
  __shared__ float sa[256], sb[256], sc[256], wsum[8];
  // FC: world positions of the four foot joints per frame ([3 k + axis][f]) and kappa(f, k) m(f) m(f + 1) ([k][f])
  __shared__ float fpos[FC ? 12 * 256 : 1];
  __shared__ uint8_t fw[FC ? 4 * 256 : 1];
  // OB: this sample's obstacles (c_x, c_z, r)
  __shared__ float obs[OB ? 3 * kMaxObstacles : 1];
  const int b = blockIdx.x, f = threadIdx.x, L = p.L;
  const bool live = f < L;
  const long long base = (long long)b * p.sb + (long long)f * p.sf;
  const float s = p.x0_u ? p.text_scale[b] : 0.f;
  const float w = p.x0_n ? p.keyframe_scale[b] : 0.f;
  // de-normalised feature c of this thread's frame, x0_hat formed as guidance_seed_kernel forms it
  auto feat = [&](int c) -> float {
    const long long o = base + (long long)c * p.sc;
    float hat = p.x0[o];
    if (p.x0_n) {
      const float u = p.x0_u[o], nf = p.x0_n[o];
      hat = __fadd_rn(__fadd_rn(nf, __fmul_rn(w, __fsub_rn(u, nf))), __fmul_rn(s, __fsub_rn(hat, u)));
    } else if (p.x0_u) {
      const float u = p.x0_u[o];
      hat = __fadd_rn(u, __fmul_rn(s, __fsub_rn(hat, u)));
    }
    return __fadd_rn(__fmul_rn(hat, p.stdv[c]), p.mean[c]);
  };
  float d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;
  if (live) { d0 = feat(0); d1 = feat(1); d2 = feat(2); d3 = feat(3); }
  // ---- forward: heading and root (recover_root_rot_pos) ----
  float ang = d0, rx = d1, rz = d2, vx = 0.f, vz = 0.f, r_x = 0.f, r_z = 0.f;
  if (!p.abs_3d) {
    sa[f] = d0; sb[f] = d1; sc[f] = d2;
    __syncthreads();
    const bool prev = live && f >= 1;
    ang = block_scan_256(prev ? sa[f - 1] : 0.f, wsum);  // exclusive prefix sum of the angular velocity
    vx = prev ? sb[f - 1] : 0.f;
    vz = prev ? sc[f - 1] : 0.f;
    float c0, s0;
    sincosf(ang, &s0, &c0);
    rot_y(c0, s0, vx, vz, r_x, r_z);
    rx = block_scan_256(r_x, wsum);                       // root x, z: inclusive prefix sums of the rotated velocity
    rz = block_scan_256(r_z, wsum);
  }
  float sn, cs;
  sincosf(ang, &sn, &cs);
  const float C2 = __fsub_rn(1.f, __fmul_rn(2.f, __fmul_rn(sn, sn))), S2 = __fmul_rn(2.f, __fmul_rn(sn, cs));
  // ---- the coefficients of the terms (FC / OB: the joint seed applies them itself) ----
  float cj = 1.f, cc = 0.f, co = 0.f;
  if constexpr (FC || OB) {
    constexpr int stride = OB ? 3 : 2;
    if (p.step_ptr) {
      const int t = *p.step_ptr;
      cj = p.coef[stride * t];
      if constexpr (FC) cc = p.coef[stride * t + 1];
      if constexpr (OB) co = p.coef[stride * t + 2];
    } else {
      cj = p.c_j;
      cc = p.c_c;
      co = p.c_o;
    }
  }
  if constexpr (OB) {
    if (f < 3 * p.n_obstacles) obs[f] = p.obstacles[(size_t)b * 3 * p.n_obstacles + f];
    __syncthreads();
  }
  // ---- FC: the foot joints' positions and contact weights, exchanged with the neighbouring frames ----
  if constexpr (FC) {
    const bool pair = live && f + 1 < L && (!p.valid || (p.valid[(size_t)b * L + f] && p.valid[(size_t)b * L + f + 1]));
    for (int k = 0; k < 4; ++k) {
      const int j = k == 0 ? 7 : k == 1 ? 10 : k == 2 ? 8 : 11;
      const int c0 = 4 + 3 * (j - 1);
      float xo = 0.f, zo = 0.f, ly = 0.f;
      bool contact = false;
      if (live) {
        const float lx = feat(c0), lz = feat(c0 + 2);
        ly = feat(c0 + 1);
        rot_y(cs, sn, lx, lz, xo, zo);
        contact = feat(kContactChannel + k) > 0.5f;
      }
      fpos[(3 * k) * 256 + f] = __fadd_rn(xo, rx);
      fpos[(3 * k + 1) * 256 + f] = ly;
      fpos[(3 * k + 2) * 256 + f] = __fadd_rn(zo, rz);
      fw[k * 256 + f] = pair && contact;
    }
    __syncthreads();
  }
  // dL_c/dP of coordinate a of foot joint k at this frame: 2 w(f - 1) (P(f) - P(f - 1)) - 2 w(f) (P(f + 1) - P(f))
  auto contact_grad = [&](int k, int a) -> float {
    const float* q = fpos + (3 * k + a) * 256;
    const float in = f >= 1 && fw[k * 256 + f - 1] ? __fmul_rn(2.f, __fsub_rn(q[f], q[f - 1])) : 0.f;
    const float out = fw[k * 256 + f] ? __fmul_rn(2.f, __fsub_rn(q[f + 1], q[f])) : 0.f;
    return __fsub_rn(in, out);
  };
  // dL_o/dP^x, dL_o/dP^z of a joint of S at world (px, pz) on this frame, L_o's 1 / L and m_o(f) included: the sum over
  // the obstacles it is inside (distance <= r) of -(P - c) / distance, 0 at distance 0 (torch's subgradients)
  const float o_scale = OB && live && (!p.obstacle_valid || p.obstacle_valid[(size_t)b * L + f]) ? __frcp_rn((float)L) : 0.f;
  auto obstacle_grad = [&](float px, float pz, float& gx, float& gz) {
    float sx = 0.f, sz = 0.f;
    for (int k = 0; k < p.n_obstacles; ++k) {
      const float dx = __fsub_rn(px, obs[3 * k]), dz = __fsub_rn(pz, obs[3 * k + 1]);
      const float d = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dz, dz)));
      if (d <= obs[3 * k + 2] && d > 0.f) {
        sx = __fadd_rn(sx, __fdiv_rn(dx, d));
        sz = __fadd_rn(sz, __fdiv_rn(dz, d));
      }
    }
    gx = -__fmul_rn(sx, o_scale);
    gz = -__fmul_rn(sz, o_scale);
  };
  auto in_s = [&](int j) { return OB && ((p.obstacle_joints >> j) & 1u); };
  // FC / OB: c_j (joint term) + c_c (contact term) + c_o (obstacle term); otherwise the joint term unscaled
  auto comb = [&](float gj, float gc, float go) -> float {
    if constexpr (!FC && !OB) return gj;
    float r = __fmul_rn(cj, gj);
    if constexpr (FC) r = __fadd_rn(r, __fmul_rn(cc, gc));
    if constexpr (OB) r = __fadd_rn(r, __fmul_rn(co, go));
    return r;
  };
  // ---- joints: residuals, the gradients of the local coordinates, and the sums over joints ----
  float g_ang = 0.f, g_rx = 0.f, g_rz = 0.f, g_ry = 0.f;
  float* o = p.out + base;
  if (live) {
    const size_t jb = ((size_t)b * L + f) * 66;
    // FC / OB without joint targets: the joint term is zero (its mask reads as all-false)
    const bool jt = !(FC || OB) || p.mask;
    const float* tg = jt ? p.target + jb : nullptr;
    const uint8_t* mk = jt ? p.mask + jb : nullptr;
    auto on = [&](int i) { return jt && mk[i]; };
    g_rx = on(0) ? __fmul_rn(2.f, __fsub_rn(rx, tg[0])) : 0.f;
    g_ry = on(1) ? __fmul_rn(2.f, __fsub_rn(d3, tg[1])) : 0.f;
    g_rz = on(2) ? __fmul_rn(2.f, __fsub_rn(rz, tg[2])) : 0.f;
    if constexpr (FC || OB) {
      float ox = 0.f, oz = 0.f;
      if (in_s(0)) obstacle_grad(rx, rz, ox, oz);
      g_rx = comb(g_rx, 0.f, ox);
      g_ry = comb(g_ry, 0.f, 0.f);
      g_rz = comb(g_rz, 0.f, oz);
    }
    for (int j = 1; j < 22; ++j) {
      const int c0 = 4 + 3 * (j - 1);
      const float lx = feat(c0), ly = feat(c0 + 1), lz = feat(c0 + 2);
      float xo, zo;
      rot_y(cs, sn, lx, lz, xo, zo);
      float gx = on(3 * j) ? __fmul_rn(2.f, __fsub_rn(__fadd_rn(xo, rx), tg[3 * j])) : 0.f;
      float gy = on(3 * j + 1) ? __fmul_rn(2.f, __fsub_rn(ly, tg[3 * j + 1])) : 0.f;
      float gz = on(3 * j + 2) ? __fmul_rn(2.f, __fsub_rn(__fadd_rn(zo, rz), tg[3 * j + 2])) : 0.f;
      if constexpr (FC || OB) {
        const int k = FC ? foot_index(j) : -1;
        float ox = 0.f, oz = 0.f;
        if (in_s(j)) obstacle_grad(__fadd_rn(xo, rx), __fadd_rn(zo, rz), ox, oz);
        gx = comb(gx, k >= 0 ? contact_grad(k, 0) : 0.f, ox);
        gy = comb(gy, k >= 0 ? contact_grad(k, 1) : 0.f, 0.f);
        gz = comb(gz, k >= 0 ? contact_grad(k, 2) : 0.f, oz);
      }
      o[(long long)c0 * p.sc] = __fmul_rn(__fadd_rn(__fmul_rn(gx, C2), __fmul_rn(gz, S2)), p.stdv[c0]);
      o[(long long)(c0 + 1) * p.sc] = __fmul_rn(gy, p.stdv[c0 + 1]);
      o[(long long)(c0 + 2) * p.sc] = __fmul_rn(__fsub_rn(__fmul_rn(gz, C2), __fmul_rn(gx, S2)), p.stdv[c0 + 2]);
      g_ang = __fadd_rn(g_ang, __fmul_rn(2.f, __fsub_rn(__fmul_rn(gz, xo), __fmul_rn(gx, zo))));
      g_rx = __fadd_rn(g_rx, gx);
      g_rz = __fadd_rn(g_rz, gz);
    }
  }
  // ---- root and heading channels ----
  float g0 = g_ang, g1 = g_rx, g2 = g_rz;
  if (!p.abs_3d) {
    // root_f = sum_{k <= f} r_k: dL/dr_k = sum_{f >= k} dL/droot_f, a suffix sum (thread t scans frame L - 1 - t)
    __syncthreads();
    sb[f] = g_rx; sc[f] = g_rz;
    __syncthreads();
    const int k = L - 1 - f;
    const float Gx = block_scan_256(k >= 0 ? sb[k] : 0.f, wsum);
    const float Gz = block_scan_256(k >= 0 ? sc[k] : 0.f, wsum);
    if (k >= 0) { sb[k] = Gx; sc[k] = Gz; }
    __syncthreads();
    float G_x = 0.f, G_z = 0.f;
    if (live) { G_x = sb[f]; G_z = sc[f]; }
    __syncthreads();
    // r_f = rot(ang_f) v_f, v_f = (d1, d2) of frame f - 1
    sb[f] = __fadd_rn(__fmul_rn(G_x, C2), __fmul_rn(G_z, S2));
    sc[f] = __fsub_rn(__fmul_rn(G_z, C2), __fmul_rn(G_x, S2));
    sa[f] = __fadd_rn(g_ang, __fmul_rn(2.f, __fsub_rn(__fmul_rn(G_z, r_x), __fmul_rn(G_x, r_z))));
    __syncthreads();
    // ang_f = sum_{k < f} d0_k: dL/dd0_k = sum_{f > k} dL/dang_f, an exclusive suffix sum
    const float ga = block_scan_256(k >= 0 && k + 1 < L ? sa[k + 1] : 0.f, wsum);
    if (k >= 0) o = p.out + (long long)b * p.sb + (long long)k * p.sf;  // this thread now writes frame k's heading
    g0 = ga;
    g1 = live && f + 1 < L ? sb[f + 1] : 0.f;
    g2 = live && f + 1 < L ? sc[f + 1] : 0.f;
    if (k >= 0) o[0] = __fmul_rn(g0, p.stdv[0]);
    o = p.out + base;
  } else if (live) {
    o[0] = __fmul_rn(g0, p.stdv[0]);
  }
  if (live) {
    o[p.sc] = __fmul_rn(g1, p.stdv[1]);
    o[2 * p.sc] = __fmul_rn(g2, p.stdv[2]);
    o[3 * p.sc] = __fmul_rn(g_ry, p.stdv[3]);
  }
  // ---- exact zeros on channels 67 .. out_cols - 1 (row-contiguous for the frame-major layout) ----
  const int nz = p.out_cols - kJointChannels;
  float* ob = p.out + (long long)b * p.sb;
  for (int i = threadIdx.x; i < L * nz; i += blockDim.x) {
    const int ff = i / nz, c = kJointChannels + i % nz;
    ob[(long long)ff * p.sf + (long long)c * p.sc] = 0.f;
  }
}

template <bool FC>
__global__ void __launch_bounds__(256) joint_seed_kernel(const JointSeedParams p) {
  joint_seed<FC, false>(p);
}

// The joint seed with obstacle-avoidance guidance (and foot-contact guidance when FC).
template <bool FC>
__global__ void __launch_bounds__(256) obstacle_seed_kernel(const JointSeedParams p) {
  joint_seed<FC, true>(p);
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
  if (p.joint_grad) {
    if (p.f16) guidance_seed_kernel<true, true><<<(unsigned)grid, 256, 0, stream>>>(p);
    else guidance_seed_kernel<false, true><<<(unsigned)grid, 256, 0, stream>>>(p);
  } else {
    if (p.f16) guidance_seed_kernel<true, false><<<(unsigned)grid, 256, 0, stream>>>(p);
    else guidance_seed_kernel<false, false><<<(unsigned)grid, 256, 0, stream>>>(p);
  }
  return cudaGetLastError();
}

cudaError_t launch_joint_seed(const JointSeedParams& p, cudaStream_t stream) {
  if (p.L < 1 || p.L > 256 || p.D < kJointChannels || p.out_cols < kJointChannels) return cudaErrorInvalidValue;
  if (p.contact && (p.D < kContactChannel + 4 || (p.step_ptr && !p.coef))) return cudaErrorInvalidValue;
  if (p.obstacle && (p.n_obstacles < 0 || p.n_obstacles > kMaxObstacles || (p.n_obstacles > 0 && !p.obstacles) ||
                     (p.obstacle_joints >> 22) != 0 || (p.step_ptr && !p.coef)))
    return cudaErrorInvalidValue;
  if (p.B == 0) return cudaSuccess;
  if (p.obstacle) {
    if (p.contact) obstacle_seed_kernel<true><<<p.B, 256, 0, stream>>>(p);
    else obstacle_seed_kernel<false><<<p.B, 256, 0, stream>>>(p);
  } else if (p.contact) {
    joint_seed_kernel<true><<<p.B, 256, 0, stream>>>(p);
  } else {
    joint_seed_kernel<false><<<p.B, 256, 0, stream>>>(p);
  }
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
