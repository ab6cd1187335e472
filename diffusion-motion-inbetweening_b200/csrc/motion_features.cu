// HumanML3D representation conversions on the GPU (C ABI in include/condmdi_b200.h):
//   cmdi_joints_to_features  extract_features (data_loaders/humanml/scripts/motion_process.py:50-187)
//   cmdi_convert_motion      abs3d_to_rel / rel_to_abs3d (data_loaders/humanml/data/dataset.py:1198-1288, :1327-1401),
//                            and inverse projection + de-normalisation + recover_from_ric on their own
//
// One CTA per sequence: the facing direction is smoothed along time and the absolute root channels are prefix sums,
// so a sequence never leaves shared memory.  The whole conversion is one launch on the caller's stream.
//
// Arithmetic follows the reference's dtypes, operation by operation.  Its quaternion helpers (common/quaternion.py
// qbetween_np / qmul_np / qrot_np / quaternion_to_cont6d_np) cast to float32 torch tensors, so inverse kinematics,
// cont6d and every rotation run in fp32 with separately rounded products and sums (__fmul_rn / __fadd_rn: no FMA
// contraction, as between two torch ops).  What numpy computes in float64 stays in fp64 here: the cross product with
// an int64 axis, gaussian_filter1d (scipy, sigma 20, truncate 4 -> radius 80, mode 'nearest') and the normalisation of
// the smoothed direction; the foot-contact threshold compares in fp64.  torch.cumsum on the CPU accumulates float in
// double (ATen acc_type), and so do the prefix sums below.  De-normalisation and normalisation run in the dataset
// statistics' own dtype (float64 statistics promote the torch expression to float64).
#include <cmath>
#include <cstdint>

#include "../../include/condmdi_b200.h"
#include "kernels.h"

using namespace cmdi;

namespace {

constexpr int kJoints = 22;
constexpr int kFeats = 263;          // 4 + 21*3 + 21*6 + 22*3 + 4
constexpr int kFrontCh = 67;         // channels recover_from_ric reads: root (4) + ric (63)
constexpr int kMaxFrames = 224;
constexpr int kRadius = 80;          // int(4 * 20 + 0.5)
constexpr int kThreads = 256;
constexpr int kRic = 4, kRot = 67, kVel = 193, kFoot = 259;

// paramUtil.t2m_raw_offsets as (axis, sign) of each joint's unit offset; t2m_kinematic_chain flattened
__constant__ int8_t c_off_axis[kJoints] = {0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 2, 2, 1, 0, 0, 2, 1, 1, 1, 1, 1, 1};
__constant__ int8_t c_off_sign[kJoints] = {0, 1, -1, 1, -1, -1, 1, -1, -1, 1, 1, 1, 1, 1, -1, 1, -1, -1, -1, -1, -1, -1};
__constant__ int8_t c_chain[26] = {0, 2, 5, 8, 11, 0, 1, 4, 7, 10, 0, 3, 6, 9, 12, 15, 9, 14, 17, 19, 21, 9, 13, 16, 18, 20};
__constant__ int8_t c_chain_start[6] = {0, 5, 10, 16, 21, 26};

enum Mode { kFromJoints = 0, kAbsToRel = 1, kRelToAbs = 2, kToJoints = 3 };

struct ConvParams {
  int mode;
  const float* in;              // kFromJoints: (seq, frame, 66); otherwise (seq, feature, frame) by the strides below
  long long is, ic, iff;        // input strides: sequence, feature / joint-coordinate, frame
  int B, L;
  int front_abs;                // recover_from_ric(abs_3d=...) of the front end
  const float* inv_proj;        // [263, 263] row-major or null
  const double* mean_in;        // de-normalisation (x * std + mean) or null
  const double* std_in;
  int in_f64;
  const double* mean_out;       // normalisation ((x - mean) / std) of the output, or null (de-normalised features)
  const double* std_out;
  int out_f64;
  double feet_thre;
  float* out;
  long long os, oc, of;         // output strides: sequence, feature (or joint*3 + coordinate), frame
};

struct Q {
  float w, x, y, z;
};

__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }

__device__ __forceinline__ float3 cross(float3 a, float3 b) {  // torch.cross
  return make_float3(sub(mul(a.y, b.z), mul(a.z, b.y)), sub(mul(a.z, b.x), mul(a.x, b.z)), sub(mul(a.x, b.y), mul(a.y, b.x)));
}
__device__ __forceinline__ float sumsq3(float3 v) { return add(add(mul(v.x, v.x), mul(v.y, v.y)), mul(v.z, v.z)); }
__device__ __forceinline__ float3 unit(float3 v) {  // v / np.sqrt((v**2).sum(-1)) in float32
  const float n = __fsqrt_rn(sumsq3(v));
  return make_float3(__fdiv_rn(v.x, n), __fdiv_rn(v.y, n), __fdiv_rn(v.z, n));
}
__device__ __forceinline__ float3 sub3(float3 a, float3 b) { return make_float3(sub(a.x, b.x), sub(a.y, b.y), sub(a.z, b.z)); }

// quaternion.py qrot: v + 2 * (w * uv + uuv), uv = qvec x v, uuv = qvec x uv
__device__ __forceinline__ float3 qrot(Q q, float3 v) {
  const float3 qv = make_float3(q.x, q.y, q.z);
  const float3 uv = cross(qv, v), uuv = cross(qv, uv);
  return make_float3(add(v.x, mul(2.f, add(mul(q.w, uv.x), uuv.x))), add(v.y, mul(2.f, add(mul(q.w, uv.y), uuv.y))),
                     add(v.z, mul(2.f, add(mul(q.w, uv.z), uuv.z))));
}
// quaternion.py qmul: terms[i][j] = r_i * q_j summed left to right
__device__ __forceinline__ Q qmul(Q q, Q r) {
  Q o;
  o.w = sub(sub(sub(mul(r.w, q.w), mul(r.x, q.x)), mul(r.y, q.y)), mul(r.z, q.z));
  o.x = add(sub(add(mul(r.w, q.x), mul(r.x, q.w)), mul(r.y, q.z)), mul(r.z, q.y));
  o.y = sub(add(add(mul(r.w, q.y), mul(r.x, q.z)), mul(r.y, q.w)), mul(r.z, q.x));
  o.z = add(add(sub(mul(r.w, q.z), mul(r.x, q.y)), mul(r.y, q.x)), mul(r.z, q.w));
  return o;
}
__device__ __forceinline__ Q qinv(Q q) { return Q{q.w, -q.x, -q.y, -q.z}; }
__device__ __forceinline__ Q qnormalize(Q q) {
  const float n = __fsqrt_rn(add(add(add(mul(q.w, q.w), mul(q.x, q.x)), mul(q.y, q.y)), mul(q.z, q.z)));
  return Q{__fdiv_rn(q.w, n), __fdiv_rn(q.x, n), __fdiv_rn(q.y, n), __fdiv_rn(q.z, n)};
}
// quaternion.py qbetween: normalize([sqrt(|v0|^2 |v1|^2) + v0.v1, v0 x v1])
__device__ __forceinline__ Q qbetween(float3 v0, float3 v1) {
  const float3 c = cross(v0, v1);
  const float w = add(__fsqrt_rn(mul(sumsq3(v0), sumsq3(v1))), add(add(mul(v0.x, v1.x), mul(v0.y, v1.y)), mul(v0.z, v1.z)));
  return qnormalize(Q{w, c.x, c.y, c.z});
}
// the y-axis rotation (cos a, 0, sin a, 0) of recover_root_rot_pos, inverted, applied to (x, 0, z)
__device__ __forceinline__ float2 rot_y_inv(float c, float s, float x, float z) {
  const float qy = -s;
  const float uv0 = mul(qy, z), uv2 = -mul(qy, x);
  const float uuv0 = mul(qy, uv2), uuv2 = -mul(qy, uv0);
  return make_float2(add(x, mul(2.f, add(mul(c, uv0), uuv0))), add(z, mul(2.f, add(mul(c, uv2), uuv2))));
}

__device__ __forceinline__ float denorm(const ConvParams& p, float x, int c) {
  if (p.in_f64) return (float)__dadd_rn(__dmul_rn((double)x, p.std_in[c]), p.mean_in[c]);
  return add(mul(x, (float)p.std_in[c]), (float)p.mean_in[c]);
}
__device__ __forceinline__ float norm_out(const ConvParams& p, float x, int c) {
  if (!p.mean_out) return x;
  if (p.out_f64) return (float)__ddiv_rn(__dsub_rn((double)x, p.mean_out[c]), p.std_out[c]);
  return __fdiv_rn(sub(x, (float)p.mean_out[c]), (float)p.std_out[c]);
}

__global__ void __launch_bounds__(kThreads) motion_convert_kernel(const ConvParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int L = p.L, tid = threadIdx.x;
  double* fwd = reinterpret_cast<double*>(smem_raw);  // [L][2] raw forward direction (x, z); y is 0
  double* gw = fwd + 2 * L;                           // [kRadius + 1] gaussian weights, centre first
  Q* rq = reinterpret_cast<Q*>(gw + kRadius + 1 + 1); // [L] root quaternions (r_rot)
  float* J = reinterpret_cast<float*>(rq + L);        // [L][22][3] joint positions
  float* dn = J + L * kJoints * 3;                    // [L][67] de-normalised input channels (front end)
  float* r0 = dn + L * kFrontCh;                      // [3][L] root scratch: heading / x / z
  float* r1 = r0 + L;
  float* r2 = r1 + L;
  const long long b = blockIdx.x;
  const float* in = p.in + b * p.is;
  float* out = p.out + b * p.os;
  const bool conv = p.mode == kAbsToRel || p.mode == kRelToAbs;

  // ---- front end: [x @ inv_proj] -> x * std + mean -> recover_from_ric ------------------------------------------
  if (p.mode != kFromJoints) {
    for (int i = tid; i < kFrontCh * L; i += kThreads) {
      const int c = i / L, f = i - c * L;
      float x;
      if (p.inv_proj) {  // np.matmul(data, inv_proj): fp32 dot over the 263 features of the frame
        float acc = 0.f;
        const float* xf = in + f * p.iff;
        for (int k = 0; k < kFeats; ++k) acc = fmaf(xf[k * p.ic], p.inv_proj[k * kFeats + c], acc);
        x = acc;
      } else {
        x = in[c * p.ic + f * p.iff];
      }
      dn[f * kFrontCh + c] = p.mean_in ? denorm(p, x, c) : x;
    }
    __syncthreads();
    // recover_root_rot_pos: heading r0, root x r1, root z r2
    if (p.front_abs) {
      for (int f = tid; f < L; f += kThreads) {
        r0[f] = dn[f * kFrontCh];
        r1[f] = dn[f * kFrontCh + 1];
        r2[f] = dn[f * kFrontCh + 2];
      }
      __syncthreads();
    } else {
      if (tid == 0) {  // r_rot_ang = cumsum([0, w_0, ..., w_{L-2}])
        double acc = 0.0;
        r0[0] = 0.f;
        for (int f = 1; f < L; ++f) {
          acc += (double)dn[(f - 1) * kFrontCh];
          r0[f] = (float)acc;
        }
      }
      __syncthreads();
      for (int f = tid; f < L; f += kThreads) {
        float2 v = make_float2(0.f, 0.f);
        if (f > 0) v = rot_y_inv(cosf(r0[f]), sinf(r0[f]), dn[(f - 1) * kFrontCh + 1], dn[(f - 1) * kFrontCh + 2]);
        r1[f] = v.x;
        r2[f] = v.y;
      }
      __syncthreads();
      if (tid < 2) {
        float* a = tid == 0 ? r1 : r2;
        double acc = 0.0;
        for (int f = 0; f < L; ++f) {
          acc += (double)a[f];
          a[f] = (float)acc;
        }
      }
      __syncthreads();
    }
    for (int i = tid; i < L * kJoints; i += kThreads) {
      const int f = i / kJoints, j = i - f * kJoints;
      float3 v;
      if (j == 0) {
        v = make_float3(r1[f], dn[f * kFrontCh + 3], r2[f]);
      } else {
        const float* ric = dn + f * kFrontCh + kRic + 3 * (j - 1);
        const float2 xz = rot_y_inv(cosf(r0[f]), sinf(r0[f]), ric[0], ric[2]);
        v = make_float3(add(xz.x, r1[f]), ric[1], add(xz.y, r2[f]));
      }
      if (p.mode == kToJoints) {
        float* o = out + f * p.of + (3 * j) * p.oc;
        o[0] = v.x;
        o[p.oc] = v.y;
        o[2 * p.oc] = v.z;
      } else {
        float* o = J + (f * kJoints + j) * 3;
        o[0] = v.x;
        o[1] = v.y;
        o[2] = v.z;
      }
    }
    if (p.mode == kToJoints) return;
  } else {
    for (int i = tid; i < L * kJoints * 3; i += kThreads) {
      const int f = i / (kJoints * 3), r = i - f * (kJoints * 3);
      J[i] = in[f * p.iff + r];
    }
  }
  // gaussian_filter1d weights: exp(-0.5 / sigma^2 * x^2) / sum, x = -80..80
  if (tid <= kRadius) gw[tid] = exp(-0.5 / 400.0 * (double)(tid * tid));
  __syncthreads();
  auto joint = [&](int f, int j) { const float* q = J + (f * kJoints + j) * 3; return make_float3(q[0], q[1], q[2]); };

  // ---- facing direction: across = (r_hip - l_hip) + (sdr_r - sdr_l), forward = (0, 1, 0) x across --------------
  for (int f = tid; f < L; f += kThreads) {
    const float3 a1 = sub3(joint(f, 1), joint(f, 2)), a2 = sub3(joint(f, 17), joint(f, 16));
    const float3 across = unit(make_float3(add(a1.x, a2.x), add(a1.y, a2.y), add(a1.z, a2.z)));
    fwd[2 * f] = (double)across.z;
    fwd[2 * f + 1] = -(double)across.x;
  }
  if (tid == 0) {
    double s = 0.0;
    for (int x = -kRadius; x <= kRadius; ++x) s += gw[x < 0 ? -x : x];
    gw[kRadius + 1] = s;
  }
  __syncthreads();
  const double gsum = gw[kRadius + 1];
  // smoothed, normalised, root_quat = qbetween(forward, +z); frame 0 forced to identity (skeleton.py:81)
  for (int f = tid; f < L; f += kThreads) {
    if (f == 0) {
      rq[0] = Q{1.f, 0.f, 0.f, 0.f};
      continue;
    }
    double sx = __dmul_rn(fwd[2 * f], gw[0] / gsum), sz = __dmul_rn(fwd[2 * f + 1], gw[0] / gsum);
    for (int r = kRadius; r >= 1; --r) {  // scipy's symmetric correlate: centre, then (x[-r] + x[r]) * w[r], far first
      const int lo = max(f - r, 0), hi = min(f + r, L - 1);
      const double w = gw[r] / gsum;
      sx = __dadd_rn(sx, __dmul_rn(__dadd_rn(fwd[2 * lo], fwd[2 * hi]), w));
      sz = __dadd_rn(sz, __dmul_rn(__dadd_rn(fwd[2 * lo + 1], fwd[2 * hi + 1]), w));
    }
    const double n = sqrt(__dadd_rn(__dmul_rn(sx, sx), __dmul_rn(sz, sz)));
    const float3 v0 = make_float3((float)__ddiv_rn(sx, n), 0.f, (float)__ddiv_rn(sz, n));
    rq[f] = qbetween(v0, make_float3(0.f, 0.f, 1.f));
  }
  __syncthreads();

  const int rows = L - 1;
  // emit a feature of row f (< rows); converted rows are normalised and the last row is duplicated (dataset.py:1214)
  auto emit = [&](int f, int c, float v) {
    const float y = norm_out(p, v, c);
    out[f * p.of + c * p.oc] = y;
    if (conv && f == rows - 1) out[rows * p.of + c * p.oc] = y;
  };

  // ---- inverse kinematics down each chain, R restarting at the root quaternion; cont6d of each local rotation ---
  for (int i = tid; i < rows * 5; i += kThreads) {
    const int f = i / 5, ch = i - f * 5;
    Q R = rq[f];
    for (int k = c_chain_start[ch]; k + 1 < c_chain_start[ch + 1]; ++k) {
      const int j0 = c_chain[k], j1 = c_chain[k + 1];
      float3 u = make_float3(0.f, 0.f, 0.f);
      const float sg = (float)c_off_sign[j1];
      if (c_off_axis[j1] == 0) u.x = sg; else if (c_off_axis[j1] == 1) u.y = sg; else u.z = sg;
      const Q rl = qmul(qinv(R), qbetween(u, unit(sub3(joint(f, j1), joint(f, j0)))));
      R = qmul(R, rl);
      // quaternion_to_matrix, columns 0 and 1
      const float two_s = __fdiv_rn(2.f, add(add(add(mul(rl.w, rl.w), mul(rl.x, rl.x)), mul(rl.y, rl.y)), mul(rl.z, rl.z)));
      const float r = rl.w, a = rl.x, bq = rl.y, c = rl.z;
      const float m00 = sub(1.f, mul(two_s, add(mul(bq, bq), mul(c, c))));
      const float m10 = mul(two_s, add(mul(a, bq), mul(c, r)));
      const float m20 = mul(two_s, sub(mul(a, c), mul(bq, r)));
      const float m01 = mul(two_s, sub(mul(a, bq), mul(c, r)));
      const float m11 = sub(1.f, mul(two_s, add(mul(a, a), mul(c, c))));
      const float m21 = mul(two_s, add(mul(bq, c), mul(a, r)));
      const int base = kRot + 6 * (j1 - 1);
      emit(f, base + 0, m00);
      emit(f, base + 1, m10);
      emit(f, base + 2, m20);
      emit(f, base + 3, m01);
      emit(f, base + 4, m11);
      emit(f, base + 5, m21);
    }
  }
  // ---- RIFKE positions, root height and local velocities ------------------------------------------------------
  for (int i = tid; i < rows * kJoints; i += kThreads) {
    const int f = i / kJoints, j = i - f * kJoints;
    const float3 pj = joint(f, j), root = joint(f, 0);
    const float3 ric = qrot(rq[f], make_float3(sub(pj.x, root.x), pj.y, sub(pj.z, root.z)));
    if (j == 0) {
      emit(f, 3, ric.y);
    } else {
      emit(f, kRic + 3 * (j - 1), ric.x);
      emit(f, kRic + 3 * (j - 1) + 1, ric.y);
      emit(f, kRic + 3 * (j - 1) + 2, ric.z);
    }
    const float3 vel = qrot(rq[f], sub3(joint(f + 1, j), pj));
    emit(f, kVel + 3 * j, vel.x);
    emit(f, kVel + 3 * j + 1, vel.y);
    emit(f, kVel + 3 * j + 2, vel.z);
  }
  // ---- root angular / linear velocity and foot contacts ---------------------------------------------------------
  for (int f = tid; f < rows; f += kThreads) {
    const Q rv = qmul(rq[f + 1], qinv(rq[f]));
    r0[f] = asinf(rv.y);
    const float3 v = qrot(rq[f + 1], sub3(joint(f + 1, 0), joint(f, 0)));
    r1[f] = v.x;
    r2[f] = v.z;
    const int feet[4] = {7, 10, 8, 11};  // fid_l, then fid_r
    for (int k = 0; k < 4; ++k) {
      const float3 d = sub3(joint(f + 1, feet[k]), joint(f, feet[k]));
      const float s = add(add(mul(d.x, d.x), mul(d.y, d.y)), mul(d.z, d.z));
      emit(f, kFoot + k, (double)s < p.feet_thre ? 1.f : 0.f);
    }
  }
  __syncthreads();
  if (p.mode != kRelToAbs) {
    for (int f = tid; f < rows; f += kThreads) {
      emit(f, 0, r0[f]);
      emit(f, 1, r1[f]);
      emit(f, 2, r2[f]);
    }
    return;
  }
  // ---- rel_to_abs3d: recover_root_rot_pos(abs_3d=False) over the L rows (last one duplicated), channels 0..2 -----
  // r0/r1/r2 hold rows 0..L-2; the prefix sums only read rows 0..L-2 (row f uses row f-1)
  float* ang = dn;               // [L] the front end is done with dn
  float* px = dn + L;
  float* pz = dn + 2 * L;
  if (tid == 0) {
    double acc = 0.0;
    ang[0] = 0.f;
    for (int f = 1; f < L; ++f) {
      acc += (double)r0[f - 1];
      ang[f] = (float)acc;
    }
  }
  __syncthreads();
  for (int f = tid; f < L; f += kThreads) {
    float2 v = make_float2(0.f, 0.f);
    if (f > 0) v = rot_y_inv(cosf(ang[f]), sinf(ang[f]), r1[f - 1], r2[f - 1]);
    px[f] = v.x;
    pz[f] = v.y;
  }
  __syncthreads();
  if (tid < 2) {
    float* a = tid == 0 ? px : pz;
    double acc = 0.0;
    for (int f = 0; f < L; ++f) {
      acc += (double)a[f];
      a[f] = (float)acc;
    }
  }
  __syncthreads();
  for (int f = tid; f < L; f += kThreads) {
    out[f * p.of] = norm_out(p, ang[f], 0);
    out[f * p.of + p.oc] = norm_out(p, px[f], 1);
    out[f * p.of + 2 * p.oc] = norm_out(p, pz[f], 2);
  }
}

size_t smem_bytes(int L) {
  return (size_t)(2 * L + kRadius + 2) * sizeof(double) + (size_t)L * sizeof(Q) +
         (size_t)(L * kJoints * 3 + L * kFrontCh + 3 * L) * sizeof(float);
}

cudaError_t launch(const ConvParams& p, cudaStream_t stream) {
  if (p.B <= 0) return cudaSuccess;
  const size_t smem = smem_bytes(p.L);
  cudaError_t e = cudaFuncSetAttribute(motion_convert_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  return launch_kernel(motion_convert_kernel, dim3(p.B), dim3(kThreads), smem, stream, p);
}

#define CK(expr)                                                                                    \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) {                                                                        \
      set_last_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__);   \
      return 1;                                                                                     \
    }                                                                                               \
  } while (0)

int check_shape(const char* fn, int num_seqs, int nframes, int joints_num) {
  if (joints_num != kJoints) {
    set_last_error("%s: joints_num must be 22 (HumanML3D skeleton), got %d", fn, joints_num);
    return 1;
  }
  if (nframes < 2 || nframes > kMaxFrames) {
    set_last_error("%s: nframes must satisfy 2 <= nframes <= %d, got %d", fn, kMaxFrames, nframes);
    return 1;
  }
  if (num_seqs < 0) {
    set_last_error("%s: num_seqs must be >= 0, got %d", fn, num_seqs);
    return 1;
  }
  return 0;
}

}  // namespace

extern "C" int cmdi_joints_to_features(const float* joints, long long stride_seq, long long stride_frame, int num_seqs,
                                       int nframes, int joints_num, double feet_thre, float* out, long long ostride_seq,
                                       long long ostride_frame, long long ostride_feat, void* stream) {
  if (check_shape("cmdi_joints_to_features", num_seqs, nframes, joints_num)) return 1;
  if (!joints || !out) {
    set_last_error("cmdi_joints_to_features: null pointer");
    return 1;
  }
  ConvParams p{};
  p.mode = kFromJoints;
  p.in = joints;
  p.is = stride_seq;
  p.iff = stride_frame;
  p.B = num_seqs;
  p.L = nframes;
  p.feet_thre = feet_thre;
  p.out = out;
  p.os = ostride_seq;
  p.of = ostride_frame;
  p.oc = ostride_feat;
  CK(launch(p, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

extern "C" int cmdi_convert_motion(int direction, const float* in, long long stride_seq, long long stride_feat,
                                   long long stride_frame, int num_seqs, int nframes, int nfeats, const float* inv_proj,
                                   const double* mean_in, const double* std_in, int in_f64, const double* mean_out,
                                   const double* std_out, int out_f64, double feet_thre, float* out, long long ostride_seq,
                                   long long ostride_feat, long long ostride_frame, void* stream) {
  if (check_shape("cmdi_convert_motion", num_seqs, nframes, kJoints)) return 1;
  if (nfeats != kFeats) {
    set_last_error("cmdi_convert_motion: nfeats must be 263 (HumanML3D), got %d", nfeats);
    return 1;
  }
  if (direction < CMDI_MOTION_ABS3D_TO_REL || direction > CMDI_MOTION_ABS3D_TO_JOINTS) {
    set_last_error("cmdi_convert_motion: unknown direction %d", direction);
    return 1;
  }
  const bool to_joints = direction == CMDI_MOTION_REL_TO_JOINTS || direction == CMDI_MOTION_ABS3D_TO_JOINTS;
  if (!in || !out || !mean_in || !std_in || (!to_joints && (!mean_out || !std_out))) {
    set_last_error("cmdi_convert_motion: null pointer (input and output, and both statistics pairs unless converting to joints)");
    return 1;
  }
  ConvParams p{};
  p.mode = direction == CMDI_MOTION_ABS3D_TO_REL ? kAbsToRel : direction == CMDI_MOTION_REL_TO_ABS3D ? kRelToAbs : kToJoints;
  p.in = in;
  p.is = stride_seq;
  p.ic = stride_feat;
  p.iff = stride_frame;
  p.B = num_seqs;
  p.L = nframes;
  p.front_abs = direction == CMDI_MOTION_ABS3D_TO_REL || direction == CMDI_MOTION_ABS3D_TO_JOINTS;
  p.inv_proj = inv_proj;
  p.mean_in = mean_in;
  p.std_in = std_in;
  p.in_f64 = in_f64 != 0;
  p.mean_out = to_joints ? nullptr : mean_out;
  p.std_out = to_joints ? nullptr : std_out;
  p.out_f64 = out_f64 != 0;
  p.feet_thre = feet_thre;
  p.out = out;
  p.os = ostride_seq;
  p.oc = ostride_feat;
  p.of = ostride_frame;
  CK(launch(p, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
