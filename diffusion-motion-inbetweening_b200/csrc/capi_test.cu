// Kernel-level C-ABI entry points used by the parity tests (declared in include/condmdi_b200.h).
// They stage fp32 inputs into the bf16 hi/lo planes the kernels consume, build the TMA descriptors,
// launch the production kernel and hand back fp32 results.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/condmdi_b200.h"
#include "kernels.h"

using namespace cmdi;

namespace {

#define CK(expr)                                                                   \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess) {                                                       \
      set_last_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return 1;                                                                    \
    }                                                                              \
  } while (0)

struct DevBuf {
  void* p = nullptr;
  ~DevBuf() {
    if (p) cudaFree(p);
  }
  cudaError_t alloc(size_t bytes) {
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) e = cudaMemset(p, 0, bytes);
    return e;
  }
  template <class T>
  T* as() {
    return reinterpret_cast<T*>(p);
  }
};

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

int num_sms_of_current_device() {
  int dev = 0, n = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n;
}

}  // namespace

extern "C" int cmdi_test_linear(const float* A, const float* W, const float* bias, const float* residual, float* C, int M,
                                int N, int K, int act, int precision, int block_n, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int bn_abs = block_n < 0 ? -block_n : block_n;
  const int Kp = round_up(K, 8), Mp = round_up(M, 256), Np = round_up(N, bn_abs);
  DevBuf a_hi, a_lo, w_hi, w_lo;
  CK(a_hi.alloc((size_t)Mp * Kp * 2));
  CK(a_lo.alloc((size_t)Mp * Kp * 2));
  CK(w_hi.alloc((size_t)Np * Kp * 2));
  CK(w_lo.alloc((size_t)Np * Kp * 2));
  // precision 2 (CMDI_PRECISION_FP16): one fp16 plane per operand, bias and results rounded to fp16 like autocast
  const bool f16 = precision == 2;
  if (f16) {
    CK(launch_conv_weight_planes(A, M, K, 1, K, a_hi.as<__nv_bfloat16>(), nullptr, Kp, stream, true));
    CK(launch_conv_weight_planes(W, N, K, 1, K, w_hi.as<__nv_bfloat16>(), nullptr, Kp, stream, true));
    precision = 1;
  } else {
    CK(launch_split_planes(A, M, K, K, a_hi.as<__nv_bfloat16>(), a_lo.as<__nv_bfloat16>(), Kp, stream));
    CK(launch_split_planes(W, N, K, K, w_hi.as<__nv_bfloat16>(), w_lo.as<__nv_bfloat16>(), Kp, stream));
  }
  const bool pair = true;  // every linear layer runs on the CTA-pair kernel (the sign of block_n is accepted and ignored)
  if (block_n < 0) block_n = -block_n;
  CUtensorMap ma_hi, ma_lo, mw_hi, mw_lo;
  if (make_tmap_bf16_2d(&ma_hi, a_hi.p, Mp, Kp, Kp, 64, 128)) return 1;
  if (make_tmap_bf16_2d(&ma_lo, a_lo.p, Mp, Kp, Kp, 64, 128)) return 1;
  if (make_tmap_bf16_2d(&mw_hi, w_hi.p, Np, Kp, Kp, 64, pair ? block_n / 2 : block_n)) return 1;
  if (make_tmap_bf16_2d(&mw_lo, w_lo.p, Np, Kp, Kp, 64, pair ? block_n / 2 : block_n)) return 1;
  CUtensorMap mc_f32;
  if (make_tmap_2d(&mc_f32, C, 4, M, N, N, 32, 32)) return 1;
  LinearStoreMaps stm;
  stm.f32 = &mc_f32;
  const LinearStoreMaps* stp = getenv("CMDI_EPI") && !strcmp(getenv("CMDI_EPI"), "stg") ? nullptr : &stm;
  LinearParams p{};
  p.M = M; p.N = N; p.K = K; p.nsplit = precision;
  p.bias = bias; p.residual = residual; p.ld_res = N;
  DevBuf ln_g, ln_b, ln_s;
  if (residual && N == 512 && getenv("CMDI_TEST_RES_LN")) {
    // the residual is LayerNorm(`residual`) (gamma = 1.5, beta = -0.25), re-derived in the epilogue from the
    // statistics the LayerNorm kernel publishes
    std::vector<float> hg(512, 1.5f), hb(512, -0.25f);
    CK(ln_g.alloc(512 * 4)); CK(ln_b.alloc(512 * 4)); CK(ln_s.alloc((size_t)M * sizeof(float2)));
    CK(cudaMemcpyAsync(ln_g.p, hg.data(), 512 * 4, cudaMemcpyHostToDevice, stream));
    CK(cudaMemcpyAsync(ln_b.p, hb.data(), 512 * 4, cudaMemcpyHostToDevice, stream));
    CK(cudaStreamSynchronize(stream));
    CK(launch_layernorm512(residual, ln_g.as<float>(), ln_b.as<float>(), 1e-5f, M, nullptr, nullptr, nullptr, stream, ln_s.as<float2>()));
    p.residual = nullptr; p.ln_src = residual; p.ld_ln = N; p.ln_stats = ln_s.as<float2>();
    p.ln_gamma = ln_g.as<float>(); p.ln_beta = ln_b.as<float>();
  }
  p.act = act; p.rowmap = ROWMAP_IDENTITY;
  p.out_f32 = C; p.ld_f32 = N;
  p.nsplit_out = precision;
  if (pair) {
    CK(configure_linear2_kernels());
    DevBuf dbg, o_hi, o_lo;
    CUtensorMap mo_hi, mo_lo;
    const bool want_dbg = getenv("CMDI_TEST_DBG") != nullptr;
    if (const char* d = getenv("CMDI_DEBUG")) p.debug = atoi(d);
    if (want_dbg) {
      CK(dbg.alloc(148 * 16 * 8));
      p.dbg_cycles = dbg.as<long long>();
      CK(o_hi.alloc((size_t)Mp * Np * 2));
      CK(o_lo.alloc((size_t)Mp * Np * 2));
      if (make_tmap_bf16_2d(&mo_hi, o_hi.p, Mp, Np, Np, 64, 32)) return 1;
      if (make_tmap_bf16_2d(&mo_lo, o_lo.p, Mp, Np, Np, 64, 32)) return 1;
      stm.hi = &mo_hi;
      stm.lo = &mo_lo;
      p.out_hi = o_hi.as<__nv_bfloat16>();  // realistic stores: bf16 planes like the engine's QKV / FFN1
      p.out_lo = o_lo.as<__nv_bfloat16>();
      p.ld_bf = Np;
      if (getenv("CMDI_TEST_NOF32")) p.out_f32 = nullptr;
      CK(launch_linear_pair(ma_hi, ma_lo, mw_hi, mw_lo, p, block_n, num_sms_of_current_device(), stream, stp, f16));
    }
    CK(launch_linear_pair(ma_hi, ma_lo, mw_hi, mw_lo, p, block_n, num_sms_of_current_device(), stream, stp, f16));
    if (want_dbg) {
      std::vector<long long> h(148 * 16);
      CK(cudaStreamSynchronize(stream));
      CK(cudaMemcpy(h.data(), dbg.p, h.size() * 8, cudaMemcpyDeviceToHost));
      double acc[16] = {0};
      int n_lead = 0, n_all = 0;
      for (int b = 0; b < 148; ++b) {
        if (h[b * 16 + 4] == 0) continue;
        ++n_all;
        for (int k = 4; k < 8; ++k) acc[k] += (double)h[b * 16 + k];
        if (h[b * 16 + 0]) { ++n_lead; for (int k = 0; k < 3; ++k) acc[k] += (double)h[b * 16 + k]; }
      }
      printf("dbg cycles (mean per CTA): mma total=%.0f wait_tmem_empty=%.0f wait_full=%.0f | epi total=%.0f wait_tmem_full=%.0f work=%.0f arrive=%.0f (leaders %d, ctas %d)\n",
             acc[0] / n_lead, acc[1] / n_lead, acc[2] / n_lead, acc[4] / n_all, acc[5] / n_all, acc[6] / n_all, acc[7] / n_all, n_lead, n_all);
      fflush(stdout);
    }
  }
  CK(cudaStreamSynchronize(stream));  // staging buffers are freed on return
  return 0;
}

extern "C" int cmdi_test_layernorm(const float* v, const float* gamma, const float* beta, float* out, int rows,
                                   void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  CK(launch_layernorm512(v, gamma, beta, 1e-5f, rows, out, nullptr, nullptr, stream));
  return 0;
}

namespace {
int test_attention(const float* qkv, float* O, int num_seqs, int S, int H, int precision, int nsplit_out, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (S > kAttnKeyPad) {
    set_last_error("cmdi_test_attention: S=%d exceeds %d", S, kAttnKeyPad);
    return 1;
  }
  const int rows = num_seqs * S;
  const int rows_p = round_up(rows, 128) + 256;  // tiles of the last sequence read past its end
  const int ld = 3 * H * 128, ldo = H * 128;
  DevBuf q_hi, q_lo, o_hi, o_lo;
  CK(q_hi.alloc((size_t)rows_p * ld * 2));
  CK(q_lo.alloc((size_t)rows_p * ld * 2));
  CK(o_hi.alloc((size_t)rows_p * ldo * 2));
  CK(o_lo.alloc((size_t)rows_p * ldo * 2));
  CK(launch_split_planes(qkv, rows, ld, ld, q_hi.as<__nv_bfloat16>(), q_lo.as<__nv_bfloat16>(), ld, stream));
  CUtensorMap mq_hi, mq_lo, mkv_hi, mkv_lo;
  if (make_tmap_bf16_2d(&mq_hi, q_hi.p, rows_p, ld, ld, 64, 128)) return 1;
  if (make_tmap_bf16_2d(&mq_lo, q_lo.p, rows_p, ld, ld, 64, 128)) return 1;
  if (make_tmap_bf16_2d(&mkv_hi, q_hi.p, rows_p, ld, ld, 64, kAttnKeyPad)) return 1;
  if (make_tmap_bf16_2d(&mkv_lo, q_lo.p, rows_p, ld, ld, 64, kAttnKeyPad)) return 1;
  CUtensorMap mkh_hi, mkh_lo;
  if (make_tmap_bf16_2d(&mkh_hi, q_hi.p, rows_p, ld, ld, 64, kAttnKeyPad / 2)) return 1;
  if (make_tmap_bf16_2d(&mkh_lo, q_lo.p, rows_p, ld, ld, 64, kAttnKeyPad / 2)) return 1;
  CUtensorMap mo_hi, mo_lo;
  if (make_tmap_bf16_2d(&mo_hi, o_hi.p, rows_p, ldo, ldo, 64, 32)) return 1;
  if (make_tmap_bf16_2d(&mo_lo, o_lo.p, rows_p, ldo, ldo, 64, 32)) return 1;
  CK(configure_attention_kernel());
  const AttnMaps am{&mq_hi, &mq_lo, &mkh_hi, &mkh_lo, &mkv_hi, &mkv_lo, &mo_hi, &mo_lo};
  AttnParams p{};
  p.num_seqs = num_seqs; p.seq_len = S; p.num_heads = H; p.nsplit = precision; p.nsplit_out = nsplit_out;
  p.out_hi = o_hi.as<__nv_bfloat16>(); p.out_lo = o_lo.as<__nv_bfloat16>(); p.ld_out = ldo;
  if (const char* g = getenv("CMDI_ATTN_SPLIT")) p.trunc_split = strcmp(g, "trunc") == 0;
  DevBuf adbg;
  const int nctas = ((S + 127) / 128) * H * num_seqs;
  if (getenv("CMDI_TEST_DBG")) {
    CK(adbg.alloc((size_t)nctas * 16 * 8));
    CK(cudaMemset(adbg.p, 0, (size_t)nctas * 16 * 8));
    p.dbg_cycles = adbg.as<long long>();
    CK(launch_attention(am, p, stream));
  }
  CK(launch_attention(am, p, stream));
  if (p.dbg_cycles) {
    std::vector<long long> h((size_t)nctas * 16);
    CK(cudaStreamSynchronize(stream));
    CK(cudaMemcpy(h.data(), adbg.p, h.size() * 8, cudaMemcpyDeviceToHost));
    double a[16] = {0};
    {
      // per-CTA-pair sums over its items; slot 7 = item count
      double items = 0;
      for (int c = 0; c < nctas; ++c) items += (double)h[(size_t)c * 16 + 7];
      for (int c = 0; c < nctas; ++c) for (int k = 0; k < 12; ++k) a[k] += (double)h[(size_t)c * 16 + k] / items;
      printf("attention dbg cycles (mean per item): MMA thread wait_q=%.0f wait_k=%.0f S-issue=%.0f wait_P=%.0f wait_V=%.0f PV-issue=%.0f wait_PV_retired=%.0f | "
             "softmax warp: wait_S=%.0f softmax=%.0f last_wait_O=%.0f output=%.0f (items %.0f)\n",
             a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[8], a[9], a[10], a[11], items);
      double pro = 0, tot_max = 0, n = 0;
      for (int c = 0; c < nctas; ++c) {
        if (h[(size_t)c * 16 + 7] == 0) continue;
        n += 1;
        pro += (double)h[(size_t)c * 16 + 12];
        if ((double)h[(size_t)c * 16 + 13] > tot_max) tot_max = (double)h[(size_t)c * 16 + 13];
      }
      printf("attention dbg: CTA pairs=%.0f prologue=%.0f cycles, longest pair (MMA thread) %.0f cycles\n", n, pro / n, tot_max);
      fflush(stdout);
      p.dbg_cycles = nullptr;
    }
  }
  // O = hi + lo (fp32) for the test; at nsplit_out = 1 the lo plane is still the zeros it was allocated with
  {
    std::vector<uint16_t> hh((size_t)rows * ldo), hl((size_t)rows * ldo);
    std::vector<float> ho((size_t)rows * ldo);
    CK(cudaStreamSynchronize(stream));
    CK(cudaMemcpy(hh.data(), o_hi.p, hh.size() * 2, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hl.data(), o_lo.p, hl.size() * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < ho.size(); ++i) {
      uint32_t a = (uint32_t)hh[i] << 16, b = (uint32_t)hl[i] << 16;
      float fa, fb;
      memcpy(&fa, &a, 4);
      memcpy(&fb, &b, 4);
      ho[i] = fa + fb;
    }
    CK(cudaMemcpy(O, ho.data(), ho.size() * 4, cudaMemcpyHostToDevice));
  }
  return 0;
}

}  // namespace

extern "C" int cmdi_test_attention(const float* qkv, float* O, int num_seqs, int S, int H, int precision, void* stream) {
  return test_attention(qkv, O, num_seqs, S, H, precision, 3, stream);
}
extern "C" int cmdi_test_attention_hi(const float* qkv, float* O, int num_seqs, int S, int H, int precision, void* stream) {
  return test_attention(qkv, O, num_seqs, S, H, precision, 1, stream);
}

extern "C" int cmdi_test_normal_aten(float* out, long long numel, unsigned long long seed, unsigned long long offset,
                                     unsigned int threads, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (threads == 0 || (offset & 3) || numel < 0) {
    set_last_error("cmdi_test_normal_aten: threads must be > 0 and offset a multiple of 4");
    return 1;
  }
  CK(launch_fill_normal_aten(out, (size_t)numel, seed, offset, threads, stream));
  return 0;
}

extern "C" int cmdi_test_normal(float* out, int B, long long per_sample, unsigned long long seed, unsigned long long stream_id,
                                unsigned long long sample_offset, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  CK(launch_fill_normal_ref(out, B, (size_t)per_sample, seed, stream_id, sample_offset, stream));
  return 0;
}

extern "C" int cmdi_test_layernorm_bwd(const float* dy, const float* v, const float* gamma, float* dv, int rows, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  DevBuf hi;
  CK(hi.alloc((size_t)rows * 512 * 2));
  CK(launch_layernorm512_bwd(dy, v, gamma, 1e-5f, rows, dv, hi.as<__nv_bfloat16>(), nullptr, stream));
  CK(cudaStreamSynchronize(stream));
  return 0;
}

// qkv: fp32 [num_seqs*S, 3*H*128], dO: fp32 [num_seqs*S, H*128] -> dqkv fp32 (hi + lo of the kernel's planes)
extern "C" int cmdi_test_attention_bwd_at(const float* qkv, const float* dO, float* dqkv, int num_seqs, int S, int H, int precision,
                                          void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int rows = num_seqs * S, ld = 3 * H * 128, ldo = H * 128;
  const int rows_p = round_up(rows, 128) + 256;  // tiles of the last sequence read past its end
  DevBuf q_hi, q_lo, d_hi, d_lo, g_hi, g_lo, stats;
  CK(q_hi.alloc((size_t)rows_p * ld * 2)); CK(q_lo.alloc((size_t)rows_p * ld * 2));
  CK(d_hi.alloc((size_t)rows_p * ldo * 2)); CK(d_lo.alloc((size_t)rows_p * ldo * 2));
  CK(g_hi.alloc((size_t)rows_p * ld * 2)); CK(g_lo.alloc((size_t)rows_p * ld * 2));
  CK(stats.alloc((size_t)rows_p * H * sizeof(float2)));
  CK(cudaMemsetAsync(q_hi.p, 0, (size_t)rows_p * ld * 2, stream)); CK(cudaMemsetAsync(q_lo.p, 0, (size_t)rows_p * ld * 2, stream));
  CK(cudaMemsetAsync(d_hi.p, 0, (size_t)rows_p * ldo * 2, stream)); CK(cudaMemsetAsync(d_lo.p, 0, (size_t)rows_p * ldo * 2, stream));
  CK(launch_split_planes(qkv, rows, ld, ld, q_hi.as<__nv_bfloat16>(), q_lo.as<__nv_bfloat16>(), ld, stream));
  CK(launch_split_planes(dO, rows, ldo, ldo, d_hi.as<__nv_bfloat16>(), d_lo.as<__nv_bfloat16>(), ldo, stream));
  AttnBwdParams p{};
  p.num_seqs = num_seqs; p.seq_len = S; p.num_heads = H; p.qkv_hi = q_hi.as<__nv_bfloat16>(); p.qkv_lo = q_lo.as<__nv_bfloat16>();
  p.do_hi = d_hi.as<__nv_bfloat16>(); p.do_lo = d_lo.as<__nv_bfloat16>(); p.ld_do = ldo;
  p.dqkv_hi = g_hi.as<__nv_bfloat16>(); p.dqkv_lo = g_lo.as<__nv_bfloat16>();
  p.ld_dqkv = ld; p.nsplit = precision; p.stats = stats.as<float2>();
  if (!getenv("CMDI_TEST_ATTN_BWD_SIMT")) {
    CUtensorMap qt_hi, qt_lo, qf_hi, qf_lo, dt_hi, dt_lo, df_hi, df_lo, o_hi, o_lo;
    if (make_tmap_bf16_2d(&qt_hi, q_hi.p, rows_p, ld, ld, 64, 128)) return 1;
    if (make_tmap_bf16_2d(&qt_lo, q_lo.p, rows_p, ld, ld, 64, 128)) return 1;
    if (make_tmap_bf16_2d(&qf_hi, q_hi.p, rows_p, ld, ld, 64, kAttnKeyPad)) return 1;
    if (make_tmap_bf16_2d(&qf_lo, q_lo.p, rows_p, ld, ld, 64, kAttnKeyPad)) return 1;
    if (make_tmap_bf16_2d(&dt_hi, d_hi.p, rows_p, ldo, ldo, 64, 128)) return 1;
    if (make_tmap_bf16_2d(&dt_lo, d_lo.p, rows_p, ldo, ldo, 64, 128)) return 1;
    if (make_tmap_bf16_2d(&df_hi, d_hi.p, rows_p, ldo, ldo, 64, kAttnKeyPad)) return 1;
    if (make_tmap_bf16_2d(&df_lo, d_lo.p, rows_p, ldo, ldo, 64, kAttnKeyPad)) return 1;
    if (make_tmap_bf16_2d(&o_hi, g_hi.p, rows_p, ld, ld, 64, 32)) return 1;
    if (make_tmap_bf16_2d(&o_lo, g_lo.p, rows_p, ld, ld, 64, 32)) return 1;
    CK(configure_attention_bwd_tc_kernel());
    AttnBwdTcMaps bm{&qt_hi, &qt_lo, &qf_hi, &qf_lo, &dt_hi, &dt_lo, &df_hi, &df_lo, &o_hi, &o_lo};
    CK(launch_attention_bwd_tc(bm, p, stream));
  } else {
    CK(configure_attention_bwd_kernel());
    CK(launch_attention_bwd(p, stream));
  }
  CK(cudaStreamSynchronize(stream));
  std::vector<uint16_t> hh((size_t)rows * ld), hl((size_t)rows * ld);
  std::vector<float> ho((size_t)rows * ld);
  CK(cudaMemcpy(hh.data(), g_hi.p, hh.size() * 2, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(hl.data(), g_lo.p, hl.size() * 2, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < ho.size(); ++i) {
    uint32_t a = (uint32_t)hh[i] << 16, b = (uint32_t)hl[i] << 16;
    float fa, fb;
    memcpy(&fa, &a, 4);
    memcpy(&fb, &b, 4);
    ho[i] = fa + fb;
  }
  CK(cudaMemcpy(dqkv, ho.data(), ho.size() * 4, cudaMemcpyHostToDevice));
  return 0;
}

extern "C" int cmdi_test_attention_bwd(const float* qkv, const float* dO, float* dqkv, int num_seqs, int S, int H, void* stream) {
  return cmdi_test_attention_bwd_at(qkv, dO, dqkv, num_seqs, S, H, 3, stream);
}

// The phase list mirrors get_chain_tables (engine.cu) for a layer l with 0 < l < layers - 1; what the engine keeps in
// xseq_p / x1_p / ffh_p / qkv_p / stats1 / stats2 / chain_ctr are local buffers here.
extern "C" int cmdi_test_chain_layer(const float* const* in, float* const* out, int M, int precision, float stale_lo,
                                     void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M < 1 || (precision != 1 && precision != 3)) {
    set_last_error("cmdi_test_chain_layer: M=%d precision=%d", M, precision);
    return 1;
  }
  enum { ATTN, V2P, G2P, BE2P, WO, BO, G1, BE1, W1, B1, W2, B2, G2, BE2, WQKV, BQKV };
  constexpr int kD = 512, kFF = 1024, kBn = 256;
  const int Mp = round_up(M, 256), m_pairs = Mp / 256;
  struct Pl {
    DevBuf hi, lo;
    int ld = 0;
    CUtensorMap a_hi, a_lo, st_hi, st_lo;
  };
  uint32_t stale_bits;
  memcpy(&stale_bits, &stale_lo, 4);
  const std::vector<uint16_t> stale((size_t)Mp * 3 * kD, (uint16_t)(stale_bits >> 16));
  // rows x ld planes; box_rows: A operand {64, 128} or W operand {64, kBn / 2}; st_cols: 32 (residual phases) or 64 (wide phases)
  auto planes = [&](Pl& pl, int rows, int ld, int box_rows, int st_cols, bool prefill) -> int {
    pl.ld = ld;
    CK(pl.hi.alloc((size_t)rows * ld * 2));
    CK(pl.lo.alloc((size_t)rows * ld * 2));
    if (prefill) CK(cudaMemcpy(pl.lo.p, stale.data(), (size_t)rows * ld * 2, cudaMemcpyHostToDevice));
    if (make_tmap_bf16_2d(&pl.a_hi, pl.hi.p, rows, ld, ld, 64, box_rows)) return 1;
    if (make_tmap_bf16_2d(&pl.a_lo, pl.lo.p, rows, ld, ld, 64, box_rows)) return 1;
    if (make_tmap_bf16_2d(&pl.st_hi, pl.hi.p, rows, ld, ld, st_cols, 32)) return 1;
    if (make_tmap_bf16_2d(&pl.st_lo, pl.lo.p, rows, ld, ld, st_cols, 32)) return 1;
    return 0;
  };
  Pl attn, xseq, x1, ffh, qkv, wo, w1f, w2, wqf;
  if (planes(attn, Mp, kD, 128, 32, false) || planes(xseq, Mp, kD, 128, 32, false) || planes(x1, Mp, kD, 128, 32, true) ||
      planes(ffh, Mp, kFF, 128, 64, true) || planes(qkv, Mp, 3 * kD, 128, 64, true) || planes(wo, kD, kD, kBn / 2, 32, false) ||
      planes(w1f, kFF, kD, kBn / 2, 32, false) || planes(w2, kD, kFF, kBn / 2, 32, false) || planes(wqf, 3 * kD, kD, kBn / 2, 32, false))
    return 1;
  auto split = [&](Pl& pl, const float* src, int rows) {
    return launch_split_planes(src, rows, pl.ld, pl.ld, pl.hi.as<__nv_bfloat16>(), pl.lo.as<__nv_bfloat16>(), pl.ld, stream);
  };
  CK(split(attn, in[ATTN], M));
  CK(split(xseq, in[V2P], M));  // what the previous layer's FFN2 phase leaves in xseq_p
  CK(split(wo, in[WO], kD));
  CK(split(w2, in[W2], kD));
  DevBuf folded, c1, d1, cq, dq, beta_bo, beta_b2, stats1, stats2, ctr, phases;
  CK(folded.alloc((size_t)3 * kD * kD * 4));
  CK(c1.alloc(kFF * 4)); CK(d1.alloc(kFF * 4)); CK(cq.alloc(3 * kD * 4)); CK(dq.alloc(3 * kD * 4));
  CK(beta_bo.alloc(kD * 4)); CK(beta_b2.alloc(kD * 4));
  CK(launch_fold_ln(in[W1], kFF, kD, in[G1], in[BE1], in[B1], folded.as<float>(), c1.as<float>(), d1.as<float>(), stream));
  CK(split(w1f, folded.as<float>(), kFF));
  CK(launch_fold_ln(in[WQKV], 3 * kD, kD, in[G2], in[BE2], in[BQKV], folded.as<float>(), cq.as<float>(), dq.as<float>(), stream));
  CK(split(wqf, folded.as<float>(), 3 * kD));
  CK(launch_add_vectors(in[BE2P], in[BO], beta_bo.as<float>(), kD, stream));
  CK(launch_add_vectors(in[BE1], in[B2], beta_b2.as<float>(), kD, stream));
  // partial statistics of v2_prev as its producer publishes them (LinearParams::stats_out): (mean, sum of squared
  // deviations) of each 128-column quarter in the first 4 of a row's 16 slots
  CK(stats1.alloc((size_t)Mp * 16 * sizeof(float2)));
  CK(stats2.alloc((size_t)Mp * 16 * sizeof(float2)));
  {
    std::vector<float> v((size_t)M * kD);
    std::vector<float2> st((size_t)M * 16, make_float2(0.f, 0.f));
    CK(cudaStreamSynchronize(stream));
    CK(cudaMemcpy(v.data(), in[V2P], v.size() * 4, cudaMemcpyDeviceToHost));
    for (int r = 0; r < M; ++r)
      for (int q = 0; q < 4; ++q) {
        const float* x = &v[(size_t)r * kD + q * 128];
        double mean = 0, m2 = 0;
        for (int j = 0; j < 128; ++j) mean += x[j];
        mean /= 128;
        for (int j = 0; j < 128; ++j) m2 += (x[j] - mean) * (x[j] - mean);
        st[(size_t)r * 16 + q] = make_float2((float)mean, (float)m2);
      }
    CK(cudaMemcpy(stats2.p, st.data(), st.size() * sizeof(float2), cudaMemcpyHostToDevice));
  }
  CK(ctr.alloc((size_t)3 * m_pairs * sizeof(int)));
  ChainPhaseDesc ph[kMaxChainPhases];
  auto base = [&](ChainPhaseDesc& d, const Pl& a, const Pl& w, int N, int K) {
    memset(&d, 0, sizeof(d));
    d.a_hi = a.a_hi; d.a_lo = a.a_lo; d.w_hi = w.a_hi; d.w_lo = w.a_lo;
    d.o_hi = a.a_hi; d.o_lo = a.a_hi; d.o_f32 = a.a_hi;  // placeholders unless set below
    ChainPhaseInfo& pi = d.info;
    pi.p.M = M; pi.p.N = N; pi.p.K = K; pi.p.nsplit = precision; pi.p.nsplit_out = precision; pi.p.rowmap = ROWMAP_IDENTITY;
    pi.p.tma_store = 1;
    pi.block_n = kBn; pi.num_m_pairs = m_pairs; pi.num_n_blocks = (N + kBn - 1) / kBn; pi.num_k_blocks = (K + 63) / 64;
    pi.publish_now = 1;
  };
  int* const c = ctr.as<int>();
  // a phase whose output planes are a later phase's residual source (v = hi + lo) writes both planes at either precision
  auto residual_phase = [&](ChainPhaseDesc& d, Pl& src, const float* gamma, const float* beta, const float2* partials, Pl& dst,
                            float2* stats_out) {
    LinearParams& p = d.info.p;
    p.ld_ln = kD; p.ln_partials = partials; p.ln_gamma = gamma; p.ln_beta = beta;
    p.ln_src_hi = src.hi.as<__nv_bfloat16>(); p.ln_src_lo = src.lo.as<__nv_bfloat16>();
    p.out_hi = dst.hi.as<__nv_bfloat16>(); p.out_lo = dst.lo.as<__nv_bfloat16>(); p.ld_bf = kD; p.nsplit_out = 3;
    p.stats_out = stats_out;
    d.o_hi = dst.st_hi; d.o_lo = dst.st_lo;
  };
  auto folded_phase = [&](ChainPhaseDesc& d, const float* cvec, const float* dvec, const float2* stats, Pl& dst) {
    LinearParams& p = d.info.p;
    p.bias = dvec; p.fold_c = cvec; p.fold_stats = stats;
    p.out_hi = dst.hi.as<__nv_bfloat16>(); p.out_lo = dst.lo.as<__nv_bfloat16>(); p.ld_bf = dst.ld;
    d.info.wide = 1; d.o_hi = dst.st_hi; d.o_lo = dst.st_lo;
  };
  base(ph[0], attn, wo, kD, kD);
  residual_phase(ph[0], xseq, in[G2P], beta_bo.as<float>(), stats2.as<float2>(), x1, stats1.as<float2>());
  ph[0].info.done_ctr = c;
  base(ph[1], x1, w1f, kFF, kD);
  folded_phase(ph[1], c1.as<float>(), d1.as<float>(), stats1.as<float2>(), ffh);
  ph[1].info.p.act = 1;
  ph[1].info.wait_ctr = c; ph[1].info.wait_target = ph[0].info.num_n_blocks * 2; ph[1].info.done_ctr = c + m_pairs;
  base(ph[2], ffh, w2, kD, kFF);
  residual_phase(ph[2], x1, in[G1], beta_b2.as<float>(), stats1.as<float2>(), xseq, stats2.as<float2>());
  ph[2].info.wait_ctr = c + m_pairs; ph[2].info.wait_target = ph[1].info.num_n_blocks * 2; ph[2].info.done_ctr = c + 2 * m_pairs;
  base(ph[3], xseq, wqf, 3 * kD, kD);
  folded_phase(ph[3], cq.as<float>(), dq.as<float>(), stats2.as<float2>(), qkv);
  ph[3].info.wait_ctr = c + 2 * m_pairs; ph[3].info.wait_target = ph[2].info.num_n_blocks * 2;
  int tiles = 0;
  for (int i = 0; i < kMaxChainPhases; ++i) {
    ph[i].info.tile_begin = tiles;
    tiles += ph[i].info.num_m_pairs * ph[i].info.num_n_blocks;
    ph[i].info.tile_end = tiles;
  }
  CK(phases.alloc(sizeof(ph)));
  CK(cudaMemcpy(phases.p, ph, sizeof(ph), cudaMemcpyHostToDevice));
  CK(configure_linear_chain_kernel());
  // ph[2] overwrites, row pair by row pair, the planes and statistics ph[0] read v2_prev from, as in the engine (xseq_p,
  // stats2): a row pair's ph[2] tiles wait for its ph[1] tiles, and those for all of its ph[0] tiles
  CK(launch_linear_chain(phases.as<ChainPhaseDesc>(), kMaxChainPhases, tiles, precision, num_sms_of_current_device(), stream));
  CK(cudaStreamSynchronize(stream));
  auto read_back = [&](const Pl& pl, bool with_lo, float* dst) -> int {
    const size_t n = (size_t)M * pl.ld;
    std::vector<uint16_t> hh(n), hl(n);
    std::vector<float> ho(n);
    CK(cudaMemcpy(hh.data(), pl.hi.p, n * 2, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hl.data(), pl.lo.p, n * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; ++i) {
      const uint32_t a = (uint32_t)hh[i] << 16, b = (uint32_t)hl[i] << 16;
      float fa, fb;
      memcpy(&fa, &a, 4);
      memcpy(&fb, &b, 4);
      ho[i] = with_lo ? fa + fb : fa;
    }
    CK(cudaMemcpy(dst, ho.data(), n * 4, cudaMemcpyHostToDevice));
    return 0;
  };
  if (read_back(x1, true, out[0]) || read_back(ffh, precision == 3, out[1]) || read_back(xseq, true, out[2]) ||
      read_back(qkv, precision == 3, out[3]))
    return 1;
  return 0;
}
