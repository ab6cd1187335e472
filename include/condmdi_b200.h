/*
 * condmdi_b200 -- C ABI of the B200-native CondMDI sampling engine (libcondmdi_b200.so).
 *
 * This is the boundary a maintainer of setarehc/diffusion-motion-inbetweening binds to (ctypes stub in
 * INTEGRATION.md).  The reference has no FFI of its own: its "operator API" for this path is three
 * Python call signatures.  Each entry point below names the reference interface it replaces
 * (paths relative to the reference repository root).
 *
 *   cmdi_engine_create      model hyper-parameters  <- utils/model_util.py:40-119 (get_model_args), model/mdm.py:11-165
 *   cmdi_load_weights       MDM.state_dict()        <- utils/model_util.py:168-182 (load_saved_model), model/mdm.py:97-165
 *   cmdi_set_schedule       diffusion tables        <- diffusion/gaussian_diffusion.py:183-217, diffusion/respace.py:74-91
 *   cmdi_model_forward      one denoiser pass       <- model/mdm.py:239-306 (MDM.forward),
 *                                                      model/cfg_sampler.py:25-35 (ClassifierFreeSampleModel.forward)
 *   cmdi_sample             the sampling loop       <- diffusion/gaussian_diffusion.py:1149-1297 (p_sample_loop[_progressive]),
 *                                                      :1454-1587 (ddim_sample_loop[_progressive]),
 *                                                      :1589-1804 (plms_sample_loop[_progressive]),
 *                                                      :1418-1452 (ddim_reverse_sample, looped),
 *                                                      :352-534 (p_mean_variance), :656-713 (p_sample), :1358-1416 (ddim_sample_with_grad)
 *
 * Conventions
 *   - All tensors are plain pointers + sizes; no framework types cross this boundary.
 *   - "ref layout" is the reference's (B, njoints, nfeats=1, nframes) contiguous fp32 layout, frames fastest.
 *   - Pointers are DEVICE pointers unless the call's `host_buffers` flag says otherwise.
 *   - Work is enqueued on the caller's CUDA stream (cudaStream_t passed as void*); calls are
 *     stream-ordered and never call cudaDeviceSynchronize (host_buffers = 1 synchronises the stream once
 *     at the end so the host output is valid on return, like `sample.cpu()` in the reference scripts).
 *   - Every function returns 0 on success, non-zero on error; cmdi_last_error() describes the failure.
 *     There is no CPU fallback: a missing GPU / wrong architecture is an error.
 */
#ifndef CONDMDI_B200_H_
#define CONDMDI_B200_H_

#include <stdint.h>

#if defined(__GNUC__)
#define CMDI_API __attribute__((visibility("default")))
#else
#define CMDI_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cmdi_engine cmdi_engine;

/* numerics of the tensor-core contractions */
enum {
  CMDI_PRECISION_BF16X3 = 3, /* bf16 hi/lo operand split, 3 MMAs per product, fp32 accumulate: meets the fp32 parity gate */
  CMDI_PRECISION_BF16 = 1,   /* single bf16 MMA, fp32 accumulate: "fast" mode, does NOT meet rtol 1e-3 / atol 1e-4 */
  CMDI_PRECISION_FP16 = 2    /* "autocast", MDM_UNET only: what torch.autocast("cuda", float16) computes -- fp16 conv / linear
                                operands and outputs (one MMA, fp32 accumulate), GroupNorm / AdaGN / Mish / residual sums in
                                fp32 -- the arithmetic of checkpoints trained and sampled with use_fp16 */
};

/* PLMS: pseudo linear multistep (plms_sample_loop, gaussian_diffusion.py:1589-1804): deterministic, no per-step noise */
/* DDIM_REVERSE: DDIM inversion (ddim_reverse_sample, gaussian_diffusion.py:1418-1452, eta = 0), the deterministic
   encoder x_t -> x_{t+1}.  The loop ascends from t0 = skip_timesteps (the iterations already done, counted upwards);
   x_T is the start state (e.g. x_0) and is required; num_steps as for the other samplers (0 = up to t = T - 1).
   eta must be 0 and noise_tape, init_image, dump_xstart, plms_order and plms_old_eps_out unset: the call fails
   naming the field otherwise.  pred_xstart_out receives the last step's x0. */
/* DPM_SOLVER: DPM-Solver++ multistep (Lu et al. 2022; data prediction, solver type `dpmsolver`) on the spaced steps,
   orders 1..3 (dpm_order), one denoiser pass per step.  Deterministic after x_T; the step at s uses order
   min(dpm_order, iterations since the history started + 1, s + 1), and the last step returns x0 as DDIM's does.
   skip_timesteps / init_image / resume as for DDIM (init_image only on a call that starts a history); eta must be 0 and
   noise_tape, dump_xstart, plms_order and plms_old_eps_out unset: the call fails naming the field otherwise. */
/* UNIPC: UniPC (Zhao et al. 2023; multistep, data prediction) on the spaced steps, orders 1..3 (unipc_order), variant
   bh1 or bh2 (unipc_variant), with or without the UniC corrector (unipc_corrector), one denoiser pass per step.  The
   pass at s evaluates the uncorrected state; its x0 then corrects the state of s (with the order of the predictor
   step into s) and predicts s - 1 with order min(unipc_order, iterations since the history started + 1, s + 1).  The
   corrected state stays on the device; the last step returns x0 as DDIM's does.  skip_timesteps / init_image / resume
   as for DPM_SOLVER; eta must be 0 and noise_tape, dump_xstart, plms_order, plms_old_eps_out and dpm_order unset: the
   call fails naming the field otherwise. */
/* DPM_SOLVER_SDE: SDE-DPM-Solver++ (Lu et al. 2022; the SDE multistep solver in data prediction, midpoint form) on the
   spaced steps, orders 1..2 (dpm_order), one denoiser pass per step.  Stochastic like DDPM, with DDPM's noise contract:
   one draw per step including the last (tape, CMDI_RNG_TORCH stream or engine generator, numbered from the call's
   first step), whose value the last step does not use.  Order 1 is the DDPM posterior step.  The step at s uses order
   min(dpm_order, iterations since the history started + 1, s + 1); the last step returns x0.  skip_timesteps /
   init_image / resume as for DPM_SOLVER; eta must be 0 and dump_xstart, plms_order, plms_old_eps_out and the unipc_*
   fields unset: the call fails naming the field otherwise. */
/* REPAINT: RePaint resampling (Lugmayr et al. 2022, "time travel") around DDPM, for in-betweening with imputation.  The
   walk starts at position t0 = T - 1 - skip_timesteps (position p: the state step p takes as input) and is a sequence
   of +-1 ops: a denoise op at p is p_sample at step p, exactly DDPM's step (CFG, keyframe input, imputation and
   reconstruction guidance decided by p); an undo op into p is one forward step of the spaced chain,
   x <- fp32(sqrt(1 - beta_p)) x + fp32(sqrt(beta_p)) z.  The walk descends; the first time it arrives at a jump point t
   (t % repaint_jump_length == 0, t + repaint_jump_length <= t0) it goes up repaint_jump_length positions by undo ops and
   comes back down by denoise ops, repaint_jump_n_sample - 1 times.  With repaint_jump_n_sample = 1 it is DDPM.  Noise:
   one draw per op in walk order (tape slice, CMDI_RNG_TORCH stream, numbered from the call's first op); the engine
   generator keys the first denoise op at p by DDPM's stream for p and every other op by its index in the walk.
   num_steps counts denoise ops; the undo ops before each run in the same call.  resume = 1 continues the running walk
   (same jump fields and batch) with skip_timesteps = T - 1 - the position the walk has reached.  eta must be 0 and
   dump_xstart, plms_order, plms_old_eps_out, dpm_order and the unipc_* fields unset: the call fails naming the field
   otherwise. */
enum { CMDI_SAMPLER_DDPM = 0, CMDI_SAMPLER_DDIM = 1, CMDI_SAMPLER_PLMS = 2, CMDI_SAMPLER_DDIM_REVERSE = 3,
       CMDI_SAMPLER_DPM_SOLVER = 4, CMDI_SAMPLER_UNIPC = 5, CMDI_SAMPLER_DPM_SOLVER_SDE = 6, CMDI_SAMPLER_REPAINT = 7 };
enum { CMDI_UNIPC_BH1 = 1, CMDI_UNIPC_BH2 = 2 };  /* unipc_variant: B(h) = h or e^h - 1 */
enum { CMDI_ARCH_TRANS_ENC = 0, CMDI_ARCH_UNET = 1 };
enum { CMDI_RNG_ENGINE = 0, CMDI_RNG_TORCH = 1 };

typedef struct {
  int32_t njoints;     /* 263 (input_feats = njoints * nfeats, nfeats == 1)                      mdm.py:64 */
  int32_t nframes;     /* 196                                                                    synthesize.py:23-29 */
  int32_t latent_dim;  /* 512 (only value supported)                                             parser_util.py:37-49 */
  int32_t ff_size;     /* 1024                                                                   */
  int32_t num_layers;  /* 8                                                                      */
  int32_t num_heads;   /* 4  (head dim must be 128)                                              model_util.py:98 */
  int32_t max_batch;   /* largest B a call may use (buffers are sized for 2*max_batch sequences) */
  int32_t has_text;    /* cond_mode contains 'text': embed_text weights are expected             mdm.py:137-139 */
  int32_t precision;   /* CMDI_PRECISION_* */
  /* denoiser architecture: the MDM transformer encoder above, or MDM_UNET (model/mdm_unet.py, arch='unet', AdaGN) */
  int32_t arch;                  /* CMDI_ARCH_TRANS_ENC / CMDI_ARCH_UNET                          model_util.py:26-35 */
  int32_t unet_levels;           /* len(dim_mults), 2..4                                           configs/model.py:28-67 */
  int32_t unet_dim_mults[4];     /* channels of level l = latent_dim * unet_dim_mults[l] (equal across levels) */
  int32_t keyframe_conditioned;  /* the input is cat([obs_x0*M + x*~M, M]) (2 * njoints channels)  mdm_unet.py:636-643, :778-783 */
} cmdi_model_cfg;

typedef struct {
  const char* name;  /* state-dict key, e.g. "seqTransEncoder.layers.0.self_attn.in_proj_weight" */
  const float* data; /* fp32, contiguous */
  int64_t numel;
  int32_t on_host;   /* 1: host pointer, 0: device pointer */
} cmdi_tensor_desc;

/* One denoiser evaluation: out = model(x, timesteps, y).  With cfg != 0 the cond and uncond passes run as one
 * batch-doubled pass and out = out_uncond + text_scale[b] * (out_cond - out_uncond). */
typedef struct {
  int32_t batch;
  const float* x;             /* ref layout (B, 263, 1, 196) */
  int32_t timestep;           /* ORIGINAL-process timestep (already mapped through timestep_map); same for all b */
  const float* cond_emb;      /* (B, 512) text embedding (output of encode_text) or NULL for no_cond */
  int32_t uncond;             /* y['uncond']: mask the text embedding to zeros (mdm.py:188-191) */
  int32_t cfg;                /* ClassifierFreeSampleModel.forward */
  const float* text_scale;    /* (B,) when cfg */
  int32_t host_buffers;
  const float* obs_x0;        /* ref layout observed keyframes and ... */
  const uint8_t* obs_mask;    /* ... their bool mask: the obs_x0 / obs_mask arguments of MDM_UNET.forward (mdm_unet.py:765);
                                 NULL for the transformer (which ignores them, SURVEY 8b note 2) */
} cmdi_forward_args;

typedef struct {
  int32_t batch;
  int32_t sampler;              /* CMDI_SAMPLER_* */
  float eta;                    /* DDIM eta (0 in the reference's callers) */
  int32_t skip_timesteps;       /* gaussian_diffusion.py:1252-1260: the loop starts at t0 = T - 1 - skip_timesteps */
  int32_t num_steps;            /* loop iterations to run; 0 = all the way down to t = 0 */
  int32_t resume;               /* 1: x_T already IS the state x_t0 (no q_sample of init_image); used to continue a
                                   loop chunk by chunk, e.g. for the *_progressive generators (:1217, :1514) */
  const float* init_image;      /* ref layout or NULL (zeros when skip_timesteps > 0, :1252-1253) */
  /* noise: either a tape or the engine's counter-based generator */
  const float* x_T;             /* ref layout initial noise (p_sample_loop's `noise=` / randn(*shape), :1245-1248) or NULL */
  const float* noise_tape;      /* (num_steps, B, 263, 1, 196): tape[k] is the k-th randn_like draw of the loop
                                   (k = 0 is the first, i.e. largest-t, step), or NULL */
  uint64_t seed;                /* used when x_T / noise_tape are NULL */
  uint64_t sample_offset;       /* global index of local sample 0: results are independent of how a batch is sharded */
  int32_t rng_mode;             /* CMDI_RNG_ENGINE (seed / sample_offset above) or CMDI_RNG_TORCH: reproduce the stream of
                                   torch.randn / randn_like on this device (gaussian_diffusion.py:696, :1248, :1407) from
                                   generator state (seed, aten_offset): x_T first when x_T is NULL, then one draw per step */
  uint64_t aten_offset;         /* philox offset of torch's CUDA generator at loop entry (multiple of 4) */
  uint64_t aten_increment;      /* offset one randn of B*263*196 elements consumes (ATen: calls per thread x 4) */
  uint32_t aten_threads;        /* 256 x grid of ATen's distribution kernel for that numel on this device */
  /* conditioning */
  const float* cond_emb;        /* (B, 512) or NULL */
  int32_t uncond;               /* y['uncond'] on a plain (non-CFG) model: zero the text embedding (mdm.py:188-191) */
  int32_t cfg;                  /* model is wrapped in ClassifierFreeSampleModel */
  const float* text_scale;      /* (B,) y['text_scale'] */
  const uint8_t* y_mask;        /* (B, 196) y['mask'] as bytes, or NULL (= all true) */
  /* keyframe imputation, gaussian_diffusion.py:427-435 + utils/editing_util.py:336-346 */
  int32_t imputate;
  int32_t stop_imputation_at;
  const float* inpainted_motion;   /* ref layout */
  const uint8_t* inpainting_mask;  /* ref layout, bool bytes */
  /* reconstruction guidance, gaussian_diffusion.py:405-425 + utils/editing_util.py:325-333: at steps t >= stop_recguidance_at
   * x0_hat is moved along -d/dz sum((inpainted_motion - x0_hat(z))^2 * M) (a backward pass through the denoiser) */
  int32_t recon_guidance;
  int32_t stop_recguidance_at;
  const float* recon_coef;         /* HOST array [T]: w_r[t] * reconstruction_weight * sqrt(alphas_cumprod[t]) / 2, fp32 */
  /* outputs */
  float* pred_xstart_out;       /* ref layout, last step's pred_xstart, or NULL */
  float* dump_xstart;           /* (n_dump, B, 263, 1, 196) pred_xstart at the loop iterations listed in dump_steps, or NULL */
  const int32_t* dump_steps;    /* host array of loop-iteration indices (ascending), p_sample_loop's dump_steps (:1208-1213) */
  int32_t n_dump;
  int32_t host_buffers;         /* 1: every pointer above and `out` are HOST pointers (copies happen inside the call) */
  int32_t use_graph;            /* 0: plain launches; 1: one captured CUDA graph replayed per step for calls of >= 3 steps
                                   (default); 2: also for one-step calls (the *_progressive generators) */
  /* keyframe INPUT conditioning of MDM_UNET: model_kwargs['obs_x0'] / ['obs_mask'] (sample/conditional_synthesis.py:159-162),
     constant over the loop; NULL for models that do not consume them */
  const float* obs_x0;          /* ref layout */
  const uint8_t* obs_mask;      /* ref layout, bool bytes (NOT and-ed with y['mask']) */
  /* CMDI_SAMPLER_PLMS only.  The eps history stays on the device: a call with resume = 0 starts a new one, a call with
     resume = 1 continues it (x_T = the previous call's sample, skip_timesteps advanced by its steps).  noise_tape and
     dump_xstart must be NULL: the only draw is x_T. */
  int32_t plms_order;           /* 2..4 (plms_sample's `order`) */
  float* plms_old_eps_out;      /* NULL, or (min(steps so far, plms_order - 1), B, 263, 1, 196): the reference's old_eps
                                   list after the last step, oldest first (ref layout) */
  /* CMDI_SAMPLER_DPM_SOLVER and CMDI_SAMPLER_DPM_SOLVER_SDE only (0 for every other sampler).  The x0 history stays on
     the device like PLMS's eps history: resume = 1 continues it with the same sampler, order and batch. */
  int32_t dpm_order;            /* 1..3 (DPM_SOLVER), 1..2 (DPM_SOLVER_SDE) */
  /* CMDI_SAMPLER_UNIPC only (all 0 for every other sampler).  The x0 history and the corrected state stay on the device:
     resume = 1 continues them with the same order, variant, corrector and batch. */
  int32_t unipc_order;          /* 1..3 */
  int32_t unipc_variant;        /* CMDI_UNIPC_BH1 / CMDI_UNIPC_BH2 */
  int32_t unipc_corrector;      /* 0 / 1 */
  /* CMDI_SAMPLER_REPAINT only (both 0 for every other sampler); RePaint's names */
  int32_t repaint_jump_length;  /* >= 1: positions an undo run goes up */
  int32_t repaint_jump_n_sample; /* >= 1: passes over each jumped stretch (1 = no resampling) */
  /* Overlapping windows: a motion of global_frames = N frames, longer than the engine's nframes = F, sampled as
     window_count = K windows of F frames whose x0 is blended at every step (all four fields 0 / NULL: off).  Row
     s * K + k of the batch is window k of global sample s and covers global frames [window_frames0[k],
     window_frames0[k] + F); batch counts windows (max_batch too), so batch = B_global * K.
       - window_frames0[0] = 0, window_frames0[K - 1] = N - F, strictly ascending, and consecutive windows leave no gap.
       - x0 (after CFG, guidance and imputation) of a frame covered by several windows is sum_k w_k x0_k / sum_k w_k over
         them in ascending k, fp32 with round-to-nearest products, sums and quotient, w_k = 1 + the frame's distance to
         the nearer end of window k; a frame covered by one window keeps its x0.  Every covering window stores the same
         bits at a shared frame (state, pred_xstart, multistep histories).
       - Global layout (B_global, njoints, 1, N): x_T, noise_tape ((num_steps, B_global, njoints, 1, N)), out,
         pred_xstart_out and dump_xstart; the engine crops x_T into the windows once per call and gathers the outputs
         from the first window covering each frame.  Every draw is that of the global tensor: the CMDI_RNG_TORCH stream of
         B_global * njoints * N elements (aten_increment / aten_threads for that numel), the engine generator keyed by
         (global sample, element c * N + g).
       - Window layout (batch, ...): cond_emb, text_scale, y_mask, inpainted_motion, inpainting_mask, obs_x0, obs_mask
         and init_image, cropped by the caller (a window may carry its own prompt).
     Samplers DDPM, DDIM, PLMS, DPM_SOLVER, UNIPC and DPM_SOLVER_SDE; plms_old_eps_out must be NULL. */
  int32_t window_count;         /* K >= 1, or 0: no windows */
  const int32_t* window_frames0; /* HOST array [K]: first global frame of each window */
  int32_t global_frames;        /* N */
  float* window_out;            /* test aid: NULL, or (batch, njoints, 1, F) the windows' final states (window layout) */
} cmdi_sample_args;

CMDI_API int cmdi_engine_create(const cmdi_model_cfg* cfg, int device, cmdi_engine** out);
CMDI_API int cmdi_engine_destroy(cmdi_engine* e);
CMDI_API int cmdi_load_weights(cmdi_engine* e, const cmdi_tensor_desc* tensors, int n);
/* betas: the (respaced) float64 betas of the sampler, length T; timestep_map[t] = original timestep of step t */
CMDI_API int cmdi_set_schedule(cmdi_engine* e, const double* betas, int T, const int64_t* timestep_map);
CMDI_API int cmdi_model_forward(cmdi_engine* e, const cmdi_forward_args* args, float* out, void* stream);
CMDI_API int cmdi_sample(cmdi_engine* e, const cmdi_sample_args* args, float* out, void* stream);
/* number of kernels of this library launched (directly or through graph replay) by the engine so far */
CMDI_API int64_t cmdi_launch_count(const cmdi_engine* e);
CMDI_API const char* cmdi_last_error(void);
CMDI_API const char* cmdi_version(void);

/* ---- kernel-level entry points (used by the parity tests; device pointers, fp32 row-major) ---- */
/* C[M,N] = act(A[M,K] W[N,K]^T + bias) (+ residual); block_n in {128, 256}: one CTA per tile; {-128, -256}: CTA-pair kernel.
   precision: CMDI_PRECISION_*; with CMDI_PRECISION_FP16 A, W and bias are rounded to fp16 and C holds fp16 values */
CMDI_API int cmdi_test_linear(const float* A, const float* W, const float* bias, const float* residual, float* C, int M, int N,
                     int K, int act, int precision, int block_n, void* stream);
/* O = softmax(Q K^T / sqrt(128)) V for `num_seqs` sequences of length S and H heads; qkv: [num_seqs*S, 3*H*128];
   O = hi + lo of the output planes (nsplit_out = 3) */
CMDI_API int cmdi_test_attention(const float* qkv, float* O, int num_seqs, int S, int H, int precision, void* stream);
/* the same launch with nsplit_out = 1, the engine's setting at CMDI_PRECISION_BF16: the kernel writes the hi plane only
   and O is that plane */
CMDI_API int cmdi_test_attention_hi(const float* qkv, float* O, int num_seqs, int S, int H, int precision, void* stream);
CMDI_API int cmdi_test_layernorm(const float* v, const float* gamma, const float* beta, float* out, int rows, void* stream);
/* one diffusion-step update on ref-layout tensors (all device): see StepParams in csrc/kernels.h */
CMDI_API int cmdi_test_step(cmdi_engine* e, int sampler, float eta, int t, int B, const float* model_out_c, const float* model_out_u,
                   const float* text_scale, const float* x_t, const float* noise, int impute, int stop_imputation_at,
                   const float* x_obs, const uint8_t* mask, float* x_next, float* pred_xstart, void* stream);

/* one guided evaluation (args as cmdi_model_forward, device pointers) and its input-VJP, as a reconstruction-guided step runs
 * them: grad receives d/dx of sum((inpainted_motion - x0_hat)^2 * inpainting_mask) through each pass, (cfg ? 2 : 1) x
 * (B, njoints, 1, nframes), the cond pass first (the sampler adds the two and masks them).  MDM_UNET: CMDI_PRECISION_FP16 only */
CMDI_API int cmdi_test_input_vjp(cmdi_engine* e, const cmdi_forward_args* args, const float* inpainted_motion,
                        const uint8_t* inpainting_mask, float* grad, void* stream);
/* backward pieces of reconstruction guidance (fp32 in / out) */
CMDI_API int cmdi_test_layernorm_bwd(const float* dy, const float* v, const float* gamma, float* dv, int rows, void* stream);
CMDI_API int cmdi_test_attention_bwd(const float* qkv, const float* dO, float* dqkv, int num_seqs, int S, int H, void* stream);
/* cmdi_test_attention_bwd (which runs CMDI_PRECISION_BF16X3) at `precision` = CMDI_PRECISION_BF16X3 or CMDI_PRECISION_BF16,
   the wgmma kernel's nsplit; dqkv = hi + lo of its output planes */
CMDI_API int cmdi_test_attention_bwd_at(const float* qkv, const float* dO, float* dqkv, int num_seqs, int S, int H, int precision,
                               void* stream);
/* One middle encoder layer's chained launch (out-proj + residual LN2'(v2_prev) -> v1; FFN1 with norm1 folded + GELU -> h;
 * FFN2 + residual LN1(v1) -> v2; the next layer's QKV projection with norm2 folded), phases set up as the engine sets them.
 * in[16], fp32 device: attn [M,512], v2_prev [M,512] (the previous layer's pre-norm2 sum), prev norm2 weight, bias [512],
 *   out_proj weight [512,512], bias, norm1 weight, bias, linear1 weight [1024,512], bias, linear2 weight [512,1024], bias,
 *   norm2 weight, bias, next in_proj weight [1536,512], bias.
 * out[4], fp32 device: v1 [M,512], h [M,1024], v2 [M,512], qkv [M,1536], read back from the bf16 planes the launch wrote:
 *   v1 and v2 (residual sources) as hi + lo, h and qkv as hi + lo at CMDI_PRECISION_BF16X3 and hi at CMDI_PRECISION_BF16.
 * Every lo plane the launch may write or read, except v2_prev's, is prefilled with bf16(stale_lo): results must not depend on it. */
CMDI_API int cmdi_test_chain_layer(const float* const* in, float* const* out, int M, int precision, float stale_lo, void* stream);
/* per-launch device times (ms, mean over `repeats` back-to-back launches of each kernel) of one denoiser pass at
 * `batch` (x2 sequences when cfg), in launch order:
 * token_rows, frame_embed, {qkv, attention, out_proj, ln1, ffn1, ffn2, ln2} x num_layers, out_head */
CMDI_API int cmdi_profile_pass(cmdi_engine* e, int batch, int cfg, int repeats, float* ms, int capacity, int* count, void* stream);
/* the engine's counter-based N(0,1) generator: out[b, i] depends only on (seed, stream_id, sample_offset + b, i) */
CMDI_API int cmdi_test_normal(float* out, int B, long long per_sample, unsigned long long seed, unsigned long long stream_id,
                     unsigned long long sample_offset, void* stream);

/* HumanML3D feature vectors -> joint positions: recover_root_rot_pos + recover_from_ric
 * (data_loaders/humanml/scripts/motion_process.py:402-441, :474-489), optionally fused with the de-normalisation
 * data * std + mean (data_loaders/humanml/data/dataset.py:378-382) and the permutes around them
 * (sample/synthesize.py:153-157).  Device pointers; strides in elements.
 *   data : element (sequence b, frame f, feature c) at data[b*stride_seq + f*stride_frame + c*stride_feat]
 *          -- (B,263,1,196) sampler output: strides (263*196, 1, 196); (B,1,196,263) reference input: (196*263, 263, 1)
 *   mean, std : [nfeats] or both NULL (data already de-normalised)
 *   out  : joints_num x 3 positions per frame, element (b, f, joint j, coordinate k) at
 *          out[b*ostride_seq + f*ostride_frame + j*ostride_joint + k*ostride_coord]
 *   joints_num : 22 (HumanML3D, 263 features) or 21 (KIT, 251); nfeats >= 4 + 3*(joints_num-1); nframes <= 2048 */
CMDI_API int cmdi_recover_from_ric(const float* data, long long stride_seq, long long stride_frame, long long stride_feat,
                          const float* mean, const float* std, int num_seqs, int nframes, int nfeats, int joints_num,
                          int abs_3d, float* out, long long ostride_seq, long long ostride_frame, long long ostride_joint,
                          long long ostride_coord, void* stream);
/* HumanML3D representation conversions, 22-joint skeleton only (paramUtil.t2m_raw_offsets / t2m_kinematic_chain,
 * face joints [2, 1, 17, 16], feet [8, 11] / [7, 10]).  One CTA per sequence, one launch on the caller's stream, no host
 * synchronisation.  Device pointers; strides in elements.  Limits: 2 <= nframes <= 224, joints_num == 22, nfeats == 263.
 *
 * cmdi_joints_to_features: extract_features (data_loaders/humanml/scripts/motion_process.py:50-187)
 *   joints : (num_seqs, nframes, 22, 3) fp32, sequence b / frame f at joints[b*stride_seq + f*stride_frame], the 66
 *            coordinates of a frame contiguous
 *   out    : (num_seqs, nframes - 1, 263) de-normalised features, element (b, f, c) at
 *            out[b*ostride_seq + f*ostride_frame + c*ostride_feat]; contacts compare the squared displacement to feet_thre */
CMDI_API int cmdi_joints_to_features(const float* joints, long long stride_seq, long long stride_frame, int num_seqs,
                            int nframes, int joints_num, double feet_thre, float* out, long long ostride_seq,
                            long long ostride_frame, long long ostride_feat, void* stream);

enum {
  CMDI_MOTION_ABS3D_TO_REL = 0,    /* dataset.py:1327-1361 abs3d_to_rel                                               */
  CMDI_MOTION_REL_TO_ABS3D = 1,    /* dataset.py:1364-1401 rel_to_abs3d                                               */
  CMDI_MOTION_REL_TO_JOINTS = 2,   /* inv_transform + recover_from_ric(abs_3d=False)                                 */
  CMDI_MOTION_ABS3D_TO_JOINTS = 3  /* inv_transform + recover_from_ric(abs_3d=True) (sample_to_motion, dataset.py:1301) */
};
/* cmdi_convert_motion: a normalised (num_seqs, 263, 1, nframes) batch, element (b, c, f) at
 * in[b*stride_seq + c*stride_feat + f*stride_frame], through
 *   [x @ inv_proj] (inv_random_projection, dataset.py:536-539; inv_proj [263, 263] row-major or NULL)
 *   -> x * std_in + mean_in (inv_transform, dataset.py:378-382) -> recover_from_ric (motion_process.py:474-489)
 * and, for the two representation directions,
 *   -> extract_features -> duplicate the last row (dataset.py:1214) -> [ABS3D_TO_REL] (x - mean_out) / std_out
 *                                                                     [REL_TO_ABS3D] channels 0..2 replaced by rot_ang and
 *      r_pos.xz of recover_root_rot_pos(abs_3d=False) (dataset.py:1276-1279), then (x - mean_out) / std_out
 * out: the same layout as `in` (ostride_*), or for the *_TO_JOINTS directions positions (num_seqs, 22, 3, nframes) with
 *      element (b, joint j, coordinate k, f) at out[b*ostride_seq + (3*j + k)*ostride_feat + f*ostride_frame] (mean_out /
 *      std_out unused).
 * Statistics are float64 arrays; in_f64 / out_f64 = 1 computes that (de-)normalisation in float64, as the reference does
 * for float64 statistics, 0 in float32 (the statistics then hold float32 values). */
CMDI_API int cmdi_convert_motion(int direction, const float* in, long long stride_seq, long long stride_feat,
                        long long stride_frame, int num_seqs, int nframes, int nfeats, const float* inv_proj,
                        const double* mean_in, const double* std_in, int in_f64, const double* mean_out,
                        const double* std_out, int out_f64, double feet_thre, float* out, long long ostride_seq,
                        long long ostride_feat, long long ostride_frame, void* stream);

/* out[i] = element i of torch.randn(numel, device=this GPU) under generator state (seed, offset); `threads` as
 * cmdi_sample_args.aten_threads */
CMDI_API int cmdi_test_normal_aten(float* out, long long numel, unsigned long long seed, unsigned long long offset,
                          unsigned int threads, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CONDMDI_B200_H_ */
