/* b200mdm.h -- C ABI of libb200mdm.so: the H100 (sm_90a) sampling engine that replaces the per-step hot path of
 * GuyTevet/motion-diffusion-model (paths below are relative to the reference repository root).
 *
 * The reference is pure Python, so there is no existing FFI to mirror; each entry point states which
 * reference function(s) it replaces.  The Python host mirror (motion-diffusion-model_b200/) binds these with
 * ctypes (see INTEGRATION.md) and passes torch tensors as raw pointers (`tensor.data_ptr()`), the CUDA stream
 * as `torch.cuda.current_stream().cuda_stream`.
 *
 * Conventions
 *   - every function returns 0 on success, a negative B200MDM_E* code on failure; b200mdm_last_error() returns a
 *     thread-local description of the most recent failure;
 *   - pointers named *_dev are device pointers, *_host host pointers; no ownership is transferred;
 *   - tensors use the reference's layouts: motion x [B, njoints, nfeats, T] fp32 (T contiguous),
 *     text embedding [B, cond_dim] fp32 (the reference's [1, B, C] with the leading 1 dropped);
 *   - nothing allocates on the per-step path: b200mdm_set_cond selects the workspace of a (B, T, CFG) triple -- built
 *     on first use, then kept (with its captured step graph) in a small pool;
 *   - kernels are specialised for latent_dim 512, 4 heads of 128 and sequences of at most 256 tokens (every released
 *     MDM / DiP model; 196 frames + 1 token); other shapes -> B200MDM_ENOTIMPL;
 *   - no call synchronises the stream except where stated.
 */
#ifndef B200MDM_H_
#define B200MDM_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200MDM_OK 0
#define B200MDM_EINVAL (-1)   /* contract violation (the reference raises AssertionError / ValueError) */
#define B200MDM_ECUDA (-2)    /* CUDA runtime / driver error */
#define B200MDM_ESTATE (-3)   /* call order violated (weights not finalised, schedule / cond missing ...) */
#define B200MDM_ENOTIMPL (-4) /* configuration the engine does not implement (reference: NotImplementedError) */

#define B200MDM_ARCH_TRANS_ENC 0
#define B200MDM_ARCH_TRANS_DEC 1

#define B200MDM_COND_NONE 0
#define B200MDM_COND_TEXT 1
#define B200MDM_COND_ACTION 2

#define B200MDM_MODE_X0 0   /* model output only */
#define B200MDM_MODE_DDPM 1 /* p_sample */
#define B200MDM_MODE_DDIM 2 /* ddim_sample */
/* (3-5: the PLMS steps inside b200mdm_plms_loop_range / b200mdm_plms_step, 7: the DPM-Solver++ step inside
 * b200mdm_dpm_loop_range, 8: the bound step inside b200mdm_vb_loop_range; not valid modes of the calls below) */
#define B200MDM_MODE_DDIM_REVERSE 6 /* ddim_reverse_sample: b200mdm_sample_step only (noise_dev may be NULL) */

#define B200MDM_FLAG_CONST_NOISE 1   /* p_sample(const_noise=True): eps row 0 repeated (gaussian_diffusion.py:527-528) */
#define B200MDM_FLAG_CLIP_DENOISED 2 /* clip_denoised=True: clamp x0 to [-1,1] (gaussian_diffusion.py:348-352) */
#define B200MDM_FLAG_PHILOX_NOISE 4  /* loops only: eps comes from the engine's counter-based stream (b200mdm_set_noise_stream)
                                        instead of a caller-provided tape -- replaces th.randn_like, gaussian_diffusion.py:525 */

#define B200MDM_SCHED_STRIDE 8 /* floats per schedule row, see b200mdm_set_schedule */

typedef struct b200mdm_engine b200mdm_engine;

/* Mirrors the keyword arguments utils/model_util.py:24-71 (get_model_args) passes to MDM.__init__
 * (model/mdm.py:12-135) that matter to the forward pass. */
typedef struct b200mdm_config {
  int32_t arch;              /* B200MDM_ARCH_*            (args.arch) */
  int32_t latent_dim;        /* 512                       (args.latent_dim) */
  int32_t ff_size;           /* 1024                      (hard-wired model_util.py:63) */
  int32_t num_layers;        /* 8                         (args.layers) */
  int32_t num_heads;         /* 4                         (hard-wired model_util.py:63) */
  int32_t njoints;           /* 263 humanml / 25 a2m */
  int32_t nfeats;            /* 1 humanml / 6 a2m */
  int32_t cond_mode;         /* B200MDM_COND_*            (utils/parser_util.py:269-276) */
  int32_t cond_dim;          /* 512 CLIP / 768 DistilBERT (model/mdm.py:121) */
  int32_t num_actions;       /* rows of embed_action.action_embedding */
  int32_t mask_frames;       /* args.mask_frames (model/mdm.py:241-247) */
  int32_t pos_embed_max_len; /* args.pos_embed_max_len: rows of the positional table */
  int32_t temb_rows;         /* model timesteps to pre-embed (>= original_num_steps of the diffusion) */
  int32_t context_len;       /* trans_dec (DiP) prefix completion: args.context_len frames precede x (model/mdm.py:58-61) */
  /* Target-location conditioning (args.multi_target_cond, model/mdm.py:64-73,197-199); 0 / 0 / 0 = none. */
  int32_t target_encoder;    /* B200MDM_TARGET_*          (args.multi_encoder_type) */
  int32_t target_enc_layers; /* args.target_enc_layers (single / split; the multi encoder always has one hidden layer) */
  int32_t target_joints;     /* n_ext = len(all_goal_joint_names) + 2 ('traj', 'heading'): 8 for HumanML3D */
  /* trans_dec only (model/mdm.py:241-270); 0 / 0 = DiP: BERT token memory, no timestep token. */
  int32_t emb_trans_dec;     /* args.emb_trans_dec: the timestep embedding is sequence token 0 (pe[0]), frames follow */
  int32_t dec_memory;        /* B200MDM_DEC_MEMORY_*: what the cross-attention of every decoder layer attends to */
  int32_t reserved[1];
} b200mdm_config;

/* Decoder memory kinds.  trans_dec accepts MEMORY_CLIP only with emb_trans_dec = 1 and context_len = 0 (the
 * humanml-decoder-with-emb checkpoint), and emb_trans_dec = 1 only with MEMORY_CLIP; other pairs -> B200MDM_ENOTIMPL. */
#define B200MDM_DEC_MEMORY_TOKENS 0 /* text-token features + padding mask (DiP, text_encoder_type 'bert') */
#define B200MDM_DEC_MEMORY_CLIP 1   /* one CLIP feature row per sample: memory = embed_text(clip) + time_emb (mdm.py:262-264).
                                       A softmax over one key is 1, so each layer's cross-attention block reduces to
                                       the per-sample row c_l = out_proj(W_v m + b_v), added before norm2. */

#define B200MDM_TARGET_NONE 0
#define B200MDM_TARGET_SINGLE 1 /* EmbedTargetLocSingle: one MLP on cat(target, valid) [4 n_ext] */
#define B200MDM_TARGET_MULTI 2  /* EmbedTargetLocMulti: an MLP per valid joint, combined by WeightedSum */
#define B200MDM_TARGET_SPLIT 3  /* EmbedTargetLocSplit: a mini-MLP of width d / n_ext per joint, concatenated */

const char* b200mdm_last_error(void);
int b200mdm_version(void);

/* MDM.__init__ (model/mdm.py:12-135): allocates the weight store for `cfg` on the current CUDA device. */
int b200mdm_create(const b200mdm_config* cfg, b200mdm_engine** out);
int b200mdm_destroy(b200mdm_engine* e);

/* load_model_wo_clip / load_state_dict(strict=False) (utils/model_util.py:8-15): one call per state_dict entry,
 * `name` is the reference key (SURVEY.md A.4), data fp32, host or device memory.  "sequence_pos_encoder.pe"
 * ([max_len, d]; the buffer the reference recomputes in PositionalEncoding.__init__, model/mdm.py:301-308) is
 * accepted here as well.  Unknown names -> B200MDM_EINVAL (the reference asserts no unexpected keys).
 * With target_encoder != 0 the embed_target_cond.* keys are accepted too; the multi encoder's per-joint keys name the
 * joint by its position in the extended joint list: "embed_target_cond.target_loc_emb.<index>.{0,2}.{weight,bias}". */
int b200mdm_load_weight(b200mdm_engine* e, const char* name, const float* data, const int64_t* shape, int32_t ndim);

/* Repack for the tensor cores (fp16 K-major copies, hi/lo split of the in/out projections), precompute the
 * timestep-embedding MLP (TimestepEmbedder.forward, model/mdm.py:329-330) for every model timestep.
 * Fails with B200MDM_ESTATE listing the first missing tensor. */
int b200mdm_finalize_weights(b200mdm_engine* e, void* stream);

/* SpacedDiffusion / GaussianDiffusion tables (diffusion/respace.py:74-88, gaussian_diffusion.py:166-205) after the
 * fp64->fp32 cast of _extract_into_tensor (gaussian_diffusion.py:1612).  rows_host: n_steps rows of
 *   [0] posterior_mean_coef1  [1] posterior_mean_coef2  [2] (t!=0) * exp(0.5*posterior_log_variance_clipped)
 *   [3] sqrt_recip_alphas_cumprod  [4] sqrt_recipm1_alphas_cumprod  [5] sqrt(alphas_cumprod_prev)
 *   [6] sqrt(1 - alphas_cumprod_prev - sigma_ddim^2)  [7] (t!=0) * sigma_ddim(eta)
 * timestep_map_host: _WrappedModel's map (respace.py:125-127), n_steps int32.  Synchronous copy. */
int b200mdm_set_schedule(b200mdm_engine* e, int32_t n_steps, const float* rows_host, const int32_t* timestep_map_host);

/* The DDIM inversion's table (ddim_reverse_sample, gaussian_diffusion.py:866-872), n_steps rows of
 *   [0] sqrt(alphas_cumprod_next)  [1] sqrt(1 - alphas_cumprod_next)
 * with alphas_cumprod_next cast fp64 -> fp32 first, then fp32 arithmetic (the last row is 0, 1).  n_steps must equal
 * the current schedule's; every b200mdm_set_schedule makes the table stale, and a reverse call against a stale table
 * fails with B200MDM_ESTATE.  Synchronous copy. */
#define B200MDM_SCHED_NEXT_STRIDE 2
int b200mdm_set_schedule_next(b200mdm_engine* e, int32_t n_steps, const float* rows_host);

/* The DPM-Solver++ table (no reference counterpart; DESIGN.md section 1), n_steps rows of
 *   [0] c_x = sigma_{i-1}/sigma_i  [1] c0 = alpha_{i-1} - alpha_i*sigma_{i-1}/sigma_i  [2] c_cur = c0*(1 + 1/(2r))
 *   [3] c_prev = -c0/(2r)
 * with alpha = sqrt(ac), sigma = sqrt(1 - ac), target index i - 1 taken from alphas_cumprod_prev, r = h_prev / h the
 * ratio of the log-SNR steps, every value computed in fp64 and rounded once.  Row 0 is (0, 1, ., .).  Staleness as for
 * b200mdm_set_schedule_next.  Synchronous copy. */
#define B200MDM_SCHED_DPM_STRIDE 4
int b200mdm_set_schedule_dpm(b200mdm_engine* e, int32_t n_steps, const float* rows_host);

/* The variational-bound table (calc_bpd_loop), n_steps rows of fp32 values as the reference's fp32 tensors hold them:
 *   [0] posterior_mean_coef1  [1] posterior_mean_coef2  [2] posterior_log_variance_clipped  [3] the model's fixed
 *   log-variance (FIXED_SMALL: = [2]; FIXED_LARGE: log(append(posterior_variance[1], betas[1:])))
 *   [4] sqrt_recip_alphas_cumprod  [5] sqrt_recipm1_alphas_cumprod  [6] sqrt_alphas_cumprod
 *   [7] sqrt_one_minus_alphas_cumprod  [8] ((-1 + [3]) - [2]) + exp([2] - [3])  [9] exp(-[3])  [10] exp(-(0.5 * [3]))
 *   [11] (-1 - log(1 - ac)) + exp(log(1 - ac))
 * ([8]-[11] in fp32 arithmetic from the fp32 entries; DESIGN.md section 1).  Staleness as for b200mdm_set_schedule_next.
 * Synchronous copy. */
#define B200MDM_SCHED_VB_STRIDE 12
int b200mdm_set_schedule_vb(b200mdm_engine* e, int32_t n_steps, const float* rows_host);

/* Canonicalises model_kwargs['y'] (data_loaders/tensors.py:22-64 + callers) once per loop and (re)builds the
 * workspace for (batch, nframes):
 *   cond_embed_dev : y['text_embed'][0]  [batch, cond_dim] fp32 device, or NULL (cond_mode none / action)
 *   lengths_host   : y['lengths'] int64 [batch] or NULL => no key mask (also ignored unless cfg.mask_frames)
 *   scale_dev      : y['scale'] fp32 [batch] device => ClassifierFreeSampleModel semantics (cond/uncond pair
 *                    packed into one batch of 2*batch, utils/sampler_util.py:27-34); NULL => single forward
 *   force_uncond   : y.get('uncond', False) for the single-forward case (model/mdm.py:208)
 *   action_host    : y['action'][:,0] int64 [batch] or NULL
 * The text projection embed_text(mask_cond(.)) (model/mdm.py:218) is evaluated here, once.  Every call starts a new
 * loop's conditioning: it clears the target (b200mdm_set_target) and the inpainting inputs (b200mdm_set_inpaint), also
 * at an unchanged shape; a PLMS / DPM-Solver++ loop of the selected workspace can still be continued. */
int b200mdm_set_cond(b200mdm_engine* e, int32_t batch, int32_t nframes, const float* cond_embed_dev,
                     const int64_t* lengths_host, const float* scale_dev, int32_t force_uncond,
                     const int64_t* action_host, void* stream);

/* Like b200mdm_set_cond, it clears the target (b200mdm_set_target) and the inpainting inputs (b200mdm_set_inpaint).
 * trans_dec (DiP, model/mdm.py:203-206,255-270): conditioning for arch = B200MDM_ARCH_TRANS_DEC.
 *   enc_text_dev   : y['text_embed'][0], BERT token features [n_tokens, batch, cond_dim] fp32 device (reference layout)
 *   text_mask_host : y['text_embed'][1], uint8 [batch, n_tokens], 1 = padding (memory_key_padding_mask)
 *   nframes        : frames of x (pred_len); the sequence is context_len + nframes tokens, no conditioning token
 *   n_tokens       : 1..512 (DistilBERT's position limit; B200MDM_EINVAL above).  Up to 64 tokens the cross-attention
 *                    core holds a sample's keys in registers; above, it streams them in blocks of 64.  The text-memory
 *                    buffers grow linearly in n_tokens (at 512 tokens and 128 guided rows, ~1.4 GB).
 * lengths / scale / force_uncond as in b200mdm_set_cond.  Must be followed by b200mdm_set_prefix when context_len > 0.
 * dec_memory = B200MDM_DEC_MEMORY_CLIP (emb_trans_dec): enc_text_dev is y['text_embed'] [1, batch, 512], the CLIP row
 * as the one memory token; n_tokens must be 1 (else B200MDM_EINVAL) and text_mask_host all zero (the reference passes
 * no memory mask).  The sequence is the timestep token + nframes frames; with cfg.mask_frames and lengths, token 0
 * and `lengths` frames are valid keys (mdm.py:241-247).  The per-sample part of every layer's cross-attention row,
 * out_proj(W_v (embed_text(clip) + g) + b_v), is evaluated here (and again by b200mdm_set_target), in fp32. */
int b200mdm_set_cond_dec(b200mdm_engine* e, int32_t batch, int32_t nframes, const float* enc_text_dev,
                         const uint8_t* text_mask_host, int32_t n_tokens, const int64_t* lengths_host,
                         const float* scale_dev, int32_t force_uncond, void* stream);
/* y['prefix'] [batch, njoints, nfeats, context_len] fp32 device: the frames x is a continuation of. */
int b200mdm_set_prefix(b200mdm_engine* e, const float* prefix_dev, void* stream);

/* Target-location conditioning (model/mdm.py:197-199) for an engine created with target_encoder != 0.  Call it after
 * b200mdm_set_cond / b200mdm_set_cond_dec (they size the workspace, and clear any previous target):
 *   target_dev : y['target_cond'] [batch, target_joints, 3] fp32 device
 *   valid_host : uint8 [batch, target_joints], 1 for each joint named in y['target_joint_names'][b], plus 'heading'
 *                when y['is_heading'][b]
 * g = embed_target_cond(target, valid) [batch, d] is evaluated here, in fp32, once per loop.  Every forward then adds
 * it to the timestep embedding, in both halves of a CFG pair: the conditioning token is cond + (temb[t] + g[b]) for
 * trans_enc, each text-memory token text_emb + (temb[t] + g[b]) for DiP.  y['target_uncond'] = True is a call that is
 * never made. */
int b200mdm_set_target(b200mdm_engine* e, const float* target_dev, const uint8_t* valid_host, void* stream);

/* y['inpainting_mask'] (bool as uint8) / y['inpainted_motion'] [B,J,F,T] device pointers
 * (gaussian_diffusion.py:300-304); NULL, NULL clears.  Call it after b200mdm_set_cond / b200mdm_set_cond_dec, which
 * clear it.  The pointers are read by every sampler step and loop (and so the pred_xstart of b200mdm_sample_step, as the
 * reference's p_mean_variance forms it), never by b200mdm_denoise or b200mdm_test_forward_taps, and must stay valid
 * until the work enqueued with them has completed. */
int b200mdm_set_inpaint(b200mdm_engine* e, const uint8_t* mask_dev, const float* motion_dev);

/* MDM.forward / ClassifierFreeSampleModel.forward (model/mdm.py:189-283, utils/sampler_util.py:27-34):
 * out = model(x, timesteps, y), without inpainting (the sampler's, not the model's).  timesteps_host: int32 [batch] MODEL
 * timesteps (already mapped). */
int b200mdm_denoise(b200mdm_engine* e, const float* x_dev, const int32_t* timesteps_host, float* out_dev, void* stream);

/* One p_sample / ddim_sample (gaussian_diffusion.py:489-541 / 729-779) at schedule index `index`:
 * x_out = step(x_t, eps).  pred_xstart_dev may be NULL.  x_out_dev may alias x_t_dev.
 * mode B200MDM_MODE_DDIM_REVERSE: one ddim_reverse_sample (gaussian_diffusion.py:838-874, eta = 0), x at index i ->
 * x at index i + 1: eps = (sr*x - x0)/srm1, x_out = x0*sqrt(abn) + sqrt(1 - abn)*eps.  noise_dev is not read (may be
 * NULL), the only valid flag is B200MDM_FLAG_CLIP_DENOISED, and b200mdm_set_schedule_next must have been called for
 * the current schedule. */
int b200mdm_sample_step(b200mdm_engine* e, int32_t mode, int32_t index, const float* x_t_dev, const float* noise_dev,
                        int32_t flags, float* x_out_dev, float* pred_xstart_dev, void* stream);

/* p_sample_loop / ddim_sample_loop (gaussian_diffusion.py:591-727 / 876-990) without returning to the host:
 * steps index = n_steps-1-skip_timesteps ... 0 are enqueued (one CUDA graph of a single step, replayed, when
 * use_graph != 0; the graph runs on an engine-owned stream ordered against `stream` with events).
 * x_T_dev: the initial sample (after any q_sample of init_image), not modified; x_0_dev: result (may alias x_T_dev).
 * noise_tape_dev: eps for the k-th executed step at noise_tape_dev + k*noise_step_stride elements.
 * flags: B200MDM_FLAG_*.  The tape must stay alive until the work enqueued here has completed. */
int b200mdm_sample_loop(b200mdm_engine* e, int32_t mode, int32_t skip_timesteps, const float* x_T_dev, float* x_0_dev,
                        const float* noise_tape_dev, int64_t noise_step_stride, int32_t flags, int32_t use_graph,
                        void* stream);

/* The same loop body for a sub-range of the schedule: indices first_index, first_index-1, ... (n_run of them).  This is
 * what lets the host draw the reference's per-step th.randn_like (gaussian_diffusion.py:525) in bounded chunks instead
 * of materialising an O(n_steps) tape.  x_in_dev NULL: continue from the state the previous call left in the engine;
 * x_out_dev NULL: leave the result there.  noise_tape_dev: eps of the k-th step OF THIS CALL at + k*noise_step_stride
 * (ignored with B200MDM_FLAG_PHILOX_NOISE). */
int b200mdm_sample_loop_range(b200mdm_engine* e, int32_t mode, int32_t first_index, int32_t n_run, const float* x_in_dev,
                              float* x_out_dev, const float* noise_tape_dev, int64_t noise_step_stride, int32_t flags,
                              int32_t use_graph, void* stream);

/* ddim_reverse_sample (gaussian_diffusion.py:838-874) repeated without returning to the host: schedule indices
 * first_index, first_index+1, ... (n_run of them, up to n_steps - 1) on the engine's working buffer, one CUDA graph of a
 * single step replayed when use_graph != 0.  x_in_dev / x_out_dev NULL as in b200mdm_sample_loop_range.  flags:
 * B200MDM_FLAG_CLIP_DENOISED or 0.  No noise is drawn.  Needs b200mdm_set_schedule_next for the current schedule. */
int b200mdm_ddim_reverse_loop_range(b200mdm_engine* e, int32_t first_index, int32_t n_run, const float* x_in_dev,
                                    float* x_out_dev, int32_t flags, int32_t use_graph, void* stream);

/* plms_sample_loop (gaussian_diffusion.py:1076-1187) without returning to the host: schedule indices first_index,
 * first_index-1, ... (n_run of them) on the engine's working buffer, order 1..4.  x_in_dev != NULL starts a fresh loop
 * from it, whose first step is the pseudo improved-Euler step (two forwards, the second at index i - 1, wrapping to
 * n_steps - 1 at i = 0); every later step is one Adams-Bashforth forward (one CUDA graph, replayed, when use_graph != 0).
 * A fresh loop of order 1 -> B200MDM_EINVAL (the reference fails on its missing history).  x_in_dev NULL continues
 * the PLMS loop the previous call of the same order left in the engine; x_out_dev NULL leaves the result there.
 * flags: B200MDM_FLAG_CLIP_DENOISED or 0.  No noise is drawn.  The eps history (3 x [B, JF, T] fp32), a scratch sample
 * and a pred_xstart buffer are allocated in the workspace on first use.  The loop to continue is the workspace's: a
 * b200mdm_set_cond* that selects another (batch, nframes, CFG) and then this one again, a b200mdm_set_cond* at the same
 * shape, b200mdm_denoise, b200mdm_sample_step, b200mdm_set_schedule and loops on other workspaces keep it; any other loop
 * on this workspace, b200mdm_plms_step, a weight reload and the eviction of the parked workspace from the pool end it
 * (B200MDM_ESTATE). */
int b200mdm_plms_loop_range(b200mdm_engine* e, int32_t order, int32_t first_index, int32_t n_run, const float* x_in_dev,
                            float* x_out_dev, int32_t flags, int32_t use_graph, void* stream);

/* One plms_sample (gaussian_diffusion.py:992-1074) at schedule index `index`: old_eps_dev is a host array of n_old
 * device pointers to [B, JF, T] fp32 eps, oldest first (old_out['old_eps']), and may be empty (n_old == 0: one
 * Adams-Bashforth forward at cur_order 1, as the reference does for an empty history).  old_eps_dev NULL (with
 * n_old == 0) is old_out = None: the improved-Euler step, order 2..4.  x_out_dev (may alias x_t_dev) receives the sample, pred_xstart_dev (may be NULL) the first
 * evaluation's x0, eps_out_dev (may be NULL) this step's eps -- the entry the caller appends to its history. */
int b200mdm_plms_step(b200mdm_engine* e, int32_t index, int32_t order, const float* x_t_dev, const float* const* old_eps_dev,
                      int32_t n_old, int32_t flags, float* x_out_dev, float* pred_xstart_dev, float* eps_out_dev,
                      void* stream);

/* Multistep DPM-Solver++ in its data-prediction form (Lu et al. 2022, Algorithm 2; no reference counterpart) without
 * returning to the host: schedule indices first_index, first_index-1, ... (n_run of them) on the engine's working
 * buffer, order 1 or 2, each step one forward (one CUDA graph per order, replayed, when use_graph != 0).  Step k of a
 * loop at index i: x0 as the DDIM step forms it (CFG, inpainting, clamp), kept in slot k % 2 of an x0 history, then
 *   x_out = fmaf(c0, x0, c_x*x)                                   at k == 0, i == 0 or order 1,
 *   x_out = fmaf(c_prev, x0 of step k - 1, fmaf(c_cur, x0, c_x*x)) otherwise (2M),
 * from row i of the b200mdm_set_schedule_dpm table (stale table -> B200MDM_ESTATE).  x_in_dev != NULL starts a fresh
 * loop (k = 0); NULL continues the DPM-Solver++ loop the previous call of the same order left in the engine, history
 * included; x_out_dev NULL leaves the result there.  flags: B200MDM_FLAG_CLIP_DENOISED or 0.  No noise is drawn.  The
 * history (2 x [B, JF, T] fp32) is allocated in the workspace on first use.  What keeps and what ends the loop to
 * continue is as for b200mdm_plms_loop_range, except that b200mdm_plms_step does not end it. */
int b200mdm_dpm_loop_range(b200mdm_engine* e, int32_t order, int32_t first_index, int32_t n_run, const float* x_in_dev,
                           float* x_out_dev, int32_t flags, int32_t use_graph, void* stream);
/* out_dev [B, JF, T] fp32 <- the x0 (pred_xstart) of the last step of that loop.  Enqueued on `stream`. */
int b200mdm_dpm_pred_xstart(b200mdm_engine* e, float* out_dev, void* stream);

/* The variational lower bound (calc_bpd_loop, gaussian_diffusion.py:1544-1599) at schedule indices first_index,
 * first_index-1, ... (n_run of them), each step one forward (one CUDA graph, replayed, when use_graph != 0):
 *   x_t = sqrt_ac*x_start + sqrt_1mac*eps (eps: step k of noise_tape_dev, or the engine's Philox stream with
 *   B200MDM_FLAG_PHILOX_NOISE, as in b200mdm_sample_loop_range); x0 as p_mean_variance forms it (CFG, inpainting, clamp
 *   under B200MDM_FLAG_CLIP_DENOISED); the KL term (the decoder NLL at index 0) in bits, (x0 - x_start)^2 and
 *   (eps(x_t, x0) - eps)^2, each averaged over the sample (padded frames included) with per-chunk partial sums in fixed
 *   slots and a fixed-order final sum: two runs on the same inputs give the same bits.
 * x_start_dev != NULL starts a fresh loop (x_start [B, JF, T] is copied in and never overwritten; every column is
 * cleared); NULL continues the bound loop left in the engine (b200mdm_set_cond* ends it).  terms_dev (nullable)
 * [3, B, n_steps] fp32 receives vb, xstart_mse, mse with column c = schedule index n_steps - 1 - c (columns no call of
 * this loop has reached hold 0).  bpd_dev (nullable) [2, B] receives total_bpd = the sum of the vb row (columns in order)
 * + prior_bpd, and prior_bpd, when this call ends at schedule index 0.  Stale bound table -> B200MDM_ESTATE.  The
 * buffers (about 2 x [B, JF, T] fp32) are allocated in the workspace on first use. */
int b200mdm_vb_loop_range(b200mdm_engine* e, int32_t first_index, int32_t n_run, const float* x_start_dev,
                          const float* noise_tape_dev, int64_t noise_step_stride, int32_t flags, float* terms_dev,
                          float* bpd_dev, int32_t use_graph, void* stream);

/* The engine's own noise stream (no reference counterpart: the reference draws from torch's global generator).
 * Philox4x32-10 keyed by `seed`, counter = (element/4, schedule index of the consuming step, global sample index);
 * Box-Muller on the 4 output words (exact recipe: csrc/kernels.cuh, restated in oracle/philox_oracle.py).  A sample's
 * noise depends only on (seed, its global index, step, element): sharding the batch over GPUs, or drawing the steps in
 * chunks, cannot change it.  sample_index_base = global index of this engine's sample 0. */
int b200mdm_set_noise_stream(b200mdm_engine* e, uint64_t seed, int64_t sample_index_base);
/* out[b, :] = that stream for step_id (x_T uses step_id = -1), b = 0..batch-1, n_per_sample fp32 each. */
int b200mdm_philox_normal(float* out_dev, int32_t batch, int64_t n_per_sample, uint64_t seed, int64_t sample_index_base,
                          int32_t step_id, void* stream);

/* q_sample (gaussian_diffusion.py:226-244) at schedule index `index`: out = sqrt_ac*x_start + sqrt_1mac*noise;
 * x_start_dev NULL => zeros (gaussian_diffusion.py:693-694).  sqrt_ac / sqrt_1mac are the fp32 table values. */
int b200mdm_q_sample(b200mdm_engine* e, float sqrt_ac, float sqrt_1mac, const float* x_start_dev,
                     const float* noise_dev, float* out_dev, int64_t n, void* stream);

/* Kernels launched by this engine since creation / since the last reset (bench.py's gpu_launches). */
int64_t b200mdm_launch_count(b200mdm_engine* e, int32_t reset);

/* ---- post-loop step (SURVEY.md 8f rank 2): sample/generate.py:161-166 for data_rep 'hml_vec' -- inv_transform
 * (data * std + mean, data_loaders/humanml/data/dataset.py:309-310) + recover_from_ric (data_loaders/humanml/scripts/
 * motion_process.py:366-385,437-452) in one kernel, any input / output layout through element strides:
 *   data element (b, feature f, frame t)       at data_dev[b*stride_b + f*stride_f + t*stride_t]
 *   out  element (b, frame t, joint j, axis c) at out_dev[b*ostride_b + t*ostride_t + (3j + c)*ostride_c]
 * mean_dev / std_dev: fp32 [features] or both NULL (input already de-normalised).  njoints 22 (263 features) / 21 (251). */
int b200mdm_recover_from_ric(const float* data_dev, int64_t stride_b, int64_t stride_f, int64_t stride_t,
                             const float* mean_dev, const float* std_dev, float* out_dev, int64_t ostride_b,
                             int64_t ostride_t, int64_t ostride_c, int32_t batch, int32_t nframes, int32_t njoints,
                             void* stream);

/* ---- kernel-level entry points (used by tests/ to check each kernel against a torch fp32 restatement) ---- */
/* out16[M,N] = fp16(act(A16[M,K] @ W16[N,K]^T + bias)); act: 0 none, 1 exact GELU.  K % 8 == 0, N % 8 == 0,
 * block_n must be 128: 128 x 128 tiles, the kernel every projection GEMM of the step runs on (B200MDM_EINVAL
 * otherwise, before the device is touched). */
int b200mdm_test_gemm_f16(const void* a16_dev, const void* w16_dev, const float* bias_dev, void* out16_dev, int32_t M,
                          int32_t N, int32_t K, int32_t act, int32_t block_n, void* stream);
/* The two projection-GEMM epilogues b200mdm_test_gemm_f16 does not reach, on 128 x 128 tiles; a16 [M,K], w16 [N,K] fp16,
 * bias fp32 [N], K % 8 == 0:
 *   epi 0: EpiBiasF16Wide<GELU> (the DiP FFN up-projection): out16 fp16 [M, 2N], columns [0, N) = hi, [N, 2N) = lo with
 *          hi + lo = gelu(A W^T + bias) to ~22 bits.  N % 64 == 0, N <= 2048.
 *   epi 1: EpiBiasF16Global (the DiP K/V projection of all layers): out16 fp16 [M, N] = fp16(A W^T + bias), bias read
 *          from global memory per tile, so N is not limited by the staged-vector size.  N % 32 == 0. */
int b200mdm_test_gemm_epi(const void* a16_dev, const void* w16_dev, const float* bias_dev, void* out16_dev, int32_t M,
                          int32_t N, int32_t K, int32_t epi, void* stream);
/* The embedding launches of the step (InputProcess + positional encoding, model/mdm.py:238,252,343-349) through scratch
 * buffers allocated on `stream`: pack_input (frame t -> row s = s_off + t), split_weight of w_in, pe_bias, then the
 * split-precision EpiEmbed GEMM.  x fp32 [B, JF, T]; w_in fp32 [d, JF]; b_in fp32 [d]; pe fp32 [>= T + s_off, d].
 * hres16 fp16 [halves*B*S, 2d] (S = T + s_off) receives [hi | lo] of x W^T + b_in + pe[s] in rows (b, s) of each CFG
 * half (rows s < s_off: b_in + pe[s]).  d % 64 == 0, d <= 2048, halves 1 or 2. */
int b200mdm_test_embed(const float* x_dev, const float* w_in_dev, const float* b_in_dev, const float* pe_dev, void* hres16_dev,
                       int32_t B, int32_t JF, int32_t T, int32_t d, int32_t s_off, int32_t halves, void* stream);
/* The output launches of the step through scratch buffers allocated on `stream`: blend_split of the residual stream, then
 * the split-weight EpiOut<OutStep> GEMM (BLOCK_N 96) with the sampler update, schedule row `sched_row` (8 floats, device; see
 * b200mdm_set_schedule) as a one-row table at index 0.
 * hres16 fp16 [halves*B*S, 2d] = [hi | lo] (S = T + s_off; rows s >= s_off are frames); scale fp32 [B] (NULL when
 * halves == 1); w_out fp32 [JF, d]; b_out fp32 [JF]; x_t, noise, x_out, pred_xstart fp32 [B, JF, T] (x_out may alias
 * x_t; noise may be NULL for mode B200MDM_MODE_X0); mode B200MDM_MODE_*; flags B200MDM_FLAG_CONST_NOISE (noise [JF, T]
 * for every sample) | B200MDM_FLAG_CLIP_DENOISED; inpaint_mask uint8 / inpaint_motion fp32 [B, JF, T] or both NULL. */
int b200mdm_test_out_step(const void* hres16_dev, const float* scale_dev, const float* w_out_dev, const float* b_out_dev,
                          const float* x_t_dev, const float* noise_dev, const float* sched_row_dev, int32_t mode, int32_t flags,
                          const uint8_t* inpaint_mask_dev, const float* inpaint_motion_dev, float* x_out_dev,
                          float* pred_xstart_dev, int32_t B, int32_t JF, int32_t T, int32_t d, int32_t s_off, int32_t halves,
                          void* stream);
/* The same output launches with the EpiOut<OutDpm> epilogue of b200mdm_dpm_loop_range, as step `step` (k) of a loop of
 * order 1 or 2 at schedule index `index`: dpm_row (4 floats, device; see b200mdm_set_schedule_dpm) is row `index` of
 * the table.  x0_hist fp32 [2, B, JF, T]: slot (k - 1) % 2 is read as the previous x0 (second-order steps only), slot
 * k % 2 receives this step's x0; x_out [B, JF, T] (may alias x_t) the update.  flags: B200MDM_FLAG_CLIP_DENOISED or 0;
 * other arguments as in b200mdm_test_out_step.  Invalid arguments return B200MDM_EINVAL before any CUDA call. */
int b200mdm_test_out_dpm(const void* hres16_dev, const float* scale_dev, const float* w_out_dev, const float* b_out_dev,
                         const float* x_t_dev, const float* dpm_row_dev, int32_t index, int32_t step, int32_t order,
                         int32_t flags, const uint8_t* inpaint_mask_dev, const float* inpaint_motion_dev,
                         float* x0_hist_dev, float* x_out_dev, int32_t B, int32_t JF, int32_t T, int32_t d, int32_t s_off,
                         int32_t halves, void* stream);
/* The same output launches with the EpiOut<OutVb> epilogue of b200mdm_vb_loop_range and its per-sample reduction, as
 * the bound step at schedule index `index` of an n_steps schedule: vb_row (12 floats, device; see b200mdm_set_schedule_vb)
 * is row `index` of the table; x_t, x_start, noise [B, JF, T].  pred_xstart (nullable) receives x0, elem (nullable)
 * [3, B, JF, T] the per-element terms before averaging, terms [3, B, n_steps] column n_steps - 1 - index the per-sample
 * means (the other columns are left as they are).  flags: B200MDM_FLAG_CLIP_DENOISED or 0; other arguments as in
 * b200mdm_test_out_step.  Invalid arguments return B200MDM_EINVAL before any CUDA call. */
int b200mdm_test_out_vb(const void* hres16_dev, const float* scale_dev, const float* w_out_dev, const float* b_out_dev,
                        const float* x_t_dev, const float* x_start_dev, const float* noise_dev, const float* vb_row_dev,
                        int32_t index, int32_t n_steps, int32_t flags, const uint8_t* inpaint_mask_dev,
                        const float* inpaint_motion_dev, float* pred_xstart_dev, float* elem_dev, float* terms_dev, int32_t B,
                        int32_t JF, int32_t T, int32_t d, int32_t s_off, int32_t halves, void* stream);
/* Self-attention core (tensor-core kernel, S <= 256): softmax(q k^T / sqrt(128) + mask) v per (sample, head);
 * qkv16 [n*S, 3d]; kvlen int32 [n] device (valid keys per sample, a prefix).
 * impl 0: out16 fp16 [n*S, d] (the encoder); impl 1: out16 fp16 [n*S, 2d] = [hi | lo] with hi + lo = the fp32 result
 * to ~22 bits (the DiP decoder). */
int b200mdm_test_attention(const void* qkv16_dev, void* out16_dev, const int32_t* kvlen_dev, int32_t n_samples,
                           int32_t S, int32_t d, int32_t impl, void* stream);
/* Cross-attention core of the trans_dec (DiP) layers, nn.MultiheadAttention(query = sequence, key = value = text memory)
 * between its in- and out-projections (model/mdm.py:219-224 via nn.TransformerDecoderLayer): d = 512, 4 heads.
 * q16 fp16 [n*S, 512]; kv16 fp16 rows (sample, token) of pitch ld_kv >= 1024 holding k | v; mask uint8 [n, n_tokens]
 * (1 = padding token, any pattern); out16 fp16 [n*S, 1024]: columns [0, 512) are written.  1 <= n_tokens <= 512: the
 * engine's dispatch, cross_attention_kernel for n_tokens <= 64 and cross_attention_long_kernel above.  Invalid arguments
 * return B200MDM_EINVAL before any CUDA call. */
int b200mdm_test_cross_attention(const void* q16_dev, const void* kv16_dev, const unsigned char* mask_dev, void* out16_dev,
                                 int32_t n_samples, int32_t S, int32_t n_tokens, int32_t ld_kv, void* stream);
/* QKV projection + attention core of an encoder layer (nn.MultiheadAttention up to its output projection,
 * model/mdm.py:77-84), the two kernels the step launches, through a scratch qkv buffer allocated on `stream`:
 * out16[n*S, 512] = concat_h softmax((h Wq_h^T + bq)(h Wk_h^T + bk)^T / sqrt(128) + mask)(h Wv_h^T + bv), q, k, v rounded to fp16.
 * h16: fp16 [n*S, ld] (first 512 columns used), wqkv16: in_proj_weight fp16 [1536, 512], bqkv fp32 [1536],
 * kvlen int32 [n] device (valid keys per sample), S <= 256. */
int b200mdm_test_qkv_attention(const void* h16_dev, int32_t ld, const void* wqkv16_dev, const float* bqkv_dev,
                               void* out16_dev, const int32_t* kvlen_dev, int32_t n_samples, int32_t S, void* stream);
/* h[M,512] <- LayerNorm(h + A16[M,K] @ W16[512,K]^T + bias; gamma, beta, 1e-5) in place (the fused out-projection /
 * FFN-down kernel of the transformer layer).  h is the engine's residual-stream format: fp16 [M, 1024] = [hi | lo],
 * value = hi + lo, read and written only with TMA (rows past M are never touched).  K % 8 == 0; a16, w16 and hres16
 * 16-byte aligned. */
int b200mdm_test_gemm_resid_ln(const void* a16_dev, const void* w16_dev, const float* bias_dev, const float* gamma_dev,
                               const float* beta_dev, void* hres16_dev, int32_t M, int32_t K, void* stream);
/* The target encoder of b200mdm_set_target on the engine's finalised weights, for any batch, through a scratch buffer
 * allocated on `stream`: out fp32 [batch, d] = embed_target_cond(target [batch, target_joints, 3], valid uint8 host). */
int b200mdm_test_target(b200mdm_engine* e, const float* target_dev, const uint8_t* valid_host, int32_t batch,
                        float* out_dev, void* stream);
/* The per-step cross-attention rows of a B200MDM_DEC_MEMORY_CLIP engine for its current workspace (after
 * b200mdm_set_cond_dec, and b200mdm_set_target when used), every sample at model timestep `timestep`:
 * out fp32 [num_layers, Bp, 512], Bp = 2 x batch with CFG (conditional rows, then unconditional), else batch;
 * row (l, b') = out_proj_l(W_v,l (embed_text(clip[b'] or 0) + temb[timestep] + g[b' mod batch]) + b_v,l). */
int b200mdm_test_cross_rows(b200mdm_engine* e, int32_t timestep, float* out_dev, void* stream);
/* The step's row-bias LayerNorm of such an engine: h[r] <- LayerNorm(h[r] + c[r / S]; gamma, beta, 1e-5) in place, for
 * r < M; h fp16 [M, 1024] = [hi | lo] (value hi + lo, d = 512), c fp32 [(M + S - 1) / S, 512]. */
int b200mdm_test_row_bias_ln(void* hres16_dev, const float* c_dev, const float* gamma_dev, const float* beta_dev,
                             int32_t M, int32_t S, void* stream);

/* Stage taps of the engine's own forward: one b200mdm_denoise (the same launches, programmatic dependent launch as
 * configured), and after the launch that produces tap point k the engine copies the workspace buffer behind it into
 * tap_dev[k] (a caller device buffer of the size below, or NULL to skip it) on `stream`.  Per-layer points (L_*) are taken
 * for layer `layer` only.  Nothing else changes: no graph, no loop state, no launch count.  A non-NULL buffer for a point
 * the model does not have, a bad layer or n_taps outside 0..B200MDM_TAP_COUNT return B200MDM_EINVAL before any CUDA call.
 * Synchronises the stream once (like b200mdm_denoise) before the forward is enqueued.
 * Sizes, with M = halves*B*S rows (S = T + 1, or context_len + T for DiP), Bp = halves*B, kw = 2 for DiP else 1, Mt the
 * text tokens, ff = ff_size, d = 512; h = fp16, f = fp32; hres rows are [hi | lo]: */
#define B200MDM_TAP_EMBED 0     /* h [M, 2d]  residual stream after the embedding GEMM, before token 0 */
#define B200MDM_TAP_TOK0 1      /* h [M, 2d]  after token 0 / the DiP memory build / the CLIP decoder's cross rows */
#define B200MDM_TAP_CONDPROJ 2  /* f [Bp, d]  conditioning rows (not DiP) */
#define B200MDM_TAP_TEMB 3      /* f [B, d]   timestep-embedding rows temb[timesteps[b]] */
#define B200MDM_TAP_MEM16 4     /* h [Bp*Mt, 2d] DiP: text memory + temb, [hi | lo] */
#define B200MDM_TAP_CROSS_C 5   /* f [L, Bp, d] CLIP decoder: every layer's cross-attention row of this step */
#define B200MDM_TAP_KVC16 6     /* h [Bp*Mt, L*2d] DiP: the K | V projections of every layer */
#define B200MDM_TAP_L_IN 7      /* h [M, 2d]  residual stream at the layer's entry */
#define B200MDM_TAP_L_QKV 8     /* h [M, 3d]  after the QKV GEMM */
#define B200MDM_TAP_L_ATT 9     /* h [M, kw*d] after the self-attention core */
#define B200MDM_TAP_L_LN1 10    /* h [M, 2d]  after out-proj + LN1 */
#define B200MDM_TAP_L_QC 11     /* h [M, d]   DiP: after the cross-attention Q GEMM */
#define B200MDM_TAP_L_XATT 12   /* h [M, kw*d] DiP: after the cross-attention core (columns [0, d)) */
#define B200MDM_TAP_L_LN2 13    /* h [M, 2d]  decoders: after cross out-proj + LN2 (DiP) / the row-bias LN2 (CLIP) */
#define B200MDM_TAP_L_FFN 14    /* h [M, kw*ff] after FFN-up (GELU) */
#define B200MDM_TAP_L_LN3 15    /* h [M, 2d]  after FFN-down + LN (norm2, decoders norm3) */
#define B200MDM_TAP_BLEND 16    /* h [B*T, 3d] CFG blend [hi | lo | hi], the output GEMM's A operand */
#define B200MDM_TAP_COUNT 17
int b200mdm_test_forward_taps(b200mdm_engine* e, const float* x_dev, const int32_t* timesteps_host, float* out_dev,
                              int32_t layer, void* const* tap_dev, int32_t n_taps, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200MDM_H_ */
