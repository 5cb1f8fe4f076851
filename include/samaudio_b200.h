/* samaudio_b200.h — C ABI of libsamaudio_b200.so: the H100 (sm_90a) implementation of the
 * SAMAudio.separate() inference hot path of facebookresearch/sam-audio.
 *
 * The reference has no FFI: its seam is the Python class surface (SURVEY.md §8b).  Each entry point
 * below names the reference method it replaces (paths relative to the reference tree); the Python
 * host mirror (sam_audio_b200/model.py) and INTEGRATION.md show the binding.
 *
 * Conventions
 *  - plain C types only; every device pointer is BORROWED (the caller — PyTorch in the Python mirror —
 *    owns activations and I/O buffers); the library owns its packed weights and workspace.
 *  - every function returns 0 on success, non-zero on failure; sab_last_error() gives the message
 *    (reference convention is Python exceptions; the mirror raises RuntimeError from it).
 *  - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises
 *    unless stated.  A handle is not thread-safe.
 *  - layouts: "rows x cols" row-major, fp32 unless stated; T = latent frames (25 Hz), S = samples.
 */
#ifndef SAMAUDIO_B200_H
#define SAMAUDIO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sab_engine sab_engine;

/* Shapes of the model (reference: sam_audio/model/config.py:86-130 TransformerConfig,
 * :10-41 DACVAEConfig, :204-231 SAMAudioConfig). */
typedef struct sab_config {
  int32_t dim;              /* transformer.dim (multiple of 128)            */
  int32_t n_heads;          /* transformer.n_heads (head_dim must be 128)   */
  int32_t n_layers;         /* transformer.n_layers                         */
  int32_t ffn_hidden;       /* SwiGLU hidden width (transformer.py:179-185) */
  int32_t out_channels;     /* 256                                          */
  int32_t in_channels;      /* SAMAudioConfig.in_channels = 768             */
  int32_t text_dim;         /* 768                                          */
  int32_t vision_dim;       /* 1024                                         */
  int32_t n_anchor_tokens;  /* num_anchors + 1 = 4                          */
  int32_t anchor_dim;       /* 128                                          */
  int32_t max_positions;    /* RoPE table length (10000)                    */
  float   rope_theta;       /* max(10000, 2*max_positions)                  */
  float   norm_eps;         /* 1e-5                                         */
  /* DAC-VAE codec */
  int32_t codec_encoder_dim;      /* 64   */
  int32_t codec_latent_dim;       /* 1024 */
  int32_t codec_decoder_dim;      /* 1536 */
  int32_t codec_codebook_dim;     /* 128  */
  int32_t codec_n_rates;          /* 4    */
  int32_t codec_encoder_rates[8]; /* 2,8,10,12 */
  int32_t codec_decoder_rates[8]; /* 12,10,8,2 */
} sab_config;

const char* sab_last_error(void);
int sab_version(void);

/* Lifecycle.  replaces: SAMAudio.__init__ (model.py:79-102). */
int sab_create(const sab_config* cfg, int device, sab_engine** out);
int sab_destroy(sab_engine* e);

/* Weights.  replaces: BaseModel._from_pretrained / load_state_dict (base.py:47-61, model.py:346-359).
 * `name` is the reference state-dict key (e.g. "transformer.layers.0.attention.wq.weight"; codec keys
 * "audio_codec.encoder.block.0.weight", weight-norm already folded).  `data` is fp32, contiguous, on host
 * (is_device=0) or device (is_device=1); it is consumed (repacked to bf16 / permuted) before returning.
 * Unknown names fail.  sab_finalize_weights() checks completeness and builds derived tables; with
 * allow_missing != 0 (load_state_dict(strict=False)) missing tensors keep their zero initialisation and their
 * names are written, newline-separated, into missing_out (may be NULL). */
int sab_load_weight(sab_engine* e, const char* name, const float* data, const int64_t* shape, int ndim,
                    int is_device, void* stream);
int sab_finalize_weights(sab_engine* e, int allow_missing, char* missing_out, int64_t missing_cap, void* stream);

/* Codec analysis.  replaces: DACVAE.forward (codec.py:65-78) + SAMAudio._get_audio_features (model.py:182-184).
 * wav [B, S] mono fp32 (S already padded to a multiple of hop by the caller = codec.py:72-78);
 * features [B, T, 2*codebook_dim] fp32: the 128-d mean latent duplicated along channels. */
int sab_encode(sab_engine* e, const float* wav, int B, int64_t S, float* features, void* stream);

/* Conditioning, once per separate() call.  replaces the time-independent part of SAMAudio.forward:
 * align_inputs (model.py:108-128), AlignModalities (align.py:30-50), EmbedAnchors (model.py:54-65),
 * memory_proj (model.py:92,172), and _repeat_for_reranking (model.py:193-203): every input is per CLIP
 * and the `candidates` sequences of a clip (candidate-minor, sequence = clip * candidates + k) share it
 * without being materialised; the ODE state has B * candidates sequences.
 *  features       [B, T, 256]      (sab_encode output)
 *  text_features  [B, L, text_dim] ; text_mask [B, L] uint8 (1 = token)
 *  video_features [B, vision_dim, T] or NULL (= zeros, model.py:188-189)
 *  anchor_ids [B, n_ids] int64 ; anchor_alignment [B, T] int64 ; audio_pad_mask [B, T] uint8 (1 = frame)
 *  flags: SAB_PREP_* — the three `None` cases of SAMAudio.forward (separate() never passes None). */
#define SAB_PREP_NO_VIDEO_TERM 1 /* masked_video_features=None: AlignModalities returns its input (align.py:41-42) */
#define SAB_PREP_NO_ANCHORS 2    /* anchor_ids=None: EmbedAnchors returns its input (model.py:57-58); ids may be NULL */
#define SAB_PREP_NO_TEXT 4       /* text_features=None: memory = time embedding only (model.py:170-172); L must be 1 */
int sab_prepare(sab_engine* e, int B, int candidates, int T, int L, const float* features, const float* text_features,
                const uint8_t* text_mask, const float* video_features, const int64_t* anchor_ids, int n_ids,
                const int64_t* anchor_alignment, const uint8_t* audio_pad_mask, int flags, void* stream);

/* One ODE function evaluation.  replaces: SAMAudio.forward / DiT.forward (model.py:130-180,
 * transformer.py:473-524) on the conditioning installed by sab_prepare.
 * noisy [Bc, T, 256], time [Bc] (device), velocity out [Bc, T, 256]. */
int sab_dit_forward(sab_engine* e, const float* noisy, const float* time, float* velocity, void* stream);

/* The ODE solve.  replaces: torchdiffeq.odeint(method=..., options={"step_size": 1/n_steps}) as called at
 * model.py:285-290 with the reference's **ode_opt: fixed-grid midpoint (the default, 2*n_steps evaluations), euler
 * (n_steps) or rk4 (torchdiffeq's 3/8 rule, 4*n_steps).  noise [Bc, T, 256] in, latent [Bc, T, 256] out (may alias). */
#define SAB_ODE_MIDPOINT 0
#define SAB_ODE_EULER 1
#define SAB_ODE_RK4 2
int sab_solve(sab_engine* e, const float* noise, int n_steps, int method, float* latent, void* stream);

/* Codec synthesis.  replaces: DACVAE.decode (codec.py:86-89) as called at model.py:291-295.
 * latent [Bc, T, 256] (target half = channels [0,128), residual half = [128,256));
 * wav [Bc, 2, T*hop] fp32 (row 0 target, row 1 residual). */
int sab_decode(sab_engine* e, const float* latent, int Bc, int T, float* wav, void* stream);

/* Introspection for benchmarks/tests: kernels launched by this engine since creation / last reset. */
int64_t sab_launch_count(sab_engine* e, int reset);
/* Workspace bytes currently held. */
int64_t sab_workspace_bytes(sab_engine* e);
/* Plan residency.  sab_prepare fills the DiT plan of its (B, candidates, T, L), building it if it is not resident, and
 * sab_solve / sab_dit_forward run the plan the last sab_prepare filled; each plan keeps its own workspace, time tables
 * and captured solve graph.  At most dit_plans DiT plans and codec_plans_per_direction codec plans per direction
 * (keyed by (items per chunk, length)) stay resident; the least recently used go first.  The defaults are 1 and 3.
 * Lowering a limit evicts at once (after a device synchronise).  Both limits must be >= 1. */
int sab_set_plan_limits(sab_engine* e, int dit_plans, int codec_plans_per_direction);
/* Counts since sab_create: DiT plans built, solve graphs captured, codec plans built (both directions); and the plans
 * resident now (codec: both directions).  Any pointer may be NULL. */
int sab_plan_stats(sab_engine* e, int64_t* dit_plan_builds, int64_t* graph_captures, int64_t* codec_plan_builds,
                   int* dit_plans_resident, int* codec_plans_resident);
/* Live per-kernel timing for roofline reporting: with profiling on, one CUDA event is recorded in front of
 * every launch on `stream`; sab_profile_report aggregates the inter-event times per kernel tag as JSON
 * ({"tag": {"launches","ms","flops","bytes"}}) and clears the log. */
int sab_profile(sab_engine* e, int enable, void* stream);
int sab_profile_report(sab_engine* e, char* json_out, int64_t capacity, void* stream);

/* ---- T5 text encoder (SURVEY §8f-3 "next" row) ----
 * replaces: the T5EncoderModel call inside T5TextEncoder.forward (reference sam_audio/model/text_encoder.py:29-35;
 * HF transformers T5Stack arithmetic).  Tokenisation stays on the host (HF tokenizer, text_encoder.py:21-27).
 * Weight names are the HF T5EncoderModel state-dict keys ("shared.weight",
 * "encoder.block.N.layer.0.SelfAttention.q.weight", ...). */
typedef struct sab_t5 sab_t5;
typedef struct sab_t5_config {
  int32_t vocab_size;   /* 32128 */
  int32_t d_model;      /* 768   */
  int32_t d_kv;         /* 64    */
  int32_t d_ff;         /* 3072  */
  int32_t n_layers;     /* 12    */
  int32_t n_heads;      /* 12    */
  int32_t n_buckets;    /* relative_attention_num_buckets = 32 */
  float   eps;          /* layer_norm_epsilon = 1e-6 */
} sab_t5_config;
int sab_t5_create(const sab_t5_config* cfg, int device, sab_t5** out);
int sab_t5_destroy(sab_t5* e);
int sab_t5_load_weight(sab_t5* e, const char* name, const float* data, const int64_t* shape, int ndim, int is_device,
                       void* stream);
int sab_t5_finalize(sab_t5* e, void* stream);
/* ids [B, L] int64, mask [B, L] uint8 (1 = token), rel_bucket [2L-1] int32 = T5's relative-position bucket of
 * (key - query) + L - 1 (computed by the host exactly as transformers does); out [B, L, d_model] fp32. */
int sab_t5_forward(sab_t5* e, const int64_t* ids, const uint8_t* mask, const int32_t* rel_bucket, int B, int L, float* out,
                   void* stream);
int64_t sab_t5_launch_count(sab_t5* e, int reset);

/* ---- unit-test seams (used by tests/ only; stable but not part of the drop-in surface) ---- */
/* C[M,N] (fp32) = A[M,K] (bf16) * B[N,K]^T (bf16) through the wgmma GEMM (tile BN x BK; cg = 1: one CTA per
 * 128-row tile, cg = 2: 2-CTA clusters on 256-row tiles sharing the B tile, cg = 0: the engine's default choice). */
int sab_test_gemm(int M, int N, int K, const void* a_bf16, const void* b_bf16, float* c, int bn, int bk, int cg,
                  void* stream);

/* The whole GEMM contract (sam_audio_b200/csrc/gemm_tc.cuh): one launch planned by the engine's own planner
 * (tile counts, TMA maps, cluster choice) with every epilogue field of GemmParams under the caller's control.
 * The descriptor and the epilogue combination are checked by the same rules as every engine plan, before any CUDA
 * call; a rejected descriptor returns non-zero with the rule in sab_last_error(). */
typedef struct sab_test_gemm_run {
  int32_t row_shift;  /* added to the tile's first row; rows outside [0, a_rows) read as zero */
  int32_t a_col;      /* first A column of the run */
  int32_t nkb;        /* number of bk-wide k-blocks */
} sab_test_gemm_run;
typedef struct sab_test_gemm_desc {
  int32_t struct_bytes;     /* = sizeof(sab_test_gemm_desc), checked first */
  /* tile */
  int32_t mode;             /* 0 affine, 1 SwiGLU, 2 QKV, 3 affine + fused-RMSNorm producer */
  int32_t bn, bk, cg, b2b;  /* cg = 0: the engine's choice; b2b: back-to-back second GEMM (codec residual unit) */
  /* A (bf16): a_cols visible columns, a_rows rows per item, a_items items; pitches in elements (0: packed) */
  const void* a;
  int64_t a_cols, a_rows, a_items, a_row_pitch, a_item_pitch;
  /* B (bf16) [n, sum of the run list's k-blocks * bk], K-major; w1: the b2b second weight [n, n] */
  const void* b;
  int32_t n;
  const void* w1;
  /* K runs: list 1 applies to the n-tiles with n_period > 0 and (n0 % n_period) >= n_switch */
  int32_t n_runs[2];
  sab_test_gemm_run runs[2][8];
  int32_t n_period, n_switch;
  /* schedule overrides, 0 = the engine's default */
  int32_t grid_ctas, group_m, reverse_m;
  /* epilogue: the GemmParams fields of the same names, with the same meaning */
  const float* bias; int32_t bias_mod;
  const float* gate; int32_t gate_ld, gate_div;
  float alpha; int32_t relu;
  const float* res; int64_t res_ld;
  float* out_f32; int64_t out_f32_ld;
  void* out_bf16; int64_t out_bf16_ld;
  void* out_act; int64_t out_act_ld; const float* snake_alpha;
  const float* colscale; int64_t colscale_ld;
  void* out_scaled; int64_t out_scaled_ld;
  float* ssq_out; int32_t ssq_ld;
  const float* ssq_in; int32_t ssq_n; float ssq_inv_dim;
  const float* ibias; int64_t ibias_ld; int32_t ibias_div;
  const float* b2b_bias; const float* b2b_alpha;
  const float* qnorm_w; const float* knorm_w;
  int32_t n_q_end, n_k_end, qkv_period, norm_w_stride;
  const void* rope; int32_t rope_T, use_rope; float eps;   /* rope: [rope_T, 64] (cos, sin) float pairs */
  const void* xa_kv; int64_t xa_kv_ld; int32_t xa_v_col0, xa_Tk, xa_T;
  const uint8_t* xa_mask; float xa_scale_log2;
  /* per-clip B: item i multiplies rows (i / b_clip_div) * b_clip_rows + [0, n) of b, which then has
   * ceil(a_items / b_clip_div) * b_clip_rows rows of b_cols visible columns at pitch b_ld (0: the run list's K) */
  int32_t b_clip_rows, b_clip_div;
  int64_t b_cols, b_ld;
  /* fused cross-attention writes its probabilities [rows, xa_Tk * heads] (bf16, column j * heads + h) here instead of O */
  void* xa_p; int64_t xa_p_ld;
} sab_test_gemm_desc;
int sab_test_gemm_ex(const sab_test_gemm_desc* d, void* stream);
/* The cross-attention fold (sam_audio_b200/csrc/xattn_fold.cuh) for `layers` layers:
 *   ut[l * ut_layer_stride + (b * d + n) * ldu + j * heads + h] = bf16(sum_c Wo_l[n, h*128 + c] * V_l[b*L + j, h*128 + c])
 * with d = heads * 128, Wo_l = wo_table[l] (a DEVICE array of layers pointers to [d, d] bf16) and
 * V_l[r, c] = kv[r * kv_ld + l * kv_layer_cols + v_col0 + c] (bf16, clips * L rows); columns [heads * L, ldu) are 0. */
int sab_test_xattn_fold(int layers, int clips, int L, int heads, const void* wo_table, const void* kv, int64_t kv_ld,
                        int64_t kv_layer_cols, int v_col0, void* ut, int ldu, int64_t ut_layer_stride, void* stream);
/* O = softmax(Q K^T / sqrt(128) + mask) V through the attention kernel; all [items*T, heads*128] bf16. */
int sab_test_attention(int items, int heads, int Tq, int Tk, const void* q, const void* k, const void* v,
                       const uint8_t* key_mask, void* o, void* stream);

/* Same, through the wgmma self-attention kernel (attention_tc2.cuh; Tq == Tk == T <= 256): shift_log2 > 0 =
 * single-pass softmax with that logit bound, < 0 = exact two-pass, 0 = the folded variant (q already scaled by
 * log2(e)/sqrt(128), logits bounded by 50); poly = pairs of every 8 exponentials evaluated on the FMA pipe
 * (0, 2, 3, 4; < 0: default). */
int sab_test_attention_tc2(int items, int heads, int T, const void* q_bf16, const void* k_bf16, const void* v_bf16,
                           const uint8_t* key_mask, void* o_bf16, float shift_log2, int poly, void* stream);

/* Same, through the wgmma streaming self-attention kernel (attention_stream_tc.cuh; any T, the engine uses it for
 * T > 256): shift_log2 < 0 = exact online softmax, >= 0 = the bounded variant (q already scaled by log2(e)/sqrt(128),
 * every |logit| <= shift_log2 <= 50 in the log2 domain; 0 stands for 50); poly as above. */
int sab_test_attention_stream(int items, int heads, int T, const void* q_bf16, const void* k_bf16, const void* v_bf16,
                              const uint8_t* key_mask, void* o_bf16, float shift_log2, int poly, void* stream);

/* The SIMT kernels of the DiT, codec and T5 paths, each through the launch helper the engine itself calls (same kernels,
 * grids and variant choice).  Every argument rule is checked before any CUDA call; a refusal returns non-zero with the rule
 * in sab_last_error().  All pointers are device addresses; fp32 unless stated.
 *
 * Fused RMSNorm + adaLN modulate (rmsnorm_mod_kernel<d/128>, d/128 in {2,4,8,12,16,20,22,24,32}), x [M, d]:
 *   out[m, :] = bf16(x[m,:] * rsqrt(mean(x[m,:]^2) + eps) * w * (1 + scale[b,:]) + shift[b,:]),  b = m / rows_per_item,
 *   shift / scale rows b at b * mod_ld (0: one row for all); reverse = 1 walks the rows last first (same values). */
int sab_test_rmsnorm_mod(int M, int d, const float* x, const float* w, const float* shift, const float* scale,
                         int64_t mod_ld, int rows_per_item, float eps, int reverse, void* out_bf16, void* stream);
/* GroupNorm(1 group) + SiLU (gn_stats_kernel + gn_silu_kernel) of `items` slabs x [items, n_per_item] (C channels
 * innermost): y = bf16(silu((x - mean) * rsqrt(var + eps) * gamma[c] + beta[c])), mean / biased var over the slab. */
int sab_test_group_norm_silu(int items, int64_t n_per_item, int C, const float* x, const float* gamma, const float* beta,
                             float eps, void* y_bf16, void* stream);
/* Time features of R = B * cand sequences; each output may be NULL (its kernel is skipped):
 *   tfreq [R, 256] bf16 = (cos, sin)(time[r] * exp(-ln(1e4) k / 128)), k < 128          (tfreq_kernel)
 *   mem_in [R/cand * L, d] bf16 = mem_base + (cos, sin)(time[b*cand] * exp(-ln(1e4) k / (d/2)))   (mem_time_kernel)
 *   mod [n_layers, R, 6, d] = tables[l] + t0[r] ([6, d] rows); fin [R, 2, d] = ftable + t[r]   (build_mod_kernel)
 *   cs [2 n_layers, R, d] = norm_w[k] * (1 + mod[k/2, r, 3(k%2) + 1]); shift [2 n_layers, R, d] bf16 = bf16(mod[k/2, r,
 *   3(k%2)])                                                                               (norm_tables_kernel) */
int sab_test_time_features(int R, int cand, int d, int n_layers, int L, const float* time, void* tfreq_bf16,
                           const float* mem_base, void* mem_in_bf16, const float* tables, const float* t0, const float* ftable,
                           const float* t, float* mod, float* fin, const float* norm_w, float* cs, void* shift_bf16,
                           void* stream);
/* Conditioning finish of sab_prepare for M = B * cand * T sequence rows (flags: SAB_PREP_NO_VIDEO_TERM, SAB_PREP_NO_ANCHORS):
 *   vconst = LayerNorm(vid_bias) * ln_w + ln_b (eps 1e-5)                                   (ln_vector_kernel)
 *   anchor_table [n_anchor, d] = anchor_embed [n_anchor, anchor_dim] @ anchor_proj [d, anchor_dim]^T   (small_abt_kernel)
 *   cond[m] = cond_clip[c] + tanh(gate_v) * (vproj ? LayerNorm(vproj[c]) * ln_w + ln_b : vconst)
 *             + tanh(gate_a) * anchor_table[anchor_ids[b, anchor_align[c]]]                   (cond_finish_kernel)
 *   with clip b = m / T / cand, clip row c = b * T + m % T; cond == cond_clip (in place) exactly when cand == 1. */
int sab_test_cond_finish(int B, int cand, int T, int d, float* cond, const float* cond_clip, const float* vproj,
                         const float* ln_w, const float* ln_b, const float* vid_bias, float* vconst, const float* gate_v,
                         const float* anchor_embed, const float* anchor_proj, int n_anchor, int anchor_dim,
                         float* anchor_table, const int64_t* anchor_ids, int n_ids, const int64_t* anchor_align,
                         const float* gate_a, int flags, void* stream);
/* RoPE table (rope_table_kernel): out [T, hd/2] (cos, sin) float pairs of pos * theta^(-2i/hd). */
int sab_test_rope_table(int T, int hd, float theta, float* out, void* stream);
/* The codec's 1-channel end layers; variant -1 = the engine's choice, 0 = the generic kernel, 1 = the register kernel.
 *  which 0, encoder.block.0 (enc_conv0{,_reg}_kernel): in = wav [items, S], w [C, 7], bias [C], alpha [C]:
 *    x_out [items, S, C] = bias[c] + sum_k w[c, k] wav[t + k - 3] (zero outside [0, S)); a_out bf16 = bf16(Snake_alpha(x_out))
 *  which 1, decoder last conv (dec_last_kernel, dec_last_reg_kernel<C/32> for C = 64, 96, 128): in = a bf16 [items, S, C],
 *    w [C, 7], bias [1]:  wav_out [items, S] = tanh(bias + sum_{k,c} w[c, k] a[t + k - 3, c]). */
int sab_test_codec_end(int which, int variant, int items, int64_t S, int C, const void* in, const float* w,
                       const float* bias, const float* alpha, float* x_out, void* a_out_bf16, float* wav_out, void* stream);
/* Cross-attention through the engine's dispatcher (xattn_small_kernel for Tk <= 16, attention_kernel above), the `cand`
 * query items of a clip sharing its text: O[i] = softmax(Q[i] K[i/cand]^T / sqrt(128) + mask[i/cand]) V[i/cand];
 * q, o [items*Tq, heads*128], k, v [items/cand*Tk, heads*128] bf16, key_mask [items/cand, Tk] (1 = attend) or NULL. */
int sab_test_attention_cross(int items, int heads, int Tq, int Tk, int cand, const void* q, const void* k, const void* v,
                             const uint8_t* key_mask, void* o, void* stream);
/* T5LayerNorm (t5_norm_kernel): y = x * rsqrt(mean(x^2) + eps) * w, x [rows, d]; out_bf16 and / or out_f32 (NULL: skipped). */
int sab_test_t5_norm(int64_t rows, int d, const float* x, const float* w, float eps, void* out_bf16, float* out_f32,
                     void* stream);
/* T5 self-attention of sab_t5_forward (t5_bias_table_kernel + t5_attention_kernel), 1 <= L <= 512:
 *   bias [H, 2L-1] = rel_bias_w[rel_bucket[delta], h] (rel_bias_w [buckets, H]);
 *   out[b*L + i, h*64 + c] = bf16(sum_j softmax_j(q_i . k_j + bias[h, j - i + L - 1], mask[b, j]) v_j[c]),
 *   q | k | v = qkv [B*L, 3*H*64] bf16 column blocks; no 1/sqrt(d) scaling. */
int sab_test_t5_attention(int B, int L, int H, const void* qkv, const float* rel_bias_w, const int32_t* rel_bucket,
                          float* bias, const uint8_t* mask, void* out_bf16, void* stream);

/* Time tiling of long clips in the codec (decoder != 0: sab_decode, else sab_encode) for a clip of T latent frames under
 * the current workspace budget: halo_frames = latent frames of context an output frame needs on each side, derived from
 * the codec's layer list; tile_frames = length of the tiles the clip is cut into, 0 when it runs whole. */
int sab_codec_tiling(sab_engine* e, int decoder, int T, int* halo_frames, int* tile_frames);

/* Visual prompting, frame pre-processing.  replaces: PerceptionEncoder.get_transform (vision_encoder.py:91-113) =
 * torchvision Resize((S, S), BICUBIC, antialias) on uint8 frames, x / 255, Normalize(0.5, 0.5).
 * frames [n_frames, 3, H, W] uint8 (device), workspace [n_frames, 3, H, S] fp32 (device), out [n_frames, 3, S, S] fp32.
 * Engine-independent (no weights). */
int sab_preprocess_frames(const uint8_t* frames, int n_frames, int H, int W, int out_size, float* workspace, float* out,
                          void* stream);
/* Long recordings, cross-fade of overlapping windows.  replaces: nothing — the reference has no windowing (its RoPE table
 * ends at max_positions, rope.py:152); SAMAudio.separate() solves a batch longer than the table as windows of Tw frames
 * and blends them with this (DESIGN.md section 3).  Engine-independent (no weights).
 *  win_latent [n_win, Tw, 256] fp32; per window (device arrays): win_seq = destination sequence in [0, Bc),
 *  win_start = its first frame, win_flags = SAB_WIN_FIRST | SAB_WIN_LAST (first / last window of its clip);
 *  starts may be negative or past T, so latent can be a frame range of a longer timeline (streams pass starts relative
 *  to the first frame they blend);
 *  latent [Bc, T, 256] fp32 out, every frame written:
 *    latent[s, t] = sum_k w_k x_k[t - start_k] / sum_k w_k over the windows k of s covering t, ascending k, fp32;
 *    w = min(ramp_in, ramp_out) at local position j, ramp_in = min(1, (j + 0.5) / ramp) (1 for a first window),
 *    ramp_out = min(1, (Tw - j - 0.5) / ramp) (1 for a last window); frames no window covers are 0. */
#define SAB_WIN_FIRST 1
#define SAB_WIN_LAST 2
int sab_blend_windows(const float* win_latent, int n_win, int Tw, const int32_t* win_seq, const int32_t* win_start,
                      const uint8_t* win_flags, int ramp, float* latent, int Bc, int T, void* stream);
/* Resampling.  replaces: torchaudio.functional.resample (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99), which
 * the reference's processor applies to files; streams and SAMAudio.resample() use it to bring audio at any rate to the
 * codec's rate and back (DESIGN.md section 3).  With g = gcd(orig, new), o = orig / g, n = new / g, output
 * q = m * n + j (j < n) is y[q] = sum_{k < K} w[j][k] * x[m * o + lo[j] + k], a K-term fp32 FMA chain in ascending k;
 * input samples outside [0, length) are zero and the output length is ceil(n * length / o).  orig == new is the
 * identity (K = 1, w = 1).  The table of each rate pair is built on first use and kept, counted in sab_workspace_bytes,
 * until sab_destroy.  One call runs every segment in one launch; an output's bits depend only on the signal and the
 * table, never on how the outputs are split into segments.
 *  Each segment: rates in [8000, 192000], 1 <= channels <= 8; input [channels, in_count] at channel stride
 *  in_channel_stride holds signal samples [in_first, in_first + in_count), and the mono signal is their channel mean
 *  (summed in ascending channel order, then divided by channels); length < 0 = not known yet, in which case only
 *  negative indices read as zero; outputs [out_first, out_first + out_count) go to out (contiguous fp32).  Every input
 *  index an output reads inside [0, length) must lie in the buffer.  Every rule is checked on the host before any CUDA
 *  call; the descriptors go to the device asynchronously on `stream` (calls of one engine must be ordered on one
 *  stream).  Not for graph capture. */
typedef struct sab_resample_seg {
  int32_t struct_bytes;     /* = sizeof(sab_resample_seg), checked first */
  int32_t orig_rate, new_rate, channels;
  const float* in;
  int64_t in_channel_stride, in_first, in_count;
  int64_t length;
  float* out;
  int64_t out_first, out_count;
} sab_resample_seg;
int sab_resample(sab_engine* e, const sab_resample_seg* segs, int n_segs, void* stream);
/* Host-only: the table sab_resample uses for a rate pair: *K taps, lo [n] (n = new / gcd) and, when w is not NULL,
 * w [n, K] fp32 (cap = floats w holds).  lo and w may be NULL to query K alone. */
int sab_resample_taps(int orig_rate, int new_rate, int64_t cap, int* K, int* lo, float* w);
/* Multichannel stems.  replaces: nothing — this goes beyond the reference, which is mono (its examples separate the
 * channel mean); streams with keep_channels and SAMAudio.spread_channels() use it (DESIGN.md section 3).  At the
 * codec's rate, with N = 2048, hop a = 512, the periodic Hann window w[n] = 0.5 - 0.5 cos(2 pi n / N) and frame j >= 0
 * covering samples [j a - 3 a, j a + a): M_j[k] = (|T_j[k]|^2 + d) / (|T_j[k]|^2 + |R_j[k]|^2 + 2 d), d = 1e-10, from the
 * rfft of the windowed mono target T and residual R; target_c[s] = (2/3) sum_j w[s - start_j] irfft(M_j X_c,j)[s -
 * start_j] over the four frames covering s, ascending j, with X_c,j the rfft of the windowed channel c; residual_c[s] =
 * x_c[s] - target_c[s] (one fp32 subtraction).  Samples outside a signal's known range are zero.  One call runs every
 * segment in one launch; an output's bits depend only on its inputs, never on how the outputs are split into segments.
 *  Each segment: 1 <= channels <= 8; target / residual hold samples [tr_first, tr_first + tr_count) of the mono stems
 *  (tr_length = their length, < 0 = not known yet); mix [channels, mix_count] at mix_channel_stride holds samples
 *  [mix_first, mix_first + mix_count) of the channels (mix_length likewise, at most tr_length when both are known);
 *  outputs [out_first, out_first + out_count) go to out_target / out_residual [channels, out_count] at
 *  out_channel_stride, and lie below tr_length when it is known.  Every input index an output reads must lie in its
 *  window or past its signal's known end.  Every rule is checked on the host before any CUDA call; the descriptors go
 *  to the device asynchronously on `stream` (calls of one engine must be ordered on one stream).  Not for graph
 *  capture. */
typedef struct sab_spread_seg {
  int32_t struct_bytes;     /* = sizeof(sab_spread_seg), checked first */
  int32_t channels;
  const float* target;
  const float* residual;
  int64_t tr_first, tr_count, tr_length;
  const float* mix;
  int64_t mix_channel_stride, mix_first, mix_count, mix_length;
  float* out_target;
  float* out_residual;
  int64_t out_channel_stride, out_first, out_count;
} sab_spread_seg;
int sab_spread_channels(sab_engine* e, const sab_spread_seg* segs, int n_segs, void* stream);

/* host-only test seam: evaluation times of sab_solve's grid (method = SAB_ODE_*), in evaluation order */
int sab_test_solver_grid(int method, int n_steps, int cap, int* n_evals, float* times);
/* host-only test seam: tap window start / count / normalised weights ([out_size, cap], zero padded) of one axis */
int sab_test_aa_taps(int in_size, int out_size, int cap, int* taps, int* lo, int* cnt, float* w);

#ifdef __cplusplus
}
#endif
#endif /* SAMAUDIO_B200_H */
