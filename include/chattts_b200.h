/*
 * chattts_b200 - C ABI of the H100-native (sm_90a) ChatTTS hot paths.
 *
 * The reference (2noise/ChatTTS) has no FFI boundary: its seams are Python objects
 * (SURVEY.md 8b).  This header is the boundary a maintainer binds from Python with
 * ctypes (see INTEGRATION.md); every entry point names the reference interface it
 * replaces.  Conventions:
 *   - plain C types, raw *device* pointers + sizes + a cudaStream_t passed as void*;
 *     no torch types; the caller owns every buffer it passes in;
 *   - int return: 0 = ok, negative = error, message via ctb_last_error() (thread local);
 *   - one handle per device per model; a handle is not re-entrant, different handles are;
 *   - nothing here ever runs on the CPU: if no CUDA device is usable, calls fail.
 */
#ifndef CHATTTS_B200_H
#define CHATTTS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTB_OK 0
#define CTB_ERR_ARG (-1)
#define CTB_ERR_CUDA (-2)
#define CTB_ERR_STATE (-3)
#define CTB_ERR_NOMEM (-4)

#define CTB_ABI_VERSION 4

/* ---- library ------------------------------------------------------------------- */
int ctb_abi_version(void);
const char* ctb_last_error(void);
/* number of kernels this library has launched in this process (bench "gpu_launches") */
uint64_t ctb_launch_count(void);

/* ---- GPT decode loop: replaces ChatTTS/model/gpt.py:315-618 (GPT.generate) ------ */

/* Model shape.  Mirrors the fields of the HF LlamaConfig the reference reads
 * (gpt.py:52,75; SURVEY.md quirk Q22) plus the Embed sizes (embed.py:8-35). */
typedef struct ctb_gpt_config {
  int32_t hidden_size;        /* 768  */
  int32_t intermediate_size;  /* 3072 */
  int32_t num_layers;         /* 20   */
  int32_t num_heads;          /* 12   */
  int32_t num_kv_heads;       /* 12 (GQA group = num_heads / num_kv_heads) */
  int32_t head_dim;           /* 64   */
  int32_t num_vq;             /* 4    */
  int32_t num_audio_tokens;   /* 626  */
  int32_t num_text_tokens;    /* 21178 */
  int32_t max_positions;      /* 4096: rows of the RoPE table */
  float rms_eps;              /* 1e-6 */
  int32_t max_batch;          /* rows this handle can decode at once */
  int32_t max_context;        /* prompt + generated tokens per row (KV pages are sized from it) */
} ctb_gpt_config;

/* Element offsets (in floats) of every tensor inside the packed fp32 weight blob the
 * caller uploads (one cudaMalloc / one NCCL broadcast).  Per-layer tensors are at
 * layer0 + l * layer_stride + <field>. Row-major [out_features, in_features], i.e. the
 * nn.Linear layout of the checkpoint (SURVEY.md 8b state-dict names). */
typedef struct ctb_gpt_layout {
  int64_t layer0, layer_stride;
  int64_t wqkv;      /* [(Hq + 2*Hkv)*hd, d]  q rows, then k rows, then v rows */
  int64_t wo;        /* [d, Hq*hd] */
  int64_t wgate_up;  /* [2*I, d]  gate rows then up rows */
  int64_t wdown;     /* [d, I] */
  int64_t ln1, ln2;  /* [d] each */
  int64_t final_norm;  /* [d] */
  int64_t head_code;   /* [num_vq*num_audio, d]  weight-norm already folded (embed.py:23-35) */
  int64_t head_text;   /* [num_text, d]          weight-norm already folded */
  int64_t emb_code;    /* [num_vq*num_audio, d] */
  int64_t emb_text;    /* [num_text, d] */
  int64_t rope_cos;    /* [max_positions, hd]  host-built exactly like HF LlamaRotaryEmbedding */
  int64_t rope_sin;    /* [max_positions, hd] */
  int64_t total;       /* floats in the blob */
} ctb_gpt_layout;

int ctb_gpt_layout_query(const ctb_gpt_config* cfg, ctb_gpt_layout* out);

/* Sampling tail: gpt.py:487-508 + processors.py:18-58 + HF TopP/TopK warpers.
 * Order: temperature -> repetition penalty -> top-p -> top-k -> [greedy mask] ->
 * (step < min_new: EOS ban) -> softmax -> argmax(p / q)  (== torch.multinomial).
 * Ties: the top-p and top-k cuts are value thresholds, so every token equal to the smallest kept value is kept.  At
 * the top-p cut HF removes tied tokens by their position in torch.sort's output, an order among equal values that is
 * not defined; the kept set here contains HF's and differs from it only in tokens equal to the cut value.  -0.0 and
 * +0.0 are equal values. */
typedef struct ctb_sampler_config {
  float temperature[8];     /* per codebook (row r uses temperature[r % rows_per_item]) */
  float top_p;              /* <0: warper absent (gen_logits top_P=None) */
  int32_t top_k;            /* <=0: warper absent; else the number kept, used as given: HF's TopKLogitsWarper has
                               already taken max(top_k, its own min_tokens_to_keep) */
  int32_t min_tokens_to_keep; /* top-p's (TopPLogitsWarper.min_tokens_to_keep; 3 at processors.py:45) */
  int32_t penalty_on;       /* 0: no CustomRepetitionPenaltyLogitsProcessorRepeat (penalty == 1) */
  float penalty_lut[32];    /* penalty ** count for count = 0..past_window, built by the host
                               with the same torch.pow call as processors.py:28 */
  int32_t past_window;      /* 16 */
  int32_t penalty_max_ids;  /* rows >= this get no penalty (processors.py:24-27 quirk) */
  int32_t greedy;           /* 1: keep only the row arg-max before softmax (bench config C2);
                               2: arg-max over the non-EOS tokens (EOS removed as well) */
  int32_t eos_token;
  int32_t min_new_token;
  float top_p_removed_max;  /* float32(1 - top_P) evaluated by the host exactly like HF TopPLogitsWarper (python double
                               arithmetic, then the fp32 comparison `cum <= 1 - top_p`); used when has_removed_max != 0,
                               otherwise the kernel derives it from the fp32 top_p (ABI v1 behaviour) */
  int32_t has_removed_max;
  uint64_t philox_seed;     /* used only when q_noise == NULL (manual_seed=None path) */
} ctb_sampler_config;

typedef struct ctb_gpt ctb_gpt;

/* weights_dev: packed blob laid out per ctb_gpt_layout_query, already on the device and
 * kept alive by the caller for the life of the handle. */
int ctb_gpt_create(const ctb_gpt_config* cfg, const float* weights_dev, ctb_gpt** out);
int ctb_gpt_destroy(ctb_gpt* h);

/* Which decode step serves a static batch of B rows on this handle (ctb_gpt_begin with that B and infer_text): the
 * predicates the launch code uses, evaluated for B without touching the handle.  The choice depends on the device
 * (the one-kernel steps need 128 SMs or more; k_flow at most 191) and on the environment at ctb_gpt_create:
 * CTB_NO_FLOW, CTB_FLOW_MAX_BATCH, CTB_FLOW_NO_INK, CTB_NO_MEGA, CTB_MEGA_MAX_BATCH, CTB_GPT_TC, CTB_GPT_FMA.
 *   CTB_STEP_FLOW_INK  k_flow with the sampling tail inside, up to 64 steps per launch (audio rows, B <= 2)
 *   CTB_STEP_FLOW      k_flow, one step per launch, sampled by k_sample
 *   CTB_STEP_MEGA      k_step, the grid-barrier one-kernel step
 *   CTB_STEP_FMA       the per-layer FMA kernels, chained by programmatic dependent launch
 *   CTB_STEP_WGMMA     the per-layer wgmma 3xTF32 GEMM kernels
 * Returns one of these (all > 0), or CTB_ERR_ARG for a null handle or B outside [1, max_batch]. */
#define CTB_STEP_FLOW_INK 1
#define CTB_STEP_FLOW 2
#define CTB_STEP_MEGA 3
#define CTB_STEP_FMA 4
#define CTB_STEP_WGMMA 5
int ctb_gpt_step_kind(const ctb_gpt* h, int32_t B, int32_t infer_text);

/* Start one generate() call.  Replaces gpt.py:343-381 (buffer set-up) and the i == 0
 * iteration (prefill + first sample).
 *   emb_dev      [B, T0, d] fp32   prompt embeddings (Embed.forward output, embed.py:51-79)
 *   mask_dev     [B, T0]   uint8   attention_mask; every row's valid tokens must be a contiguous SUFFIX (left padding,
 *                                  tokenizer.py:79-110) with the last column valid - the host mirror checks it
 *   q_noise_dev  [rows, V] fp32    Exp(1) noise of the seeded torch generator (gpt.py:504-508),
 *                                  rows = B*num_vq (audio) or B (text); NULL => device Philox
 *   ids_out_dev  [B, max_new, num_vq] int32   sampled ids (text: id replicated, gpt.py:521-523)
 *   hiddens_out_dev [B, max_new, d] fp32 or NULL (return_hidden, gpt.py:435-436)
 * Runs the whole prompt and the first sampling step on `stream`; does not synchronise. */
int ctb_gpt_begin(ctb_gpt* h, int32_t B, int32_t T0, const float* emb_dev, const uint8_t* mask_dev,
                  const ctb_sampler_config* sampler, const float* q_noise_dev, int32_t max_new_token,
                  int32_t infer_text, int32_t* ids_out_dev, float* hiddens_out_dev, void* stream);

/* Enqueue up to n_steps more iterations of the loop gpt.py:394-596.  Steps after every row
 * has finished (gpt.py:592) are no-ops on the device.  Does not synchronise. */
int ctb_gpt_decode(ctb_gpt* h, int32_t n_steps, void* stream);

typedef struct ctb_gpt_status {
  int32_t steps_done;     /* loop iterations executed so far (incl. the first one) */
  int32_t all_finished;   /* finish.all() (gpt.py:592) */
  int32_t any_finished_first_step; /* i == 0 and finish.any() (gpt.py:527) */
  int32_t reserved;
} ctb_gpt_status;

/* Synchronises `stream`, then reports loop state and copies per-row results:
 *   end_idx_host[B] int32 (gpt.py:345,576-577), finish_host[B] uint8; either may be NULL. */
int ctb_gpt_status_query(ctb_gpt* h, ctb_gpt_status* out, int32_t* end_idx_host, uint8_t* finish_host,
                         void* stream);

/* Attention maps of the static batch in flight (the reference's return_attn=True: GenerationOutputs.attentions, eager
 * attention's softmax probabilities of every layer at every step), for query columns [q0, q0 + n): the whole prompt
 * (q0 = 0, n >= T0) and/or the fed tokens of steps 1, 2, ... (column T0 + i - 1 is step i's query, the id sampled at
 * step i - 1).  A query-only pass over the K / V the decode wrote: it changes no decode state, so it may run between
 * ctb_gpt_decode calls.  Enqueued on `stream` (it reads the mask and the rows' end_idx there); does not synchronise.
 *   emb_dev [B, n, hidden] fp32: the embeddings of columns q0 .. q0 + n - 1 (the prompt's, and ctb_gpt_embed_prompt
 *     of the generated ids); mask_dev [B, T0]: the ctb_gpt_begin mask.
 *   out_dev: the blocks of the steps of those columns, in order; step 0 [L, B, Hq, T0, T0], step i >= 1
 *     [L, B, Hq, 1, T0 + i] fp32, key columns as the reference's (left padding included).  A padded key column is 0, a
 *     padded prompt row is uniform (1 / T0) as eager attention gives a fully masked row, and a row's steps after its
 *     end_idx are 0 (the device appends no KV for a finished row).
 * CTB_ERR_STATE: no static batch in flight (no ctb_gpt_begin, or a slot engine owns the handle); CTB_ERR_ARG: B / T0
 * are not the batch's, or the columns are not whole steps among those the enqueued steps fed. */
int ctb_gpt_attention_maps(ctb_gpt* h, int32_t B, int32_t T0, int32_t q0, int32_t n, const float* emb_dev,
                           const uint8_t* mask_dev, float* out_dev, void* stream);

/* Teacher-forced scoring on the fp32 model: the log-probability of given tokens under a prompt, computed in one causal
 * prefill pass (the prefill kernels of ctb_gpt_begin, k_prefill_attn_tiled above 1,024 columns) instead of sampled.
 * Row b has a prompt of n_prompt[b] positions and n_given[b] given tokens; its P + n - 1 columns (the prompt, then the
 * given tokens but the last) are the last columns of its T, left padded.  For given token j of row b, the column before
 * it (P - 1 + j of the row) gives the raw head logits z (code heads, V = num_audio_tokens, q < num_vq; or the text
 * head, V = num_text_tokens, q = 0) and out = log softmax(z)[token] at temperature 1, the quantity
 * ctb_gpt_engine_logprobs returns for sampled ids, with the same kernel (k_token_logprob).
 *   emb_dev [B, T, hidden] fp32: each row's prompt embeddings then ctb_gpt_embed_prompt of its given tokens but the
 *     last, in its last P + n - 1 columns (the padded columns are not read into any scored value)
 *   n_prompt, n_given [B] (host): P >= 1, n >= 1, P + n - 1 <= T
 *   targets_dev [m, rpi] int32, m = sum of n_given, rows in order (rpi = num_vq, or 1 with infer_text); out_dev the
 *     same shape fp32.  An id outside [0, V) gives NaN for that entry alone.
 * Enqueued on `stream` after one synchronisation that uploads the row layout.  The pass takes the handle as
 * ctb_gpt_begin does: a static batch in flight ends (ctb_gpt_decode, ctb_gpt_status_query and
 * ctb_gpt_attention_maps return CTB_ERR_STATE until the next ctb_gpt_begin), and so does a slot engine with no work.
 * Errors: CTB_ERR_ARG for a null argument, B outside [1, max_batch], T outside [8, max_context] or a row that does
 * not fit T; CTB_ERR_STATE while a slot engine has a slot pending, running or with a prompt in progress (the handle
 * as it was). */
int ctb_gpt_score(ctb_gpt* h, int32_t B, int32_t T, const float* emb_dev, const int32_t* n_prompt,
                  const int32_t* n_given, const int32_t* targets_dev, int32_t infer_text, float* out_dev,
                  void* stream);

/* ctb_gpt_score, and for every scored position the n_top ids with the largest z and their log softmax(z), as
 * ctb_gpt_engine_top_logprobs describes (same kernel, k_token_top_logprobs, over the same logits rows):
 *   top_ids_dev [m, rpi, n_top] int32, top_lp_dev [m, rpi, n_top] fp32.
 * out_dev is bit-equal to ctb_gpt_score's.  Errors: those of ctb_gpt_score; CTB_ERR_ARG for a null top buffer or n_top
 * outside [1, 20]. */
int ctb_gpt_score_ex(ctb_gpt* h, int32_t B, int32_t T, const float* emb_dev, const int32_t* n_prompt,
                     const int32_t* n_given, const int32_t* targets_dev, int32_t infer_text, float* out_dev,
                     int32_t n_top, int32_t* top_ids_dev, float* top_lp_dev, void* stream);

/* ---- slot engine: continuous batching of audio-code generation (no reference counterpart; the reference serves
 * this with the vLLM fork behind Chat.load(use_vllm=True)).  The handle's rows become S independent slots; each holds
 * one request (one utterance) at its own point of generation, with its own sampling parameters, noise and max_new,
 * and produces exactly what ctb_gpt_begin / ctb_gpt_decode produce for that request alone (B = 1).  Requests enter
 * free slots between ctb_gpt_decode calls; ctb_gpt_decode is used unchanged (steps advance every running slot; with
 * no running slot they are no-ops).  ctb_gpt_begin returns the handle to static batches. */

#define CTB_SLOT_IDLE 0
#define CTB_SLOT_RUNNING 1
#define CTB_SLOT_FINISHED 2

/* Turn the handle into S slots (2 <= S <= max_batch), all idle.  Every slot owns a fixed KV page range of
 * max_context tokens (S x max_context tokens in all).  Engines of 9 <= S <= 64 slots run the wgmma step whatever the
 * handle's max_batch (CTB_GPT_FMA=1 keeps them on the PDL chain), building its state on a handle that lacks it; the
 * others run the PDL chain.
 *   ids_out_dev      [S, max_new_cap, num_vq] int32   slot b's tokens: ids_out_dev[b, 0 : end_idx[b]]
 *   hiddens_out_dev  [S, max_new_cap, d] fp32 or NULL  its last hidden states, same rows */
int ctb_gpt_engine_begin(ctb_gpt* h, int32_t S, int32_t max_new_cap, int32_t* ids_out_dev, float* hiddens_out_dev,
                         void* stream);

/* ctb_gpt_engine_begin with precision flags (flags = 0 is ctb_gpt_engine_begin).  The half-precision engine is the
 * model the reference serves with its vLLM fork (dtype "auto" runs a float32 checkpoint in float16), except that the
 * heads stay fp32 as in every reference mode:
 *   CTB_ENGINE_FP16_WEIGHTS  the four matrices of every layer are stored in fp16, rounded to nearest even: Wqkv and
 *                            [Wgate; Wup] after the fp32 fold of input_layernorm / post_attention_layernorm into
 *                            their columns (the activations then enter as x * rsqrt(mean(x^2) + eps)), Wo and Wdown as
 *                            they are.  Prefill uses the same rounded values.
 *   CTB_ENGINE_FP16_KV       K (after RoPE) and V are rounded to fp16 as they are appended; every attention, prompt
 *                            and decode, reads the rounded values.  K/V overflow is not checked (nor is it in the
 *                            reference's fp16 modes).
 * Embeddings, RMSNorm statistics, RoPE, activations, attention arithmetic, the heads, the sampler and the hidden
 * states in hiddens_out_dev stay fp32.  A flagged engine always runs the wgmma step with 16 (S <= 16), 32 (S <= 32) or
 * 64 padded rows and builds what the handle lacks for it; the fp16 copies (377.5 MB for the 20 layers, plus their 755 MB fp32
 * image read by the prefill GEMMs) are built by the first CTB_ENGINE_FP16_WEIGHTS engine and kept until
 * ctb_gpt_destroy.  The KV pool is sized in bytes and shared by every call on the handle.
 * Errors (CTB_ERR_ARG): unknown flag bits; S > 64 with a flag set; a flag set while CTB_GPT_FMA=1; a layer weight
 * (norm folded) with |w| > 65504, named by layer and matrix in ctb_last_error - the handle is left as it was. */
#define CTB_ENGINE_FP16_WEIGHTS 1
#define CTB_ENGINE_FP16_KV 2
int ctb_gpt_engine_begin_ex(ctb_gpt* h, int32_t S, int32_t max_new_cap, int32_t flags, int32_t* ids_out_dev,
                            float* hiddens_out_dev, void* stream);

/* Admit n requests into the idle or finished slots slots[0..n) (host array): prefill their prompts (token-parallel,
 * left padded, 8 <= T0 <= max_context - 1: pad shorter prompts with masked columns) into those slots and sample each
 * one's first token; no other slot's state, outputs or KV pages are touched.  Up to T0 = 1024 the prompt's attention is
 * the one ctb_gpt_begin's prefill runs, bit for bit; a wider admission runs a tiled causal attention (fp32 arithmetic,
 * results within float rounding of the column walk ctb_gpt_begin uses for such prompts, not bit-equal to it).  Which
 * one runs depends on T0 alone, and a prompt's results do not depend on the other prompts of its admission.
 *   emb_dev [n, T0, d] fp32, mask_dev [n, T0] uint8 (valid tokens a suffix of each row, as for ctb_gpt_begin)
 *   samplers[n] (host)   sampling parameters of each request (audio codes; penalty_max_ids applies to its own rows
 *                        0..num_vq-1, as in a batch of one)
 *   q_noise_dev          [n, num_vq, num_audio] fp32 Exp(1) rows of each request's seeded generator, or NULL: device
 *                        Philox from samplers[i].philox_seed
 *   max_new[n] (host)    tokens each request may generate (<= max_new_cap, T0 + max_new <= max_context)
 * Enqueued on `stream`; the host arrays may be released on return. */
int ctb_gpt_engine_admit(ctb_gpt* h, int32_t n, const int32_t* slots, int32_t T0, const float* emb_dev,
                         const uint8_t* mask_dev, const ctb_sampler_config* samplers, const float* q_noise_dev,
                         const int32_t* max_new, void* stream);

/* ctb_gpt_engine_admit for text requests (GPT.generate(infer_text=True) for a batch of one): the slots take text
 * tokens - emb_text input, the text head, one sampled row (temperature[0]; penalty_max_ids applies to row 0).  Text
 * and code slots decode in the same ctb_gpt_decode steps.  Each token is written to all num_vq columns of
 * ids_out_dev[b, n]; no hidden states are written for text slots.
 *   q_noise_dev  [n, num_text] fp32 Exp(1) rows of each request's seeded generator, or NULL: device Philox
 * Other arguments as for ctb_gpt_engine_admit. */
int ctb_gpt_engine_admit_text(ctb_gpt* h, int32_t n, const int32_t* slots, int32_t T0, const float* emb_dev,
                              const uint8_t* mask_dev, const ctb_sampler_config* samplers, const float* q_noise_dev,
                              const int32_t* max_new, void* stream);

/* Prefill columns [c0, c0 + n) of a prompt of T0 columns (8 <= T0 <= max_context - 1, every column valid, no padding)
 * into the idle or finished slot `slot`, whose KV pages hold columns [0, c0) from the earlier chunks of the same
 * prompt.  A prompt prefilled in chunks gives the same bits - KV pages, first token, and every later token and hidden
 * state - as the same prompt admitted by one ctb_gpt_engine_admit / _admit_text call: each chunk row runs the layers
 * as that call runs it, and its attention is the kernel that call would choose for T0 (not for n), over keys 0 .. its
 * position read from the pages.  c0, and n unless the chunk is the final one (c0 + n == T0), are multiples of
 * CTB_PREFILL_CHUNK_ALIGN, which keeps every row's GEMM tile and every query's attention tile where one call puts them.
 *   emb_dev [n, d] fp32  the chunk's prompt embeddings (columns c0 .. c0 + n - 1)
 *   text                 0: an audio-code request (ctb_gpt_engine_admit), 1: a text request (_admit_text)
 *   sampler (host), q_noise_dev ([num_vq, num_audio] or [1, num_text] fp32, or NULL), max_new: one request's, as for
 *                        those calls; read on the final chunk only (sampler may be NULL before it)
 * A chunk before the final one touches nothing but the slot's pages: the slot keeps its state (idle or finished), and
 * decode steps in between neither read nor append its pages.  The final chunk admits the request as those calls do:
 * the slot becomes pending and its first token is sampled.  The handle records each slot's prompt in progress (T0,
 * columns done); ctb_gpt_engine_admit / _admit_text / _cancel on the slot and ctb_gpt_engine_begin* drop it.
 * Enqueued on `stream` after one synchronisation (two on the final chunk); the host arguments may be released on return.
 * Errors leave the handle usable and the prompt in progress as it was:
 *   CTB_ERR_STATE  outside engine mode; a chunk that does not continue the slot's prompt in progress (other c0 or T0),
 *                  a first chunk with c0 != 0, or a slot that is running or pending
 *   CTB_ERR_ARG    a null argument; slot out of range; T0 outside [8, max_context - 1]; [c0, c0 + n) not inside
 *                  [0, T0); c0, or a non-final n, not a multiple of CTB_PREFILL_CHUNK_ALIGN; max_new outside
 *                  [1, max_new_cap] or T0 + max_new > max_context; on the final chunk, a sampler ctb_gpt_engine_admit
 *                  refuses */
#define CTB_PREFILL_CHUNK_ALIGN 128
int ctb_gpt_engine_prefill_chunk(ctb_gpt* h, int32_t slot, int32_t T0, int32_t c0, int32_t n, const float* emb_dev,
                                 int32_t text, const ctb_sampler_config* sampler, const float* q_noise_dev,
                                 int32_t max_new, void* stream);

/* Synchronises `stream`, then reports per-slot results (each array [S], any may be NULL): state_host CTB_SLOT_*,
 * end_idx_host tokens of the slot's request, finish_host 1 if it ended at EOS.  A finished slot with end_idx 0 and
 * finish 1 sampled EOS as its first token (gpt.py:527: the request ends empty).  out->steps_done counts decode steps
 * with at least one running slot; out->all_finished = no running slot. */
int ctb_gpt_engine_status(ctb_gpt* h, ctb_gpt_status* out, int32_t* state_host, int32_t* end_idx_host,
                          uint8_t* finish_host, void* stream);

/* Stop the requests in `slots` (host array of n distinct slot indices, 1 <= n <= S): a server whose client went away
 * frees the slot for the next request at once instead of decoding to EOS or max_new.  Enqueued on `stream`, no
 * synchronisation; the host array may be released on return.
 * A listed slot that is running or pending becomes CTB_SLOT_FINISHED with finish 0; its ids_out / hiddens_out rows
 * 0 .. end_idx-1 stay valid.  Idle and already finished slots are left as they are (not an error): the host cannot
 * know that a row did not finish on the device since its last status read.  Afterwards all_finished = no running
 * slot, so later ctb_gpt_decode steps with nothing running stay no-ops and do not count in steps_done.  A cancelled
 * slot takes a new request through ctb_gpt_engine_admit / _admit_text.
 * Errors: CTB_ERR_STATE outside engine mode; CTB_ERR_ARG for a null argument, n outside [1, S], a slot out of range
 * or repeated, or an engine of more than 1024 slots. */
int ctb_gpt_engine_cancel(ctb_gpt* h, int32_t n, const int32_t* slots, void* stream);

/* ---- KV pages on demand: a slot engine whose KV memory is a bounded pool shared by its slots.
 * ctb_gpt_engine_begin_ex with two differences: the pool holds pool_pages pages of every layer (one page: 16 tokens
 * of K and V, 2 x num_kv_heads x 16 x head_dim values per layer, fp32 or fp16 by CTB_ENGINE_FP16_KV), and no slot
 * owns any page.  Page 0 is the zero page: never handed out, always zero, and every block-table entry that maps no
 * page points at it, so a read of a position a slot does not own sees zeros.  The handle keeps the free list.
 * A request's results do not depend on which pages hold its KV: ctb_gpt_engine_admit / _admit_text /
 * _prefill_chunk / _cancel and ctb_gpt_decode keep their contracts, and the first three, and ctb_gpt_decode, refuse
 * (CTB_ERR_STATE, nothing enqueued) a slot whose pages do not cover the positions they are about to write.
 * With CTB_KV_POISON=1 in the environment at this call, the pool (all but the zero page) and every released page
 * are filled with quiet-NaN bits instead of zeros, so a read of a page a request does not own shows in its outputs.
 * Errors: those of ctb_gpt_engine_begin_ex; CTB_ERR_ARG for pool_pages < 2 or max_context over 8,192 tokens;
 * CTB_ERR_NOMEM if the pool does not fit. */
#define CTB_ERR_POOL (-5)
int ctb_gpt_engine_begin_paged(ctb_gpt* h, int32_t S, int32_t max_new_cap, int32_t flags, int32_t pool_pages,
                               int32_t* ids_out_dev, float* hiddens_out_dev, void* stream);

/* Map pages so that each slot slots[i] (host array of n distinct slots) holds positions [0, tokens[i]) (0 <= tokens[i]
 * <= max_context; a slot that holds them already is left as it is).  All or nothing: when the free list cannot cover
 * the whole call it returns CTB_ERR_POOL and the handle is unchanged.  Enqueued on `stream` (the new block-table
 * entries travel by value), no synchronisation.
 * Errors: CTB_ERR_STATE outside a paged engine; CTB_ERR_ARG for a null argument, n outside [1, S], a slot out of
 * range or repeated, or tokens outside [0, max_context]. */
int ctb_gpt_engine_reserve(ctb_gpt* h, int32_t n, const int32_t* slots, const int32_t* tokens, void* stream);

/* Return the pages of the idle or finished slots slots[0..n) to the free list and point their entries back at the
 * zero page (CTB_KV_POISON=1: the pages are filled with quiet-NaN bits).  Synchronises `stream` once to read the
 * slots' states.  Errors: CTB_ERR_STATE outside a paged engine, or for a slot that is running, pending or has a
 * prompt in progress (nothing is released); CTB_ERR_ARG as for ctb_gpt_engine_reserve. */
int ctb_gpt_engine_release(ctb_gpt* h, int32_t n, const int32_t* slots, void* stream);

/* The pool's pages as the block table maps them now: *in_use physical pages mapped, each counted once however many
 * slots map it, and *shared of them mapped by more than one block-table entry (shared prompts).  Host bookkeeping
 * only: no device work, no synchronisation.  Errors: CTB_ERR_STATE outside a paged engine; CTB_ERR_ARG for a null
 * argument. */
int ctb_gpt_engine_pages(ctb_gpt* h, int32_t* in_use, int32_t* shared);

/* A suspended slot's image in a pinned host buffer: this header, then the sections at the offsets it records. */
#define CTB_SLOT_IMAGE_MAGIC 0x4b565031u
typedef struct ctb_slot_image {
  uint32_t magic;
  int32_t prec;            /* the engine's CTB_ENGINE_FP16_* flags */
  int32_t seq_len, pos, end_idx, finish;
  int32_t n_gen;           /* tokens in the ids / hiddens sections */
  int32_t npages;          /* KV pages: positions [0, 16 * npages) of every layer */
  int32_t page_bytes;      /* one page of one layer */
  int32_t num_vq, hidden_size, noise_floats;
  int32_t has_hidden;      /* the hiddens section exists */
  int32_t row[8];          /* the slot's loop state (n_gen, step, state, max_new, has_noise, eos, text, -) */
  int32_t reserved[3];
  ctb_sampler_config sampler;
  uint64_t off_noise;      /* float[noise_floats]: the slot's Exp(1) rows */
  uint64_t off_ids;        /* int32[n_gen][num_vq] */
  uint64_t off_hiddens;    /* float[n_gen][hidden_size], if has_hidden */
  uint64_t off_kv;         /* [layer][npages] pages as the pool stores them */
  uint64_t bytes;          /* the whole image */
} ctb_slot_image;

/* Bytes of the image ctb_gpt_engine_suspend would write for the running slot `slot` now.  Synchronises `stream`.
 * Errors: CTB_ERR_STATE outside a paged engine or for a slot that is not running; CTB_ERR_ARG for a null argument
 * or a slot out of range. */
int ctb_gpt_engine_suspend_bytes(ctb_gpt* h, int32_t slot, uint64_t* bytes, void* stream);

/* Move the running slot `slot` out of the engine into host_buf (pinned host memory of host_bytes bytes, at least
 * ctb_gpt_engine_suspend_bytes): its KV for positions [0, seq_len) of every layer (k_kv_pack: one launch, 16-byte
 * stores straight into the mapped buffer), its loop state, sampler, noise row, seq_len / pos / finish / end_idx, and
 * its ids_out / hiddens_out rows 0 .. n_gen-1.  Its pages are then released and the slot becomes idle.  The header is
 * written before the call returns; the rest is enqueued on `stream` (synchronise it before reading them on the host).
 * Errors (the handle as it was): CTB_ERR_STATE outside a paged engine, for a slot that is not running or has a prompt
 * in progress; CTB_ERR_ARG for a null argument, a slot out of range, a buffer that is not pinned or too small. */
int ctb_gpt_engine_suspend(ctb_gpt* h, int32_t slot, void* host_buf, uint64_t host_bytes, void* stream);

/* Restore the image in host_buf into `slot` - any idle or finished slot whose pages already hold the image's
 * positions [0, seq_len) - and set it running (k_kv_unpack scatters the pages).  The request then continues exactly
 * as it would have without the move.  Enqueued on `stream` after one synchronisation; host_buf must stay alive until
 * the stream has passed this call.  Errors (the handle as it was): CTB_ERR_STATE outside a paged engine, for a slot
 * that is running, pending or has a prompt in progress, or whose pages do not cover the image; CTB_ERR_ARG for a null
 * argument, a slot out of range, a buffer that is not pinned or smaller than the image, or an image of another
 * engine shape (magic, precision, page, noise or hidden-state layout, max_new_cap). */
int ctb_gpt_engine_resume(ctb_gpt* h, int32_t slot, const void* host_buf, uint64_t host_bytes, void* stream);

/* ---- Shared prompts: a request whose prompt equals the one slot `src` was admitted with takes that slot's KV for
 * prompt columns [0, c0) instead of prefilling them.  Sets up slot `dst` as a prompt of T0 columns in progress with
 * [0, c0) done; the next call for it must be its final chunk, ctb_gpt_engine_prefill_chunk(dst, T0, c0, T0 - c0, ...),
 * which samples its first token with its own sampler and noise.  Its results are then bit for bit those of admitting
 * the request normally, provided the two prompts are equal: the handle cannot check that, and c0 being a chunk
 * boundary (CTB_PREFILL_CHUNK_ALIGN) is what makes the final chunk after [0, c0) equal a one-call admission.
 *   A fixed engine copies positions [0, c0) of every layer from src's pages to dst's (k_kv_copy, enqueued on
 *   `stream`).  A paged engine copies nothing: dst's block-table entries [0, c0 / 16) map src's pages, whose
 *   reference counts rise, and entries [c0 / 16, ceil(T0 / 16)) map pages of dst's own.  A page returns to the free
 *   list (and is poisoned under CTB_KV_POISON=1) when its last entry is released; ctb_gpt_engine_suspend releases the
 *   suspended slot's entries, so a resumed request holds private pages only.  No call writes a page that more than one
 *   entry maps: admissions, chunks, decode steps and resumes that would are refused with CTB_ERR_STATE.
 * `src` is a slot whose admitted prompt's KV is still in place: running, or finished and neither released nor given
 * another prompt, prefill or image since (a resumed request is no source).  Synchronises `stream` once to read both
 * slots' states.
 * Errors (the handle as it was): CTB_ERR_STATE outside a slot engine, when src holds no admitted prompt or one of fewer
 * than c0 positions, or when dst is running, pending, has a prompt in progress or (paged) has pages mapped;
 * CTB_ERR_ARG for src == dst, a slot out of range, T0 outside [8, max_context - 1], c0 that is not a positive
 * multiple of CTB_PREFILL_CHUNK_ALIGN below T0, or T0 and src's prompt width on different sides of 1,024 columns
 * (different prefill attention kernels); CTB_ERR_POOL (paged) when the free list cannot map dst's own pages. */
int ctb_gpt_engine_share_prompt(ctb_gpt* h, int32_t src, int32_t dst, int32_t T0, int32_t c0, void* stream);

/* ---- Token log-probabilities: attach logprobs_out_dev, [S, max_new_cap, num_vq] fp32 (device), to the slot engine
 * just begun.  From then on every sampler launch of the engine (admissions, final prefill chunks, decode steps, and the
 * decode graphs captured after this call) is followed by k_token_logprob, which writes, for every row it sampled,
 *   logprobs_out_dev[slot][n][q] = log softmax(z)[id]
 * where n is the index the id is written at in ids_out, q the codebook (text requests: q = 0 only) and z the fp32
 * head logits row the sampler read: the model's distribution at temperature 1, before the repetition penalty, top-P,
 * top-K and the min_new_token EOS ban.  The step that samples a terminating EOS writes no id, and its entry is not
 * part of the request's output.  The row max is taken in fp32, the denominator summed in double in a fixed order and
 * the result rounded once to fp32, so the same logits give the same bits.  Ids, hidden states and every other output
 * are those of the engine without the buffer.  No kernel reads the buffer: a suspended request's entries are not in
 * its ctb_slot_image, and the caller moves them with it.  The call zeroes the buffer on `stream`.  Every
 * ctb_gpt_engine_begin* starts without a buffer.
 * Errors (the handle as it was): CTB_ERR_ARG for a null argument; CTB_ERR_STATE outside a slot engine, or once the
 * engine has admitted, prefilled a chunk for or resumed a request. */
int ctb_gpt_engine_logprobs(ctb_gpt* h, float* logprobs_out_dev, void* stream);

/* ---- Top log-probabilities: attach ids_out_dev [S, max_new_cap, num_vq, n_top] int32 and lp_out_dev (same shape,
 * fp32), both device, to the slot engine just begun.  From then on every sampler launch of the engine (where
 * ctb_gpt_engine_logprobs' kernel runs, after it when both are attached) is followed by k_token_top_logprobs, which
 * writes, for every row it sampled, at [slot][n][q][k] for k < n_top:
 *   ids_out_dev = the k-th id of z's order (z descending, the smaller id first among equal z)
 *   lp_out_dev  = (float)((double)(z[id] - max) - log(den))
 * with z, n and q as in ctb_gpt_engine_logprobs, and max and den computed as k_token_logprob computes them: an entry
 * whose id is the sampled one equals that call's value bit for bit.  Ids, hidden states and log-probabilities are those
 * of the engine without the buffers; no kernel reads them, and a suspended request's entries are not in its
 * ctb_slot_image.  The call zeroes both buffers on `stream`.  Every ctb_gpt_engine_begin* starts without them.
 * Errors (the handle as it was): CTB_ERR_ARG for a null argument or n_top outside [1, 20]; CTB_ERR_STATE outside a
 * slot engine, or once the engine has admitted, prefilled a chunk for or resumed a request. */
int ctb_gpt_engine_top_logprobs(ctb_gpt* h, int32_t n_top, int32_t* ids_out_dev, float* lp_out_dev, void* stream);

/* Measurement hook for bench.py's roofline: launches ONE kernel kind once per layer on the
 * state left by the last generate call (kind 0 qkv, 1 attention, 2 o-proj, 3 gate/up, 4 down;
 * 5 = heads, 6 = sampler, 7 = one decode step as ONE kernel launch (k_flow / k_step), 8 = 16 decode steps in one
 * k_flow launch with the sampling tail inside).  7 and 8 advance the generation.  No reference counterpart. */
int ctb_gpt_profile_kernel(ctb_gpt* h, int32_t kind, void* stream);

/* Profiling aid: with CTB_MEGA_TRACE=1 in the environment at ctb_gpt_create, the one-kernel decode step records
 * a %globaltimer stamp (ns) of CTA 0 after every grid barrier of the most recent step; copies up to n of them. */
int ctb_gpt_debug_trace(ctb_gpt* h, unsigned long long* host_out, int n);

/* Prompt embedding mix: replaces Embed.forward (ChatTTS/model/embed.py:51-79).
 *   ids_dev [B, T, num_vq] int64 (tokenizer output), text_mask_dev [B, T] uint8, tables inside the packed blob of `h`;
 *   out_dev [B, T, d] fp32: text positions get emb_text[ids[...,0]], the others sum_q emb_code[q][ids[...,q]].
 * Reads only the handle's weights and configuration, so unlike the other calls on a handle it may run in one thread
 * while another thread drives the handle (a server embeds new prompts while its slot engine decodes); it must keep
 * writing nothing the handle owns. */
int ctb_gpt_embed_prompt(ctb_gpt* h, const int64_t* ids_dev, const uint8_t* text_mask_dev, int32_t B, int32_t T,
                         float* out_dev, void* stream);

/* Stand-alone sampling tail over caller-provided logits (minimum slice of SURVEY.md 7.2;
 * same kernel the decode loop uses).
 *   logits_dev [rows, V] fp32 (not modified); gen_ids_dev [rows/rpi, gen_stride, rpi] int32 with
 *   n_gen tokens generated so far; out_idx_dev [rows] int32. */
int ctb_sample(const float* logits_dev, int32_t rows, int32_t V, int32_t rows_per_item,
               const ctb_sampler_config* sampler, const float* q_noise_dev, const int32_t* gen_ids_dev,
               int32_t gen_stride, int32_t n_gen, int32_t step, int32_t* out_idx_dev, void* stream);

/* Stand-alone token log-probability (the kernel ctb_gpt_engine_logprobs launches): for each of `rows` rows of
 * logits_dev [rows, V] fp32, out_dev[r] = log softmax(logits_dev[r])[ids_dev[r]] (NaN for an id outside [0, V)),
 * with the arithmetic described there.  Enqueued on `stream`.  Errors: CTB_ERR_ARG for a null argument, rows < 1 or
 * V < 1. */
int ctb_token_logprobs(const float* logits_dev, int32_t rows, int32_t V, const int32_t* ids_dev, float* out_dev,
                       void* stream);

/* Stand-alone top log-probabilities (the kernel ctb_gpt_engine_top_logprobs launches): for each of `rows` rows of
 * logits_dev [rows, V] fp32, ids_out_dev [rows, n_top] int32 and lp_out_dev [rows, n_top] fp32 as described there.
 * Enqueued on `stream`.  Errors: CTB_ERR_ARG for a null argument, n_top outside [1, 20], rows < 1, V < n_top or a row
 * over 200 KiB (V > 51,200). */
int ctb_token_top_logprobs(const float* logits_dev, int32_t rows, int32_t V, int32_t n_top, int32_t* ids_out_dev,
                           float* lp_out_dev, void* stream);

/* ---- token -> waveform: replaces ChatTTS/core.py:512-539 (_decode_to_wavs) ------ */

typedef struct ctb_convstack_config {
  int32_t idim, odim, hidden, n_layer, bn_dim, kernel, dilation; /* dvae.py:131-172 */
  int32_t out_dim;    /* DVAE(dim=...) : out_conv input channels; 100 mel bins out (dvae.py:236) */
  int32_t vq_dim, vq_groups, vq_residual; /* GFSQ (dvae.py:69-97); vq_dim = 0: no VQ layer */
  int32_t vq_levels;  /* low byte: levels per dim (5); bits 8..15: residual scale base (0 => levels-1);
                       * bit 16 (encode only): 1 = do NOT bound() the projected input before the first residual stage */
} ctb_convstack_config;

typedef struct ctb_vocos_config {
  int32_t input_channels, dim, intermediate_dim, num_layers, n_fft, hop_length; /* config.py:74-121 */
} ctb_vocos_config;

typedef struct ctb_decoder ctb_decoder;

/* Element offsets inside the packed decoder blob (DVAE stack + out_conv + coef [+ VQ]). */
int64_t ctb_dvae_blob_floats(const ctb_convstack_config* cfg);
int64_t ctb_vocos_blob_floats(const ctb_vocos_config* cfg);

int ctb_decoder_create(const ctb_convstack_config* dvae_cfg, const float* dvae_blob_dev,
                       const ctb_vocos_config* vocos_cfg, const float* vocos_blob_dev, int32_t max_batch,
                       int32_t max_tokens, ctb_decoder** out);
int ctb_decoder_destroy(ctb_decoder* h);

/* DVAE.forward(mode="decode") (dvae.py:276-297).  in_layout selects what in_dev holds:
 *   0: hidden path, channels-first [B, C, T] fp32 (C = 2*idim) - the layout DVAE.__call__ receives
 *      from core.py:519-534;
 *   1: hidden path, token-major [B, T, C] fp32 - what ctb_gpt_* writes to hiddens_out_dev; the
 *      frame doubling of dvae.py:281-287 is then a pure re-interpretation (no copy);
 *   2: code path, ids [B, num_vq, T] int32 through GFSQ._embed (dvae.py:87-97).
 *   mel_dev [B, 100, 2T] fp32 channels-first, or NULL to keep the mel only inside the handle
 *   (time-major) for a following ctb_vocos_decode(mel_dev = NULL). */
int ctb_dvae_decode(ctb_decoder* h, const void* in_dev, int32_t in_layout, int32_t B, int32_t T, float* mel_dev,
                    void* stream);
/* Vocos.decode (core.py:505-510): mel [B,100,F] channels-first (NULL: the mel left in the handle by
 * the last ctb_dvae_decode) -> wav [B, hop*(F-1)] fp32 */
int ctb_vocos_decode(ctb_decoder* h, const float* mel_dev, int32_t B, int32_t F, float* wav_dev, void* stream);
/* Ragged batch of independent token sequences -> waveforms.  Row k is decoded exactly as ctb_dvae_decode +
 * ctb_vocos_decode decode it alone (B = 1, T = n_tokens[k]): bit-identical, on either back end (CTB_DECODER_FMA).
 *   kind 1: rows_dev[k] -> [n_k, 2*idim] fp32 token-major hidden states (e.g. a slice of the engine's hiddens_out),
 *           16-byte aligned
 *   kind 2: rows_dev[k] -> [n_k, num_vq] int32 token-major codes (e.g. a slice of the engine's ids_out)
 *   rows_dev, n_tokens: host arrays of B entries, n_k >= 1; they may be released on return
 *   wav_dev [B, wav_ld] fp32: row k receives hop*(2 n_k - 1) samples; the rest of the row is not written.
 * CTB_ERR_ARG when B * 2 * max(n_k) exceeds the handle's max_batch * 2 * max_tokens frames.  Needs both weight sets. */
int ctb_decode_rows(ctb_decoder* h, int32_t kind, int32_t B, const void* const* rows_dev, const int32_t* n_tokens,
                    float* wav_dev, int64_t wav_ld, void* stream);

/* ---- waveform -> codes: replaces DVAE.forward(mode="encode") (ChatTTS/model/dvae.py:265-274), i.e. ------
 * MelSpectrogramFeatures (dvae.py:175-206; n_fft 1024, hop 256, 100 mel bins, center/reflect, power 1, log(clip 1e-5))
 * -> / coef -> downsample_conv (dvae.py:231-236) -> encoder DVAEDecoder stack (dvae.py:131-172) -> GFSQ.forward indices
 * (dvae.py:102-128).  Caller: Chat.sample_audio_speaker (core.py:179-180) and the automatic speaker sample of
 * multi-sentence infer() (core.py:435-453).
 * cfg: idim = DVAE dim (512), odim = vq_dim (1024), hidden / n_layer / bn_dim / kernel / dilation of the encoder stack,
 * vq_* as for the decoder.  The blob holds the analysis window, the mel filterbank, coef, the two downsample convs,
 * the stack and the FSQ project_in matrices (order: chattts_b200/decoder.py::pack_dvae_encoder). */
typedef struct ctb_encoder ctb_encoder;
int64_t ctb_dvae_encoder_blob_floats(const ctb_convstack_config* enc_cfg);
int ctb_dvae_encoder_create(const ctb_convstack_config* enc_cfg, const float* blob_dev, int64_t max_samples,
                            ctb_encoder** out);
int ctb_dvae_encoder_destroy(ctb_encoder* h);
/* wav_dev [n_samples] fp32 (24 kHz) -> ids_dev [G*R, T] int32 with T = (n_samples / 256 + 1) / 2 written to the HOST
 * int *n_tokens_out; ids_capacity_tokens = tokens ids_dev (and margin_dev) can hold per code row.
 * mel_dev (optional) [100, n_samples / 256 + 1]: the log-mel BEFORE the division by coef is not kept; this is mel / coef.
 * margin_dev (optional) [G*R, T] fp32: distance of the closest pre-rounding value to a rounding edge (0 .. 0.5), the
 * decision margin the parity tests use to tell a real mismatch from fp32 reordering noise. */
int ctb_dvae_encode(ctb_encoder* h, const float* wav_dev, int64_t n_samples, int32_t* ids_dev,
                    int32_t ids_capacity_tokens, int32_t* n_tokens_out, float* mel_dev, float* margin_dev, void* stream);
/* Ragged batch of independent waveforms -> codes in one pass.  Row k is encoded exactly as ctb_dvae_encode encodes it
 * alone: its ids and margins are bit-identical, on either back end (CTB_DECODER_FMA).
 *   wavs_dev, n_samples: host arrays of B entries (they may be released on return); wavs_dev[k] -> n_k fp32 samples at
 *                        24 kHz on the device, read in place (e.g. a row of ctb_decode_rows' wav_dev)
 *   ids_dev [B, G*R, ids_ld] int32; margin_dev (optional) the same shape in fp32
 *   n_tokens_out: host array of B entries, T_k = (n_k / 256 + 1) / 2
 * CTB_ERR_ARG for B < 1, a null argument, n_k <= 512, n_k > max_samples or T_k > ids_ld.  The handle's scratch grows on
 * demand to B rows of the widest one (CTB_ERR_NOMEM if it cannot).  Not re-entrant with the handle's other calls. */
int ctb_dvae_encode_rows(ctb_encoder* h, int32_t B, const float* const* wavs_dev, const int64_t* n_samples,
                         int32_t* ids_dev, int32_t ids_ld, int32_t* n_tokens_out, float* margin_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CHATTTS_B200_H */
