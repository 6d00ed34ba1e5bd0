// extern "C" entry points for hot path 1 (see include/chattts_b200.h).
#include <stdarg.h>

#include <map>
#include <mutex>
#include <vector>

#include <cudaTypedefs.h>

#define CTB_GPT_KERNELS_IMPL
#include "gpt_kernels.cuh"
#include "tc_decode.cuh"
#include "mega.cuh"
#include "flow.cuh"
#include "prefill.cuh"
#include "tc_gemm.cuh"
#include "kv_pool.cuh"

namespace ctb {

thread_local char g_err[512] = {0};
std::atomic<uint64_t> g_launches{0};

int set_err(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int g_num_sms = 132;  // set from the device in ctb_gpt_create


static int bt_for(int B) {
  int bt = 1;
  while (bt < B && bt < 32) bt <<= 1;
  return bt;
}

}  // namespace ctb

using namespace ctb;
using ctb::g_num_sms;

// What the host knows of one slot of a slot engine (ctb_gpt::slot); all zero when ctb_gpt_engine_begin* starts it
struct SlotRecord {
  int chunk_T0, chunk_done;  // prompt being prefilled in chunks: its width (0: none), the columns in the slot's pages
  int pr_len, pr_W;  // admitted prompt its pages hold (a share's source): its positions (0: none), the kernels' width
  int pages;         // block-table entries mapped (paged engines)
  int hi;            // positions its request may hold after the steps enqueued so far (0: none)
  int cap;           // and at most: prompt + max_new - 1
};

struct ctb_gpt {
  ctb_gpt_config cfg;
  ctb_gpt_layout lay;
  const float* W;
  int pages_per_row, nsplit_max, bpad_max;
  // device state
  float *x, *qbuf, *attn, *mlp, *logits, *kv, *part;
  int *block_table, *seq_len, *pos, *counter, *end_idx;
  int32_t* idx;
  uint8_t *active, *finish;
  LoopState* st;
  size_t kv_layer_elems;  // elements (fp32, or fp16 for a CTB_ENGINE_FP16_KV engine) of one layer's share of the pool
  size_t kv_bytes;        // size of the pool
  int bt_B; size_t bt_per_row;  // shape the uploaded block table was built for
  // per generate() call
  int B, T0, max_new, infer_text, started;
  ctb_sampler_config sampler;
  const float* q_noise;
  const float* emb;
  const uint8_t* mask;
  int32_t* ids_out;
  float* hiddens_out;
  cudaGraphExec_t graph_exec;
  uint64_t graph_kernels;  // kernel nodes captured in graph_exec
  cudaStream_t cap_stream;
  // ---- tensor-core decode path (tc_decode.cuh)
  bool use_tc, tc_ready;
  int tc_min_batch;
  // ---- batched prefill (prefill.cuh): lazily allocated
  bool pf_enabled;
  float *gw_hi, *gw_lo;            // tf32 hi / lo copies of the per-layer weight region of the blob
  float *pf_resid, *pf_xn, *pf_qkv, *pf_q, *pf_attn, *pf_gu, *pf_h, *pf_ones, *pf_zeros;
  int *pf_npre, *pf_nvalid;
  uint8_t* pf_mask;                // [pf_rows] a prompt chunk's column mask (all ones)
  size_t pf_rows;                  // capacity (B * T0) of the pf_* activation buffers
  bool mega_ok;      // one-kernel decode step (mega.cuh), built for B <= 8
  int mega_max_batch; // batches that use it (default 4; CTB_MEGA_MAX_BATCH overrides)
  unsigned* bar;     // its grid-barrier counter
  unsigned long long* trace;  // CTB_MEGA_TRACE=1: per-phase timestamps of the last step
  bool flow_ok;      // dataflow decode step (flow.cuh), built for B <= 4
  int flow_R;        // replicas of the broadcast exchange regions (CTB_FLOW_R)
  int flow_l2_ahead;  // weight tasks prefetched one layer ahead into L2 (CTB_FLOW_L2_AHEAD)
  int flow_max_batch; // batches that use it (CTB_FLOW_MAX_BATCH, default 1)
  bool flow_no_ink;   // CTB_FLOW_NO_INK: k_flow runs one step per launch, sampled by k_sample / k_finalize
  unsigned long long* flow_arena;
  unsigned* flow_epoch;
  int steps_enqueued;  // loop iterations enqueued since ctb_gpt_begin (host-side bound for ctb_gpt_decode)
  float *tc_wqkv, *tc_wgu, *tc_heads_code, *tc_heads_text;  // permuted / norm-folded weight copies
  float *x_hi, *x_lo, *attn_hi, *attn_lo, *h_hi, *h_lo;      // [tc_rows][K] tf32-split activations
  int tc_rows;                                               // 32, or 64 on a handle whose max_batch exceeds 32
  CUtensorMap *m_wqkv, *m_wo, *m_wgu, *m_wd;                 // [layers] host arrays
  CUtensorMap m_hcode, m_htext;
  CUtensorMap m_x[3][2], m_attn[3][2], m_h[3][2];            // [npad16|32|64][hi|lo] (npad 64: tc_rows == 64 only)
  bool use_graph;
  // ---- slot engine (ctb_gpt_engine_*): B = S slots, max_new = the per-slot capacity of ids_out / hiddens_out
  int engine;                 // 1 between ctb_gpt_engine_begin and the next ctb_gpt_begin
  int phase;                  // rows the heads / sampler / finalize serve: RS_RUNNING (decode) or RS_PENDING (admission)
  RowState* rows;             // [Bpad] per-slot loop state
  ctb_sampler_config* cfgs;   // [max_batch] per-slot sampling parameters
  float* eng_noise;           // [max_batch, noise_stride(h)] per-slot Exp(1) rows ([num_vq, num_audio] or [1, num_text])
  int* eng_slot;              // [max_batch] slot of each prompt of the admission being prefilled
  float* eng_text_logits;     // [max_batch, num_text] text-head logits of text slots (h->logits holds the code rows)
  int32_t* eng_text_idx;      // [max_batch] the text sampler's ids
  // 1 while a text slot may be pending or running (set by ctb_gpt_engine_admit_text, cleared by the status read that
  // finds none): steps carry the text head / sampler launches only then, from their own captured graph
  int eng_text;
  cudaGraphExec_t graph_exec_text;
  uint64_t graph_kernels_text;
  float* eng_logprobs;        // [S, max_new, num_vq] token log-probabilities (ctb_gpt_engine_logprobs), or nullptr
  int eng_served;             // 1 once the engine has admitted, chunked or resumed a request
  int eng_top_n;              // N of the top log-probability buffers (ctb_gpt_engine_top_logprobs), 0 without them
  int32_t* eng_top_ids;       // [S, max_new, num_vq, N] the N most likely ids of every sampled row
  float* eng_top_lp;          // [S, max_new, num_vq, N] their log-probabilities
  std::vector<SlotRecord> slot;  // [S] host-side record of each slot
  // ---- half-precision slot engine (ctb_gpt_engine_begin_ex)
  int prec;                   // CTB_ENGINE_FP16_* bits of the current engine (0 for fp32 engines and generate())
  bool tc_base;               // tensor-core activation scratch, head copies and their tensor maps exist (tc_setup_base)
  __half *w16_qkv, *w16_wo, *w16_gu, *w16_wd;  // fp16 decode copies of the layer matrices (built once, kept)
  CUtensorMap *m16_wqkv, *m16_wo, *m16_wgu, *m16_wd;
  float* gw16;                // the same rounded values as fp32 in the blob's layer layout: prefill W_hi
  float* pf_wzero;            // prefill W_lo of the rounded weights (exactly zero), as large as the largest matrix
  // ---- on-demand KV pages (ctb_gpt_engine_begin_paged); pg_pages == 0: the fixed page ranges of kv_reserve
  int pg_pages;               // pages in the pool, page 0 the zero page
  bool pg_poison;             // CTB_KV_POISON=1 at begin: free pages hold quiet-NaN bits
  std::vector<int> pg_free;   // free pages, taken from the back
  std::vector<int> pg_bt;     // [S][pages_per_row] host copy of the block table
  std::vector<int> pg_ref;    // [pool_pages] block-table entries that map each page (above 1: a shared prompt's)
  int pg_shared;              // pages whose count is above 1
  char* pg_stage;             // KV_STAGE_BYTES of device staging for suspend / resume (allocated by the first one)
  // ---- teacher-forced scoring (ctb_gpt_score): built or grown by the first call that needs them, then kept
  float *sc_head_hi[2], *sc_head_lo[2];  // tf32 hi / lo copies of head_code [num_vq * V, d] and head_text [V, d]
  float *sc_xn, *sc_logits;   // [SCORE_ROWS, d] final-normed scored columns; [SCORE_ROWS, widest head used] logits
  size_t sc_logits_cols;
  int* sc_src;                // [sc_src_cap] prefill row of each scored column
  size_t sc_src_cap;
};

static size_t kv_elem_bytes(const ctb_gpt* h) { return (h->prec & CTB_ENGINE_FP16_KV) ? 2 : 4; }
// layer l's share of the KV pool, in the element type the current call's kernels use
static float* kv_layer(const ctb_gpt* h, int l) {
  return reinterpret_cast<float*>(reinterpret_cast<char*>(h->kv) + (size_t)l * h->kv_layer_elems * kv_elem_bytes(h));
}
static size_t page_elems(const ctb_gpt* h) { return (size_t)2 * h->cfg.num_kv_heads * kPageTokens * h->cfg.head_dim; }
static size_t page_bytes(const ctb_gpt* h) { return page_elems(h) * kv_elem_bytes(h); }  // one page of one layer

// floats of one slot's noise in the engine's buffer: room for a code request's or a text request's rows
static size_t noise_stride(const ctb_gpt* h) {
  return std::max((size_t)h->cfg.num_vq * h->cfg.num_audio_tokens, (size_t)h->cfg.num_text_tokens);
}

static int check_engine(const ctb_gpt* h) {
  return h->engine ? CTB_OK : set_err(CTB_ERR_STATE, "ctb_gpt_engine_begin has not been called");
}

static int check_paged(const ctb_gpt* h) {
  if (!h->engine || !h->pg_pages) return set_err(CTB_ERR_STATE, "not a paged slot engine (ctb_gpt_engine_begin_paged)");
  return CTB_OK;
}

static int check_slot_list(const ctb_gpt* h, int n, const int32_t* slots) {
  if (n < 1 || n > h->B) return set_err(CTB_ERR_ARG, "n=%d outside [1,%d]", n, h->B);
  std::vector<char> seen((size_t)h->B, 0);
  for (int i = 0; i < n; ++i) {
    if (slots[i] < 0 || slots[i] >= h->B || seen[slots[i]])
      return set_err(CTB_ERR_ARG, "slot %d out of range or repeated", slots[i]);
    seen[slots[i]] = 1;
  }
  return CTB_OK;
}

static int check_slot(const ctb_gpt* h, int slot) {
  if (slot < 0 || slot >= h->B) return set_err(CTB_ERR_ARG, "slot %d outside [0,%d)", slot, h->B);
  if (h->slot[slot].chunk_T0) return set_err(CTB_ERR_STATE, "slot %d has a prompt in progress", slot);
  return CTB_OK;
}

// prompts over 1,024 columns take the tiled prefill attention; every slot owns max_context tokens of pages
static int check_T0(const ctb_gpt* h, int T0) {
  if (T0 < 8 || T0 > h->cfg.max_context - 1)
    return set_err(CTB_ERR_ARG, "T0=%d outside [8,%d]: left-pad shorter prompts to 8", T0, h->cfg.max_context - 1);
  return CTB_OK;
}

static int check_max_new(const ctb_gpt* h, int b, int T0, int max_new) {
  if (max_new < 1 || max_new > h->max_new || T0 + max_new > h->cfg.max_context)
    return set_err(CTB_ERR_ARG, "slot %d: max_new=%d (capacity %d) with T0=%d exceeds max_context=%d", b, max_new,
                   h->max_new, T0, h->cfg.max_context);
  return CTB_OK;
}

// every slot's RowState (bpad_max: an admission writes them all back); synchronises s and the caller's copies on it
static int read_rows(ctb_gpt* h, std::vector<RowState>& rows, cudaStream_t s) {
  rows.resize((size_t)h->bpad_max);
  CTB_CUDA(cudaMemcpyAsync(rows.data(), h->rows, sizeof(RowState) * rows.size(), cudaMemcpyDeviceToHost, s));
  CTB_CUDA(cudaStreamSynchronize(s));
  return CTB_OK;
}

static int check_not_generating(const RowState& r, int b) {
  if (r.state == RS_RUNNING || r.state == RS_PENDING) return set_err(CTB_ERR_STATE, "slot %d is still generating", b);
  return CTB_OK;
}

// CTB_ERR_STATE unless a paged engine's slot b has pages for positions [0, hi)
static int check_covers(const ctb_gpt* h, int b, int hi) {
  const int held = h->slot[b].pages * kPageTokens;
  if (h->pg_pages && held < hi)
    return set_err(CTB_ERR_STATE, "slot %d: its pages hold %d positions, the call writes up to %d", b, held, hi);
  return CTB_OK;
}

// CTB_ERR_STATE unless a paged engine's slot b has pages for the positions [lo, hi) a call writes, none of them mapped
// by another entry too (kernels never write a shared prompt's pages, ctb_gpt_engine_share_prompt)
static int check_writes(const ctb_gpt* h, int b, int lo, int hi) {
  if (!h->pg_pages) return CTB_OK;
  if (int rc = check_covers(h, b, hi)) return rc;
  for (int k = lo / kPageTokens; k * kPageTokens < hi && k < h->slot[b].pages; ++k)
    if (h->pg_ref[h->pg_bt[(size_t)b * h->pages_per_row + k]] > 1)
      return set_err(CTB_ERR_STATE, "slot %d: positions [%d,%d) reach page entry %d, which is shared", b, lo, hi, k);
  return CTB_OK;
}

extern "C" int ctb_abi_version(void) { return CTB_ABI_VERSION; }
extern "C" const char* ctb_last_error(void) { return g_err; }
extern "C" uint64_t ctb_launch_count(void) { return g_launches.load(); }

extern "C" int ctb_gpt_layout_query(const ctb_gpt_config* c, ctb_gpt_layout* o) {
  if (!c || !o) return set_err(CTB_ERR_ARG, "null argument");
  const int64_t d = c->hidden_size, I = c->intermediate_size, hd = c->head_dim;
  const int64_t nq = (int64_t)c->num_heads * hd, nkv = (int64_t)c->num_kv_heads * hd;
  int64_t off = 0;
  o->wqkv = off; off += (nq + 2 * nkv) * d;
  o->wo = off; off += d * nq;
  o->wgate_up = off; off += 2 * I * d;
  o->wdown = off; off += d * I;
  o->ln1 = off; off += d;
  o->ln2 = off; off += d;
  o->layer_stride = off;
  o->layer0 = 0;
  off = o->layer_stride * c->num_layers;
  o->final_norm = off; off += d;
  o->head_code = off; off += (int64_t)c->num_vq * c->num_audio_tokens * d;
  o->head_text = off; off += (int64_t)c->num_text_tokens * d;
  o->emb_code = off; off += (int64_t)c->num_vq * c->num_audio_tokens * d;
  o->emb_text = off; off += (int64_t)c->num_text_tokens * d;
  o->rope_cos = off; off += (int64_t)c->max_positions * hd;
  o->rope_sin = off; off += (int64_t)c->max_positions * hd;
  o->total = off;
  return CTB_OK;
}

template <typename T>
static int dalloc(T** p, size_t n) {
  CTB_CUDA(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
  CTB_CUDA(cudaMemset(*p, 0, n * sizeof(T)));
  return CTB_OK;
}

namespace ctb {
__global__ void k_build_tc_weight(const float* __restrict__ W, const float* __restrict__ scale, float* __restrict__ out,
                                  int rows, int K, int mode, int qk_rows, int hd, int I) {
  const int r = blockIdx.x;
  if (r >= rows) return;
  int pr = r;
  if (mode == 1 && r < qk_rows) {
    const int h = r / hd, j = r % hd, half = hd / 2;
    pr = h * hd + (j < half ? 2 * j : 2 * (j - half) + 1);
  } else if (mode == 2) {
    pr = (r < I) ? 2 * r : 2 * (r - I) + 1;
  }
  for (int k = threadIdx.x; k < K; k += blockDim.x)
    out[(size_t)pr * K + k] = scale ? __fmul_rn(W[(size_t)r * K + k], scale[k]) : W[(size_t)r * K + k];
}

__global__ void k_build_tc_weight16(const float* __restrict__ W, const float* __restrict__ scale, __half* __restrict__ out16,
                                    float* __restrict__ out32, int rows, int K, int mode, int qk_rows, int hd, int I,
                                    int* __restrict__ bad) {
  const int r = blockIdx.x;
  if (r >= rows) return;
  int pr = r;  // the row permutation of k_build_tc_weight
  if (mode == 1 && r < qk_rows) {
    const int h = r / hd, j = r % hd, half = hd / 2;
    pr = h * hd + (j < half ? 2 * j : 2 * (j - half) + 1);
  } else if (mode == 2) {
    pr = (r < I) ? 2 * r : 2 * (r - I) + 1;
  }
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float v = scale ? __fmul_rn(W[(size_t)r * K + k], scale[k]) : W[(size_t)r * K + k];
    if (fabsf(v) > 65504.f) *bad = 1;
    const __half w = __float2half_rn(v);
    out16[(size_t)pr * K + k] = w;
    out32[(size_t)r * K + k] = __half2float(w);
  }
}
}  // namespace ctb

static int encode_map_2d(CUtensorMap* m, const void* base, uint64_t rows, uint64_t K, uint32_t box_rows,
                         bool f16 = false) {
  static PFN_cuTensorMapEncodeTiled_v12000 enc = nullptr;
  if (!enc) {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return set_err(CTB_ERR_CUDA, "cuTensorMapEncodeTiled unavailable");
    enc = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fp);
  }
  // fp32: 128-byte rows of 32 k, swizzled for wgmma; fp16 (weights the kernel widens): dense 64-byte rows
  const cuuint64_t dims[2] = {K, rows};
  const cuuint64_t strides[1] = {K * (f16 ? 2 : 4)};
  const cuuint32_t box[2] = {32, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base),
                   dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   f16 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_err(CTB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return CTB_OK;
}

// the shared-memory attribute of k_tc_dec<EPI, NPAD, CS, PREC> for the 16-, 32- and 64-row tiles
template <int EPI, int CS, int PREC = 0>
static int set_tc_attr() {
  constexpr bool w16 = (PREC & TD_W16) != 0;
  int rc;
  if ((rc = ensure_smem_attr((const void*)k_tc_dec<EPI, 16, CS, PREC>, TdCfg<16, w16>::SMEM_BYTES)) ||
      (rc = ensure_smem_attr((const void*)k_tc_dec<EPI, 32, CS, PREC>, TdCfg<32, w16>::SMEM_BYTES)))
    return rc;
  return ensure_smem_attr((const void*)k_tc_dec<EPI, 64, CS, PREC>, TdCfg<64, w16>::SMEM_BYTES);
}

// cluster sizes of the split-K (K slices per 128-row tile)
constexpr int CS_QKV = 4, CS_O = 8, CS_GU = 2, CS_DOWN = 8, CS_HEADS = 4;

static int tc_setup_base(ctb_gpt* h);

// the fp32 wgmma step: norm-folded, permuted fp32 copies of Wqkv and [Wgate; Wup] (Wo and Wdown are read in place)
static int tc_setup(ctb_gpt* h) {
  const ctb_gpt_config& c = h->cfg;
  const ctb_gpt_layout& L = h->lay;
  const size_t d = c.hidden_size, I = c.intermediate_size;
  const size_t nqkv = (size_t)(c.num_heads + 2 * c.num_kv_heads) * c.head_dim;
  int rc;
  if ((rc = tc_setup_base(h))) return rc;
  if ((rc = dalloc(&h->tc_wqkv, (size_t)c.num_layers * nqkv * d))) return rc;
  if ((rc = dalloc(&h->tc_wgu, (size_t)c.num_layers * 2 * I * d))) return rc;
  h->m_wqkv = new CUtensorMap[c.num_layers]; h->m_wo = new CUtensorMap[c.num_layers];
  h->m_wgu = new CUtensorMap[c.num_layers]; h->m_wd = new CUtensorMap[c.num_layers];
  const int qk_rows = (c.num_heads + c.num_kv_heads) * c.head_dim;
  for (int l = 0; l < c.num_layers; ++l) {
    const float* Wl = h->W + L.layer0 + (int64_t)l * L.layer_stride;
    float* wq = h->tc_wqkv + (size_t)l * nqkv * d;
    float* wg = h->tc_wgu + (size_t)l * 2 * I * d;
    k_build_tc_weight<<<(unsigned)nqkv, 256>>>(Wl + L.wqkv, Wl + L.ln1, wq, (int)nqkv, (int)d, 1, qk_rows, c.head_dim, 0);
    k_build_tc_weight<<<(unsigned)(2 * I), 256>>>(Wl + L.wgate_up, Wl + L.ln2, wg, (int)(2 * I), (int)d, 2, 0, 0, (int)I);
    if ((rc = encode_map_2d(&h->m_wqkv[l], wq, nqkv, d, 128))) return rc;
    if ((rc = encode_map_2d(&h->m_wo[l], Wl + L.wo, d, (size_t)c.num_heads * c.head_dim, 128))) return rc;
    if ((rc = encode_map_2d(&h->m_wgu[l], wg, 2 * I, d, 128))) return rc;
    if ((rc = encode_map_2d(&h->m_wd[l], Wl + L.wdown, d, I, 128))) return rc;
  }
  CTB_CUDA(cudaDeviceSynchronize());
  if ((rc = set_tc_attr<DE_QKV, CS_QKV>()) || (rc = set_tc_attr<DE_OPROJ, CS_O>()) ||
      (rc = set_tc_attr<DE_GATEUP, CS_GU>()))
    return rc;
  return set_tc_attr<DE_DOWN, CS_DOWN>();
}

// what every wgmma step shares: the tf32-split activation scratch (32 rows; 64 on a handle whose max_batch exceeds 32,
// for engines of up to 64 slots), the fp32 norm-folded head copies and the tensor maps over them
static int tc_setup_base(ctb_gpt* h) {
  if (h->tc_base) return CTB_OK;
  const ctb_gpt_config& c = h->cfg;
  const ctb_gpt_layout& L = h->lay;
  const size_t d = c.hidden_size, I = c.intermediate_size;
  int rc;
  if ((rc = dalloc(&h->tc_heads_code, (size_t)c.num_vq * c.num_audio_tokens * d))) return rc;
  if ((rc = dalloc(&h->tc_heads_text, (size_t)c.num_text_tokens * d))) return rc;
  const size_t R = c.max_batch > 32 ? 64 : 32;
  if ((rc = dalloc(&h->x_hi, R * d))) return rc;
  if ((rc = dalloc(&h->x_lo, R * d))) return rc;
  if ((rc = dalloc(&h->attn_hi, R * d))) return rc;
  if ((rc = dalloc(&h->attn_lo, R * d))) return rc;
  if ((rc = dalloc(&h->h_hi, R * I))) return rc;
  if ((rc = dalloc(&h->h_lo, R * I))) return rc;
  h->tc_rows = (int)R;
  const int nhc = c.num_vq * c.num_audio_tokens;
  k_build_tc_weight<<<nhc, 256>>>(h->W + L.head_code, h->W + L.final_norm, h->tc_heads_code, nhc, (int)d, 0, 0, 0, 0);
  k_build_tc_weight<<<c.num_text_tokens, 256>>>(h->W + L.head_text, h->W + L.final_norm, h->tc_heads_text,
                                                c.num_text_tokens, (int)d, 0, 0, 0, 0);
  CTB_CUDA(cudaDeviceSynchronize());
  if ((rc = encode_map_2d(&h->m_hcode, h->tc_heads_code, nhc, d, 128))) return rc;
  if ((rc = encode_map_2d(&h->m_htext, h->tc_heads_text, c.num_text_tokens, d, 128))) return rc;
  for (int n = 0; n < (R > 32 ? 3 : 2); ++n) {
    const uint32_t npad = 16u << n;
    if ((rc = encode_map_2d(&h->m_x[n][0], h->x_hi, R, d, npad))) return rc;
    if ((rc = encode_map_2d(&h->m_x[n][1], h->x_lo, R, d, npad))) return rc;
    if ((rc = encode_map_2d(&h->m_attn[n][0], h->attn_hi, R, d, npad))) return rc;
    if ((rc = encode_map_2d(&h->m_attn[n][1], h->attn_lo, R, d, npad))) return rc;
    if ((rc = encode_map_2d(&h->m_h[n][0], h->h_hi, R, I, npad))) return rc;
    if ((rc = encode_map_2d(&h->m_h[n][1], h->h_lo, R, I, npad))) return rc;
  }
  if ((rc = set_tc_attr<DE_HEADS, CS_HEADS>())) return rc;
  h->tc_base = true;
  return CTB_OK;
}

static void fp16_free(ctb_gpt* h) {
  void* ptrs[] = {h->w16_qkv, h->w16_wo, h->w16_gu, h->w16_wd, h->gw16, h->pf_wzero};
  for (void* p : ptrs) if (p) cudaFree(p);
  h->w16_qkv = h->w16_wo = h->w16_gu = h->w16_wd = nullptr; h->gw16 = h->pf_wzero = nullptr;
  delete[] h->m16_wqkv; delete[] h->m16_wo; delete[] h->m16_wgu; delete[] h->m16_wd;
  h->m16_wqkv = h->m16_wo = h->m16_wgu = h->m16_wd = nullptr;
}

// The half-precision engine's weights, built by the first such engine and kept for the life of the handle: fp16
// decode copies of the four layer matrices (Wqkv and [Wgate; Wup] norm-folded in fp32 first, then rounded; Wo and
// Wdown rounded) and the same values as fp32 for the prefill GEMMs.  A value outside fp16's range refuses them.
static int fp16_setup(ctb_gpt* h) {
  if (h->w16_qkv) return CTB_OK;
  const ctb_gpt_config& c = h->cfg;
  const ctb_gpt_layout& L = h->lay;
  const size_t d = c.hidden_size, I = c.intermediate_size, nq = (size_t)c.num_heads * c.head_dim;
  const size_t nqkv = (size_t)(c.num_heads + 2 * c.num_kv_heads) * c.head_dim;
  const int nl = c.num_layers, qk_rows = (c.num_heads + c.num_kv_heads) * c.head_dim;
  int rc;
  if ((rc = tc_setup_base(h))) return rc;
  int* bad = nullptr;
  if ((rc = dalloc(&h->w16_qkv, nl * nqkv * d)) || (rc = dalloc(&h->w16_wo, nl * d * nq)) ||
      (rc = dalloc(&h->w16_gu, nl * 2 * I * d)) || (rc = dalloc(&h->w16_wd, nl * d * I)) ||
      (rc = dalloc(&h->gw16, (size_t)L.layer_stride * nl)) ||
      (rc = dalloc(&h->pf_wzero, std::max(std::max(nqkv * d, d * nq), std::max(2 * I * d, d * I)))) ||
      (rc = dalloc(&bad, (size_t)4 * nl))) {
    fp16_free(h);
    if (bad) cudaFree(bad);
    return rc;
  }
  for (int l = 0; l < nl; ++l) {
    const float* Wl = h->W + L.layer0 + (int64_t)l * L.layer_stride;
    float* gl = h->gw16 + (int64_t)l * L.layer_stride;
    k_build_tc_weight16<<<(unsigned)nqkv, 256>>>(Wl + L.wqkv, Wl + L.ln1, h->w16_qkv + l * nqkv * d, gl + L.wqkv,
                                                 (int)nqkv, (int)d, 1, qk_rows, c.head_dim, 0, bad + 4 * l);
    k_build_tc_weight16<<<(unsigned)d, 256>>>(Wl + L.wo, nullptr, h->w16_wo + l * d * nq, gl + L.wo, (int)d, (int)nq, 0,
                                              0, 0, 0, bad + 4 * l + 1);
    k_build_tc_weight16<<<(unsigned)(2 * I), 256>>>(Wl + L.wgate_up, Wl + L.ln2, h->w16_gu + l * 2 * I * d,
                                                    gl + L.wgate_up, (int)(2 * I), (int)d, 2, 0, 0, (int)I, bad + 4 * l + 2);
    k_build_tc_weight16<<<(unsigned)d, 256>>>(Wl + L.wdown, nullptr, h->w16_wd + l * d * I, gl + L.wdown, (int)d, (int)I,
                                              0, 0, 0, 0, bad + 4 * l + 3);
  }
  std::vector<int> hbad((size_t)4 * nl);
  const cudaError_t e = cudaMemcpy(hbad.data(), bad, hbad.size() * sizeof(int), cudaMemcpyDeviceToHost);
  cudaFree(bad);
  if (e != cudaSuccess) { fp16_free(h); return set_err(CTB_ERR_CUDA, "fp16 weight copies: %s", cudaGetErrorString(e)); }
  static const char* names[4] = {"self_attn.qkv (x input_layernorm)", "self_attn.o_proj",
                                 "mlp.gate_up (x post_attention_layernorm)", "mlp.down_proj"};
  for (int i = 0; i < 4 * nl; ++i)
    if (hbad[i]) {
      fp16_free(h);
      return set_err(CTB_ERR_ARG, "fp16 engine: layer %d %s has a weight with |w| > 65504 (outside fp16's range)", i / 4,
                     names[i % 4]);
    }
  h->m16_wqkv = new CUtensorMap[nl]; h->m16_wo = new CUtensorMap[nl];
  h->m16_wgu = new CUtensorMap[nl]; h->m16_wd = new CUtensorMap[nl];
  for (int l = 0; l < nl; ++l) {
    if ((rc = encode_map_2d(&h->m16_wqkv[l], h->w16_qkv + l * nqkv * d, nqkv, d, 128, true)) ||
        (rc = encode_map_2d(&h->m16_wo[l], h->w16_wo + l * d * nq, d, nq, 128, true)) ||
        (rc = encode_map_2d(&h->m16_wgu[l], h->w16_gu + l * 2 * I * d, 2 * I, d, 128, true)) ||
        (rc = encode_map_2d(&h->m16_wd[l], h->w16_wd + l * d * I, d, I, 128, true))) {
      fp16_free(h);
      return rc;
    }
  }
  if ((rc = set_tc_attr<DE_QKV, CS_QKV, 1>()) || (rc = set_tc_attr<DE_QKV, CS_QKV, 3>()) ||
      (rc = set_tc_attr<DE_OPROJ, CS_O, 1>()) || (rc = set_tc_attr<DE_GATEUP, CS_GU, 1>()))
    return rc;
  return set_tc_attr<DE_DOWN, CS_DOWN, 1>();
}

extern "C" int ctb_gpt_create(const ctb_gpt_config* c, const float* weights_dev, ctb_gpt** out) {
  if (!c || !weights_dev || !out) return set_err(CTB_ERR_ARG, "null argument");
  if (c->hidden_size != KC) return set_err(CTB_ERR_ARG, "hidden_size must be %d", KC);
  if (c->intermediate_size % KC) return set_err(CTB_ERR_ARG, "intermediate_size must be a multiple of %d", KC);
  if (c->head_dim != 64) return set_err(CTB_ERR_ARG, "head_dim must be 64");
  if (c->num_heads % c->num_kv_heads) return set_err(CTB_ERR_ARG, "num_heads %% num_kv_heads != 0");
  if (c->num_vq > 8 || c->num_vq < 1) return set_err(CTB_ERR_ARG, "num_vq out of range");
  if (c->max_batch < 1 || c->max_context < 1 || c->max_context > c->max_positions)
    return set_err(CTB_ERR_ARG, "bad max_batch/max_context");
  int dev_count = 0;
  CTB_CUDA(cudaGetDeviceCount(&dev_count));
  if (dev_count < 1) return set_err(CTB_ERR_CUDA, "no CUDA device: chattts_b200 has no CPU path");
  {
    int dev = 0, sms = 0;
    CTB_CUDA(cudaGetDevice(&dev));
    CTB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    g_num_sms = sms;
  }
  ctb_gpt* h = new ctb_gpt();
  memset(h, 0, sizeof(*h));
  h->cfg = *c;
  ctb_gpt_layout_query(c, &h->lay);
  h->W = weights_dev;
  h->pages_per_row = (c->max_context + kPageTokens - 1) / kPageTokens;
  h->nsplit_max = (c->max_context + ATT_SPLIT_UNIT - 1) / ATT_SPLIT_UNIT;
  const int bt = bt_for(c->max_batch);
  h->bpad_max = ((c->max_batch + bt - 1) / bt) * bt;
  const size_t Bp = h->bpad_max, d = c->hidden_size;
  const size_t nq = (size_t)c->num_heads * c->head_dim;
  int rc;
#define TRY(e) if ((rc = (e)) != CTB_OK) { ctb_gpt_destroy(h); return rc; }
  TRY(dalloc(&h->x, Bp * d));
  TRY(dalloc(&h->qbuf, Bp * nq));
  TRY(dalloc(&h->attn, Bp * nq));
  TRY(dalloc(&h->mlp, Bp * c->intermediate_size));
  const size_t nlog = std::max((size_t)c->num_vq * c->num_audio_tokens, (size_t)c->num_text_tokens);
  TRY(dalloc(&h->logits, Bp * nlog));
  // The KV pool is sized by what a generate() call can actually touch (ctb_gpt_begin -> kv_reserve), not by
  // max_batch x max_context: a handle that allows 32 rows x 4096 tokens costs nothing until such a call arrives.
  h->kv = nullptr; h->kv_layer_elems = 0; h->kv_bytes = 0;
  TRY(dalloc(&h->part, (size_t)c->max_batch * c->num_heads * h->nsplit_max * (c->head_dim + 2)));
  TRY(dalloc(&h->block_table, (size_t)c->max_batch * h->pages_per_row));
  TRY(dalloc(&h->seq_len, Bp));
  TRY(dalloc(&h->pos, Bp));
  TRY(dalloc(&h->counter, (size_t)c->max_batch * c->num_heads));
  TRY(dalloc(&h->end_idx, Bp));
  TRY(dalloc(&h->idx, Bp * c->num_vq));
  TRY(dalloc(&h->active, Bp));
  TRY(dalloc(&h->finish, Bp));
  TRY(dalloc(&h->st, 1));
  TRY(dalloc(&h->bar, 4));
  if (getenv("CTB_MEGA_TRACE")) TRY(dalloc(&h->trace, FL_TR_WORDS));
  h->flow_ok = getenv("CTB_NO_FLOW") == nullptr && g_num_sms >= 128 && g_num_sms <= 191 && c->intermediate_size == 4 * KC &&
               c->num_heads == c->num_kv_heads && c->num_heads * c->head_dim == KC && c->num_heads <= FL_HEADS;
  if (h->flow_ok) {
    TRY(dalloc(&h->flow_arena, FL_ARENA_WORDS));
    TRY(dalloc(&h->flow_epoch, 4));
    const unsigned e0 = FL_EPOCH_STEP;
    cudaMemcpy(h->flow_epoch, &e0, sizeof(e0), cudaMemcpyHostToDevice);
    // one copy of the exchange words by default (replicas multiply the 8-byte stores; CTB_FLOW_R selects more for
    // tools/flow_check.py to compare)
    h->flow_R = getenv("CTB_FLOW_R") ? std::max(1, std::min(FL_RMAX, atoi(getenv("CTB_FLOW_R")))) : 1;
    h->flow_l2_ahead = getenv("CTB_FLOW_L2_AHEAD") ? atoi(getenv("CTB_FLOW_L2_AHEAD")) : 0;
    // H100, 512-token passes: k_flow<1> 239 ms vs k_step<1> 309 ms, but at B = 2 / 3 / 4 k_step is faster (332 / 379 / 395 ms
    // vs 342 / 530 / 550 ms), so the dataflow step serves B = 1 by default
    h->flow_max_batch = getenv("CTB_FLOW_MAX_BATCH") ? std::max(0, std::min(FL_BMAX, atoi(getenv("CTB_FLOW_MAX_BATCH")))) : 1;
    h->flow_no_ink = getenv("CTB_FLOW_NO_INK") != nullptr;
  }
#undef TRY
  h->use_graph = getenv("CTB_NO_GRAPH") == nullptr;
  h->pf_enabled = getenv("CTB_NO_BATCHED_PREFILL") == nullptr;
  h->mega_ok = getenv("CTB_NO_MEGA") == nullptr && g_num_sms >= 128 && c->intermediate_size == 4 * KC &&
               (c->hidden_size / 2 + g_num_sms - 1) / g_num_sms <= MG_DOWN_PAIRS;
  h->mega_max_batch = getenv("CTB_MEGA_MAX_BATCH") ? std::min(8, atoi(getenv("CTB_MEGA_MAX_BATCH"))) : 4;
  // tensor-core decode GEMMs (tc_decode.cuh): CTB_GPT_TC=1 forces them for every batch, CTB_GPT_FMA=1 disables
  // them; by default they serve batches of 9 rows and more, where the FMA kernels' batch tile grows to 16 rows
  // (H100, 512-token passes: 726 / 786 ms vs 881 / 962 ms at B = 10 / 16; at B = 8 the FMA kernels take 481 ms).
  constexpr int kTcMinBatch = 9;
  h->tc_ready = getenv("CTB_GPT_FMA") == nullptr && c->max_batch <= 32 &&
                (getenv("CTB_GPT_TC") != nullptr || c->max_batch >= kTcMinBatch);
  h->tc_min_batch = getenv("CTB_GPT_TC") != nullptr ? 1 : kTcMinBatch;
  if (h->tc_ready && (rc = tc_setup(h)) != CTB_OK) { ctb_gpt_destroy(h); return rc; }
  *out = h;
  return CTB_OK;
}

extern "C" int ctb_gpt_destroy(ctb_gpt* h) {
  if (!h) return CTB_OK;
  if (h->graph_exec) cudaGraphExecDestroy(h->graph_exec);
  if (h->graph_exec_text) cudaGraphExecDestroy(h->graph_exec_text);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  void* ptrs[] = {h->x, h->qbuf, h->attn, h->mlp, h->logits, h->kv, h->part, h->block_table, h->seq_len,
                  h->pos, h->counter, h->end_idx, h->idx, h->active, h->finish, h->st, h->tc_wqkv, h->tc_wgu,
                  h->tc_heads_code, h->tc_heads_text, h->x_hi, h->x_lo, h->attn_hi, h->attn_lo, h->h_hi, h->h_lo, h->bar, h->trace, h->flow_arena, h->flow_epoch, h->gw_hi, h->gw_lo, h->pf_resid, h->pf_xn, h->pf_qkv, h->pf_q,
                  h->pf_attn, h->pf_gu, h->pf_h, h->pf_ones, h->pf_zeros, h->pf_npre, h->pf_nvalid,
                  h->pf_mask, h->rows, h->cfgs, h->eng_noise, h->eng_slot, h->eng_text_logits, h->eng_text_idx,
                  h->pg_stage, h->sc_head_hi[0], h->sc_head_hi[1], h->sc_head_lo[0], h->sc_head_lo[1], h->sc_xn,
                  h->sc_logits, h->sc_src};
  delete[] h->m_wqkv; delete[] h->m_wo; delete[] h->m_wgu; delete[] h->m_wd;
  for (void* p : ptrs) if (p) cudaFree(p);
  fp16_free(h);
  delete h;
  return CTB_OK;
}

// ------------------------------------------------------------------ launches
template <int BT, int EPI>
static int launch_gemv_t(const GemvP& p, int ntiles, cudaStream_t s) {
  const size_t smem = (size_t)BT * KC * sizeof(float);
  { int rc = ensure_smem_attr((const void*)k_gemv<BT, EPI>, (int)smem); if (rc) return rc; }
  // persistent: one CTA per SM strides over the warp tasks (DOWN: clusters of DOWN_SPLIT CTAs)
  int ctas = std::min(g_num_sms, (p.ntasks + GEMV_WARPS - 1) / GEMV_WARPS);
  unsigned cluster = 1;
  if (EPI == EPI_DOWN) {
    cluster = DOWN_SPLIT;
    // clusters of 4 cannot use every SM at once (GPC granularity): size one wave by what the device reports
    static int max_groups = 0;
    if (!max_groups) {
      cudaLaunchConfig_t qc{};
      qc.gridDim = dim3(DOWN_SPLIT * (g_num_sms / DOWN_SPLIT)); qc.blockDim = dim3(GEMV_WARPS * 32); qc.dynamicSmemBytes = smem;
      cudaLaunchAttribute qa[1];
      qa[0].id = cudaLaunchAttributeClusterDimension;
      qa[0].val.clusterDim.x = DOWN_SPLIT; qa[0].val.clusterDim.y = 1; qa[0].val.clusterDim.z = 1;
      qc.attrs = qa; qc.numAttrs = 1;
      CTB_CUDA(cudaOccupancyMaxActiveClusters(&max_groups, k_gemv<BT, EPI>, &qc));
      if (max_groups < 1) return set_err(CTB_ERR_STATE, "DOWN kernel: no cluster of %d CTAs fits the device", DOWN_SPLIT);
    }
    const int groups = std::max(1, std::min(max_groups, (p.ntasks + GEMV_WARPS - 1) / GEMV_WARPS));
    if ((p.ntasks + groups * GEMV_WARPS - 1) / (groups * GEMV_WARPS) > DOWN_MAX_TASKS)
      return set_err(CTB_ERR_STATE, "DOWN kernel: too few SMs (%d) for %d tasks", g_num_sms, p.ntasks);
    ctas = groups * DOWN_SPLIT;
  }
  dim3 grid(ctas, ntiles);
  CTB_CUDA(launch_pdl_cluster(k_gemv<BT, EPI>, grid, dim3(GEMV_WARPS * 32), smem, s, cluster, p));
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

template <int EPI>
static int launch_gemv(int bt, const GemvP& p, int ntiles, cudaStream_t s) {
  switch (bt) {
    case 1: return launch_gemv_t<1, EPI>(p, ntiles, s);
    case 2: return launch_gemv_t<2, EPI>(p, ntiles, s);
    case 4: return launch_gemv_t<4, EPI>(p, ntiles, s);
    case 8: return launch_gemv_t<8, EPI>(p, ntiles, s);
    case 16: return launch_gemv_t<16, EPI>(p, ntiles, s);
    default: return launch_gemv_t<32, EPI>(p, ntiles, s);
  }
}

template <int BT>
static int launch_gateup_small_t(const GemvP& p, cudaStream_t s) {
  const size_t smem = ((size_t)BT * KC + GU_ZONE_FLOATS) * sizeof(float);
  { int rc = ensure_smem_attr((const void*)k_gateup_small<BT>, (int)smem); if (rc) return rc; }
  CTB_CUDA(launch_pdl(k_gateup_small<BT>, dim3(g_num_sms), dim3(GEMV_WARPS * 32), smem, s, p));
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}
static int launch_gateup_small(int bt, const GemvP& p, cudaStream_t s) {
  switch (bt) {
    case 1: return launch_gateup_small_t<1>(p, s);
    case 2: return launch_gateup_small_t<2>(p, s);
    case 4: return launch_gateup_small_t<4>(p, s);
    case 8: return launch_gateup_small_t<8>(p, s);
    default: return launch_gateup_small_t<16>(p, s);
  }
}

template <int BT>
static int launch_down_small_t(const GemvP& p, cudaStream_t s) {
  const size_t smem = (size_t)BT * p.K * sizeof(float);
  { int rc = ensure_smem_attr((const void*)k_down_small<BT>, (int)smem); if (rc) return rc; }
  CTB_CUDA(launch_pdl(k_down_small<BT>, dim3(g_num_sms), dim3(GEMV_WARPS * 32), smem, s, p));
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}
static int launch_down_small(int bt, const GemvP& p, cudaStream_t s) {
  switch (bt) {
    case 1: return launch_down_small_t<1>(p, s);
    case 2: return launch_down_small_t<2>(p, s);
    case 4: return launch_down_small_t<4>(p, s);
    case 8: return launch_down_small_t<8>(p, s);
    default: return launch_down_small_t<16>(p, s);
  }
}

template <bool ENGINE>
static int launch_sample_t(const SampleP& sp, cudaStream_t s) {
  const size_t smem = (size_t)sp.V * sizeof(float) + 2 * 1024 * sizeof(uint32_t);
  { int rc = ensure_smem_attr((const void*)k_sample<ENGINE>, (int)smem); if (rc) return rc; }
  CTB_CUDA(launch_pdl(k_sample<ENGINE>, dim3(sp.rows), dim3(SAMPLE_THREADS), smem, s, sp));
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}
static int launch_sample(const SampleP& sp, cudaStream_t s) {
  return sp.rstate != nullptr ? launch_sample_t<true>(sp, s) : launch_sample_t<false>(sp, s);
}

struct StepCtx {
  GemvP g;
  AttnP a;
  int bt, ntiles, decode;
};

static StepCtx make_ctx(ctb_gpt* h, int decode) {
  const ctb_gpt_config& c = h->cfg;
  const ctb_gpt_layout& L = h->lay;
  StepCtx x{};
  x.decode = decode;
  x.bt = bt_for(h->B);
  x.ntiles = (h->B + x.bt - 1) / x.bt;
  GemvP& g = x.g;
  g.B = h->B; g.st = h->st; g.check_finished = decode; g.eps = c.rms_eps;
  g.block_table = h->block_table; g.pages_per_row = h->pages_per_row; g.pos = h->pos; g.active = h->active;
  g.rope_cos = h->W + L.rope_cos; g.rope_sin = h->W + L.rope_sin;
  g.Hq = c.num_heads; g.Hkv = c.num_kv_heads; g.hd = c.head_dim; g.I = c.intermediate_size; g.xres = h->x;
  AttnP& a = x.a;
  a.st = h->st; a.check_finished = decode; a.q = h->qbuf; a.block_table = h->block_table;
  a.pages_per_row = h->pages_per_row; a.pos = h->pos; a.active = h->active; a.out = h->attn; a.part = h->part;
  a.out_hi = h->use_tc ? h->attn_hi : nullptr; a.out_lo = h->use_tc ? h->attn_lo : nullptr;
  a.counter = h->counter; a.Hq = c.num_heads; a.Hkv = c.num_kv_heads; a.hd = c.head_dim;
  a.nsplit_max = h->nsplit_max; a.scaling = 1.0f / sqrtf((float)c.head_dim);
  return x;
}

// kind: 0 qkv(+rope+kv append), 1 attention, 2 o-proj(+residual), 3 gate/up(+silu*mul), 4 down(+residual)
static int launch_layer_kernel(ctb_gpt* h, const StepCtx& x, int l, int kind, cudaStream_t s) {
  const ctb_gpt_config& c = h->cfg;
  const ctb_gpt_layout& L = h->lay;
  const int d = c.hidden_size, I = c.intermediate_size, hd = c.head_dim;
  const float* Wl = h->W + L.layer0 + (int64_t)l * L.layer_stride;
  float* kvl = kv_layer(h, l);
  GemvP p = x.g;
  switch (kind) {
    case 0:
      p.W = Wl + L.wqkv; p.K = d; p.nrows = (c.num_heads + 2 * c.num_kv_heads) * hd; p.ntasks = p.nrows / 2;
      p.xin = h->x; p.normw = Wl + L.ln1; p.out = h->qbuf; p.kv = kvl;
      return launch_gemv<EPI_QKV>(x.bt, p, x.ntiles, s);
    case 1: {
      AttnP a = x.a;
      a.kv = kvl;
      // context after this call <= T0 + max_new: only launch splits that can be populated (a slot engine's rows may
      // reach max_context)
      const int max_ctx = h->engine ? c.max_context : std::min(c.max_context, h->T0 + h->max_new);
      // enough CTAs to fill the chip twice; a CTA walks chunks c, c + grid.x, ... with a running softmax,
      // so large batches need no cross-CTA merge at all
      const int want = (2 * g_num_sms + c.num_heads * h->B - 1) / (c.num_heads * h->B);
      dim3 agrid(std::max(1, std::min(want, (max_ctx + ATT_CHUNK - 1) / ATT_CHUNK)), c.num_heads, h->B);
      if (h->prec & CTB_ENGINE_FP16_KV)
        CTB_CUDA(launch_pdl(k_attn<__half>, agrid, dim3(ATT_THREADS), 0, s, a));
      else
        CTB_CUDA(launch_pdl(k_attn<float>, agrid, dim3(ATT_THREADS), 0, s, a));
      CTB_LAUNCH_CHECK();
      return CTB_OK;
    }
    case 2:
      p.W = Wl + L.wo; p.K = c.num_heads * hd; p.nrows = d; p.ntasks = d / 2; p.xin = h->attn; p.normw = nullptr;
      return launch_gemv<EPI_OPROJ>(x.bt, p, x.ntiles, s);
    case 3:
      p.W = Wl + L.wgate_up; p.K = d; p.nrows = 2 * I; p.ntasks = I; p.xin = h->x; p.normw = Wl + L.ln2;
      p.out = h->mlp;
      if (x.bt <= 8 && x.ntiles == 1 && (I + g_num_sms * GEMV_WARPS - 1) / (g_num_sms * GEMV_WARPS) <= GU_TASKS &&
          getenv("CTB_GATEUP_GENERIC") == nullptr)
        return launch_gateup_small(x.bt, p, s);
      return launch_gemv<EPI_GATEUP>(x.bt, p, x.ntiles, s);
    case 4:
      p.W = Wl + L.wdown; p.K = I; p.nrows = d; p.ntasks = d / 2; p.xin = h->mlp; p.normw = nullptr;
      if (x.bt <= 16 && x.ntiles == 1 && I == 4 * KC && (d / 2 + g_num_sms - 1) / g_num_sms <= DS_PAIRS &&
          getenv("CTB_DOWN_CLUSTER") == nullptr)
        return launch_down_small(x.bt, p, s);
      return launch_gemv<EPI_DOWN>(x.bt, p, x.ntiles, s);
  }
  return set_err(CTB_ERR_ARG, "bad kernel kind %d", kind);
}

static int launch_heads(ctb_gpt* h, const StepCtx& x, cudaStream_t s) {
  const ctb_gpt_config& c = h->cfg;
  const int rpi = h->infer_text ? 1 : c.num_vq;
  const int V = h->infer_text ? c.num_text_tokens : c.num_audio_tokens;
  GemvP hp = x.g;
  hp.W = h->W + (h->infer_text ? h->lay.head_text : h->lay.head_code);
  hp.K = c.hidden_size; hp.nrows = rpi * V; hp.ntasks = (hp.nrows + 1) / 2; hp.xin = h->x;
  hp.normw = h->W + h->lay.final_norm; hp.out = h->logits; hp.rows_per_item = rpi; hp.V = V;
  hp.hidden_out = h->hiddens_out; hp.hidden_stride = h->max_new * c.hidden_size;
  hp.rows = h->engine ? h->rows : nullptr; hp.want = h->phase;
  const int rc = launch_gemv<EPI_HEADS>(x.bt, hp, x.ntiles, s);
  if (rc || !h->engine || !h->eng_text) return rc;
  // slot engine: the code heads above served the code rows; the text head serves the text rows, into its own logits
  // buffer and without hidden states (its CTAs leave at once when no text row is in state `phase`)
  hp.W = h->W + h->lay.head_text; hp.nrows = c.num_text_tokens; hp.ntasks = (hp.nrows + 1) / 2;
  hp.out = h->eng_text_logits; hp.rows_per_item = 1; hp.V = c.num_text_tokens; hp.hidden_out = nullptr;
  hp.want = h->phase | WANT_TEXT;
  return launch_gemv<EPI_HEADS>(x.bt, hp, x.ntiles, s);
}

// the log-probabilities of the ids the k_sample<true> launch `sp` just wrote, at the index k_finalize_rows writes them
static int launch_logprob(ctb_gpt* h, const SampleP& sp, cudaStream_t s) {
  LogprobP lp{};
  lp.st = sp.st; lp.check_finished = sp.check_finished; lp.logits = sp.logits; lp.V = sp.V;
  lp.rows_per_item = sp.rows_per_item; lp.idx = sp.out_idx; lp.rstate = sp.rstate; lp.want = sp.want;
  lp.out = h->eng_logprobs; lp.max_new = h->max_new; lp.num_vq = h->cfg.num_vq;
  CTB_CUDA(launch_pdl(k_token_logprob, dim3(sp.rows), dim3(LOGPROB_THREADS), 0, s, lp));
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

static int launch_top_logprobs(const TopLogprobP& tp, int rows, cudaStream_t s) {
  const int smem = tp.V * (int)sizeof(float);
  { int rc = ensure_smem_attr((const void*)k_token_top_logprobs, smem); if (rc) return rc; }
  CTB_CUDA(launch_pdl(k_token_top_logprobs, dim3(rows), dim3(LOGPROB_THREADS), (size_t)smem, s, tp));
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

// the N most likely ids and their log-probabilities for the rows the k_sample<true> launch `sp` just served, at the
// index k_finalize_rows writes the sampled id
static int launch_top_logprobs(ctb_gpt* h, const SampleP& sp, cudaStream_t s) {
  TopLogprobP tp{};
  tp.st = sp.st; tp.check_finished = sp.check_finished; tp.logits = sp.logits; tp.V = sp.V;
  tp.rows_per_item = sp.rows_per_item; tp.rstate = sp.rstate; tp.want = sp.want; tp.n_top = h->eng_top_n;
  tp.ids = h->eng_top_ids; tp.lp = h->eng_top_lp; tp.max_new = h->max_new; tp.num_vq = h->cfg.num_vq;
  return launch_top_logprobs(tp, sp.rows, s);
}

static int launch_sampler(ctb_gpt* h, const StepCtx& x, cudaStream_t s) {
  const ctb_gpt_config& c = h->cfg;
  const int rpi = h->infer_text ? 1 : c.num_vq;
  SampleP sp{};
  sp.st = h->st; sp.check_finished = x.decode; sp.logits = h->logits; sp.rows = h->B * rpi;
  sp.V = h->infer_text ? c.num_text_tokens : c.num_audio_tokens;
  sp.rows_per_item = rpi; sp.cfg = h->sampler; sp.q_noise = h->q_noise; sp.gen_ids = h->ids_out;
  sp.gen_stride = h->max_new; sp.gen_inner = c.num_vq; sp.out_idx = h->idx;
  if (!h->engine) return launch_sample(sp, s);
  sp.rstate = h->rows; sp.cfgs = h->cfgs; sp.want = h->phase; sp.q_noise = h->eng_noise;
  sp.noise_stride = (int)noise_stride(h);
  int rc = launch_sample(sp, s);
  if (!rc && h->eng_logprobs) rc = launch_logprob(h, sp, s);
  if (!rc && h->eng_top_n) rc = launch_top_logprobs(h, sp, s);
  if (rc || !h->eng_text) return rc;
  // text rows: one row per slot over the text head's logits, as a batch of one samples them
  sp.logits = h->eng_text_logits; sp.rows = h->B; sp.V = c.num_text_tokens; sp.rows_per_item = 1;
  sp.out_idx = h->eng_text_idx; sp.want = h->phase | WANT_TEXT;
  if ((rc = launch_sample(sp, s)) || (h->eng_logprobs && (rc = launch_logprob(h, sp, s)))) return rc;
  return h->eng_top_n ? launch_top_logprobs(h, sp, s) : CTB_OK;
}

// npad 16 for B <= 16, 32 for B <= 32, 64 for B <= 64 (a 64-row scratch only: tc_rows == 64)
static int tc_npad_index(int B) { return B > 32 ? 2 : (B > 16 ? 1 : 0); }

template <int EPI, int CS, int PREC = 0>
static int launch_tc(int npad, const CUtensorMap& mw, const CUtensorMap& mxh, const CUtensorMap& mxl, const TcDecP& p,
                     cudaStream_t s) {
  constexpr bool W16 = (PREC & TD_W16) != 0;
  const int tiles = (p.nrows + 127) / 128;
  dim3 grid(tiles * CS);
  if (npad == 16)
    CTB_CUDA(launch_pdl_cluster(k_tc_dec<EPI, 16, CS, PREC>, grid, dim3(TD_THREADS), (size_t)TdCfg<16, W16>::SMEM_BYTES, s, (unsigned)CS, mw, mxh, mxl, p));
  else if (npad == 32)
    CTB_CUDA(launch_pdl_cluster(k_tc_dec<EPI, 32, CS, PREC>, grid, dim3(TD_THREADS), (size_t)TdCfg<32, W16>::SMEM_BYTES, s, (unsigned)CS, mw, mxh, mxl, p));
  else
    CTB_CUDA(launch_pdl_cluster(k_tc_dec<EPI, 64, CS, PREC>, grid, dim3(TD_THREADS), (size_t)TdCfg<64, W16>::SMEM_BYTES, s, (unsigned)CS, mw, mxh, mxl, p));
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

static TcDecP make_tc(ctb_gpt* h) {
  const ctb_gpt_config& c = h->cfg;
  TcDecP p{};
  p.B = h->B; p.eps = c.rms_eps; p.d = c.hidden_size; p.xres = h->x; p.x_hi = h->x_hi; p.x_lo = h->x_lo;
  p.qbuf = h->qbuf; p.block_table = h->block_table; p.pages_per_row = h->pages_per_row; p.pos = h->pos;
  p.active = h->active; p.rope_cos = h->W + h->lay.rope_cos; p.rope_sin = h->W + h->lay.rope_sin;
  p.Hq = c.num_heads; p.Hkv = c.num_kv_heads; p.hd = c.head_dim; p.h_hi = h->h_hi; p.h_lo = h->h_lo;
  p.I = c.intermediate_size; p.st = h->st;
  return p;
}

// PREC: the engine's CTB_ENGINE_FP16_* bits (only the QKV GEMM sees the KV bit)
template <int PREC>
static int launch_layer_kernel_tc_t(ctb_gpt* h, int l, int kind, cudaStream_t s) {
  constexpr int PW = PREC & TD_W16;
  const ctb_gpt_config& c = h->cfg;
  const int n = tc_npad_index(h->B), npad = 16 << n;
  const int d = c.hidden_size, I = c.intermediate_size;
  TcDecP p = make_tc(h);
  switch (kind) {
    case 0:
      p.K = d; p.kslice = d / CS_QKV; p.nrows = (c.num_heads + 2 * c.num_kv_heads) * c.head_dim; p.xraw = h->x;
      p.kv = kv_layer(h, l);
      return launch_tc<DE_QKV, CS_QKV, PREC>(npad, PW ? h->m16_wqkv[l] : h->m_wqkv[l], h->m_x[n][0], h->m_x[n][1], p, s);
    case 2:
      p.K = c.num_heads * c.head_dim; p.kslice = p.K / CS_O; p.nrows = d; p.xraw = nullptr;
      return launch_tc<DE_OPROJ, CS_O, PW>(npad, PW ? h->m16_wo[l] : h->m_wo[l], h->m_attn[n][0], h->m_attn[n][1], p, s);
    case 3:
      p.K = d; p.kslice = d / CS_GU; p.nrows = 2 * I; p.xraw = h->x;
      return launch_tc<DE_GATEUP, CS_GU, PW>(npad, PW ? h->m16_wgu[l] : h->m_wgu[l], h->m_x[n][0], h->m_x[n][1], p, s);
    case 4:
      p.K = I; p.kslice = I / CS_DOWN; p.nrows = d; p.xraw = nullptr;
      return launch_tc<DE_DOWN, CS_DOWN, PW>(npad, PW ? h->m16_wd[l] : h->m_wd[l], h->m_h[n][0], h->m_h[n][1], p, s);
  }
  return set_err(CTB_ERR_ARG, "bad tc kernel kind %d", kind);
}

static int launch_layer_kernel_tc(ctb_gpt* h, int l, int kind, cudaStream_t s) {
  switch (h->prec) {
    case 0: return launch_layer_kernel_tc_t<0>(h, l, kind, s);
    case CTB_ENGINE_FP16_WEIGHTS: return launch_layer_kernel_tc_t<CTB_ENGINE_FP16_WEIGHTS>(h, l, kind, s);
    case CTB_ENGINE_FP16_KV: return launch_layer_kernel_tc_t<CTB_ENGINE_FP16_KV>(h, l, kind, s);
    default: return launch_layer_kernel_tc_t<CTB_ENGINE_FP16_WEIGHTS | CTB_ENGINE_FP16_KV>(h, l, kind, s);
  }
}

static int launch_heads_tc(ctb_gpt* h, cudaStream_t s) {
  const ctb_gpt_config& c = h->cfg;
  const int n = tc_npad_index(h->B), npad = 16 << n;
  TcDecP p = make_tc(h);
  const int rpi = h->infer_text ? 1 : c.num_vq;
  const int V = h->infer_text ? c.num_text_tokens : c.num_audio_tokens;
  p.K = c.hidden_size; p.kslice = p.K / CS_HEADS; p.nrows = rpi * V; p.xraw = h->x;
  p.logits = h->logits; p.rows_per_item = rpi; p.V = V; p.hidden_out = h->hiddens_out;
  p.hidden_stride = h->max_new * c.hidden_size; p.final_norm_w = h->W + h->lay.final_norm;
  p.rows = h->engine ? h->rows : nullptr; p.want = h->phase;
  const int rc = launch_tc<DE_HEADS, CS_HEADS>(npad, h->infer_text ? h->m_htext : h->m_hcode, h->m_x[n][0], h->m_x[n][1], p, s);
  if (rc || !h->engine || !h->eng_text) return rc;
  // slot engine: the text head over the text rows (see launch_heads)
  p.nrows = c.num_text_tokens; p.logits = h->eng_text_logits; p.rows_per_item = 1; p.V = c.num_text_tokens;
  p.hidden_out = nullptr; p.want = h->phase | WANT_TEXT;
  return launch_tc<DE_HEADS, CS_HEADS>(npad, h->m_htext, h->m_x[n][0], h->m_x[n][1], p, s);
}

template <int BT>
static int launch_step_mega_t(const MegaP& mp, cudaStream_t s) {
  // [BT][768] activations + the 144 KiB landing zone (gate/up weights; reused as merge scratch and for the down
  // phase's [BT][3072] activations)
  const size_t smem = (size_t)BT * KC * sizeof(float) + (size_t)MG_GW_FLOATS * sizeof(float);
  { int rc = ensure_smem_attr((const void*)k_step<BT>, (int)smem); if (rc) return rc; }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(g_num_sms); cfg.blockDim = dim3(MG_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;  // every CTA must be resident: the phases meet at grid barriers
  attr[0].val.cooperative = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  CTB_CUDA(cudaLaunchKernelEx(&cfg, k_step<BT>, mp));
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

static int launch_step_mega(ctb_gpt* h, int col, bool sample, cudaStream_t s) {
  const ctb_gpt_config& c = h->cfg;
  const ctb_gpt_layout& L = h->lay;
  MegaP m{};
  m.W = h->W; m.layer0 = L.layer0; m.layer_stride = L.layer_stride; m.o_wqkv = L.wqkv; m.o_wo = L.wo; m.o_wgu = L.wgate_up;
  m.o_wd = L.wdown; m.o_ln1 = L.ln1; m.o_ln2 = L.ln2; m.o_final_norm = L.final_norm;
  m.o_head = h->infer_text ? L.head_text : L.head_code; m.o_emb_code = L.emb_code; m.o_emb_text = L.emb_text;
  m.o_cos = L.rope_cos; m.o_sin = L.rope_sin;
  m.L = c.num_layers; m.d = c.hidden_size; m.I = c.intermediate_size; m.Hq = c.num_heads; m.Hkv = c.num_kv_heads;
  m.hd = c.head_dim; m.eps = c.rms_eps; m.scaling = 1.0f / sqrtf((float)c.head_dim);
  m.x = h->x; m.qbuf = h->qbuf; m.attn = h->attn; m.mlp = h->mlp; m.logits = h->logits; m.kv = h->kv; m.part = h->part;
  m.kv_layer_floats = h->kv_layer_elems; m.block_table = h->block_table; m.pages_per_row = h->pages_per_row;
  m.seq_len = h->seq_len; m.counter = h->counter; m.nsplit_max = h->nsplit_max; m.st = h->st; m.bar = h->bar;
  m.decode = col < 0; m.col = col < 0 ? 0 : col; m.T0 = h->T0; m.sample = sample ? 1 : 0;
  m.emb = h->emb; m.mask = h->mask; m.ids_out = h->ids_out; m.max_new = h->max_new; m.num_vq = c.num_vq;
  m.num_audio = c.num_audio_tokens; m.infer_text = h->infer_text; m.B = h->B;
  m.hidden_out = h->hiddens_out; m.hidden_stride = h->max_new * c.hidden_size;
  m.rows_per_item = h->infer_text ? 1 : c.num_vq; m.V = h->infer_text ? c.num_text_tokens : c.num_audio_tokens;
  m.trace = h->trace;
  CTB_CUDA(cudaMemsetAsync(h->bar, 0, sizeof(unsigned), s));
  switch (bt_for(h->B)) {
    case 1: return launch_step_mega_t<1>(m, s);
    case 2: return launch_step_mega_t<2>(m, s);
    case 4: return launch_step_mega_t<4>(m, s);
    default: return launch_step_mega_t<8>(m, s);
  }
}

template <int BT>
static int launch_step_flow_t(const FlowP& fp, cudaStream_t s) {
  const size_t smem = (size_t)FL_RING_BYTES + (size_t)BT * KC * sizeof(float);
  { int rc = ensure_smem_attr((const void*)k_flow<BT>, (int)smem); if (rc) return rc; }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(g_num_sms); cfg.blockDim = dim3(FL_LAUNCH_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;  // every CTA must be resident: CTAs wait for each other's words
  attr[0].val.cooperative = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  CTB_CUDA(cudaLaunchKernelEx(&cfg, k_flow<BT>, fp));
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

static bool flow_ink(const ctb_gpt* h);

// nsteps > 0: multi-step decode with the sampling tail inside the kernel (requires flow_ink(h)); 0: one step, logits out
static int launch_step_flow(ctb_gpt* h, int col, bool sample, cudaStream_t s, int nsteps = 0) {
  const ctb_gpt_config& c = h->cfg;
  const ctb_gpt_layout& L = h->lay;
  FlowP m{};
  m.W = h->W; m.layer0 = L.layer0; m.layer_stride = L.layer_stride; m.o_wqkv = L.wqkv; m.o_wo = L.wo; m.o_wgu = L.wgate_up;
  m.o_wd = L.wdown; m.o_ln1 = L.ln1; m.o_ln2 = L.ln2; m.o_final_norm = L.final_norm;
  m.o_head = h->infer_text ? L.head_text : L.head_code; m.o_emb_code = L.emb_code; m.o_emb_text = L.emb_text;
  m.o_cos = L.rope_cos; m.o_sin = L.rope_sin;
  m.L = c.num_layers; m.I = c.intermediate_size; m.Hq = c.num_heads; m.hd = c.head_dim; m.eps = c.rms_eps;
  m.scaling = 1.0f / sqrtf((float)c.head_dim);
  m.logits = h->logits; m.kv = h->kv; m.kv_layer_floats = h->kv_layer_elems; m.block_table = h->block_table;
  m.pages_per_row = h->pages_per_row; m.seq_len = h->seq_len; m.st = h->st;
  m.decode = col < 0; m.col = col < 0 ? 0 : col; m.T0 = h->T0; m.sample = sample ? 1 : 0;
  m.emb = h->emb; m.mask = h->mask; m.ids_out = h->ids_out; m.max_new = h->max_new; m.num_vq = c.num_vq;
  m.num_audio = c.num_audio_tokens; m.infer_text = h->infer_text; m.B = h->B;
  m.hidden_out = h->hiddens_out; m.hidden_stride = h->max_new * c.hidden_size;
  m.rows_per_item = h->infer_text ? 1 : c.num_vq; m.V = h->infer_text ? c.num_text_tokens : c.num_audio_tokens;
  m.arena = h->flow_arena; m.epoch = h->flow_epoch; m.R = h->flow_R; m.trace = h->trace;
  m.l2_ahead = h->flow_l2_ahead;
  m.ink = nsteps > 0 ? 1 : 0; m.nsteps = nsteps > 0 ? nsteps : 1; m.samp = h->sampler; m.q_noise = h->q_noise;
  m.finish = h->finish; m.end_idx = h->end_idx; m.ids_w = h->ids_out;
  switch (bt_for(h->B)) {
    case 1: return launch_step_flow_t<1>(m, s);
    case 2: return launch_step_flow_t<2>(m, s);
    default: return launch_step_flow_t<4>(m, s);
  }
}

// Which step serves a static batch of B rows (tc: the wgmma step's GEMMs are on, tc_for).  The one-kernel steps
// (k_flow, k_step) keep the batch's loop counters in LoopState: never used by a slot engine.
static bool tc_for(const ctb_gpt* h, int B) { return h->tc_ready && B >= h->tc_min_batch; }
static bool flow_for(const ctb_gpt* h, int B, bool tc) { return h->flow_ok && !tc && B <= h->flow_max_batch; }
static bool mega_for(const ctb_gpt* h, int B, bool tc) { return h->mega_ok && !tc && B <= h->mega_max_batch; }
// decode steps of audio generation at B <= 2 sample inside k_flow and run many steps per launch
static bool ink_for(const ctb_gpt* h, int B, bool text, bool tc) {
  return !h->flow_no_ink && flow_for(h, B, tc) && !text && B <= 2 && h->cfg.num_audio_tokens <= FL_VPAD &&
         B * h->cfg.num_vq <= FL_SROWS && h->cfg.num_vq <= 8;
}
static bool use_flow(const ctb_gpt* h) { return !h->engine && flow_for(h, h->B, h->use_tc); }
static bool flow_ink(const ctb_gpt* h) { return !h->engine && ink_for(h, h->B, h->infer_text, h->use_tc); }

extern "C" int ctb_gpt_step_kind(const ctb_gpt* h, int32_t B, int32_t infer_text) {
  if (!h) return set_err(CTB_ERR_ARG, "null argument");
  if (B < 1 || B > h->cfg.max_batch) return set_err(CTB_ERR_ARG, "B=%d outside [1,%d]", B, h->cfg.max_batch);
  const bool tc = tc_for(h, B);
  if (ink_for(h, B, infer_text != 0, tc)) return CTB_STEP_FLOW_INK;
  if (flow_for(h, B, tc)) return CTB_STEP_FLOW;
  if (mega_for(h, B, tc)) return CTB_STEP_MEGA;
  return tc ? CTB_STEP_WGMMA : CTB_STEP_FMA;
}

static int launch_finalize(ctb_gpt* h, cudaStream_t s) {
  const ctb_gpt_config& c = h->cfg;
  FinalP fp{};
  fp.st = h->st; fp.B = h->B; fp.rows_per_item = h->infer_text ? 1 : c.num_vq; fp.num_vq = c.num_vq;
  fp.max_new = h->max_new; fp.eos = h->sampler.eos_token; fp.idx = h->idx; fp.ids_out = h->ids_out;
  fp.finish = h->finish; fp.end_idx = h->end_idx;
  if (h->engine) {
    fp.rows = h->rows; fp.want = h->phase; fp.idx_text = h->eng_text_idx;
    CTB_CUDA(launch_pdl(k_finalize_rows, dim3(1), dim3(256), 0, s, fp));
  } else {
    CTB_CUDA(launch_pdl(k_finalize, dim3(1), dim3(256), 0, s, fp));
  }
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

// One loop iteration.  col >= 0: prefill column `col` of the prompt; col < 0: decode step.
// sample: run heads + sampler + finalize (last prompt column and every decode step).
static int enqueue_step(ctb_gpt* h, int col, bool sample, cudaStream_t s) {
  const ctb_gpt_config& c = h->cfg;
  const ctb_gpt_layout& L = h->lay;
  const int decode = col < 0;
  int rc;

  if (use_flow(h) || (!h->engine && mega_for(h, h->B, h->use_tc))) {
    // small batches: the whole step (input -> 20 layers -> heads) is one persistent cooperative kernel
    if ((rc = use_flow(h) ? launch_step_flow(h, col, sample, s) : launch_step_mega(h, col, sample, s))) return rc;
    if (!sample) return CTB_OK;
    const StepCtx xm = make_ctx(h, decode);
    if ((rc = launch_sampler(h, xm, s))) return rc;
    FinalP fm{};
    fm.st = h->st; fm.B = h->B; fm.rows_per_item = h->infer_text ? 1 : c.num_vq; fm.num_vq = c.num_vq;
    fm.max_new = h->max_new; fm.eos = h->sampler.eos_token; fm.idx = h->idx; fm.ids_out = h->ids_out;
    fm.finish = h->finish; fm.end_idx = h->end_idx;
    CTB_CUDA(launch_pdl(k_finalize, dim3(1), dim3(256), 0, s, fm));
    CTB_LAUNCH_CHECK();
    return CTB_OK;
  }

  InputP ip{};
  ip.st = h->st; ip.decode = decode; ip.B = h->B; ip.d = c.hidden_size; ip.col = decode ? 0 : col; ip.T0 = h->T0;
  ip.emb = h->emb; ip.mask = h->mask;
  ip.emb_code = h->W + L.emb_code; ip.emb_text = h->W + L.emb_text;
  ip.ids_out = h->ids_out; ip.max_new = h->max_new; ip.num_vq = c.num_vq; ip.num_audio = c.num_audio_tokens;
  ip.infer_text = h->infer_text;
  ip.x = h->x; ip.seq_len = h->seq_len; ip.pos = h->pos; ip.active = h->active;
  ip.x_hi = h->use_tc ? h->x_hi : nullptr; ip.x_lo = h->use_tc ? h->x_lo : nullptr;
  ip.rows = h->engine ? h->rows : nullptr;
  CTB_CUDA(launch_pdl(k_input, dim3(h->B), dim3(256), 0, s, ip));
  CTB_LAUNCH_CHECK();

  const StepCtx x = make_ctx(h, decode);
  for (int l = 0; l < c.num_layers; ++l)
    for (int kind = 0; kind < 5; ++kind)
      if ((rc = (h->use_tc && kind != 1) ? launch_layer_kernel_tc(h, l, kind, s) : launch_layer_kernel(h, x, l, kind, s)))
        return rc;
  if (!sample) return CTB_OK;
  if ((rc = h->use_tc ? launch_heads_tc(h, s) : launch_heads(h, x, s))) return rc;
  if ((rc = launch_sampler(h, x, s))) return rc;
  return launch_finalize(h, s);
}

// Measurement hook (bench.py roofline): launch ONE kernel kind for every layer (20 launches over
// 20 different weight slabs, so nothing is L2-resident between launches) on the state left by the
// last generate call.  kind 0..4 as above, 5 = heads, 6 = sampler.  Results of a later decode are
// undefined after this call (the residual stream is overwritten); call ctb_gpt_begin again.
extern "C" int ctb_gpt_profile_kernel(ctb_gpt* h, int32_t kind, void* stream) {
  if (!h || !h->started) return set_err(CTB_ERR_STATE, "ctb_gpt_begin has not been called");
  cudaStream_t s = (cudaStream_t)stream;
  StepCtx x = make_ctx(h, 0);
  x.g.check_finished = 0; x.a.check_finished = 0;
  int rc;
  if (kind == 5) return h->use_tc ? launch_heads_tc(h, s) : launch_heads(h, x, s);
  if (kind == 6) return launch_sampler(h, x, s);
  if (kind == 8) {  // 16 decode iterations in ONE launch of the dataflow step kernel (sampling tail inside)
    if (!flow_ink(h)) return set_err(CTB_ERR_STATE, "multi-step dataflow kernel unavailable for this handle/batch");
    if (h->steps_enqueued + 16 > h->max_new || h->T0 + h->steps_enqueued + 16 > h->cfg.max_context)
      return set_err(CTB_ERR_STATE, "no room for 16 more steps (max_new / max_context reached)");
    h->steps_enqueued += 16;
    return launch_step_flow(h, -1, true, s, 16);
  }
  if (kind == 7) {  // the one-kernel decode step alone (context grows by one token per call)
    if (h->steps_enqueued >= h->max_new || h->T0 + h->steps_enqueued >= h->cfg.max_context)
      return set_err(CTB_ERR_STATE, "no room for another step (max_new / max_context reached)");
    h->steps_enqueued++;
    if (use_flow(h)) return launch_step_flow(h, -1, true, s, flow_ink(h) ? 1 : 0);
    if (!(h->mega_ok && h->B <= 8)) return set_err(CTB_ERR_STATE, "one-kernel step unavailable for this handle/batch");
    return launch_step_mega(h, -1, true, s);
  }
  for (int l = 0; l < h->cfg.num_layers; ++l)
    if ((rc = (h->use_tc && kind != 1) ? launch_layer_kernel_tc(h, l, kind, s) : launch_layer_kernel(h, x, l, kind, s)))
      return rc;
  return CTB_OK;
}

// ------------------------------------------------------------------ batched prefill
static int prefill_reserve(ctb_gpt* h, size_t rows) {
  const ctb_gpt_config& c = h->cfg;
  const size_t d = c.hidden_size, I = c.intermediate_size, nqkv = (size_t)(c.num_heads + 2 * c.num_kv_heads) * c.head_dim;
  int rc;
  if (!h->gw_hi && !(h->prec & CTB_ENGINE_FP16_WEIGHTS)) {  // a half-precision engine's prefill reads h->gw16
    const size_t n = (size_t)h->lay.layer_stride * c.num_layers;
    if ((rc = dalloc(&h->gw_hi, n))) return rc;
    if ((rc = dalloc(&h->gw_lo, n))) return rc;
    k_split_tf32_t<0><<<2048, 256>>>(h->W + h->lay.layer0, h->gw_hi, h->gw_lo, (int64_t)n);
    CTB_CUDA(cudaDeviceSynchronize());
  }
  if (!h->pf_ones) {
    if ((rc = dalloc(&h->pf_ones, 2 * I))) return rc;
    if ((rc = dalloc(&h->pf_zeros, 2 * I))) return rc;
    std::vector<float> ones(2 * I, 1.0f);
    CTB_CUDA(cudaMemcpy(h->pf_ones, ones.data(), ones.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  if (rows > h->pf_rows) {
    float** bufs[] = {&h->pf_resid, &h->pf_xn, &h->pf_qkv, &h->pf_q, &h->pf_attn, &h->pf_gu, &h->pf_h};
    for (float** b : bufs) if (*b) { cudaFree(*b); *b = nullptr; }
    if (h->pf_npre) { cudaFree(h->pf_npre); h->pf_npre = nullptr; }
    if (h->pf_nvalid) { cudaFree(h->pf_nvalid); h->pf_nvalid = nullptr; }
    if (h->pf_mask) { cudaFree(h->pf_mask); h->pf_mask = nullptr; }
    if ((rc = dalloc(&h->pf_resid, rows * d))) return rc;
    if ((rc = dalloc(&h->pf_xn, rows * d))) return rc;
    if ((rc = dalloc(&h->pf_qkv, rows * nqkv))) return rc;
    if ((rc = dalloc(&h->pf_q, rows * d))) return rc;
    if ((rc = dalloc(&h->pf_attn, rows * d))) return rc;
    if ((rc = dalloc(&h->pf_gu, rows * 2 * I))) return rc;
    if ((rc = dalloc(&h->pf_h, rows * I))) return rc;
    if ((rc = dalloc(&h->pf_npre, rows))) return rc;
    if ((rc = dalloc(&h->pf_nvalid, (size_t)std::max(h->cfg.max_batch, 2)))) return rc;
    if ((rc = dalloc(&h->pf_mask, rows))) return rc;
    h->pf_rows = rows;
  }
  return CTB_OK;
}

// The 20 layers over the B x T0 prompt columns in h->pf_resid (positions, mask and slots in pp), the prompt's K / V
// appended to the rows' pages.  attn(pp, l) launches layer l's causal attention.  append_kv == false: the queries
// alone, against the K / V already in the pages (the attention-map pass), which then stops after the last attention.
template <typename Attn>
static int prefill_layers(ctb_gpt* h, PrefillP& pp, Attn attn, cudaStream_t s, bool append_kv = true) {
  const ctb_gpt_config& c = h->cfg;
  const ctb_gpt_layout& L = h->lay;
  const int B = pp.B, T0 = pp.T0, M = B * T0;
  const int d = c.hidden_size, I = c.intermediate_size, nqkv = (c.num_heads + 2 * c.num_kv_heads) * c.head_dim;
  int rc;
  pp.Hq = c.num_heads; pp.Hkv = c.num_kv_heads; pp.hd = c.head_dim; pp.d = d;
  pp.npre = h->pf_npre; pp.nvalid = h->pf_nvalid; pp.qkv = h->pf_qkv; pp.q = h->pf_q; pp.block_table = h->block_table;
  pp.pages_per_row = h->pages_per_row; pp.rope_cos = h->W + L.rope_cos; pp.rope_sin = h->W + L.rope_sin;
  pp.permute_qk = h->use_tc ? 1 : 0; pp.attn = h->pf_attn; pp.scaling = 1.0f / sqrtf((float)c.head_dim);
  const int rms_blocks = (M + 7) / 8;
  // a half-precision engine: the rounded weights (norms folded in before rounding) with W_lo = 0 and unit norms
  const bool w16 = (h->prec & CTB_ENGINE_FP16_WEIGHTS) != 0, kv16 = (h->prec & CTB_ENGINE_FP16_KV) != 0;
  for (int l = 0; l < c.num_layers; ++l) {
    const int64_t lo = (int64_t)l * L.layer_stride;
    const float* Wl = h->W + L.layer0 + lo;
    const float *Whi = (w16 ? h->gw16 : h->gw_hi) + lo, *Wlo = w16 ? nullptr : h->gw_lo + lo;
    auto wlo = [&](int64_t off) { return w16 ? h->pf_wzero : Wlo + off; };
    pp.kv = kv_layer(h, l);
    k_rms_rows<<<rms_blocks, 256, 0, s>>>(h->pf_resid, w16 ? h->pf_ones : Wl + L.ln1, h->pf_xn, M, d, c.rms_eps);
    CTB_LAUNCH_CHECK();
    if ((rc = tc_gemm_launch<GE_NONE>(s, h->pf_xn, d, B, T0, nqkv, d, 1, d, 1, 0, Whi + L.wqkv, wlo(L.wqkv), nullptr,
                                      nullptr, nullptr, 0, h->pf_qkv, nqkv))) return rc;
    if (!append_kv) k_prefill_rope_q<<<dim3(T0, B), 256, 0, s>>>(pp);
    else if (kv16) k_prefill_rope_kv<__half><<<dim3(T0, B), 256, 0, s>>>(pp);
    else k_prefill_rope_kv<float><<<dim3(T0, B), 256, 0, s>>>(pp);
    CTB_LAUNCH_CHECK();
    attn(pp, l);
    CTB_LAUNCH_CHECK();
    if (!append_kv && l == c.num_layers - 1) break;
    if ((rc = tc_gemm_launch<GE_SCALE_RES>(s, h->pf_attn, d, B, T0, d, d, 1, d, 1, 0, Whi + L.wo, wlo(L.wo), h->pf_zeros,
                                           h->pf_ones, h->pf_resid, d, h->pf_resid, d))) return rc;
    k_rms_rows<<<rms_blocks, 256, 0, s>>>(h->pf_resid, w16 ? h->pf_ones : Wl + L.ln2, h->pf_xn, M, d, c.rms_eps);
    CTB_LAUNCH_CHECK();
    if ((rc = tc_gemm_launch<GE_NONE>(s, h->pf_xn, d, B, T0, 2 * I, d, 1, d, 1, 0, Whi + L.wgate_up, wlo(L.wgate_up),
                                      nullptr, nullptr, nullptr, 0, h->pf_gu, 2 * I))) return rc;
    k_silu_mul<<<(unsigned)(((size_t)M * I + 255) / 256), 256, 0, s>>>(h->pf_gu, h->pf_h, M, I);
    CTB_LAUNCH_CHECK();
    if ((rc = tc_gemm_launch<GE_SCALE_RES>(s, h->pf_h, I, B, T0, d, I, 1, I, 1, 0, Whi + L.wdown, wlo(L.wdown),
                                           h->pf_zeros, h->pf_ones, h->pf_resid, d, h->pf_resid, d))) return rc;
  }
  return CTB_OK;
}

// The last column of each of the B prefilled rows (width T0) becomes its decode row's state (seq_len = nvalid[b]), then
// heads -> sampler -> finalize give the first token of every row in state h->phase (the i == 0 iteration of gpt.py:394)
static int prefill_first_token(ctb_gpt* h, int B, int T0, const int* nvalid, const int* slot, cudaStream_t s) {
  int rc;
  k_prefill_finish<<<B, 256, 0, s>>>(h->pf_resid, h->x, h->use_tc ? h->x_hi : nullptr, h->use_tc ? h->x_lo : nullptr,
                                     nvalid, h->seq_len, h->pos, h->active, T0, h->cfg.hidden_size, slot);
  CTB_LAUNCH_CHECK();
  const StepCtx x = make_ctx(h, 0);
  if ((rc = h->use_tc ? launch_heads_tc(h, s) : launch_heads(h, x, s))) return rc;
  if ((rc = launch_sampler(h, x, s))) return rc;
  return launch_finalize(h, s);
}

// Columns [q0, q0 + n) of B prompts of T columns -> decode rows slots[b] (slots: host array, copied to h->eng_slot by
// the admission or written there by k_prefill_chunk_positions; nullptr: rows 0..B-1), whose pages hold columns [0, q0).
//   whole prompts (q0 = 0, n = T): left padded, the positions counted from `mask` [B, T] (device)
//   a chunk (mask == nullptr, B = 1): every column valid, positions q0 + j; q0, and n unless the chunk is the last, are
//     multiples of CTB_PREFILL_CHUNK_ALIGN, so each row and query is computed as in the one-call prefill of T columns
// Each query attends to keys 0 .. its position, read from the pages, with the kernel chosen by T: k_prefill_attn up to
// PF_ATT_MAX_T0, else k_prefill_attn_tiled.  The call that ends the prompts (q0 + n == T) then hands each row's last
// column to its decode row and samples the first token of every row in state h->phase (all h->B rows of a static batch;
// the admitted slots of a slot engine); an earlier chunk touches nothing but the pf_* scratch and the slot's pages.
// prefill_columns is the pass alone: it leaves every column's final residual in h->pf_resid [B * n, d].
static int prefill_columns(ctb_gpt* h, int B, int T, int q0, int n, const float* emb, const uint8_t* mask,
                           const int32_t* slots, cudaStream_t s) {
  const ctb_gpt_config& c = h->cfg;
  const int M = B * n;
  int rc;
  if ((rc = prefill_reserve(h, (size_t)M))) return rc;
  CTB_CUDA(cudaMemcpyAsync(h->pf_resid, emb, (size_t)M * c.hidden_size * sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (mask) k_prefill_positions<<<B, 32, 0, s>>>(mask, h->pf_npre, h->pf_nvalid, T);
  else k_prefill_chunk_positions<<<(n + 255) / 256, 256, 0, s>>>(h->pf_mask, h->pf_npre, h->pf_nvalid, h->eng_slot,
                                                                 slots[0], q0, n);
  CTB_LAUNCH_CHECK();
  PrefillP pp{};
  pp.B = B; pp.T0 = n; pp.mask = mask ? mask : h->pf_mask; pp.slot = slots ? h->eng_slot : nullptr;
  const bool kv16 = (h->prec & CTB_ENGINE_FP16_KV) != 0, tiled = T > PF_ATT_MAX_T0;
  if (tiled &&
      (rc = kv16 ? ensure_smem_attr((const void*)k_prefill_attn_tiled<__half>, PftSmem<__half>::BYTES)
                 : ensure_smem_attr((const void*)k_prefill_attn_tiled<float>, PftSmem<float>::BYTES)))
    return rc;
  auto attn = [&](const PrefillP& p, int) {
    if (tiled) {
      const dim3 tgrid((n + PFT_TILE - 1) / PFT_TILE, c.num_heads, B);
      if (kv16) k_prefill_attn_tiled<__half><<<tgrid, PFT_THREADS, PftSmem<__half>::BYTES, s>>>(p, q0);
      else k_prefill_attn_tiled<float><<<tgrid, PFT_THREADS, PftSmem<float>::BYTES, s>>>(p, q0);
    } else {
      const dim3 agrid((n + PF_ATT_WARPS - 1) / PF_ATT_WARPS, c.num_heads, B);
      const size_t smem = (size_t)PF_ATT_WARPS * (q0 + n) * sizeof(float);
      if (kv16) k_prefill_attn<__half><<<agrid, PF_ATT_WARPS * 32, smem, s>>>(p, q0);
      else k_prefill_attn<float><<<agrid, PF_ATT_WARPS * 32, smem, s>>>(p, q0);
    }
  };
  return prefill_layers(h, pp, attn, s);
}

static int prefill(ctb_gpt* h, int B, int T, int q0, int n, const float* emb, const uint8_t* mask,
                   const int32_t* slots, cudaStream_t s) {
  int rc;
  if ((rc = prefill_columns(h, B, T, q0, n, emb, mask, slots, s))) return rc;
  if (q0 + n < T) return CTB_OK;
  // a chunk's k_prefill_chunk_positions puts the row's token count q0 + n in nvalid[1]
  return prefill_first_token(h, B, n, mask ? h->pf_nvalid : h->pf_nvalid + 1, slots ? h->eng_slot : nullptr, s);
}

// Pages for B rows of up to `tokens` tokens each: grow the pool if needed (page = 16 tokens x K|V x heads x 64 values per
// layer, fp32 or fp16 by the call's CTB_ENGINE_FP16_KV bit; the pool is sized in bytes, so calls of either type reuse
// it) and assign row b the pages [b * need, (b + 1) * need) - kernels only ever see the block table.
static size_t pool_bytes(const ctb_gpt* h, size_t pages) { return pages * page_bytes(h) * h->cfg.num_layers; }

// A pool of `pages` pages of every layer in place of the current one, which kernels on s may still read (CTB_ERR_NOMEM,
// and no pool, when it does not fit); the callers keep a pool that serves them
static int kv_alloc(ctb_gpt* h, size_t pages, cudaStream_t s) {
  CTB_CUDA(cudaStreamSynchronize(s));
  if (h->kv) { cudaFree(h->kv); h->kv = nullptr; h->kv_bytes = 0; }
  if (cudaMalloc(reinterpret_cast<void**>(&h->kv), pool_bytes(h, pages)) != cudaSuccess) {
    cudaGetLastError();
    return set_err(CTB_ERR_NOMEM, "KV pool: %zu pages x %d layers (%.2f GB) do not fit", pages, h->cfg.num_layers,
                   (double)pool_bytes(h, pages) / 1e9);
  }
  h->kv_bytes = pool_bytes(h, pages);
  return CTB_OK;
}

static int kv_reserve(ctb_gpt* h, int B, int tokens, cudaStream_t s) {
  const size_t per_row = ((size_t)tokens + kPageTokens - 1) / kPageTokens;
  const size_t need = per_row * (size_t)B;
  if (pool_bytes(h, need) > h->kv_bytes) {
    if (int rc = kv_alloc(h, need + need / 8, s)) return rc;  // head-room against re-allocation on slightly longer calls
    CTB_CUDA(cudaMemsetAsync(h->kv, 0, h->kv_bytes, s));
    h->bt_B = 0;
  }
  h->kv_layer_elems = h->kv_bytes / pool_bytes(h, 1) * page_elems(h);
  if (h->bt_B == B && h->bt_per_row == per_row) return CTB_OK;  // table already describes this shape: nothing to upload
  std::vector<int> bt((size_t)B * h->pages_per_row, 0);
  for (int b = 0; b < B; ++b)
    for (size_t i = 0; i < per_row; ++i) bt[(size_t)b * h->pages_per_row + i] = (int)((size_t)b * per_row + i);
  CTB_CUDA(cudaMemcpyAsync(h->block_table, bt.data(), bt.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaStreamSynchronize(s));  // bt is a host temporary
  h->bt_B = B; h->bt_per_row = per_row;
  return CTB_OK;
}

static int check_sampler(const ctb_sampler_config& sc) {
  if (sc.past_window > 31 || sc.past_window < 0) return set_err(CTB_ERR_ARG, "past_window out of range");
  if (sc.min_tokens_to_keep < 1) return set_err(CTB_ERR_ARG, "min_tokens_to_keep must be >= 1");
  return CTB_OK;
}

// A new static batch or slot engine: the captured decode graphs were built for the old one, and the wgmma step's
// activation scratch starts from zeros (h->use_tc already chosen)
static int restart_decode(ctb_gpt* h, cudaStream_t s) {
  if (h->graph_exec) { cudaGraphExecDestroy(h->graph_exec); h->graph_exec = nullptr; }
  if (h->graph_exec_text) { cudaGraphExecDestroy(h->graph_exec_text); h->graph_exec_text = nullptr; }
  if (h->use_tc) {
    const size_t d = h->cfg.hidden_size, I = h->cfg.intermediate_size;
    float* z768[] = {h->x_hi, h->x_lo, h->attn_hi, h->attn_lo};
    for (float* zp : z768) CTB_CUDA(cudaMemsetAsync(zp, 0, h->tc_rows * d * sizeof(float), s));
    CTB_CUDA(cudaMemsetAsync(h->h_hi, 0, h->tc_rows * I * sizeof(float), s));
    CTB_CUDA(cudaMemsetAsync(h->h_lo, 0, h->tc_rows * I * sizeof(float), s));
  }
  return CTB_OK;
}

extern "C" int ctb_gpt_begin(ctb_gpt* h, int32_t B, int32_t T0, const float* emb_dev, const uint8_t* mask_dev,
                             const ctb_sampler_config* sampler, const float* q_noise_dev, int32_t max_new_token,
                             int32_t infer_text, int32_t* ids_out_dev, float* hiddens_out_dev, void* stream) {
  if (!h || !emb_dev || !mask_dev || !sampler || !ids_out_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (B < 1 || B > h->cfg.max_batch) return set_err(CTB_ERR_ARG, "B=%d outside [1,%d]", B, h->cfg.max_batch);
  if (T0 < 1 || max_new_token < 1 || T0 + max_new_token > h->cfg.max_context)
    return set_err(CTB_ERR_ARG, "T0=%d + max_new=%d exceeds max_context=%d", T0, max_new_token, h->cfg.max_context);
  int rc;
  if ((rc = check_sampler(*sampler))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  h->B = B; h->T0 = T0; h->max_new = max_new_token; h->infer_text = infer_text ? 1 : 0;
  h->engine = 0; h->phase = RS_RUNNING; h->prec = 0; h->pg_pages = 0;
  h->use_tc = tc_for(h, B);
  h->sampler = *sampler; h->q_noise = q_noise_dev; h->emb = emb_dev; h->mask = mask_dev;
  h->ids_out = ids_out_dev; h->hiddens_out = hiddens_out_dev;
  if ((rc = restart_decode(h, s)) || (rc = kv_reserve(h, B, T0 + max_new_token, s))) return rc;
  CTB_CUDA(cudaMemsetAsync(h->st, 0, sizeof(LoopState), s));
  CTB_CUDA(cudaMemsetAsync(h->seq_len, 0, sizeof(int) * h->bpad_max, s));
  CTB_CUDA(cudaMemsetAsync(h->finish, 0, h->bpad_max, s));
  CTB_CUDA(cudaMemsetAsync(h->end_idx, 0, sizeof(int) * h->bpad_max, s));
  CTB_CUDA(cudaMemsetAsync(h->counter, 0, sizeof(int) * h->cfg.max_batch * h->cfg.num_heads, s));
  if (h->flow_ok) {
    // the dataflow step numbers its launches from 1 within a generate() call: tag base and arrival counters restart
    static const unsigned e0 = FL_EPOCH_STEP;
    CTB_CUDA(cudaMemcpyAsync(h->flow_epoch, &e0, sizeof(e0), cudaMemcpyHostToDevice, s));
    CTB_CUDA(cudaMemsetAsync(h->flow_arena, 0, FL_ARENA_WORDS * sizeof(unsigned long long), s));
  }
  if (h->pf_enabled && T0 >= 8 && T0 <= 1024) {
    // whole prompt as token-parallel wgmma GEMMs (prefill.cuh)
    if ((rc = prefill(h, B, T0, 0, T0, emb_dev, mask_dev, nullptr, s))) return rc;
  } else {
    // short prompts: walk the columns through the decode kernels (left padding keeps every row's last prompt
    // token in the last column, like the reference's batches)
    for (int col = 0; col < T0; ++col)
      if ((rc = enqueue_step(h, col, col == T0 - 1, s))) return rc;
  }
  h->started = 1;
  h->steps_enqueued = 1;
  return CTB_OK;
}

extern "C" int ctb_gpt_decode(ctb_gpt* h, int32_t n_steps, void* stream) {
  if (!h || !h->started) return set_err(CTB_ERR_STATE, "ctb_gpt_begin has not been called");
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  // ids_out / hiddens_out hold max_new steps and the KV pages max_context tokens: never enqueue past either
  // (a slot engine's rows stop at their own max_new, checked against both at admission)
  if (!h->engine) n_steps = std::min(n_steps, h->max_new - h->steps_enqueued);
  if (n_steps <= 0) return CTB_OK;
  if (h->pg_pages) {  // a paged engine: every slot that may run must hold the positions these steps append
    for (int b = 0; b < h->B; ++b)
      if (h->slot[b].hi && (rc = check_writes(h, b, h->slot[b].hi, std::min(h->slot[b].hi + n_steps, h->slot[b].cap))))
        return rc;
    for (SlotRecord& r : h->slot)
      if (r.hi) r.hi = std::min(r.hi + n_steps, r.cap);
  }
  h->steps_enqueued += n_steps;
  if (flow_ink(h)) {
    // the whole loop body (step, sampling tail, finish bookkeeping) is inside k_flow: many iterations per launch
    const int per_launch = h->trace ? 1 : 64;
    for (int done = 0; done < n_steps; done += per_launch)
      if ((rc = launch_step_flow(h, -1, true, s, std::min(per_launch, n_steps - done)))) return rc;
    return CTB_OK;
  }
  // a slot engine with text slots replays the graph that carries the text head and sampler
  cudaGraphExec_t& graph_exec = (h->engine && h->eng_text) ? h->graph_exec_text : h->graph_exec;
  uint64_t& graph_kernels = (h->engine && h->eng_text) ? h->graph_kernels_text : h->graph_kernels;
  if (h->use_graph && !graph_exec) {
    // capture on a private stream (the caller's may be the legacy default stream, which cannot
    // be captured); the instantiated graph is then launched on the caller's stream
    cudaGraph_t graph;
    if (!h->cap_stream) CTB_CUDA(cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking));
    CTB_CUDA(cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal));
    const uint64_t before = g_launches.load();
    rc = enqueue_step(h, -1, true, h->cap_stream);
    graph_kernels = g_launches.load() - before;
    g_launches.store(before);  // captured, not launched
    cudaError_t e = cudaStreamEndCapture(h->cap_stream, &graph);
    if (rc) return rc;
    if (e != cudaSuccess) return set_err(CTB_ERR_CUDA, "graph capture failed: %s", cudaGetErrorString(e));
    CTB_CUDA(cudaGraphInstantiate(&graph_exec, graph, 0));
    cudaGraphDestroy(graph);
  }
  for (int i = 0; i < n_steps; ++i) {
    if (graph_exec) {
      CTB_CUDA(cudaGraphLaunch(graph_exec, s));
      g_launches.fetch_add(graph_kernels, std::memory_order_relaxed);
    } else if ((rc = enqueue_step(h, -1, true, s))) {
      return rc;
    }
  }
  return CTB_OK;
}

// ------------------------------------------------------------------ attention maps of a static batch
// A query-only teacher-forced pass: columns [q0, q0 + n) of the B rows go through the prefill layers, whose attention
// (k_attn_probs) reads the K / V the decode wrote and writes each layer's probabilities; no page is written.  Columns
// without a map row (padded prompt columns, steps after a row's end) are computed too and get their fill rows.  The
// pass touches only the pf_* scratch, which no decode step reads (a static batch's decode state is x, the pages,
// seq_len / pos / active, the loop state and the k_flow arena), and runs in chunks of at most AM_ROWS (row, column)
// pairs, so pf_* stays within that of a 2-row prompt of 1,024 columns.  It reads the rows' padding and end_idx on the
// device, so it never synchronises.
static constexpr int AM_ROWS = 2048;

extern "C" int ctb_gpt_attention_maps(ctb_gpt* h, int32_t B, int32_t T0, int32_t q0, int32_t n, const float* emb_dev,
                                      const uint8_t* mask_dev, float* out_dev, void* stream) {
  if (!h || !emb_dev || !mask_dev || !out_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (!h->started || h->engine) return set_err(CTB_ERR_STATE, "attention maps: no static batch in flight (ctb_gpt_begin)");
  if (B != h->B || T0 != h->T0) return set_err(CTB_ERR_ARG, "attention maps: B=%d T0=%d, the batch has B=%d T0=%d", B, T0, h->B, h->T0);
  const int fed = T0 + h->steps_enqueued - 1;  // columns fed by the steps enqueued so far
  if (n < 1 || q0 < 0 || (q0 < T0 && (q0 != 0 || n < T0)) || q0 + n > fed)
    return set_err(CTB_ERR_ARG, "attention maps: columns [%d, %d) are not whole steps of the %d columns fed", q0, q0 + n, fed);
  const ctb_gpt_config& c = h->cfg;
  if (c.head_dim != 64) return set_err(CTB_ERR_ARG, "attention maps: head_dim %d (64 supported)", c.head_dim);
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  // only ever raised past the 48 KB every kernel may use without the attribute
  const int probs_smem = (AM_SMEM_FLOATS + q0 + n) * (int)sizeof(float);
  if (probs_smem > 48 * 1024 && (rc = ensure_smem_attr((const void*)k_attn_probs, probs_smem))) return rc;
  const int chunk = std::max(1, AM_ROWS / B), d = c.hidden_size;
  AttnMapP ap{};
  ap.out = out_dev; ap.L = c.num_layers; ap.B = B; ap.Hq = c.num_heads; ap.Hkv = c.num_kv_heads; ap.T0 = T0; ap.q0 = q0;
  ap.block_table = h->block_table; ap.pages_per_row = h->pages_per_row; ap.scaling = 1.0f / sqrtf((float)c.head_dim);
  for (int a = q0; a < q0 + n; a += chunk) {
    const int nc = std::min(chunk, q0 + n - a);
    if ((rc = prefill_reserve(h, (size_t)B * nc))) return rc;
    CTB_CUDA(cudaMemcpy2DAsync(h->pf_resid, (size_t)nc * d * sizeof(float), emb_dev + (size_t)(a - q0) * d,
                               (size_t)n * d * sizeof(float), (size_t)nc * d * sizeof(float), B,
                               cudaMemcpyDeviceToDevice, s));
    k_attn_map_positions<<<B, 256, 0, s>>>(mask_dev, h->end_idx, T0, a, nc, h->pf_mask, h->pf_npre);
    CTB_LAUNCH_CHECK();
    PrefillP pp{};
    pp.B = B; pp.T0 = nc; pp.mask = h->pf_mask; pp.slot = nullptr;
    ap.a = a; ap.nc = nc; ap.q = h->pf_q; ap.attn = h->pf_attn; ap.mask = h->pf_mask; ap.npre = h->pf_npre;
    auto attn = [&](const PrefillP& p, int l) {
      ap.kv = p.kv; ap.layer = l;
      k_attn_probs<<<dim3(nc, c.num_heads, B), AM_THREADS, (size_t)probs_smem, s>>>(ap);
    };
    if ((rc = prefill_layers(h, pp, attn, s, /*append_kv=*/false))) return rc;
  }
  return CTB_OK;
}

// ------------------------------------------------------------------ teacher-forced scoring
// One causal prefill over the B x T columns of the rows to score (prompt, then the given tokens but the last), then the
// heads over the columns that predict a given token and k_token_logprob over their logits.  The heads run in chunks of
// at most SCORE_ROWS columns into one logits scratch: 173 MB for the text head's 21,178 columns.
static constexpr int SCORE_ROWS = 2048;

namespace ctb {
// The final RMSNorm (k_rms_rows' arithmetic: fp32 statistics, out = w * (x * rinv)) of prefill rows src[i] of `resid`
// into out row i, for i < n: one warp per row of 768
__global__ void __launch_bounds__(256) k_score_gather(const float* __restrict__ resid, const int* __restrict__ src, int n,
                                                      const float* __restrict__ w, float* __restrict__ out, int d,
                                                      float eps) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= n) return;
  const float4* xr = reinterpret_cast<const float4*>(resid + (size_t)src[row] * d);
  float4 v[6];
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    v[i] = xr[i * 32 + lane];
    ss = fmaf(v[i].x, v[i].x, ss); ss = fmaf(v[i].y, v[i].y, ss); ss = fmaf(v[i].z, v[i].z, ss); ss = fmaf(v[i].w, v[i].w, ss);
  }
  ss = warp_sum(ss);
  const float rinv = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fdiv_rn(ss, (float)d), eps)));
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(w) + i * 32 + lane);
    float4 o;
    o.x = __fmul_rn(g.x, __fmul_rn(v[i].x, rinv)); o.y = __fmul_rn(g.y, __fmul_rn(v[i].y, rinv));
    o.z = __fmul_rn(g.z, __fmul_rn(v[i].z, rinv)); o.w = __fmul_rn(g.w, __fmul_rn(v[i].w, rinv));
    reinterpret_cast<float4*>(out + (size_t)row * d)[i * 32 + lane] = o;
  }
}
}  // namespace ctb

// What scoring m columns with the code (text = 0) or text head needs: the head's tf32 hi / lo copies, the normed-column
// and logits scratch, and room for m source rows
static int score_setup(ctb_gpt* h, int text, size_t m) {
  const ctb_gpt_config& c = h->cfg;
  const size_t d = c.hidden_size, N = text ? (size_t)c.num_text_tokens : (size_t)c.num_vq * c.num_audio_tokens;
  int rc;
  if (!h->sc_head_hi[text]) {
    if ((rc = dalloc(&h->sc_head_hi[text], N * d)) || (rc = dalloc(&h->sc_head_lo[text], N * d))) {
      cudaFree(h->sc_head_hi[text]); cudaFree(h->sc_head_lo[text]);
      h->sc_head_hi[text] = h->sc_head_lo[text] = nullptr;
      return rc;
    }
    k_split_tf32_t<0><<<2048, 256>>>(h->W + (text ? h->lay.head_text : h->lay.head_code), h->sc_head_hi[text],
                                     h->sc_head_lo[text], (int64_t)(N * d));
    CTB_LAUNCH_CHECK();
    CTB_CUDA(cudaDeviceSynchronize());
  }
  if (!h->sc_xn && (rc = dalloc(&h->sc_xn, (size_t)SCORE_ROWS * d))) return rc;
  if (h->sc_logits_cols < N) {
    cudaFree(h->sc_logits); h->sc_logits = nullptr; h->sc_logits_cols = 0;
    if ((rc = dalloc(&h->sc_logits, (size_t)SCORE_ROWS * N))) return rc;
    h->sc_logits_cols = N;
  }
  if (h->sc_src_cap < m) {
    cudaFree(h->sc_src); h->sc_src = nullptr; h->sc_src_cap = 0;
    if ((rc = dalloc(&h->sc_src, m))) return rc;
    h->sc_src_cap = m;
  }
  return CTB_OK;
}

// ctb_gpt_score (n_top == 0) and ctb_gpt_score_ex
static int score_pass(ctb_gpt* h, int32_t B, int32_t T, const float* emb_dev, const int32_t* n_prompt, const int32_t* n_given,
                      const int32_t* targets_dev, int32_t infer_text, float* out_dev, int32_t n_top, int32_t* top_ids_dev,
                      float* top_lp_dev, void* stream) {
  if (!h || !emb_dev || !n_prompt || !n_given || !targets_dev || !out_dev) return set_err(CTB_ERR_ARG, "null argument");
  const ctb_gpt_config& c = h->cfg;
  if (B < 1 || B > c.max_batch) return set_err(CTB_ERR_ARG, "score: B=%d outside [1,%d]", B, c.max_batch);
  if (T < 8 || T > c.max_context)
    return set_err(CTB_ERR_ARG, "score: T=%d outside [8,%d]: left-pad shorter rows to 8", T, c.max_context);
  size_t m = 0;
  for (int b = 0; b < B; ++b) {
    if (n_prompt[b] < 1 || n_given[b] < 1 || (int64_t)n_prompt[b] + n_given[b] - 1 > T)
      return set_err(CTB_ERR_ARG, "score: row %d: prompt %d + given tokens %d - 1 outside [1,%d]", b, n_prompt[b],
                     n_given[b], T);
    m += (size_t)n_given[b];
  }
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  if (h->engine) {  // a slot engine's pages and decode state stay as they are while any slot has work
    std::vector<RowState> rows;
    if ((rc = read_rows(h, rows, s))) return rc;
    for (int b = 0; b < h->B; ++b) {
      if ((rc = check_not_generating(rows[b], b))) return rc;
      if (h->slot[b].chunk_T0) return set_err(CTB_ERR_STATE, "slot %d has a prompt in progress", b);
    }
  }
  if ((rc = score_setup(h, infer_text ? 1 : 0, m))) return rc;
  // the pass takes the handle as ctb_gpt_begin does: the pages and prefill scratch are the fp32 model's, so a static
  // batch or slot engine before it is over (ctb_gpt_decode, ctb_gpt_status_query, ... CTB_ERR_STATE until the next begin)
  h->started = 0; h->engine = 0; h->prec = 0; h->pg_pages = 0; h->use_tc = false;
  if ((rc = kv_reserve(h, B, T, s)) || (rc = prefill_reserve(h, (size_t)B * T))) return rc;
  std::vector<uint8_t> mask((size_t)B * T, 0);  // row b: left padded, its P + n - 1 columns at the end
  std::vector<int> src(m);                      // the prefill row of each scored column, rows in order
  for (int b = 0, r = 0; b < B; ++b) {
    const int pad = T - (n_prompt[b] + n_given[b] - 1);
    memset(mask.data() + (size_t)b * T + pad, 1, (size_t)(T - pad));
    for (int j = 0; j < n_given[b]; ++j) src[r++] = b * T + pad + n_prompt[b] - 1 + j;
  }
  CTB_CUDA(cudaMemcpyAsync(h->pf_mask, mask.data(), mask.size(), cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaMemcpyAsync(h->sc_src, src.data(), m * sizeof(int), cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaStreamSynchronize(s));  // host temporaries
  if ((rc = prefill_columns(h, B, T, 0, T, emb_dev, h->pf_mask, nullptr, s))) return rc;
  const int rpi = infer_text ? 1 : c.num_vq, V = infer_text ? c.num_text_tokens : c.num_audio_tokens, N = rpi * V;
  const int d = c.hidden_size, k = infer_text ? 1 : 0;
  for (size_t r0 = 0; r0 < m; r0 += SCORE_ROWS) {
    const int mc = (int)std::min((size_t)SCORE_ROWS, m - r0);
    k_score_gather<<<(mc + 7) / 8, 256, 0, s>>>(h->pf_resid, h->sc_src + r0, mc, h->W + h->lay.final_norm, h->sc_xn, d,
                                                c.rms_eps);
    CTB_LAUNCH_CHECK();
    if ((rc = tc_gemm_launch<GE_NONE>(s, h->sc_xn, d, 1, mc, N, d, 1, d, 1, 0, h->sc_head_hi[k], h->sc_head_lo[k],
                                      nullptr, nullptr, nullptr, 0, h->sc_logits, N)))
      return rc;
    LogprobP lp{};
    lp.logits = h->sc_logits; lp.V = V; lp.rows_per_item = 1; lp.idx = targets_dev + r0 * rpi; lp.out = out_dev + r0 * rpi;
    CTB_CUDA(launch_pdl(k_token_logprob, dim3((unsigned)(mc * rpi)), dim3(LOGPROB_THREADS), 0, s, lp));
    CTB_LAUNCH_CHECK();
    if (n_top) {
      TopLogprobP tp{};
      tp.logits = h->sc_logits; tp.V = V; tp.rows_per_item = 1; tp.n_top = n_top;
      tp.ids = top_ids_dev + r0 * rpi * n_top; tp.lp = top_lp_dev + r0 * rpi * n_top;
      if ((rc = launch_top_logprobs(tp, mc * rpi, s))) return rc;
    }
  }
  return CTB_OK;
}

extern "C" int ctb_gpt_score(ctb_gpt* h, int32_t B, int32_t T, const float* emb_dev, const int32_t* n_prompt,
                             const int32_t* n_given, const int32_t* targets_dev, int32_t infer_text, float* out_dev,
                             void* stream) {
  return score_pass(h, B, T, emb_dev, n_prompt, n_given, targets_dev, infer_text, out_dev, 0, nullptr, nullptr, stream);
}

extern "C" int ctb_gpt_score_ex(ctb_gpt* h, int32_t B, int32_t T, const float* emb_dev, const int32_t* n_prompt,
                                const int32_t* n_given, const int32_t* targets_dev, int32_t infer_text, float* out_dev,
                                int32_t n_top, int32_t* top_ids_dev, float* top_lp_dev, void* stream) {
  if (!top_ids_dev || !top_lp_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (n_top < 1 || n_top > TOP_LOGPROBS_MAX) return set_err(CTB_ERR_ARG, "N=%d outside [1,%d]", n_top, TOP_LOGPROBS_MAX);
  return score_pass(h, B, T, emb_dev, n_prompt, n_given, targets_dev, infer_text, out_dev, n_top, top_ids_dev,
                    top_lp_dev, stream);
}

// ------------------------------------------------------------------ slot engine (continuous batching)
extern "C" int ctb_gpt_engine_begin(ctb_gpt* h, int32_t S, int32_t max_new_cap, int32_t* ids_out_dev,
                                    float* hiddens_out_dev, void* stream) {
  return ctb_gpt_engine_begin_ex(h, S, max_new_cap, 0, ids_out_dev, hiddens_out_dev, stream);
}

static_assert((int)TD_W16 == CTB_ENGINE_FP16_WEIGHTS && (int)TD_KV16 == CTB_ENGINE_FP16_KV, "precision bits");

static int kv_pool_paged(ctb_gpt* h, int S, int pool_pages, cudaStream_t s);

// ctb_gpt_engine_begin_ex (pool_pages == 0) and ctb_gpt_engine_begin_paged
static int engine_begin(ctb_gpt* h, int32_t S, int32_t max_new_cap, int32_t flags, int32_t pool_pages,
                        int32_t* ids_out_dev, float* hiddens_out_dev, void* stream) {
  if (!h || !ids_out_dev) return set_err(CTB_ERR_ARG, "null argument");
  const ctb_gpt_config& c = h->cfg;
  if (S < 2 || S > c.max_batch) return set_err(CTB_ERR_ARG, "S=%d outside [2,%d]", S, c.max_batch);
  if (max_new_cap < 1 || max_new_cap >= c.max_context)
    return set_err(CTB_ERR_ARG, "max_new_cap=%d outside [1,%d)", max_new_cap, c.max_context);
  if (flags & ~(CTB_ENGINE_FP16_WEIGHTS | CTB_ENGINE_FP16_KV)) return set_err(CTB_ERR_ARG, "unknown engine flags 0x%x", flags);
  if (flags && S > 64) return set_err(CTB_ERR_ARG, "S=%d: a half-precision engine serves up to 64 slots", S);
  if (flags && getenv("CTB_GPT_FMA"))
    return set_err(CTB_ERR_ARG, "a half-precision engine runs on the wgmma step, which CTB_GPT_FMA=1 disables");
  cudaStream_t s = (cudaStream_t)stream;
  int rc;
  // the wgmma step serves every half-precision engine and fp32 engines of tc_min_batch..64 slots, whatever the handle's
  // max_batch (CTB_GPT_FMA=1 keeps fp32 engines on the PDL chain); wider fp32 engines run the chain
  const bool use_tc = flags ? true : getenv("CTB_GPT_FMA") == nullptr && S >= h->tc_min_batch && S <= 64;
  if (use_tc) {
    // build what this handle lacks (a handle whose max_batch is below 9 or above 32 has no tensor-core state yet)
    if ((flags & CTB_ENGINE_FP16_WEIGHTS) ? (rc = fp16_setup(h)) : (!h->tc_wqkv && (rc = tc_setup(h)))) return rc;
    if ((flags & CTB_ENGINE_FP16_KV) && !(flags & CTB_ENGINE_FP16_WEIGHTS) &&
        (rc = set_tc_attr<DE_QKV, CS_QKV, CTB_ENGINE_FP16_KV>()))
      return rc;
  }
  if (!h->rows) {
    if ((rc = dalloc(&h->rows, (size_t)h->bpad_max))) return rc;
    if ((rc = dalloc(&h->cfgs, (size_t)c.max_batch))) return rc;
    if ((rc = dalloc(&h->eng_noise, (size_t)c.max_batch * noise_stride(h)))) return rc;
    if ((rc = dalloc(&h->eng_slot, (size_t)c.max_batch))) return rc;
    if ((rc = dalloc(&h->eng_text_logits, (size_t)c.max_batch * c.num_text_tokens))) return rc;
    if ((rc = dalloc(&h->eng_text_idx, (size_t)c.max_batch))) return rc;
  }
  // S rows of audio codes or text, each slot owning a fixed page range of max_context tokens; PDL chain (S <= 8 or S > 64)
  // or wgmma step (9 <= S <= 64, and every half-precision engine) - the one-kernel steps are never selected (use_flow,
  // enqueue_step)
  h->engine = 1; h->phase = RS_RUNNING; h->prec = flags;
  h->B = S; h->T0 = 0; h->max_new = max_new_cap; h->infer_text = 0;
  h->use_tc = use_tc;
  h->q_noise = h->eng_noise; h->emb = nullptr; h->mask = nullptr;
  h->ids_out = ids_out_dev; h->hiddens_out = hiddens_out_dev; h->eng_text = 0; h->pg_pages = 0;
  h->eng_logprobs = nullptr; h->eng_served = 0;
  h->eng_top_n = 0; h->eng_top_ids = nullptr; h->eng_top_lp = nullptr;
  if ((rc = restart_decode(h, s)) ||
      (rc = pool_pages ? kv_pool_paged(h, S, pool_pages, s) : kv_reserve(h, S, c.max_context, s)))
    return rc;
  static const LoopState idle_state = {0, 1, 0, 0, 0};  // no running slot: decode steps are no-ops
  CTB_CUDA(cudaMemcpyAsync(h->st, &idle_state, sizeof(LoopState), cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaMemsetAsync(h->rows, 0, sizeof(RowState) * h->bpad_max, s));  // every slot RS_IDLE
  CTB_CUDA(cudaMemsetAsync(h->seq_len, 0, sizeof(int) * h->bpad_max, s));
  CTB_CUDA(cudaMemsetAsync(h->pos, 0, sizeof(int) * h->bpad_max, s));
  CTB_CUDA(cudaMemsetAsync(h->active, 0, h->bpad_max, s));
  CTB_CUDA(cudaMemsetAsync(h->finish, 0, h->bpad_max, s));
  CTB_CUDA(cudaMemsetAsync(h->end_idx, 0, sizeof(int) * h->bpad_max, s));
  CTB_CUDA(cudaMemsetAsync(h->counter, 0, sizeof(int) * c.max_batch * c.num_heads, s));
  CTB_CUDA(cudaMemsetAsync(h->x, 0, sizeof(float) * h->bpad_max * c.hidden_size, s));
  CTB_CUDA(cudaStreamSynchronize(s));  // idle_state is read by the copy engine
  h->slot.assign((size_t)S, SlotRecord{});
  h->started = 1;
  h->steps_enqueued = 0;
  return CTB_OK;
}

extern "C" int ctb_gpt_engine_begin_ex(ctb_gpt* h, int32_t S, int32_t max_new_cap, int32_t flags, int32_t* ids_out_dev,
                                       float* hiddens_out_dev, void* stream) {
  return engine_begin(h, S, max_new_cap, flags, 0, ids_out_dev, hiddens_out_dev, stream);
}

// Admit n requests into `slots` (host): prefill columns [q0, T0) of their prompts - whole prompts (q0 = 0) with
// `mask`, or the final chunk of one slot's prompt (mask == nullptr) - and sample their first tokens.  Every slot is
// validated before anything is written, so a refused call leaves the handle as it was; the host arrays are copied
// before the call returns (synchronised), so the caller may free them at once.
static int admit(ctb_gpt* h, int n, const int32_t* slots, int T0, int q0, const float* emb_dev, const uint8_t* mask_dev,
                 const ctb_sampler_config* samplers, const float* q_noise_dev, const int32_t* max_new, int text,
                 cudaStream_t s) {
  const ctb_gpt_config& c = h->cfg;
  const int S = h->B;
  int rc;
  std::vector<uint8_t> mask_h;  // the positions each whole prompt writes (its pages, and the prompt it can share)
  if (mask_dev) {
    mask_h.resize((size_t)n * T0);
    CTB_CUDA(cudaMemcpyAsync(mask_h.data(), mask_dev, mask_h.size(), cudaMemcpyDeviceToHost, s));
  }
  std::vector<RowState> rows;
  if ((rc = read_rows(h, rows, s))) return rc;
  std::vector<int> held((size_t)n, T0);  // positions [0, held[i]) of slot slots[i] after the prefill
  for (size_t j = 0; j < mask_h.size(); ++j) held[j / T0] -= mask_h[j] == 0;
  std::vector<char> taken((size_t)S, 0);
  for (int i = 0; i < n; ++i) {
    const int b = slots[i];
    const ctb_sampler_config& sc = samplers[i];
    if (b < 0 || b >= S || taken[b]) return set_err(CTB_ERR_ARG, "slot %d out of range or repeated", b);
    taken[b] = 1;
    if ((rc = check_not_generating(rows[b], b)) || (rc = check_max_new(h, b, T0, max_new[i])) ||
        (rc = check_sampler(sc)) || (rc = check_writes(h, b, q0, held[i])))
      return rc;
    RowState& r = rows[b];
    r.n_gen = 0; r.step = 0; r.state = RS_PENDING; r.max_new = max_new[i]; r.has_noise = q_noise_dev != nullptr;
    r.eos = sc.eos_token; r.text = text;
  }
  for (int i = 0; i < n; ++i) {
    SlotRecord& r = h->slot[slots[i]];
    r.chunk_T0 = 0;  // the slot's prompt in progress, if any, is dropped
    r.pr_len = held[i]; r.pr_W = T0;
    r.hi = held[i]; r.cap = held[i] + max_new[i] - 1;
  }
  CTB_CUDA(cudaMemcpyAsync(h->rows, rows.data(), sizeof(RowState) * rows.size(), cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaMemcpyAsync(h->eng_slot, slots, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
  const size_t nrow = text ? (size_t)c.num_text_tokens : (size_t)c.num_vq * c.num_audio_tokens;
  for (int i = 0; i < n; ++i) {
    const int b = slots[i];
    CTB_CUDA(cudaMemcpyAsync(h->cfgs + b, samplers + i, sizeof(ctb_sampler_config), cudaMemcpyHostToDevice, s));
    if (q_noise_dev)
      CTB_CUDA(cudaMemcpyAsync(h->eng_noise + b * noise_stride(h), q_noise_dev + i * nrow, nrow * sizeof(float),
                               cudaMemcpyDeviceToDevice, s));
    CTB_CUDA(cudaMemsetAsync(h->finish + b, 0, 1, s));
    CTB_CUDA(cudaMemsetAsync(h->end_idx + b, 0, sizeof(int), s));
  }
  CTB_CUDA(cudaStreamSynchronize(s));
  // prompts -> their slots' pages, then heads / sampler / finalize for the RS_PENDING rows only
  if (text) h->eng_text = 1;
  h->eng_served = 1;
  h->phase = RS_PENDING;
  rc = prefill(h, n, T0, q0, T0 - q0, emb_dev, mask_dev, slots, s);
  h->phase = RS_RUNNING;
  return rc;
}

static int engine_admit(ctb_gpt* h, int32_t n, const int32_t* slots, int32_t T0, const float* emb_dev,
                        const uint8_t* mask_dev, const ctb_sampler_config* samplers, const float* q_noise_dev,
                        const int32_t* max_new, int text, void* stream) {
  if (!h || !slots || !emb_dev || !mask_dev || !samplers || !max_new) return set_err(CTB_ERR_ARG, "null argument");
  if (int rc = check_engine(h)) return rc;
  if (n < 1 || n > h->B) return set_err(CTB_ERR_ARG, "n=%d outside [1,%d]", n, h->B);
  if (int rc = check_T0(h, T0)) return rc;
  return admit(h, n, slots, T0, 0, emb_dev, mask_dev, samplers, q_noise_dev, max_new, text, (cudaStream_t)stream);
}

extern "C" int ctb_gpt_engine_admit(ctb_gpt* h, int32_t n, const int32_t* slots, int32_t T0, const float* emb_dev,
                                    const uint8_t* mask_dev, const ctb_sampler_config* samplers,
                                    const float* q_noise_dev, const int32_t* max_new, void* stream) {
  return engine_admit(h, n, slots, T0, emb_dev, mask_dev, samplers, q_noise_dev, max_new, 0, stream);
}

extern "C" int ctb_gpt_engine_admit_text(ctb_gpt* h, int32_t n, const int32_t* slots, int32_t T0, const float* emb_dev,
                                         const uint8_t* mask_dev, const ctb_sampler_config* samplers,
                                         const float* q_noise_dev, const int32_t* max_new, void* stream) {
  return engine_admit(h, n, slots, T0, emb_dev, mask_dev, samplers, q_noise_dev, max_new, 1, stream);
}

extern "C" int ctb_gpt_engine_prefill_chunk(ctb_gpt* h, int32_t slot, int32_t T0, int32_t c0, int32_t n,
                                            const float* emb_dev, int32_t text, const ctb_sampler_config* sampler,
                                            const float* q_noise_dev, int32_t max_new, void* stream) {
  if (!h || !emb_dev) return set_err(CTB_ERR_ARG, "null argument");
  int rc;
  if ((rc = check_engine(h))) return rc;
  if (slot < 0 || slot >= h->B) return set_err(CTB_ERR_ARG, "slot %d outside [0,%d)", slot, h->B);
  if ((rc = check_T0(h, T0))) return rc;
  if (c0 < 0 || n < 1 || c0 + n > T0) return set_err(CTB_ERR_ARG, "chunk [%d,%d) outside the prompt [0,%d)", c0, c0 + n, T0);
  const bool final = c0 + n == T0;
  if (c0 % CTB_PREFILL_CHUNK_ALIGN || (!final && n % CTB_PREFILL_CHUNK_ALIGN))
    return set_err(CTB_ERR_ARG, "chunk [%d,%d): c0 and a non-final chunk's n must be multiples of %d", c0, c0 + n,
                   CTB_PREFILL_CHUNK_ALIGN);
  if ((rc = check_max_new(h, slot, T0, max_new))) return rc;
  if (final) {
    if (!sampler) return set_err(CTB_ERR_ARG, "null sampler on the final chunk");
    if ((rc = check_sampler(*sampler))) return rc;
  }
  SlotRecord& rec = h->slot[slot];
  const int pT0 = rec.chunk_T0, pdone = rec.chunk_done;
  if (pT0 == 0 && c0 != 0)
    return set_err(CTB_ERR_STATE, "slot %d: chunk [%d,%d) but no prompt in progress (a first chunk starts at 0)", slot,
                   c0, c0 + n);
  if (pT0 != 0 && (T0 != pT0 || c0 != pdone))
    return set_err(CTB_ERR_STATE, "slot %d: chunk [%d,%d) of T0=%d does not continue the prompt in progress ([0,%d) of "
                   "T0=%d done)", slot, c0, c0 + n, T0, pdone, pT0);
  cudaStream_t s = (cudaStream_t)stream;
  // the final chunk admits the request as ctb_gpt_engine_admit / _admit_text do for one slot
  if (final) return admit(h, 1, &slot, T0, c0, emb_dev, nullptr, sampler, q_noise_dev, &max_new, text ? 1 : 0, s);
  std::vector<RowState> rows;
  if ((rc = read_rows(h, rows, s)) || (rc = check_not_generating(rows[slot], slot)) ||
      (rc = check_writes(h, slot, c0, c0 + n)))
    return rc;
  rec.pr_len = 0;  // its pages now hold part of a prompt
  h->eng_served = 1;
  if ((rc = prefill(h, 1, T0, c0, n, emb_dev, nullptr, &slot, s))) { rec.chunk_T0 = 0; return rc; }
  rec.chunk_T0 = T0; rec.chunk_done = c0 + n;
  return CTB_OK;
}

extern "C" int ctb_gpt_engine_logprobs(ctb_gpt* h, float* logprobs_out_dev, void* stream) {
  if (!h || !logprobs_out_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (int rc = check_engine(h)) return rc;
  if (h->eng_served)
    return set_err(CTB_ERR_STATE, "the engine has served a request: attach the log-probability buffer right after begin");
  CTB_CUDA(cudaMemsetAsync(logprobs_out_dev, 0, (size_t)h->B * h->max_new * h->cfg.num_vq * sizeof(float),
                           (cudaStream_t)stream));
  h->eng_logprobs = logprobs_out_dev;
  // decode graphs captured so far (steps of the idle engine) lack the k_token_logprob nodes
  if (h->graph_exec) { cudaGraphExecDestroy(h->graph_exec); h->graph_exec = nullptr; }
  if (h->graph_exec_text) { cudaGraphExecDestroy(h->graph_exec_text); h->graph_exec_text = nullptr; }
  return CTB_OK;
}

extern "C" int ctb_gpt_engine_top_logprobs(ctb_gpt* h, int32_t n_top, int32_t* ids_out_dev, float* lp_out_dev,
                                           void* stream) {
  if (!h || !ids_out_dev || !lp_out_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (n_top < 1 || n_top > TOP_LOGPROBS_MAX) return set_err(CTB_ERR_ARG, "N=%d outside [1,%d]", n_top, TOP_LOGPROBS_MAX);
  if (int rc = check_engine(h)) return rc;
  if (h->eng_served)
    return set_err(CTB_ERR_STATE, "the engine has served a request: attach the top log-probability buffers right after begin");
  const size_t n = (size_t)h->B * h->max_new * h->cfg.num_vq * n_top;
  cudaStream_t s = (cudaStream_t)stream;
  CTB_CUDA(cudaMemsetAsync(ids_out_dev, 0, n * sizeof(int32_t), s));
  CTB_CUDA(cudaMemsetAsync(lp_out_dev, 0, n * sizeof(float), s));
  h->eng_top_n = n_top; h->eng_top_ids = ids_out_dev; h->eng_top_lp = lp_out_dev;
  // decode graphs captured so far (steps of the idle engine) lack the k_token_top_logprobs nodes
  if (h->graph_exec) { cudaGraphExecDestroy(h->graph_exec); h->graph_exec = nullptr; }
  if (h->graph_exec_text) { cudaGraphExecDestroy(h->graph_exec_text); h->graph_exec_text = nullptr; }
  return CTB_OK;
}

extern "C" int ctb_gpt_engine_status(ctb_gpt* h, ctb_gpt_status* out, int32_t* state_host, int32_t* end_idx_host,
                                     uint8_t* finish_host, void* stream) {
  if (!h || !out) return set_err(CTB_ERR_ARG, "null argument");
  if (int rc = check_engine(h)) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<RowState> rows((size_t)h->B);
  CTB_CUDA(cudaMemcpyAsync(rows.data(), h->rows, sizeof(RowState) * h->B, cudaMemcpyDeviceToHost, s));
  if (int rc = ctb_gpt_status_query(h, out, end_idx_host, finish_host, stream)) return rc;  // synchronises `stream`
  if (state_host)
    for (int b = 0; b < h->B; ++b) state_host[b] = rows[b].state;
  for (int b = 0; b < h->B; ++b)  // a slot seen idle or finished appends nothing until its next admission
    if (rows[b].state != RS_RUNNING && rows[b].state != RS_PENDING) h->slot[b].hi = 0;
  if (h->eng_text) {  // the stream is synchronised: the rows are current
    h->eng_text = 0;
    for (int b = 0; b < h->B; ++b)
      if (rows[b].text && (rows[b].state == RS_RUNNING || rows[b].state == RS_PENDING)) h->eng_text = 1;
  }
  return CTB_OK;
}

extern "C" int ctb_gpt_engine_cancel(ctb_gpt* h, int32_t n, const int32_t* slots, void* stream) {
  if (!h || !slots) return set_err(CTB_ERR_ARG, "null argument");
  int rc;
  if ((rc = check_engine(h)) || (rc = check_slot_list(h, n, slots))) return rc;
  const int S = h->B;
  if (S > CANCEL_MAX_SLOTS) return set_err(CTB_ERR_ARG, "S=%d: cancellation serves up to %d slots", S, CANCEL_MAX_SLOTS);
  CancelP p{};
  p.st = h->st; p.rows = h->rows; p.finish = h->finish; p.B = S;
  for (int i = 0; i < n; ++i) {
    p.mask[slots[i] >> 5] |= 1u << (slots[i] & 31);
    h->slot[slots[i]].chunk_T0 = 0;  // a prompt in progress there is dropped
  }
  // h->eng_text stays as it is: the next ctb_gpt_engine_status recomputes it from the rows
  k_cancel_rows<<<1, 256, 0, (cudaStream_t)stream>>>(p);
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

// ------------------------------------------------------------------ KV pages on demand (ctb_gpt_engine_begin_paged)
static_assert(sizeof(RowState) == 8 * sizeof(int32_t), "ctb_slot_image.row");

static unsigned move_blocks(size_t words) { return (unsigned)std::min<size_t>((words + 255) / 256, (size_t)g_num_sms * 8); }

// the poison pattern (quiet NaN of the cache's element type) into n pages of every layer: list[0..n), or p0 .. p0 + n - 1
static int kv_poison(ctb_gpt* h, const int* list, int p0, int n, cudaStream_t s) {
  KvFillP p{};
  p.kv = reinterpret_cast<char*>(h->kv); p.layer_bytes = h->kv_layer_elems * kv_elem_bytes(h);
  p.page_bytes = page_bytes(h); p.layers = h->cfg.num_layers; p.p0 = p0; p.use_list = list != nullptr;
  p.word = (h->prec & CTB_ENGINE_FP16_KV) ? 0x7e007e00u : 0x7fc00000u;
  for (int k = 0; k < n; k += KV_BT_MAX) {
    p.n = std::min(KV_BT_MAX, n - k);
    if (list) std::copy(list + k, list + k + p.n, p.list);
    else p.p0 = p0 + k;
    k_kv_fill<<<move_blocks((size_t)p.layers * p.n * p.page_bytes / 16), 256, 0, s>>>(p);
    CTB_LAUNCH_CHECK();
  }
  return CTB_OK;
}

// block-table entries (index into [S][pages_per_row], page), KV_BT_MAX per launch
static int bt_write(ctb_gpt* h, const std::vector<std::pair<int, int>>& e, cudaStream_t s) {
  BtWriteP p{};
  p.bt = h->block_table;
  for (size_t k = 0; k < e.size(); k += KV_BT_MAX) {
    p.n = (int)std::min<size_t>(KV_BT_MAX, e.size() - k);
    for (int j = 0; j < p.n; ++j) { p.idx[j] = e[k + j].first; p.page[j] = e[k + j].second; }
    k_bt_write<<<1, 256, 0, s>>>(p);
    CTB_LAUNCH_CHECK();
  }
  return CTB_OK;
}

// Slot b's next block-table entry onto `page` (another entry's) or, for page < 0, the back of the free list: the page's
// count goes up and the entry joins e, for bt_write.  With unmap_slot, the only writer of pg_free, pg_bt and pg_ref.
static void map_page(ctb_gpt* h, int b, int page, std::vector<std::pair<int, int>>& e) {
  if (page < 0) { page = h->pg_free.back(); h->pg_free.pop_back(); }
  if (++h->pg_ref[page] == 2) ++h->pg_shared;
  const int idx = b * h->pages_per_row + h->slot[b].pages++;
  h->pg_bt[idx] = page;
  e.emplace_back(idx, page);
}

// Every entry of slot b onto the zero page (joining e, for bt_write): each page's count goes down, and a page no entry
// maps any more returns to the free list, to be taken again in the order it had.  Returns those pages.
static std::vector<int> unmap_slot(ctb_gpt* h, int b, std::vector<std::pair<int, int>>& e) {
  std::vector<int> freed;
  for (int k = 0; k < h->slot[b].pages; ++k) {
    const int idx = b * h->pages_per_row + k;
    const int page = h->pg_bt[idx];
    if (--h->pg_ref[page] == 0) freed.push_back(page);
    else if (h->pg_ref[page] == 1) --h->pg_shared;
    h->pg_bt[idx] = 0;
    e.emplace_back(idx, 0);
  }
  h->pg_free.insert(h->pg_free.end(), freed.rbegin(), freed.rend());
  h->slot[b].pages = 0;
  return freed;
}

// A pool of exactly pool_pages pages, zeroed (poisoned past the zero page with CTB_KV_POISON=1), every entry of the S
// slots' block table on the zero page and every other page free
static int kv_pool_paged(ctb_gpt* h, int S, int pool_pages, cudaStream_t s) {
  int rc;
  if (pool_bytes(h, pool_pages) != h->kv_bytes && (rc = kv_alloc(h, pool_pages, s))) return rc;
  h->kv_layer_elems = (size_t)pool_pages * page_elems(h);
  h->bt_B = 0;  // kv_reserve uploads its table again
  CTB_CUDA(cudaMemsetAsync(h->kv, 0, h->kv_bytes, s));
  const char* poison = getenv("CTB_KV_POISON");
  h->pg_poison = poison != nullptr && atoi(poison) == 1;
  if (h->pg_poison && (rc = kv_poison(h, nullptr, 1, pool_pages - 1, s))) return rc;
  CTB_CUDA(cudaMemsetAsync(h->block_table, 0, sizeof(int) * (size_t)S * h->pages_per_row, s));
  h->pg_free.clear();
  for (int p = pool_pages - 1; p >= 1; --p) h->pg_free.push_back(p);
  h->pg_bt.assign((size_t)S * h->pages_per_row, 0);
  h->pg_ref.assign((size_t)pool_pages, 0);
  h->pg_pages = pool_pages; h->pg_shared = 0;
  return CTB_OK;
}

extern "C" int ctb_gpt_engine_begin_paged(ctb_gpt* h, int32_t S, int32_t max_new_cap, int32_t flags, int32_t pool_pages,
                                          int32_t* ids_out_dev, float* hiddens_out_dev, void* stream) {
  if (!h) return set_err(CTB_ERR_ARG, "null argument");
  if (pool_pages < 2) return set_err(CTB_ERR_ARG, "pool_pages=%d: the zero page and at least one more", pool_pages);
  if (h->pages_per_row > KV_MOVE_MAX_PAGES)
    return set_err(CTB_ERR_ARG, "max_context=%d: a paged engine serves up to %d tokens per slot", h->cfg.max_context,
                   KV_MOVE_MAX_PAGES * kPageTokens);
  return engine_begin(h, S, max_new_cap, flags, pool_pages, ids_out_dev, hiddens_out_dev, stream);
}

extern "C" int ctb_gpt_engine_reserve(ctb_gpt* h, int32_t n, const int32_t* slots, const int32_t* tokens, void* stream) {
  if (!h || !slots || !tokens) return set_err(CTB_ERR_ARG, "null argument");
  int rc;
  if ((rc = check_paged(h)) || (rc = check_slot_list(h, n, slots))) return rc;
  size_t need = 0;
  for (int i = 0; i < n; ++i) {
    if (tokens[i] < 0 || tokens[i] > h->cfg.max_context)
      return set_err(CTB_ERR_ARG, "slot %d: tokens=%d outside [0,%d]", slots[i], tokens[i], h->cfg.max_context);
    need += (size_t)std::max(0, (tokens[i] + kPageTokens - 1) / kPageTokens - h->slot[slots[i]].pages);
  }
  if (need > h->pg_free.size())
    return set_err(CTB_ERR_POOL, "KV pool: %zu more pages needed, %zu of %d free", need, h->pg_free.size(),
                   h->pg_pages - 1);
  std::vector<std::pair<int, int>> e;
  for (int i = 0; i < n; ++i)
    while (h->slot[slots[i]].pages * kPageTokens < tokens[i]) map_page(h, slots[i], -1, e);
  return bt_write(h, e, (cudaStream_t)stream);
}

// slot b's pages and the positions they hold released, its prompt no longer shareable (neither caller leaves a prompt
// in progress there)
static int release_pages(ctb_gpt* h, int b, cudaStream_t s) {
  std::vector<std::pair<int, int>> e;
  const std::vector<int> freed = unmap_slot(h, b, e);
  h->slot[b] = SlotRecord{};
  int rc;
  if ((rc = bt_write(h, e, s))) return rc;
  return h->pg_poison ? kv_poison(h, freed.data(), 0, (int)freed.size(), s) : CTB_OK;
}

extern "C" int ctb_gpt_engine_release(ctb_gpt* h, int32_t n, const int32_t* slots, void* stream) {
  if (!h || !slots) return set_err(CTB_ERR_ARG, "null argument");
  int rc;
  if ((rc = check_paged(h)) || (rc = check_slot_list(h, n, slots))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<RowState> rows;
  if ((rc = read_rows(h, rows, s))) return rc;
  for (int i = 0; i < n; ++i) {
    if ((rc = check_not_generating(rows[slots[i]], slots[i])) || (rc = check_slot(h, slots[i]))) return rc;
  }
  for (int i = 0; i < n; ++i)
    if ((rc = release_pages(h, slots[i], s))) return rc;
  return CTB_OK;
}

extern "C" int ctb_gpt_engine_pages(ctb_gpt* h, int32_t* in_use, int32_t* shared) {
  if (!h || !in_use || !shared) return set_err(CTB_ERR_ARG, "null argument");
  if (int rc = check_paged(h)) return rc;
  *in_use = h->pg_pages - 1 - (int32_t)h->pg_free.size();  // every page but the zero page is mapped or free
  *shared = h->pg_shared;
  return CTB_OK;
}

// the sections of an image of n_gen tokens and seq_len positions on this engine, each 256-byte aligned
static void image_layout(const ctb_gpt* h, int n_gen, int seq_len, ctb_slot_image* img) {
  const ctb_gpt_config& c = h->cfg;
  auto up = [](uint64_t x) { return (x + 255) & ~(uint64_t)255; };
  img->magic = CTB_SLOT_IMAGE_MAGIC; img->prec = h->prec; img->n_gen = n_gen; img->seq_len = seq_len;
  img->npages = (seq_len + kPageTokens - 1) / kPageTokens; img->page_bytes = (int32_t)page_bytes(h);
  img->num_vq = c.num_vq; img->hidden_size = c.hidden_size; img->noise_floats = (int32_t)noise_stride(h);
  img->has_hidden = h->hiddens_out != nullptr;
  img->off_noise = up(sizeof(ctb_slot_image));
  img->off_ids = up(img->off_noise + (uint64_t)img->noise_floats * sizeof(float));
  img->off_hiddens = up(img->off_ids + (uint64_t)n_gen * c.num_vq * sizeof(int32_t));
  img->off_kv = up(img->off_hiddens + (img->has_hidden ? (uint64_t)n_gen * c.hidden_size * sizeof(float) : 0));
  img->bytes = img->off_kv + (uint64_t)c.num_layers * img->npages * img->page_bytes;
}

// slot's loop state and counters (synchronises s)
static int read_slot(ctb_gpt* h, int slot, ctb_slot_image* img, cudaStream_t s) {
  uint8_t fin = 0;
  CTB_CUDA(cudaMemcpyAsync(img->row, h->rows + slot, sizeof(RowState), cudaMemcpyDeviceToHost, s));
  CTB_CUDA(cudaMemcpyAsync(&img->seq_len, h->seq_len + slot, sizeof(int), cudaMemcpyDeviceToHost, s));
  CTB_CUDA(cudaMemcpyAsync(&img->pos, h->pos + slot, sizeof(int), cudaMemcpyDeviceToHost, s));
  CTB_CUDA(cudaMemcpyAsync(&img->end_idx, h->end_idx + slot, sizeof(int), cudaMemcpyDeviceToHost, s));
  CTB_CUDA(cudaMemcpyAsync(&fin, h->finish + slot, 1, cudaMemcpyDeviceToHost, s));
  CTB_CUDA(cudaStreamSynchronize(s));
  img->finish = fin;
  return CTB_OK;
}

// CTB_ERR_ARG unless host_buf is pinned host memory (the copies through it are asynchronous)
static int check_pinned(const void* host_buf) {
  void* p = nullptr;
  if (cudaHostGetDevicePointer(&p, const_cast<void*>(host_buf), 0) != cudaSuccess) {
    cudaGetLastError();
    return set_err(CTB_ERR_ARG, "the image buffer is not pinned host memory");
  }
  return CTB_OK;
}

static int launch_set_row(ctb_gpt* h, int slot, const RowState& r, cudaStream_t s) {
  SetRowP p{};
  p.st = h->st; p.rows = h->rows; p.B = h->B; p.b = slot; p.row = r;
  k_set_row<<<1, 256, 0, s>>>(p);
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

// A slot's KV pages <-> the image's KV section in pinned host memory, through the device staging buffer: as many
// image pages as it holds at a time, k_kv_pack into it and one cudaMemcpyAsync out (or one copy in and k_kv_unpack).
// Measured on an H100 (DESIGN.md §4): resumes this way took 25-30 % less time than k_kv_unpack reading mapped pinned
// memory directly, and one copy out of the staging buffer runs at about 40 GB/s.
static int kv_move(ctb_gpt* h, int slot, char* img, int npages, bool pack, cudaStream_t s) {
  if (npages == 0) return CTB_OK;
  int rc;
  if (!h->pg_stage && (rc = dalloc(&h->pg_stage, KV_STAGE_BYTES))) return rc;
  KvMoveP p{};
  p.kv = reinterpret_cast<char*>(h->kv); p.img = reinterpret_cast<uint4*>(h->pg_stage);
  p.layer_bytes = h->kv_layer_elems * kv_elem_bytes(h); p.page_words = (int)(page_bytes(h) / 16);
  p.layers = h->cfg.num_layers; p.npages = npages;
  for (int i = 0; i < npages; ++i) p.pages[i] = h->pg_bt[(size_t)slot * h->pages_per_row + i];
  const size_t pb = page_bytes(h);
  const int per = (int)(KV_STAGE_BYTES / pb), total = p.layers * npages;
  for (p.pg0 = 0; p.pg0 < total; p.pg0 = p.pg1) {
    p.pg1 = std::min(total, p.pg0 + per);
    const size_t bytes = (size_t)(p.pg1 - p.pg0) * pb;
    char* hp = img + (size_t)p.pg0 * pb;
    const unsigned grid = (unsigned)std::min(p.pg1 - p.pg0, g_num_sms * 4);
    if (pack) {
      k_kv_pack<<<grid, 256, 0, s>>>(p);
      CTB_LAUNCH_CHECK();
      CTB_CUDA(cudaMemcpyAsync(hp, h->pg_stage, bytes, cudaMemcpyDeviceToHost, s));
    } else {
      CTB_CUDA(cudaMemcpyAsync(h->pg_stage, hp, bytes, cudaMemcpyHostToDevice, s));
      k_kv_unpack<<<grid, 256, 0, s>>>(p);
      CTB_LAUNCH_CHECK();
    }
  }
  return CTB_OK;
}

// the running slot's state (synchronises s) and its image's layout
static int running_image(ctb_gpt* h, int slot, ctb_slot_image* img, cudaStream_t s) {
  int rc;
  if ((rc = check_paged(h)) || (rc = check_slot(h, slot)) || (rc = read_slot(h, slot, img, s))) return rc;
  RowState r;
  memcpy(&r, img->row, sizeof(r));
  if (r.state != RS_RUNNING) return set_err(CTB_ERR_STATE, "slot %d is not running (state %d)", slot, r.state);
  image_layout(h, r.n_gen, img->seq_len, img);
  return check_covers(h, slot, img->seq_len);
}

extern "C" int ctb_gpt_engine_suspend_bytes(ctb_gpt* h, int32_t slot, uint64_t* bytes, void* stream) {
  if (!h || !bytes) return set_err(CTB_ERR_ARG, "null argument");
  ctb_slot_image img{};
  int rc;
  if ((rc = running_image(h, slot, &img, (cudaStream_t)stream))) return rc;
  *bytes = img.bytes;
  return CTB_OK;
}

extern "C" int ctb_gpt_engine_suspend(ctb_gpt* h, int32_t slot, void* host_buf, uint64_t host_bytes, void* stream) {
  if (!h || !host_buf) return set_err(CTB_ERR_ARG, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  const ctb_gpt_config& c = h->cfg;
  ctb_slot_image img{};
  int rc;
  if ((rc = running_image(h, slot, &img, s)) || (rc = check_pinned(host_buf))) return rc;
  if (host_bytes < img.bytes)
    return set_err(CTB_ERR_ARG, "image buffer of %llu bytes, slot %d needs %llu", (unsigned long long)host_bytes, slot,
                   (unsigned long long)img.bytes);
  char* hb = static_cast<char*>(host_buf);
  memcpy(hb, &img, sizeof(img));  // the header; the device fills in the sampler and the sections
  const int n_gen = img.n_gen;
  CTB_CUDA(cudaMemcpyAsync(hb + offsetof(ctb_slot_image, sampler), h->cfgs + slot, sizeof(ctb_sampler_config),
                           cudaMemcpyDeviceToHost, s));
  CTB_CUDA(cudaMemcpyAsync(hb + img.off_noise, h->eng_noise + slot * noise_stride(h), img.noise_floats * sizeof(float),
                           cudaMemcpyDeviceToHost, s));
  CTB_CUDA(cudaMemcpyAsync(hb + img.off_ids, h->ids_out + (size_t)slot * h->max_new * c.num_vq,
                           (size_t)n_gen * c.num_vq * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
  if (img.has_hidden)
    CTB_CUDA(cudaMemcpyAsync(hb + img.off_hiddens, h->hiddens_out + (size_t)slot * h->max_new * c.hidden_size,
                             (size_t)n_gen * c.hidden_size * sizeof(float), cudaMemcpyDeviceToHost, s));
  if ((rc = kv_move(h, slot, hb + img.off_kv, img.npages, true, s)) || (rc = release_pages(h, slot, s)))
    return rc;
  return launch_set_row(h, slot, RowState{}, s);  // RS_IDLE
}

extern "C" int ctb_gpt_engine_resume(ctb_gpt* h, int32_t slot, const void* host_buf, uint64_t host_bytes, void* stream) {
  if (!h || !host_buf) return set_err(CTB_ERR_ARG, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  const ctb_gpt_config& c = h->cfg;
  int rc;
  if ((rc = check_paged(h)) || (rc = check_slot(h, slot)) || (rc = check_pinned(host_buf))) return rc;
  if (host_bytes < sizeof(ctb_slot_image)) return set_err(CTB_ERR_ARG, "image buffer of %llu bytes", (unsigned long long)host_bytes);
  const ctb_slot_image* img = static_cast<const ctb_slot_image*>(host_buf);
  RowState r;
  memcpy(&r, img->row, sizeof(r));
  ctb_slot_image want{};
  image_layout(h, img->n_gen, img->seq_len, &want);
  if (img->magic != want.magic || img->prec != want.prec || img->page_bytes != want.page_bytes ||
      img->num_vq != want.num_vq || img->hidden_size != want.hidden_size || img->noise_floats != want.noise_floats ||
      img->has_hidden != want.has_hidden || img->npages != want.npages || img->off_noise != want.off_noise ||
      img->off_ids != want.off_ids || img->off_hiddens != want.off_hiddens || img->off_kv != want.off_kv ||
      img->bytes != want.bytes || img->n_gen < 1 || img->seq_len < 1 || r.state != RS_RUNNING ||
      r.n_gen != img->n_gen || r.max_new > h->max_new)
    return set_err(CTB_ERR_ARG, "the buffer holds no slot image of this engine");
  if (host_bytes < img->bytes)
    return set_err(CTB_ERR_ARG, "image buffer of %llu bytes, the image has %llu", (unsigned long long)host_bytes,
                   (unsigned long long)img->bytes);
  std::vector<RowState> rows;
  if ((rc = check_writes(h, slot, 0, img->seq_len)) || (rc = read_rows(h, rows, s)) ||
      (rc = check_not_generating(rows[slot], slot)))
    return rc;
  h->slot[slot].pr_len = 0;  // the image does not record its prompt: a resumed request is no source to share from
  h->eng_served = 1;
  const char* hb = static_cast<const char*>(host_buf);
  const int n_gen = img->n_gen;
  CTB_CUDA(cudaMemcpyAsync(h->cfgs + slot, &img->sampler, sizeof(ctb_sampler_config), cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaMemcpyAsync(h->eng_noise + slot * noise_stride(h), hb + img->off_noise, img->noise_floats * sizeof(float),
                           cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaMemcpyAsync(h->ids_out + (size_t)slot * h->max_new * c.num_vq, hb + img->off_ids,
                           (size_t)n_gen * c.num_vq * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  if (img->has_hidden)
    CTB_CUDA(cudaMemcpyAsync(h->hiddens_out + (size_t)slot * h->max_new * c.hidden_size, hb + img->off_hiddens,
                             (size_t)n_gen * c.hidden_size * sizeof(float), cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaMemcpyAsync(h->seq_len + slot, &img->seq_len, sizeof(int), cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaMemcpyAsync(h->pos + slot, &img->pos, sizeof(int), cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaMemcpyAsync(h->end_idx + slot, &img->end_idx, sizeof(int), cudaMemcpyHostToDevice, s));
  CTB_CUDA(cudaMemsetAsync(h->finish + slot, img->finish ? 1 : 0, 1, s));
  if ((rc = kv_move(h, slot, const_cast<char*>(hb) + img->off_kv, img->npages, false, s)) ||
      (rc = launch_set_row(h, slot, r, s)))
    return rc;
  h->slot[slot].hi = img->seq_len;
  h->slot[slot].cap = img->seq_len + r.max_new - r.n_gen;
  if (r.text) h->eng_text = 1;
  return CTB_OK;
}

// ------------------------------------------------------------------ shared prompts (ctb_gpt_engine_share_prompt)
extern "C" int ctb_gpt_engine_share_prompt(ctb_gpt* h, int32_t src, int32_t dst, int32_t T0, int32_t c0, void* stream) {
  if (!h) return set_err(CTB_ERR_ARG, "null argument");
  int rc;
  if ((rc = check_engine(h))) return rc;
  const int S = h->B;
  if (src < 0 || src >= S || dst < 0 || dst >= S || src == dst)
    return set_err(CTB_ERR_ARG, "slots %d -> %d: two distinct slots of [0,%d)", src, dst, S);
  if ((rc = check_T0(h, T0))) return rc;
  if (c0 < CTB_PREFILL_CHUNK_ALIGN || c0 % CTB_PREFILL_CHUNK_ALIGN || c0 >= T0)
    return set_err(CTB_ERR_ARG, "c0=%d: a positive multiple of %d below T0=%d", c0, CTB_PREFILL_CHUNK_ALIGN, T0);
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<RowState> rows;
  if ((rc = read_rows(h, rows, s))) return rc;
  const SlotRecord& from = h->slot[src];
  SlotRecord& to = h->slot[dst];
  // a finished source still holds its KV until the slot is released or admitted again (pr_len is then 0)
  if ((rows[src].state != RS_RUNNING && rows[src].state != RS_FINISHED) || from.pr_len == 0)
    return set_err(CTB_ERR_STATE, "slot %d holds no admitted prompt (state %d)", src, rows[src].state);
  if ((rc = check_not_generating(rows[dst], dst)) || (rc = check_slot(h, dst))) return rc;
  if (h->pg_pages && to.pages) return set_err(CTB_ERR_STATE, "slot %d has pages mapped", dst);
  if (from.pr_len < c0)
    return set_err(CTB_ERR_STATE, "slot %d holds a prompt of %d positions, fewer than c0=%d", src, from.pr_len, c0);
  if ((T0 > PF_ATT_MAX_T0) != (from.pr_W > PF_ATT_MAX_T0))
    return set_err(CTB_ERR_ARG, "T0=%d and slot %d's prompt width %d take different prefill attention kernels", T0, src,
                   from.pr_W);
  const int shared = c0 / kPageTokens;
  if (h->pg_pages) {  // dst's entries [0, shared) map src's pages; [shared, ceil(T0 / 16)) map pages of its own
    const int own = (T0 + kPageTokens - 1) / kPageTokens - shared;
    if ((size_t)own > h->pg_free.size())
      return set_err(CTB_ERR_POOL, "KV pool: %d more pages needed, %zu of %d free", own, h->pg_free.size(),
                     h->pg_pages - 1);
    std::vector<std::pair<int, int>> e;
    for (int k = 0; k < shared + own; ++k)
      map_page(h, dst, k < shared ? h->pg_bt[(size_t)src * h->pages_per_row + k] : -1, e);
    if ((rc = bt_write(h, e, s))) return rc;
  } else {  // a fixed engine: row b owns pages [b * bt_per_row, (b + 1) * bt_per_row)
    KvCopyP p{};
    p.kv = reinterpret_cast<char*>(h->kv); p.layer_bytes = h->kv_layer_elems * kv_elem_bytes(h);
    p.page_words = (int)(page_bytes(h) / 16); p.layers = h->cfg.num_layers; p.npages = shared;
    p.src0 = src * (int)h->bt_per_row; p.dst0 = dst * (int)h->bt_per_row;
    k_kv_copy<<<(unsigned)std::min(p.layers * shared, g_num_sms * 8), 256, 0, s>>>(p);
    CTB_LAUNCH_CHECK();
  }
  to.chunk_T0 = T0; to.chunk_done = c0;  // the final chunk [c0, T0) admits the request
  to.pr_len = 0;
  return CTB_OK;
}

namespace ctb {
// Embed.forward (embed.py:51-79): one CTA per prompt position
__global__ void k_embed_prompt(const int64_t* __restrict__ ids, const uint8_t* __restrict__ text_mask,
                               const float* __restrict__ emb_text, const float* __restrict__ emb_code, int num_vq,
                               int num_audio, int num_text, int d, float* __restrict__ out) {
  const size_t pos = blockIdx.x;
  const int64_t* id = ids + pos * num_vq;
  float* o = out + pos * d;
  if (text_mask[pos]) {
    const int64_t t = min(max(id[0], (int64_t)0), (int64_t)num_text - 1);
    const float* e = emb_text + (size_t)t * d;
    for (int k = threadIdx.x; k < d; k += blockDim.x) o[k] = e[k];
  } else {
    for (int k = threadIdx.x; k < d; k += blockDim.x) {
      float s = 0.f;
      for (int q = 0; q < num_vq; ++q) {
        const int64_t c = min(max(id[q], (int64_t)0), (int64_t)num_audio - 1);
        s += emb_code[((size_t)q * num_audio + c) * d + k];
      }
      o[k] = s;
    }
  }
}
}  // namespace ctb

extern "C" int ctb_gpt_embed_prompt(ctb_gpt* h, const int64_t* ids_dev, const uint8_t* text_mask_dev, int32_t B, int32_t T,
                                    float* out_dev, void* stream) {
  if (!h || !ids_dev || !text_mask_dev || !out_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (B < 1 || T < 1) return set_err(CTB_ERR_ARG, "bad shape");
  const ctb_gpt_config& c = h->cfg;
  k_embed_prompt<<<(unsigned)((size_t)B * T), 256, 0, (cudaStream_t)stream>>>(
      ids_dev, text_mask_dev, h->W + h->lay.emb_text, h->W + h->lay.emb_code, c.num_vq, c.num_audio_tokens,
      c.num_text_tokens, c.hidden_size, out_dev);
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

extern "C" int ctb_gpt_debug_trace(ctb_gpt* h, unsigned long long* host_out, int n) {
  if (!h || !h->trace) return set_err(CTB_ERR_STATE, "trace disabled (set CTB_MEGA_TRACE=1 before ctb_gpt_create)");
  CTB_CUDA(cudaMemcpy(host_out, h->trace, sizeof(unsigned long long) * (size_t)std::min(n, FL_TR_WORDS), cudaMemcpyDeviceToHost));
  return CTB_OK;
}

extern "C" int ctb_gpt_status_query(ctb_gpt* h, ctb_gpt_status* out, int32_t* end_idx_host, uint8_t* finish_host,
                                    void* stream) {
  if (!h || !out) return set_err(CTB_ERR_ARG, "null argument");
  if (!h->started) return set_err(CTB_ERR_STATE, "no static batch or slot engine in flight (ctb_gpt_begin*)");
  cudaStream_t s = (cudaStream_t)stream;
  LoopState st;
  CTB_CUDA(cudaMemcpyAsync(&st, h->st, sizeof(st), cudaMemcpyDeviceToHost, s));
  if (end_idx_host) CTB_CUDA(cudaMemcpyAsync(end_idx_host, h->end_idx, sizeof(int) * h->B, cudaMemcpyDeviceToHost, s));
  if (finish_host) CTB_CUDA(cudaMemcpyAsync(finish_host, h->finish, h->B, cudaMemcpyDeviceToHost, s));
  CTB_CUDA(cudaStreamSynchronize(s));
  if (st.err != 0)
    return set_err(CTB_ERR_STATE, "decode kernel reported error 0x%x (watchdog: a cross-CTA wait never completed)", st.err);
  out->steps_done = st.step;
  out->all_finished = st.all_finished;
  out->any_finished_first_step = st.any_first;
  out->reserved = 0;
  return CTB_OK;
}

extern "C" int ctb_sample(const float* logits_dev, int32_t rows, int32_t V, int32_t rows_per_item,
                          const ctb_sampler_config* sampler, const float* q_noise_dev, const int32_t* gen_ids_dev,
                          int32_t gen_stride, int32_t n_gen, int32_t step, int32_t* out_idx_dev, void* stream) {
  if (!logits_dev || !sampler || !out_idx_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (rows < 1 || V < 1 || rows_per_item < 1 || rows % rows_per_item) return set_err(CTB_ERR_ARG, "bad shape");
  if ((size_t)V * 4 + 8192 > 200 * 1024) return set_err(CTB_ERR_ARG, "V=%d too large for the sampler", V);
  if (sampler->penalty_on && n_gen > 0 && !gen_ids_dev) return set_err(CTB_ERR_ARG, "gen_ids required");
  if (int rc = check_sampler(*sampler)) return rc;
  SampleP sp{};
  sp.st = nullptr; sp.check_finished = 0; sp.logits = logits_dev; sp.rows = rows; sp.V = V;
  sp.rows_per_item = rows_per_item; sp.cfg = *sampler; sp.q_noise = q_noise_dev; sp.gen_ids = gen_ids_dev;
  sp.gen_stride = gen_stride; sp.gen_inner = rows_per_item; sp.n_gen_fixed = n_gen; sp.step_fixed = step; sp.out_idx = out_idx_dev;
  return launch_sample(sp, (cudaStream_t)stream);
}

extern "C" int ctb_token_logprobs(const float* logits_dev, int32_t rows, int32_t V, const int32_t* ids_dev, float* out_dev,
                                  void* stream) {
  if (!logits_dev || !ids_dev || !out_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (rows < 1 || V < 1) return set_err(CTB_ERR_ARG, "bad shape");
  LogprobP lp{};
  lp.logits = logits_dev; lp.V = V; lp.rows_per_item = 1; lp.idx = ids_dev; lp.out = out_dev;
  CTB_CUDA(launch_pdl(k_token_logprob, dim3(rows), dim3(LOGPROB_THREADS), 0, (cudaStream_t)stream, lp));
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

extern "C" int ctb_token_top_logprobs(const float* logits_dev, int32_t rows, int32_t V, int32_t n_top, int32_t* ids_out_dev,
                                      float* lp_out_dev, void* stream) {
  if (!logits_dev || !ids_out_dev || !lp_out_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (n_top < 1 || n_top > TOP_LOGPROBS_MAX) return set_err(CTB_ERR_ARG, "N=%d outside [1,%d]", n_top, TOP_LOGPROBS_MAX);
  if (rows < 1 || V < n_top) return set_err(CTB_ERR_ARG, "bad shape: rows=%d, V=%d, N=%d", rows, V, n_top);
  if ((size_t)V * 4 > 200 * 1024) return set_err(CTB_ERR_ARG, "V=%d: a row does not fit in shared memory", V);
  TopLogprobP tp{};
  tp.logits = logits_dev; tp.V = V; tp.rows_per_item = 1; tp.n_top = n_top; tp.ids = ids_out_dev; tp.lp = lp_out_dev;
  return launch_top_logprobs(tp, rows, (cudaStream_t)stream);
}
