// Decode-step kernels for hot path 1 (GPT.generate, reference ChatTTS/model/gpt.py:394-596).
//
// One "step" = k_input -> 20 x [k_gemv<QKV> -> k_attn -> k_gemv<OPROJ> -> k_gemv<GATEUP> -> k_gemv<DOWN>]
//            -> k_gemv<HEADS> -> k_sample -> k_finalize.
// All loop state (positions, finish flags, step counter) lives in device memory so a captured
// CUDA graph of one step can be replayed without host involvement.
//
// Numerics: fp32 weights, fp32 FMA accumulation everywhere.  The parity target is the fp32 CPU
// reference (SURVEY.md 7 "hard parts"): sampled ids must match, so no reduced precision here.
#pragma once
#include "common.cuh"

namespace ctb {

struct LoopState {
  int step;            // loop iterations completed (gpt.py: i)
  int all_finished;    // finish.all()
  int any_first;       // i == 0 and finish.any()
  int n_gen;           // tokens appended to ids_out so far
  int err;             // != 0: a device-side watchdog fired (flow.cuh); reported by ctb_gpt_status_query
};

// Slot engine (ctb_gpt_engine_*): every batch row is a slot holding one request at its own point of generation, so
// the loop counters live per row.  The static path passes rows == nullptr and keeps using LoopState's counters.
enum RowStateKind { RS_IDLE = 0, RS_RUNNING = 1, RS_FINISHED = 2, RS_PENDING = 3 /* prefilled, first token not yet sampled */ };
struct RowState {
  int n_gen;      // tokens this row has appended to ids_out
  int step;       // loop iterations this row has run (its own gpt.py `i`)
  int state;      // RowStateKind
  int max_new;    // the row finishes after this many tokens
  int has_noise;  // 1: Exp(1) rows in the engine's noise buffer (seeded request); 0: device Philox
  int eos;
  int text;       // 1: text tokens (emb_text input, text head, one sampled row); 0: audio codes
  int pad;
};

// The heads and the sampler of a slot engine run once for code rows and once for text rows: their `want` is a
// RowStateKind, plus WANT_TEXT when the launch serves text rows.  k_finalize_rows serves both kinds in one launch.
constexpr int WANT_TEXT = 8;
__device__ __forceinline__ bool row_wanted(const RowState* r, int want) {
  return ldg_cg(&r->state) == (want & ~WANT_TEXT) && (ldg_cg(&r->text) != 0) == ((want & WANT_TEXT) != 0);
}
// CTA-uniform: does any of the B rows match `want`?  (every warp reads the <= 32 row states itself)
__device__ __forceinline__ bool any_row_wanted(const RowState* rows, int B, int want) {
  bool any = false;
  for (int b = threadIdx.x & 31; b < B; b += 32) any |= row_wanted(rows + b, want);
  return __any_sync(0xffffffffu, any);
}

constexpr int KC = 768;        // K chunk staged in shared memory (= hidden size of the model)
constexpr int GEMV_WARPS = 8;  // warps per CTA, one 2-row task per warp
constexpr int ATT_CHUNK = 128;      // keys per k_attn chunk: 8 warps x 16 keys, all K/V rows of a chunk in flight at once
constexpr int ATT_THREADS = 256;
constexpr int ATT_SPLIT_UNIT = 64;  // granularity the split/partial buffers are sized with (k_step uses 64-key chunks)

enum Epi { EPI_QKV = 0, EPI_OPROJ = 1, EPI_GATEUP = 2, EPI_DOWN = 3, EPI_HEADS = 4 };

struct GemvP {
  const float* W;        // [rows, K] row-major
  int K;                 // 768 or a multiple of 768
  int ntasks;            // 2-row warp tasks
  int nrows;             // valid rows of W
  const float* xin;      // [Bpad, K]
  const float* normw;    // RMSNorm weight (prologue) or nullptr
  float eps;
  int B;                 // real batch rows
  const LoopState* st;   // nullptr: never skip
  int check_finished;    // decode steps early-exit once all rows finished
  // --- epilogue targets
  float* xres;           // residual stream [Bpad, d]   (OPROJ / DOWN: +=)
  float* out;            // GATEUP: mlp [Bpad, I]; HEADS: logits; QKV: q buffer [Bpad, Hq*hd]
  float* kv;             // QKV: KV pool of this layer
  const int* block_table;
  int pages_per_row;
  const int* pos;        // [Bpad] position of the current token per row
  const uint8_t* active; // [Bpad]
  const float* rope_cos; // [max_pos, hd]
  const float* rope_sin;
  int Hq, Hkv, hd, I;
  // HEADS
  int rows_per_item;     // num_vq (audio) or 1 (text)
  int V;
  float* hidden_out;     // [B, max_new, d] or nullptr
  int hidden_stride;     // max_new * d
  const RowState* rows;  // slot engine: only rows matching `want` (row_wanted) get logits / hidden states; nullptr: every row
  int want;
};

// KV pool layout of one layer: [page][2 (K,V)][Hkv][16 tokens][hd]
__device__ __forceinline__ size_t kv_off(int page, int which, int h, int slot, int Hkv, int hd) {
  return ((((size_t)page * 2 + which) * Hkv + h) * kPageTokens + slot) * hd;
}

// ---- cluster / async-copy helpers (sm_90+)
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float ld_dsmem(const float* local_smem_ptr, uint32_t rank) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(local_smem_ptr);
  uint32_t r; float v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
  asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(r) : "memory");
  return v;
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

constexpr int DOWN_SPLIT = 4;       // K = 3072 split over a 4-CTA cluster, partials merged through DSMEM
constexpr int DOWN_MAX_TASKS = 4;   // row-pair tasks per warp in the DOWN kernel (ceil(384 / (groups*8)) <= 4 for >= 12 groups)

// Persistent weight-streaming GEMV / skinny GEMM:  y[b, r] = sum_k W[r, k] * x[b, k]  for a batch tile of
// BT rows.  grid.x CTAs (one per SM) stride over 2-row warp tasks; the batch tile's activations are staged
// ONCE per CTA in shared memory with cp.async (L2-coherent), the RMSNorm prologue runs on that copy, and each
// warp streams its rows' weights with 128-bit non-allocating loads, next task prefetched under the FMAs.
// EPI_DOWN: launched as clusters of DOWN_SPLIT CTAs; rank r owns K-chunk r of the same rows, the partial sums
// meet in rank 0 through distributed shared memory in a fixed order (deterministic, no atomics).
template <int BT, int EPI>
__global__ void __launch_bounds__(GEMV_WARPS * 32) k_gemv(const GemvP p) {
  pdl_trigger();
  extern __shared__ __align__(16) float xs[];  // [BT][KC]
  __shared__ float rinv[BT];
  __shared__ float red[(EPI == EPI_DOWN) ? GEMV_WARPS * DOWN_MAX_TASKS * 2 * BT : 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int bbase = blockIdx.y * BT;        // batch tile (B > 32 re-streams the weights per tile)
  const int nb = min(BT, p.B - bbase);      // live rows in this tile
  const int kc = (EPI == EPI_DOWN) ? (int)cluster_ctarank() : 0;
  const int cta = (EPI == EPI_DOWN) ? blockIdx.x / DOWN_SPLIT : blockIdx.x;
  const int ncta = (EPI == EPI_DOWN) ? gridDim.x / DOWN_SPLIT : gridDim.x;
  const int tstride = ncta * GEMV_WARPS;
  const int task0 = cta * GEMV_WARPS + warp;

  auto task_rows = [&](int task, int& r0, int& r1) {
    if (EPI == EPI_QKV) {
      // task -> (q|k|v, head, j): rows j and j + hd/2 of one head so RoPE pairs stay in-warp
      const int half = p.hd / 2;
      int t = task, base = 0;
      const int nq = p.Hq * half, nk = p.Hkv * half;
      if (t >= nq + nk) { t -= nq + nk; base = (p.Hq + p.Hkv) * p.hd; }
      else if (t >= nq) { t -= nq; base = p.Hq * p.hd; }
      r0 = base + (t / half) * p.hd + (t % half);
      r1 = r0 + half;
    } else if (EPI == EPI_GATEUP) {
      r0 = task; r1 = p.I + task;
    } else {
      r0 = 2 * task; r1 = min(2 * task + 1, p.nrows - 1);
    }
  };
  auto load_w = [&](int task, float4 (&w0)[6], float4 (&w1)[6]) {
    int r0, r1;
    task_rows(task, r0, r1);
    const float4* w0p = reinterpret_cast<const float4*>(p.W + (size_t)r0 * p.K + kc * KC) + lane;
    const float4* w1p = reinterpret_cast<const float4*>(p.W + (size_t)r1 * p.K + kc * KC) + lane;
#pragma unroll
    for (int i = 0; i < 6; ++i) { w0[i] = ldg_stream(w0p + i * 32); w1[i] = ldg_stream(w1p + i * 32); }
  };

  // the first task's weights do not depend on earlier kernels: request them before the PDL wait.  A slot engine's
  // text head streams nothing until the row states show a text row to serve.
  const bool text_rows = EPI == EPI_HEADS && p.rows != nullptr && (p.want & WANT_TEXT);
  float4 w0[6], w1[6];
  if (task0 < p.ntasks && !text_rows) load_w(task0, w0, w1);
  pdl_wait();  // everything below reads activations / loop state written by earlier kernels
  if (p.check_finished && ldg_cg(&p.st->all_finished)) {
    if (EPI == EPI_DOWN) { cluster_sync_all(); cluster_sync_all(); }
    return;
  }
  if (text_rows) {
    if (!any_row_wanted(p.rows, p.B, p.want)) return;
    if (task0 < p.ntasks) load_w(task0, w0, w1);
  }

  // ---- stage the batch tile's activations (K chunk kc) once per CTA
  for (int i = tid; i < BT * (KC / 4); i += GEMV_WARPS * 32) {
    const int b = i / (KC / 4), k4 = i % (KC / 4);
    if (b < nb) cp_async16(&xs[i * 4], p.xin + (size_t)(bbase + b) * p.K + kc * KC + k4 * 4);
    else reinterpret_cast<float4*>(xs)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  cp_async_wait_all();
  __syncthreads();
  if (p.normw != nullptr) {
    // RMSNorm prologue (K == KC): HF LlamaRMSNorm  w * (x * rsqrt(mean(x^2) + eps))
    for (int b = warp; b < BT; b += GEMV_WARPS) {
      float ss = 0.f;
#pragma unroll
      for (int k = lane; k < KC; k += 32) { const float v = xs[b * KC + k]; ss = fmaf(v, v, ss); }
      ss = warp_sum(ss);
      if (lane == 0) rinv[b] = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fdiv_rn(ss, (float)KC), p.eps)));
    }
    __syncthreads();
    for (int i = tid; i < BT * KC; i += GEMV_WARPS * 32) {
      const int b = i / KC, k = i % KC;
      xs[i] = __fmul_rn(__ldg(p.normw + k), __fmul_rn(xs[i], rinv[b]));
    }
    __syncthreads();
    if (EPI == EPI_HEADS && p.hidden_out != nullptr && blockIdx.x == 0) {
      // last_hidden_state of this step (gpt.py:430-436), written once per batch tile
      if (p.rows == nullptr) {
        const int step = ldg_cg(&p.st->n_gen);
        for (int i = tid; i < nb * KC; i += GEMV_WARPS * 32) {
          const int b = i / KC, k = i % KC;
          p.hidden_out[(size_t)(bbase + b) * p.hidden_stride + (size_t)step * KC + k] = xs[i];
        }
      } else {
        for (int b = 0; b < nb; ++b) {
          const RowState* r = p.rows + bbase + b;
          if (!row_wanted(r, p.want)) continue;
          const int step = ldg_cg(&r->n_gen);
          for (int k = tid; k < KC; k += GEMV_WARPS * 32)
            p.hidden_out[(size_t)(bbase + b) * p.hidden_stride + (size_t)step * KC + k] = xs[b * KC + k];
        }
      }
    }
  }

  constexpr int LPB = 32 / BT;  // lanes per batch row after the reduce-scatter
  int jtask = 0;
  for (int task = task0; task < p.ntasks; task += tstride, ++jtask) {
    float4 n0[6], n1[6];
    const bool more = task + tstride < p.ntasks;
    if (more) load_w(task + tstride, n0, n1);
    float acc0[BT], acc1[BT];
#pragma unroll
    for (int b = 0; b < BT; ++b) { acc0[b] = 0.f; acc1[b] = 0.f; }
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
      for (int b = 0; b < BT; ++b) {
        const float4 xv = reinterpret_cast<const float4*>(xs)[b * (KC / 4) + i * 32 + lane];
        acc0[b] = fmaf(w0[i].x, xv.x, acc0[b]); acc0[b] = fmaf(w0[i].y, xv.y, acc0[b]);
        acc0[b] = fmaf(w0[i].z, xv.z, acc0[b]); acc0[b] = fmaf(w0[i].w, xv.w, acc0[b]);
        acc1[b] = fmaf(w1[i].x, xv.x, acc1[b]); acc1[b] = fmaf(w1[i].y, xv.y, acc1[b]);
        acc1[b] = fmaf(w1[i].z, xv.z, acc1[b]); acc1[b] = fmaf(w1[i].w, xv.w, acc1[b]);
      }
    }
    if (more) {
#pragma unroll
      for (int i = 0; i < 6; ++i) { w0[i] = n0[i]; w1[i] = n1[i]; }
    }
    warp_reduce_scatter<BT>(acc0);
    warp_reduce_scatter<BT>(acc1);
    const bool writer = (lane % LPB) == 0 && (lane / LPB) < nb;
    const int b = bbase + lane / LPB;
    const float v0 = acc0[0], v1 = acc1[0];
    int r0, r1;
    task_rows(task, r0, r1);
    const bool r1_valid = (EPI == EPI_QKV || EPI == EPI_GATEUP) ? true : (2 * task + 1 < p.nrows);

    if (EPI == EPI_DOWN) {
      // partial over K chunk kc -> this CTA's smem; merged by cluster rank 0 below
      if ((lane % LPB) == 0 && jtask < DOWN_MAX_TASKS) {
        float* r = red + ((warp * DOWN_MAX_TASKS + jtask) * 2) * BT + lane / LPB;
        r[0] = v0; r[BT] = v1;
      }
      continue;
    }
    if (!writer) continue;
    if (EPI == EPI_QKV) {
      if (!ldg_cg(&p.active[b])) continue;
      const int half = p.hd / 2;
      const int nq = p.Hq * half, nk = p.Hkv * half;
      int t = task, which = 0;
      if (t >= nq + nk) { which = 2; t -= nq + nk; }
      else if (t >= nq) { which = 1; t -= nq; }
      const int h = t / half, j = t % half;
      const int pos = ldg_cg(&p.pos[b]);
      float o0 = v0, o1 = v1;
      if (which < 2) {
        // HF apply_rotary_pos_emb: q*cos + rotate_half(q)*sin, each product rounded separately
        const float c0 = __ldg(p.rope_cos + (size_t)pos * p.hd + j), s0 = __ldg(p.rope_sin + (size_t)pos * p.hd + j);
        const float c1 = __ldg(p.rope_cos + (size_t)pos * p.hd + j + half), s1 = __ldg(p.rope_sin + (size_t)pos * p.hd + j + half);
        o0 = __fadd_rn(__fmul_rn(v0, c0), __fmul_rn(-v1, s0));
        o1 = __fadd_rn(__fmul_rn(v1, c1), __fmul_rn(v0, s1));
      }
      if (which == 0) {
        p.out[(size_t)b * p.Hq * p.hd + h * p.hd + j] = o0;
        p.out[(size_t)b * p.Hq * p.hd + h * p.hd + j + half] = o1;
      } else {
        const int page = __ldg(p.block_table + b * p.pages_per_row + pos / kPageTokens);
        float* dst = p.kv + kv_off(page, which - 1, h, pos % kPageTokens, p.Hkv, p.hd);
        dst[j] = o0; dst[j + half] = o1;
      }
    } else if (EPI == EPI_OPROJ) {
      const int d = p.nrows;
      p.xres[(size_t)b * d + r0] = __fadd_rn(ldg_cg(&p.xres[(size_t)b * d + r0]), v0);
      if (r1_valid) p.xres[(size_t)b * d + r1] = __fadd_rn(ldg_cg(&p.xres[(size_t)b * d + r1]), v1);
    } else if (EPI == EPI_GATEUP) {
      // LlamaMLP: silu(gate) * up ; silu(x) = x / (1 + exp(-x))
      const float sg = __fdiv_rn(v0, __fadd_rn(1.0f, expf(-v0)));
      p.out[(size_t)b * p.I + task] = __fmul_rn(sg, v1);
    } else {  // EPI_HEADS: logits rows ordered (b, q) like gpt.py:459-464
      if (p.rows != nullptr && !row_wanted(p.rows + b, p.want)) continue;
      const int q0 = r0 / p.V, c0 = r0 % p.V;
      p.out[((size_t)b * p.rows_per_item + q0) * p.V + c0] = v0;
      if (r1_valid) {
        const int q1 = (2 * task + 1) / p.V, c1 = (2 * task + 1) % p.V;
        p.out[((size_t)b * p.rows_per_item + q1) * p.V + c1] = v1;
      }
    }
  }

  if (EPI == EPI_DOWN) {
    cluster_sync_all();  // every rank's partials are in its shared memory
    if (kc == 0) {
      const int d = p.nrows;
      int j = 0;
      for (int task = task0; task < p.ntasks && j < DOWN_MAX_TASKS; task += tstride, ++j) {
        if ((lane % LPB) != 0 || (lane / LPB) >= nb) continue;
        const int b = bbase + lane / LPB;
        const float* r = red + ((warp * DOWN_MAX_TASKS + j) * 2) * BT + lane / LPB;
        float v0 = r[0], v1 = r[BT];
#pragma unroll
        for (uint32_t rk = 1; rk < DOWN_SPLIT; ++rk) {  // fixed order: chunk 0 + 1 + 2 + 3
          v0 = __fadd_rn(v0, ld_dsmem(r, rk));
          v1 = __fadd_rn(v1, ld_dsmem(r + BT, rk));
        }
        const int r0 = 2 * task, r1 = 2 * task + 1;
        p.xres[(size_t)b * d + r0] = __fadd_rn(ldg_cg(&p.xres[(size_t)b * d + r0]), v0);
        if (r1 < d) p.xres[(size_t)b * d + r1] = __fadd_rn(ldg_cg(&p.xres[(size_t)b * d + r1]), v1);
      }
    }
    cluster_sync_all();  // keep the other ranks' shared memory alive until rank 0 has read it
  }
}

// Down projection (K = I = 4 * KC) for batch tiles <= 16: no cluster.  Every CTA owns up to DS_PAIRS row pairs, its 8 warps
// split K (I/8 each), ALL of the warp's weights are requested before griddepcontrol.wait (one DRAM round trip), the
// batch tile's [BT][I] activations are staged once with cp.async, partial sums meet in shared memory in a fixed order.
constexpr int DS_PAIRS = 3;  // ceil((d/2) / grid) for grid >= 128 CTAs
template <int BT>
__global__ void __launch_bounds__(GEMV_WARPS * 32) k_down_small(const GemvP p) {
  pdl_trigger();
  extern __shared__ __align__(16) float xs[];  // [BT][I]
  __shared__ float red[DS_PAIRS][GEMV_WARPS][2][BT];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int I = p.K, d = p.nrows, npairs = d / 2, I4 = I / 4, ks4 = I4 / GEMV_WARPS;  // float4 per K slice (96)
  float4 dw[DS_PAIRS][2][3];
#pragma unroll
  for (int j = 0; j < DS_PAIRS; ++j) {
    const int pair = blockIdx.x + j * gridDim.x;
    if (pair < npairs) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float4* wp = reinterpret_cast<const float4*>(p.W + (size_t)(2 * pair + r) * I) + warp * ks4 + lane;
#pragma unroll
        for (int i = 0; i < 3; ++i) dw[j][r][i] = ldg_stream(wp + i * 32);
      }
    }
  }
  pdl_wait();
  if (p.check_finished && ldg_cg(&p.st->all_finished)) return;
  const int nb = p.B;
  for (int i = tid; i < BT * I4; i += GEMV_WARPS * 32) {
    const int b = i / I4, k4 = i % I4;
    if (b < nb) cp_async16(&xs[i * 4], p.xin + (size_t)b * I + k4 * 4);
    else reinterpret_cast<float4*>(xs)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  // residual values of the final-reduce elements (one per thread), requested together with the activations
  float rx = 0.f;
  const bool fin = tid < DS_PAIRS * 2 * BT;
  const int fb = tid % BT, fr = (tid / BT) % 2, fj = tid / (2 * BT);
  const int fpair = blockIdx.x + fj * gridDim.x;
  if (fin && fpair < npairs && fb < nb) rx = ldg_cg(p.xres + (size_t)fb * d + 2 * fpair + fr);
  cp_async_wait_all();
  __syncthreads();
  constexpr int LPB = 32 / BT;
#pragma unroll
  for (int j = 0; j < DS_PAIRS; ++j) {
    const int pair = blockIdx.x + j * gridDim.x;
    if (pair >= npairs) break;
    float acc0[BT], acc1[BT];
#pragma unroll
    for (int b = 0; b < BT; ++b) { acc0[b] = 0.f; acc1[b] = 0.f; }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
      for (int b = 0; b < BT; ++b) {
        const float4 xv = reinterpret_cast<const float4*>(xs)[b * I4 + warp * ks4 + i * 32 + lane];
        acc0[b] = fmaf(dw[j][0][i].x, xv.x, acc0[b]); acc0[b] = fmaf(dw[j][0][i].y, xv.y, acc0[b]);
        acc0[b] = fmaf(dw[j][0][i].z, xv.z, acc0[b]); acc0[b] = fmaf(dw[j][0][i].w, xv.w, acc0[b]);
        acc1[b] = fmaf(dw[j][1][i].x, xv.x, acc1[b]); acc1[b] = fmaf(dw[j][1][i].y, xv.y, acc1[b]);
        acc1[b] = fmaf(dw[j][1][i].z, xv.z, acc1[b]); acc1[b] = fmaf(dw[j][1][i].w, xv.w, acc1[b]);
      }
    }
    warp_reduce_scatter<BT>(acc0);
    warp_reduce_scatter<BT>(acc1);
    if ((lane % LPB) == 0) { red[j][warp][0][lane / LPB] = acc0[0]; red[j][warp][1][lane / LPB] = acc1[0]; }
  }
  __syncthreads();
  if (fin && fpair < npairs && fb < nb) {
    float v = red[fj][0][fr][fb];
#pragma unroll
    for (int w = 1; w < GEMV_WARPS; ++w) v = __fadd_rn(v, red[fj][w][fr][fb]);  // K slices in the order 0..7
    p.xres[(size_t)fb * d + 2 * fpair + fr] = __fadd_rn(rx, v);
  }
}

// Gate/up projection for batch tiles <= 16: the (<= GU_TASKS) 2-row tasks of every warp land in a shared-memory zone through
// cp.async issued BEFORE griddepcontrol.wait (no registers, every request in flight at once), so after the wait the kernel
// only stages x, normalises and multiplies.  One CTA per SM.
constexpr int GU_TASKS = 3;  // ceil(I / (grid * 8)) for grid >= 128 CTAs
constexpr int GU_ZONE_FLOATS = GEMV_WARPS * GU_TASKS * 2 * KC;
template <int BT>
__global__ void __launch_bounds__(GEMV_WARPS * 32) k_gateup_small(const GemvP p) {
  pdl_trigger();
  extern __shared__ __align__(16) float gsm[];  // [BT][KC] activations | weight zone
  __shared__ float rinv[BT];
  float* xs = gsm;
  float* zone = gsm + BT * KC;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tstride = gridDim.x * GEMV_WARPS;
#pragma unroll
  for (int j = 0; j < GU_TASKS; ++j) {
    const int task = blockIdx.x * GEMV_WARPS + warp + j * tstride;
    if (task < p.I) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const float* src = p.W + (size_t)(r ? p.I + task : task) * KC;
        float* dst = zone + ((size_t)(warp * GU_TASKS + j) * 2 + r) * KC;
#pragma unroll
        for (int i = 0; i < 6; ++i) cp_async16(dst + (i * 32 + lane) * 4, src + (i * 32 + lane) * 4);
      }
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  pdl_wait();
  if (p.check_finished && ldg_cg(&p.st->all_finished)) { cp_async_wait_all(); return; }
  const int nb = p.B;
  for (int i = tid; i < BT * (KC / 4); i += GEMV_WARPS * 32) {
    const int b = i / (KC / 4), k4 = i % (KC / 4);
    if (b < nb) cp_async16(&xs[i * 4], p.xin + (size_t)b * KC + k4 * 4);
    else reinterpret_cast<float4*>(xs)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  cp_async_wait_all();  // activations and the weight zone
  __syncthreads();
  for (int b = warp; b < BT; b += GEMV_WARPS) {
    float ss = 0.f;
#pragma unroll
    for (int k = lane; k < KC; k += 32) { const float v = xs[b * KC + k]; ss = fmaf(v, v, ss); }
    ss = warp_sum(ss);
    if (lane == 0) rinv[b] = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fdiv_rn(ss, (float)KC), p.eps)));
  }
  __syncthreads();
  for (int i = tid; i < BT * KC; i += GEMV_WARPS * 32) {
    const int b = i / KC, k = i % KC;
    xs[i] = __fmul_rn(__ldg(p.normw + k), __fmul_rn(xs[i], rinv[b]));
  }
  __syncthreads();
  constexpr int LPB = 32 / BT;
#pragma unroll
  for (int j = 0; j < GU_TASKS; ++j) {
    const int task = blockIdx.x * GEMV_WARPS + warp + j * tstride;
    if (task >= p.I) break;
    const float4* g0 = reinterpret_cast<const float4*>(zone + ((size_t)(warp * GU_TASKS + j) * 2) * KC);
    const float4* g1 = g0 + KC / 4;
    float acc0[BT], acc1[BT];
#pragma unroll
    for (int b = 0; b < BT; ++b) { acc0[b] = 0.f; acc1[b] = 0.f; }
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      const float4 a = g0[i * 32 + lane], bq = g1[i * 32 + lane];
#pragma unroll
      for (int b = 0; b < BT; ++b) {
        const float4 xv = reinterpret_cast<const float4*>(xs)[b * (KC / 4) + i * 32 + lane];
        acc0[b] = fmaf(a.x, xv.x, acc0[b]); acc0[b] = fmaf(a.y, xv.y, acc0[b]);
        acc0[b] = fmaf(a.z, xv.z, acc0[b]); acc0[b] = fmaf(a.w, xv.w, acc0[b]);
        acc1[b] = fmaf(bq.x, xv.x, acc1[b]); acc1[b] = fmaf(bq.y, xv.y, acc1[b]);
        acc1[b] = fmaf(bq.z, xv.z, acc1[b]); acc1[b] = fmaf(bq.w, xv.w, acc1[b]);
      }
    }
    warp_reduce_scatter<BT>(acc0);
    warp_reduce_scatter<BT>(acc1);
    if ((lane % LPB) == 0 && (lane / LPB) < nb) {
      const float v0 = acc0[0], v1 = acc1[0];
      const float sg = __fdiv_rn(v0, __fadd_rn(1.0f, expf(-v0)));
      p.out[(size_t)(lane / LPB) * p.I + task] = __fmul_rn(sg, v1);
    }
  }
}

// ------------------------------------------------------------------ step input
struct InputP {
  LoopState* st;
  int decode;             // 0: prefill column, 1: decode step
  int B, d, col, T0;
  const float* emb;       // [B, T0, d] prompt embeddings
  const uint8_t* mask;    // [B, T0]
  const float* emb_code;  // [num_vq*num_audio, d]
  const float* emb_text;  // [num_text, d]
  const int32_t* ids_out; // [B, max_new, num_vq]
  int max_new, num_vq, num_audio, infer_text;
  float* x;               // [Bpad, d]
  float* x_hi; float* x_lo; // tensor-core path: tf32 hi / lo split of x (nullptr on the FMA path)
  int* seq_len;           // [Bpad]
  int* pos;               // [Bpad]
  uint8_t* active;        // [Bpad]
  const RowState* rows;   // slot engine: decode only running rows, each at its own n_gen; nullptr: static batch
};

#ifdef CTB_GPT_KERNELS_IMPL
__global__ void k_input(const InputP p) {
  const int b = blockIdx.x;
  pdl_trigger();
  pdl_wait();
  if (p.decode && ldg_cg(&p.st->all_finished)) return;
  float* x = p.x + (size_t)b * p.d;
  bool act;
  if (!p.decode) {
    act = p.mask[(size_t)b * p.T0 + p.col] != 0;
    const float* e = p.emb + ((size_t)b * p.T0 + p.col) * p.d;
    for (int k = threadIdx.x; k < p.d; k += blockDim.x) x[k] = act ? e[k] : 0.f;
  } else {
    act = true;
    int n_gen, text = p.infer_text;
    if (p.rows != nullptr) {
      // idle / finished slots append no KV and keep their position: only the active flag is written
      if (ldg_cg(&p.rows[b].state) != RS_RUNNING) {
        if (threadIdx.x == 0) p.active[b] = 0;
        return;
      }
      n_gen = ldg_cg(&p.rows[b].n_gen);
      text = ldg_cg(&p.rows[b].text);
    } else {
      n_gen = ldg_cg(&p.st->n_gen);
    }
    const int32_t* id = p.ids_out + ((size_t)b * p.max_new + (n_gen - 1)) * p.num_vq;
    if (text) {
      const float* e = p.emb_text + (size_t)ldg_cg(&id[0]) * p.d;
      for (int k = threadIdx.x; k < p.d; k += blockDim.x) x[k] = e[k];
    } else {
      // gpt.py:409-413: stack(code_emb, 3).sum(3)
      int idq[8];
      for (int q = 0; q < p.num_vq; ++q) idq[q] = ldg_cg(&id[q]);
      for (int k = threadIdx.x; k < p.d; k += blockDim.x) {
        float s = 0.f;
        for (int q = 0; q < p.num_vq; ++q) s += p.emb_code[((size_t)q * p.num_audio + idq[q]) * p.d + k];
        x[k] = s;
      }
    }
  }
  if (p.x_hi != nullptr) {
    __syncthreads();
    for (int k = threadIdx.x; k < p.d; k += blockDim.x) {
      const float v = x[k];
      uint32_t hb;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(v));
      const float hi = __uint_as_float(hb);
      uint32_t lb;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(v - hi));
      p.x_hi[(size_t)b * p.d + k] = hi;
      p.x_lo[(size_t)b * p.d + k] = __uint_as_float(lb);
    }
  }
  if (threadIdx.x == 0) {
    const int n = ldg_cg(&p.seq_len[b]);
    p.pos[b] = n;               // position id = #valid tokens before this one (gpt.py:234-241)
    p.active[b] = act ? 1 : 0;
    if (act) p.seq_len[b] = n + 1;
  }
}

#endif  // CTB_GPT_KERNELS_IMPL

// ------------------------------------------------------------------ decode attention
struct AttnP {
  const LoopState* st; int check_finished;
  const float* q;        // [Bpad, Hq*hd]
  const float* kv;       // this layer's pool (elements of k_attn's KVT)
  const int* block_table; int pages_per_row;
  const int* pos; const uint8_t* active;
  float* out;            // [Bpad, Hq*hd]
  float* out_hi; float* out_lo;  // tensor-core path copies (nullptr on the FMA path)
  float* part;           // [B, Hq, nsplit_max, hd + 2]
  int* counter;          // [B, Hq]
  int Hq, Hkv, hd, nsplit_max;
  float scaling;
};

// grid (nsplit_max, Hq, B); block ATT_THREADS (4 warps).  hd == 64 (checked on the host).
// Each warp owns ATT_CHUNK/4 keys of the CTA's chunk: 8 lanes per key row, all K and V rows of the warp
// are requested up front (one memory round trip), softmax statistics stay in registers; the four warps
// merge through shared memory and the CTA publishes (m, l, o[64]); the last CTA of a (row, head)
// merges the splits (flash-decoding).  KVT: the cache's element type (float, or __half for a half-precision slot
// engine: each 8-dim slice is one 16-byte load widened to fp32; the arithmetic is the same).
#ifdef CTB_GPT_KERNELS_IMPL
template <typename KVT>
__global__ void __launch_bounds__(ATT_THREADS) k_attn(const AttnP p) {
  pdl_trigger();
  pdl_wait();
  if (p.check_finished && ldg_cg(&p.st->all_finished)) return;
  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int HD = 64, NW = ATT_THREADS / 32, PER_WARP = ATT_CHUNK / NW, ITER = PER_WARP / 4;
  float* outp = p.out + (size_t)b * p.Hq * HD + h * HD;
  auto store_out = [&](float v) {
    outp[tid] = v;
    if (p.out_hi != nullptr) {
      uint32_t hb, lb;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(v));
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(v - __uint_as_float(hb)));
      p.out_hi[(size_t)b * p.Hq * HD + h * HD + tid] = __uint_as_float(hb);
      p.out_lo[(size_t)b * p.Hq * HD + h * HD + tid] = __uint_as_float(lb);
    }
  };
  if (!ldg_cg(&p.active[b])) { if (split == 0 && tid < HD) store_out(0.f); return; }
  const int n = ldg_cg(&p.pos[b]) + 1;  // keys 0..pos
  const int nchunk = (n + ATT_CHUNK - 1) / ATT_CHUNK;
  const int nsplit = min(nchunk, (int)gridDim.x);  // CTAs working on this (row, head): chunk c -> CTA c % gridDim.x
  if (split >= nsplit) return;
  const int hk = h / (p.Hq / p.Hkv);
  const int* bt = p.block_table + b * p.pages_per_row;
  const int sub = lane & 7, grp = lane >> 3;

  __shared__ float s_m[NW], s_l[NW];
  __shared__ __align__(16) float s_o[NW][HD];
  __shared__ int s_last;

  const float* qp = p.q + (size_t)b * p.Hq * HD + h * HD + sub * 8;
  const float4 q0 = ldg_cg(reinterpret_cast<const float4*>(qp));
  const float4 q1 = ldg_cg(reinterpret_cast<const float4*>(qp + 4));
  float M = -INFINITY, L = 0.f, O = 0.f;  // running softmax state of this CTA (thread d < 64 owns dim d)
  for (int chunk = split; chunk < nchunk; chunk += gridDim.x) {
    const int tbase = chunk * ATT_CHUNK + warp * PER_WARP + grp;
    float4 k0[ITER], k1[ITER], v0[ITER], v1[ITER];
#pragma unroll
    for (int i = 0; i < ITER; ++i) {
      const int t = tbase + 4 * i;
      k0[i] = k1[i] = v0[i] = v1[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t < n) {
        const int page = bt[t / kPageTokens];
        const KVT* kv = reinterpret_cast<const KVT*>(p.kv);
        ld_kv8(kv + kv_off(page, 0, hk, t % kPageTokens, p.Hkv, HD) + sub * 8, k0[i], k1[i]);
        ld_kv8(kv + kv_off(page, 1, hk, t % kPageTokens, p.Hkv, HD) + sub * 8, v0[i], v1[i]);
      }
    }
    float sc[ITER], m = -INFINITY;
#pragma unroll
    for (int i = 0; i < ITER; ++i) {
      float s = q0.x * k0[i].x + q0.y * k0[i].y + q0.z * k0[i].z + q0.w * k0[i].w + q1.x * k1[i].x + q1.y * k1[i].y +
                q1.z * k1[i].z + q1.w * k1[i].w;
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      sc[i] = (tbase + 4 * i < n) ? s * p.scaling : -INFINITY;
      m = fmaxf(m, sc[i]);
    }
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
    float l = 0.f, o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (m > -INFINITY) {
#pragma unroll
      for (int i = 0; i < ITER; ++i) {
        const float e = expf(sc[i] - m);  // exp(-inf) = 0 for masked keys
        l += e;
        o[0] = fmaf(e, v0[i].x, o[0]); o[1] = fmaf(e, v0[i].y, o[1]); o[2] = fmaf(e, v0[i].z, o[2]);
        o[3] = fmaf(e, v0[i].w, o[3]); o[4] = fmaf(e, v1[i].x, o[4]); o[5] = fmaf(e, v1[i].y, o[5]);
        o[6] = fmaf(e, v1[i].z, o[6]); o[7] = fmaf(e, v1[i].w, o[7]);
      }
    }
    // merge the 4 key groups of the warp (same `sub`, different `grp`)
    l += __shfl_xor_sync(0xffffffffu, l, 8);
    l += __shfl_xor_sync(0xffffffffu, l, 16);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[j] += __shfl_xor_sync(0xffffffffu, o[j], 8);
      o[j] += __shfl_xor_sync(0xffffffffu, o[j], 16);
    }
    __syncthreads();  // previous chunk's merge has finished reading s_o / s_m / s_l
    if (lane < 8) {
      *reinterpret_cast<float4*>(&s_o[warp][lane * 8]) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(&s_o[warp][lane * 8 + 4]) = make_float4(o[4], o[5], o[6], o[7]);
      if (lane == 0) { s_m[warp] = m; s_l[warp] = l; }
    }
    __syncthreads();
    // ---- merge the warps of this chunk into the CTA's running state
    if (tid < HD) {
      float cm = M;
#pragma unroll
      for (int w = 0; w < NW; ++w) cm = fmaxf(cm, s_m[w]);
      const float fo = (M > -INFINITY) ? expf(M - cm) : 0.f;
      L *= fo; O *= fo;
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        const float f = (s_m[w] > -INFINITY) ? expf(s_m[w] - cm) : 0.f;
        L = fmaf(f, s_l[w], L);
        O = fmaf(f, s_o[w][tid], O);
      }
      M = cm;
    }
  }
  if (nsplit == 1) {
    if (tid < HD) store_out(O / L);
    return;
  }
  float* part = p.part + (((size_t)b * p.Hq + h) * p.nsplit_max + split) * (HD + 2);
  if (tid < HD) part[tid] = O;
  if (tid == 0) { part[HD] = M; part[HD + 1] = L; }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(&p.counter[b * p.Hq + h], 1) == nsplit - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* pb = p.part + (((size_t)b * p.Hq + h) * p.nsplit_max) * (HD + 2);
  float GM = -INFINITY;
  for (int s = 0; s < nsplit; ++s) GM = fmaxf(GM, __ldcg(pb + s * (HD + 2) + HD));
  float GL = 0.f, GO = 0.f;
  for (int s = 0; s < nsplit; ++s) {
    const float w = expf(__ldcg(pb + s * (HD + 2) + HD) - GM);
    GL = fmaf(w, __ldcg(pb + s * (HD + 2) + HD + 1), GL);
    if (tid < HD) GO = fmaf(w, __ldcg(pb + s * (HD + 2) + tid), GO);
  }
  if (tid < HD) store_out(GO / GL);
  if (tid == 0) p.counter[b * p.Hq + h] = 0;
}
#endif  // CTB_GPT_KERNELS_IMPL

// ------------------------------------------------------------------ sampler
struct SampleP {
  const LoopState* st; int check_finished;
  const float* logits;   // [rows, V]
  int rows, V, rows_per_item;
  ctb_sampler_config cfg;
  const float* q_noise;  // [rows, V] or nullptr
  const int32_t* gen_ids; // [rows/rpi, gen_stride, gen_inner]
  int gen_stride, gen_inner;
  int n_gen_fixed, step_fixed;  // used when st == nullptr (stand-alone ctb_sample)
  int32_t* out_idx;      // [rows]
  // slot engine (k_sample<true>): counters, noise flag and state per item from `rstate`, the sampling parameters of
  // item b from cfgs[b] (device memory, so a captured decode graph serves every admitted request); only items
  // matching `want` (row_wanted) are sampled.  Item b's noise rows start at q_noise + b * noise_stride.
  const RowState* rstate;
  const ctb_sampler_config* cfgs;
  int want;
  int noise_stride;
};

constexpr int SAMPLE_THREADS = 1024;
template <bool ENGINE>
__global__ void k_sample(const SampleP p);

// k_token_logprob: log softmax(logits row)[id] of the id a sampler just chose, at temperature 1 and before any logits
// processing.  Its launch mirrors the k_sample<true> it follows (same rows, rows_per_item, want and st), and each served
// row r of item b, codebook q = r % rows_per_item writes out[(b * max_new + n_gen(b)) * num_vq + q], the index
// k_finalize_rows then writes the id at.  rstate == nullptr (ctb_token_logprobs): every row, out[r], ids from idx[r].
struct LogprobP {
  const LoopState* st; int check_finished;
  const float* logits;   // [rows, V]
  int V, rows_per_item;
  const int32_t* idx;    // [rows] the sampled ids
  const RowState* rstate;
  int want;
  float* out;            // slot engine: [B, max_new, num_vq]; stand-alone: [rows]
  int max_new, num_vq;
};
constexpr int LOGPROB_THREADS = 256;
__global__ void k_token_logprob(const LogprobP p);

// k_token_top_logprobs: the n_top ids of a logits row with the largest z (z descending, the smaller id first among equal
// z) and their log softmax(z), with k_token_logprob's row max and denominator.  Launched beside k_token_logprob with the
// same rows, rows_per_item, want and st; each served row writes its n_top entries at
// [((b * max_new + n_gen(b)) * num_vq + q) * n_top + k].  rstate == nullptr (ctb_token_top_logprobs, scoring): every
// row, at [r * n_top + k].  Dynamic shared memory: V floats (the row).
struct TopLogprobP {
  const LoopState* st; int check_finished;
  const float* logits;   // [rows, V]
  int V, rows_per_item;
  const RowState* rstate;
  int want;
  int n_top;             // 1..TOP_LOGPROBS_MAX
  int32_t* ids;          // slot engine: [B, max_new, num_vq, n_top]; stand-alone: [rows, n_top]
  float* lp;             // same shape as ids
  int max_new, num_vq;
};
constexpr int TOP_LOGPROBS_MAX = 20;
__global__ void k_token_top_logprobs(const TopLogprobP p);

struct FinalP {
  LoopState* st;
  int B, rows_per_item, num_vq, max_new, eos;
  const int32_t* idx;    // [B*rpi]
  int32_t* ids_out;      // [B, max_new, num_vq]
  uint8_t* finish; int32_t* end_idx;
  RowState* rows;        // k_finalize_rows only
  int want;
  const int32_t* idx_text;  // k_finalize_rows: [B] the text sampler's ids (text rows)
};
__global__ void k_finalize(const FinalP p);
__global__ void k_finalize_rows(const FinalP p);

// ctb_gpt_engine_cancel: the slots to stop travel by value as a bit set, so the launch needs no host-to-device copy
constexpr int CANCEL_MAX_SLOTS = 1024;
struct CancelP {
  LoopState* st;
  RowState* rows;
  uint8_t* finish;
  int B;
  uint32_t mask[CANCEL_MAX_SLOTS / 32];  // bit b: stop slot b
};
__global__ void k_cancel_rows(const CancelP p);

}  // namespace ctb
