// Batched prefill (SURVEY.md 8f N1; reference gpt.py:396-427 at i == 0): the whole left-padded prompt batch
// [B, T0, 768] goes through the 20 layers as token-parallel GEMMs on wgmma (k_tc_gemm, 3xTF32 =
// fp32-equivalent) instead of one decode step per prompt column.  Each batch row is one "utterance" of T0 frames
// for the GEMM tiler; pad columns are computed but never written to the KV cache nor attended to.
//
//   per layer:  k_rms_rows -> GEMM(Wqkv) -> k_prefill_rope_kv (RoPE, q buffer, paged-KV append)
//               -> k_prefill_attn (causal over the row's valid tokens; k_prefill_attn_tiled when T0 > 1024)
//               -> GEMM(Wo)+residual
//               -> k_rms_rows -> GEMM([Wgate;Wup]) -> k_silu_mul -> GEMM(Wdown)+residual
//   then k_prefill_finish hands the last column's residual to the decode-loop state (x, seq_len) and the
//   regular heads -> sampler -> finalize kernels produce the first token.
// A slot-engine prompt may also be prefilled in 128-aligned chunks (ctb_gpt_engine_prefill_chunk): the same layers over
// the chunk's rows (k_prefill_chunk_positions), and the attention kernel of the whole prompt's width with the chunk's
// first position as its query offset q0, reading the earlier chunks' keys from the pages.  A whole prompt is the chunk
// with q0 = 0.
#pragma once
#include <type_traits>

#include "gpt_kernels.cuh"

namespace ctb {

#ifdef CTB_GPT_KERNELS_IMPL

// HF LlamaRMSNorm over rows of 768: out = w * (x * rsqrt(mean(x^2) + eps)); one warp per row
__global__ void __launch_bounds__(256) k_rms_rows(const float* __restrict__ x, const float* __restrict__ w,
                                                  float* __restrict__ out, int M, int d, float eps) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= M) return;
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * d);
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

struct PrefillP {
  int B, T0, Hq, Hkv, hd, d;
  const uint8_t* mask;      // [B, T0]
  const int* npre;          // [B, T0] number of valid tokens strictly before column c (= position id)
  const int* nvalid;        // [B]
  const float* qkv;         // [B*T0, (Hq + 2 Hkv) * hd]
  float* q;                 // [B*T0, Hq*hd] (RoPE applied)
  float* kv; const int* block_table; int pages_per_row;
  const float* rope_cos; const float* rope_sin;
  int permute_qk;           // tensor-core decode path keeps q/k rows pair-interleaved (tc_decode.cuh)
  float* attn;              // [B*T0, Hq*hd]
  float scaling;
  const int* slot;          // [B] decode row (block-table row) of prompt b; nullptr: row b
};

// RoPE + KV append for every valid prompt token; grid (T0, B), 256 threads over (which, head, j).  KVT: the cache's
// element type (__half: K and V are rounded to nearest even as they are appended).
template <typename KVT>
__global__ void k_prefill_rope_kv(const PrefillP p) {
  const int c = blockIdx.x, b = blockIdx.y;
  if (!p.mask[(size_t)b * p.T0 + c]) return;
  const int pos = p.npre[(size_t)b * p.T0 + c];
  const int half = p.hd / 2, nq = p.Hq * p.hd, nkv = p.Hkv * p.hd;
  const float* src = p.qkv + ((size_t)b * p.T0 + c) * (nq + 2 * nkv);
  const int page = p.block_table[(p.slot ? p.slot[b] : b) * p.pages_per_row + pos / kPageTokens];
  const int npairs = (p.Hq + 2 * p.Hkv) * half;
  for (int i = threadIdx.x; i < npairs; i += blockDim.x) {
    const int which = i < p.Hq * half ? 0 : (i < (p.Hq + p.Hkv) * half ? 1 : 2);
    const int t = i - (which == 0 ? 0 : (which == 1 ? p.Hq * half : (p.Hq + p.Hkv) * half));
    const int h = t / half, j = t % half;
    const int base = (which == 0 ? 0 : (which == 1 ? nq : nq + nkv)) + h * p.hd;
    const float v0 = src[base + j], v1 = src[base + j + half];
    float o0 = v0, o1 = v1;
    if (which < 2) {
      const float c0 = p.rope_cos[(size_t)pos * p.hd + j], s0 = p.rope_sin[(size_t)pos * p.hd + j];
      const float c1 = p.rope_cos[(size_t)pos * p.hd + j + half], s1 = p.rope_sin[(size_t)pos * p.hd + j + half];
      o0 = __fadd_rn(__fmul_rn(v0, c0), __fmul_rn(-v1, s0));
      o1 = __fadd_rn(__fmul_rn(v1, c1), __fmul_rn(v0, s1));
    }
    const int i0 = (which < 2 && p.permute_qk) ? 2 * j : j;
    const int i1 = (which < 2 && p.permute_qk) ? 2 * j + 1 : j + half;
    if (which == 0) {
      float* dst = p.q + ((size_t)b * p.T0 + c) * nq + h * p.hd;
      dst[i0] = o0; dst[i1] = o1;
    } else {
      KVT* dst = reinterpret_cast<KVT*>(p.kv) + kv_off(page, which - 1, h, pos % kPageTokens, p.Hkv, p.hd);
      dst[i0] = KVT(o0); dst[i1] = KVT(o1);
    }
  }
}

// RoPE of the queries alone, as k_prefill_rope_kv computes them, with no KV append: the attention-map pass
// (ctb_gpt_attention_maps) reads the K / V the decode wrote and leaves them as they are.  Grid (T0, B), 256 threads.
__global__ void k_prefill_rope_q(const PrefillP p) {
  const int c = blockIdx.x, b = blockIdx.y;
  if (!p.mask[(size_t)b * p.T0 + c]) return;
  const int pos = p.npre[(size_t)b * p.T0 + c];
  const int half = p.hd / 2, nq = p.Hq * p.hd, nkv = p.Hkv * p.hd;
  const float* src = p.qkv + ((size_t)b * p.T0 + c) * (nq + 2 * nkv);
  float* dst = p.q + ((size_t)b * p.T0 + c) * nq;
  for (int i = threadIdx.x; i < p.Hq * half; i += blockDim.x) {
    const int h = i / half, j = i % half;
    const float v0 = src[h * p.hd + j], v1 = src[h * p.hd + j + half];
    const float c0 = p.rope_cos[(size_t)pos * p.hd + j], s0 = p.rope_sin[(size_t)pos * p.hd + j];
    const float c1 = p.rope_cos[(size_t)pos * p.hd + j + half], s1 = p.rope_sin[(size_t)pos * p.hd + j + half];
    const float o0 = __fadd_rn(__fmul_rn(v0, c0), __fmul_rn(-v1, s0));
    const float o1 = __fadd_rn(__fmul_rn(v1, c1), __fmul_rn(v0, s1));
    dst[h * p.hd + (p.permute_qk ? 2 * j : j)] = o0;
    dst[h * p.hd + (p.permute_qk ? 2 * j + 1 : j + half)] = o1;
  }
}

// The attention-map pass (ctb_gpt_attention_maps) over columns [a, a + nc) of the B rows of a static batch: which
// columns have a map row, and their positions.  mask_out / npre_out [B, nc] (k_prefill_rope_q's mask and positions):
// column c of row b is valid when pad_b <= c < T0 + end_idx[b] (steps up to the row's end), at position c - pad_b,
// pad_b the zeros of the row's prompt mask.  Grid B, 256 threads.
__global__ void k_attn_map_positions(const uint8_t* __restrict__ prompt_mask, const int* __restrict__ end_idx, int T0,
                                     int a, int nc, uint8_t* __restrict__ mask_out, int* __restrict__ npre_out) {
  __shared__ int s_pad;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) s_pad = 0;
  __syncthreads();
  int z = 0;
  for (int c = threadIdx.x; c < T0; c += blockDim.x) z += prompt_mask[(size_t)b * T0 + c] == 0;
  atomicAdd(&s_pad, z);
  __syncthreads();
  const int pad = s_pad, last = T0 + end_idx[b];
  for (int j = threadIdx.x; j < nc; j += blockDim.x) {
    const int c = a + j;
    mask_out[(size_t)b * nc + j] = c >= pad && c < last;
    npre_out[(size_t)b * nc + j] = c - pad;
  }
}

// Attention of the map pass, and its probabilities written where the reference's GenerationOutputs.attentions has
// them.  The output is the blocks of steps i0, i0 + 1, ... (step of column q0), each [L, B, Hq, rows, cols] fp32:
// step 0 (columns 0 .. T0 - 1) has rows = cols = T0, step i >= 1 (column T0 + i - 1) rows = 1, cols = T0 + i.  Key
// column k of row b holds its position k - pad_b.
struct AttnMapP {
  const float* q;          // [B * nc, Hq * 64] queries of the chunk's columns (RoPE applied, the pages' q / k layout)
  float* attn;             // [B * nc, Hq * 64] attention output (zero for columns without a map row)
  const uint8_t* mask;     // [B, nc] column has a map row (k_attn_map_positions)
  const int* npre;         // [B, nc] its position
  const float* kv;         // the layer's pages (fp32)
  const int* block_table; int pages_per_row;
  float* out;
  int L, B, Hq, Hkv, T0, q0, a, nc, layer;
  float scaling;
};

// Grid (nc, Hq, B), AM_THREADS threads: one CTA per (column, head, row).  A column without a map row writes its fill
// row: a padded prompt row 1 / T0 everywhere (eager attention's fully masked row), a step after the row's end zeros
// (the device appends no KV for a finished row).  A valid column scores its keys 0 .. t (t its position) as
// k_prefill_attn does (the same fmaf chain over the 64 dims, then the scale), takes the max and the sum in a fixed
// order (thread-strided partials, xor butterfly, warps in order), so the same inputs give the same bits, writes the
// whole map row (padded key columns and keys after the query 0, the others e / sum rounded once) and the attention
// output sum_k p_k v_k (dims split over two halves of the CTA, keys even / odd, added in that order).  Dynamic
// shared memory: AM_SMEM_FLOATS + the call's widest row (q0 + n floats).
constexpr int AM_THREADS = 128, AM_SMEM_FLOATS = 64 + AM_THREADS / 32 + 64;
__global__ void __launch_bounds__(AM_THREADS) k_attn_probs(const AttnMapP p) {
  constexpr int HD = 64, NW = AM_THREADS / 32;
  const int j = blockIdx.x, h = blockIdx.y, b = blockIdx.z, c = p.a + j, tid = threadIdx.x;
  const size_t row = (size_t)b * p.nc + j;
  const int step = c < p.T0 ? 0 : c - p.T0 + 1, i0 = p.q0 < p.T0 ? 0 : p.q0 - p.T0 + 1;
  const int rows = step ? 1 : p.T0, cols = step ? p.T0 + step : p.T0;
  int64_t blk = 0;  // elements per (layer, row, head) of the blocks of steps i0 .. step - 1
  if (step > 0) {
    const int64_t j0 = i0 > 0 ? i0 : 1;
    blk = (i0 == 0 ? (int64_t)p.T0 * p.T0 : 0) + (step - j0) * p.T0 + (j0 + step - 1) * (step - j0) / 2;
  }
  float* o = p.out + blk * p.L * p.B * p.Hq +
             ((((int64_t)p.layer * p.B + b) * p.Hq + h) * rows + (step ? 0 : c)) * cols;
  float* ao = p.attn + (row * p.Hq + h) * HD;
  if (!p.mask[row]) {
    const float v = step == 0 ? 1.0f / (float)p.T0 : 0.f;
    for (int k = tid; k < cols; k += AM_THREADS) o[k] = v;
    if (tid < HD) ao[tid] = 0.f;
    return;
  }
  extern __shared__ float am_smem[];
  float* s_q = am_smem;                // [64]
  float* s_red = am_smem + HD;         // [NW]
  float* s_o = s_red + NW;             // [64] the odd keys' half of the output
  float* s_p = am_smem + AM_SMEM_FLOATS;  // [t + 1]
  const int t = p.npre[row], pad = c - t;
  const int hk = h / (p.Hq / p.Hkv), lane = tid & 31, warp = tid >> 5;
  const int* bt = p.block_table + (size_t)b * p.pages_per_row;
  if (tid < HD) s_q[tid] = p.q[(row * p.Hq + h) * HD + tid];
  __syncthreads();
  const float4* q4 = reinterpret_cast<const float4*>(s_q);
  float m = -INFINITY;
  for (int k = tid; k <= t; k += AM_THREADS) {
    const float4* kr = reinterpret_cast<const float4*>(p.kv + kv_off(bt[k / kPageTokens], 0, hk, k % kPageTokens, p.Hkv, HD));
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < HD / 4; ++i) {
      const float4 kk = kr[i], qq = q4[i];
      s = fmaf(qq.x, kk.x, s); s = fmaf(qq.y, kk.y, s); s = fmaf(qq.z, kk.z, s); s = fmaf(qq.w, kk.w, s);
    }
    s *= p.scaling;
    s_p[k] = s;
    m = fmaxf(m, s);
  }
  m = warp_max(m);
  if (lane == 0) s_red[warp] = m;
  __syncthreads();
  m = s_red[0];
#pragma unroll
  for (int w = 1; w < NW; ++w) m = fmaxf(m, s_red[w]);
  __syncthreads();  // s_red is reused for the sum
  float sum = 0.f;
  for (int k = tid; k <= t; k += AM_THREADS) { const float e = expf(s_p[k] - m); s_p[k] = e; sum += e; }
  sum = warp_sum(sum);
  if (lane == 0) s_red[warp] = sum;
  __syncthreads();  // also: every e is in s_p
  sum = s_red[0];
#pragma unroll
  for (int w = 1; w < NW; ++w) sum += s_red[w];
  for (int k = tid; k < cols; k += AM_THREADS) {
    const int kp = k - pad;  // padded key columns and keys after the query: probability 0
    o[k] = (kp >= 0 && kp <= t) ? __fdiv_rn(s_p[kp], sum) : 0.f;
  }
  // attention output: dim d = tid % 64 over keys of parity tid / 64, V read a page row at a time
  const int d = tid & (HD - 1), par = tid >> 6;
  float acc = 0.f;
  for (int k = par; k <= t; k += 2)
    acc = fmaf(s_p[k], p.kv[kv_off(bt[k / kPageTokens], 1, hk, k % kPageTokens, p.Hkv, HD) + d], acc);
  if (par) s_o[d] = acc;
  __syncthreads();
  if (!par) ao[d] = (acc + s_o[d]) / sum;  // V (and the output) is never permuted
}

// Causal attention over the row's valid prompt tokens, query-parallel: grid (ceil(T0 / 8), Hq, B), 8 warps per CTA,
// ONE WARP PER QUERY (hd == 64).  Pass 1: lane-per-key scores into the warp's shared-memory row (same fma order per score
// as the decode kernels), warp max; pass 2: exponentials + sum; pass 3: P.V with lane = two output dims, keys in order.
// (Round 1 walked the queries of a (row, head) serially in one 128-thread CTA: 12 CTAs on 132 SMs and O(T^2) per CTA -
// fine for 16-token prompts, hopeless for speaker-prompt prefixes of hundreds of tokens.)
// KVT: the cache's element type, widened to fp32 as it is read.
//
// q0: position of the call's first query (a chunk of a longer prompt whose columns 0 .. q0 - 1 are already in the row's
// pages, with B = 1 and T0 = the chunk's columns, all valid; 0 for a whole prompt).  Query j of the call is prompt
// position q0 + j and attends to keys 0 .. q0 + j, each with the arithmetic a one-call prefill gives that position.
// Shared memory: 8 x (q0 + T0) floats.
constexpr int PF_ATT_WARPS = 8;
template <typename KVT>
__global__ void __launch_bounds__(PF_ATT_WARPS * 32) k_prefill_attn(const PrefillP p, int q0) {
  constexpr int HD = 64;
  const int h = blockIdx.y, b = blockIdx.z, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = p.nvalid[b];
  const int j = blockIdx.x * PF_ATT_WARPS + warp;  // query among the call's valid tokens
  if (j >= n) return;                              // warp-uniform; the kernel has no block-wide barrier
  const int t = q0 + j;                            // its position in the prompt
  extern __shared__ float pa_smem[];
  float* s_p = pa_smem + (size_t)warp * (q0 + p.T0);  // [q0 + T0] scores / probabilities of this warp's query
  const int hk = h / (p.Hq / p.Hkv);
  const int* bt = p.block_table + (p.slot ? p.slot[b] : b) * p.pages_per_row;
  const int c0 = p.T0 - n;                        // first valid column (left padding)
  const size_t qrow = ((size_t)b * p.T0 + c0 + j) * p.Hq * HD + h * HD;
  float4 q[HD / 4];
#pragma unroll
  for (int i = 0; i < HD / 4; ++i) q[i] = __ldg(reinterpret_cast<const float4*>(p.q + qrow) + i);
  const KVT* kv = reinterpret_cast<const KVT*>(p.kv);
  float m = -INFINITY;
  for (int k = lane; k <= t; k += 32) {
    float s = 0.f;
    if constexpr (std::is_same<KVT, float>::value) {
      const float4* kr = reinterpret_cast<const float4*>(kv + kv_off(bt[k / kPageTokens], 0, hk, k % kPageTokens, p.Hkv, HD));
#pragma unroll
      for (int i = 0; i < HD / 4; ++i) {
        const float4 kk = kr[i];
        s = fmaf(q[i].x, kk.x, s); s = fmaf(q[i].y, kk.y, s); s = fmaf(q[i].z, kk.z, s); s = fmaf(q[i].w, kk.w, s);
      }
    } else {
      const uint4* kr = reinterpret_cast<const uint4*>(kv + kv_off(bt[k / kPageTokens], 0, hk, k % kPageTokens, p.Hkv, HD));
#pragma unroll
      for (int i = 0; i < HD / 8; ++i) {
        const uint4 u = kr[i];
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&w[2 * j]));
          const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&w[2 * j + 1]));
          const float4 qq = q[2 * i + j];
          s = fmaf(qq.x, a.x, s); s = fmaf(qq.y, a.y, s); s = fmaf(qq.z, b.x, s); s = fmaf(qq.w, b.y, s);
        }
      }
    }
    s *= p.scaling;
    s_p[k] = s;
    m = fmaxf(m, s);
  }
  m = warp_max(m);
  float l = 0.f;
  for (int k = lane; k <= t; k += 32) { const float e = expf(s_p[k] - m); s_p[k] = e; l += e; }
  l = warp_sum(l);
  __syncwarp();
  float o0 = 0.f, o1 = 0.f;
#pragma unroll 4
  for (int k = 0; k <= t; ++k) {
    const KVT* vp = kv + kv_off(bt[k / kPageTokens], 1, hk, k % kPageTokens, p.Hkv, HD) + 2 * lane;
    float2 v;
    if constexpr (std::is_same<KVT, float>::value) v = *reinterpret_cast<const float2*>(vp);
    else v = __half22float2(*reinterpret_cast<const __half2*>(vp));
    const float pk = s_p[k];
    o0 = fmaf(pk, v.x, o0); o1 = fmaf(pk, v.y, o1);
  }
  *reinterpret_cast<float2*>(p.attn + qrow + 2 * lane) = make_float2(o0 / l, o1 / l);  // V (and the output) is never permuted
}

// k_prefill_attn keeps a query's whole score row in shared memory (8 x T0 floats per CTA): prompts wider than this
// take k_prefill_attn_tiled.  The choice depends on T0 alone, so a prompt of up to 1,024 columns is computed as before.
constexpr int PF_ATT_MAX_T0 = 1024;

// Tiled causal attention for prompts over PF_ATT_MAX_T0 columns: grid (ceil(T0 / 64), Hq, B), 256 threads.  A CTA takes
// 64 consecutive queries t of one (row, head) and walks the key tiles 0 .. t / 64 (tiles wholly above the diagonal are
// never loaded), each 64 keys = 4 pages of the row's block table, staged into shared memory once for all 64 queries with
// cp.async and double-buffered.  Online softmax in fp32: running max and sum per query, the accumulator rescaled when
// the max grows; causal mask inside the diagonal tile.  Thread (ty, tx) = (tid / 16, tid % 16) owns queries
// 4 ty .. 4 ty + 3, and keys tx + 16 j of a tile for the scores, dims 4 tx .. 4 tx + 3 for P.V.  A score is the same
// fmaf chain over the 64 dims as k_prefill_attn's.  Shared memory is fixed (PftSmem), whatever T0.  KVT: the cache's
// element type, staged as it is stored and widened to fp32 as it is read.
constexpr int PFT_TILE = 64, PFT_THREADS = 256;
template <typename KVT>
struct PftSmem {
  static constexpr int QS = PFT_TILE + 4;                         // Q / P row stride (floats): 16-byte rows, one pad
  static constexpr int KS = PFT_TILE + 16 / (int)sizeof(KVT);     // K / V row stride (elements): one 16-byte pad
  static constexpr int CH = PFT_TILE * (int)sizeof(KVT) / 16;     // 16-byte chunks per K / V row
  static constexpr int Q_FLOATS = PFT_TILE * QS;
  static constexpr int KV_ELEMS = PFT_TILE * KS;                  // one K or V tile
  static constexpr int BYTES = 2 * Q_FLOATS * 4 + 2 * 2 * KV_ELEMS * (int)sizeof(KVT);  // Q, P, 2 stages of K and V
};

__device__ __forceinline__ void pft_cp16(void* smem_dst, const void* gsrc, bool valid) {
  // 16 bytes global -> shared; !valid: no read, 16 zero bytes
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void pft_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void pft_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// 8 consecutive staged values as fp32
__device__ __forceinline__ void pft_ld8(const float* p, float4& a, float4& b) {
  a = *reinterpret_cast<const float4*>(p); b = *reinterpret_cast<const float4*>(p + 4);
}
__device__ __forceinline__ void pft_ld8(const __half* p, float4& a, float4& b) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
  const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  const float2 f2 = __half22float2(*reinterpret_cast<const __half2*>(&u.z));
  const float2 f3 = __half22float2(*reinterpret_cast<const __half2*>(&u.w));
  a = make_float4(f0.x, f0.y, f1.x, f1.y); b = make_float4(f2.x, f2.y, f3.x, f3.y);
}
// 4 consecutive staged values as fp32
__device__ __forceinline__ float4 pft_ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 pft_ld4(const __half* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
  const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(f0.x, f0.y, f1.x, f1.y);
}

//
// q0 (a multiple of 64) as in k_prefill_attn: the call's query tile qj is the prompt's tile q0 / 64 + qj, the same 64
// queries a one-call prefill gives one CTA, and keys past q0 + n - 1 are zero-filled as keys past a whole prompt's last
// are (the pages there hold an earlier request's values).
template <typename KVT>
__global__ void __launch_bounds__(PFT_THREADS) k_prefill_attn_tiled(const PrefillP p, int q0) {
  using SM = PftSmem<KVT>;
  constexpr int HD = 64, T = PFT_TILE;
  const int h = blockIdx.y, b = blockIdx.z, tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int n = p.nvalid[b];                   // queries of the call
  const int kn = q0 + n;                       // keys: positions 0 .. kn - 1
  const int qj = gridDim.x - 1 - blockIdx.x;  // the longest walks start first
  if (qj * T >= n) return;                     // CTA-uniform, before any barrier
  const int qt = q0 / T + qj;                  // query tile of the prompt
  extern __shared__ __align__(16) unsigned char pft_smem[];
  float* sQ = reinterpret_cast<float*>(pft_smem);
  float* sP = sQ + SM::Q_FLOATS;
  KVT* sKV = reinterpret_cast<KVT*>(sP + SM::Q_FLOATS);  // [stage][K, V][T][KS]
  const int hk = h / (p.Hq / p.Hkv);
  const int* bt = p.block_table + (p.slot ? p.slot[b] : b) * p.pages_per_row;
  const int c0 = p.T0 - n;                     // first valid column (left padding)
  const KVT* kv = reinterpret_cast<const KVT*>(p.kv);
  const size_t row0 = (size_t)b * p.T0 + c0;   // column of query / key 0

  // queries qt*64 .. qt*64+63 (zeros past the row's last)
  for (int i = tid; i < T * 16; i += PFT_THREADS) {
    const int r = i >> 4, c = i & 15, t = qj * T + r;
    const float* src = t < n ? p.q + ((row0 + t) * p.Hq + h) * HD + c * 4 : p.q;
    pft_cp16(sQ + r * SM::QS + c * 4, src, t < n);
  }
  // keys / values of tile kt into stage st (zeros past the row's last key)
  auto load_kv = [&](int kt, int st) {
    KVT* dst = sKV + (size_t)st * 2 * SM::KV_ELEMS;
    for (int i = tid; i < 2 * T * SM::CH; i += PFT_THREADS) {
      const int which = i / (T * SM::CH), r = (i / SM::CH) % T, c = i % SM::CH, k = kt * T + r;
      constexpr int E = 16 / (int)sizeof(KVT);
      const KVT* src = k < kn ? kv + kv_off(bt[k / kPageTokens], which, hk, k % kPageTokens, p.Hkv, HD) + c * E : kv;
      pft_cp16(dst + which * SM::KV_ELEMS + r * SM::KS + c * E, src, k < kn);
    }
  };
  load_kv(0, 0);
  pft_commit();

  float m[4], l[4], o[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m[i] = -INFINITY; l[i] = 0.f;
#pragma unroll
    for (int e = 0; e < 4; ++e) o[i][e] = 0.f;
  }
  for (int kt = 0; kt <= qt; ++kt) {
    const int st = kt & 1;
    if (kt < qt) { load_kv(kt + 1, st ^ 1); pft_commit(); pft_wait<1>(); }
    else pft_wait<0>();
    __syncthreads();
    const KVT* sK = sKV + (size_t)st * 2 * SM::KV_ELEMS;
    const KVT* sV = sK + SM::KV_ELEMS;
    // scores of queries 4 ty + i against keys tx + 16 j
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 2
    for (int d = 0; d < HD; d += 8) {
      float4 qa[4], qb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        qa[i] = *reinterpret_cast<const float4*>(sQ + (ty * 4 + i) * SM::QS + d);
        qb[i] = *reinterpret_cast<const float4*>(sQ + (ty * 4 + i) * SM::QS + d + 4);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float4 ka, kb;
        pft_ld8(sK + (tx + 16 * j) * SM::KS + d, ka, kb);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float a = s[i][j];
          a = fmaf(qa[i].x, ka.x, a); a = fmaf(qa[i].y, ka.y, a); a = fmaf(qa[i].z, ka.z, a); a = fmaf(qa[i].w, ka.w, a);
          a = fmaf(qb[i].x, kb.x, a); a = fmaf(qb[i].y, kb.y, a); a = fmaf(qb[i].z, kb.z, a); a = fmaf(qb[i].w, kb.w, a);
          s[i][j] = a;
        }
      }
    }
    // causal mask, online softmax (a query's 64 scores are spread over the 16 lanes tx of its half-warp)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int t = min(q0 + qj * T + ty * 4 + i, kn - 1);  // queries past the row's last see its keys, and are not written
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int k = kt * T + tx + 16 * j;
        s[i][j] = k <= t ? s[i][j] * p.scaling : -INFINITY;
        mx = fmaxf(mx, s[i][j]);
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      const float mn = fmaxf(m[i], mx);            // finite: key kt * 64 <= t is never masked
      const float alpha = expf(m[i] - mn);         // 0 on the first tile
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float e = expf(s[i][j] - mn);
        sP[(ty * 4 + i) * SM::QS + tx + 16 * j] = e;
        sum += e;
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
      l[i] = l[i] * alpha + sum;
      m[i] = mn;
#pragma unroll
      for (int e = 0; e < 4; ++e) o[i][e] *= alpha;
    }
    __syncthreads();
    // o += P . V over the tile's keys in order
#pragma unroll 2
    for (int k = 0; k < T; k += 4) {
      float4 pr[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) pr[i] = *reinterpret_cast<const float4*>(sP + (ty * 4 + i) * SM::QS + k);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const float4 v = pft_ld4(sV + (k + kk) * SM::KS + tx * 4);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float pk = kk == 0 ? pr[i].x : kk == 1 ? pr[i].y : kk == 2 ? pr[i].z : pr[i].w;
          o[i][0] = fmaf(pk, v.x, o[i][0]); o[i][1] = fmaf(pk, v.y, o[i][1]);
          o[i][2] = fmaf(pk, v.z, o[i][2]); o[i][3] = fmaf(pk, v.w, o[i][3]);
        }
      }
    }
    __syncthreads();  // stage st and P are rewritten by the next tile
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int t = qj * T + ty * 4 + i;
    if (t < n)  // V (and the output) is never permuted
      *reinterpret_cast<float4*>(p.attn + ((row0 + t) * p.Hq + h) * HD + tx * 4) =
          make_float4(o[i][0] / l[i], o[i][1] / l[i], o[i][2] / l[i], o[i][3] / l[i]);
  }
}

// h = silu(gate) * up over [M, 2I] -> [M, I]
__global__ void k_silu_mul(const float* __restrict__ gu, float* __restrict__ h, int M, int I) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)M * I) return;
  const size_t m = i / I, n = i % I;
  const float g = gu[m * 2 * I + n], u = gu[m * 2 * I + I + n];
  h[i] = __fmul_rn(__fdiv_rn(g, __fadd_rn(1.0f, expf(-g))), u);
}

// prompt positions: npre[b, c] = #valid columns before c ; nvalid[b]
__global__ void k_prefill_positions(const uint8_t* __restrict__ mask, int* __restrict__ npre, int* __restrict__ nvalid, int T0) {
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    int n = 0;
    for (int c = 0; c < T0; ++c) { npre[(size_t)b * T0 + c] = n; n += mask[(size_t)b * T0 + c] != 0; }
    nvalid[b] = n;
  }
}

// a chunk of n columns of one prompt, at positions q0 .. q0 + n - 1, into decode row `slot`: every column valid
// (k_prefill_rope_kv's mask and positions), nvalid[0] = n (the chunk's queries), nvalid[1] = q0 + n (the row's tokens
// after it: k_prefill_finish's seq_len on the final chunk), slot_dev[0] = slot
__global__ void k_prefill_chunk_positions(uint8_t* __restrict__ mask, int* __restrict__ npre, int* __restrict__ nvalid,
                                          int* __restrict__ slot_dev, int slot, int q0, int n) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) { mask[c] = 1; npre[c] = q0 + c; }
  if (blockIdx.x == 0 && threadIdx.x == 0) { nvalid[0] = n; nvalid[1] = q0 + n; slot_dev[0] = slot; }
}

// hand the last prompt column's residual to the decode-loop state of decode row slot[b] (slot == nullptr: row b)
__global__ void k_prefill_finish(const float* __restrict__ resid, float* __restrict__ x, float* __restrict__ x_hi,
                                 float* __restrict__ x_lo, const int* __restrict__ nvalid, int* __restrict__ seq_len,
                                 int* __restrict__ pos, uint8_t* __restrict__ active, int T0, int d,
                                 const int* __restrict__ slot) {
  const int b = blockIdx.x, sb = slot ? slot[b] : b;
  const float* r = resid + ((size_t)b * T0 + T0 - 1) * d;
  for (int k = threadIdx.x; k < d; k += blockDim.x) {
    const float v = r[k];
    x[(size_t)sb * d + k] = v;
    if (x_hi != nullptr) {
      uint32_t hb, lb;
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(v));
      asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(v - __uint_as_float(hb)));
      x_hi[(size_t)sb * d + k] = __uint_as_float(hb);
      x_lo[(size_t)sb * d + k] = __uint_as_float(lb);
    }
  }
  if (threadIdx.x == 0) {
    const int n = nvalid[b];
    seq_len[sb] = n; pos[sb] = n - 1; active[sb] = 1;
  }
}

#endif  // CTB_GPT_KERNELS_IMPL

}  // namespace ctb
