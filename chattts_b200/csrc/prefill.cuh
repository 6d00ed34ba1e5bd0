// Batched prefill (SURVEY.md 8f N1; reference gpt.py:396-427 at i == 0): the whole left-padded prompt batch
// [B, T0, 768] goes through the 20 layers as token-parallel GEMMs on wgmma (k_tc_gemm, 3xTF32 =
// fp32-equivalent) instead of one decode step per prompt column.  Each batch row is one "utterance" of T0 frames
// for the GEMM tiler; pad columns are computed but never written to the KV cache nor attended to.
//
//   per layer:  k_rms_rows -> GEMM(Wqkv) -> k_prefill_rope_kv (RoPE, q buffer, paged-KV append)
//               -> k_prefill_attn (causal over the row's valid tokens) -> GEMM(Wo)+residual
//               -> k_rms_rows -> GEMM([Wgate;Wup]) -> k_silu_mul -> GEMM(Wdown)+residual
//   then k_prefill_finish hands the last column's residual to the decode-loop state (x, seq_len) and the
//   regular heads -> sampler -> finalize kernels produce the first token.
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

// Causal attention over the row's valid prompt tokens, query-parallel: grid (ceil(T0 / 8), Hq, B), 8 warps per CTA,
// ONE WARP PER QUERY (hd == 64).  Pass 1: lane-per-key scores into the warp's shared-memory row (same fma order per score
// as the decode kernels), warp max; pass 2: exponentials + sum; pass 3: P.V with lane = two output dims, keys in order.
// (Round 1 walked the queries of a (row, head) serially in one 128-thread CTA: 12 CTAs on 132 SMs and O(T^2) per CTA -
// fine for 16-token prompts, hopeless for speaker-prompt prefixes of hundreds of tokens.)
// KVT: the cache's element type, widened to fp32 as it is read.
constexpr int PF_ATT_WARPS = 8;
template <typename KVT>
__global__ void __launch_bounds__(PF_ATT_WARPS * 32) k_prefill_attn(const PrefillP p) {
  constexpr int HD = 64;
  const int h = blockIdx.y, b = blockIdx.z, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = p.nvalid[b];
  const int t = blockIdx.x * PF_ATT_WARPS + warp;  // query position among the row's valid tokens
  if (t >= n) return;                              // warp-uniform; the kernel has no block-wide barrier
  extern __shared__ float pa_smem[];
  float* s_p = pa_smem + (size_t)warp * p.T0;      // [T0] scores / probabilities of this warp's query
  const int hk = h / (p.Hq / p.Hkv);
  const int* bt = p.block_table + (p.slot ? p.slot[b] : b) * p.pages_per_row;
  const int c0 = p.T0 - n;                        // first valid column (left padding)
  const size_t qrow = ((size_t)b * p.T0 + c0 + t) * p.Hq * HD + h * HD;
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
