// Decode-step GEMMs on wgmma tensor cores (swap-AB, 3xTF32, split-K over a thread-block cluster).
//
//   Y[b, r] = sum_k W[r, k] * x[b, k]        W: [rows, K] fp32 streamed from HBM exactly once by TMA
//
//   * swap-AB: the 128 weight rows of a tile are the MMA M dimension (two m64 wgmmas), the (padded) batch is N = NPAD.
//   * fp32-equivalent accuracy for the bit-exact-ids contract: W = W_hi + W_lo is split in shared memory by
//     the worker warpgroup (cvt.rna.tf32; weights cannot be pre-split without doubling HBM traffic), the
//     activations arrive pre-split (x_hi, x_lo written by the producing kernel's epilogue).  Two MMAs per
//     k-step:  W_hi x [x_hi ; x_lo] (N = 2*NPAD, one pass over the W_hi tile) and W_lo x x_hi (N = NPAD).
//   * split-K: the CS CTAs of a cluster own consecutive K slices of the same 128 rows, so 6..48 row tiles
//     still put ~100+ SMs on the HBM stream; partial accumulators meet through distributed shared memory
//     in a fixed order (deterministic), and the rank that owns a row slice runs the fused epilogue:
//     RMSNorm scale (norm weight folded into W at load, 1/rms applied here), RoPE + paged-KV append,
//     residual add, SiLU*up, logits.  Row pairs that must meet in one thread (RoPE j / j+32, gate_n / up_n)
//     are made adjacent by a row permutation applied once when the tensor-core weight copy is built.
//   * 4-stage TMA/mbarrier ring; weight tiles of the first stages are requested BEFORE griddepcontrol.wait
//     (PDL), activations after it.
//   * half-precision slot engine (PREC & TD_W16): the weight copy is fp16 (8 KiB tiles by TMA, unswizzled).  The
//     worker warpgroup widens a tile into the fp32 128-byte-swizzled tile the descriptors read; an fp16 value is
//     exactly a tf32 value, so W_lo = 0 and one MMA per k-step, W x [x_hi ; x_lo], is the whole product.  k order,
//     split-K and epilogues are those of the fp32 kernel (same results on fp16-representable weights).
//     PREC & TD_KV16: the QKV epilogue appends K/V to an fp16 cache.
#pragma once
#include "gpt_kernels.cuh"
#include "tc_common.cuh"

namespace ctb {

enum DecEpi { DE_QKV = 0, DE_OPROJ = 1, DE_GATEUP = 2, DE_DOWN = 3, DE_HEADS = 4 };
enum DecPrec { TD_W16 = 1, TD_KV16 = 2 };  // the bits of CTB_ENGINE_FP16_WEIGHTS / CTB_ENGINE_FP16_KV

// 3 stages of 28-40 KiB at NPAD 16 / 32: two CTAs (this kernel + its PDL successor) fit one SM; at NPAD 64 (40 KiB
// fp16 / 48 KiB fp32 stages, 121.5 / 145.5 KiB in all) one CTA per SM
constexpr int TD_STAGES = 3;
constexpr int TD_THREADS = 160;  // warps 0-3: one warpgroup (rms, W split, wgmma, epilogue); warp 4: TMA
constexpr int TD_A_BYTES = 128 * 32 * 4;  // 16 KiB weight tile (128 rows x 32 k)
constexpr int TD_A16_BYTES = 128 * 32 * 2;  // 8 KiB fp16 weight tile as TMA lands it

template <int NPAD, bool W16 = false>
struct TdCfg {
  static constexpr int X_BYTES = NPAD * 128;                       // one x tile (NPAD rows x 32 k)
  // fp32: W | W_lo | x_hi | x_lo      fp16: W (widened) | x_hi | x_lo | W16
  static constexpr int X_OFF = W16 ? TD_A_BYTES : 2 * TD_A_BYTES;
  static constexpr int W16_OFF = X_OFF + 2 * X_BYTES;
  static constexpr int W_TX = W16 ? TD_A16_BYTES : TD_A_BYTES;  // weight bytes TMA brings per stage
  static constexpr int STAGE_BYTES = W16 ? W16_OFF + TD_A16_BYTES : 2 * TD_A_BYTES + 2 * X_BYTES;
  static constexpr int SMEM_BYTES = TD_STAGES * STAGE_BYTES + 1024 + 512;
};

struct TcDecP {
  int K, kslice, nrows, B;
  const float* xraw;      // [Bpad][K] raw residual rows for 1/rms (nullptr: no norm)
  float eps;
  float* xres; float* x_hi; float* x_lo; int d;                      // OPROJ / DOWN
  float* qbuf; float* kv; const int* block_table; int pages_per_row;  // QKV
  const int* pos; const uint8_t* active; const float* rope_cos; const float* rope_sin;
  int Hq, Hkv, hd;
  float* h_hi; float* h_lo; int I;                                    // GATEUP
  float* logits; int rows_per_item, V;                                // HEADS
  float* hidden_out; int hidden_stride; const float* final_norm_w; const LoopState* st;
  const RowState* rows; int want;  // HEADS in slot-engine mode: only rows matching `want` (nullptr: every row)
};

template <int EPI, int NPAD, int CS, int PREC>
__global__ void __launch_bounds__(TD_THREADS, 1)
k_tc_dec(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_xhi,
         const __grid_constant__ CUtensorMap map_xlo, const TcDecP p) {
  constexpr bool W16 = (PREC & TD_W16) != 0;
  using Cfg = TdCfg<NPAD, W16>;
  pdl_trigger();
  extern __shared__ uint8_t td_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(td_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TD_STAGES * Cfg::STAGE_BYTES);
  uint64_t* full = bars;                  // [stages]  TMA bytes landed
  uint64_t* empty = bars + TD_STAGES;     // [stages]  the stage's MMAs retired
  float* s_rinv = reinterpret_cast<float*>(bars + 2 * TD_STAGES);  // [NPAD]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rank = (CS > 1) ? (int)cluster_ctarank() : 0;
  const int tile = blockIdx.x / CS;
  const int r_tile = tile * 128;
  const int kbase = rank * p.kslice;
  const int nk = p.kslice / 32;

  if (threadIdx.x == 128) {  // TMA warp: hide the descriptor fetch latency
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_xhi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_xlo) : "memory");
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < TD_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 128); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (EPI == DE_HEADS && p.rows != nullptr && (p.want & WANT_TEXT)) {
    // a slot engine's text head: no weight request before the row states show a text row to serve (every CTA of
    // the cluster reads the same states and leaves together, before any cluster barrier)
    pdl_wait();
    if (!any_row_wanted(p.rows, p.B, p.want)) return;
  }

  if (warp == 4) {
    // ===================== TMA producer
    if (lane == 0) {
      const int pre = min(nk, TD_STAGES);
      constexpr int W_DST = W16 ? Cfg::W16_OFF : 0;
      for (int t = 0; t < pre; ++t) {  // weights do not depend on earlier kernels
        uint8_t* st = smem + t * Cfg::STAGE_BYTES;
        mbar_expect_tx(&full[t], Cfg::W_TX + 2 * Cfg::X_BYTES);
        tma_load_2d(st + W_DST, &map_w, &full[t], kbase + t * 32, r_tile);
      }
      pdl_wait();  // activations below were written by the previous kernel
      for (int t = 0; t < pre; ++t) {
        uint8_t* st = smem + t * Cfg::STAGE_BYTES;
        tma_load_2d(st + Cfg::X_OFF, &map_xhi, &full[t], kbase + t * 32, 0);
        tma_load_2d(st + Cfg::X_OFF + Cfg::X_BYTES, &map_xlo, &full[t], kbase + t * 32, 0);
      }
      for (int t = pre; t < nk; ++t) {
        const int s = t % TD_STAGES, it = t / TD_STAGES;
        mbar_wait(&empty[s], (it - 1) & 1);
        uint8_t* st = smem + s * Cfg::STAGE_BYTES;
        mbar_expect_tx(&full[s], Cfg::W_TX + 2 * Cfg::X_BYTES);
        tma_load_2d(st + W_DST, &map_w, &full[s], kbase + t * 32, r_tile);
        tma_load_2d(st + Cfg::X_OFF, &map_xhi, &full[s], kbase + t * 32, 0);
        tma_load_2d(st + Cfg::X_OFF + Cfg::X_BYTES, &map_xlo, &full[s], kbase + t * 32, 0);
      }
    }
  } else {
    // ===================== workers
    pdl_wait();
    if (p.xraw != nullptr) {  // 1/rms of the raw residual rows (HF LlamaRMSNorm statistics)
      // rows b = warp, warp + 4, ...: all loads of all rows are issued before the first reduction
      constexpr int RPW = NPAD / 4;
      float ss[RPW];
#pragma unroll
      for (int i = 0; i < RPW; ++i) {
        const int b = warp + 4 * i;
        ss[i] = 0.f;
        if (b < p.B) {
          const float4* xr = reinterpret_cast<const float4*>(p.xraw + (size_t)b * p.K);
#pragma unroll
          for (int k4 = 0; k4 < 6; ++k4) {  // K == 768 on every normed GEMM: 6 float4 per lane
            const float4 v = ldg_cg(xr + k4 * 32 + lane);
            ss[i] = fmaf(v.x, v.x, ss[i]); ss[i] = fmaf(v.y, v.y, ss[i]);
            ss[i] = fmaf(v.z, v.z, ss[i]); ss[i] = fmaf(v.w, v.w, ss[i]);
          }
        }
      }
#pragma unroll
      for (int i = 0; i < RPW; ++i) {
        const float t = warp_sum(ss[i]);
        if (lane == 0) s_rinv[warp + 4 * i] = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fdiv_rn(t, (float)p.K), p.eps)));
      }
      if (EPI == DE_HEADS && p.hidden_out != nullptr && blockIdx.x == 0) {
        // last_hidden_state (gpt.py:430-436): w * (x * rinv), written once
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (p.rows == nullptr) {
          const int step = ldg_cg(&p.st->n_gen);
          for (int i = threadIdx.x; i < p.B * p.K; i += 128) {
            const int b = i / p.K, k = i % p.K;
            p.hidden_out[(size_t)b * p.hidden_stride + (size_t)step * p.K + k] =
                __fmul_rn(__ldg(p.final_norm_w + k), __fmul_rn(ldg_cg(p.xraw + i), s_rinv[b]));
          }
        } else {
          for (int b = 0; b < p.B; ++b) {
            if (!row_wanted(p.rows + b, p.want)) continue;
            const int step = ldg_cg(&p.rows[b].n_gen);
            for (int k = threadIdx.x; k < p.K; k += 128)
              p.hidden_out[(size_t)b * p.hidden_stride + (size_t)step * p.K + k] =
                  __fmul_rn(__ldg(p.final_norm_w + k), __fmul_rn(ldg_cg(p.xraw + (size_t)b * p.K + k), s_rinv[b]));
          }
        }
      }
    }
    // accumulators of weight rows [64 hf, 64 hf + 64): columns [0, NPAD) x_hi, [NPAD, 2 NPAD) x_lo
    float acc[2][NPAD];
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int i = 0; i < NPAD; ++i) acc[hf][i] = 0.f;
    int prev = 0;
    for (int t = 0; t < nk; ++t) {
      const int s = t % TD_STAGES, it = t / TD_STAGES;
      mbar_wait(&full[s], it & 1);
      float4* a = reinterpret_cast<float4*>(smem + s * Cfg::STAGE_BYTES);
      if constexpr (W16) {
        // [128 rows][32 k] fp16, 64 B per row -> fp32 rows of 128 B, 16-byte chunk c stored at chunk c ^ (row & 7)
        // (the 128-byte swizzle TMA applies to the fp32 tiles)
        const uint4* w16 = reinterpret_cast<const uint4*>(smem + s * Cfg::STAGE_BYTES + Cfg::W16_OFF);
#pragma unroll
        for (int j = 0; j < TD_A16_BYTES / 16 / 128; ++j) {
          const int i = threadIdx.x + 128 * j, r = i >> 2, c = 2 * (i & 3);
          const uint4 u = w16[i];
          const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
          const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
          const float2 f2 = __half22float2(*reinterpret_cast<const __half2*>(&u.z));
          const float2 f3 = __half22float2(*reinterpret_cast<const __half2*>(&u.w));
          a[r * 8 + (c ^ (r & 7))] = make_float4(f0.x, f0.y, f1.x, f1.y);
          a[r * 8 + ((c + 1) ^ (r & 7))] = make_float4(f2.x, f2.y, f3.x, f3.y);
        }
      } else {
        float4* lo = reinterpret_cast<float4*>(smem + s * Cfg::STAGE_BYTES + TD_A_BYTES);
#pragma unroll
        for (int j = 0; j < TD_A_BYTES / 16 / 128; ++j) {
          const int i = threadIdx.x + 128 * j;
          const float4 v = a[i];
          float4 h, l;
          h.x = to_tf32(v.x); h.y = to_tf32(v.y); h.z = to_tf32(v.z); h.w = to_tf32(v.w);
          l.x = to_tf32(v.x - h.x); l.y = to_tf32(v.y - h.y); l.z = to_tf32(v.z - h.z); l.w = to_tf32(v.w - h.w);
          a[i] = h; lo[i] = l;
        }
      }
      fence_async_smem();  // generic-proxy writes -> visible to the tensor core (async proxy)
      warpgroup_bar(2);
      const uint32_t st = smem_u32(smem + s * Cfg::STAGE_BYTES);
      const uint32_t w_hi = st, w_lo = st + TD_A_BYTES, x_hl = st + Cfg::X_OFF;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t ko = k * 32;
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {
          const uint32_t ro = hf * (TD_A_BYTES / 2);  // 64 rows x 128 B
          // cols [0,NPAD) += W_hi x_hi ; cols [NPAD,2NPAD) += W_hi x_lo   (x_hi | x_lo tiles are contiguous)
          // cols [0,NPAD) += W_lo x_hi   (fp32 weights only)
          if constexpr (NPAD == 16) {
            wgmma_tf32_n32(acc[hf], wgmma_desc_sw128(w_hi + ro + ko), wgmma_desc_sw128(x_hl + ko), (t | k) ? 1u : 0u);
            if constexpr (!W16) wgmma_tf32_n16(acc[hf], wgmma_desc_sw128(w_lo + ro + ko), wgmma_desc_sw128(x_hl + ko), 1u);
          } else if constexpr (NPAD == 32) {
            wgmma_tf32_n64(acc[hf], wgmma_desc_sw128(w_hi + ro + ko), wgmma_desc_sw128(x_hl + ko), (t | k) ? 1u : 0u);
            if constexpr (!W16) wgmma_tf32_n32(acc[hf], wgmma_desc_sw128(w_lo + ro + ko), wgmma_desc_sw128(x_hl + ko), 1u);
          } else {
            wgmma_tf32_n128(acc[hf], wgmma_desc_sw128(w_hi + ro + ko), wgmma_desc_sw128(x_hl + ko), (t | k) ? 1u : 0u);
            if constexpr (!W16) wgmma_tf32_n64(acc[hf], wgmma_desc_sw128(w_lo + ro + ko), wgmma_desc_sw128(x_hl + ko), 1u);
          }
        }
      }
      wgmma_commit();
      if (t > 0) {  // the previous stage's MMAs have retired: hand it back to the producer
        wgmma_wait<1>();
        mbar_arrive(&empty[prev]);
      }
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc[0]);
    wgmma_fence_operands(acc[1]);
    // ---- accumulator -> this CTA's partial tile in shared memory [128 rows][NPAD]
    float* part = reinterpret_cast<float*>(smem);  // stage 0 is free: every MMA has retired
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int i = 0; i < NPAD / 2; ++i) {  // register layout: see wgmma_tf32_n*
        const int row = hf * 64 + warp * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
        const int b = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        part[row * NPAD + b] = acc[hf][i] + acc[hf][i + NPAD / 2];  // x_hi and x_lo halves
      }
  }

  // ===================== split-K merge through DSMEM + fused epilogue (worker warps)
  if (CS > 1) cluster_sync_all(); else __syncthreads();
  if (warp < 4) {
    const float* part = reinterpret_cast<const float*>(smem);
    constexpr int RPR = 128 / CS;  // rows owned by this rank
    const int nitems = (RPR / 2) * p.B;
    for (int item = threadIdx.x; item < nitems; item += 128) {
      const int b = item % p.B, pi = item / p.B;
      const int lr = rank * RPR + 2 * pi;  // local row of the pair
      float v0 = 0.f, v1 = 0.f;
#pragma unroll
      for (int rk = 0; rk < CS; ++rk) {  // fixed order: K slice 0, 1, ... (deterministic)
        if (CS > 1) {
          v0 = __fadd_rn(v0, ld_dsmem(part + lr * NPAD + b, rk));
          v1 = __fadd_rn(v1, ld_dsmem(part + (lr + 1) * NPAD + b, rk));
        } else {
          v0 = part[lr * NPAD + b]; v1 = part[(lr + 1) * NPAD + b];
        }
      }
      const int R = r_tile + lr;  // global (permuted) weight row of the pair's first member
      if (R >= p.nrows) continue;
      const float rinv = p.xraw ? s_rinv[b] : 1.0f;
      if (EPI == DE_QKV) {
        if (!ldg_cg(&p.active[b])) continue;
        const int nq = p.Hq * p.hd, nkv = p.Hkv * p.hd, half = p.hd / 2;
        const float y0 = __fmul_rn(v0, rinv), y1 = __fmul_rn(v1, rinv);
        const int pos = ldg_cg(&p.pos[b]);
        const int which = R < nq ? 0 : (R < nq + nkv ? 1 : 2);
        const int rr = R - (which == 0 ? 0 : (which == 1 ? nq : nq + nkv));
        const int h = rr / p.hd, pp = rr % p.hd;  // pp even: RoPE pair (j, j + hd/2) sits at (2j, 2j+1)
        float o0 = y0, o1 = y1;
        if (which < 2) {
          const int j = pp / 2;
          const float c0 = __ldg(p.rope_cos + (size_t)pos * p.hd + j), s0 = __ldg(p.rope_sin + (size_t)pos * p.hd + j);
          const float c1 = __ldg(p.rope_cos + (size_t)pos * p.hd + j + half), s1 = __ldg(p.rope_sin + (size_t)pos * p.hd + j + half);
          o0 = __fadd_rn(__fmul_rn(y0, c0), __fmul_rn(-y1, s0));
          o1 = __fadd_rn(__fmul_rn(y1, c1), __fmul_rn(y0, s1));
        }
        if (which == 0) {
          *reinterpret_cast<float2*>(p.qbuf + (size_t)b * nq + h * p.hd + pp) = make_float2(o0, o1);
        } else {
          const int page = __ldg(p.block_table + b * p.pages_per_row + pos / kPageTokens);
          const size_t off = kv_off(page, which - 1, h, pos % kPageTokens, p.Hkv, p.hd) + pp;
          if constexpr ((PREC & TD_KV16) != 0) st_kv2(reinterpret_cast<__half*>(p.kv) + off, o0, o1);
          else *reinterpret_cast<float2*>(p.kv + off) = make_float2(o0, o1);
        }
      } else if (EPI == DE_OPROJ || EPI == DE_DOWN) {
        float* xr = p.xres + (size_t)b * p.d + R;
        const float n0 = __fadd_rn(ldg_cg(xr), v0), n1 = __fadd_rn(ldg_cg(xr + 1), v1);
        *reinterpret_cast<float2*>(xr) = make_float2(n0, n1);
        const float h0 = to_tf32(n0), h1 = to_tf32(n1);
        *reinterpret_cast<float2*>(p.x_hi + (size_t)b * p.d + R) = make_float2(h0, h1);
        *reinterpret_cast<float2*>(p.x_lo + (size_t)b * p.d + R) = make_float2(to_tf32(n0 - h0), to_tf32(n1 - h1));
      } else if (EPI == DE_GATEUP) {
        const float g = __fmul_rn(v0, rinv), u = __fmul_rn(v1, rinv);  // rows (2n, 2n+1) = (gate_n, up_n)
        const float hv = __fmul_rn(__fdiv_rn(g, __fadd_rn(1.0f, expf(-g))), u);
        const float hh = to_tf32(hv);
        p.h_hi[(size_t)b * p.I + R / 2] = hh;
        p.h_lo[(size_t)b * p.I + R / 2] = to_tf32(hv - hh);
      } else {  // DE_HEADS
        if (p.rows != nullptr && !row_wanted(p.rows + b, p.want)) continue;
        const int q0 = R / p.V, c0 = R % p.V;
        p.logits[((size_t)b * p.rows_per_item + q0) * p.V + c0] = __fmul_rn(v0, rinv);
        if (R + 1 < p.nrows) {
          const int q1 = (R + 1) / p.V, c1 = (R + 1) % p.V;
          p.logits[((size_t)b * p.rows_per_item + q1) * p.V + c1] = __fmul_rn(v1, rinv);
        }
      }
    }
  }
  if (CS > 1) cluster_sync_all();  // partial tiles stay alive until every rank has read them
}

// ---- one-time construction of the tensor-core weight copy (device side, from the fp32 blob)
// out[(perm(r)) * K + k] = W[r * K + k] * (scale ? scale[k] : 1)
//   mode 0: identity rows; mode 1: q/k heads -> RoPE pairs adjacent (row j -> 2j, row j+hd/2 -> 2j+1), v rows
//   unchanged; mode 2: [gate; up] -> interleaved (gate_n -> 2n, up_n -> 2n+1)
__global__ void k_build_tc_weight(const float* __restrict__ W, const float* __restrict__ scale, float* __restrict__ out,
                                  int rows, int K, int mode, int qk_rows, int hd, int I);
// the half-precision engine's copies of one layer matrix: v = W[r * K + k] * (scale ? scale[k] : 1) in fp32, then
// out16[perm(r) * K + k] = fp16_rne(v) (decode layout, as above) and out32[r * K + k] = fp16_rne(v) as fp32 (the
// blob's layout, for the prefill GEMMs); *bad = 1 if some |v| > 65504 (not representable in fp16)
__global__ void k_build_tc_weight16(const float* __restrict__ W, const float* __restrict__ scale, __half* __restrict__ out16,
                                    float* __restrict__ out32, int rows, int K, int mode, int qk_rows, int hd, int I,
                                    int* __restrict__ bad);

}  // namespace ctb
