// wgmma / TMA GEMM with fp32-equivalent accuracy (3xTF32) for the dense contractions of
// hot path 2 (and prefill):   C[m, n] = epi( sum_kk A[m, kk] * W[n, kk] )
//
//   * A: time-major activations [B][F][lda] fp32, read by a 3-D TMA tensor map (c, f, b).  A Conv1d tap
//     is a shift of the f coordinate; frames outside [0, F) are zero-filled by TMA = the conv's zero
//     padding, per utterance - no im2col, no boundary code.
//   * W: [N][K] fp32, pre-split on the host into tf32-rounded `hi` and `lo = tf32(w - hi)` copies (weights
//     are constants), two 2-D TMA maps.
//   * 3xTF32:  A*W ~= A_hi*W_hi + A_hi*W_lo + A_lo*W_hi, accumulated in fp32 registers.  A is split in shared
//     memory by the warpgroup that consumes it (cvt.rna.tf32).
//   * warp roles: warpgroups 0-1 consume (each splits and multiplies 64 of the tile's 128 rows with
//     wgmma.m64n128k8.tf32, then runs the epilogue from its registers), warp 8 = TMA producer.
//   * tile 128 (frames of one utterance) x 128 (channels) x 32 (k) per stage, 3 stages of 64 KiB:
//     [A | A_lo | W_hi | W_lo], 128-byte swizzle (TMA and wgmma descriptors agree).
//   * persistent: a CTA walks tiles (n fastest, so concurrent CTAs share A rows in L2); the producer runs ahead into
//     the next tile's stages while the consumers run the epilogue of the current one.
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>

#include "decoder_kernels.cuh"
#include "tc_common.cuh"

namespace ctb {

constexpr int TC_BM = 128, TC_BN = 128, TC_BK = 32, TC_STAGES = 3;
constexpr int TC_TILE_BYTES = TC_BM * TC_BK * 4;          // 16 KiB
constexpr int TC_STAGE_BYTES = 4 * TC_TILE_BYTES;         // A, A_lo, W_hi, W_lo
constexpr int TC_SMEM_BYTES = TC_STAGES * TC_STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
constexpr int TC_CONSUMERS = 256;                         // two warpgroups
constexpr int TC_THREADS = TC_CONSUMERS + 32;             // + the TMA warp

struct TcGemmP {
  int N, K;                   // K = taps * Cin, multiple of 32
  int taps, Cin, dil, pad, F, B;
  const float* bias; const float* gamma;
  const float* res; int ldres;
  float* C; int ldc;
  const int* fr;              // ragged mode: frames of each utterance (F = the widest); rows f >= fr[b] are written as 0
};


// Epilogue of two adjacent output columns (n even) of one output row m.
template <int EPI>
__device__ __forceinline__ void tc_epi_store2(const TcGemmP& p, float v0, float v1, size_t m, int n) {
  if (EPI == GE_BIAS || EPI == GE_GELU || EPI == GE_SCALE_RES || EPI == GE_SPEC) {
    const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + n));
    v0 += bb.x; v1 += bb.y;
  }
  if (EPI == GE_GELU) {
    v0 = gelu_erf(v0); v1 = gelu_erf(v1);
  } else if (EPI == GE_SCALE_RES) {
    const float2 g = __ldg(reinterpret_cast<const float2*>(p.gamma + n));
    const float2 rr = *reinterpret_cast<const float2*>(p.res + m * p.ldres + n);
    v0 = __fadd_rn(__fmul_rn(v0, g.x), rr.x); v1 = __fadd_rn(__fmul_rn(v1, g.y), rr.y);
  } else if (EPI == GE_COEF) {
    const float2 g = __ldg(reinterpret_cast<const float2*>(p.gamma + n));
    v0 *= g.x; v1 *= g.y;
  } else if (EPI == GE_SPEC) {  // columns (2j, 2j+1) = (log-magnitude, phase) of one bin
    const float mag = fminf(expf(v0), 100.0f);
    float sn, cs;
    sincosf(v1, &sn, &cs);
    v0 = mag * cs; v1 = mag * sn;
  }
  *reinterpret_cast<float2*>(p.C + m * p.ldc + n) = make_float2(v0, v1);
}

__device__ __forceinline__ void mbar_wait_or_trap(uint64_t* bar, uint32_t parity) {
  for (uint32_t spin = 0; !mbar_try_wait(bar, parity); ++spin)
    if (spin > (1u << 28)) __trap();   // a protocol bug must end the kernel, not hang the GPU
}

// RAGGED: the utterances have fr[b] <= F frames each.  Rows past an utterance's end are written as exact zeros, so a
// later tapped layer reads there what TMA's out-of-bounds fill gives an utterance decoded alone, and every output row
// of the utterance is bit-identical to that decode (same tile origin, same operands, same k order).
template <int EPI, bool RAGGED = false>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_tc_gemm(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_whi,
          const __grid_constant__ CUtensorMap map_wlo, const TcGemmP p) {
  extern __shared__ uint8_t tc_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TC_STAGES * TC_STAGE_BYTES);
  uint64_t* full = bars;                  // [stages]  TMA bytes landed
  uint64_t* empty = bars + TC_STAGES;     // [stages]  both warpgroups' MMAs of the stage retired

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_per_utt = (p.F + TC_BM - 1) / TC_BM;
  const int n_tiles = (p.N + TC_BN - 1) / TC_BN;
  const int total = n_tiles * tiles_per_utt * p.B;
  const int nk = p.K / TC_BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < TC_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], TC_CONSUMERS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == TC_CONSUMERS / 32) {
    // ===================== TMA producer
    if (lane == 0) {
      int g = 0;
      for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int nt = tile % n_tiles, mt = tile / n_tiles;
        const int b = mt / tiles_per_utt, f0 = (mt % tiles_per_utt) * TC_BM, n0 = nt * TC_BN;
        for (int t = 0; t < nk; ++t, ++g) {
          const int s = g % TC_STAGES, it = g / TC_STAGES;
          if (it > 0) mbar_wait_or_trap(&empty[s], (it - 1) & 1);
          uint8_t* st = smem + s * TC_STAGE_BYTES;
          const int k0 = t * TC_BK;
          const int tap = k0 / p.Cin, c0 = k0 - tap * p.Cin;
          mbar_expect_tx(&full[s], 3 * TC_TILE_BYTES);
          tma_load_3d(st, &map_a, &full[s], c0, f0 + (tap - p.pad) * p.dil, b);
          tma_load_2d(st + 2 * TC_TILE_BYTES, &map_whi, &full[s], k0, n0);
          tma_load_2d(st + 3 * TC_TILE_BYTES, &map_wlo, &full[s], k0, n0);
        }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64)
  const int wg = warp >> 2, tid = threadIdx.x & 127;
  const uint32_t half_off = wg * (TC_TILE_BYTES / 2);   // 64 rows x 128 B: whole 1024-byte swizzle atoms
  int g = 0;
  for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
    const int nt = tile % n_tiles, mt = tile / n_tiles;
    const int b = mt / tiles_per_utt, f0 = (mt % tiles_per_utt) * TC_BM, n0 = nt * TC_BN;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    int prev = 0;
    for (int t = 0; t < nk; ++t, ++g) {
      const int s = g % TC_STAGES, it = g / TC_STAGES;
      mbar_wait_or_trap(&full[s], it & 1);
      uint8_t* st = smem + s * TC_STAGE_BYTES;
      float4* a = reinterpret_cast<float4*>(st + half_off);
      float4* lo = reinterpret_cast<float4*>(st + TC_TILE_BYTES + half_off);
#pragma unroll
      for (int j = 0; j < TC_TILE_BYTES / 2 / 16 / 128; ++j) {
        const int e = tid + 128 * j;  // elementwise: the swizzle pattern is the same in both tiles
        const float4 v = a[e];
        float4 h, l;
        h.x = to_tf32(v.x); h.y = to_tf32(v.y); h.z = to_tf32(v.z); h.w = to_tf32(v.w);
        l.x = to_tf32(v.x - h.x); l.y = to_tf32(v.y - h.y); l.z = to_tf32(v.z - h.z); l.w = to_tf32(v.w - h.w);
        a[e] = h; lo[e] = l;
      }
      fence_async_smem();  // generic-proxy writes -> visible to the tensor core (async proxy)
      warpgroup_bar(2 + wg);
      const uint32_t su = smem_u32(st);
      const uint32_t a_hi = su + half_off, a_lo = su + TC_TILE_BYTES + half_off;
      const uint32_t w_hi = su + 2 * TC_TILE_BYTES, w_lo = su + 3 * TC_TILE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 8; ++k) {
        const uint32_t ko = k * 32;  // 8 tf32 = 32 bytes inside the 128-byte swizzle row
        wgmma_tf32_n128(acc, wgmma_desc_sw128(a_hi + ko), wgmma_desc_sw128(w_hi + ko), (t | k) ? 1u : 0u);
        wgmma_tf32_n128(acc, wgmma_desc_sw128(a_hi + ko), wgmma_desc_sw128(w_lo + ko), 1u);
        wgmma_tf32_n128(acc, wgmma_desc_sw128(a_lo + ko), wgmma_desc_sw128(w_hi + ko), 1u);
      }
      wgmma_commit();
      if (t > 0) {  // the previous stage's MMAs have retired: hand it back to the producer
        wgmma_wait<1>();
        mbar_arrive(&empty[prev]);
      }
      prev = s;
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    mbar_arrive(&empty[prev]);
    // epilogue straight from the accumulator registers (layout: see wgmma_tf32_n*)
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int f = f0 + r0 + 8 * h;
      if (f >= p.F) continue;
      const size_t m = (size_t)b * p.F + f;
      if (RAGGED && f >= p.fr[b]) {
#pragma unroll
        for (int j = 0; j < TC_BN / 8; ++j) {
          const int n = n0 + 8 * j + 2 * (lane & 3);
          if (n < p.N) *reinterpret_cast<float2*>(p.C + m * p.ldc + n) = make_float2(0.f, 0.f);
        }
        continue;
      }
#pragma unroll
      for (int j = 0; j < TC_BN / 8; ++j) {
        const int n = n0 + 8 * j + 2 * (lane & 3);
        if (n < p.N) tc_epi_store2<EPI>(p, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], m, n);
      }
    }
  }
}

// ---------------------------------------------------------------- host launcher (shared by both C APIs)
inline int tc_make_map(CUtensorMap* m, const float* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                       const cuuint32_t* box) {
  static PFN_cuTensorMapEncodeTiled_v12000 enc = nullptr;
  if (!enc) {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return set_err(CTB_ERR_CUDA, "cuTensorMapEncodeTiled unavailable");
    enc = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fp);
  }
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<float*>(base), dims, strides_bytes, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_err(CTB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return CTB_OK;
}

// C[B*F rows, N] = epi(A (x) W^T): A time-major [B][F][lda], W given as tf32 hi / lo copies [N][K].
// fr (device [B], ragged mode): frames of each utterance, see k_tc_gemm.
template <int EPI, bool RAGGED = false>
inline int tc_gemm_launch(cudaStream_t s, const float* A, int lda, int B, int F, int N, int K, int taps, int Cin, int dil,
                          int pad, const float* W_hi, const float* W_lo, const float* bias, const float* gamma,
                          const float* res, int ldres, float* C, int ldc, const int* fr = nullptr) {
  // CTB_TC_NONPERSISTENT=1: one tile per CTA, the schedule the persistent one is cross-checked against
  const bool persistent = getenv("CTB_TC_NONPERSISTENT") == nullptr;
  { int arc = ensure_smem_attr((const void*)k_tc_gemm<EPI, RAGGED>, TC_SMEM_BYTES); if (arc) return arc; }
  CUtensorMap ma, mh, ml;
  const cuuint64_t adims[3] = {(cuuint64_t)lda, (cuuint64_t)F, (cuuint64_t)B};
  const cuuint64_t astr[2] = {(cuuint64_t)lda * 4, (cuuint64_t)F * lda * 4};
  const cuuint32_t abox[3] = {TC_BK, TC_BM, 1};
  const cuuint64_t wdims[2] = {(cuuint64_t)K, (cuuint64_t)N};
  const cuuint64_t wstr[1] = {(cuuint64_t)K * 4};
  const cuuint32_t wbox[2] = {TC_BK, TC_BN};
  int rc;
  if ((rc = tc_make_map(&ma, A, 3, adims, astr, abox))) return rc;
  if ((rc = tc_make_map(&mh, W_hi, 2, wdims, wstr, wbox))) return rc;
  if ((rc = tc_make_map(&ml, W_lo, 2, wdims, wstr, wbox))) return rc;
  TcGemmP p{};
  p.N = N; p.K = K; p.taps = taps; p.Cin = Cin; p.dil = dil; p.pad = pad; p.F = F; p.B = B;
  p.bias = bias; p.gamma = gamma; p.res = res; p.ldres = ldres; p.C = C; p.ldc = ldc; p.fr = fr;
  static int sms = 0;
  if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
  const int total = ((N + TC_BN - 1) / TC_BN) * B * ((F + TC_BM - 1) / TC_BM);
  k_tc_gemm<EPI, RAGGED><<<persistent ? std::min(total, sms) : total, TC_THREADS, TC_SMEM_BYTES, s>>>(ma, mh, ml, p);
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

// tf32 hi / lo split of a weight buffer (device side, once at load)
template <int DUMMY = 0>
__global__ void k_split_tf32_t(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float x = w[i], h = to_tf32(x);
    hi[i] = h;
    lo[i] = to_tf32(x - h);
  }
}

}  // namespace ctb
