// Kernels of hot path 2: DVAE decoder + Vocos + iSTFT  (reference ChatTTS/core.py:505-539,
// ChatTTS/model/dvae.py:14-66,87-97,131-172,276-297; vocos [3p]).
//
// Internal activation layout is TIME-MAJOR: [B*F rows, C channels], channel fastest.  With it
//   * every Conv1d(k, dilation) / Linear is one "NT" GEMM  C[m, n] = sum_kk A[m, kk] * W[n, kk]
//     whose A operand is gathered on the fly from shifted rows (kk = tap * Cin + c): no im2col;
//   * the frame-doubling reshape of dvae.py:281-287 applied to the decode loop's [B, T, 768]
//     hidden states is a pure re-interpretation ([B, 2T, 384]) - zero bytes moved;
//   * LayerNorm / depthwise conv read and write fully coalesced rows.
// The inverse STFT is a GEMM against a constant windowed inverse-DFT basis followed by an
// overlap-add/envelope kernel.  fp32 FMA throughout (waveform tolerance 1e-4 RMS).
#pragma once
#include "common.cuh"

namespace ctb {

enum GemmEpi { GE_NONE = 0, GE_BIAS = 1, GE_GELU = 2, GE_SCALE_RES = 3, GE_COEF = 4, GE_SPEC = 5 };

struct GemmP {
  const float* A; int lda;   // time-major activations
  int M, N, K;               // K = taps * Cin (multiple of 16)
  int taps, Cin, dil, pad, F;  // A[m, tap*Cin + c] = X[row of frame f + (tap - pad)*dil of the same utterance]
  const float* W;            // [N, K] row-major
  const float* bias;         // [N]
  const float* gamma;        // GE_SCALE_RES: layer scale; GE_COEF: per-channel coefficient
  const float* res; int ldres;
  float* C; int ldc;
  const int* fr;             // ragged mode: frames of each utterance (F = the widest); rows f >= fr[b] are written as 0
};

constexpr int GBM = 128, GBN = 128, GBK = 16;

__device__ __forceinline__ float gelu_erf(float x) {  // nn.GELU() default (exact erf form)
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}

template <int EPI, bool RAGGED = false>
__global__ void __launch_bounds__(256) k_sgemm_nt(const GemmP p) {
  __shared__ __align__(16) float As[2][GBK][GBM];
  __shared__ __align__(16) float Bs[2][GBK][GBN];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * GBM, n0 = blockIdx.x * GBN;
  // loader mapping: 2 float4 per operand per thread; row = tid/4 + 64*i, k quad = tid%4
  const int lrow = tid >> 2, lkq = (tid & 3) * 4;
  // compute mapping: 16x16 threads, each 2x2 blocks of 4x4 (rows ty*4 + {0,64}, cols tx*4 + {0,64})
  const int tx = tid & 15, ty = tid >> 4;

  int arow_b[2], arow_f[2];
  bool arow_ok[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = m0 + lrow + 64 * i;
    arow_ok[i] = m < p.M;
    const int mm = arow_ok[i] ? m : 0;
    arow_b[i] = mm / p.F; arow_f[i] = mm - arow_b[i] * p.F;
  }
  const int ntile = p.K / GBK;

  auto load_tile = [&](int t, float4 (&ra)[2], float4 (&rb)[2]) {
    const int k0 = t * GBK;
    const int tap = k0 / p.Cin, c0 = k0 - tap * p.Cin;
    const int shift = (tap - p.pad) * p.dil;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int f = arow_f[i] + shift;
      ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (arow_ok[i] && f >= 0 && f < p.F)
        ra[i] = *reinterpret_cast<const float4*>(p.A + ((size_t)arow_b[i] * p.F + f) * p.lda + c0 + lkq);
      const int n = n0 + lrow + 64 * i;
      rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (n < p.N) rb[i] = __ldg(reinterpret_cast<const float4*>(p.W + (size_t)n * p.K + k0 + lkq));
    }
  };
  auto store_tile = [&](int buf, const float4 (&ra)[2], const float4 (&rb)[2]) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = lrow + 64 * i;
      As[buf][lkq + 0][r] = ra[i].x; As[buf][lkq + 1][r] = ra[i].y;
      As[buf][lkq + 2][r] = ra[i].z; As[buf][lkq + 3][r] = ra[i].w;
      Bs[buf][lkq + 0][r] = rb[i].x; Bs[buf][lkq + 1][r] = rb[i].y;
      Bs[buf][lkq + 2][r] = rb[i].z; Bs[buf][lkq + 3][r] = rb[i].w;
    }
  };

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra[2], rb[2];
  load_tile(0, ra, rb);
  store_tile(0, ra, rb);
  __syncthreads();
  for (int t = 0; t < ntile; ++t) {
    const int buf = t & 1;
    if (t + 1 < ntile) load_tile(t + 1, ra, rb);
#pragma unroll
    for (int k = 0; k < GBK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4 + 64]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4 + 64]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (t + 1 < ntile) {
      store_tile(buf ^ 1, ra, rb);
      __syncthreads();
    }
  }

  // ---- epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + ty * 4 + (i & 3) + (i >> 2) * 64;
    if (m >= p.M) continue;
    bool pad_row = false;
    if (RAGGED) { const int b = m / p.F; pad_row = m - b * p.F >= p.fr[b]; }
#pragma unroll
    for (int jb = 0; jb < 2; ++jb) {
      const int n = n0 + tx * 4 + jb * 64;
      if (n >= p.N) continue;  // N is a multiple of 4 for every layer here
      if (RAGGED && pad_row) {
        *reinterpret_cast<float4*>(p.C + (size_t)m * p.ldc + n) = make_float4(0.f, 0.f, 0.f, 0.f);
        continue;
      }
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = acc[i][jb * 4 + j];
      if (EPI == GE_BIAS || EPI == GE_GELU || EPI == GE_SCALE_RES || EPI == GE_SPEC) {
        const float4 bb = __ldg(reinterpret_cast<const float4*>(p.bias + n));
        v[0] += bb.x; v[1] += bb.y; v[2] += bb.z; v[3] += bb.w;
      }
      if (EPI == GE_GELU) {
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = gelu_erf(v[j]);
      } else if (EPI == GE_SCALE_RES) {
        // ConvNeXt tail (dvae.py:59-63): y *= gamma ; x = y + residual
        const float4 g = __ldg(reinterpret_cast<const float4*>(p.gamma + n));
        const float4 r = *reinterpret_cast<const float4*>(p.res + (size_t)m * p.ldres + n);
        v[0] = __fadd_rn(__fmul_rn(v[0], g.x), r.x); v[1] = __fadd_rn(__fmul_rn(v[1], g.y), r.y);
        v[2] = __fadd_rn(__fmul_rn(v[2], g.z), r.z); v[3] = __fadd_rn(__fmul_rn(v[3], g.w), r.w);
      } else if (EPI == GE_COEF) {
        const float4 g = __ldg(reinterpret_cast<const float4*>(p.gamma + n));
        v[0] *= g.x; v[1] *= g.y; v[2] *= g.z; v[3] *= g.w;
      } else if (EPI == GE_SPEC) {
        // ISTFTHead: columns are interleaved (log-magnitude, phase) pairs.
        // mag = clip(exp(.), max=1e2); S = mag * (cos p + i sin p)   (exporter.py:395-404)
#pragma unroll
        for (int j = 0; j < 4; j += 2) {
          const float mag = fminf(expf(v[j]), 100.0f);
          float sn, cs;
          sincosf(v[j + 1], &sn, &cs);
          v[j] = mag * cs; v[j + 1] = mag * sn;
        }
      }
      *reinterpret_cast<float4*>(p.C + (size_t)m * p.ldc + n) = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
}

// Depthwise Conv1d(k = 7, dilation) + bias + LayerNorm(eps) over channels, time-major in/out.
// taps == 0: LayerNorm only.  One warp per frame row, C = 32 * 4 * NV channels.
struct DwLnP {
  const float* x; float* out;
  int M, F, C, taps, dil;
  const float* w;     // [taps][C]
  const float* b;     // [C]
  const float* lnw; const float* lnb;
  float eps;
  const int* fr;      // ragged mode: frames of each utterance; rows f >= fr[b] are written as 0
};

// RAGGED: the taps stop at the utterance's own last frame, exactly as for F = fr[b] (no fmaf with a padding zero)
template <int NV, bool RAGGED = false>
__global__ void __launch_bounds__(256) k_dwconv_ln(const DwLnP p) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= p.M) return;
  const int m = warp, b = m / p.F, f = m - b * p.F;
  const int Fb = RAGGED ? p.fr[b] : p.F;
  if (RAGGED && f >= Fb) {
#pragma unroll
    for (int i = 0; i < NV; ++i)
      *reinterpret_cast<float4*>(p.out + (size_t)m * p.C + (i * 32 + lane) * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  float4 v[NV];
  if (p.taps == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i)
      v[i] = *reinterpret_cast<const float4*>(p.x + (size_t)m * p.C + (i * 32 + lane) * 4);
  } else {
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = __ldg(reinterpret_cast<const float4*>(p.b + (i * 32 + lane) * 4));
    const int half = p.taps / 2;
    for (int t = 0; t < p.taps; ++t) {
      const int ff = f + (t - half) * p.dil;
      if (ff < 0 || ff >= Fb) continue;
      const float* xr = p.x + ((size_t)b * p.F + ff) * p.C;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = (i * 32 + lane) * 4;
        const float4 xv = *reinterpret_cast<const float4*>(xr + c);
        const float4 wv = __ldg(reinterpret_cast<const float4*>(p.w + (size_t)t * p.C + c));
        v[i].x = fmaf(wv.x, xv.x, v[i].x); v[i].y = fmaf(wv.y, xv.y, v[i].y);
        v[i].z = fmaf(wv.z, xv.z, v[i].z); v[i].w = fmaf(wv.w, xv.w, v[i].w);
      }
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) / (float)p.C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, bq = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += (a * a + bq * bq) + (c * c + d * d);
  }
  const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)p.C + p.eps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = (i * 32 + lane) * 4;
    const float4 g = __ldg(reinterpret_cast<const float4*>(p.lnw + c));
    const float4 bb = __ldg(reinterpret_cast<const float4*>(p.lnb + c));
    float4 o;
    o.x = (v[i].x - mean) * rstd * g.x + bb.x; o.y = (v[i].y - mean) * rstd * g.y + bb.y;
    o.z = (v[i].z - mean) * rstd * g.z + bb.z; o.w = (v[i].w - mean) * rstd * g.w + bb.w;
    *reinterpret_cast<float4*>(p.out + (size_t)m * p.C + c) = o;
  }
}

#ifdef CTB_DECODER_KERNELS_IMPL  // non-template kernels: defined once, in decoder_api.cu
// [B, Cin2, T] channels-first -> time-major [B, 2T, Cin2/2] with the frame-doubling of
// dvae.py:281-287 (channel c < C/2 -> even frame, c + C/2 -> odd frame).  Tiled transpose.
__global__ void k_cf_to_tm_doubled(const float* __restrict__ in, float* __restrict__ out, int B, int C2, int T) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, c0 = blockIdx.y * 32, t0 = blockIdx.x * 32;
  const int Ch = C2 / 2;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C2 && t < T) ? in[((size_t)b * C2 + c) * T + t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (c < C2 && t < T) {
      const int s = c / Ch, cc = c - s * Ch;
      out[((size_t)b * 2 * T + 2 * t + s) * Ch + cc] = tile[threadIdx.x][i];
    }
  }
}

// generic [B, C, F] channels-first <-> [B, F, ld] time-major (pad channels written as 0)
__global__ void k_cf_to_tm(const float* __restrict__ in, float* __restrict__ out, int B, int C, int F, int ld) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, c0 = blockIdx.y * 32, f0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, f = f0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && f < F) ? in[((size_t)b * C + c) * F + f] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int f = f0 + i, c = c0 + threadIdx.x;
    if (c < ld && f < F) out[((size_t)b * F + f) * ld + c] = tile[threadIdx.x][i];
  }
}
__global__ void k_tm_to_cf(const float* __restrict__ in, float* __restrict__ out, int B, int C, int F, int ld) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, c0 = blockIdx.y * 32, f0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int f = f0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && f < F) ? in[((size_t)b * F + f) * ld + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, f = f0 + threadIdx.x;
    if (c < C && f < F) out[((size_t)b * C + c) * F + f] = tile[threadIdx.x][i];
  }
}

// GFSQ._embed (dvae.py:87-97) + frame doubling: ids [B, G*R, T] -> time-major [B, 2T (= G frames per
// token when G == 2), dim/G].  code(i)_k = ((i / 5^k) % 5 - 2) / 2 ; z = sum_r base^-r * code ; Linear(4 -> dim/G).
struct GfsqP {
  const int32_t* ids; float* out;
  int B, T, G, R, levels, nlev, per_group;
  float scale_base;
  const float* w;   // [G][per_group][nlev]
  const float* b;   // [G][per_group]
};
__global__ void k_gfsq_dequant(const GfsqP p) {
  const int frame = blockIdx.x;  // b * T * G + t * G + g
  const int g = frame % p.G, t = (frame / p.G) % p.T, b = frame / (p.G * p.T);
  float z[8];
  for (int k = 0; k < p.nlev; ++k) z[k] = 0.f;
  float sc = 1.f;
  const float half = (float)(p.levels / 2);
  for (int r = 0; r < p.R; ++r) {
    int id = p.ids[((size_t)b * p.G * p.R + g * p.R + r) * p.T + t];
    for (int k = 0; k < p.nlev; ++k) {
      const int li = id % p.levels;
      id /= p.levels;
      z[k] += (((float)li - half) / half) * sc;
    }
    sc /= p.scale_base;
  }
  for (int c = threadIdx.x; c < p.per_group; c += blockDim.x) {
    const float* w = p.w + ((size_t)g * p.per_group + c) * p.nlev;
    float a = 0.f;
    for (int k = 0; k < p.nlev; ++k) a = fmaf(z[k], w[k], a);
    p.out[(size_t)frame * p.per_group + c] = a + p.b[g * p.per_group + c];
  }
}

// torch.istft tail: overlap-add of windowed frames, divide by the window-square envelope, trim
// n_fft/2 on both sides (center=True).  frames [B, F, n_fft] (already multiplied by the window
// through the DFT basis) -> wav [B, hop * (F - 1)].
// RAGGED: utterance b has fr[b] <= F frames (its envelope, trim and length follow them); wav is [B, wav_ld] and
// row b receives hop * (fr[b] - 1) samples.
template <bool RAGGED = false>
__global__ void k_overlap_add(const float* __restrict__ frames, const float* __restrict__ window,
                              float* __restrict__ wav, int B, int F, int n_fft, int hop, const int* __restrict__ fr = nullptr,
                              int64_t wav_ld = 0) {
  const int L = hop * (F - 1);
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * L) return;
  const int b = (int)(i / L), j = (int)(i - (size_t)b * L);
  const int Fb = RAGGED ? fr[b] : F;
  if (RAGGED && j >= hop * (Fb - 1)) return;
  const int pidx = j + n_fft / 2;
  const int f_hi = min(Fb - 1, pidx / hop);
  const int f_lo = pidx >= n_fft ? (pidx - n_fft) / hop + 1 : 0;
  float s = 0.f, env = 0.f;
  for (int f = f_lo; f <= f_hi; ++f) {
    const int n = pidx - f * hop;
    const float w = window[n];
    s += frames[((size_t)b * F + f) * n_fft + n];
    env = fmaf(w, w, env);
  }
  if (RAGGED)
    wav[(size_t)b * wav_ld + j] = s / env;
  else
    wav[i] = s / env;
}

// Ragged-mode inputs, staged time-major [B, 2W, idim] with rows f >= 2 n_b zero (W = the widest row's tokens).
// Hidden rows: token-major [n_b, 2 idim] fp32, whose frame doubling is a re-interpretation as [2 n_b, idim].
__global__ void k_gather_hidden_rows(const float* const* __restrict__ rows, const int* __restrict__ fr,
                                     float* __restrict__ out, int W, int idim) {
  const int b = blockIdx.y, f = blockIdx.x;
  float4* o = reinterpret_cast<float4*>(out + ((size_t)b * 2 * W + f) * idim);
  const bool in = f < fr[b];
  const float4* src = in ? reinterpret_cast<const float4*>(rows[b] + (size_t)f * idim) : nullptr;
  for (int c = threadIdx.x; c < idim / 4; c += blockDim.x) o[c] = in ? src[c] : make_float4(0.f, 0.f, 0.f, 0.f);
}

// GFSQ._embed of k_gfsq_dequant for ragged token-major codes: row b is [n_b, G*R] int32; frame (t, g) of row b goes to
// staged row b * 2W + t * G + g.  The arithmetic is k_gfsq_dequant's, term for term (that kernel is left as it is).
struct GfsqRowsP {
  const int32_t* const* rows; const int* fr; float* out;
  int W, G, R, levels, nlev, per_group;
  float scale_base;
  const float* w; const float* b;
};
__global__ void k_gfsq_dequant_rows(const GfsqRowsP p) {
  const int frame = blockIdx.x;  // t * G + g of row blockIdx.y
  const int b = blockIdx.y, g = frame % p.G, t = frame / p.G;
  float* out = p.out + ((size_t)b * 2 * p.W + frame) * p.per_group;
  if (frame >= p.fr[b]) {
    for (int c = threadIdx.x; c < p.per_group; c += blockDim.x) out[c] = 0.f;
    return;
  }
  float z[8];
  for (int k = 0; k < p.nlev; ++k) z[k] = 0.f;
  float sc = 1.f;
  const float half = (float)(p.levels / 2);
  const int32_t* ids = p.rows[b] + (size_t)t * p.G * p.R + g * p.R;
  for (int r = 0; r < p.R; ++r) {
    int id = ids[r];
    for (int k = 0; k < p.nlev; ++k) {
      const int li = id % p.levels;
      id /= p.levels;
      z[k] += (((float)li - half) / half) * sc;
    }
    sc /= p.scale_base;
  }
  for (int c = threadIdx.x; c < p.per_group; c += blockDim.x) {
    const float* w = p.w + ((size_t)g * p.per_group + c) * p.nlev;
    float a = 0.f;
    for (int k = 0; k < p.nlev; ++k) a = fmaf(z[k], w[k], a);
    out[c] = a + p.b[g * p.per_group + c];
  }
}

// ---------------------------------------------------------------- DVAE encode branch (dvae.py:175-206,265-274,102-128)
// torch.stft(center=True, pad_mode="reflect") framing: padded[i] = wav[reflect(i - n_fft/2)]; frame f = padded[f*hop .. +n_fft).
__global__ void k_reflect_pad(const float* __restrict__ wav, float* __restrict__ out, int64_t L, int64_t total, int half) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int64_t j = i - half;
  if (j < 0) j = -j;
  if (j >= L) j = 2 * (L - 1) - j;
  out[i] = (j >= 0 && j < L) ? wav[j] : 0.f;   // rows past the last frame are never read as a full window
}

// |STFT| (power = 1) of one frame per block row, evaluated as a direct DFT in DOUBLE precision: thread = frequency bin,
// x[n] * hann[n] (exact in double) times an exact-index twiddle table cos/sin(2 pi ((k n) mod N) / N).  The reference runs
// an fp32 FFT (torch.stft); a direct fp32 DFT would carry ~10x its rounding error, and the log that follows amplifies any
// error in the bins far below the frame's peak into the codes.  In double the result is the correctly rounded magnitude,
// i.e. at least as close to the exact value as the reference's own output.  Cost: 1 M DFMA per frame - negligible.
template <int NFFT>
__global__ void __launch_bounds__(256) k_stft_mag(const float* __restrict__ padded, const float* __restrict__ window, int hop,
                                                   int nbin, float* __restrict__ mag, int ldmag) {
  __shared__ double s_c[NFFT], s_s[NFFT], s_x[NFFT];
  const float* x = padded + (size_t)blockIdx.x * hop;
  for (int j = threadIdx.x; j < NFFT; j += 256) {
    double sn, cs;
    sincospi(2.0 * (double)j / (double)NFFT, &sn, &cs);
    s_c[j] = cs; s_s[j] = sn;
    s_x[j] = (double)x[j] * (double)window[j];
  }
  __syncthreads();
  const int k = blockIdx.y * 256 + threadIdx.x;
  if (k >= nbin) return;
  double re = 0.0, im = 0.0;
#pragma unroll 8
  for (int n = 0; n < NFFT; ++n) {
    const int j = (k * n) & (NFFT - 1);
    re = fma(s_x[n], s_c[j], re);
    im = fma(s_x[n], s_s[j], im);
  }
  mag[(size_t)blockIdx.x * ldmag + k] = (float)sqrt(re * re + im * im);
}

// mel filterbank -> log(clip(., 1e-5)) / coef  (dvae.py:199-206,267-268), one frame per block.  mag [F, ldmag];
// fb [nbin][MELP] (bin-major, mel padded with zero columns); out time-major [F, MELP], pad channels written as 0.
template <int MELP>
__global__ void __launch_bounds__(MELP) k_mel_log(const float* __restrict__ mag, int ldmag, int nbin,
                                                   const float* __restrict__ fb, const float* __restrict__ coef, int n_mels,
                                                   float* __restrict__ out) {
  extern __shared__ float s_mag[];
  const float* row = mag + (size_t)blockIdx.x * ldmag;
  for (int k = threadIdx.x; k < nbin; k += MELP) s_mag[k] = row[k];
  __syncthreads();
  const int m = threadIdx.x;
  float a = 0.f;
  for (int k = 0; k < nbin; ++k) a = fmaf(s_mag[k], fb[(size_t)k * MELP + m], a);
  out[(size_t)blockIdx.x * MELP + m] = m < n_mels ? logf(fmaxf(a, 1e-5f)) / coef[m] : 0.f;
}

// GFSQ.forward (dvae.py:102-128) -> GroupedResidualFSQ [3p]: per (frame, group) project_in Linear(dim/G -> nlev), then
// R residual FSQ stages: q = round(bound(res / s_r)), code = q / (levels / 2), res -= code * s_r, s_r = base^-r;
// index_r = sum_k (q_k + levels / 2) * levels^k.  x time-major [T, G * per_group]; ids [G * R, T] (c = g * R + r).
struct FsqQuantP {
  const float* x; int32_t* ids; float* margin;  // margin (optional) [G * R, T]: distance of the closest bound() to a rounding edge
  int T, G, R, levels, nlev, per_group;
  float scale_base; int bound_input;
  const float* w;   // [G][nlev][per_group]
  const float* b;   // [G][nlev]
  // ragged mode (ctb_dvae_encode_rows): row b's x is [F rows, G * per_group] at x + b * F * G * per_group, its ids and
  // margins [G * R, T] (T = the row stride) at + b * G * R * T; only its first tn[b] tokens are quantised
  const int* tn; int F;
};
__device__ __forceinline__ float fsq_bound(float z, int levels) {
  const float half_l = (float)(levels - 1) * (1.0f + 1e-3f) * 0.5f;
  const float offset = (levels & 1) ? 0.0f : 0.5f;
  const float shift = atanhf(offset / half_l);
  return tanhf(z + shift) * half_l - offset;
}
// RAGGED: grid (F * G, B); blocks past a row's tn[b] tokens return at once.  A token's arithmetic is the lone kernel's.
template <bool RAGGED = false>
__global__ void __launch_bounds__(128) k_fsq_quant(const FsqQuantP p) {
  const int t = blockIdx.x / p.G, g = blockIdx.x % p.G;
  size_t xoff = 0, ioff = 0;
  if (RAGGED) {
    if (t >= p.tn[blockIdx.y]) return;
    xoff = (size_t)blockIdx.y * p.F * p.G * p.per_group;
    ioff = (size_t)blockIdx.y * p.G * p.R * p.T;
  }
  const float* x = p.x + xoff + ((size_t)t * p.G + g) * p.per_group;
  __shared__ float s_part[4][8];
  float acc[8];
  for (int k = 0; k < p.nlev; ++k) acc[k] = 0.f;
  for (int c = threadIdx.x; c < p.per_group; c += 128) {
    const float xv = x[c];
    for (int k = 0; k < p.nlev; ++k) acc[k] = fmaf(xv, p.w[((size_t)g * p.nlev + k) * p.per_group + c], acc[k]);
  }
  for (int k = 0; k < p.nlev; ++k) {
    float v = acc[k];
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5][k] = v;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  float res[8];
  for (int k = 0; k < p.nlev; ++k) {
    const float z = ((s_part[0][k] + s_part[1][k]) + (s_part[2][k] + s_part[3][k])) + p.b[g * p.nlev + k];
    res[k] = p.bound_input ? fsq_bound(z, p.levels) : z;
  }
  const float half_w = (float)(p.levels / 2);
  float sc = 1.f;
  for (int r = 0; r < p.R; ++r) {
    int idx = 0, mul = 1;
    float mg = 1.f;
    for (int k = 0; k < p.nlev; ++k) {
      const float bz = fsq_bound(res[k] / sc, p.levels);
      const float q = rintf(bz);                       // torch.round: half to even
      mg = fminf(mg, 0.5f - fabsf(bz - q));
      res[k] -= (q / half_w) * sc;
      idx += ((int)q + p.levels / 2) * mul;
      mul *= p.levels;
    }
    p.ids[ioff + ((size_t)g * p.R + r) * p.T + t] = idx;
    if (p.margin) p.margin[ioff + ((size_t)g * p.R + r) * p.T + t] = mg;
    sc /= p.scale_base;
  }
}

#endif  // CTB_DECODER_KERNELS_IMPL

}  // namespace ctb
