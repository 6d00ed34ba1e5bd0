// extern "C" entry points for hot path 2 (token -> waveform); see include/chattts_b200.h.
#define CTB_DECODER_KERNELS_IMPL
#include <vector>

#include "tc_gemm.cuh"

using namespace ctb;

__global__ void k_split_tf32(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, int64_t n);

namespace {

struct BlockOff {  // one ConvNeXt block inside a blob (float offsets)
  int64_t dw_w, dw_b, ln_w, ln_b, pw1_w, pw1_b, pw2_w, pw2_b, gamma;
};

struct DvaeOff {
  int64_t in0_w, in0_b, in2_w, in2_b, conv_out_w, out_conv_w, coef, vq_w, vq_b, total;
  BlockOff blk[64];
};
struct VocosOff {
  int64_t embed_w, embed_b, norm_w, norm_b, fin_w, fin_b, head_w, head_b, basis, window, total;
  BlockOff blk[64];
};

constexpr int MEL = 100, MEL_PAD = 128;

int64_t take(int64_t& off, int64_t n) { const int64_t o = off; off += (n + 3) / 4 * 4; return o; }

void block_layout(BlockOff& b, int64_t& off, int C, int inter) {
  b.dw_w = take(off, 7LL * C); b.dw_b = take(off, C); b.ln_w = take(off, C); b.ln_b = take(off, C);
  b.pw1_w = take(off, (int64_t)inter * C); b.pw1_b = take(off, inter);
  b.pw2_w = take(off, (int64_t)C * inter); b.pw2_b = take(off, C); b.gamma = take(off, C);
}

// Blob order (all fp32, every tensor padded to a multiple of 4 floats); the Python packer in
// chattts_b200/decoder.py writes the same sequence and checks the total against these functions.
DvaeOff dvae_layout(const ctb_convstack_config& c) {
  DvaeOff o{};
  int64_t off = 0;
  o.in0_w = take(off, (int64_t)c.bn_dim * 3 * c.idim);       // [bn, 3*idim]  tap-major K
  o.in0_b = take(off, c.bn_dim);
  o.in2_w = take(off, (int64_t)c.hidden * 3 * c.bn_dim);     // [hidden, 3*bn]
  o.in2_b = take(off, c.hidden);
  for (int i = 0; i < c.n_layer; ++i) block_layout(o.blk[i], off, c.hidden, 4 * c.hidden);
  o.conv_out_w = take(off, (int64_t)c.odim * c.hidden);      // [odim, hidden]
  o.out_conv_w = take(off, (int64_t)MEL_PAD * 3 * c.out_dim); // [128 (100 + zero rows), 3*out_dim]
  o.coef = take(off, MEL_PAD);
  if (c.vq_dim > 0) {
    const int per_group = c.vq_dim / c.vq_groups;
    o.vq_w = take(off, (int64_t)c.vq_groups * per_group * 4); // [G][dim/G][4]
    o.vq_b = take(off, (int64_t)c.vq_groups * per_group);
  }
  o.total = off;
  return o;
}

int spec_k(const ctb_vocos_config& c) { return ((c.n_fft + 2) + 31) / 32 * 32; }  // 1026 -> 1056

VocosOff vocos_layout(const ctb_vocos_config& c) {
  VocosOff o{};
  int64_t off = 0;
  o.embed_w = take(off, (int64_t)c.dim * 7 * MEL_PAD);       // [dim, 7*128] (mel channels padded)
  o.embed_b = take(off, c.dim);
  o.norm_w = take(off, c.dim); o.norm_b = take(off, c.dim);
  for (int i = 0; i < c.num_layers; ++i) block_layout(o.blk[i], off, c.dim, c.intermediate_dim);
  o.fin_w = take(off, c.dim); o.fin_b = take(off, c.dim);
  o.head_w = take(off, (int64_t)spec_k(c) * c.dim);          // rows interleaved (mag_k, phase_k), zero pad rows
  o.head_b = take(off, spec_k(c));
  o.basis = take(off, (int64_t)c.n_fft * spec_k(c));         // [n_fft, spec_k] windowed inverse real DFT
  o.window = take(off, c.n_fft);
  o.total = off;
  return o;
}

}  // namespace

struct ctb_decoder {
  ctb_convstack_config dc;
  ctb_vocos_config vc;
  DvaeOff dl;
  VocosOff vl;
  const float* dW;
  const float* vW;
  int max_batch, max_tokens;
  size_t max_rows;  // max_batch * 2 * max_tokens frames
  size_t cap_rows;  // frames the activation buffers currently hold
  float *bufA, *bufB, *bufH, *mel_tm, *staged_in;
  void* rows_meta;      // ctb_decode_rows: [B] row pointers + [B] frame counts, grown with B
  int rows_meta_cap;
  // tensor-core path: tf32-rounded hi / lo copies of both blobs (same offsets as the fp32 blobs)
  float *dW_hi, *dW_lo, *vW_hi, *vW_lo;
  bool use_tc;
};

extern "C" int64_t ctb_dvae_blob_floats(const ctb_convstack_config* c) { return c ? dvae_layout(*c).total : -1; }
extern "C" int64_t ctb_vocos_blob_floats(const ctb_vocos_config* c) { return c ? vocos_layout(*c).total : -1; }

extern "C" int ctb_decoder_destroy(ctb_decoder* h) {
  if (!h) return CTB_OK;
  void* ptrs[] = {h->bufA, h->bufB, h->bufH, h->mel_tm, h->staged_in, h->dW_hi, h->dW_lo, h->vW_hi, h->vW_lo,
                  h->rows_meta};
  for (void* p : ptrs) if (p) cudaFree(p);
  delete h;
  return CTB_OK;
}

// grow the activation buffers to `rows` frames (time-major [rows, C]); the contents are scratch
static int dec_reserve(ctb_decoder* h, size_t rows, cudaStream_t s) {
  if (rows <= h->cap_rows) return CTB_OK;
  CTB_CUDA(cudaStreamSynchronize(s));
  float** bufs[] = {&h->bufA, &h->bufB, &h->bufH, &h->mel_tm, &h->staged_in};
  for (float** b : bufs) if (*b) { cudaFree(*b); *b = nullptr; }
  h->cap_rows = 0;
  const ctb_convstack_config& dc = h->dc;
  const ctb_vocos_config& vc = h->vc;
  const size_t R = std::min(h->max_rows, rows + rows / 8);
  const size_t wide = std::max((size_t)std::max(4 * dc.hidden, vc.intermediate_dim), (size_t)vc.n_fft);
  const size_t narrow = std::max((size_t)std::max(std::max(dc.hidden, dc.idim), vc.dim), (size_t)dc.odim);
  cudaError_t e = cudaSuccess;
  auto A = [&](float** p, size_t n) { if (e == cudaSuccess) e = cudaMalloc((void**)p, n * sizeof(float)); };
  A(&h->bufA, R * std::max(narrow, (size_t)spec_k(vc)));
  A(&h->bufB, R * narrow);
  A(&h->bufH, R * wide);
  A(&h->mel_tm, R * MEL_PAD);
  A(&h->staged_in, R * dc.idim);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return set_err(CTB_ERR_NOMEM, "decoder buffers for %zu frames: %s", R, cudaGetErrorString(e));
  }
  h->cap_rows = R;
  return CTB_OK;
}

extern "C" int ctb_decoder_create(const ctb_convstack_config* dc, const float* dvae_blob_dev,
                                  const ctb_vocos_config* vc, const float* vocos_blob_dev, int32_t max_batch,
                                  int32_t max_tokens, ctb_decoder** out) {
  // either blob may be NULL: the handle then serves only the other half (DVAE-only / Vocos-only)
  if (!dc || !vc || (!dvae_blob_dev && !vocos_blob_dev) || !out) return set_err(CTB_ERR_ARG, "null argument");
  if (dc->kernel != 7 || dc->n_layer > 64 || vc->num_layers > 64) return set_err(CTB_ERR_ARG, "unsupported conv stack");
  if (dc->idim % 16 || dc->bn_dim % 16 || dc->hidden % 128 || dc->hidden > 512 || dc->odim % 16 || dc->out_dim % 16)
    return set_err(CTB_ERR_ARG, "dvae channel counts must be multiples of 16 (hidden: of 128, <= 512)");
  if (vc->input_channels != MEL || vc->dim % 128 || vc->dim > 512 || vc->intermediate_dim % 16 || vc->n_fft % 16 ||
      vc->hop_length * 4 != vc->n_fft)
    return set_err(CTB_ERR_ARG, "unsupported vocos shape");
  if (dc->vq_dim > 0 && (dc->vq_levels < 2 || dc->vq_dim % dc->vq_groups || dc->vq_dim / dc->vq_groups != dc->idim))
    return set_err(CTB_ERR_ARG, "vq_dim / vq_groups must equal the stack's idim");
  int ndev = 0;
  CTB_CUDA(cudaGetDeviceCount(&ndev));
  if (ndev < 1) return set_err(CTB_ERR_CUDA, "no CUDA device: chattts_b200 has no CPU path");
  ctb_decoder* h = new ctb_decoder();
  memset(h, 0, sizeof(*h));
  h->dc = *dc; h->vc = *vc; h->dl = dvae_layout(*dc); h->vl = vocos_layout(*vc);
  h->dW = dvae_blob_dev; h->vW = vocos_blob_dev;
  h->max_batch = max_batch; h->max_tokens = max_tokens;
  h->max_rows = (size_t)max_batch * 2 * max_tokens;
  cudaError_t e = cudaSuccess;
  auto A = [&](float** p, size_t n) { if (e == cudaSuccess) e = cudaMalloc((void**)p, n * sizeof(float)); };
  // activation buffers are sized by the largest call seen so far (dec_reserve), not by max_batch x max_tokens
  h->use_tc = getenv("CTB_DECODER_FMA") == nullptr;
  if (h->use_tc) {
    if (h->dW) { A(&h->dW_hi, h->dl.total); A(&h->dW_lo, h->dl.total); }
    if (h->vW) { A(&h->vW_hi, h->vl.total); A(&h->vW_lo, h->vl.total); }
  }
  if (e != cudaSuccess) {
    ctb_decoder_destroy(h);
    return set_err(CTB_ERR_NOMEM, "decoder buffers: %s", cudaGetErrorString(e));
  }
  if (h->use_tc) {
    if (h->dW) k_split_tf32<<<1024, 256>>>(h->dW, h->dW_hi, h->dW_lo, h->dl.total);
    if (h->vW) k_split_tf32<<<1024, 256>>>(h->vW, h->vW_hi, h->vW_lo, h->vl.total);
    CTB_CUDA(cudaDeviceSynchronize());
  }
  *out = h;
  return CTB_OK;
}

// ------------------------------------------------------------------ launch helpers
__global__ void k_split_tf32(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float x = w[i], h = to_tf32(x);
    hi[i] = h;
    lo[i] = to_tf32(x - h);
  }
}

struct GemmCtx {  // which blob a weight pointer lives in, for the hi / lo lookup of the tensor-core path
  const float* W; const float* hi; const float* lo; bool tc;
};

// fr (device [M / F], or null): ragged mode, the utterances have fr[b] <= F frames each and every layer writes zeros
// in the rows past them (see k_tc_gemm)
template <int EPI>
static int gemm(cudaStream_t s, const GemmCtx& gc, const float* A, int lda, int M, int N, int K, int taps, int Cin,
                int dil, int pad, int F, const float* W, const float* bias, const float* gamma, const float* res,
                int ldres, float* C, int ldc, const int* fr = nullptr) {
  if (gc.tc && K % TC_BK == 0 && Cin % TC_BK == 0 && M % F == 0) {
    if (fr)
      return tc_gemm_launch<EPI, true>(s, A, lda, M / F, F, N, K, taps, Cin, dil, pad, gc.hi + (W - gc.W),
                                       gc.lo + (W - gc.W), bias, gamma, res, ldres, C, ldc, fr);
    return tc_gemm_launch<EPI>(s, A, lda, M / F, F, N, K, taps, Cin, dil, pad, gc.hi + (W - gc.W), gc.lo + (W - gc.W), bias,
                               gamma, res, ldres, C, ldc);
  }
  GemmP p{};
  p.A = A; p.lda = lda; p.M = M; p.N = N; p.K = K; p.taps = taps; p.Cin = Cin; p.dil = dil; p.pad = pad; p.F = F;
  p.W = W; p.bias = bias; p.gamma = gamma; p.res = res; p.ldres = ldres; p.C = C; p.ldc = ldc; p.fr = fr;
  dim3 grid((N + GBN - 1) / GBN, (M + GBM - 1) / GBM);
  if (fr)
    k_sgemm_nt<EPI, true><<<grid, 256, 0, s>>>(p);
  else
    k_sgemm_nt<EPI><<<grid, 256, 0, s>>>(p);
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

template <bool RAGGED>
static void dwln_launch(cudaStream_t s, const DwLnP& p, int blocks) {
  switch (p.C / 128) {
    case 1: k_dwconv_ln<1, RAGGED><<<blocks, 256, 0, s>>>(p); break;
    case 2: k_dwconv_ln<2, RAGGED><<<blocks, 256, 0, s>>>(p); break;
    case 3: k_dwconv_ln<3, RAGGED><<<blocks, 256, 0, s>>>(p); break;
    default: k_dwconv_ln<4, RAGGED><<<blocks, 256, 0, s>>>(p); break;
  }
}

static int dwln(cudaStream_t s, const float* x, float* out, int M, int F, int C, int taps, int dil, const float* w,
                const float* b, const float* lnw, const float* lnb, const int* fr = nullptr) {
  DwLnP p{x, out, M, F, C, taps, dil, w, b, lnw, lnb, 1e-6f, fr};
  const int blocks = (M + 7) / 8;
  if (fr)
    dwln_launch<true>(s, p, blocks);
  else
    dwln_launch<false>(s, p, blocks);
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

// x (time-major [M, C]) -> x through one ConvNeXt block; tmp = [M, C], hbuf = [M, inter]
static int convnext(cudaStream_t s, const GemmCtx& gc, const float* W, const BlockOff& b, float* x, float* tmp, float* hbuf, int M,
                    int F, int C, int inter, int dil, const int* fr = nullptr) {
  int rc;
  if ((rc = dwln(s, x, tmp, M, F, C, 7, dil, W + b.dw_w, W + b.dw_b, W + b.ln_w, W + b.ln_b, fr))) return rc;
  if ((rc = gemm<GE_GELU>(s, gc, tmp, C, M, inter, C, 1, C, 1, 0, F, W + b.pw1_w, W + b.pw1_b, nullptr, nullptr, 0, hbuf,
                          inter, fr))) return rc;
  return gemm<GE_SCALE_RES>(s, gc, hbuf, inter, M, C, inter, 1, inter, 1, 0, F, W + b.pw2_w, W + b.pw2_b, W + b.gamma, x,
                            C, x, C, fr);
}

// in_layout: 0 = channels-first [B, C, T] fp32 (DVAE.__call__ layout), 1 = token-major [B, T, C] fp32
// (the decode loop's hidden states; frame doubling is then a re-interpretation), 2 = codes [B, G*R, T] int32.
// fr: ragged mode (ctb_decode_rows), layout 1 with rows past each utterance's fr[b] frames zero.
static int dvae_run(ctb_decoder* h, const void* in, int layout, int B, int T, float* mel_cf, cudaStream_t s,
                    const int* fr = nullptr) {
  const ctb_convstack_config& c = h->dc;
  const DvaeOff& L = h->dl;
  const float* W = h->dW;
  const int F = 2 * T, M = B * F;
  const GemmCtx gc{h->dW, h->dW_hi, h->dW_lo, h->use_tc};
  int rc;
  const float* x0;
  if (layout == 1) {
    x0 = static_cast<const float*>(in);
  } else if (layout == 0) {
    dim3 g((T + 31) / 32, (2 * c.idim + 31) / 32, B);
    k_cf_to_tm_doubled<<<g, dim3(32, 8), 0, s>>>(static_cast<const float*>(in), h->staged_in, B, 2 * c.idim, T);
    CTB_LAUNCH_CHECK();
    x0 = h->staged_in;
  } else {
    if (c.vq_dim <= 0) return set_err(CTB_ERR_ARG, "this decoder has no VQ layer (use_decoder=True model)");
    if (c.vq_groups != 2) return set_err(CTB_ERR_ARG, "vq_groups must be 2 (one group per doubled frame)");
    GfsqP g{};
    g.ids = static_cast<const int32_t*>(in); g.out = h->staged_in; g.B = B; g.T = T; g.G = c.vq_groups;
    g.R = c.vq_residual; g.levels = c.vq_levels & 0xff; g.nlev = 4; g.per_group = c.vq_dim / c.vq_groups;
    g.scale_base = (float)(((c.vq_levels >> 8) & 0xff) ? ((c.vq_levels >> 8) & 0xff) : (g.levels - 1));
    g.w = W + L.vq_w; g.b = W + L.vq_b;
    k_gfsq_dequant<<<B * T * c.vq_groups, 128, 0, s>>>(g);
    CTB_LAUNCH_CHECK();
    x0 = h->staged_in;
  }
  // conv_in: Conv1d(idim -> bn, k3, p1) + GELU + Conv1d(bn -> hidden, k3, p1)   (dvae.py:144-148)
  if ((rc = gemm<GE_GELU>(s, gc, x0, c.idim, M, c.bn_dim, 3 * c.idim, 3, c.idim, 1, 1, F, W + L.in0_w, W + L.in0_b,
                          nullptr, nullptr, 0, h->bufB, c.bn_dim, fr))) return rc;
  if ((rc = gemm<GE_BIAS>(s, gc, h->bufB, c.bn_dim, M, c.hidden, 3 * c.bn_dim, 3, c.bn_dim, 1, 1, F, W + L.in2_w,
                          W + L.in2_b, nullptr, nullptr, 0, h->bufA, c.hidden, fr))) return rc;
  for (int i = 0; i < c.n_layer; ++i)
    if ((rc = convnext(s, gc, W, L.blk[i], h->bufA, h->bufB, h->bufH, M, F, c.hidden, 4 * c.hidden, c.dilation, fr)))
      return rc;
  // conv_out 1x1 (no bias), out_conv k3 (no bias) * coef        (dvae.py:159,236,289-297)
  if ((rc = gemm<GE_NONE>(s, gc, h->bufA, c.hidden, M, c.odim, c.hidden, 1, c.hidden, 1, 0, F, W + L.conv_out_w, nullptr,
                          nullptr, nullptr, 0, h->bufB, c.odim, fr))) return rc;
  if ((rc = gemm<GE_COEF>(s, gc, h->bufB, c.out_dim, M, MEL_PAD, 3 * c.out_dim, 3, c.out_dim, 1, 1, F, W + L.out_conv_w,
                          nullptr, W + L.coef, nullptr, 0, h->mel_tm, MEL_PAD, fr))) return rc;
  if (mel_cf) {
    dim3 g((F + 31) / 32, (MEL + 31) / 32, B);
    k_tm_to_cf<<<g, dim3(32, 8), 0, s>>>(h->mel_tm, mel_cf, B, MEL, F, MEL_PAD);
    CTB_LAUNCH_CHECK();
  }
  return CTB_OK;
}

// fr: ragged mode (ctb_decode_rows); wav is then [B, wav_ld] and row b receives hop * (fr[b] - 1) samples
static int vocos_run(ctb_decoder* h, const float* mel_cf, int B, int F, float* wav, cudaStream_t s,
                     const int* fr = nullptr, int64_t wav_ld = 0) {
  const ctb_vocos_config& c = h->vc;
  const VocosOff& L = h->vl;
  const float* W = h->vW;
  const int M = B * F, SK = spec_k(c);
  const GemmCtx gc{h->vW, h->vW_hi, h->vW_lo, h->use_tc};
  int rc;
  if (mel_cf) {
    dim3 g((F + 31) / 32, (MEL_PAD + 31) / 32, B);
    k_cf_to_tm<<<g, dim3(32, 8), 0, s>>>(mel_cf, h->mel_tm, B, MEL, F, MEL_PAD);
    CTB_LAUNCH_CHECK();
  }
  // backbone: Conv1d(100 -> dim, k7, p3) -> LN -> ConvNeXt x num_layers -> LN
  if ((rc = gemm<GE_BIAS>(s, gc, h->mel_tm, MEL_PAD, M, c.dim, 7 * MEL_PAD, 7, MEL_PAD, 1, 3, F, W + L.embed_w,
                          W + L.embed_b, nullptr, nullptr, 0, h->bufB, c.dim, fr))) return rc;
  if ((rc = dwln(s, h->bufB, h->bufA, M, F, c.dim, 0, 1, nullptr, nullptr, W + L.norm_w, W + L.norm_b, fr))) return rc;
  for (int i = 0; i < c.num_layers; ++i)
    if ((rc = convnext(s, gc, W, L.blk[i], h->bufA, h->bufB, h->bufH, M, F, c.dim, c.intermediate_dim, 1, fr))) return rc;
  if ((rc = dwln(s, h->bufA, h->bufB, M, F, c.dim, 0, 1, nullptr, nullptr, W + L.fin_w, W + L.fin_b, fr))) return rc;
  // ISTFTHead: Linear(dim -> n_fft + 2) -> (mag, phase) -> complex spectrum (interleaved re/im)
  if ((rc = gemm<GE_SPEC>(s, gc, h->bufB, c.dim, M, SK, c.dim, 1, c.dim, 1, 0, F, W + L.head_w, W + L.head_b, nullptr,
                          nullptr, 0, h->bufA, SK, fr))) return rc;
  // inverse real DFT * window as a GEMM against the constant basis, then overlap-add / envelope
  if ((rc = gemm<GE_NONE>(s, gc, h->bufA, SK, M, c.n_fft, SK, 1, SK, 1, 0, F, W + L.basis, nullptr, nullptr, nullptr, 0,
                          h->bufH, c.n_fft, fr))) return rc;
  const size_t total = (size_t)B * c.hop_length * (F - 1);
  if (fr)
    k_overlap_add<true><<<(unsigned)((total + 255) / 256), 256, 0, s>>>(h->bufH, W + L.window, wav, B, F, c.n_fft,
                                                                        c.hop_length, fr, wav_ld);
  else
    k_overlap_add<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(h->bufH, W + L.window, wav, B, F, c.n_fft, c.hop_length);
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

extern "C" int ctb_dvae_decode(ctb_decoder* h, const void* in_dev, int32_t in_layout, int32_t B, int32_t T,
                               float* mel_dev, void* stream) {
  if (!h || !in_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (!h->dW) return set_err(CTB_ERR_STATE, "handle was created without DVAE weights");
  if (B < 1 || T < 1 || (size_t)B * 2 * T > h->max_rows)
    return set_err(CTB_ERR_ARG, "B=%d x T=%d exceeds this handle (max_batch=%d, max_tokens=%d)", B, T, h->max_batch,
                   h->max_tokens);
  if (in_layout < 0 || in_layout > 2) return set_err(CTB_ERR_ARG, "bad in_layout");
  { int rc = dec_reserve(h, (size_t)B * 2 * T, (cudaStream_t)stream); if (rc) return rc; }
  return dvae_run(h, in_dev, in_layout, B, T, mel_dev, (cudaStream_t)stream);
}

extern "C" int ctb_vocos_decode(ctb_decoder* h, const float* mel_dev, int32_t B, int32_t F, float* wav_dev,
                                void* stream) {
  if (!h || !wav_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (!h->vW) return set_err(CTB_ERR_STATE, "handle was created without Vocos weights");
  if (B < 1 || F < 2 || (size_t)B * F > h->max_rows) return set_err(CTB_ERR_ARG, "B x F exceeds this handle");
  if (mel_dev == nullptr && (size_t)B * F > h->cap_rows)
    return set_err(CTB_ERR_STATE, "no mel of this shape was left in the handle by ctb_dvae_decode");
  { int rc = dec_reserve(h, (size_t)B * F, (cudaStream_t)stream); if (rc) return rc; }
  return vocos_run(h, mel_dev, B, F, wav_dev, (cudaStream_t)stream);
}

extern "C" int ctb_decode_rows(ctb_decoder* h, int32_t kind, int32_t B, const void* const* rows_dev,
                               const int32_t* n_tokens, float* wav_dev, int64_t wav_ld, void* stream) {
  if (!h || !rows_dev || !n_tokens || !wav_dev) return set_err(CTB_ERR_ARG, "null argument");
  if (!h->dW || !h->vW) return set_err(CTB_ERR_STATE, "ctb_decode_rows needs a handle with DVAE and Vocos weights");
  if (kind != 1 && kind != 2) return set_err(CTB_ERR_ARG, "bad kind %d (1: hidden states, 2: codes)", kind);
  if (B < 1) return set_err(CTB_ERR_ARG, "B=%d", B);
  const ctb_convstack_config& c = h->dc;
  if (kind == 2 && (c.vq_dim <= 0 || c.vq_groups != 2))
    return set_err(CTB_ERR_ARG, "codes need a decoder with a VQ layer of 2 groups (use_decoder=False model)");
  int W = 0;
  for (int k = 0; k < B; ++k) {
    if (n_tokens[k] < 1) return set_err(CTB_ERR_ARG, "row %d has %d tokens", k, n_tokens[k]);
    if (!rows_dev[k] || (kind == 1 && (reinterpret_cast<uintptr_t>(rows_dev[k]) & 15)))
      return set_err(CTB_ERR_ARG, "row %d: null or (hidden states) not 16-byte aligned", k);
    W = std::max(W, (int)n_tokens[k]);
  }
  const int hop = h->vc.hop_length;
  if (wav_ld < (int64_t)hop * (2 * W - 1)) return set_err(CTB_ERR_ARG, "wav_ld %lld < %d", (long long)wav_ld, hop * (2 * W - 1));
  if ((size_t)B * 2 * W > h->max_rows)
    return set_err(CTB_ERR_ARG, "B=%d rows x %d tokens exceed this handle's %zu frames", B, W, h->max_rows);
  cudaStream_t s = (cudaStream_t)stream;
  { int rc = dec_reserve(h, (size_t)B * 2 * W, s); if (rc) return rc; }
  // one upload of the row table: [B] pointers then [B] frame counts (2 n_k).  From pageable memory the copy is staged
  // before cudaMemcpyAsync returns, so the caller's arrays may go away; stream order protects the device table.
  if (B > h->rows_meta_cap) {
    CTB_CUDA(cudaStreamSynchronize(s));
    if (h->rows_meta) { cudaFree(h->rows_meta); h->rows_meta = nullptr; h->rows_meta_cap = 0; }
    CTB_CUDA(cudaMalloc(&h->rows_meta, (size_t)B * (sizeof(void*) + sizeof(int))));
    h->rows_meta_cap = B;
  }
  std::vector<uint8_t> meta((size_t)B * (sizeof(void*) + sizeof(int)));
  memcpy(meta.data(), rows_dev, (size_t)B * sizeof(void*));
  int* fr_host = reinterpret_cast<int*>(meta.data() + (size_t)B * sizeof(void*));
  for (int k = 0; k < B; ++k) fr_host[k] = 2 * n_tokens[k];
  CTB_CUDA(cudaMemcpyAsync(h->rows_meta, meta.data(), meta.size(), cudaMemcpyHostToDevice, s));
  const void* const* rows_d = static_cast<const void* const*>(h->rows_meta);
  const int* fr = reinterpret_cast<const int*>(static_cast<uint8_t*>(h->rows_meta) + (size_t)B * sizeof(void*));
  if (kind == 1) {
    k_gather_hidden_rows<<<dim3(2 * W, B), 128, 0, s>>>(reinterpret_cast<const float* const*>(rows_d), fr, h->staged_in, W,
                                                        c.idim);
  } else {
    GfsqRowsP g{};
    g.rows = reinterpret_cast<const int32_t* const*>(rows_d); g.fr = fr; g.out = h->staged_in; g.W = W;
    g.G = c.vq_groups; g.R = c.vq_residual; g.levels = c.vq_levels & 0xff; g.nlev = 4; g.per_group = c.vq_dim / c.vq_groups;
    g.scale_base = (float)(((c.vq_levels >> 8) & 0xff) ? ((c.vq_levels >> 8) & 0xff) : (g.levels - 1));
    g.w = h->dW + h->dl.vq_w; g.b = h->dW + h->dl.vq_b;
    k_gfsq_dequant_rows<<<dim3(2 * W, B), 128, 0, s>>>(g);
  }
  CTB_LAUNCH_CHECK();
  int rc;
  if ((rc = dvae_run(h, h->staged_in, 1, B, W, nullptr, s, fr))) return rc;
  return vocos_run(h, nullptr, B, 2 * W, wav_dev, s, fr, wav_ld);
}

// ------------------------------------------------------------------ DVAE encode branch (speaker enrolment)
// DVAE.forward(mode="encode") (dvae.py:265-274): wav -> log-mel / coef -> downsample_conv -> encoder stack -> GFSQ indices.
namespace {

constexpr int ENC_NFFT = 1024, ENC_HOP = 256, ENC_NBIN = ENC_NFFT / 2 + 1, ENC_LDMAG = 516;  // MelSpectrogramFeatures defaults (dvae.py:176-181)

struct EncOff {
  int64_t window, fb, coef, ds0_w, ds0_b, ds1_w, ds1_b, in0_w, in0_b, in2_w, in2_b, conv_out_w, vq_w, vq_b, total;
  BlockOff blk[64];
};

// Blob order of the encode branch; chattts_b200/decoder.py::pack_dvae_encoder writes the same sequence.
EncOff enc_layout(const ctb_convstack_config& c) {
  EncOff o{};
  int64_t off = 0;
  o.window = take(off, ENC_NFFT);                             // analysis window (periodic Hann, fp32 like torch.hann_window)
  o.fb = take(off, (int64_t)ENC_NBIN * MEL_PAD);              // [513][128] mel filterbank, bin-major
  o.coef = take(off, MEL_PAD);
  o.ds0_w = take(off, (int64_t)c.idim * 3 * MEL_PAD);         // Conv1d(100 -> dim, k3, p1), mel channels padded to 128
  o.ds0_b = take(off, c.idim);
  o.ds1_w = take(off, (int64_t)c.idim * 3 * 2 * c.idim);      // Conv1d(dim -> dim, k4, s2, p1) over frame PAIRS: 3 taps x 2*dim
  o.ds1_b = take(off, c.idim);
  o.in0_w = take(off, (int64_t)c.bn_dim * 3 * c.idim);
  o.in0_b = take(off, c.bn_dim);
  o.in2_w = take(off, (int64_t)c.hidden * 3 * c.bn_dim);
  o.in2_b = take(off, c.hidden);
  for (int i = 0; i < c.n_layer; ++i) block_layout(o.blk[i], off, c.hidden, 4 * c.hidden);
  o.conv_out_w = take(off, (int64_t)c.odim * c.hidden);
  const int nlev = 4;
  o.vq_w = take(off, (int64_t)c.vq_groups * nlev * (c.vq_dim / c.vq_groups));  // project_in [G][4][dim/G]
  o.vq_b = take(off, (int64_t)c.vq_groups * nlev);
  o.total = off;
  return o;
}

}  // namespace

struct ctb_encoder {
  ctb_convstack_config c;
  EncOff L;
  const float* W;
  float *W_hi, *W_lo;
  bool use_tc;
  int64_t max_samples;
  int max_frames;
  float *padded, *spec, *mel_tm, *bufX, *bufY, *bufA, *bufB, *bufH;
  // what the buffers hold (enc_reserve): cap_frames STFT / mel / bufX frames (bufY..bufH: half as many token rows),
  // cap_padded samples of reflect-padded audio
  size_t cap_frames, cap_padded;
  int* rows_meta;  // ctb_dvae_encode_rows: [B] frame counts + [B] token counts, grown with B
  int rows_meta_cap;
};

extern "C" int64_t ctb_dvae_encoder_blob_floats(const ctb_convstack_config* c) { return c ? enc_layout(*c).total : -1; }

extern "C" int ctb_dvae_encoder_destroy(ctb_encoder* h) {
  if (!h) return CTB_OK;
  void* ptrs[] = {h->W_hi, h->W_lo, h->padded, h->spec, h->mel_tm, h->bufX, h->bufY, h->bufA, h->bufB, h->bufH,
                  h->rows_meta};
  for (void* p : ptrs) if (p) cudaFree(p);
  delete h;
  return CTB_OK;
}

extern "C" int ctb_dvae_encoder_create(const ctb_convstack_config* c, const float* blob_dev, int64_t max_samples,
                                       ctb_encoder** out) {
  if (!c || !blob_dev || !out) return set_err(CTB_ERR_ARG, "null argument");
  if (c->kernel != 7 || c->n_layer > 64 || c->idim % 32 || c->bn_dim % 16 || c->hidden % 128 || c->hidden > 512 || c->odim % 16)
    return set_err(CTB_ERR_ARG, "unsupported encoder stack");
  if (c->vq_dim != c->odim || c->vq_groups < 1 || c->vq_dim % c->vq_groups || c->vq_residual < 1 || (c->vq_levels & 0xff) < 2)
    return set_err(CTB_ERR_ARG, "the encoder's odim must equal vq_dim (GFSQ input)");
  if (max_samples <= ENC_NFFT / 2 || max_samples > (int64_t)1 << 28) return set_err(CTB_ERR_ARG, "max_samples out of range");
  int ndev = 0;
  CTB_CUDA(cudaGetDeviceCount(&ndev));
  if (ndev < 1) return set_err(CTB_ERR_CUDA, "no CUDA device: chattts_b200 has no CPU path");
  ctb_encoder* h = new ctb_encoder();
  memset(h, 0, sizeof(*h));
  h->c = *c; h->L = enc_layout(*c); h->W = blob_dev; h->max_samples = max_samples;
  h->max_frames = (int)(max_samples / ENC_HOP) + 1;
  h->use_tc = getenv("CTB_DECODER_FMA") == nullptr;
  const size_t F = h->max_frames, FP = (F + 1) / 2;
  cudaError_t e = cudaSuccess;
  auto A = [&](float** p, size_t n) { if (e == cudaSuccess) e = cudaMalloc((void**)p, n * sizeof(float)); };
  A(&h->padded, (F + 3) * ENC_HOP);
  A(&h->spec, F * ENC_LDMAG);
  A(&h->mel_tm, F * MEL_PAD);
  A(&h->bufX, 2 * FP * c->idim);
  A(&h->bufY, FP * c->idim);
  A(&h->bufA, FP * std::max(c->hidden, c->bn_dim));
  A(&h->bufB, FP * std::max(std::max(c->hidden, c->bn_dim), c->odim));
  A(&h->bufH, FP * 4 * c->hidden);
  if (h->use_tc) { A(&h->W_hi, h->L.total); A(&h->W_lo, h->L.total); }
  if (e != cudaSuccess) {
    cudaGetLastError();
    ctb_dvae_encoder_destroy(h);
    return set_err(CTB_ERR_NOMEM, "encoder buffers: %s", cudaGetErrorString(e));
  }
  if (h->use_tc) {
    k_split_tf32<<<1024, 256>>>(h->W, h->W_hi, h->W_lo, h->L.total);
    CTB_CUDA(cudaDeviceSynchronize());
  }
  h->cap_frames = F;
  h->cap_padded = (F + 3) * ENC_HOP;
  *out = h;
  return CTB_OK;
}

// grow the activation buffers to `frames` frames (bufY..bufH: frames / 2 token rows) and `padded` samples; the contents
// are scratch.  They never shrink below what ctb_dvae_encode needs for max_samples.
static int enc_reserve(ctb_encoder* h, size_t frames, size_t padded, cudaStream_t s) {
  if (frames <= h->cap_frames && padded <= h->cap_padded) return CTB_OK;
  CTB_CUDA(cudaStreamSynchronize(s));
  float** bufs[] = {&h->padded, &h->spec, &h->mel_tm, &h->bufX, &h->bufY, &h->bufA, &h->bufB, &h->bufH};
  for (float** b : bufs) if (*b) { cudaFree(*b); *b = nullptr; }
  h->cap_frames = h->cap_padded = 0;
  const ctb_convstack_config& c = h->c;
  const size_t F1 = (size_t)h->max_frames + 1;  // the lone call's 2 * FP frames
  const size_t R = std::max(F1, (frames + frames / 8 + 1) & ~(size_t)1);
  const size_t P = std::max((F1 + 2) * ENC_HOP, padded + padded / 8);
  cudaError_t e = cudaSuccess;
  auto A = [&](float** p, size_t n) { if (e == cudaSuccess) e = cudaMalloc((void**)p, n * sizeof(float)); };
  A(&h->padded, P);
  A(&h->spec, R * ENC_LDMAG);
  A(&h->mel_tm, R * MEL_PAD);
  A(&h->bufX, R * c.idim);
  A(&h->bufY, R / 2 * c.idim);
  A(&h->bufA, R / 2 * std::max(c.hidden, c.bn_dim));
  A(&h->bufB, R / 2 * std::max(std::max(c.hidden, c.bn_dim), c.odim));
  A(&h->bufH, R / 2 * 4 * c.hidden);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return set_err(CTB_ERR_NOMEM, "encoder buffers for %zu frames: %s", R, cudaGetErrorString(e));
  }
  h->cap_frames = R;
  h->cap_padded = P;
  return CTB_OK;
}

extern "C" int ctb_dvae_encode(ctb_encoder* h, const float* wav_dev, int64_t n_samples, int32_t* ids_dev,
                               int32_t ids_capacity_tokens, int32_t* n_tokens_out, float* mel_dev, float* margin_dev,
                               void* stream) {
  if (!h || !wav_dev || !ids_dev || !n_tokens_out) return set_err(CTB_ERR_ARG, "null argument");
  if (n_samples <= ENC_NFFT / 2) return set_err(CTB_ERR_ARG, "reflect padding needs more than %d samples", ENC_NFFT / 2);
  if (n_samples > h->max_samples) return set_err(CTB_ERR_ARG, "%lld samples exceed this handle (max_samples=%lld)",
                                                 (long long)n_samples, (long long)h->max_samples);
  const ctb_convstack_config& c = h->c;
  const EncOff& L = h->L;
  const float* W = h->W;
  cudaStream_t s = (cudaStream_t)stream;
  const int F = (int)(n_samples / ENC_HOP) + 1;     // torch.stft(center=True)
  const int T = F / 2;                              // Conv1d(k4, s2, p1): floor((F + 2 - 4) / 2) + 1
  *n_tokens_out = T;
  if (T < 1) return set_err(CTB_ERR_ARG, "audio too short for one token");
  if (T > ids_capacity_tokens) return set_err(CTB_ERR_ARG, "ids buffer holds %d tokens, %d needed", ids_capacity_tokens, T);
  const GemmCtx gc{h->W, h->W_hi, h->W_lo, h->use_tc};
  int rc;
  // a no-op unless a failed ctb_dvae_encode_rows growth left the handle without buffers
  if ((rc = enc_reserve(h, h->max_frames, (size_t)(h->max_frames + 3) * ENC_HOP, s))) return rc;
  // framing (reflect padding) -> |STFT| as a double-precision direct DFT -> mel filterbank, log, / coef
  const int64_t total = (int64_t)(F + 3) * ENC_HOP;
  k_reflect_pad<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(wav_dev, h->padded, n_samples, total, ENC_NFFT / 2);
  CTB_LAUNCH_CHECK();
  k_stft_mag<ENC_NFFT><<<dim3(F, (ENC_NBIN + 255) / 256), 256, 0, s>>>(h->padded, W + L.window, ENC_HOP, ENC_NBIN, h->spec, ENC_LDMAG);
  CTB_LAUNCH_CHECK();
  k_mel_log<MEL_PAD><<<F, MEL_PAD, ENC_NBIN * sizeof(float), s>>>(h->spec, ENC_LDMAG, ENC_NBIN, W + L.fb, W + L.coef, MEL, h->mel_tm);
  CTB_LAUNCH_CHECK();
  if (mel_dev) {
    dim3 g((F + 31) / 32, (MEL + 31) / 32, 1);
    k_tm_to_cf<<<g, dim3(32, 8), 0, s>>>(h->mel_tm, mel_dev, 1, MEL, F, MEL_PAD);
    CTB_LAUNCH_CHECK();
  }
  // downsample_conv (dvae.py:231-236): Conv1d(100 -> dim, k3, p1) + GELU; Conv1d(dim -> dim, k4, s2, p1) + GELU.
  // The stride-2 conv runs over frame pairs [F/2 rows, 2*dim]: out[t] = W0 x[2t-1] + W1 x[2t] + W2 x[2t+1] + W3 x[2t+2]
  // = 3 taps over pair rows with the weights re-packed (zeros where a pair half is not touched).
  const int FP = (F + 1) / 2;
  if (F & 1) CTB_CUDA(cudaMemsetAsync(h->bufX + (size_t)F * c.idim, 0, (size_t)c.idim * sizeof(float), s));
  if ((rc = gemm<GE_GELU>(s, gc, h->mel_tm, MEL_PAD, F, c.idim, 3 * MEL_PAD, 3, MEL_PAD, 1, 1, F, W + L.ds0_w, W + L.ds0_b,
                          nullptr, nullptr, 0, h->bufX, c.idim))) return rc;
  if ((rc = gemm<GE_GELU>(s, gc, h->bufX, 2 * c.idim, FP, c.idim, 3 * 2 * c.idim, 3, 2 * c.idim, 1, 1, FP, W + L.ds1_w,
                          W + L.ds1_b, nullptr, nullptr, 0, h->bufY, c.idim))) return rc;
  // encoder = DVAEDecoder(idim -> odim) over the first T rows (dvae.py:131-172)
  if ((rc = gemm<GE_GELU>(s, gc, h->bufY, c.idim, T, c.bn_dim, 3 * c.idim, 3, c.idim, 1, 1, T, W + L.in0_w, W + L.in0_b,
                          nullptr, nullptr, 0, h->bufB, c.bn_dim))) return rc;
  if ((rc = gemm<GE_BIAS>(s, gc, h->bufB, c.bn_dim, T, c.hidden, 3 * c.bn_dim, 3, c.bn_dim, 1, 1, T, W + L.in2_w, W + L.in2_b,
                          nullptr, nullptr, 0, h->bufA, c.hidden))) return rc;
  for (int i = 0; i < c.n_layer; ++i)
    if ((rc = convnext(s, gc, W, L.blk[i], h->bufA, h->bufB, h->bufH, T, T, c.hidden, 4 * c.hidden, c.dilation))) return rc;
  if ((rc = gemm<GE_NONE>(s, gc, h->bufA, c.hidden, T, c.odim, c.hidden, 1, c.hidden, 1, 0, T, W + L.conv_out_w, nullptr,
                          nullptr, nullptr, 0, h->bufB, c.odim))) return rc;
  FsqQuantP q{};
  q.x = h->bufB; q.ids = ids_dev; q.margin = margin_dev; q.T = T; q.G = c.vq_groups; q.R = c.vq_residual;
  q.levels = c.vq_levels & 0xff; q.nlev = 4; q.per_group = c.vq_dim / c.vq_groups;
  q.scale_base = (float)(((c.vq_levels >> 8) & 0xff) ? ((c.vq_levels >> 8) & 0xff) : (q.levels - 1));
  q.bound_input = ((c.vq_levels >> 16) & 1) ? 0 : 1;
  q.w = W + L.vq_w; q.b = W + L.vq_b;
  k_fsq_quant<<<T * c.vq_groups, 128, 0, s>>>(q);
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}

// Ragged batch of the encode branch.  Row k's frames live at a frame stride FW (the widest row's F, rounded up to even,
// so a frame pair never straddles two rows) and its tokens at a stride FW / 2.  Every buffer a tapped conv reads holds
// exact +0 in row k's frames f >= F_k (tokens t >= T_k), which is what TMA's out-of-bounds fill (or the FMA kernel's
// range check) gives the lone call; every output element then keeps its operands and reduction order.
extern "C" int ctb_dvae_encode_rows(ctb_encoder* h, int32_t B, const float* const* wavs_dev, const int64_t* n_samples,
                                    int32_t* ids_dev, int32_t ids_ld, int32_t* n_tokens_out, float* margin_dev,
                                    void* stream) {
  if (!h || !wavs_dev || !n_samples || !ids_dev || !n_tokens_out) return set_err(CTB_ERR_ARG, "null argument");
  if (B < 1) return set_err(CTB_ERR_ARG, "B=%d", B);
  int Fmax = 0;
  for (int k = 0; k < B; ++k) {
    if (!wavs_dev[k]) return set_err(CTB_ERR_ARG, "row %d: null wav", k);
    if (n_samples[k] <= ENC_NFFT / 2)
      return set_err(CTB_ERR_ARG, "row %d: reflect padding needs more than %d samples", k, ENC_NFFT / 2);
    if (n_samples[k] > h->max_samples)
      return set_err(CTB_ERR_ARG, "row %d: %lld samples exceed this handle (max_samples=%lld)", k,
                     (long long)n_samples[k], (long long)h->max_samples);
    const int F = (int)(n_samples[k] / ENC_HOP) + 1;
    if (F / 2 > ids_ld) return set_err(CTB_ERR_ARG, "row %d: ids_ld %d < %d tokens", k, ids_ld, F / 2);
    Fmax = std::max(Fmax, F);
  }
  const ctb_convstack_config& c = h->c;
  const EncOff& L = h->L;
  const float* W = h->W;
  cudaStream_t s = (cudaStream_t)stream;
  const int FW = (Fmax + 1) & ~1, TW = FW / 2;
  int rc;
  if ((rc = enc_reserve(h, (size_t)B * FW, (size_t)B * (FW + 3) * ENC_HOP, s))) return rc;
  // one upload of the row table: [B] frame counts then [B] token counts (staged from pageable memory before
  // cudaMemcpyAsync returns; stream order protects the device copy)
  if (B > h->rows_meta_cap) {
    CTB_CUDA(cudaStreamSynchronize(s));
    if (h->rows_meta) { cudaFree(h->rows_meta); h->rows_meta = nullptr; h->rows_meta_cap = 0; }
    CTB_CUDA(cudaMalloc((void**)&h->rows_meta, (size_t)B * 2 * sizeof(int)));
    h->rows_meta_cap = B;
  }
  std::vector<int> meta((size_t)2 * B);
  for (int k = 0; k < B; ++k) {
    meta[k] = (int)(n_samples[k] / ENC_HOP) + 1;
    meta[B + k] = n_tokens_out[k] = meta[k] / 2;
  }
  CTB_CUDA(cudaMemcpyAsync(h->rows_meta, meta.data(), meta.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  const int* fr = h->rows_meta;
  const int* tn = h->rows_meta + B;
  const GemmCtx gc{h->W, h->W_hi, h->W_lo, h->use_tc};
  // framing, |STFT| and log-mel are frame-local: the lone kernels run per row, and the mel frames past F_k are +0
  for (int k = 0; k < B; ++k) {
    const int F = meta[k];
    float* padded = h->padded + (size_t)k * (FW + 3) * ENC_HOP;
    float* spec = h->spec + (size_t)k * FW * ENC_LDMAG;
    float* mel = h->mel_tm + (size_t)k * FW * MEL_PAD;
    const int64_t total = (int64_t)(F + 3) * ENC_HOP;
    k_reflect_pad<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(wavs_dev[k], padded, n_samples[k], total, ENC_NFFT / 2);
    CTB_LAUNCH_CHECK();
    k_stft_mag<ENC_NFFT><<<dim3(F, (ENC_NBIN + 255) / 256), 256, 0, s>>>(padded, W + L.window, ENC_HOP, ENC_NBIN, spec,
                                                                         ENC_LDMAG);
    CTB_LAUNCH_CHECK();
    k_mel_log<MEL_PAD><<<F, MEL_PAD, ENC_NBIN * sizeof(float), s>>>(spec, ENC_LDMAG, ENC_NBIN, W + L.fb, W + L.coef, MEL,
                                                                     mel);
    CTB_LAUNCH_CHECK();
    if (F < FW) CTB_CUDA(cudaMemsetAsync(mel + (size_t)F * MEL_PAD, 0, (size_t)(FW - F) * MEL_PAD * sizeof(float), s));
  }
  // ds0 writes +0 in frames f >= F_k, so each row's frame pairs past its own are zero, the frame at F_k of an odd F_k
  // included (the lone call's memset).  ds1 writes +0 in token rows t >= T_k: the lone call computes rows T..FP-1 but
  // its stack reads them only as out-of-bounds zeros.
  if ((rc = gemm<GE_GELU>(s, gc, h->mel_tm, MEL_PAD, B * FW, c.idim, 3 * MEL_PAD, 3, MEL_PAD, 1, 1, FW, W + L.ds0_w,
                          W + L.ds0_b, nullptr, nullptr, 0, h->bufX, c.idim, fr))) return rc;
  if ((rc = gemm<GE_GELU>(s, gc, h->bufX, 2 * c.idim, B * TW, c.idim, 3 * 2 * c.idim, 3, 2 * c.idim, 1, 1, TW,
                          W + L.ds1_w, W + L.ds1_b, nullptr, nullptr, 0, h->bufY, c.idim, tn))) return rc;
  if ((rc = gemm<GE_GELU>(s, gc, h->bufY, c.idim, B * TW, c.bn_dim, 3 * c.idim, 3, c.idim, 1, 1, TW, W + L.in0_w,
                          W + L.in0_b, nullptr, nullptr, 0, h->bufB, c.bn_dim, tn))) return rc;
  if ((rc = gemm<GE_BIAS>(s, gc, h->bufB, c.bn_dim, B * TW, c.hidden, 3 * c.bn_dim, 3, c.bn_dim, 1, 1, TW, W + L.in2_w,
                          W + L.in2_b, nullptr, nullptr, 0, h->bufA, c.hidden, tn))) return rc;
  for (int i = 0; i < c.n_layer; ++i)
    if ((rc = convnext(s, gc, W, L.blk[i], h->bufA, h->bufB, h->bufH, B * TW, TW, c.hidden, 4 * c.hidden, c.dilation,
                       tn))) return rc;
  if ((rc = gemm<GE_NONE>(s, gc, h->bufA, c.hidden, B * TW, c.odim, c.hidden, 1, c.hidden, 1, 0, TW, W + L.conv_out_w,
                          nullptr, nullptr, nullptr, 0, h->bufB, c.odim, tn))) return rc;
  FsqQuantP q{};
  q.x = h->bufB; q.ids = ids_dev; q.margin = margin_dev; q.T = ids_ld; q.G = c.vq_groups; q.R = c.vq_residual;
  q.levels = c.vq_levels & 0xff; q.nlev = 4; q.per_group = c.vq_dim / c.vq_groups;
  q.scale_base = (float)(((c.vq_levels >> 8) & 0xff) ? ((c.vq_levels >> 8) & 0xff) : (q.levels - 1));
  q.bound_input = ((c.vq_levels >> 16) & 1) ? 0 : 1;
  q.w = W + L.vq_w; q.b = W + L.vq_b;
  q.tn = tn; q.F = TW;
  k_fsq_quant<true><<<dim3(TW * c.vq_groups, B), 128, 0, s>>>(q);
  CTB_LAUNCH_CHECK();
  return CTB_OK;
}
