// Fused sampling tail (reference gpt.py:487-525 + processors.py:18-58 + HF TopP/TopK warpers).
// One CTA of 1024 threads per logits row.
#include "gpt_kernels.cuh"

namespace ctb {

namespace {

template <int NT = SAMPLE_THREADS>
__device__ __forceinline__ double block_sum_d(double v, double* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum_d(v);
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  double t = 0.0;
#pragma unroll 8
  for (int w = 0; w < NT / 32; ++w) t += s_red[w];  // fixed order => deterministic
  return t;
}

__device__ __forceinline__ int block_sum_i(int v, int* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = __reduce_add_sync(0xffffffffu, v);
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  int t = 0;
#pragma unroll 8
  for (int w = 0; w < SAMPLE_THREADS / 32; ++w) t += s_red[w];
  return t;
}

template <int NT = SAMPLE_THREADS>
__device__ __forceinline__ float block_max_f(float v, float* s_red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float t = -INFINITY;
#pragma unroll 8
  for (int w = 0; w < NT / 32; ++w) t = fmaxf(t, s_red[w]);
  return t;
}

}  // namespace

template <bool ENGINE>
__global__ void __launch_bounds__(SAMPLE_THREADS) k_sample(const SampleP p) {
  pdl_trigger();
  pdl_wait();
  if (p.check_finished && ldg_cg(&p.st->all_finished)) return;
  const int row = blockIdx.x, V = p.V, rpi = p.rows_per_item;
  const int item = row / rpi, qi = row % rpi;
  __shared__ ctb_sampler_config s_cfg;
  if (ENGINE) {
    if (!row_wanted(p.rstate + item, p.want)) return;  // CTA-uniform
    static_assert(sizeof(ctb_sampler_config) % 4 == 0, "config is copied as words");
    const uint32_t* src = reinterpret_cast<const uint32_t*>(p.cfgs + item);
    for (int i = threadIdx.x; i < (int)(sizeof(ctb_sampler_config) / 4); i += SAMPLE_THREADS)
      reinterpret_cast<uint32_t*>(&s_cfg)[i] = __ldg(src + i);
    __syncthreads();
  }
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* s_x = reinterpret_cast<float*>(smem_raw);                 // [V] processed logits
  uint32_t* s_key = reinterpret_cast<uint32_t*>(s_x + p.V);        // [2][1024] sort path only
  __shared__ double s_redd[SAMPLE_THREADS / 32];
  __shared__ int s_redi[SAMPLE_THREADS / 32];
  __shared__ float s_redf[SAMPLE_THREADS / 32];
  __shared__ int s_win[32];
  __shared__ uint32_t s_thr;

  const int tid = threadIdx.x;
  const int n_gen = ENGINE ? ldg_cg(&p.rstate[item].n_gen) : (p.st ? ldg_cg(&p.st->n_gen) : p.n_gen_fixed);
  const int step = ENGINE ? ldg_cg(&p.rstate[item].step) : (p.st ? ldg_cg(&p.st->step) : p.step_fixed);
  const ctb_sampler_config& c = ENGINE ? s_cfg : p.cfg;
  const float* lg = p.logits + (size_t)row * V;
  // a slot's request is sampled as if it were decoded alone (B = 1): its logits row index is the codebook index
  const int prow = ENGINE ? qi : row;

  // ---- S2 window of the last <= past_window generated ids of this (item, codebook) row
  int nwin = 0;
  const bool pen = c.penalty_on && prow < c.penalty_max_ids;
  if (pen) {
    nwin = min(n_gen, c.past_window);
    if (tid < nwin) s_win[tid] = ldg_cg(&p.gen_ids[((size_t)item * p.gen_stride + (n_gen - nwin + tid)) * p.gen_inner + qi]);
  }
  __syncthreads();
  // ---- S1 temperature, S2 penalty
  const float temp = c.temperature[qi];
  for (int v = tid; v < V; v += SAMPLE_THREADS) {
    float x = __fdiv_rn(ldg_cg(&lg[v]), temp);
    if (pen) {
      int cnt = 0;
      for (int w = 0; w < nwin; ++w) cnt += (s_win[w] == v);
      const float a = c.penalty_lut[cnt];
      x = (x < 0.f) ? __fmul_rn(x, a) : __fdiv_rn(x, a);
    }
    s_x[v] = x;
  }
  __syncthreads();

  // ---- row max and softmax denominator of the unfiltered row (top-p's own softmax)
  float mx = -INFINITY;
  for (int v = tid; v < V; v += SAMPLE_THREADS) mx = fmaxf(mx, s_x[v]);
  mx = block_max_f(mx, s_redf);

  // top_k is taken as given: TopKLogitsWarper has already folded its own min_tokens_to_keep into it, and
  // c.min_tokens_to_keep is top-p's alone.  Both cuts are key thresholds, so a tie group at either cut is kept whole:
  // top-p keeps every token equal to the smallest kept one, where HF removes by position in its sorted row (an order
  // among equal values no deterministic kernel can reproduce; only the number HF removes is defined).
  const bool use_p = c.top_p >= 0.f;
  const int kk = c.top_k > 0 ? min(c.top_k, V) : 0;
  const int min_keep = min(c.min_tokens_to_keep, V);
  uint32_t thr_key = 0;  // keep x iff float_key(x) >= thr_key

  if (use_p || kk > 0) {
    double den = 0.0;
    if (use_p) {
      for (int v = tid; v < V; v += SAMPLE_THREADS) den += (double)expf(s_x[v] - mx);
      den = block_sum_d(den, s_redd);
    }
    const float denf = (float)den;
    const float pthr = c.has_removed_max ? c.top_p_removed_max : (float)(1.0 - (double)c.top_p);  // `cum <= (1 - top_p)` evaluated in fp32
    if (V <= 1024) {
      // ---------- sort path: bitonic sort of 1024 keys (pads = 0 sort first).  One key per thread in a register;
      // compare-exchange distances < 32 are warp shuffles, the 15 longer ones go through two alternating
      // shared-memory buffers (one barrier each instead of 55 barriers for an all-shared-memory network).
      uint32_t key = tid < V ? float_key(s_x[tid]) : 0u;
      int sb = 0;
      for (int k = 2; k <= 1024; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
          uint32_t other;
          if (j >= 32) {
            uint32_t* buf = s_key + sb * 1024;
            buf[tid] = key;
            __syncthreads();
            other = buf[tid ^ j];
            sb ^= 1;
          } else {
            other = __shfl_xor_sync(0xffffffffu, key, j);
          }
          const bool up = (tid & k) == 0, lower = (tid & j) == 0;
          key = (lower == up) ? min(key, other) : max(key, other);
        }
      }
      __syncthreads();
      s_key[tid] = key;
      __syncthreads();
      uint32_t t_p = 0;
      if (use_p) {
        // inclusive scan (double, like ATen's CPU cumsum) of softmax(sorted) ascending
        const uint32_t key = s_key[tid];
        double pv = key ? (double)__fdiv_rn(expf(key_float(key) - mx), denf) : 0.0;
        const int lane = tid & 31, warp = tid >> 5;
        double inc = pv;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const double n = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += n;
        }
        if (lane == 31) s_redd[warp] = inc;
        __syncthreads();
        double base = 0.0;
        for (int w = 0; w < warp; ++w) base += s_redd[w];
        const float cum = (float)(base + inc);
        const int removed = (cum <= pthr) && (tid < 1024 - min_keep);
        const int nrem = __syncthreads_count(removed);  // removed set is a prefix of the sorted row
        t_p = s_key[nrem];
      }
      const uint32_t t_k = kk > 0 ? s_key[1024 - kk] : 0u;
      thr_key = max(t_p, t_k);
    } else {
      // ---------- search path (text head, V = 21178): bisection on the key space
      uint32_t t_p = 0;
      if (use_p) {
        // smallest key t with float(sum_{key_j <= t} p_j) > pthr
        uint32_t lo = 0u, hi = 0xffffffffu;
        while (lo < hi) {
          const uint32_t mid = lo + ((hi - lo) >> 1);
          double s = 0.0;
          for (int v = tid; v < V; v += SAMPLE_THREADS) {
            const float x = s_x[v];
            if (float_key(x) <= mid) s += (double)__fdiv_rn(expf(x - mx), denf);
          }
          s = block_sum_d(s, s_redd);
          if ((float)s > pthr) hi = mid; else lo = mid + 1;
        }
        t_p = lo;
        // always keep the min_keep largest: largest t with count(key >= t) >= min_keep
        uint32_t lo2 = 0u, hi2 = 0xffffffffu;
        while (lo2 < hi2) {
          const uint32_t mid = lo2 + (uint32_t)(((uint64_t)hi2 - lo2 + 1) >> 1);
          int cnt = 0;
          for (int v = tid; v < V; v += SAMPLE_THREADS) cnt += (float_key(s_x[v]) >= mid);
          cnt = block_sum_i(cnt, s_redi);
          if (cnt >= min_keep) lo2 = mid; else hi2 = mid - 1;
        }
        t_p = min(t_p, lo2);
      }
      uint32_t t_k = 0;
      if (kk > 0) {
        uint32_t lo2 = 0u, hi2 = 0xffffffffu;
        while (lo2 < hi2) {
          const uint32_t mid = lo2 + (uint32_t)(((uint64_t)hi2 - lo2 + 1) >> 1);
          int cnt = 0;
          for (int v = tid; v < V; v += SAMPLE_THREADS) cnt += (float_key(s_x[v]) >= mid);
          cnt = block_sum_i(cnt, s_redi);
          if (cnt >= kk) lo2 = mid; else hi2 = mid - 1;
        }
        t_k = lo2;
      }
      thr_key = max(t_p, t_k);
    }
  }
  if (c.greedy) {
    // bench config C2: keep only the row arg-max; greedy == 2 takes it over the non-EOS tokens so
    // that the EOS ban below can never empty the row
    float gm = -INFINITY;
    for (int v = tid; v < V; v += SAMPLE_THREADS)
      if (!(c.greedy == 2 && v == c.eos_token)) gm = fmaxf(gm, s_x[v]);
    gm = block_max_f(gm, s_redf);
    thr_key = float_key(gm);
  }
  if (tid == 0) s_thr = thr_key;
  __syncthreads();
  thr_key = s_thr;

  // ---- EOS ban (gpt.py:494-495), final softmax (gpt.py:497), argmax(p / q) (gpt.py:501-508)
  const bool ban = step < c.min_new_token;
  float mx2 = -INFINITY;
  for (int v = tid; v < V; v += SAMPLE_THREADS) {
    float x = s_x[v];
    if (float_key(x) < thr_key || ((ban || c.greedy == 2) && v == c.eos_token)) x = -INFINITY;
    s_x[v] = x;
    mx2 = fmaxf(mx2, x);
  }
  mx2 = block_max_f(mx2, s_redf);
  double den2 = 0.0;
  for (int v = tid; v < V; v += SAMPLE_THREADS) den2 += (double)expf(s_x[v] - mx2);
  den2 = block_sum_d(den2, s_redd);
  const float den2f = (float)den2;

  const bool noise = ENGINE ? ldg_cg(&p.rstate[item].has_noise) != 0 : p.q_noise != nullptr;
  float best = -1.f;
  int besti = 0x7fffffff;
  for (int v = tid; v < V; v += SAMPLE_THREADS) {
    const float pr = __fdiv_rn(expf(s_x[v] - mx2), den2f);
    const float qn = noise ? (ENGINE ? p.q_noise[(size_t)item * p.noise_stride + (size_t)qi * V + v]
                                     : p.q_noise[(size_t)row * V + v])
                           : philox_exp1(c.philox_seed, (uint32_t)prow, (uint32_t)v, (uint32_t)step);
    const float r = __fdiv_rn(pr, qn);
    if (r > best) { best = r; besti = v; }  // ascending v within a thread: first max wins
  }
  // block arg-max, lowest index on ties (ATen argmax returns the first maximum)
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
  }
  __shared__ float s_bv[SAMPLE_THREADS / 32];
  __shared__ int s_bi[SAMPLE_THREADS / 32];
  __syncthreads();
  if ((tid & 31) == 0) { s_bv[tid >> 5] = best; s_bi[tid >> 5] = besti; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < SAMPLE_THREADS / 32; ++w)
      if (s_bv[w] > best || (s_bv[w] == best && s_bi[w] < besti)) { best = s_bv[w]; besti = s_bi[w]; }
    p.out_idx[row] = besti < V ? besti : 0;  // all-NaN row: ATen argmax returns the first index
  }
}

// finish / write-back / counters (gpt.py:512-525,572-577).  One CTA, one thread per batch row.
__global__ void k_finalize(const FinalP p) {
  pdl_trigger();
  pdl_wait();
  if (ldg_cg(&p.st->all_finished)) return;
  __shared__ int s_any, s_notall;
  if (threadIdx.x == 0) { s_any = 0; s_notall = 0; }
  __syncthreads();
  const int n = ldg_cg(&p.st->n_gen);
  const int step0 = ldg_cg(&p.st->step);
  for (int b = threadIdx.x; b < p.B; b += blockDim.x) {
    bool eos = false;
    for (int q = 0; q < p.rows_per_item; ++q) eos |= (ldg_cg(&p.idx[b * p.rows_per_item + q]) == p.eos);
    const bool fin = ldg_cg(&p.finish[b]) || eos;
    p.finish[b] = fin ? 1 : 0;
    int32_t* dst = p.ids_out + ((size_t)b * p.max_new + n) * p.num_vq;
    for (int q = 0; q < p.num_vq; ++q) dst[q] = ldg_cg(&p.idx[b * p.rows_per_item + (p.rows_per_item == 1 ? 0 : q)]);
    if (fin) atomicOr(&s_any, 1); else { atomicOr(&s_notall, 1); }
    // gpt.py:527: at i == 0 with any finished row the reference returns before end_idx moves
    (void)0;
  }
  __syncthreads();
  const bool first_abort = (step0 == 0) && s_any;
  if (!first_abort)
    for (int b = threadIdx.x; b < p.B; b += blockDim.x)
      if (!p.finish[b]) p.end_idx[b] = ldg_cg(&p.end_idx[b]) + 1;
  __syncthreads();
  if (threadIdx.x == 0) {
    if (first_abort) { p.st->any_first = 1; p.st->all_finished = 1; }
    else if (!s_notall) p.st->all_finished = 1;
    p.st->n_gen = n + 1;
    p.st->step = step0 + 1;
  }
}

// Slot-engine counterpart of k_finalize: every row in state `want` (RS_RUNNING in a decode step, RS_PENDING after an
// admission's prefill) writes its token at its own n_gen and advances its own counters; a row ends at EOS or at its
// own max_new.  A B = 1 request that samples EOS first ends empty (end_idx 0, finish 1): the reference's first-step
// return (gpt.py:527) seen from a batch of one.  all_finished = no running row.
__global__ void k_finalize_rows(const FinalP p) {
  pdl_trigger();
  pdl_wait();
  const bool decode = p.want == RS_RUNNING;
  if (decode && ldg_cg(&p.st->all_finished)) return;
  __shared__ int s_running;
  if (threadIdx.x == 0) s_running = 0;
  __syncthreads();
  for (int b = threadIdx.x; b < p.B; b += blockDim.x) {
    RowState* r = p.rows + b;
    int state = ldg_cg(&r->state);
    if (state == p.want) {
      const int n = ldg_cg(&r->n_gen), eos_tok = ldg_cg(&r->eos);
      bool eos = false;
      int32_t* dst = p.ids_out + ((size_t)b * p.max_new + n) * p.num_vq;
      if (ldg_cg(&r->text)) {  // one text id, written to every column (k_finalize with rows_per_item == 1)
        const int32_t id = ldg_cg(&p.idx_text[b]);
        eos = id == eos_tok;
        for (int q = 0; q < p.num_vq; ++q) dst[q] = id;
      } else {
        for (int q = 0; q < p.rows_per_item; ++q) eos |= (ldg_cg(&p.idx[b * p.rows_per_item + q]) == eos_tok);
        for (int q = 0; q < p.num_vq; ++q) dst[q] = ldg_cg(&p.idx[b * p.rows_per_item + (p.rows_per_item == 1 ? 0 : q)]);
      }
      p.finish[b] = eos ? 1 : 0;
      if (!eos) p.end_idx[b] = ldg_cg(&p.end_idx[b]) + 1;
      r->n_gen = n + 1;
      r->step = ldg_cg(&r->step) + 1;
      state = (eos || n + 1 >= ldg_cg(&r->max_new)) ? RS_FINISHED : RS_RUNNING;
      r->state = state;
    }
    if (state == RS_RUNNING) atomicOr(&s_running, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    p.st->all_finished = s_running ? 0 : 1;
    if (decode) p.st->step = ldg_cg(&p.st->step) + 1;
  }
}

// Slot-engine cancellation (ctb_gpt_engine_cancel), launched between decode steps outside the captured graphs: every
// listed row that is running or pending ends as a row that stopped short of EOS (RS_FINISHED, finish 0) and keeps its
// end_idx, so its outputs stay a valid prefix.  Other rows are untouched.  all_finished = no running row, as in
// k_finalize_rows, so later decode steps with nothing running stay no-ops and do not advance st->step.
__global__ void k_cancel_rows(const CancelP p) {
  __shared__ int s_running;
  if (threadIdx.x == 0) s_running = 0;
  __syncthreads();
  for (int b = threadIdx.x; b < p.B; b += blockDim.x) {
    RowState* r = p.rows + b;
    int state = ldg_cg(&r->state);
    if (((p.mask[b >> 5] >> (b & 31)) & 1u) && (state == RS_RUNNING || state == RS_PENDING)) {
      p.finish[b] = 0;
      state = RS_FINISHED;
      r->state = state;
    }
    if (state == RS_RUNNING) atomicOr(&s_running, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) p.st->all_finished = s_running ? 0 : 1;
}

// Token log-probability (ctb_gpt_engine_logprobs, ctb_token_logprobs): one CTA per logits row.  The row max in fp32,
// den = sum exp(z_v - max) summed in double in a fixed order (per thread over v, then warps, then the CTA's warps in
// order, as k_sample sums its denominators), lp = (double)(z_id - max) - log(den) rounded once to fp32: the same
// logits give the same bits.  An id outside [0, V) (stand-alone calls only; k_sample never writes one) gives NaN.
__global__ void __launch_bounds__(LOGPROB_THREADS) k_token_logprob(const LogprobP p) {
  pdl_trigger();
  pdl_wait();
  if (p.check_finished && ldg_cg(&p.st->all_finished)) return;
  const int row = blockIdx.x, V = p.V;
  const int item = row / p.rows_per_item, q = row % p.rows_per_item;
  if (p.rstate != nullptr && !row_wanted(p.rstate + item, p.want)) return;  // CTA-uniform: the rows k_sample served
  __shared__ double s_redd[LOGPROB_THREADS / 32];
  __shared__ float s_redf[LOGPROB_THREADS / 32];
  const float* lg = p.logits + (size_t)row * V;
  float mx = -INFINITY;
  for (int v = threadIdx.x; v < V; v += LOGPROB_THREADS) mx = fmaxf(mx, ldg_cg(&lg[v]));
  mx = block_max_f<LOGPROB_THREADS>(mx, s_redf);
  double den = 0.0;
  for (int v = threadIdx.x; v < V; v += LOGPROB_THREADS) den += (double)expf(ldg_cg(&lg[v]) - mx);
  den = block_sum_d<LOGPROB_THREADS>(den, s_redd);
  if (threadIdx.x != 0) return;
  const int id = ldg_cg(&p.idx[row]);
  const float lp = (id >= 0 && id < V) ? (float)((double)(ldg_cg(&lg[id]) - mx) - log(den)) : __int_as_float(0x7fc00000);
  if (p.rstate == nullptr) {
    p.out[row] = lp;
  } else {
    const int n_gen = ldg_cg(&p.rstate[item].n_gen);
    p.out[((size_t)item * p.max_new + n_gen) * p.num_vq + q] = lp;
  }
}

namespace {

// One 64-bit key per column, larger = earlier in the top order: float_key(z) (one key for -0.0 and +0.0, which compare
// equal) above 0x7fffffff - v (the smaller id first among equal z).  Every key is > 0 and < ~0ull.
__device__ __forceinline__ unsigned long long top_key(float z, int v) {
  return ((unsigned long long)float_key(z) << 32) | (uint32_t)(0x7fffffff - v);
}

// the largest key below `below` among this thread's columns of s_z[0, V), 0 if none
__device__ __forceinline__ unsigned long long top_scan(const float* s_z, int V, unsigned long long below) {
  unsigned long long best = 0ull;
  for (int v = threadIdx.x; v < V; v += LOGPROB_THREADS) {
    const unsigned long long k = top_key(s_z[v], v);
    if (k < below && k > best) best = k;
  }
  return best;
}

}  // namespace

// Top log-probabilities (ctb_gpt_engine_top_logprobs, ctb_token_top_logprobs, ctb_gpt_score_ex): one CTA per logits row.
// The row goes to shared memory as k_token_logprob's max pass reads it; max and den are then k_token_logprob's (same
// CTA size, helpers and summation order), so an entry equals that kernel's value for its id bit for bit.  Selection:
// n_top rounds of a block arg-max over the column keys.  Each thread holds the best key of its columns below the last
// chosen one; only the thread that owned the round's winner rescans its columns, so a round is one rescan of V / 256
// columns and one CTA reduction, and the result depends on the keys alone.
__global__ void __launch_bounds__(LOGPROB_THREADS) k_token_top_logprobs(const TopLogprobP p) {
  pdl_trigger();
  pdl_wait();
  if (p.check_finished && ldg_cg(&p.st->all_finished)) return;
  const int row = blockIdx.x, V = p.V;
  const int item = row / p.rows_per_item, q = row % p.rows_per_item;
  if (p.rstate != nullptr && !row_wanted(p.rstate + item, p.want)) return;  // CTA-uniform: the rows k_sample served
  extern __shared__ float s_z[];  // [V]
  __shared__ double s_redd[LOGPROB_THREADS / 32];
  __shared__ float s_redf[LOGPROB_THREADS / 32];
  __shared__ unsigned long long s_best[2][LOGPROB_THREADS / 32];
  const float* lg = p.logits + (size_t)row * V;
  float mx = -INFINITY;
  for (int v = threadIdx.x; v < V; v += LOGPROB_THREADS) {
    const float z = ldg_cg(&lg[v]);
    s_z[v] = z;
    mx = fmaxf(mx, z);
  }
  mx = block_max_f<LOGPROB_THREADS>(mx, s_redf);  // its barriers also publish s_z
  double den = 0.0;
  for (int v = threadIdx.x; v < V; v += LOGPROB_THREADS) den += (double)expf(s_z[v] - mx);
  den = block_sum_d<LOGPROB_THREADS>(den, s_redd);
  const double lden = log(den);
  const size_t base = p.rstate == nullptr
      ? (size_t)row * p.n_top
      : (((size_t)item * p.max_new + ldg_cg(&p.rstate[item].n_gen)) * p.num_vq + q) * p.n_top;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long mine = top_scan(s_z, V, ~0ull);
  for (int k = 0; k < p.n_top; ++k) {
    unsigned long long w = mine;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ow = __shfl_xor_sync(0xffffffffu, w, o);
      w = ow > w ? ow : w;
    }
    // two buffers: round k + 2 writes this one only after every thread has passed round k + 1's barrier
    if (lane == 0) s_best[k & 1][warp] = w;
    __syncthreads();
    w = 0ull;
#pragma unroll
    for (int i = 0; i < LOGPROB_THREADS / 32; ++i) w = s_best[k & 1][i] > w ? s_best[k & 1][i] : w;
    if (threadIdx.x == 0) {
      const int id = w ? 0x7fffffff - (int)(uint32_t)w : -1;  // w == 0: fewer than n_top columns
      p.ids[base + k] = id;
      p.lp[base + k] = id >= 0 ? (float)((double)(s_z[id] - mx) - lden) : __int_as_float(0x7fc00000);
    }
    if (mine == w && w) mine = top_scan(s_z, V, w);
  }
}

template __global__ void k_sample<false>(const SampleP p);
template __global__ void k_sample<true>(const SampleP p);

}  // namespace ctb
