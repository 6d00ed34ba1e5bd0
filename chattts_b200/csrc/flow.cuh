// Dataflow decode step for small batches (B <= 4):  k_flow<BT>
//
// Same arithmetic as k_step (mega.cuh) - input -> 20 x [QKV+RoPE+KV append -> attention -> O-proj -> gate/up -> down]
// -> heads - in ONE persistent cooperative kernel, but the two things that kept k_step at a quarter of the HBM
// roofline are gone:
//
//  * Weight stream decoupled from the phases.  Every warp owns a private ring of FL_SLOTS x 6 KiB shared-memory
//    slots filled by 1-D TMA bulk copies (cp.async.bulk + mbarrier complete_tx).  The warp's tasks for the whole step
//    (QKV pair, K/V chunk, O row, gate/up pairs, down slices, head pairs; all layers) form one static sequence;
//    after consuming task n the warp's lane 0 issues the copy of task n + FL_SLOTS into the slot it just freed.
//    Weights (and the K/V of earlier tokens) never depend on this step's activations, so every SM's 192 KiB are always
//    in flight across phase and layer boundaries and HBM streams while a CTA waits for its inputs.
//
//  * No grid barriers.  Activations cross CTAs as 8-byte {value, tag} words ("LL" protocol): the producer stores
//    value and tag with ONE 64-bit store, the consumer polls the data words themselves until the tag of this
//    (step, layer, phase) appears.  One L2 write + one L2 read per dependent edge - no release fence, no arrival
//    counter, no separate data load after an acquire.  Broadcast vectors are written to R replicas so that the
//    grid's readers of a vector do not queue on the same L2 slices.
//
// Arithmetic order per row is independent of the batch; results differ from k_step only by fp32 reassociation in
// the RMSNorm sum (per-lane strided instead of per-warp-row).
#pragma once
#include "gpt_kernels.cuh"
#include "tc_common.cuh"

namespace ctb {

constexpr int FL_THREADS = 256;
constexpr int FL_LAUNCH_THREADS = FL_THREADS;
constexpr int FL_WARPS = 8;
constexpr int FL_SLOTS = 4;
constexpr int FL_SLOT_BYTES = 6144;
constexpr int FL_SLOT_FLOATS = FL_SLOT_BYTES / 4;
constexpr int FL_RING_BYTES = FL_WARPS * FL_SLOTS * FL_SLOT_BYTES;  // 192 KiB
constexpr int FL_SMAX = 6;   // attention splits per (row, head); 12 was measured slower (365 vs 349 us/step: register spills, wider merge)
constexpr int FL_CH = 64;    // keys per attention chunk: 8 per warp
constexpr int FL_PW = 66;    // words of one attention partial: o[64], m, l
constexpr int FL_BMAX = 4;   // batch rows the exchange arena is sized for
constexpr int FL_ROWS = 6;   // O-proj / down rows per CTA: ceil(768 / grid) for grid >= 128
constexpr int FL_GU = 3;     // gate/up pair tasks per warp: ceil(3072 / (8 * grid)) for grid >= 128
constexpr int FL_QR = 2;     // QKV pair tasks per warp
constexpr int FL_HEADS = 12; // heads the arena is sized for
constexpr int FL_RMAX = 16;  // replicas the arena is sized for

// Exchange arena, in 8-byte words.  Two parity copies (layer l uses copy l & 1); per copy FL_RMAX replicas of the
// broadcast regions followed by the point-to-point q / k_new / v_new region.
constexpr int FL_A_X = 0;                                       // [BMAX][768]  residual stream entering a layer
constexpr int FL_A_XO = FL_A_X + FL_BMAX * KC;                  // [BMAX][768]  residual stream after O-proj
constexpr int FL_A_ACT = FL_A_XO + FL_BMAX * KC;                // [BMAX][3072] silu(gate) * up
constexpr int FL_A_P = FL_A_ACT + FL_BMAX * 4 * KC;             // [BMAX][12][SMAX][66] attention partials
constexpr int FL_A_END = FL_A_P + FL_BMAX * FL_HEADS * FL_SMAX * FL_PW;
constexpr int FL_REP_STRIDE = ((FL_A_END + 1023) / 1024) * 1024;
constexpr int FL_A_Q = 0, FL_A_KN = FL_BMAX * KC, FL_A_VN = 2 * FL_BMAX * KC;
constexpr int FL_QKV_WORDS = 3 * FL_BMAX * KC;
// in-kernel sampling (audio rows, V <= 1024): logits of the <= 16 (row, codebook) rows and the sampled ids
constexpr int FL_SROWS = 16, FL_VPAD = 1024;
constexpr int FL_A_LOGITS = FL_QKV_WORDS, FL_A_IDX = FL_A_LOGITS + FL_SROWS * FL_VPAD;
constexpr int FL_TAIL_WORDS = FL_A_IDX + 64;
constexpr size_t FL_PARITY_WORDS = (size_t)FL_RMAX * FL_REP_STRIDE + FL_TAIL_WORDS;
constexpr size_t FL_ARENA_WORDS = 2 * FL_PARITY_WORDS;
constexpr unsigned FL_EPOCH_STEP = 256;  // tags of one launch: base + 8 * layer + kind
// CTB_MEGA_TRACE buffer (words): CTA 0's phase stamps and cycle probes below FL_TR_EV, then FL_TR_EVN per-CTA event
// stamps of one layer for each of up to 192 CTAs (the grids k_flow runs on)
constexpr int FL_TR_EV = 4096, FL_TR_EVN = 32, FL_TR_WORDS = FL_TR_EV + 192 * FL_TR_EVN;

enum FlowTagKind { FT_X = 0, FT_QKV = 1, FT_P = 2, FT_XO = 3, FT_ACT = 4, FT_LOGITS = 5, FT_IDX = 6 };
enum FlowStage { FS_Q0 = 0, FS_Q1 = 1, FS_KV = 2, FS_O = 3, FS_GU0 = 4, FS_GU1 = 5, FS_GU2 = 6, FS_D0 = 7, FS_D1 = 8, FS_NLAYER = 9 };

// barrier among the 8 consumer warps only (the loader warp never joins it)
__device__ __forceinline__ void fl_bar() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

struct FlowP {
  const float* W;  // packed fp32 blob
  int64_t layer0, layer_stride, o_wqkv, o_wo, o_wgu, o_wd, o_ln1, o_ln2, o_final_norm, o_head, o_emb_code, o_emb_text,
      o_cos, o_sin;
  int L, I, Hq, hd;
  float eps, scaling;
  float *logits, *kv;
  size_t kv_layer_floats;
  const int* block_table; int pages_per_row;
  int* seq_len;
  LoopState* st;
  int decode, col, T0, sample;
  const float* emb; const uint8_t* mask; const int32_t* ids_out;
  int max_new, num_vq, num_audio, infer_text, B;
  float* hidden_out; int hidden_stride, rows_per_item, V;
  unsigned long long* arena;  // FL_ARENA_WORDS, zeroed at create
  unsigned* epoch;            // tag base of the next launch (advanced by CTA 0 at the end of every launch)
  int R;                      // replicas in use (1..FL_RMAX)
  int l2_ahead;               // 1: prefetch every weight task one layer ahead into L2 (CTB_FLOW_L2_AHEAD)
  unsigned long long* trace;  // optional globaltimer stamps of CTA 0 (1 + 5 * L + 1)
  // ---- multi-step mode (decode, audio): the sampling tail and the finish bookkeeping run inside the kernel
  int nsteps;                 // decode steps this launch runs (1 when ink == 0)
  int ink;                    // 1: sample in the kernel (k_sample / k_finalize are not launched)
  ctb_sampler_config samp;
  const float* q_noise;       // [rows][V] Exp(1) noise or nullptr (device Philox)
  uint8_t* finish;            // [B]
  int* end_idx;               // [B]
  int32_t* ids_w;             // ids_out, writable
};

// ---------------------------------------------------------------- LL words
// Stores are relaxed.gpu 64-bit (single-copy atomic: value and tag can never be seen torn).  Polls use ld.global.cg
// (L2-coherent, never served from L1): a probe inside the running kernel measured 280 cycles per dependent .cg load
// against 450 for ld.relaxed.gpu and 650 for ld.volatile, and the poll period is what an edge's latency is made of.
__device__ __forceinline__ void ll_st(unsigned long long* p, float v, uint32_t tag) {
  const unsigned long long x = ((unsigned long long)tag << 32) | (unsigned long long)__float_as_uint(v);
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(x) : "memory");
}
__device__ __forceinline__ unsigned long long ll_ld(const unsigned long long* p) {
  unsigned long long x;
  asm volatile("ld.global.cg.u64 %0, [%1];" : "=l"(x) : "l"(p) : "memory");
  return x;
}
__device__ __forceinline__ void ll_ld2(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
  asm volatile("ld.global.cg.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}
__device__ __forceinline__ uint32_t ll_tag(unsigned long long x) { return (uint32_t)(x >> 32); }
__device__ __forceinline__ float ll_val(unsigned long long x) { return __uint_as_float((uint32_t)x); }

// Watchdog: a wait that does not complete in ~2^20 polls records an error in LoopState::err and every later wait of
// the thread falls through, so a protocol bug ends the kernel in about a second instead of hanging the device.
struct FlowWd {
  int* err;
  int dead;
  int spins;
};
__device__ __forceinline__ bool fl_giveup(FlowWd& wd, int code) {
  if (wd.dead) return true;
  if (++wd.spins < (1 << 20)) {
    if ((wd.spins & 8191) == 0 && __ldcg(wd.err) != 0) { wd.dead = 1; return true; }
    return false;
  }
  atomicCAS(wd.err, 0, code);
  wd.dead = 1;
  return true;
}

__device__ __forceinline__ void fl_bulk(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst),
      "l"(src), "r"(bytes), "r"(bar), "l"(pol)
      : "memory");
}
// One elected lane of a converged warp (the pattern ptxas recognises: the guarded TMA instructions take their operands
// through plain R2UR instead of a per-lane waterfall loop, which `lane == 0` produced).
__device__ __forceinline__ bool fl_elect() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void fl_expect(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool fl_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}

// Geometry every thread of a CTA agrees on.  The CTA-uniform part sits in shared memory (read by the non-inlined
// issue routine); warp / lane / gw are recomputed from threadIdx where needed.
struct FlowGeo {
  int G, NW, gw, cta, warp, lane;
  int S;                                // attention splits per (row, head)
  int u_on, u_b, u_h, u_split, u_n, u_nchunk;  // this CTA's attention unit (u_on = 0: none / masked row)
  int nheads_tasks;                     // 2-row tasks of the heads phase (0: no heads in this launch)
};

// ---- task predicates shared by the issue side and the consume side (they MUST enumerate the same sequence)
__device__ __forceinline__ bool fl_q_valid(const FlowGeo& g, int j) { return g.gw + j * g.NW < 3 * KC / 2; }
__device__ __forceinline__ bool fl_kv_more(const FlowGeo& g, int sub, int& chunk) {
  chunk = g.u_split + sub * g.S;
  return g.u_on && chunk < g.u_nchunk;
}
__device__ __forceinline__ bool fl_kv_valid(const FlowGeo& g, int chunk) { return FL_CH * chunk + 8 * g.warp < g.u_n; }
__device__ __forceinline__ bool fl_o_valid(const FlowGeo& g) { return g.warp < FL_ROWS && g.cta + g.G * g.warp < KC; }
__device__ __forceinline__ bool fl_gu_valid(const FlowGeo& g, int j, int I) { return g.gw + j * g.NW < I; }
__device__ __forceinline__ int fl_d_rows(const FlowGeo& g, int j0, int j1) {
  int n = 0;
  for (int j = j0; j < j1; ++j) n += (g.cta + g.G * j < KC);
  return n;
}
__device__ __forceinline__ bool fl_h_valid(const FlowGeo& g, int j) { return g.gw + j * g.NW < g.nheads_tasks; }

__device__ __forceinline__ void fl_qkv_rows(const FlowP& p, int task, int& r0, int& r1) {
  const int half = p.hd / 2, nq = p.Hq * half;
  int t = task, base = 0;
  if (t >= 2 * nq) { t -= 2 * nq; base = 2 * p.Hq * p.hd; }
  else if (t >= nq) { t -= nq; base = p.Hq * p.hd; }
  r0 = base + (t / half) * p.hd + (t % half);
  r1 = r0 + half;
}

// Issue side.  The task sequence of a warp is the same in every layer (only the layer base moves), so it is tabulated
// once per launch in shared memory: entry = {offset of copy 0 (floats, relative to the layer's weight / KV base),
// stride between copies (floats), bytes per copy | ncopy << 16 | kind << 20}.  Issuing task n + FL_SLOTS after task n
// is then a table lookup - the first version recomputed the sequence position with ~200 dependent integer
// instructions per task and spent a quarter of the step there.
constexpr int FL_TMAX = 40;  // table entries per warp: 2 (QKV) + K/V chunks + 1 (O) + 3 (gate/up) + 2 (down)
struct FlowIss {
  int l, k, n, ntab, hsub;  // layer, entry within the layer, tasks issued so far, entries per layer, heads sub-iterator
};

// Build this warp's per-layer table (all lanes execute it uniformly; lane 0 stores).  Returns the entry count.
__device__ __noinline__ int fl_build_table(const FlowP& p, const FlowGeo* gs, int4* tab) {
  FlowGeo g = *gs;
  g.warp = threadIdx.x >> 5; g.lane = threadIdx.x & 31; g.gw = g.cta * FL_WARPS + g.warp;
  int n = 0;
  auto put = [&](int64_t off0, int64_t stride, int bytes, int ncopy, int kind) {
    if (g.lane == 0 && n < FL_TMAX) tab[n] = make_int4((int)off0, (int)stride, bytes | (ncopy << 16) | (kind << 20), 0);
    n++;
  };
  for (int j = 0; j < FL_QR; ++j)
    if (fl_q_valid(g, j)) {
      int r0, r1;
      fl_qkv_rows(p, g.gw + j * g.NW, r0, r1);
      put(p.o_wqkv + (int64_t)r0 * KC, (int64_t)(r1 - r0) * KC, KC * 4, 2, 0);
    }
  for (int sub = 0;; ++sub) {
    int chunk;
    if (!fl_kv_more(g, sub, chunk)) break;
    if (!fl_kv_valid(g, chunk)) continue;
    const int t0 = FL_CH * chunk + 8 * g.warp;
    const int page = __ldg(p.block_table + g.u_b * p.pages_per_row + t0 / kPageTokens);
    const int64_t k0 = (int64_t)kv_off(page, 0, g.u_h, t0 % kPageTokens, p.Hq, p.hd);
    const int64_t v0 = (int64_t)kv_off(page, 1, g.u_h, t0 % kPageTokens, p.Hq, p.hd);
    put(k0, v0 - k0, 8 * 64 * 4, 2, 1);
  }
  if (fl_o_valid(g)) put(p.o_wo + (int64_t)(g.cta + g.G * g.warp) * KC, 0, KC * 4, 1, 0);
  for (int j = 0; j < FL_GU; ++j)
    if (fl_gu_valid(g, j, p.I)) put(p.o_wgu + (int64_t)(g.gw + j * g.NW) * KC, (int64_t)p.I * KC, KC * 4, 2, 0);
  for (int half = 0; half < 2; ++half) {
    const int j0 = half ? 4 : 0, j1 = half ? FL_ROWS : 4;
    const int nr = fl_d_rows(g, j0, j1);
    if (nr > 0)
      put(p.o_wd + (int64_t)(g.cta + g.G * j0) * p.I + g.warp * (p.I / FL_WARPS), (int64_t)g.G * p.I, (p.I / FL_WARPS) * 4, nr, 0);
  }
  return n;
}

// heads tasks (after the last layer): rare, computed directly
__device__ __forceinline__ void fl_issue_heads(const FlowP& p, const FlowGeo* gs, int w, int hsub, uint32_t dst, uint32_t bar, uint64_t pol_w) {
  const int gw = gs->cta * FL_WARPS + w;
  const int t = gw + hsub * gs->NW, nrows = p.rows_per_item * p.V;
  if (fl_elect()) {
    fl_expect(bar, 2u * KC * 4u);
    fl_bulk(dst, p.W + p.o_head + (size_t)(2 * t) * KC, KC * 4, bar, pol_w);
    fl_bulk(dst + KC * 4, p.W + p.o_head + (size_t)min(2 * t + 1, nrows - 1) * KC, KC * 4, bar, pol_w);
  }
}

// Post the bulk copies of consumer warp w's next task into slot it.n % FL_SLOTS (one elected lane) and advance the
// iterator.  Returns false at the end of the step's sequence.
__device__ __forceinline__ bool fl_issue(const FlowP& p, const FlowGeo* gs, const int4* tab, FlowIss& it, int w, uint32_t ring,
                                         uint32_t bars, uint64_t pol_w, uint64_t pol_kv) {
  const int slot = it.n % FL_SLOTS;
  const uint32_t bar = bars + slot * 8, dst = ring + slot * FL_SLOT_BYTES;
  if (it.l < p.L) {
    const int4 e = tab[it.k];
    if (fl_elect()) {
      const int bytes = e.z & 0xffff, ncopy = (e.z >> 16) & 0xf, kind = e.z >> 20;
      const float* src = (kind ? p.kv + (size_t)it.l * p.kv_layer_floats : p.W + p.layer0 + (int64_t)it.l * p.layer_stride) + e.x;
      fl_expect(bar, (uint32_t)(bytes * ncopy));
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (k < ncopy) fl_bulk(dst + k * bytes, src + (int64_t)k * e.y, (uint32_t)bytes, bar, kind ? pol_kv : pol_w);
      if (p.l2_ahead && kind == 0) {
        // Two-level stream: the SAME task of the next layer (of layer 0 of the next step after the last one) is pulled
        // HBM -> L2 now, so that its shared-memory copy, posted a layer later, is an L2 hit.  A global load issued after
        // a bulk copy only returns after it: a copy that completes in ~0.3 us instead of a DRAM latency holds the polls
        // behind it that much less.  One layer of weights (37.75 MB) fits the H100's 50 MB L2 next to the exchange arena.
        const float* nsrc = it.l + 1 < p.L ? src + p.layer_stride : src - (int64_t)(p.L - 1) * p.layer_stride;
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (k < ncopy)
            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(nsrc + (int64_t)k * e.y), "r"((uint32_t)bytes) : "memory");
      }
    }
    if (++it.k == it.ntab) { it.k = 0; it.l++; }
    it.n++;
    return true;
  }
  if (gs->cta * FL_WARPS + w + it.hsub * gs->NW < gs->nheads_tasks) {
    fl_issue_heads(p, gs, w, it.hsub, dst, bar, pol_w);
    it.hsub++;
    it.n++;
    return true;
  }
  return false;
}

// Per-warp ring state.  The consuming warp refills a slot itself, right after the stores of the phase that emptied it.
// Two alternatives were built and found slower (tools/flow_check.py, B = 1, 256 tokens):
//   * lazy refills inside the poll loops (one per failed poll): a longer poll period;
//   * a loader warpgroup (4 warps posting every copy of the CTA, consumers only publish a counter, registers moved
//     with setmaxnreg): the X edge grew while the copies were posted concurrently with the polls.
struct FlowW {
  float* base;      // this warp's slots (generic pointer)
  uint32_t ring;    // same, shared-space address
  uint32_t bars;    // this warp's FL_SLOTS mbarriers
  int n;            // tasks consumed so far
  int owed;         // consumed slots not yet refilled
  FlowIss it;
  const int4* tab;
  const FlowGeo* gs;
  uint64_t pol_w, pol_kv;
};
__device__ __forceinline__ void fl_refill(const FlowP& p, FlowW& w) {
  if (w.owed > 0) {
    __syncwarp();  // every lane's reads of the slot are complete before the async proxy overwrites it
    fl_issue(p, w.gs, w.tab, w.it, (int)(threadIdx.x >> 5), w.ring, w.bars, w.pol_w, w.pol_kv);
    w.owed--;
  }
}
__device__ __forceinline__ const float* fl_ring_slot_at(const FlowW& w, int k) { return w.base + ((w.n + k) % FL_SLOTS) * FL_SLOT_FLOATS; }
// non-blocking look at tasks n .. n + cnt - 1: issued before a phase polls its inputs so that the try_wait latency
// (~200 cycles) overlaps the poll / RMSNorm; the blocking wait runs only if the tasks were not in yet
__device__ __forceinline__ bool fl_ring_peek_n(const FlowP& p, FlowW& w, int cnt) {
  while (w.owed > FL_SLOTS - cnt) fl_refill(p, w);
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 3; ++k)
    if (k < cnt) { const int n = w.n + k; ok = fl_try_wait(w.bars + (n % FL_SLOTS) * 8, (uint32_t)(n / FL_SLOTS) & 1u) && ok; }
  return ok;
}
// wait for tasks n .. n + cnt - 1 (cnt <= 3) with the try_waits in flight together
__device__ __forceinline__ void fl_ring_wait_n(const FlowP& p, FlowW& w, int cnt, FlowWd& wd) {
  while (w.owed > FL_SLOTS - cnt) fl_refill(p, w);
  uint32_t bar[3], par[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int n = w.n + k;
    bar[k] = w.bars + (n % FL_SLOTS) * 8;
    par[k] = (uint32_t)(n / FL_SLOTS) & 1u;
  }
  wd.spins = 0;
  while (true) {
    bool ok[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) ok[k] = k < cnt ? fl_try_wait(bar[k], par[k]) : true;
    if (ok[0] && ok[1] && ok[2]) break;
    if (__any_sync(0xffffffffu, fl_giveup(wd, 0x120))) { wd.dead = 1; break; }
  }
}
__device__ __forceinline__ const float* fl_ring_wait(const FlowP& p, FlowW& w, FlowWd& wd) {
  fl_ring_wait_n(p, w, 1, wd);
  return fl_ring_slot_at(w, 0);
}
// A consumed slot is refilled right after the stores of the phase that emptied it.  Posting the refills after the NEXT
// phase's inputs were detected (to keep them out of the way of the polls) was measured too: 412 us/step against 321.
__device__ __forceinline__ void fl_ring_release(const FlowP& p, FlowW& w) { w.n++; w.owed++; fl_refill(p, w); }
__device__ __forceinline__ void fl_refill_all(const FlowP& p, FlowW& w) {
  while (w.owed > 0) fl_refill(p, w);
}

// ---------------------------------------------------------------- phase helpers
// Poll p.B x 768 LL words into xs (raw), zero rows >= B, block barrier.
template <int BT>
__device__ __forceinline__ void fl_stage768(const FlowP& p, const unsigned long long* src, uint32_t tag, float* xs, FlowWd& wd, FlowW& fw) {
  const int tid = threadIdx.x;
  unsigned long long v[BT][3];
  wd.spins = 0;
  while (true) {
    bool ok = true;
#pragma unroll
    for (int b = 0; b < BT; ++b)
      if (b < p.B) {
#pragma unroll
        for (int k = 0; k < 3; ++k) v[b][k] = ll_ld(src + b * KC + tid + 256 * k);
      }
#pragma unroll
    for (int b = 0; b < BT; ++b)
      if (b < p.B) {
#pragma unroll
        for (int k = 0; k < 3; ++k) ok = ok && (ll_tag(v[b][k]) == tag);
      }
    if (__all_sync(0xffffffffu, ok)) break;
    if (__any_sync(0xffffffffu, fl_giveup(wd, 0x200 + (tag & 0xff)))) { wd.dead = 1; break; }
  }
#pragma unroll
  for (int b = 0; b < BT; ++b) {
#pragma unroll
    for (int k = 0; k < 3; ++k) xs[b * KC + tid + 256 * k] = b < p.B ? ll_val(v[b][k]) : 0.f;
  }
  fl_bar();
}

// Stage the attention output of the p.B rows into xs, merging the ns = min(chunks, S) split partials of every
// (row, head) with k_step's expressions in k_step's order (s = 0 .. ns-1): every CTA computes the same bits.  Rows
// without attention units (inactive prompt columns) get 0.  Block barrier at the end.
//
// The elements tid + 256 k (k < 3) of a warp belong to three heads, (warp >> 1) + 4 k, so every warp stages on its
// own.  The partials are 12 * ns * 66 words per row: spinning on all of them would load L2 several times as hard as
// staging 768 merged words.  Lane k * FL_SMAX + s spins on the {m, l} pair of split s of the warp's head k only; the
// merge weights go lane to lane by shuffles, and the o words are read once the pairs are in and re-read only if a
// tag is stale (they are stored by other producer threads than m / l, so every word is checked).
template <int BT>
__device__ __forceinline__ void fl_stage_attn(const FlowP& p, const unsigned long long* P, uint32_t tag, float* xs, FlowWd& wd, int S,
                                              const int* s_pos, const int* s_active) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int pk = lane / FL_SMAX, ps = lane % FL_SMAX, pbase = min(pk, 2) * FL_SMAX;
#pragma unroll 1
  for (int b = 0; b < BT; ++b) {
    if (b >= p.B) break;
    float v[3] = {0.f, 0.f, 0.f};
    if (s_active[b]) {
      const int ns = min((s_pos[b] + FL_CH) / FL_CH, S);
      const unsigned long long* Pb = P + (size_t)b * FL_HEADS * FL_SMAX * FL_PW + (size_t)(warp >> 1) * FL_SMAX * FL_PW;
      const bool pl = pk < 3 && ps < ns;
      float m = -INFINITY, lv = 0.f;
      wd.spins = 0;
      while (true) {
        bool ok = true;
        if (pl) {
          unsigned long long w1, w2;
          ll_ld2(Pb + (size_t)(4 * pk * FL_SMAX + ps) * FL_PW + 64, w1, w2);
          ok = ll_tag(w1) == tag && ll_tag(w2) == tag;
          m = ll_val(w1); lv = ll_val(w2);
        }
        if (__all_sync(0xffffffffu, ok)) break;
        if (__any_sync(0xffffffffu, fl_giveup(wd, 0x400))) { wd.dead = 1; break; }
      }
      float GM = -INFINITY;  // of this lane's head
#pragma unroll
      for (int s = 0; s < FL_SMAX; ++s) {
        const float ms = __shfl_sync(0xffffffffu, m, pbase + s);
        if (s < ns) GM = fmaxf(GM, ms);
      }
      const float wgt = pl ? expf(m - GM) : 0.f;
      unsigned long long w[3][FL_SMAX];
      while (true) {
        bool ok = true;
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
          for (int s = 0; s < FL_SMAX; ++s)
            if (s < ns) w[k][s] = ll_ld(Pb + (size_t)(4 * k * FL_SMAX + s) * FL_PW + (tid & 63));
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
          for (int s = 0; s < FL_SMAX; ++s)
            if (s < ns) ok = ok && ll_tag(w[k][s]) == tag;
        if (__all_sync(0xffffffffu, ok)) break;
        if (__any_sync(0xffffffffu, fl_giveup(wd, 0x401))) { wd.dead = 1; break; }
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        float GL = 0.f, GO = 0.f;
#pragma unroll
        for (int s = 0; s < FL_SMAX; ++s) {
          const float ws = __shfl_sync(0xffffffffu, wgt, k * FL_SMAX + s);
          const float ls = __shfl_sync(0xffffffffu, lv, k * FL_SMAX + s);
          if (s < ns) {
            GL = fmaf(ws, ls, GL);
            GO = fmaf(ws, ll_val(w[k][s]), GO);
          }
        }
        v[k] = GO / GL;
      }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) xs[b * KC + tid + 256 * k] = v[k];
  }
#pragma unroll
  for (int b = 0; b < BT; ++b)
    if (b >= p.B)
      for (int k = 0; k < 3; ++k) xs[b * KC + tid + 256 * k] = 0.f;
  fl_bar();
}

template <int BT>
__device__ __forceinline__ void fl_load_x(const float* xs, float (&x)[BT][24], int lane) {
#pragma unroll
  for (int b = 0; b < BT; ++b) {
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      const float4 v = reinterpret_cast<const float4*>(xs)[b * (KC / 4) + i * 32 + lane];
      x[b][4 * i] = v.x; x[b][4 * i + 1] = v.y; x[b][4 * i + 2] = v.z; x[b][4 * i + 3] = v.w;
    }
  }
}

// HF LlamaRMSNorm on the register copy: w * (x * rsqrt(mean(x^2) + eps)); every warp computes the same sum.
template <int BT>
__device__ __forceinline__ void fl_norm(float (&x)[BT][24], const float4 (&nw)[6], float eps) {
#pragma unroll
  for (int b = 0; b < BT; ++b) {
    float s4[4] = {0.f, 0.f, 0.f, 0.f};  // four interleaved partial sums: 6-deep dependent chains instead of 24
#pragma unroll
    for (int j = 0; j < 24; ++j) s4[j & 3] = fmaf(x[b][j], x[b][j], s4[j & 3]);
    float ss = warp_sum((s4[0] + s4[1]) + (s4[2] + s4[3]));
    const float rinv = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fdiv_rn(ss, (float)KC), eps)));
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      x[b][4 * i] = __fmul_rn(nw[i].x, __fmul_rn(x[b][4 * i], rinv));
      x[b][4 * i + 1] = __fmul_rn(nw[i].y, __fmul_rn(x[b][4 * i + 1], rinv));
      x[b][4 * i + 2] = __fmul_rn(nw[i].z, __fmul_rn(x[b][4 * i + 2], rinv));
      x[b][4 * i + 3] = __fmul_rn(nw[i].w, __fmul_rn(x[b][4 * i + 3], rinv));
    }
  }
}
// Norm weights come from HBM (they are part of the streamed blob) and the L1 returns loads in issue order: a register
// load of them right before a poll made every X / XO edge wait for a DRAM round trip.  They are now fetched into shared
// memory with cp.async half a layer ahead; this waits for the thread's own copies (the phase's barrier publishes them).
// (The first version used cp.async, i.e. the LSU: its DRAM round trip then sat IN FRONT of the next phase's polls in the
// L1's in-order return queue.)  One elected thread posts a 3 KiB bulk copy on a dedicated mbarrier; every consumer thread
// waits for the barrier phase of the fetch it needs.
__device__ __forceinline__ void fl_nw_fetch(float* dst, const float* src, uint64_t* bar, uint64_t pol) {
  if (threadIdx.x == 0) {
    fl_expect(smem_u32(bar), KC * 4);
    fl_bulk(smem_u32(dst), src, KC * 4, smem_u32(bar), pol);
  }
}
__device__ __forceinline__ void fl_nw_wait(uint64_t* bar, int& count, FlowWd& wd) {
  const uint32_t b = smem_u32(bar), parity = (uint32_t)count & 1u;
  wd.spins = 0;
  while (!fl_try_wait(b, parity))
    if (__any_sync(0xffffffffu, fl_giveup(wd, 0x800))) { wd.dead = 1; break; }
  count++;
}
__device__ __forceinline__ void fl_load_nw_s(const float* s_nw, float4 (&nw)[6], int lane) {
#pragma unroll
  for (int i = 0; i < 6; ++i) nw[i] = reinterpret_cast<const float4*>(s_nw)[i * 32 + lane];
}
__device__ __forceinline__ void fl_load_nw(const float* normw, float4 (&nw)[6], int lane) {
#pragma unroll
  for (int i = 0; i < 6; ++i) nw[i] = ldg_stream(reinterpret_cast<const float4*>(normw) + i * 32 + lane);
}

// two weight rows (slot + 0, slot + 768 floats) against BT activation rows; k order as k_gemv
template <int BT>
__device__ __forceinline__ void fl_dot2(const float* slot, const float (&x)[BT][24], float (&a0)[BT], float (&a1)[BT], int lane) {
  const float4* w0 = reinterpret_cast<const float4*>(slot) + lane;
  const float4* w1 = w0 + KC / 4;
#pragma unroll
  for (int b = 0; b < BT; ++b) { a0[b] = 0.f; a1[b] = 0.f; }
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    const float4 u = w0[i * 32], v = w1[i * 32];
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      a0[b] = fmaf(u.x, x[b][4 * i], a0[b]); a0[b] = fmaf(u.y, x[b][4 * i + 1], a0[b]);
      a0[b] = fmaf(u.z, x[b][4 * i + 2], a0[b]); a0[b] = fmaf(u.w, x[b][4 * i + 3], a0[b]);
      a1[b] = fmaf(v.x, x[b][4 * i], a1[b]); a1[b] = fmaf(v.y, x[b][4 * i + 1], a1[b]);
      a1[b] = fmaf(v.z, x[b][4 * i + 2], a1[b]); a1[b] = fmaf(v.w, x[b][4 * i + 3], a1[b]);
    }
  }
}
template <int BT>
__device__ __forceinline__ void fl_dot1(const float* slot, const float (&x)[BT][24], float (&a0)[BT], int lane) {
  const float4* w0 = reinterpret_cast<const float4*>(slot) + lane;
#pragma unroll
  for (int b = 0; b < BT; ++b) a0[b] = 0.f;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    const float4 u = w0[i * 32];
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      a0[b] = fmaf(u.x, x[b][4 * i], a0[b]); a0[b] = fmaf(u.y, x[b][4 * i + 1], a0[b]);
      a0[b] = fmaf(u.z, x[b][4 * i + 2], a0[b]); a0[b] = fmaf(u.w, x[b][4 * i + 3], a0[b]);
    }
  }
}

// Value v of batch row b lives in lane b * LPB: write it to word `idx` of every replica (LPB lanes share the work).
template <int BT>
__device__ __forceinline__ void fl_bcast_store(unsigned long long* rep0, int R, size_t idx, float v, uint32_t tag, int nb, int lane) {
  constexpr int LPB = 32 / BT;
  const float vb = __shfl_sync(0xffffffffu, v, (lane / LPB) * LPB);
  if (lane / LPB < nb)
    for (int r = lane % LPB; r < R; r += LPB) ll_st(rep0 + (size_t)r * FL_REP_STRIDE + idx, vb, tag);
}

// ---------------------------------------------------------------- in-kernel sampling tail (V <= 1024)
// k_sample's arithmetic with 256 threads: thread t plays the virtual threads t, t + 256, t + 512, t + 768 of the
// 1024-thread kernel (virtual warp = warp + 8k, same lane) and every double-precision sum runs over the virtual warps
// in k_sample's order, so the sampled index is bit for bit the one k_sample returns (sampler.cu:63-268).
struct __align__(16) FlowSamp {
  float x[FL_VPAD];
  uint32_t key[2][1024];
  double redd[32];
  double pre[32];
  int redi[8];
  float redf[8];
  float bv[8];
  int bi[8];
  int win[32];
  uint32_t thr;
  int out;
};
__device__ __forceinline__ double fl_vsum_d(const double (&v)[4], double* redd) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double r[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) r[k] = warp_sum_d(v[k]);
  fl_bar();
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) redd[warp + 8 * k] = r[k];
  }
  fl_bar();
  double t = 0.0;
#pragma unroll 8
  for (int w = 0; w < 32; ++w) t += redd[w];  // fixed order => deterministic
  return t;
}
__device__ __forceinline__ float fl_bmax(float v, float* redf) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_max(v);
  fl_bar();
  if (lane == 0) redf[warp] = v;
  fl_bar();
  float t = -INFINITY;
#pragma unroll
  for (int w = 0; w < FL_WARPS; ++w) t = fmaxf(t, redf[w]);
  return t;
}
__device__ __forceinline__ int fl_bsum_i(int v, int* redi) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = __reduce_add_sync(0xffffffffu, v);
  fl_bar();
  if (lane == 0) redi[warp] = v;
  fl_bar();
  int t = 0;
#pragma unroll
  for (int w = 0; w < FL_WARPS; ++w) t += redi[w];
  return t;
}
// Bitonic sort of 1024 keys.  Thread t holds the keys of positions 4t .. 4t+3: compare-exchange distances 1 and 2
// stay in registers, 4 .. 64 are warp shuffles, only the six stages with distance >= 128 go through shared memory.
// On return key[e] is the key of sorted position 4 * tid + e (ascending).
__device__ __forceinline__ void fl_cx(uint32_t& a, uint32_t& b, bool up) {
  const uint32_t lo = min(a, b), hi = max(a, b);
  a = up ? lo : hi; b = up ? hi : lo;
}
__device__ __forceinline__ void fl_bitonic1024(uint32_t (&key)[4], uint32_t* buf0, uint32_t* buf1) {
  const int tid = threadIdx.x;
  int sb = 0;
#pragma unroll 1
  for (int k = 2; k <= 1024; k <<= 1) {
#pragma unroll 1
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (j == 1) {
        fl_cx(key[0], key[1], ((4 * tid) & k) == 0);
        fl_cx(key[2], key[3], ((4 * tid + 2) & k) == 0);
      } else if (j == 2) {
        fl_cx(key[0], key[2], ((4 * tid) & k) == 0);
        fl_cx(key[1], key[3], ((4 * tid + 1) & k) == 0);
      } else {
        const int d = j >> 2;  // partner thread distance
        uint32_t other[4];
        if (d >= 32) {
          uint32_t* buf = sb ? buf1 : buf0;
          *reinterpret_cast<uint4*>(buf + 4 * tid) = make_uint4(key[0], key[1], key[2], key[3]);
          fl_bar();
          const uint4 o = *reinterpret_cast<const uint4*>(buf + 4 * (tid ^ d));
          other[0] = o.x; other[1] = o.y; other[2] = o.z; other[3] = o.w;
          sb ^= 1;
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e) other[e] = __shfl_xor_sync(0xffffffffu, key[e], d);
        }
        const bool up = ((4 * tid) & k) == 0, lower = (tid & d) == 0;
#pragma unroll
        for (int e = 0; e < 4; ++e) key[e] = (lower == up) ? min(key[e], other[e]) : max(key[e], other[e]);
      }
    }
  }
}

// One logits row: sm.x[0..V) raw logits, sm.win[0..nwin) the repetition window.  Returns the sampled id (all threads).
__device__ __noinline__ int fl_sample_row(const ctb_sampler_config& c, const float* q_noise, FlowSamp& sm, int V, int row, int qi,
                                          int nwin, int step, unsigned long long* dbg) {
  int dk = 0;
#define FL_SK() do { if (dbg && threadIdx.x == 0) dbg[dk++] = (unsigned long long)clock64(); } while (0)
  FL_SK();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool pen = c.penalty_on && row < c.penalty_max_ids;
  const float temp = c.temperature[qi];
  float qn[4];  // Exp(1) noise of this thread's elements, requested now and used by the final arg-max
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int v = tid + 256 * k;
    qn[k] = (q_noise != nullptr && v < V) ? __ldg(q_noise + (size_t)row * V + v) : 1.f;
  }
  {
    float xr[4];
    int cnt[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 4; ++k) { const int v = tid + 256 * k; xr[k] = v < V ? __fdiv_rn(sm.x[v], temp) : 0.f; }
    if (pen) {
#pragma unroll 4
      for (int w = 0; w < nwin; ++w) {
        const int id = sm.win[w];
#pragma unroll
        for (int k = 0; k < 4; ++k) cnt[k] += (id == tid + 256 * k);
      }
    }
    fl_bar();  // every raw logit has been read
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int v = tid + 256 * k;
      if (v < V) {
        float x = xr[k];
        if (pen) { const float a = c.penalty_lut[cnt[k]]; x = (x < 0.f) ? __fmul_rn(x, a) : __fdiv_rn(x, a); }
        sm.x[v] = x;
      }
    }
  }
  fl_bar();
  float mx = -INFINITY;
  for (int v = tid; v < V; v += FL_THREADS) mx = fmaxf(mx, sm.x[v]);
  mx = fl_bmax(mx, sm.redf);
  FL_SK();

  // as k_sample: top_k taken as given (its warper's min_tokens_to_keep is already in it), and each cut is a key
  // threshold, so a tie group at the top-p or top-k cut is kept whole
  const bool use_p = c.top_p >= 0.f;
  const int kk = c.top_k > 0 ? min(c.top_k, V) : 0;
  const int min_keep = min(c.min_tokens_to_keep, V);
  uint32_t thr_key = 0;
  // greedy replaces thr_key by the arg-max key below, so the top-p / top-k threshold is dead work there (uniform branch)
  if (!c.greedy && (use_p || kk > 0)) {
    double den = 0.0;
    if (use_p) {
      double dv[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) { const int vt = tid + 256 * k; dv[k] = vt < V ? (double)expf(sm.x[vt] - mx) : 0.0; }
      den = fl_vsum_d(dv, sm.redd);
    }
    FL_SK();
    const float denf = (float)den;
    const float pthr = c.has_removed_max ? c.top_p_removed_max : (float)(1.0 - (double)c.top_p);
    uint32_t key[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { const int vt = tid + 256 * k; key[k] = vt < V ? float_key(sm.x[vt]) : 0u; }
    fl_bitonic1024(key, sm.key[0], sm.key[1]);
    FL_SK();
    fl_bar();
    uint32_t* skey = sm.key[0];
    *reinterpret_cast<uint4*>(skey + 4 * tid) = make_uint4(key[0], key[1], key[2], key[3]);  // sorted position 4 tid + e
    fl_bar();
#pragma unroll
    for (int k = 0; k < 4; ++k) key[k] = skey[tid + 256 * k];  // back to k_sample's one-key-per-virtual-thread view
    uint32_t t_p = 0;
    if (use_p) {
      double inc[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t ky = key[k];
        double a = ky ? (double)__fdiv_rn(expf(key_float(ky) - mx), denf) : 0.0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const double n = __shfl_up_sync(0xffffffffu, a, o);
          if (lane >= o) a += n;
        }
        inc[k] = a;
      }
      fl_bar();
      if (lane == 31) {
#pragma unroll
        for (int k = 0; k < 4; ++k) sm.redd[warp + 8 * k] = inc[k];
      }
      fl_bar();
      if (tid == 0) {  // exclusive prefix over the 32 virtual warps, added in k_sample's order (w = 0, 1, ...)
        double run = 0.0;
        for (int w = 0; w < 32; ++w) { const double t = sm.redd[w]; sm.pre[w] = run; run += t; }
      }
      fl_bar();
      int removed = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int vw = warp + 8 * k, vt = tid + 256 * k;
        const double base = sm.pre[vw];
        const float cum = (float)(base + inc[k]);
        removed += ((cum <= pthr) && (vt < 1024 - min_keep)) ? 1 : 0;
      }
      const int nrem = fl_bsum_i(removed, sm.redi);  // the removed set is a prefix of the sorted row
      t_p = skey[nrem];
      FL_SK();
    }
    const uint32_t t_k = kk > 0 ? skey[1024 - kk] : 0u;
    thr_key = max(t_p, t_k);
  }
  if (c.greedy) {
    float gm = -INFINITY;
    for (int v = tid; v < V; v += FL_THREADS)
      if (!(c.greedy == 2 && v == c.eos_token)) gm = fmaxf(gm, sm.x[v]);
    gm = fl_bmax(gm, sm.redf);
    thr_key = float_key(gm);
  }
  fl_bar();  // every read of sm.key / sm.x above is complete
  const bool ban = step < c.min_new_token;
  float mx2 = -INFINITY;
  for (int v = tid; v < V; v += FL_THREADS) {
    float x = sm.x[v];
    if (float_key(x) < thr_key || ((ban || c.greedy == 2) && v == c.eos_token)) x = -INFINITY;
    sm.x[v] = x;
    mx2 = fmaxf(mx2, x);
  }
  mx2 = fl_bmax(mx2, sm.redf);
  double dv2[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) { const int vt = tid + 256 * k; dv2[k] = vt < V ? (double)expf(sm.x[vt] - mx2) : 0.0; }
  const float den2f = (float)fl_vsum_d(dv2, sm.redd);
  FL_SK();
  float best = -1.f;
  int besti = 0x7fffffff;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int v = tid + 256 * k;
    if (v < V) {
      const float pr = __fdiv_rn(expf(sm.x[v] - mx2), den2f);
      const float qv = q_noise ? qn[k] : philox_exp1(c.philox_seed, (uint32_t)row, (uint32_t)v, (uint32_t)step);
      const float r = __fdiv_rn(pr, qv);
      if (r > best) { best = r; besti = v; }  // ascending v within a thread: first max wins
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
    if (ob > best || (ob == best && oi < besti)) { best = ob; besti = oi; }
  }
  fl_bar();
  if (lane == 0) { sm.bv[warp] = best; sm.bi[warp] = besti; }
  fl_bar();
  if (tid == 0) {
    for (int w = 1; w < FL_WARPS; ++w)
      if (sm.bv[w] > best || (sm.bv[w] == best && sm.bi[w] < besti)) { best = sm.bv[w]; besti = sm.bi[w]; }
    sm.out = besti < V ? besti : 0;  // all-NaN row: ATen argmax returns the first index
  }
  fl_bar();
  FL_SK();
#undef FL_SK
  return sm.out;
}

template <int BT>
__global__ void __launch_bounds__(FL_THREADS, 1) k_flow(const __grid_constant__ FlowP p) {
  extern __shared__ __align__(128) unsigned char fl_smem[];
  float* xs = reinterpret_cast<float*>(fl_smem + FL_RING_BYTES);  // [BT][768]
  __shared__ __align__(8) uint64_t s_bar[FL_WARPS * FL_SLOTS];
  __shared__ __align__(8) uint64_t s_nwbar[2];  // norm-weight fetches (attention half, MLP half)
  __shared__ int s_pos[BT], s_active[BT], s_page[BT];
  __shared__ float s_cos[BT * 64], s_sin[BT * 64];
  __shared__ float s_red[FL_ROWS][FL_WARPS][BT];
  __shared__ float s_resd[FL_ROWS * BT];
  __shared__ float s_am[FL_WARPS], s_al[FL_WARPS];
  __shared__ __align__(16) float s_ao[FL_WARPS][64];
  __shared__ FlowGeo s_geo;
  __shared__ __align__(16) float s_nw1[KC], s_nw2[KC];  // RMSNorm weights of the coming attention / MLP half, fetched a phase early
  __shared__ int4 s_tab[FL_WARPS][FL_TMAX];
  __shared__ FlowSamp s_samp_store[BT <= 2 ? 1 : 0 + (BT > 2)];
  FlowSamp& s_samp = s_samp_store[0];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int LPB = 32 / BT;
  if (tid < FL_WARPS * FL_SLOTS) mbar_init(&s_bar[tid], 1);
  if (tid < 2) mbar_init(&s_nwbar[tid], 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  pdl_trigger();
  pdl_wait();
  if (p.decode && ldg_cg(&p.st->all_finished)) return;  // uniform over the grid; nothing has been issued yet

  constexpr bool INK = BT <= 2;  // in-kernel sampling is built for the batches this kernel is the default for
  __shared__ int s_ids[BT * 8];       // ids sampled by the previous step (multi-step mode)
  __shared__ int s_fin[BT], s_end[BT];
  __shared__ int s_allfin;
  FlowWd wd{&p.st->err, 0, 0};
  uint32_t base = (uint32_t)ldg_cg(reinterpret_cast<const int*>(p.epoch));
  int tr = 0;
#define FL_TRACE() do { if (p.trace && blockIdx.x == 0 && tid == 0 && tr < 250) p.trace[tr++] = globaltimer_ns(); } while (0)
  // per-CTA event stamps of one layer (profiling aid; trace[FL_TR_EV + cta * FL_TR_EVN + k], read by tools/flow_trace.py)
#define FL_EV(k) do { if (p.trace && l == 10 && tid == 0) p.trace[FL_TR_EV + blockIdx.x * FL_TR_EVN + (k)] = globaltimer_ns(); } while (0)
  // cycle stamps inside the gate/up phase of CTA 0 / warp 0 (profiling aid; trace[3000 + k])
#define FL_CK(k) do { if (p.trace && l == 10 && tid == 0 && blockIdx.x == 0) p.trace[3000 + (k)] = (unsigned long long)clock64(); } while (0)

  // ---- loop state of this launch
  int ngen = p.decode ? ldg_cg(&p.st->n_gen) : 0;   // tokens appended to ids_out so far
  int lstep = p.decode ? ldg_cg(&p.st->step) : 0;   // loop iterations completed (gpt.py: i)
  if (tid < BT) {
    int act = 0, pos = 0;
    if (tid < p.B) {
      pos = ldg_cg(&p.seq_len[tid]);
      act = p.decode ? 1 : (p.mask[(size_t)tid * p.T0 + p.col] != 0);
    }
    s_pos[tid] = pos; s_active[tid] = act;
    s_fin[tid] = (tid < p.B && p.ink) ? (int)p.finish[tid] : 0;
    s_end[tid] = (tid < p.B && p.ink) ? ldg_cg(&p.end_idx[tid]) : 0;
  }
  const bool ink = INK && p.ink != 0;
  const int nrows_s = p.B * p.rows_per_item;           // sampler rows (one CTA each)
  const int R = p.R;
  uint64_t pol_w, pol_kv;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_w));
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol_kv));
  int nw1_cnt = 0, nw2_cnt = 0;  // completed waits on the two norm-weight barriers (their phase parity)
  FlowW fw;
  fw.base = reinterpret_cast<float*>(fl_smem) + (size_t)warp * FL_SLOTS * FL_SLOT_FLOATS;
  fw.ring = smem_u32(fw.base);
  fw.bars = smem_u32(&s_bar[warp * FL_SLOTS]);
  fw.n = 0; fw.owed = 0;
  fw.it = FlowIss{0, 0, 0, 0, 0};
  fw.tab = s_tab[warp]; fw.gs = &s_geo; fw.pol_w = pol_w; fw.pol_kv = pol_kv;
  FlowGeo g;
  g.G = gridDim.x; g.NW = g.G * FL_WARPS; g.cta = blockIdx.x; g.warp = warp; g.lane = lane; g.gw = g.cta * FL_WARPS + warp;
  g.S = max(1, min(FL_SMAX, g.G / (p.Hq * p.B)));
  g.nheads_tasks = p.sample ? (p.rows_per_item * p.V + 1) / 2 : 0;
  const int myrep = g.cta % R;
  const int o_row = g.cta + g.G * warp;  // this warp's O-proj row (valid iff fl_o_valid)
  unsigned long long* tailw = p.arena + (size_t)FL_RMAX * FL_REP_STRIDE;  // parity-0 tail: q/k/v words, logits, ids
  fl_bar();

  // the repetition window of this CTA's sampler row: the last <= past_window ids of (item, codebook)
  int nwin = 0;
  if constexpr (INK) {
    if (ink && g.cta < nrows_s) {
      const int item = g.cta / p.rows_per_item, qi = g.cta % p.rows_per_item;
      const bool pen = p.samp.penalty_on && g.cta < p.samp.penalty_max_ids;
      nwin = pen ? min(ngen, p.samp.past_window) : 0;
      if (tid < nwin) s_samp.win[tid] = ldg_cg(&p.ids_out[((size_t)item * p.max_new + (ngen - nwin + tid)) * p.num_vq + qi]);
    }
  }

  // ---- pages / unit geometry / task table of a step's positions, first FL_SLOTS tasks posted (k_input).  Used before
  // the loop and, for the NEXT step, before the sampling tail: the ring is idle then and the weights of layer 0 are in
  // shared memory by the time the sampled ids arrive.
#define FL_PREP_STEP()                                                                                                  \
  do {                                                                                                                  \
    if (tid < BT) s_page[tid] = tid < p.B ? __ldg(p.block_table + tid * p.pages_per_row + s_pos[tid] / kPageTokens) : 0; \
    {                                                                                                                   \
      const int u = g.cta;                                                                                              \
      g.u_on = 0; g.u_b = 0; g.u_h = 0; g.u_split = 0; g.u_n = 0; g.u_nchunk = 0;                                       \
      if (u < p.B * p.Hq * g.S) {                                                                                       \
        g.u_split = u % g.S; g.u_h = (u / g.S) % p.Hq; g.u_b = u / (g.S * p.Hq);                                        \
        g.u_n = s_pos[g.u_b] + 1;                                                                                       \
        g.u_nchunk = (g.u_n + FL_CH - 1) / FL_CH;                                                                       \
        g.u_on = s_active[g.u_b] && g.u_split < min(g.u_nchunk, g.S);                                                   \
      }                                                                                                                 \
    }                                                                                                                   \
    if (tid == 0) s_geo = g;                                                                                            \
    fl_bar();                                                                                                           \
    fw.it.l = 0; fw.it.k = 0; fw.it.hsub = 0; fw.owed = 0;                                                              \
    fw.it.ntab = fl_build_table(p, &s_geo, s_tab[warp]);                                                                \
    __syncwarp();                                                                                                       \
    for (int k_ = 0; k_ < FL_SLOTS; ++k_) fl_issue(p, fw.gs, fw.tab, fw.it, warp, fw.ring, fw.bars, pol_w, pol_kv);     \
    for (int i = tid; i < BT * 64; i += FL_THREADS) {                                                                   \
      const int b = i / 64;                                                                                             \
      s_cos[i] = b < p.B ? __ldg(p.W + p.o_cos + (size_t)s_pos[b] * 64 + (i % 64)) : 0.f;                               \
      s_sin[i] = b < p.B ? __ldg(p.W + p.o_sin + (size_t)s_pos[b] * 64 + (i % 64)) : 0.f;                               \
    }                                                                                                                   \
  } while (0)

  FL_PREP_STEP();
  FL_TRACE();
#pragma unroll 1
  for (int sidx = 0;; ++sidx) {
  // ======================================================================== one decode step
  FL_TRACE();
  fl_nw_fetch(s_nw1, p.W + p.layer0 + p.o_ln1, &s_nwbar[0], pol_w);
  fl_nw_fetch(s_nw2, p.W + p.layer0 + p.o_ln2, &s_nwbar[1], pol_w);
  {  // step input: prompt column or sum of the code embeddings; every load of the thread in flight together
    float ev[BT * 3][8];
#pragma unroll
    for (int it_ = 0; it_ < BT * 3; ++it_) {
      const int i = tid + it_ * FL_THREADS, b = i / KC, k = i % KC;
#pragma unroll
      for (int q = 0; q < 8; ++q) ev[it_][q] = 0.f;
      if (b < p.B) {
        if (!p.decode) {
          ev[it_][0] = s_active[b] ? p.emb[((size_t)b * p.T0 + p.col) * KC + k] : 0.f;
        } else if (p.infer_text) {
          const int id0 = ldg_cg(p.ids_out + ((size_t)b * p.max_new + (ngen - 1)) * p.num_vq);
          ev[it_][0] = p.W[p.o_emb_text + (size_t)id0 * KC + k];
        } else {
#pragma unroll
          for (int q = 0; q < 8; ++q)
            if (q < p.num_vq) {
              const int id = sidx > 0 ? s_ids[b * 8 + q] : ldg_cg(p.ids_out + ((size_t)b * p.max_new + (ngen - 1)) * p.num_vq + q);
              ev[it_][q] = p.W[p.o_emb_code + ((size_t)q * p.num_audio + id) * KC + k];
            }
        }
      }
    }
#pragma unroll
    for (int it_ = 0; it_ < BT * 3; ++it_) {
      float v = 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q) v += ev[it_][q];   // q order as Embed.forward: 0 + e0 + e1 + ...
      xs[tid + it_ * FL_THREADS] = v;
    }
  }
  fl_bar();
  FL_TRACE();

  for (int l = 0; l < p.L; ++l) {
    const float* Wl = p.W + p.layer0 + (int64_t)l * p.layer_stride;
    unsigned long long* par = p.arena + (size_t)(l & 1) * FL_PARITY_WORDS;
    unsigned long long* parn = p.arena + (size_t)((l + 1) & 1) * FL_PARITY_WORDS;
    unsigned long long* qkvw = par + (size_t)FL_RMAX * FL_REP_STRIDE;  // FL_A_Q / KN / VN at the start of the tail
    const unsigned long long* myr = par + (size_t)myrep * FL_REP_STRIDE;
    const uint32_t tagl = base + 8u * (uint32_t)l;

    // ============ A: QKV + RoPE + KV append ============
    {
      float4 nw[6];
      FL_EV(0);
      fl_nw_wait(&s_nwbar[0], nw1_cnt, wd);
      const bool q_rdy = fl_ring_peek_n(p, fw, 1);
      if (l > 0) fl_stage768<BT>(p, myr + FL_A_X, tagl + FT_X, xs, wd, fw);
      else fl_bar();
      FL_EV(1);
      fl_refill_all(p, fw);
      fl_load_nw_s(s_nw1, nw, lane);
      float x[BT][24];
      fl_load_x<BT>(xs, x, lane);
      // residual of this warp's O-proj row (raw x), kept for phase C
      float res_o = 0.f;
      if (fl_o_valid(g)) res_o = xs[(lane / LPB) * KC + o_row];
      fl_norm<BT>(x, nw, p.eps);
      float res_keep = res_o;
#pragma unroll 1
      for (int j = 0; j < FL_QR; ++j) {
        if (!fl_q_valid(g, j)) continue;
        if (!(j == 0 && q_rdy)) fl_ring_wait_n(p, fw, 1, wd);
        const float* slot = fl_ring_slot_at(fw, 0);
        FL_EV(2);
        float a0[BT], a1[BT];
        fl_dot2<BT>(slot, x, a0, a1, lane);
        warp_reduce_scatter<BT>(a0);
        warp_reduce_scatter<BT>(a1);
        const int b = lane / LPB;
        if ((lane % LPB) == 0 && b < p.B && s_active[b]) {
          const int half = p.hd / 2, nq = p.Hq * half;
          int t = g.gw + j * g.NW, which = 0;
          if (t >= 2 * nq) { which = 2; t -= 2 * nq; }
          else if (t >= nq) { which = 1; t -= nq; }
          const int h = t / half, jj = t % half;
          const float v0 = a0[0], v1 = a1[0];
          float o0 = v0, o1 = v1;
          if (which < 2) {
            const float* cs = s_cos + b * 64;
            const float* sn = s_sin + b * 64;
            o0 = __fadd_rn(__fmul_rn(v0, cs[jj]), __fmul_rn(-v1, sn[jj]));
            o1 = __fadd_rn(__fmul_rn(v1, cs[jj + half]), __fmul_rn(v0, sn[jj + half]));
          }
          unsigned long long* dst = qkvw + (which == 0 ? FL_A_Q : which == 1 ? FL_A_KN : FL_A_VN) + b * KC + h * 64;
          ll_st(dst + jj, o0, tagl + FT_QKV);
          ll_st(dst + jj + half, o1, tagl + FT_QKV);
          if (which > 0) {
            float* kd = p.kv + (size_t)l * p.kv_layer_floats + kv_off(s_page[b], which - 1, h, s_pos[b] % kPageTokens, p.Hq, p.hd);
            kd[jj] = o0; kd[jj + half] = o1;
          }
        }
        fl_ring_release(p, fw);
      }
      FL_TRACE();
      FL_EV(3);

      // ============ B: attention (one unit per CTA: row, head, key split) ============
      if (g.u_on) {
        const int sub = lane & 7, grp = lane >> 3;
        const int b = g.u_b, h = g.u_h, n = g.u_n, pos = n - 1;
        float q[8];  // q slice of this lane: dims sub*8 .. sub*8+7 (polled after the first chunk's K/V are in registers)
        float M = -INFINITY, L = 0.f, O = 0.f;
        int pend_kv = 0;
        for (int sb = 0;; ++sb) {
          int chunk;
          if (!fl_kv_more(g, sb, chunk)) break;
          const bool have = fl_kv_valid(g, chunk);
          const float* slot = have ? fl_ring_wait(p, fw, wd) : nullptr;  // usually complete long ago (prefetched a phase early)
          const int tbase = chunk * FL_CH + warp * 8 + grp;
          float4 k0[2], k1[2], v0[2], v1[2];
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int t = tbase + 4 * i;
            k0[i] = k1[i] = v0[i] = v1[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (have && t < pos) {
              const float* kr = slot + (grp + 4 * i) * 64 + sub * 8;
              const float* vr = kr + 8 * 64;
              k0[i] = *reinterpret_cast<const float4*>(kr); k1[i] = *reinterpret_cast<const float4*>(kr + 4);
              v0[i] = *reinterpret_cast<const float4*>(vr); v1[i] = *reinterpret_cast<const float4*>(vr + 4);
            }
          }
          if (sb == 0) {  // K/V of earlier tokens never depend on this step: they are loaded before q is waited for
            const unsigned long long* qp = qkvw + FL_A_Q + b * KC + h * 64 + sub * 8;
            unsigned long long w[8];
            wd.spins = 0;
            while (true) {
              bool ok = true;
#pragma unroll
              for (int k = 0; k < 4; ++k) ll_ld2(qp + 2 * k, w[2 * k], w[2 * k + 1]);
#pragma unroll
              for (int k = 0; k < 8; ++k) ok = ok && (ll_tag(w[k]) == tagl + FT_QKV);
              if (__all_sync(0xffffffffu, ok)) break;
              if (__any_sync(0xffffffffu, fl_giveup(wd, 0x300))) { wd.dead = 1; break; }
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) q[k] = ll_val(w[k]);
          }
          if (sb == 0) { FL_EV(4); fl_refill_all(p, fw); }
          // the token of THIS step: its K/V rows arrive from the QKV phase through the LL region, not the cache
          {
            const bool mine0 = (tbase == pos), mine1 = (tbase + 4 == pos);
            if (__any_sync(0xffffffffu, mine0 || mine1)) {
              const unsigned long long* kp = qkvw + FL_A_KN + b * KC + h * 64 + sub * 8;
              const unsigned long long* vp = qkvw + FL_A_VN + b * KC + h * 64 + sub * 8;
              unsigned long long kw[8], vw[8];
              wd.spins = 0;
              while (true) {
                bool ok = true;
                if (mine0 || mine1) {
#pragma unroll
                  for (int k = 0; k < 4; ++k) { ll_ld2(kp + 2 * k, kw[2 * k], kw[2 * k + 1]); ll_ld2(vp + 2 * k, vw[2 * k], vw[2 * k + 1]); }
#pragma unroll
                  for (int k = 0; k < 8; ++k) ok = ok && (ll_tag(kw[k]) == tagl + FT_QKV) && (ll_tag(vw[k]) == tagl + FT_QKV);
                }
                if (__all_sync(0xffffffffu, ok)) break;
                if (__any_sync(0xffffffffu, fl_giveup(wd, 0x301))) { wd.dead = 1; break; }
              }
              if (mine0 || mine1) {
                const int i = mine0 ? 0 : 1;
                const float4 a = make_float4(ll_val(kw[0]), ll_val(kw[1]), ll_val(kw[2]), ll_val(kw[3]));
                const float4 bq = make_float4(ll_val(kw[4]), ll_val(kw[5]), ll_val(kw[6]), ll_val(kw[7]));
                const float4 cq = make_float4(ll_val(vw[0]), ll_val(vw[1]), ll_val(vw[2]), ll_val(vw[3]));
                const float4 dq = make_float4(ll_val(vw[4]), ll_val(vw[5]), ll_val(vw[6]), ll_val(vw[7]));
                if (i == 0) { k0[0] = a; k1[0] = bq; v0[0] = cq; v1[0] = dq; }
                else { k0[1] = a; k1[1] = bq; v0[1] = cq; v1[1] = dq; }
              }
            }
          }
          float sc[2], m = -INFINITY;
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float s = q[0] * k0[i].x + q[1] * k0[i].y + q[2] * k0[i].z + q[3] * k0[i].w + q[4] * k1[i].x + q[5] * k1[i].y +
                      q[6] * k1[i].z + q[7] * k1[i].w;
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            s += __shfl_xor_sync(0xffffffffu, s, 4);
            sc[i] = (tbase + 4 * i < n) ? s * p.scaling : -INFINITY;
            m = fmaxf(m, sc[i]);
          }
          m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
          m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 16));
          float lsum = 0.f, o[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          if (m > -INFINITY) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float e = expf(sc[i] - m);
              lsum += e;
              o[0] = fmaf(e, v0[i].x, o[0]); o[1] = fmaf(e, v0[i].y, o[1]); o[2] = fmaf(e, v0[i].z, o[2]);
              o[3] = fmaf(e, v0[i].w, o[3]); o[4] = fmaf(e, v1[i].x, o[4]); o[5] = fmaf(e, v1[i].y, o[5]);
              o[6] = fmaf(e, v1[i].z, o[6]); o[7] = fmaf(e, v1[i].w, o[7]);
            }
          }
          lsum += __shfl_xor_sync(0xffffffffu, lsum, 8);
          lsum += __shfl_xor_sync(0xffffffffu, lsum, 16);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            o[j] += __shfl_xor_sync(0xffffffffu, o[j], 8);
            o[j] += __shfl_xor_sync(0xffffffffu, o[j], 16);
          }
          if (have) {
            int nxt;
            if (fl_kv_more(g, sb + 1, nxt)) fl_ring_release(p, fw);
            else pend_kv = 1;  // last chunk: refill after the partial has been stored
          }
          fl_bar();  // previous chunk's merge no longer reads s_ao / s_am / s_al
          if (lane < 8) {
            *reinterpret_cast<float4*>(&s_ao[warp][lane * 8]) = make_float4(o[0], o[1], o[2], o[3]);
            *reinterpret_cast<float4*>(&s_ao[warp][lane * 8 + 4]) = make_float4(o[4], o[5], o[6], o[7]);
            if (lane == 0) { s_am[warp] = m; s_al[warp] = lsum; }
          }
          fl_bar();
          if (tid < 64) {
            float cm = M;
#pragma unroll
            for (int w = 0; w < FL_WARPS; ++w) cm = fmaxf(cm, s_am[w]);
            const float fo = (M > -INFINITY) ? expf(M - cm) : 0.f;
            L *= fo; O *= fo;
#pragma unroll
            for (int w = 0; w < FL_WARPS; ++w) {
              const float f = (s_am[w] > -INFINITY) ? expf(s_am[w] - cm) : 0.f;
              L = fmaf(f, s_al[w], L);
              O = fmaf(f, s_ao[w][tid], O);
            }
            M = cm;
          }
        }
        // Every unit publishes its partial; the O-proj phase of every CTA merges the splits of a (row, head) itself while
        // it stages its input (fl_stage_attn), so the partials cross CTAs once instead of meeting at a split-0 unit first.
        FL_EV(14);
        if (tid < 64) {
          unsigned long long* P = par + FL_A_P + ((size_t)(b * FL_HEADS + h) * FL_SMAX + g.u_split) * FL_PW;
          for (int r = 0; r < R; ++r) {
            unsigned long long* Pr = P + (size_t)r * FL_REP_STRIDE;
            ll_st(Pr + tid, O, tagl + FT_P);
            if (tid == 0) { ll_st(Pr + 64, M, tagl + FT_P); ll_st(Pr + 65, L, tagl + FT_P); }
          }
        }
        FL_EV(15);
        if (pend_kv) fl_ring_release(p, fw);
      }
      FL_TRACE();
      FL_EV(5);

      // ============ C: O-proj + residual on the merged attention output ============
      fl_bar();  // xs (raw x) is no longer read by any warp of this CTA
      if (l + 1 < p.L || p.sample) fl_nw_fetch(s_nw1, l + 1 < p.L ? Wl + p.layer_stride + p.o_ln1 : p.W + p.o_final_norm, &s_nwbar[0], pol_w);
      const bool o_rdy = fl_o_valid(g) ? fl_ring_peek_n(p, fw, 1) : true;
      fl_stage_attn<BT>(p, myr + FL_A_P, tagl + FT_P, xs, wd, g.S, s_pos, s_active);
      fl_refill_all(p, fw);
      FL_EV(6);
      if (fl_o_valid(g)) {
        fl_load_x<BT>(xs, x, lane);
        if (!o_rdy) fl_ring_wait_n(p, fw, 1, wd);
        const float* slot = fl_ring_slot_at(fw, 0);
        FL_EV(7);
        float a0[BT];
        fl_dot1<BT>(slot, x, a0, lane);
        warp_reduce_scatter<BT>(a0);
        const float out = __fadd_rn(res_keep, a0[0]);
        fl_bcast_store<BT>(par, R, FL_A_XO + (size_t)(lane / LPB) * KC + o_row, out, tagl + FT_XO, p.B, lane);
        fl_ring_release(p, fw);
      }
      FL_TRACE();
      FL_EV(8);
    }

    // ============ D: gate/up + SiLU * mul ============
    {
      float4 nw[6];
      fl_nw_wait(&s_nwbar[1], nw2_cnt, wd);
      int ngu = 0;
#pragma unroll
      for (int j = 0; j < FL_GU; ++j) ngu += fl_gu_valid(g, j, p.I) ? 1 : 0;
      const bool gu_rdy = fl_ring_peek_n(p, fw, ngu);
      fl_bar();  // every warp is done with xs (attention output)
      FL_CK(8);
      fl_stage768<BT>(p, myr + FL_A_XO, tagl + FT_XO, xs, wd, fw);
      fl_refill_all(p, fw);
      fl_load_nw_s(s_nw2, nw, lane);
      FL_EV(9);
      FL_CK(9);
      if (tid < FL_ROWS * BT) {  // residual of the down-phase output elements (raw x')
        const int b = tid % BT, j = tid / BT, row = g.cta + g.G * j;
        s_resd[tid] = row < KC ? xs[b * KC + row] : 0.f;
      }
      float x[BT][24];
      fl_load_x<BT>(xs, x, lane);
      FL_CK(10);
      fl_norm<BT>(x, nw, p.eps);
      FL_CK(11);
      {
        // all (<= 3) gate/up pair tasks of the warp at once: one pass over the activations, ONE butterfly for the six
        // row sums, the slot refills issued after the stores (they cost ~500 cycles each and nothing waits for them)
        FL_CK(0);
        const float4* sl[FL_GU];
#pragma unroll
        for (int j = 0; j < FL_GU; ++j) sl[j] = reinterpret_cast<const float4*>(fl_ring_slot_at(fw, j)) + lane;
        if (!gu_rdy) fl_ring_wait_n(p, fw, ngu, wd);
        FL_EV(16);
        FL_CK(1);
        float acc[8 * BT];
#pragma unroll
        for (int k = 0; k < 8 * BT; ++k) acc[k] = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) {
#pragma unroll
          for (int j = 0; j < FL_GU; ++j)
            if (j < ngu) {
              const float4 u = sl[j][i * 32], v = sl[j][KC / 4 + i * 32];
#pragma unroll
              for (int b = 0; b < BT; ++b) {
                float& a0 = acc[(2 * j) * BT + b];
                float& a1 = acc[(2 * j + 1) * BT + b];
                a0 = fmaf(u.x, x[b][4 * i], a0); a0 = fmaf(u.y, x[b][4 * i + 1], a0);
                a0 = fmaf(u.z, x[b][4 * i + 2], a0); a0 = fmaf(u.w, x[b][4 * i + 3], a0);
                a1 = fmaf(v.x, x[b][4 * i], a1); a1 = fmaf(v.y, x[b][4 * i + 1], a1);
                a1 = fmaf(v.z, x[b][4 * i + 2], a1); a1 = fmaf(v.w, x[b][4 * i + 3], a1);
              }
            }
        }
        FL_CK(2);
        warp_reduce_scatter<8 * BT>(acc);
        FL_CK(3);
        // After the butterfly the 8 lanes [8j, 8j+8) hold task j: gate sums of the BT rows (LPV lanes each), then the up
        // sums.  All 8 lanes compute the activation of "their" row; the 2*LPV lanes of a row share the replica stores.
        constexpr int LPV = 32 / (8 * BT);
        const int gl = lane & 7, b = (gl / LPV) % BT, base8 = lane & ~7;
        const float gv = __shfl_sync(0xffffffffu, acc[0], base8 + b * LPV);
        const float uv = __shfl_sync(0xffffffffu, acc[0], base8 + BT * LPV + b * LPV);
        if ((lane >> 3) < ngu && b < p.B) {
          const float sg = __fdiv_rn(gv, __fadd_rn(1.0f, expf(-gv)));
          const float act = __fmul_rn(sg, uv);
          unsigned long long* d = par + FL_A_ACT + (size_t)b * p.I + (g.gw + (lane >> 3) * g.NW);
          for (int rr = (gl % LPV) + (gl >= BT * LPV ? LPV : 0); rr < R; rr += 2 * LPV) ll_st(d + (size_t)rr * FL_REP_STRIDE, act, tagl + FT_ACT);
        }
        FL_CK(5);
        for (int j = 0; j < ngu; ++j) fl_ring_release(p, fw);
        FL_CK(6);
      }
      FL_TRACE();
      FL_EV(10);
    }

    // ============ E: down + residual (K = 3072 split over the 8 warps) ============
    {
      float xd[BT][12];
      const int nr0_ = fl_d_rows(g, 0, 4), nr1_ = fl_d_rows(g, 4, FL_ROWS);
      const bool d_rdy = fl_ring_peek_n(p, fw, nr1_ > 0 ? 2 : 1);
      {
        const int kslice = p.I / FL_WARPS;  // 384
#pragma unroll
        for (int b = 0; b < BT; ++b) {
#pragma unroll
          for (int k = 0; k < 12; ++k) xd[b][k] = 0.f;
          if (b < p.B) {  // one poll loop per batch row keeps the 64-bit words of only one row live
            const unsigned long long* ap = myr + FL_A_ACT + (size_t)b * p.I + warp * kslice;
            unsigned long long w[12];
            // 132 x 8 warps reading 3 KiB each is 3.2 MB through L2 per round: spin on the first two words of every lane
            // and read the rest once they are in; every word is still validated by its own tag.  (Arrival counters
            // bumped with red.add by the producers were tried instead of the sentinel words: no faster, 356 vs 352 us.)
            wd.spins = 0;
            bool sentinel_ok = false;
            int it_s = 0, it_f = 0;
            if (b == 0) FL_CK(12);
            while (true) {
              ++it_s;
              ll_ld2(ap + lane * 4, w[0], w[1]);
              if (sentinel_ok || __all_sync(0xffffffffu, ll_tag(w[0]) == tagl + FT_ACT && ll_tag(w[1]) == tagl + FT_ACT)) {
                if (!sentinel_ok && b == 0) FL_CK(13);
                sentinel_ok = true;
                ++it_f;
                bool ok = ll_tag(w[0]) == tagl + FT_ACT && ll_tag(w[1]) == tagl + FT_ACT;
                ll_ld2(ap + lane * 4 + 2, w[2], w[3]);
#pragma unroll
                for (int i = 1; i < 3; ++i) {
                  ll_ld2(ap + (i * 32 + lane) * 4, w[4 * i], w[4 * i + 1]);
                  ll_ld2(ap + (i * 32 + lane) * 4 + 2, w[4 * i + 2], w[4 * i + 3]);
                }
#pragma unroll
                for (int k = 2; k < 12; ++k) ok = ok && (ll_tag(w[k]) == tagl + FT_ACT);
                if (__all_sync(0xffffffffu, ok)) break;
              }
              if (__any_sync(0xffffffffu, fl_giveup(wd, 0x500))) { wd.dead = 1; break; }
            }
            if (b == 0) { FL_CK(14); if (p.trace && l == 10 && tid == 0 && blockIdx.x == 0) { p.trace[3015] = it_s; p.trace[3016] = it_f; } }
#pragma unroll
            for (int k = 0; k < 12; ++k) xd[b][k] = ll_val(w[k]);
          }
        }
      }
      FL_EV(11);
      fl_refill_all(p, fw);
      int e_tasks = 0;
      {
        // both down tasks (<= 6 row slices) together, one butterfly, refills after the partial sums are in shared memory
        const int nr0 = nr0_, nr1 = nr1_;
        const float* s0 = fl_ring_slot_at(fw, 0);
        const float* s1 = nr1 > 0 ? fl_ring_slot_at(fw, 1) : s0;
        if (!d_rdy) fl_ring_wait_n(p, fw, nr1 > 0 ? 2 : 1, wd);
        FL_EV(17);
        float acc[8 * BT];
#pragma unroll
        for (int k = 0; k < 8 * BT; ++k) acc[k] = 0.f;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
#pragma unroll
          for (int k = 0; k < FL_ROWS; ++k) {
            const bool valid = k < 4 ? (k < nr0) : (k - 4 < nr1);
            if (valid) {
              const float4 u = (reinterpret_cast<const float4*>((k < 4 ? s0 : s1) + (k & 3) * (3072 / FL_WARPS)) + lane)[i * 32];
#pragma unroll
              for (int b = 0; b < BT; ++b) {
                float& a = acc[k * BT + b];
                a = fmaf(u.x, xd[b][4 * i], a); a = fmaf(u.y, xd[b][4 * i + 1], a);
                a = fmaf(u.z, xd[b][4 * i + 2], a); a = fmaf(u.w, xd[b][4 * i + 3], a);
              }
            }
          }
        }
        warp_reduce_scatter<8 * BT>(acc);
        constexpr int LPV = 32 / (8 * BT);
        const int vi = lane / LPV, k = vi / BT, b = vi % BT;
        if ((lane % LPV) == 0 && k < FL_ROWS) s_red[k][warp][b] = acc[0];
        e_tasks = nr1 > 0 ? 2 : 1;
      }
      FL_EV(12);
      fl_bar();
      if (l + 1 < p.L) fl_nw_fetch(s_nw2, Wl + p.layer_stride + p.o_ln2, &s_nwbar[1], pol_w);
      if (tid < FL_ROWS * BT * 8) {  // K slices summed in the order 0..7 (deterministic); 8 threads share an element's replicas
        const int e = tid >> 3, b = e % BT, j = e / BT, row = g.cta + g.G * j;
        if (row < KC && b < p.B) {
          float v = s_red[j][0][b];
#pragma unroll
          for (int w = 1; w < FL_WARPS; ++w) v = __fadd_rn(v, s_red[j][w][b]);
          const float out = __fadd_rn(s_resd[e], v);
          for (int r = tid & 7; r < R; r += 8)
            ll_st(parn + (size_t)r * FL_REP_STRIDE + FL_A_X + (size_t)b * KC + row, out, tagl + 8u + FT_X);
        }
      }
      for (int k = 0; k < e_tasks; ++k) fl_ring_release(p, fw);  // refills only after the layer's output is on its way
      FL_TRACE();
      FL_EV(13);
    }
  }

  // ============ heads: final norm, logits, hidden state ============
  if (p.sample) {
    const unsigned long long* myr = p.arena + (size_t)(p.L & 1) * FL_PARITY_WORDS + (size_t)myrep * FL_REP_STRIDE;
    float4 nw[6];
    fl_nw_wait(&s_nwbar[0], nw1_cnt, wd);
    fl_bar();
    fl_stage768<BT>(p, myr + FL_A_X, base + 8u * (uint32_t)p.L + FT_X, xs, wd, fw);
    fl_refill_all(p, fw);
    fl_load_nw_s(s_nw1, nw, lane);
    float x[BT][24];
    fl_load_x<BT>(xs, x, lane);
    fl_norm<BT>(x, nw, p.eps);
    if (p.hidden_out != nullptr && blockIdx.x == 0 && warp == 0) {
#pragma unroll
      for (int b = 0; b < BT; ++b)
        if (b < p.B) {
          float4* dst = reinterpret_cast<float4*>(p.hidden_out + (size_t)b * p.hidden_stride + (size_t)ngen * KC);
#pragma unroll
          for (int i = 0; i < 6; ++i) dst[i * 32 + lane] = make_float4(x[b][4 * i], x[b][4 * i + 1], x[b][4 * i + 2], x[b][4 * i + 3]);
        }
    }
    const int nrows = p.rows_per_item * p.V;
    const uint32_t tagh = base + 8u * (uint32_t)p.L + FT_LOGITS;
    for (int j = 0; fl_h_valid(g, j); ++j) {
      const int t = g.gw + j * g.NW;
      const float* slot = fl_ring_wait(p, fw, wd);
      float a0[BT], a1[BT];
      fl_dot2<BT>(slot, x, a0, a1, lane);
      warp_reduce_scatter<BT>(a0);
      warp_reduce_scatter<BT>(a1);
      const int b = lane / LPB;
      if ((lane % LPB) == 0 && b < p.B) {
        const int r0 = 2 * t, q0 = r0 / p.V, c0 = r0 % p.V;
        const int q1 = (r0 + 1) / p.V, c1 = (r0 + 1) % p.V;
        if (ink) {  // to the sampler CTA of the row through tagged words
          ll_st(tailw + FL_A_LOGITS + (size_t)(b * p.rows_per_item + q0) * FL_VPAD + c0, a0[0], tagh);
          if (r0 + 1 < nrows) ll_st(tailw + FL_A_LOGITS + (size_t)(b * p.rows_per_item + q1) * FL_VPAD + c1, a1[0], tagh);
        } else {
          p.logits[((size_t)b * p.rows_per_item + q0) * p.V + c0] = a0[0];
          if (r0 + 1 < nrows) p.logits[((size_t)b * p.rows_per_item + q1) * p.V + c1] = a1[0];
        }
      }
      fl_ring_release(p, fw);
    }
  }
  FL_TRACE();
  fl_bar();
  if (tid < p.B && s_active[tid]) s_pos[tid]++;   // positions advance once per step
  fl_bar();
  const bool more = ink && sidx + 1 < p.nsteps;
  if (more) FL_PREP_STEP();
  if constexpr (INK) {
    if (ink) {
      // ============ sampling tail (gpt.py:487-508) on one CTA per (row, codebook) ============
      const uint32_t tagi = base + 8u * (uint32_t)p.L + FT_IDX;
      if (g.cta < nrows_s) {
        const int row = g.cta, qi = row % p.rows_per_item;
        const unsigned long long* lw = tailw + FL_A_LOGITS + (size_t)row * FL_VPAD;
        unsigned long long w[4];
        wd.spins = 0;
        while (true) {
          bool ok = true;
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (tid + 256 * k < p.V) { w[k] = ll_ld(lw + tid + 256 * k); ok = ok && ll_tag(w[k]) == base + 8u * (uint32_t)p.L + FT_LOGITS; }
          if (__all_sync(0xffffffffu, ok)) break;
          if (__any_sync(0xffffffffu, fl_giveup(wd, 0x600))) { wd.dead = 1; break; }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (tid + 256 * k < p.V) s_samp.x[tid + 256 * k] = ll_val(w[k]);
        fl_bar();
        const int id = fl_sample_row(p.samp, p.q_noise, s_samp, p.V, row, qi, nwin, lstep, (p.trace && row == 0) ? p.trace + 3100 : nullptr);
        if (tid == 0) {
          ll_st(tailw + FL_A_IDX + row, __int_as_float(id), tagi);
          const bool pen = p.samp.penalty_on && row < p.samp.penalty_max_ids;
          if (pen) {  // slide the repetition window
            if (nwin < p.samp.past_window) s_samp.win[nwin] = id;
            else { for (int k = 0; k + 1 < nwin; ++k) s_samp.win[k] = s_samp.win[k + 1]; if (nwin > 0) s_samp.win[nwin - 1] = id; }
          }
        }
        if (p.samp.penalty_on && row < p.samp.penalty_max_ids && nwin < p.samp.past_window) nwin++;
        fl_bar();
      }
      FL_TRACE();
      // ============ finish / write-back / counters (gpt.py:512-525,572-577) - every CTA keeps the loop state ============
      if (tid < nrows_s) {
        unsigned long long w;
        wd.spins = 0;
        while (true) {
          w = ll_ld(tailw + FL_A_IDX + tid);
          if (ll_tag(w) == tagi) break;
          if (fl_giveup(wd, 0x601)) break;
        }
        s_ids[(tid / p.rows_per_item) * 8 + tid % p.rows_per_item] = __float_as_int(ll_val(w));
      }
      fl_bar();
      if (tid == 0) {
        int notall = 0;
        for (int b = 0; b < p.B; ++b) {
          bool eos = false;
          for (int q = 0; q < p.rows_per_item; ++q) eos |= (s_ids[b * 8 + q] == p.samp.eos_token);
          const int fin = s_fin[b] || eos;
          s_fin[b] = fin;
          if (!fin) { s_end[b]++; notall = 1; }
          if (blockIdx.x == 0) {
            int32_t* dst = p.ids_w + ((size_t)b * p.max_new + ngen) * p.num_vq;
            for (int q = 0; q < p.num_vq; ++q) dst[q] = s_ids[b * 8 + q];
            p.finish[b] = (uint8_t)fin;
            p.end_idx[b] = s_end[b];
          }
        }
        s_allfin = !notall;
        if (blockIdx.x == 0) {
          if (!notall) p.st->all_finished = 1;
          p.st->n_gen = ngen + 1;
          p.st->step = lstep + 1;
        }
      }
      fl_bar();
      FL_TRACE();
    }
  }
  ngen++; lstep++;
  base += FL_EPOCH_STEP;                           // no word of this step can satisfy the next one
  if (!more || s_allfin) {
    if (more) {  // tasks of the step that will not run are in flight: wait for them before the CTA may exit
      const int outst = fw.it.n - fw.n;
      for (int k = 0; k < outst; ++k) {
        const int n = fw.n + k;
        wd.spins = 0;
        while (!fl_try_wait(fw.bars + (n % FL_SLOTS) * 8, (uint32_t)(n / FL_SLOTS) & 1u))
          if (__any_sync(0xffffffffu, fl_giveup(wd, 0x700))) { wd.dead = 1; break; }
      }
    }
    break;
  }
  }  // step loop
  if (blockIdx.x == 0) {
    if (tid < p.B) p.seq_len[tid] = s_pos[tid];
    if (tid == 0) *p.epoch = base;
  }
#undef FL_TRACE
#undef FL_EV
#undef FL_CK
#undef FL_PREP_STEP
}

}  // namespace ctb
