// On-demand KV pages of a slot engine (ctb_gpt_engine_begin_paged): block-table writes, page fills, one slot's loop
// state, and the gather / scatter of one slot's pages between the pool and a host image (k_kv_pack / k_kv_unpack);
// and the copy of a shared prompt's pages between two rows of a fixed engine (k_kv_copy).
// The decode, prefill and attention kernels are not involved: they reach the pool only through the block table.
#pragma once
#include "gpt_kernels.cuh"

namespace ctb {

// block-table entries (and pages to fill) per launch: they travel by value, under the 4 KiB parameter limit
constexpr int KV_BT_MAX = 480;
// pages one slot image may hold (a slot of 8,192 tokens)
constexpr int KV_MOVE_MAX_PAGES = 512;
// the device staging buffer a slot's KV passes through on its way to and from host memory
constexpr size_t KV_STAGE_BYTES = (size_t)64 << 20;

struct BtWriteP {
  int* bt;
  int n;
  int idx[KV_BT_MAX];   // entries of the [S][pages_per_row] table
  int page[KV_BT_MAX];  // their new pages (0: the zero page)
};

// n pages (list[i], or p0 + i with list unused) of every layer set to `word` (4-byte pattern)
struct KvFillP {
  char* kv;
  size_t layer_bytes, page_bytes;
  int layers, n, p0, use_list;
  uint32_t word;
  int list[KV_BT_MAX];
};

struct KvMoveP {
  char* kv;             // the pool
  uint4* img;           // image pages [pg0, pg1) of [layer][i < npages] (one page of that layer, as the pool stores it)
  int pg0, pg1;
  size_t layer_bytes;   // one layer's share of the pool
  int page_words;       // 16-byte words of one page of one layer
  int layers, npages;
  int pages[KV_MOVE_MAX_PAGES];
};

// pages [0, npages) of every layer of one fixed-engine row (pages src0 + i) to another's (dst0 + i)
struct KvCopyP {
  char* kv;             // the pool
  size_t layer_bytes;   // one layer's share of the pool
  int page_words;       // 16-byte words of one page of one layer
  int layers, npages, src0, dst0;
};

struct SetRowP {
  LoopState* st;
  RowState* rows;
  int B, b;
  RowState row;
};

#ifdef CTB_GPT_KERNELS_IMPL
__global__ void k_bt_write(const __grid_constant__ BtWriteP p) {
  for (int i = threadIdx.x; i < p.n; i += blockDim.x) p.bt[p.idx[i]] = p.page[i];
}

__global__ void k_kv_fill(const __grid_constant__ KvFillP p) {
  const size_t words = p.page_bytes / 4, total = (size_t)p.layers * p.n * words;
  for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (size_t)gridDim.x * blockDim.x) {
    const size_t pg = w / words;
    const int l = (int)(pg / p.n), i = (int)(pg % p.n);
    const int page = p.use_list ? p.list[i] : p.p0 + i;
    reinterpret_cast<uint32_t*>(p.kv + l * p.layer_bytes + (size_t)page * p.page_bytes)[w % words] = p.word;
  }
}

// a CTA per (layer, page) pair in turn, its threads over the page's 16-byte words; image page pg = l * npages + i is
// page pages[i] of layer l
template <bool PACK>
__device__ __forceinline__ void kv_move(const KvMoveP& p) {
  for (int pg = p.pg0 + blockIdx.x; pg < p.pg1; pg += gridDim.x) {
    const int l = pg / p.npages, i = pg - l * p.npages;
    uint4* d = reinterpret_cast<uint4*>(p.kv + l * p.layer_bytes) + (size_t)p.pages[i] * p.page_words;
    uint4* m = p.img + (size_t)(pg - p.pg0) * p.page_words;
    for (int w = threadIdx.x; w < p.page_words; w += blockDim.x) {
      if (PACK) m[w] = d[w];
      else d[w] = m[w];
    }
  }
}
__global__ void k_kv_pack(const __grid_constant__ KvMoveP p) { kv_move<true>(p); }
__global__ void k_kv_unpack(const __grid_constant__ KvMoveP p) { kv_move<false>(p); }

// A shared prompt's KV on a fixed engine (ctb_gpt_engine_share_prompt): a CTA per (layer, page) pair in turn, its
// threads over the page's 16-byte words, four loads in flight per thread before their stores
__global__ void k_kv_copy(const __grid_constant__ KvCopyP p) {
  constexpr int U = 4;
  for (int pg = blockIdx.x; pg < p.layers * p.npages; pg += gridDim.x) {
    const int l = pg / p.npages, i = pg - l * p.npages;
    const uint4* __restrict__ s = reinterpret_cast<const uint4*>(p.kv + l * p.layer_bytes) + (size_t)(p.src0 + i) * p.page_words;
    uint4* __restrict__ d = reinterpret_cast<uint4*>(p.kv + l * p.layer_bytes) + (size_t)(p.dst0 + i) * p.page_words;
    for (int w = threadIdx.x; w < p.page_words; w += U * blockDim.x) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (w + u * (int)blockDim.x < p.page_words) v[u] = s[w + u * blockDim.x];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (w + u * (int)blockDim.x < p.page_words) d[w + u * blockDim.x] = v[u];
    }
  }
}

// slot b's RowState <- row (outside the captured graphs, between decode chunks); all_finished = no running row, as
// k_cancel_rows leaves it
__global__ void k_set_row(const __grid_constant__ SetRowP p) {
  __shared__ int s_running;
  if (threadIdx.x == 0) {
    s_running = 0;
    p.rows[p.b] = p.row;
  }
  __syncthreads();
  for (int b = threadIdx.x; b < p.B; b += blockDim.x)
    if ((b == p.b ? p.row.state : ldg_cg(&p.rows[b].state)) == RS_RUNNING) atomicOr(&s_running, 1);
  __syncthreads();
  if (threadIdx.x == 0) p.st->all_finished = s_running ? 0 : 1;
}
#endif  // CTB_GPT_KERNELS_IMPL

}  // namespace ctb
