// multiverso-b200 :: the WordEmbedding block protocol on the device, no host round trip.
//
// Reference (Applications/WordEmbedding/src): per data block
//   PrepareData            wordembedding.cpp:169-213   input_nodes = words of the block,
//                                                      output_nodes = input_nodes U (negative_num x |input| draws)
//   RequestParameter       communicator.cpp:117-155    Get(rows) of both tables into block-local copies
//   AddDeltaParameter      communicator.cpp:206-249    Add(rows, (trained - pulled) / num_workers)
// Round 1 did PrepareData with eager PyTorch (2 x torch.unique = CUB sort + host sync, boolean-mask
// indexing, randint / where / cat, two clone()s of the caches).  Here:
//
//   mvb_we_prepare     bitmap-unique + prefix sum: tokens -> bitmap (atomicOr), three tiny scan kernels
//                      turn the bitmap into (id -> slot map, slot -> id list, count), the negative pool is
//                      drawn on the device from the unigram^0.75 alias table with a hash RNG, its words are
//                      OR-ed into the output bitmap, second scan.  Counts stay on the device; every later
//                      kernel reads them there, so nothing ever synchronises with the host.
//   mvb_rows_pull      row gather from the owners' shards (over NVLink for peer shards) into the block cache
//                      AND its "pulled" copy (what clone() did): a warp per row, 128-bit loads and stores.
//   mvb_rows_push_delta   (rows.cu) (trained - pulled) * scale per row, reduced into the owner's shard with
//                      one-sided red.add.v4.f32 (element-wise atomic at the owner: the async-PS Add for
//                      stateless updaters); all-zero 16-byte deltas are skipped.
// Pull and push run ctas_per_sm register-only CTAs per SM, co-resident with the persistent K7 (see below).
#include "mvb_common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
// PrepareData
// ------------------------------------------------------------------------------------------------
// Every kernel of the side stream runs in 128-thread CTAs with <= 56 registers and (almost) no shared memory:
// the register file is split per SM sub-partition, and under the persistent K7 (11 warps x 152 registers)
// three of the four sub-partitions have 1 792 registers left -- one warp of <= 56 registers each.  A
// 256-thread CTA (two warps per sub-partition) never fits and would simply wait for K7 to finish
// (measured: `tools/probe_coresidency.py`).
constexpr int kSideThreads = 128;
constexpr int kChunkWords = 1024;      // bitmap words per scan CTA (32768 ids)
constexpr int kScanThreads = 128;      // 8 words per thread
constexpr int kWordsPerThread = kChunkWords / kScanThreads;

__global__ void __launch_bounds__(kSideThreads, 9)
prep_clear_kernel(uint32_t* __restrict__ bm, int64_t words) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += stride) bm[i] = 0u;
}

__global__ void __launch_bounds__(kSideThreads, 9)
prep_mark_tokens_kernel(const int* __restrict__ tokens, int64_t n, int vocab, uint32_t* __restrict__ bm) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int t = __ldg(tokens + i);
    if (t < 0 || t >= vocab) continue;
    const uint32_t bit = 1u << (t & 31);
    uint32_t* w = bm + (t >> 5);
    if (!(*reinterpret_cast<volatile uint32_t*>(w) & bit)) atomicOr(w, bit);   // Zipf head: mostly already set
  }
}

// scan phase A: set bits per chunk
__global__ void __launch_bounds__(kScanThreads)
prep_scan_a_kernel(const uint32_t* __restrict__ bm, int64_t words, int* __restrict__ chunk_sums) {
  __shared__ int wsum[kScanThreads / 32];
  const int64_t base = (int64_t)blockIdx.x * kChunkWords + threadIdx.x * kWordsPerThread;
  int c = 0;
#pragma unroll
  for (int j = 0; j < kWordsPerThread; ++j)
    if (base + j < words) c += __popc(bm[base + j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < kScanThreads / 32; ++w) s += wsum[w];
    chunk_sums[blockIdx.x] = s;
  }
}

// scan phase B: exclusive scan of the chunk sums (one CTA), total -> *count (clamped to cap)
__global__ void __launch_bounds__(kSideThreads, 9)
prep_scan_b_kernel(int* __restrict__ chunk_sums, int n_chunks, int* __restrict__ count, int64_t cap) {
  __shared__ int part[kSideThreads];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n_chunks; base += kSideThreads) {
    const int i = base + threadIdx.x;
    const int v = i < n_chunks ? chunk_sums[i] : 0;
    part[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < kSideThreads; o <<= 1) {   // Hillis-Steele inclusive scan
      int t = threadIdx.x >= o ? part[threadIdx.x - o] : 0;
      __syncthreads();
      part[threadIdx.x] += t;
      __syncthreads();
    }
    if (i < n_chunks) chunk_sums[i] = carry + part[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == kSideThreads - 1) carry += part[kSideThreads - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = (int)((int64_t)carry < cap ? carry : cap);
}

// scan phase C: id -> slot map (or -1) and slot -> id list
__global__ void __launch_bounds__(kScanThreads)
prep_scan_c_kernel(const uint32_t* __restrict__ bm, int64_t words, int vocab, const int* __restrict__ chunk_off,
                   int* __restrict__ map, int* __restrict__ ids, int64_t cap, uint32_t* __restrict__ bm_copy) {
  __shared__ int wsum[kScanThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = (int64_t)blockIdx.x * kChunkWords + threadIdx.x * kWordsPerThread;
  uint32_t w[kWordsPerThread];
  int c = 0;
#pragma unroll
  for (int j = 0; j < kWordsPerThread; ++j) {
    w[j] = base + j < words ? bm[base + j] : 0u;
    if (bm_copy && base + j < words) bm_copy[base + j] = w[j];      // output nodes start as the input nodes
    c += __popc(w[j]);
  }
  int incl = c;                                     // inclusive scan inside the warp
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  int woff = 0;
  for (int k = 0; k < warp; ++k) woff += wsum[k];
  int slot = chunk_off[blockIdx.x] + woff + incl - c;
#pragma unroll
  for (int j = 0; j < kWordsPerThread; ++j) {
    if (base + j >= words) break;
    const int64_t id0 = (base + j) * 32;
#pragma unroll 8
    for (int b = 0; b < 32; ++b) {
      const int64_t id = id0 + b;
      if (id >= vocab) break;
      if ((w[j] >> b) & 1u) {
        if (slot < cap) { map[id] = slot; ids[slot] = (int)id; } else { map[id] = -1; }
        ++slot;
      } else {
        map[id] = -1;
      }
    }
  }
}

// negative pool: negative x |input| draws from unigram^0.75 (alias table), OR-ed into the output bitmap
__global__ void __launch_bounds__(kSideThreads, 9)
prep_neg_pool_kernel(const int* __restrict__ n_in_ptr, int negative, int vocab, const float* __restrict__ prob,
                     const int* __restrict__ alias, uint64_t seed, int* __restrict__ pool, int64_t pool_cap,
                     uint32_t* __restrict__ bm_out, int* __restrict__ n_pool_ptr) {
  int64_t n_draw = (int64_t)(*n_in_ptr) * negative;
  if (n_draw > pool_cap) n_draw = pool_cap;
  if (blockIdx.x == 0 && threadIdx.x == 0) *n_pool_ptr = (int)n_draw;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; d < n_draw; d += stride) {
    const uint64_t r = hash64(seed ^ (uint64_t)(d + 1) * 0x9E3779B97F4A7C15ull);
    const uint32_t idx = (uint32_t)((r >> 32) % (uint64_t)vocab);
    const float u = (float)(r & 0xFFFFFF) * (1.0f / 16777216.0f);
    const int t = (u < __ldg(prob + idx)) ? (int)idx : __ldg(alias + idx);
    pool[d] = t;
    const uint32_t bit = 1u << (t & 31);
    uint32_t* w = bm_out + (t >> 5);
    if (!(*reinterpret_cast<volatile uint32_t*>(w) & bit)) atomicOr(w, bit);
  }
}

// ------------------------------------------------------------------------------------------------
// row pull (the delta push is rows.cu's add_rows_delta_kernel)
// ------------------------------------------------------------------------------------------------
struct PullDev {
  MvbRowMap m;
  const int* ids;          // slot -> row id
  const int* n_ptr;        // device count (nullptr: n_max rows)
  int64_t n_max;
  unsigned char* dst_a;    // [n x dst_ld_bytes]
  unsigned char* dst_b;    // optional second copy
  int64_t dst_ld_bytes;
  int row_bytes;           // == the shards' row pitch
};

// No shared memory and <= 56 registers: these CTAs co-reside with the persistent K7 CTAs (which own the
// SMs' shared memory but leave threads and registers), so the pull of block i+1 and the push of block i-1
// use the memory-level parallelism of ALL SMs while K7 trains block i.
// Warp per row, 128-bit accesses, two rows in flight per warp.
__global__ void __launch_bounds__(kSideThreads, 9)
rows_pull_kernel(const __grid_constant__ PullDev a) {
  const int lane = threadIdx.x & 31;
  int64_t n = a.n_ptr ? (int64_t)*a.n_ptr : a.n_max;
  if (n > a.n_max) n = a.n_max;
  const int nvec = a.row_bytes >> 4;
  for (int64_t s = warp_id() * 2; s < n; s += num_warps() * 2) {
    const unsigned char* src[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      src[u] = nullptr;
      if (s + u < n) {
        const int64_t r = (int64_t)__ldg(a.ids + s + u);
        if (r >= 0 && r < a.m.num_row) src[u] = row_ptr<const unsigned char>(a.m, r, a.row_bytes);
      }
    }
    for (int v0 = 0; v0 < nvec; v0 += 64) {
      uint4 x[2][2];
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int v = v0 + lane + 32 * j;
          if (src[u] && v < nvec) x[u][j] = ld_nc_v4(src[u] + (size_t)v * 16);
        }
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int v = v0 + lane + 32 * j;
          if (src[u] && v < nvec) {
            st_na_v4(a.dst_a + (s + u) * a.dst_ld_bytes + (size_t)v * 16, x[u][j]);
            if (a.dst_b) st_na_v4(a.dst_b + (s + u) * a.dst_ld_bytes + (size_t)v * 16, x[u][j]);
          }
        }
    }
  }
}

}  // namespace

extern "C" int mvb_we_prepare(const MvbWePrep* p, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (p->vocab <= 0 || p->n_tokens < 0) return -1;
  if (p->negative > 0 && (!p->alias_prob || !p->alias_idx || !p->neg_pool)) return -2;
  const int64_t words = ((int64_t)p->vocab + 31) / 32;
  const int n_chunks = (int)((words + kChunkWords - 1) / kChunkWords);
  const int sms = mvb_num_sms();
  auto grid_for = [&](int64_t items) {
    int64_t g = (items + kSideThreads - 1) / kSideThreads;
    if (g > 2 * sms) g = 2 * sms;
    return (int)(g < 1 ? 1 : g);
  };
  prep_clear_kernel<<<grid_for(words), kSideThreads, 0, st>>>(p->bm_in, words);
  prep_mark_tokens_kernel<<<grid_for(p->n_tokens), kSideThreads, 0, st>>>(p->tokens, p->n_tokens, p->vocab, p->bm_in);
  prep_scan_a_kernel<<<n_chunks, kScanThreads, 0, st>>>(p->bm_in, words, p->chunk_sums);
  prep_scan_b_kernel<<<1, kSideThreads, 0, st>>>(p->chunk_sums, n_chunks, p->counts + 0, p->cap_in);
  // output nodes = input nodes U negative pool: the scan of the input bitmap also copies it
  prep_scan_c_kernel<<<n_chunks, kScanThreads, 0, st>>>(p->bm_in, words, p->vocab, p->chunk_sums, p->map_in,
                                                        p->ids_in, p->cap_in, p->bm_out);
  if (p->negative > 0)
    prep_neg_pool_kernel<<<grid_for(p->pool_cap), kSideThreads, 0, st>>>(p->counts + 0, p->negative, p->vocab,
                                                                         p->alias_prob, p->alias_idx, p->seed,
                                                                         p->neg_pool, p->pool_cap, p->bm_out,
                                                                         p->counts + 2);
  prep_scan_a_kernel<<<n_chunks, kScanThreads, 0, st>>>(p->bm_out, words, p->chunk_sums);
  prep_scan_b_kernel<<<1, kSideThreads, 0, st>>>(p->chunk_sums, n_chunks, p->counts + 1, p->cap_out);
  prep_scan_c_kernel<<<n_chunks, kScanThreads, 0, st>>>(p->bm_out, words, p->vocab, p->chunk_sums, p->map_out,
                                                        p->ids_out, p->cap_out, nullptr);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_we_prepare_launches(int negative) { return negative > 0 ? 9 : 8; }

// Gather rows ids[0..n) of a row-sharded table of 4-byte elements into dst_a (and dst_b, when given).
// n is read on the device from n_ptr when given (clamped to n_max).  Row bytes must be a multiple of 16.
// The grid is ctas_per_sm (>= 1) CTAs per SM.
extern "C" int mvb_rows_pull(const MvbRowMap* m, int esz, const int* ids, const int* n_ptr, int64_t n_max,
                             void* dst_a, void* dst_b, int64_t dst_ld, int ctas_per_sm, void* stream) {
  if (!row_split_ok(m->nservers, m->rows_per_server)) return MVB_BAD_ROW_MAP;
  if (ctas_per_sm < 1) return -22;
  if (n_max <= 0) return 0;
  const int64_t row_bytes = m->num_col * esz;
  if (row_bytes % 16 || (dst_ld * esz) % 16) return -9;
  if ((reinterpret_cast<uintptr_t>(dst_a) & 15) || (reinterpret_cast<uintptr_t>(dst_b) & 15)) return -9;
  PullDev a{};
  a.m = *m;
  a.ids = ids; a.n_ptr = n_ptr; a.n_max = n_max;
  a.dst_a = (unsigned char*)dst_a; a.dst_b = (unsigned char*)dst_b; a.dst_ld_bytes = dst_ld * esz;
  a.row_bytes = (int)row_bytes;
  rows_pull_kernel<<<mvb_num_sms() * ctas_per_sm, kSideThreads, 0, (cudaStream_t)stream>>>(a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
