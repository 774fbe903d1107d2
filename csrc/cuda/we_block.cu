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
//   mvb_rows_pull_bulk row gather over NVLink on the bulk-copy engine: one warp per CTA, 32 rows per
//                      mbarrier batch, cp.async.bulk peer HBM -> smem, then smem -> the block cache AND its
//                      "pulled" copy (what clone() did) with bulk stores; ~190 KB in flight per SM, so a
//                      handful of SMs saturates the link while K7 keeps the rest.
//   mvb_rows_push_delta_bulk   (trained - pulled) * scale per row computed in smem by 4 warps, pushed into
//                      the owner's shard with cp.reduce.async.bulk.add.f32 (one-sided, element-wise atomic
//                      at the owner's L2: the async-PS Add for stateless updaters); untouched rows skipped.
#include <cstdlib>
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
// row pull / delta push on the bulk-copy engine
// ------------------------------------------------------------------------------------------------
struct RowMapDev {
  int64_t num_row, rps;
  int64_t ld_bytes;        // row pitch of the shards
  int S;
  unsigned char* shard[MVB_MAX_RANKS];
};
MVB_DEVINL unsigned char* row_addr(const RowMapDev& m, int64_t r) {
  int64_t o = r / m.rps;
  if (o > m.S - 1) o = m.S - 1;            // last server takes the remainder (matrix_table.cpp:270-273)
  return m.shard[o] + (r - o * m.rps) * m.ld_bytes;
}

struct PullDev {
  RowMapDev m;
  const int* ids;          // slot -> row id (ascending: consecutive ids are merged into one bulk copy)
  const int* n_ptr;        // device count (nullptr: n_max rows)
  int64_t n_max;
  unsigned char* dst_a;    // [n x dst_ld_bytes]
  unsigned char* dst_b;    // optional second copy
  int64_t dst_ld_bytes;
  int row_bytes;
  int q;                   // batches in flight
  int br;                  // rows per batch (32; fewer for rows too large for the shared-memory ring)
};

// Row runs of one 32-row batch: lane `l` starts a run when its row does not continue lane l-1's
// (id + 1, same owner).  The bulk engine is op-rate bound for 1.2 KB rows (~27 M ops/s per SM measured),
// and the sorted id lists of a Zipf block are mostly runs, so merging them is what makes a handful
// of SMs enough.  Returns the run length for start lanes, 0 otherwise; `hmask` = lanes with a row.
MVB_DEVINL int row_runs(const RowMapDev& m, int64_t r, bool have, int lane, uint32_t& hmask) {
  int64_t o = -1;
  if (have) {
    o = r / m.rps;
    if (o > m.S - 1) o = m.S - 1;
  }
  const int64_t r_prev = __shfl_up_sync(0xffffffffu, r, 1);
  const int64_t o_prev = __shfl_up_sync(0xffffffffu, o, 1);
  const bool start = have && (lane == 0 || r != r_prev + 1 || o != o_prev);
  hmask = __ballot_sync(0xffffffffu, have);
  const uint32_t smask = __ballot_sync(0xffffffffu, start);
  if (!start) return 0;
  const uint32_t stop = (smask | ~hmask) & ~((2u << lane) - 1u);     // next run start / missing row above me
  return stop ? (__ffs(stop) - 1 - lane) : (32 - lane);
}

__global__ void __launch_bounds__(32, 1)
rows_pull_bulk_kernel(const __grid_constant__ PullDev a) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  unsigned char* stage = smem + 128;
  const int lane = threadIdx.x;
  const int Q = a.q;
  if (lane == 0) {
    for (int s = 0; s < Q; ++s) mbar_init(full + s, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  int64_t n = a.n_ptr ? (int64_t)*a.n_ptr : a.n_max;
  if (n > a.n_max) n = a.n_max;
  const int BR = a.br;
  const int64_t n_batches = (n + BR - 1) / BR;
  // batches of this CTA: b = blockIdx.x + t * gridDim.x
  const int64_t mine = n_batches > blockIdx.x ? (n_batches - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const size_t batch_bytes = (size_t)BR * a.row_bytes;
  const bool dst_contig = a.dst_ld_bytes == a.row_bytes;

  auto batch_row = [&](int64_t t, int64_t& s, int64_t& r) {
    s = (blockIdx.x + t * gridDim.x) * BR + lane;
    const bool in = lane < BR && s < n;
    r = in ? (int64_t)__ldg(a.ids + s) : -1;
    return in && r >= 0 && r < a.m.num_row;
  };
  auto issue_load = [&](int64_t t) {
    const int q = (int)(t % Q);
    int64_t s, r;
    const bool have = batch_row(t, s, r);
    uint32_t hmask;
    const int len = row_runs(a.m, r, have, lane, hmask);
    if (lane == 0) {
      if (hmask) mbar_arrive_expect_tx(full + q, (uint32_t)__popc(hmask) * (uint32_t)a.row_bytes);
      else mbar_arrive(full + q);
    }
    __syncwarp();
    if (len > 0)
      bulk_g2s(stage + q * batch_bytes + (size_t)lane * a.row_bytes, row_addr(a.m, r),
               (uint32_t)len * (uint32_t)a.row_bytes, full + q);
  };

  // Q-2 loads in flight; a stage is re-filled two batches after its stores were committed, so the
  // newest store group may still be reading shared memory (wait_group.read 1)
  const int64_t pre = mine < Q - 2 ? mine : Q - 2;
  for (int64_t t = 0; t < pre; ++t) issue_load(t);
  for (int64_t t = 0; t < mine; ++t) {
    const int64_t tn = t + Q - 2;
    if (tn < mine) {
      bulk_wait_read<1>();      // stage (tn % Q) was stored by batch t-2: its bulk stores have read the rows
      __syncwarp();
      issue_load(tn);
    }
    const int q = (int)(t % Q);
    mbar_wait(full + q, (uint32_t)((t / Q) & 1));
    int64_t s, r;
    const bool have = batch_row(t, s, r);
    const uint32_t hmask = __ballot_sync(0xffffffffu, have);
    const unsigned char* src = stage + q * batch_bytes + (size_t)lane * a.row_bytes;
    const bool prefix = hmask != 0 && (hmask & (hmask + 1u)) == 0;      // rows 0..m-1 present, no holes
    if (dst_contig && prefix) {
      if (lane == 0) {                                                  // one store per destination
        const uint32_t bytes = (uint32_t)__popc(hmask) * (uint32_t)a.row_bytes;
        bulk_s2g(a.dst_a + s * a.dst_ld_bytes, src, bytes);
        if (a.dst_b) bulk_s2g(a.dst_b + s * a.dst_ld_bytes, src, bytes);
      }
    } else if (have) {
      bulk_s2g(a.dst_a + s * a.dst_ld_bytes, src, (uint32_t)a.row_bytes);
      if (a.dst_b) bulk_s2g(a.dst_b + s * a.dst_ld_bytes, src, (uint32_t)a.row_bytes);
    }
    bulk_commit();
  }
  bulk_wait_all();
}

struct PushDev {
  RowMapDev m;
  const int* ids;
  const int* n_ptr;
  int64_t n_max;
  const unsigned char* cur;   // trained rows  [n x ld_bytes]
  const unsigned char* old;   // pulled rows
  int64_t ld_bytes;
  int row_bytes;
  float scale;
  int q;
  int br;
};
constexpr int kPushComputeWarps = 4;

__global__ void __launch_bounds__(32 * (1 + kPushComputeWarps), 1)
rows_push_delta_bulk_kernel(const __grid_constant__ PushDev a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int Q = a.q;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);         // loads landed
  uint64_t* ready = full + Q;                                 // deltas computed (kPushComputeWarps arrivals)
  int* nz = reinterpret_cast<int*>(smem + 256);               // [Q][32] row has a non-zero delta
  unsigned char* stage = smem + 256 + Q * 32 * 4;
  stage = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(stage) + 127) / 128 * 128);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int BR = a.br;
  const size_t batch_bytes = (size_t)BR * a.row_bytes;        // cur block, then old block
  if (threadIdx.x == 0) {
    for (int s = 0; s < Q; ++s) {
      mbar_init(full + s, 1);
      mbar_init(ready + s, kPushComputeWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  int64_t n = a.n_ptr ? (int64_t)*a.n_ptr : a.n_max;
  if (n > a.n_max) n = a.n_max;
  const int64_t n_batches = (n + BR - 1) / BR;
  const int64_t mine = n_batches > blockIdx.x ? (n_batches - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const bool contig = a.ld_bytes == a.row_bytes;

  if (warp == 0) {
    // ---------------- issuer: loads of batch t+Q-1, reductions of batch t ----------------
    auto issue_load = [&](int64_t t) {
      const int q = (int)(t % Q);
      const int64_t s0 = (blockIdx.x + t * gridDim.x) * BR;
      const int rows = (int)((n - s0) < BR ? (n - s0) : BR);
      unsigned char* c0 = stage + (size_t)q * 2 * batch_bytes;
      if (lane == 0) mbar_arrive_expect_tx(full + q, 2u * (uint32_t)rows * (uint32_t)a.row_bytes);
      __syncwarp();
      if (contig) {
        if (lane == 0) {                                       // the batch is contiguous in both caches
          bulk_g2s(c0, a.cur + s0 * a.ld_bytes, (uint32_t)rows * (uint32_t)a.row_bytes, full + q);
          bulk_g2s(c0 + batch_bytes, a.old + s0 * a.ld_bytes, (uint32_t)rows * (uint32_t)a.row_bytes, full + q);
        }
      } else if (lane < rows) {
        unsigned char* c = c0 + (size_t)lane * a.row_bytes;
        bulk_g2s(c, a.cur + (s0 + lane) * a.ld_bytes, (uint32_t)a.row_bytes, full + q);
        bulk_g2s(c + batch_bytes, a.old + (s0 + lane) * a.ld_bytes, (uint32_t)a.row_bytes, full + q);
      }
    };
    const int64_t pre = mine < Q - 1 ? mine : Q - 1;
    for (int64_t t = 0; t < pre; ++t) issue_load(t);
    for (int64_t t = 0; t < mine; ++t) {
      const int64_t tn = t + Q - 1;
      if (tn < mine) {
        if (tn >= Q) {
          // stage (tn % Q) held batch tn-Q = t-1: its reductions must have read the deltas
          bulk_wait_read<0>();
          __syncwarp();
        }
        issue_load(tn);
      }
      const int q = (int)(t % Q);
      mbar_wait(ready + q, (uint32_t)((t / Q) & 1));
      const int64_t s = (blockIdx.x + t * gridDim.x) * BR + lane;
      const bool in = lane < BR && s < n;
      const int64_t r = in ? (int64_t)__ldg(a.ids + s) : -1;
      const bool have = in && r >= 0 && r < a.m.num_row;
      uint32_t hmask;
      const int len = row_runs(a.m, r, have, lane, hmask);
      const uint32_t nzmask = __ballot_sync(0xffffffffu, have && nz[q * 32 + lane] != 0);
      if (len > 0) {
        const uint32_t run = (len >= 32 ? 0xffffffffu : ((1u << len) - 1u)) << lane;
        if (run & nzmask)                                       // an untouched run adds nothing: skip it
          bulk_reduce_add_s2g(row_addr(a.m, r), stage + (size_t)q * 2 * batch_bytes + (size_t)lane * a.row_bytes,
                              (uint32_t)len * (uint32_t)a.row_bytes);
      }
      bulk_commit();
    }
    bulk_wait_all();
  } else {
    // ---------------- compute warps: delta = (cur - old) * scale, in place over cur ----------------
    const int cw = warp - 1;
    const int nvec = a.row_bytes >> 4;
    for (int64_t t = 0; t < mine; ++t) {
      const int q = (int)(t % Q);
      mbar_wait(full + q, (uint32_t)((t / Q) & 1));
      unsigned char* cb = stage + (size_t)q * 2 * batch_bytes;
      const int64_t s0 = (blockIdx.x + t * gridDim.x) * BR;
      for (int row = cw; row < BR; row += kPushComputeWarps) {
        if (s0 + row >= n) break;
        float4* c = reinterpret_cast<float4*>(cb + (size_t)row * a.row_bytes);
        const float4* o = reinterpret_cast<const float4*>(cb + batch_bytes + (size_t)row * a.row_bytes);
        int any = 0;
        for (int v = lane; v < nvec; v += 32) {
          float4 x = c[v];
          const float4 y = o[v];
          x.x = (x.x - y.x) * a.scale; x.y = (x.y - y.y) * a.scale;
          x.z = (x.z - y.z) * a.scale; x.w = (x.w - y.w) * a.scale;
          any |= (x.x != 0.f) | (x.y != 0.f) | (x.z != 0.f) | (x.w != 0.f);
          c[v] = x;
        }
        any = __any_sync(0xffffffffu, any);
        if (lane == 0) nz[q * 32 + row] = any;
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(ready + q);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Register-path variants (no shared memory, <= 40 registers): these CTAs co-reside with the persistent
// K7 CTAs (which own the SMs' shared memory but leave threads and registers), so the pull of block i+1 and
// the push of block i-1 use the memory-level parallelism of ALL SMs instead of a few reserved ones.
// Warp per row, 128-bit accesses, two rows in flight per warp.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSideThreads, 9)
rows_pull_lsu_kernel(const __grid_constant__ PullDev a) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  int64_t n = a.n_ptr ? (int64_t)*a.n_ptr : a.n_max;
  if (n > a.n_max) n = a.n_max;
  const int nvec = a.row_bytes >> 4;
  for (int64_t s = warp * 2; s < n; s += nwarps * 2) {
    const unsigned char* src[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      src[u] = nullptr;
      if (s + u < n) {
        const int64_t r = (int64_t)__ldg(a.ids + s + u);
        if (r >= 0 && r < a.m.num_row) src[u] = row_addr(a.m, r);
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

__global__ void __launch_bounds__(kSideThreads, 9)
rows_push_delta_lsu_kernel(const __grid_constant__ PushDev a) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  int64_t n = a.n_ptr ? (int64_t)*a.n_ptr : a.n_max;
  if (n > a.n_max) n = a.n_max;
  const int nvec = a.row_bytes >> 4;
  for (int64_t s = warp; s < n; s += nwarps) {
    const int64_t r = (int64_t)__ldg(a.ids + s);
    if (r < 0 || r >= a.m.num_row) continue;
    float* dst = reinterpret_cast<float*>(row_addr(a.m, r));
    const unsigned char* c = a.cur + s * a.ld_bytes;
    const unsigned char* o = a.old + s * a.ld_bytes;
    for (int v0 = 0; v0 < nvec; v0 += 96) {
      float4 x[3], y[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int v = v0 + lane + 32 * j;
        if (v < nvec) {
          x[j] = *reinterpret_cast<const float4*>(c + (size_t)v * 16);
          y[j] = *reinterpret_cast<const float4*>(o + (size_t)v * 16);
        }
      }
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const int v = v0 + lane + 32 * j;
        if (v < nvec) {
          float4 d;
          d.x = (x[j].x - y[j].x) * a.scale; d.y = (x[j].y - y[j].y) * a.scale;
          d.z = (x[j].z - y[j].z) * a.scale; d.w = (x[j].w - y[j].w) * a.scale;
          if (d.x != 0.f || d.y != 0.f || d.z != 0.f || d.w != 0.f) red_add_v4_f32(dst + (size_t)v * 4, d);
        }
      }
    }
  }
}

RowMapDev to_dev(const MvbRowMap* m, int esz) {
  RowMapDev d{};
  d.num_row = m->num_row;
  d.S = m->nservers;
  d.rps = m->rows_per_server > 0 ? m->rows_per_server : 1;
  d.ld_bytes = m->num_col * esz;
  for (int s = 0; s < MVB_MAX_RANKS; ++s)
    d.shard[s] = s < m->nservers ? reinterpret_cast<unsigned char*>(m->shard_ptrs[s]) : nullptr;
  return d;
}

int max_optin_smem() {
  int dev = 0, v = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  return v;
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

// Gather rows ids[0..n) of a row-sharded fp32/any-4-byte table into dst_a (and dst_b) over the bulk-copy
// engine.  n is read on the device from n_ptr when given (clamped to n_max).  Row bytes must be a
// multiple of 16.  max_ctas bounds the grid (0: 16 CTAs).
extern "C" int mvb_rows_pull_bulk(const MvbRowMap* m, int esz, const int* ids, const int* n_ptr, int64_t n_max,
                                  void* dst_a, void* dst_b, int64_t dst_ld, int max_ctas, void* stream) {
  if (n_max <= 0) return 0;
  const int64_t row_bytes = m->num_col * esz;
  if (row_bytes % 16 || (dst_ld * esz) % 16 || row_bytes > 16384) return -9;
  if ((reinterpret_cast<uintptr_t>(dst_a) & 15) || (reinterpret_cast<uintptr_t>(dst_b) & 15)) return -9;
  PullDev a{};
  a.m = to_dev(m, esz);
  a.ids = ids; a.n_ptr = n_ptr; a.n_max = n_max;
  a.dst_a = (unsigned char*)dst_a; a.dst_b = (unsigned char*)dst_b; a.dst_ld_bytes = dst_ld * esz;
  a.row_bytes = (int)row_bytes;
  if (max_ctas < 0) {          // register path: -max_ctas CTAs per SM, co-resident with K7
    a.q = 0; a.br = 32;
    const int g = mvb_num_sms() * (-max_ctas);
    rows_pull_lsu_kernel<<<g, kSideThreads, 0, (cudaStream_t)stream>>>(a);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  }
  const int budget = max_optin_smem() - 128;
  int br = 32, q = 0;
  for (; br >= 4; br >>= 1) {
    q = (int)(budget / (br * row_bytes));
    if (q >= 3) break;
  }
  if (q > 8) q = 8;
  if (q < 3) return -22;
  a.q = q; a.br = br;
  const size_t smem = 128 + (size_t)q * br * row_bytes;
  int grid = max_ctas > 0 ? max_ctas : 16;
  const int64_t nb = (n_max + br - 1) / br;
  if ((int64_t)grid > nb) grid = (int)nb;
  MVB_CUDA_CHECK(cudaFuncSetAttribute(rows_pull_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  rows_pull_bulk_kernel<<<grid, 32, smem, (cudaStream_t)stream>>>(a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// rows[ids[s]] += (cur[s] - old[s]) * scale for s in [0, n): fused AddDeltaParameter on the bulk engine.
extern "C" int mvb_rows_push_delta_bulk(const MvbRowMap* m, const int* ids, const int* n_ptr, int64_t n_max,
                                        const float* cur, const float* old, int64_t ld, float scale, int max_ctas,
                                        void* stream) {
  if (n_max <= 0) return 0;
  const int64_t row_bytes = m->num_col * 4;
  if (row_bytes % 16 || (ld * 4) % 16 || row_bytes > 16384) return -9;
  if ((reinterpret_cast<uintptr_t>(cur) & 15) || (reinterpret_cast<uintptr_t>(old) & 15)) return -9;
  PushDev a{};
  a.m = to_dev(m, 4);
  a.ids = ids; a.n_ptr = n_ptr; a.n_max = n_max;
  a.cur = (const unsigned char*)cur; a.old = (const unsigned char*)old; a.ld_bytes = ld * 4;
  a.row_bytes = (int)row_bytes; a.scale = scale;
  if (max_ctas < 0) {
    a.q = 0; a.br = 32;
    const int g = mvb_num_sms() * (-max_ctas);
    rows_push_delta_lsu_kernel<<<g, kSideThreads, 0, (cudaStream_t)stream>>>(a);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  }
  const int budget = max_optin_smem() - 1024;
  int br = 32, q = 0;
  for (; br >= 4; br >>= 1) {
    q = (int)(budget / (2 * br * row_bytes + 128));
    if (q >= 2) break;
  }
  if (q > 4) q = 4;
  if (q < 2) return -22;
  a.q = q; a.br = br;
  const size_t smem = 256 + (size_t)q * 32 * 4 + 128 + (size_t)q * 2 * br * row_bytes;
  int grid = max_ctas > 0 ? max_ctas : 16;
  const int64_t nb = (n_max + br - 1) / br;
  if ((int64_t)grid > nb) grid = (int)nb;
  MVB_CUDA_CHECK(cudaFuncSetAttribute(rows_push_delta_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
  rows_push_delta_bulk_kernel<<<grid, 32 * (1 + kPushComputeWarps), smem, (cudaStream_t)stream>>>(a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
