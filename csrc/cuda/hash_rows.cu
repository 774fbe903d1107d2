// multiverso-b200 :: the hash index of a HashMatrixTable: int64 keys -> rows of an fp32 MatrixTable.
//
// The KVTable's layout (kv.cu) with a row instead of a scalar per slot: server owner_of(key, S) holds a key,
// probing is linear from mix64(key), and slot j of server s IS row s P + j of the table, so once a key has a
// slot every row kernel (gather-pool, coalesced backward, updaters, mailboxes) works on it unchanged.
//
// Inserting a key (insert = 1) at the first empty slot j of its chain:
//   1. a server whose live-key counter is at floor(7 P / 8) refuses it ("table full") and takes no slot;
//   2. CAS keys[j] from empty to the key (system scope: the owner may be a peer);
//   3. the winner counts the key; inserts that raced past the limit mark the slot refused (ready[j] = 2, the key
//      stays as a tombstone so probe chains stay intact, and is never given a row: a later insert of it reports
//      "table full", a lookup that does not insert reads it as missing);
//   4. otherwise the winner writes the row's initial value into the owner's shard with 16-byte stores, then
//      fence.acq_rel.sys and st.release.sys of ready[j] = 1.
// Every other thread that meets the key (in this launch or on another rank) waits for ready[j] with an acquire
// spin under the clock64 watchdog of spin_wait_ge, so no row is returned before its initial value is visible.
// The counter only ever holds keys that got a row: a CAS comes before the count, so the thousands of lanes that
// race for a Zipf head key at first touch never over-count. Slots are never freed, so the updater state rows of
// a new key are still zero from allocation.
//
// Lanes of a warp that carry the same (table, key) are merged with __match_any_sync: one lane probes and the
// row is broadcast, so a Zipf head repeated thousands of times costs one probe per warp.
#include "mvb_common.cuh"

namespace {

constexpr long long kEmpty = (long long)0x8000000000000000ull;

MVB_DEVINL uint32_t ld_acquire_sys_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
MVB_DEVINL void st_release_sys_u32(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

constexpr uint32_t kReady = 1, kRefused = 2;   // ready[j]: 0 while the claimer initialises the row

// ready[j] once it is set (kReady / kRefused), or 0 after `budget` cycles (the backoff of spin_wait_ge)
MVB_DEVINL uint32_t wait_ready(const uint32_t* p, long long budget) {
  uint32_t r = ld_acquire_sys_u32(p);
  if (r) return r;
  const long long t0 = clock64();
  int backoff = 8;
  while (!(r = ld_acquire_sys_u32(p))) {
    __nanosleep(backoff);
    if (backoff < 256) backoff <<= 1;
    if (clock64() - t0 > budget) return 0;
  }
  return r;
}

MVB_DEVINL void set_status(int64_t* status, int kind, int table, int server) {
  const unsigned long long v = ((unsigned long long)kind << 40) | ((unsigned long long)table << 8) |
                               (unsigned long long)server;
  atomicCAS(reinterpret_cast<unsigned long long*>(status), 0ull, v);     // the first error is kept
}

// Column c of a new key's row: a pure function of the key, in explicitly rounded fp32 (no contraction).
MVB_DEVINL float init_col(const MvbHashRows& h, long long key, int64_t c) {
  if (h.init == MVB_HASH_INIT_CONST) return h.init_value;
  const uint64_t r = hash64(hash64((uint64_t)key ^ h.seed) + (uint64_t)c);
  const float u = __fmul_rn(__uint2float_rn((uint32_t)(r >> 40)), 5.9604644775390625e-8f);   // * 2^-24
  return __fadd_rn(h.lo, __fmul_rn(u, __fsub_rn(h.hi, h.lo)));
}

// The row of `key` in index `h` (descriptor `t`); the zero row when it is missing and not inserted.
MVB_DEVINL int64_t translate(const MvbHashRows& h, int t, long long key, int insert, int64_t* status,
                             long long budget) {
  const int S = h.nservers;
  const int64_t P = h.slots;
  const int64_t zero_row = (int64_t)S * P;
  if (key == kEmpty) {
    set_status(status, MVB_HASH_BAD_KEY, t, 0);
    return zero_row;
  }
  const int s = owner_of(key, S);
  long long* keys = reinterpret_cast<long long*>(h.keys[s]);
  const uint32_t* ready = reinterpret_cast<const uint32_t*>(h.ready[s]);
  unsigned long long* count = reinterpret_cast<unsigned long long*>(h.count[s]);
  const unsigned long long limit = (unsigned long long)(7 * P / 8);
  const uint64_t mask = (uint64_t)P - 1;
  uint64_t j = mix64((uint64_t)key) & mask;
  for (int64_t probe = 0; probe < P; ++probe, j = (j + 1) & mask) {
    long long cur = *reinterpret_cast<volatile long long*>(keys + j);
    if (cur == kEmpty) {
      if (!insert) return zero_row;
      if (*reinterpret_cast<volatile unsigned long long*>(count) >= limit) {   // full: take no slot
        set_status(status, MVB_HASH_FULL, t, s);
        return zero_row;
      }
      cur = (long long)atomicCAS_system(reinterpret_cast<unsigned long long*>(keys + j),
                                        (unsigned long long)kEmpty, (unsigned long long)key);
      if (cur == kEmpty) {
        // the slot is ours; the key counts once the counter admits it. Inserts racing at the limit can pass the
        // check above together: the ones past it leave the slot refused (ready = 2), never given a row
        uint32_t* rdy = const_cast<uint32_t*>(ready) + j;
        if (atomicAdd_system(count, 1ull) >= limit) {
          atomicAdd_system(count, ~0ull);
          st_release_sys_u32(rdy, kRefused);
          set_status(status, MVB_HASH_FULL, t, s);
          return zero_row;
        }
        float* row = reinterpret_cast<float*>(h.map.shard_ptrs[s]) + (int64_t)j * h.map.num_col;
        for (int64_t c = 0; c < h.map.num_col; c += 4) {
          float4 v = make_float4(init_col(h, key, c), init_col(h, key, c + 1), init_col(h, key, c + 2),
                                 init_col(h, key, c + 3));
          st_v4(row + c, *reinterpret_cast<uint4*>(&v));
        }
        fence_sys();
        st_release_sys_u32(rdy, kReady);
        return (int64_t)s * P + (int64_t)j;
      }
    }
    if (cur == key) {
      const uint32_t r = wait_ready(ready + j, budget);
      if (r == kRefused) {                   // a key refused at the limit has no row: missing, not an error
        if (insert) set_status(status, MVB_HASH_FULL, t, s);
        return zero_row;
      }
      if (r != kReady) {
        set_status(status, MVB_HASH_TIMEOUT, t, s);
        return zero_row;
      }
      return (int64_t)s * P + (int64_t)j;
    }
  }
  if (insert) set_status(status, MVB_HASH_FULL, t, s);   // a whole chain without an empty slot
  return zero_row;
}

__global__ void __launch_bounds__(256) hash_lookup_kernel(const __grid_constant__ MvbHashLookup a,
                                                          long long budget) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int insert = a.insert && (a.insert_ok == nullptr || *a.insert_ok != 0);
  for (int64_t base = warp * 32; base < a.n; base += nwarps * 32) {
    const int64_t i = base + lane;
    const bool valid = i < a.n;
    const long long key = valid ? (long long)a.keys[i] : 0;
    int t = -2;
    if (valid) {
      t = 0;
      if (a.seg_end) {
        int lo = 0, hi = a.G - 1;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (i < a.seg_end[mid]) hi = mid; else lo = mid + 1;
        }
        t = a.seg_table[lo];
      }
    }
    const unsigned same = __match_any_sync(0xffffffffu, key) & __match_any_sync(0xffffffffu, t);
    const int leader = __ffs(same) - 1;
    int64_t row = 0;
    if (valid && lane == leader)
      row = t < 0 ? (int64_t)key : translate(a.tables[t], t, key, insert, a.status, budget);
    row = __shfl_sync(0xffffffffu, row, leader);
    if (valid) a.rows[i] = row;
  }
}

__global__ void hash_init_kernel(long long* keys, uint32_t* ready, int64_t P) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < P; i += stride) {
    keys[i] = kEmpty;
    ready[i] = 0;
  }
}

__global__ void hash_count_kernel(MvbHashRows h, int64_t* out) {
  unsigned long long c = 0;
  for (int s = 0; s < h.nservers; ++s) c += *reinterpret_cast<volatile unsigned long long*>(h.count[s]);
  *out = (int64_t)c;
}

__global__ void hash_dump_kernel(const long long* keys, const uint32_t* ready, int64_t P, int64_t row_base,
                                 int64_t* out_keys, int64_t* out_rows, unsigned long long* count) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < P; j += stride) {
    const long long k = keys[j];
    if (k != kEmpty && ready[j] == kReady) {
      const unsigned long long pos = atomicAdd(count, 1ull);
      out_keys[pos] = k;
      out_rows[pos] = row_base + j;
    }
  }
}

}  // namespace

extern "C" int mvb_hash_rows_init(void* keys, void* ready, void* count, int64_t slots, void* stream) {
  if (slots <= 0 || (slots & (slots - 1))) return -4;
  cudaStream_t st = (cudaStream_t)stream;
  hash_init_kernel<<<blocks_for(slots, 256, 8), 256, 0, st>>>((long long*)keys, (uint32_t*)ready, slots);
  MVB_CUDA_CHECK(cudaGetLastError());
  MVB_CUDA_CHECK(cudaMemsetAsync(count, 0, 8, st));
  return 0;
}

extern "C" int mvb_hash_rows_lookup(const MvbHashLookup* a, void* stream) {
  if (a->n <= 0) return 0;
  hash_lookup_kernel<<<blocks_for(a->n, 256, 8), 256, 0, (cudaStream_t)stream>>>(*a,
                                                                                 watchdog_cycles(a->timeout_s, 120.0));
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_hash_rows_count(const MvbHashRows* h, int64_t* out, void* stream) {
  hash_count_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(*h, out);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_hash_rows_dump(const MvbHashRows* h, int server, int64_t* out_keys, int64_t* out_rows,
                                  int64_t* out_count, void* stream) {
  if (server < 0 || server >= h->nservers) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  MVB_CUDA_CHECK(cudaMemsetAsync(out_count, 0, 8, st));
  hash_dump_kernel<<<blocks_for(h->slots, 256, 8), 256, 0, st>>>((const long long*)h->keys[server],
                                                          (const uint32_t*)h->ready[server], h->slots,
                                                          (int64_t)server * h->slots, out_keys, out_rows,
                                                          (unsigned long long*)out_count);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
