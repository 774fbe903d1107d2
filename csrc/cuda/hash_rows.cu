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
// race for a Zipf head key at first touch never over-count. A slot is only freed by an eviction, which leaves it
// with zero updater state, so the updater state rows of a new key are zero.
//
// Lanes of a warp that carry the same (table, key) are merged with __match_any_sync: one lane probes and the
// row is broadcast, so a Zipf head repeated thousands of times costs one probe per warp.
//
// Access clock (a descriptor with last_seen): an inserting lookup stamps every key it resolves. The claimer stores
// last_seen[j] = clock before its release of ready[j]; a lookup that finds the key raises last_seen[j] to its
// clock with atomicMax_system, after a plain load shows it older, so a Zipf head costs about one atomic per clock
// value rather than one per warp. Stamps of ranks at different clocks combine by max.
//
// Admission (a descriptor with admit_after >= 2): a count-min sketch per server, 4 rows of W uint32 counters and a
// uint64 total, next to keys / ready / count. An inserting call runs hash_count_keys_kernel first: with the same grid
// and lane merge as the lookup, the leader of each group of equal (table, key) probes read-only and, when the key
// holds no slot, adds the group's size to the key's 4 counters and to the total at the owner. The translation then
// claims an empty slot for such a key only when its estimate (the minimum of its counters) reaches admit_after; a
// key below it reads the zero row and leaves no trace. Counting a whole call before admitting any of it makes the
// outcome per call: on one rank every occurrence of a key sees the same estimate. The counter of row r is
// (hash64(key + (r + 1) golden) >> 32) & (W - 1): the high half of a hash of a shifted key, unrelated to the probe
// home (the low bits of mix64(key)) and to the owner (key mod S). mvb_hash_rows_age then halves (TinyLFU's reset)
// every server whose total reached W / 2.
//
// Eviction (mvb_hash_rows_mark, mvb_hash_rows_evict) runs between barriers, with no lookup in flight. Marking sets
// ready[j] = 3 for the listed keys; the rebuild of a server then removes marked, refused and idle slots with the
// textbook in-place rehash of linear probing, one warp per cluster of non-empty slots (see mvb200.h). A cluster
// starts after an empty slot, so a survivor's probe from its home stays inside the part of the cluster already
// walked: survivors only move back toward their homes, never onto a slot not yet walked, and no copy of the shard
// or the state is needed.
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

// ready[j]: 0 while the claimer initialises the row (or for an empty slot); kMarked only during an eviction
constexpr uint32_t kReady = 1, kRefused = 2, kMarked = 3;

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

// ---- admission ----------------------------------------------------------------------------------------------------
MVB_DEVINL uint32_t* sketch_cell(const MvbHashRows& h, int s, long long key, int r) {
  const uint64_t W = (uint64_t)h.width;
  const uint64_t c = (hash64((uint64_t)key + (uint64_t)(r + 1) * 0x9E3779B97F4A7C15ull) >> 32) & (W - 1);
  return reinterpret_cast<uint32_t*>(h.sketch[s]) + (uint64_t)r * W + c;
}

MVB_DEVINL bool admitted(const MvbHashRows& h, int s, long long key) {
  if (h.admit_after < 2) return true;
  uint32_t e = 0xffffffffu;
#pragma unroll
  for (int r = 0; r < 4; ++r) e = min(e, *reinterpret_cast<volatile uint32_t*>(sketch_cell(h, s, key, r)));
  return e >= (uint32_t)h.admit_after;
}

// whether `key` holds a slot (ready, being initialised or refused) at its owner: a probe that claims nothing
MVB_DEVINL bool holds_slot(const MvbHashRows& h, long long key) {
  const long long* keys = reinterpret_cast<const long long*>(h.keys[owner_of(key, h.nservers)]);
  const uint64_t mask = (uint64_t)h.slots - 1;
  uint64_t j = mix64((uint64_t)key) & mask;
  for (int64_t probe = 0; probe < h.slots; ++probe, j = (j + 1) & mask) {
    const long long cur = *reinterpret_cast<const volatile long long*>(keys + j);
    if (cur == key) return true;
    if (cur == kEmpty) return false;
  }
  return false;
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
      if (!insert || !admitted(h, s, key)) return zero_row;        // not admitted yet: missing, not an error
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
        if (h.last_seen[s]) reinterpret_cast<long long*>(h.last_seen[s])[j] = *h.clock;
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
      if (insert && h.last_seen[s]) {
        long long* ls = reinterpret_cast<long long*>(h.last_seen[s]) + j;
        const long long now = *h.clock;
        if (*reinterpret_cast<volatile long long*>(ls) < now) atomicMax_system(ls, now);
      }
      return (int64_t)s * P + (int64_t)j;
    }
  }
  if (insert && admitted(h, s, key)) set_status(status, MVB_HASH_FULL, t, s);   // a whole chain without an empty slot
  return zero_row;
}

// the descriptor of lookup i (-1: a row id copied unchanged), -2 past the end
MVB_DEVINL int table_of(const MvbHashLookup& a, int64_t i) {
  if (i >= a.n) return -2;
  if (!a.seg_end) return 0;
  int lo = 0, hi = a.G - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (i < a.seg_end[mid]) hi = mid; else lo = mid + 1;
  }
  return a.seg_table[lo];
}

MVB_DEVINL int effective_insert(const MvbHashLookup& a) {
  return a.insert && (a.insert_ok == nullptr || *a.insert_ok != 0);
}

// the count pass of an inserting call: the grid and lane groups of hash_lookup_kernel
__global__ void __launch_bounds__(256) hash_count_keys_kernel(const __grid_constant__ MvbHashLookup a) {
  if (!effective_insert(a)) return;
  const int lane = threadIdx.x & 31;
  for (int64_t base = warp_id() * 32; base < a.n; base += num_warps() * 32) {
    const int64_t i = base + lane;
    const int t = table_of(a, i);
    const long long key = t != -2 ? (long long)a.keys[i] : 0;
    const unsigned same = __match_any_sync(0xffffffffu, key) & __match_any_sync(0xffffffffu, t);
    if (t < 0 || lane != __ffs(same) - 1 || key == kEmpty) continue;
    const MvbHashRows& h = a.tables[t];
    if (h.admit_after < 2 || holds_slot(h, key)) continue;
    const int s = owner_of(key, h.nservers);
    const unsigned n = __popc(same);
#pragma unroll
    for (int r = 0; r < 4; ++r) atomicAdd_system(sketch_cell(h, s, key, r), n);
    atomicAdd_system(reinterpret_cast<unsigned long long*>(h.total[s]), (unsigned long long)n);
  }
}

__global__ void __launch_bounds__(256) hash_lookup_kernel(const __grid_constant__ MvbHashLookup a,
                                                          long long budget) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int insert = effective_insert(a);
  for (int64_t base = warp * 32; base < a.n; base += nwarps * 32) {
    const int64_t i = base + lane;
    const bool valid = i < a.n;
    const long long key = valid ? (long long)a.keys[i] : 0;
    const int t = table_of(a, i);
    const unsigned same = __match_any_sync(0xffffffffu, key) & __match_any_sync(0xffffffffu, t);
    const int leader = __ffs(same) - 1;
    int64_t row = 0;
    if (valid && lane == leader)
      row = t < 0 ? (int64_t)key : translate(a.tables[t], t, key, insert, a.status, budget);
    row = __shfl_sync(0xffffffffu, row, leader);
    if (valid) a.rows[i] = row;
  }
}

// Aging, part 1: thread s elects itself to shift server s (a CAS of the total from what it read to the shifted value)
// and leaves the shift, 0 when the total is below W / 2 or another caller won, in age[s]
__global__ void hash_age_elect_kernel(const __grid_constant__ MvbHashRows h) {
  const int s = threadIdx.x;
  if (s >= h.nservers) return;
  unsigned long long* tot = reinterpret_cast<unsigned long long*>(h.total[s]);
  const unsigned long long R = (unsigned long long)h.width >> 1;
  unsigned k = 0;
  unsigned long long old = *reinterpret_cast<volatile unsigned long long*>(tot);
  while (old >= R) {
    unsigned kk = 1;
    while ((old >> kk) >= R) ++kk;
    const unsigned long long seen = atomicCAS_system(tot, old, old >> kk);
    if (seen == old) {
      k = kk;
      break;
    }
    old = seen;                                       // a count landed in between: decide again
  }
  reinterpret_cast<uint32_t*>(h.age)[s] = k;
}

// Aging, part 2: the elected servers' counters shifted by CAS, so a concurrent count is shifted or kept, never lost
__global__ void __launch_bounds__(256) hash_age_shift_kernel(const __grid_constant__ MvbHashRows h) {
  const int64_t n = 4 * h.width, stride = (int64_t)gridDim.x * blockDim.x;
  for (int s = 0; s < h.nservers; ++s) {
    const uint32_t k = reinterpret_cast<const uint32_t*>(h.age)[s];
    if (!k) continue;
    uint32_t* c = reinterpret_cast<uint32_t*>(h.sketch[s]);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
      uint32_t old = *reinterpret_cast<volatile uint32_t*>(c + i);
      while (old) {
        const uint32_t seen = atomicCAS_system(c + i, old, k < 32 ? old >> k : 0u);
        if (seen == old) break;
        old = seen;
      }
    }
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

// ---- eviction ---------------------------------------------------------------------------------------------------

__global__ void hash_mark_kernel(const __grid_constant__ MvbHashRows h, const int64_t* keys, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const uint64_t mask = (uint64_t)h.slots - 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long key = keys[i];
    if (key == kEmpty) continue;
    const int s = owner_of(key, h.nservers);
    const long long* ks = reinterpret_cast<const long long*>(h.keys[s]);
    volatile uint32_t* ready = reinterpret_cast<volatile uint32_t*>(h.ready[s]);
    uint64_t j = mix64((uint64_t)key) & mask;
    for (int64_t probe = 0; probe < h.slots; ++probe, j = (j + 1) & mask) {
      const long long cur = ks[j];
      if (cur == kEmpty) break;
      if (cur == key) {
        if (ready[j] == kReady) ready[j] = kMarked;   // a refused slot is a victim anyway, and holds no live key
        break;
      }
    }
  }
}

// One server's index and the payload that moves with a slot: its row, its state rows, its last_seen.
struct EvictArgs {
  long long* keys;
  uint32_t* ready;
  long long* ls;            // or nullptr
  float* rows;              // local row j = slot j, num_col floats
  int64_t num_col;
  float* st[2];             // state arrays, or nullptr
  int n_slabs;
  int64_t stride, srow;     // elements between slabs; elements per state row
  int64_t P;
  long long older_than;     // INT64_MIN: no age rule
  int64_t* counts;          // {live keys removed, survivors moved}
  long long* work;          // {clusters, first victim, cluster starts...}
  float* st2;               // a state slab with its own row length (adam's step counts), or nullptr
  int64_t srow2;
};

MVB_DEVINL void copy_f32(float* dst, const float* src, int64_t n, int lane) {
  if ((n & 3) == 0) {
    for (int64_t c = (int64_t)lane * 4; c < n; c += 128) st_v4(dst + c, ld_v4(src + c));
  } else {
    for (int64_t c = lane; c < n; c += 32) dst[c] = src[c];
  }
}
MVB_DEVINL void zero_f32(float* dst, int64_t n, int lane) {
  if ((n & 3) == 0) {
    for (int64_t c = (int64_t)lane * 4; c < n; c += 128) st_v4(dst + c, make_uint4(0, 0, 0, 0));
  } else {
    for (int64_t c = lane; c < n; c += 32) dst[c] = 0.f;
  }
}

// Empty slot j: zero state rows and last_seen, the empty key (the row keeps whatever it holds). Whole warp.
MVB_DEVINL void clear_slot(const EvictArgs& e, int64_t j, int lane) {
  for (int a = 0; a < 2; ++a)
    if (e.st[a])
      for (int k = 0; k < e.n_slabs; ++k) zero_f32(e.st[a] + k * e.stride + j * e.srow, e.srow, lane);
  if (e.st2) zero_f32(e.st2 + j * e.srow2, e.srow2, lane);
  if (lane == 0) {
    e.keys[j] = kEmpty;
    e.ready[j] = 0;
    if (e.ls) e.ls[j] = 0;
  }
  __syncwarp();
}

// Slot `from` moves to the empty slot `to`, then `from` is cleared. Whole warp.
MVB_DEVINL void move_slot(const EvictArgs& e, int64_t to, int64_t from, int lane) {
  copy_f32(e.rows + to * e.num_col, e.rows + from * e.num_col, e.num_col, lane);
  for (int a = 0; a < 2; ++a)
    if (e.st[a])
      for (int k = 0; k < e.n_slabs; ++k) {
        float* slab = e.st[a] + k * e.stride;
        copy_f32(slab + to * e.srow, slab + from * e.srow, e.srow, lane);
      }
  if (e.st2) copy_f32(e.st2 + to * e.srow2, e.st2 + from * e.srow2, e.srow2, lane);
  if (lane == 0) {
    e.keys[to] = e.keys[from];
    e.ready[to] = e.ready[from];
    if (e.ls) e.ls[to] = e.ls[from];
  }
  __syncwarp();
  clear_slot(e, from, lane);
}

// Pass 1, before any slot changes: idle live keys become marked; live victims are counted (and leave the server's
// count); every cluster start (a non-empty slot after an empty one) is listed; the lowest victim slot is kept for
// an index without an empty slot.
__global__ void hash_evict_scan_kernel(const EvictArgs e, unsigned long long* count) {
  const int lane = threadIdx.x & 31;
  const uint64_t mask = (uint64_t)e.P - 1;
  const int64_t n32 = (e.P + 31) & ~(int64_t)31;
  int64_t removed = 0;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n32; j += (int64_t)gridDim.x * blockDim.x) {
    bool live_victim = false, victim = false, start = false;
    if (j < e.P) {
      const long long k = e.keys[j];
      if (k != kEmpty) {
        uint32_t r = e.ready[j];
        if (r == kReady && e.ls && e.ls[j] < e.older_than) {
          r = kMarked;
          e.ready[j] = kMarked;
        }
        victim = r != kReady;
        live_victim = r == kMarked;
        start = e.keys[(j - 1) & mask] == kEmpty;
      }
    }
    const unsigned vb = __ballot_sync(0xffffffffu, live_victim), sb = __ballot_sync(0xffffffffu, start);
    removed += __popc(vb);
    const unsigned first = __reduce_min_sync(0xffffffffu, victim ? (unsigned)j : 0xffffffffu);
    long long base = 0;
    if (lane == 0) {
      if (first != 0xffffffffu) atomicMin(reinterpret_cast<unsigned long long*>(e.work + 1), first);
      if (sb) base = (long long)atomicAdd(reinterpret_cast<unsigned long long*>(e.work), (unsigned long long)__popc(sb));
    }
    base = __shfl_sync(0xffffffffu, base, 0);
    if (start) e.work[2 + base + __popc(sb & ((1u << lane) - 1))] = j;
  }
  if (lane == 0 && removed) {
    atomicAdd(reinterpret_cast<unsigned long long*>(e.counts), (unsigned long long)removed);
    atomicAdd(count, (unsigned long long)-removed);
  }
}

// An index without an empty slot has no cluster to cut. Its lowest victim v is deleted by backward shifting
// (Knuth's Algorithm R for linear probing): walking on from the hole, an entry whose home is not cyclically in
// (hole, j] moves into the hole, which then moves to j. The walk ends at the first empty slot, which is the last
// hole; the rest of the index is then one cluster starting after it. One warp.
__global__ void hash_evict_unwrap_kernel(const EvictArgs e) {
  const int lane = threadIdx.x & 31;
  if (e.work[0] != 0 || (unsigned long long)e.work[1] >= (unsigned long long)e.P) return;   // clusters, or no victim
  const uint64_t mask = (uint64_t)e.P - 1;
  const int64_t v = e.work[1];
  clear_slot(e, v, lane);
  int64_t hole = v, j = v;
  long long moved = 0;
  while (true) {
    j = (j + 1) & mask;
    const long long k = e.keys[j];
    if (k == kEmpty) break;
    const int64_t home = (int64_t)(mix64((uint64_t)k) & mask);
    const bool stays = hole <= j ? (hole < home && home <= j) : (hole < home || home <= j);
    if (!stays) {
      moved += e.ready[j] == kReady;
      move_slot(e, hole, j, lane);
      hole = j;
    }
  }
  if (lane == 0) {
    e.work[0] = 1;
    e.work[2] = (hole + 1) & mask;
    if (moved) atomicAdd(reinterpret_cast<unsigned long long*>(e.counts + 1), (unsigned long long)moved);
  }
}

// Pass 2: a warp walks each cluster from its first slot to the empty slot after it. Slots ahead of the walk are
// still as pass 1 saw them (moves only go backwards), so the walk ends where the old cluster did. Until the first
// victim every survivor stays, so the walk skips 32 slots per ballot; after it, each survivor probes from its home
// with ballots over 32 slots for the first empty slot before its own and moves there.
// (256, 1): without the minimum the compiler holds the walk to 64 registers and spills
__global__ void __launch_bounds__(256, 1) hash_evict_walk_kernel(const EvictArgs e) {
  const int lane = threadIdx.x & 31;
  const uint64_t mask = (uint64_t)e.P - 1;
  long long moved = 0;
  const long long nclusters = *reinterpret_cast<volatile long long*>(e.work);
  for (long long c = warp_id(); c < nclusters; c += num_warps()) {
    uint64_t x = (uint64_t)e.work[2 + c];
    // survivors before the cluster's first victim keep their slots
    bool done = false;
    while (true) {
      const uint64_t j = (x + lane) & mask;
      const long long k = e.keys[j];
      const uint32_t r = e.ready[j];
      const unsigned eb = __ballot_sync(0xffffffffu, k == kEmpty);
      unsigned vb = __ballot_sync(0xffffffffu, k != kEmpty && r != kReady);
      if (eb) vb &= (1u << (__ffs(eb) - 1)) - 1;     // the cluster ends at its first empty slot
      if (vb) {
        x += __ffs(vb) - 1;
        break;
      }
      if (eb) {
        done = true;
        break;
      }
      x += 32;
    }
    if (done) continue;
    for (;; ++x) {
      const uint64_t j = x & mask;
      const long long k = e.keys[j];
      if (k == kEmpty) break;
      if (e.ready[j] != kReady) {
        clear_slot(e, (int64_t)j, lane);
        continue;
      }
      const uint64_t home = mix64((uint64_t)k) & mask;
      const uint64_t dist = (j - home) & mask;               // the old chain home .. j has no empty slot
      for (uint64_t d0 = 0; d0 < dist; d0 += 32) {
        const uint64_t d = d0 + lane;
        const bool free = d < dist && e.keys[(home + d) & mask] == kEmpty;
        const unsigned fb = __ballot_sync(0xffffffffu, free);
        if (fb) {
          move_slot(e, (int64_t)((home + d0 + __ffs(fb) - 1) & mask), (int64_t)j, lane);
          ++moved;
          break;
        }
      }
    }
  }
  if (lane == 0 && moved) atomicAdd(reinterpret_cast<unsigned long long*>(e.counts + 1), (unsigned long long)moved);
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
  if (a->admit) {
    hash_count_keys_kernel<<<blocks_for(a->n, 256, 8), 256, 0, (cudaStream_t)stream>>>(*a);
    MVB_CUDA_CHECK(cudaGetLastError());
  }
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

static int check_index(const MvbHashRows* h) {
  if (h->nservers < 1 || h->nservers > MVB_MAX_RANKS) return -3;
  if (h->slots < 2 || h->slots > (int64_t(1) << 31) || (h->slots & (h->slots - 1))) return -4;
  return 0;
}

extern "C" int mvb_hash_rows_age(const MvbHashRows* h, void* stream) {
  if (int rc = check_index(h)) return rc;
  if (h->admit_after < 2) return -7;
  if (h->width < 2 || h->width > (int64_t(1) << 31) || (h->width & (h->width - 1))) return -8;
  if (!h->age) return -9;
  for (int s = 0; s < h->nservers; ++s)
    if (!h->sketch[s] || !h->total[s]) return -9;
  cudaStream_t st = (cudaStream_t)stream;
  hash_age_elect_kernel<<<1, MVB_MAX_RANKS, 0, st>>>(*h);
  MVB_CUDA_CHECK(cudaGetLastError());
  hash_age_shift_kernel<<<blocks_for(4 * h->width, 256, 4), 256, 0, st>>>(*h);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_hash_rows_mark(const MvbHashRows* h, const int64_t* keys, int64_t n, void* stream) {
  if (int rc = check_index(h)) return rc;
  if (n <= 0) return 0;
  hash_mark_kernel<<<blocks_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(*h, keys, n);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_hash_rows_evict(const MvbHashRows* h, int server, int64_t older_than, void* state0, void* state1,
                                   int n_slabs, int64_t state_stride, int64_t state_row, int64_t* counts,
                                   int64_t* work, void* stream) {
  return mvb_hash_rows_evict_ex(h, server, older_than, state0, state1, n_slabs, state_stride, state_row, counts, work,
                                stream, nullptr, 0);
}

extern "C" int mvb_hash_rows_evict_ex(const MvbHashRows* h, int server, int64_t older_than, void* state0,
                                      void* state1, int n_slabs, int64_t state_stride, int64_t state_row,
                                      int64_t* counts, int64_t* work, void* stream, void* state2,
                                      int64_t state2_row) {
  if (int rc = check_index(h)) return rc;
  if (server < 0 || server >= h->nservers) return -1;
  const MvbRowMap& m = h->map;
  if (!row_split_ok(m.nservers, m.rows_per_server) || m.nservers != h->nservers || m.rows_per_server < h->slots ||
      m.num_col < 4 || m.num_col % 4)
    return MVB_BAD_ROW_MAP;
  if (older_than != INT64_MIN && !h->last_seen[server]) return -5;
  if ((state0 || state1) && (n_slabs < 1 || state_row < 1 || (n_slabs > 1 && state_stride < h->slots * state_row)))
    return -6;
  if (state2 && state2_row < 1) return -6;
  cudaStream_t st = (cudaStream_t)stream;
  const EvictArgs e{(long long*)h->keys[server], (uint32_t*)h->ready[server], (long long*)h->last_seen[server],
                    (float*)m.shard_ptrs[server], m.num_col, {(float*)state0, (float*)state1}, n_slabs,
                    state_stride, state_row, h->slots, (long long)older_than, counts, (long long*)work,
                    (float*)state2, state2_row};
  MVB_CUDA_CHECK(cudaMemsetAsync(counts, 0, 16, st));
  MVB_CUDA_CHECK(cudaMemsetAsync(work, 0, 8, st));              // no cluster yet
  MVB_CUDA_CHECK(cudaMemsetAsync(work + 1, 0xff, 8, st));       // no victim yet
  hash_evict_scan_kernel<<<blocks_for(h->slots, 256, 8), 256, 0, st>>>(e, (unsigned long long*)h->count[server]);
  MVB_CUDA_CHECK(cudaGetLastError());
  hash_evict_unwrap_kernel<<<1, 32, 0, st>>>(e);
  MVB_CUDA_CHECK(cudaGetLastError());
  hash_evict_walk_kernel<<<grid_for(h->slots / 2), 256, 0, st>>>(e);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
