// multiverso-b200 :: K5, the KVTable as a GPU hash table.
//
// Reference: KVWorkerTable/KVServerTable (include/multiverso/table/kv_table.h:18-118):
// keys are hash-partitioned over servers (key % num_servers), the server keeps an
// unordered_map and ProcessAdd does table_[k] += v, ProcessGet default-constructs
// missing keys.  Here every server shard is an open-addressing table in HBM
// (int64 keys, linear probing); remote shards are reached with system-scope CAS /
// atomic adds through the peer mapping, so Add/Get are single one-sided kernels.
//
// INT64_MIN marks an empty slot, so it cannot be a key: Add skips it and sets error 5003 (the rule of the hash
// index, hash_rows.cu), Get returns 0 for it without probing. A CAS of an empty slot from "empty" to INT64_MIN
// would succeed without claiming it, and the value added there would then belong to the next key in that slot.
#include "mvb_common.cuh"

namespace {

constexpr long long kEmpty = (long long)0x8000000000000000ull;

struct KVDev {
  int S;
  int64_t cap;
  long long* keys[MVB_MAX_RANKS];
  void* vals[MVB_MAX_RANKS];
};

template <typename V>
MVB_DEVINL void atomic_add_sys(V* p, V v);
template <>
MVB_DEVINL void atomic_add_sys<float>(float* p, float v) { atomicAdd_system(p, v); }
template <>
MVB_DEVINL void atomic_add_sys<double>(double* p, double v) { atomicAdd_system(p, v); }
template <>
MVB_DEVINL void atomic_add_sys<int>(int* p, int v) { atomicAdd_system(p, v); }
template <>
MVB_DEVINL void atomic_add_sys<long long>(long long* p, long long v) {
  atomicAdd_system(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
}

__global__ void kv_init_kernel(long long* keys, int64_t cap) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += stride)
    keys[i] = kEmpty;
}

template <typename V>
__global__ void kv_add_kernel(const __grid_constant__ KVDev kv, const long long* __restrict__ keys,
                              const V* __restrict__ vals, int64_t n, int* err) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long key = keys[i];
    if (key == kEmpty) {
      if (err) atomicExch(err, 5003);   // reserved key
      continue;
    }
    const int o = owner_of(key, kv.S);
    long long* tk = kv.keys[o];
    V* tv = reinterpret_cast<V*>(kv.vals[o]);
    uint64_t slot = mix64((uint64_t)key) & (uint64_t)(kv.cap - 1);
    bool done = false;
    for (int64_t probe = 0; probe < kv.cap; ++probe) {
      long long cur = *reinterpret_cast<volatile long long*>(tk + slot);
      if (cur == kEmpty) {
        cur = (long long)atomicCAS_system(reinterpret_cast<unsigned long long*>(tk + slot),
                                          (unsigned long long)kEmpty, (unsigned long long)key);
        if (cur == kEmpty) cur = key;
      }
      if (cur == key) {
        atomic_add_sys<V>(tv + slot, vals[i]);
        done = true;
        break;
      }
      slot = (slot + 1) & (uint64_t)(kv.cap - 1);
    }
    if (!done && err) atomicExch(err, 5001);  // table full
  }
}

template <typename V>
__global__ void kv_get_kernel(const __grid_constant__ KVDev kv, const long long* __restrict__ keys,
                              V* __restrict__ out, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long key = keys[i];
    if (key == kEmpty) {                 // reserved key: never stored
      out[i] = (V)0;
      continue;
    }
    const int o = owner_of(key, kv.S);
    const long long* tk = kv.keys[o];
    const V* tv = reinterpret_cast<const V*>(kv.vals[o]);
    uint64_t slot = mix64((uint64_t)key) & (uint64_t)(kv.cap - 1);
    V result = (V)0;
    for (int64_t probe = 0; probe < kv.cap; ++probe) {
      long long cur = *reinterpret_cast<const volatile long long*>(tk + slot);
      if (cur == key) {
        result = *reinterpret_cast<const volatile V*>(tv + slot);
        break;
      }
      if (cur == kEmpty) break;
      slot = (slot + 1) & (uint64_t)(kv.cap - 1);
    }
    out[i] = result;
  }
}

template <typename V>
__global__ void kv_dump_kernel(const long long* keys, const V* vals, int64_t cap,
                               long long* out_keys, V* out_vals, unsigned long long* count) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += stride) {
    long long k = keys[i];
    if (k != kEmpty) {
      unsigned long long pos = atomicAdd(count, 1ull);
      out_keys[pos] = k;
      out_vals[pos] = vals[i];
    }
  }
}

// growth: number of live keys of a shard, and re-insertion of a shard into a larger local table
__global__ void kv_count_kernel(const long long* keys, int64_t cap, unsigned long long* count) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long c = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += stride) c += keys[i] != kEmpty;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}
template <typename V>
__global__ void kv_rehash_kernel(const long long* okeys, const V* ovals, int64_t ocap, long long* nkeys, V* nvals,
                                 int64_t ncap, int* err) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ocap; i += stride) {
    const long long key = okeys[i];
    if (key == kEmpty) continue;
    uint64_t slot = mix64((uint64_t)key) & (uint64_t)(ncap - 1);
    bool done = false;
    for (int64_t probe = 0; probe < ncap; ++probe) {
      const long long cur = (long long)atomicCAS(reinterpret_cast<unsigned long long*>(nkeys + slot),
                                                 (unsigned long long)kEmpty, (unsigned long long)key);
      if (cur == kEmpty) { nvals[slot] = ovals[i]; done = true; break; }   // keys are unique in the old table
      slot = (slot + 1) & (uint64_t)(ncap - 1);
    }
    if (!done && err) atomicExch(err, 5002);
  }
}

KVDev to_dev(const MvbKV* h) {
  KVDev d{};
  d.S = h->nservers;
  d.cap = h->capacity;
  for (int s = 0; s < MVB_MAX_RANKS; ++s) {
    d.keys[s] = s < h->nservers ? (long long*)h->keys[s] : nullptr;
    d.vals[s] = s < h->nservers ? h->vals[s] : nullptr;
  }
  return d;
}

}  // namespace

extern "C" int mvb_kv_init(void* keys, int64_t capacity, void* stream) {
  kv_init_kernel<<<blocks_for(capacity, 256, 8), 256, 0, (cudaStream_t)stream>>>((long long*)keys, capacity);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_kv_add(const MvbKV* kv, const int64_t* keys, const void* vals, int64_t n,
                          int* err_flag, void* stream) {
  if (kv->nservers < 1 || kv->nservers > MVB_MAX_RANKS) return -3;
  if (kv->capacity < 1 || (kv->capacity & (kv->capacity - 1))) return -4;
  if (n <= 0) return 0;
  const KVDev d = to_dev(kv);
  return with_dtype<float, double, int, long long>(kv->vtype, [&](auto t) {
    using T = typename decltype(t)::type;
    kv_add_kernel<T><<<blocks_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(d, (const long long*)keys,
                                                                               (const T*)vals, n, err_flag);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  });
}
extern "C" int mvb_kv_get(const MvbKV* kv, const int64_t* keys, void* out_vals, int64_t n,
                          void* stream) {
  if (kv->nservers < 1 || kv->nservers > MVB_MAX_RANKS) return -3;
  if (kv->capacity < 1 || (kv->capacity & (kv->capacity - 1))) return -4;
  if (n <= 0) return 0;
  const KVDev d = to_dev(kv);
  return with_dtype<float, double, int, long long>(kv->vtype, [&](auto t) {
    using T = typename decltype(t)::type;
    kv_get_kernel<T><<<blocks_for(n, 256, 8), 256, 0, (cudaStream_t)stream>>>(d, (const long long*)keys,
                                                                               (T*)out_vals, n);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  });
}
extern "C" int mvb_kv_dump(int vtype, const void* keys, const void* vals, int64_t capacity,
                           int64_t* out_keys, void* out_vals, int64_t* out_count, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  return with_dtype<float, double, int, long long>(vtype, [&](auto t) {
    using T = typename decltype(t)::type;
    MVB_CUDA_CHECK(cudaMemsetAsync(out_count, 0, 8, st));
    kv_dump_kernel<T><<<blocks_for(capacity, 256, 8), 256, 0, st>>>((const long long*)keys, (const T*)vals, capacity,
                                                                     (long long*)out_keys, (T*)out_vals,
                                                                     (unsigned long long*)out_count);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  });
}

// Live keys of one shard (device count, zeroed here).
extern "C" int mvb_kv_count(const void* keys, int64_t capacity, int64_t* out_count, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  MVB_CUDA_CHECK(cudaMemsetAsync(out_count, 0, 8, st));
  kv_count_kernel<<<blocks_for(capacity, 256, 8), 256, 0, st>>>((const long long*)keys, capacity, (unsigned long long*)out_count);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
// Re-insert every live (key, value) of a shard into a new, initialised, larger LOCAL table (growth).
extern "C" int mvb_kv_rehash(int vtype, const void* old_keys, const void* old_vals, int64_t old_cap, void* new_keys,
                             void* new_vals, int64_t new_cap, int* err_flag, void* stream) {
  if (new_cap < 1 || (new_cap & (new_cap - 1))) return -4;
  return with_dtype<float, double, int, long long>(vtype, [&](auto t) {
    using T = typename decltype(t)::type;
    kv_rehash_kernel<T><<<blocks_for(old_cap, 256, 8), 256, 0, (cudaStream_t)stream>>>(
        (const long long*)old_keys, (const T*)old_vals, old_cap, (long long*)new_keys, (T*)new_vals, new_cap, err_flag);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  });
}
