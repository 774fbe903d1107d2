// multiverso-b200 :: key-addressed shard kernels for application-defined tables (the device-side extension
// point; reference example: Applications/LogisticRegression/src/util/sparse_table.h:16-294 SparseTable<T> and
// ftrl_sparse_table.h:11-86 FTRLTable<T>: size_t keys range-partitioned over the servers, server storage
// -= value, a per-key "touched" flag so that a whole-table Get only returns the keys anybody ever wrote).
//
// A table is S shards of `per` keys (last server takes the remainder) x `width` fp32 values each, in
// symmetric HBM, plus one touched bitmap per shard.  All ops are one-sided single kernels over peer memory:
//   keys_add   thread per (key, component): red.add of sign * value into the owner's shard, atomicOr of the
//              touched bit (commutative => race-free async-PS semantics, like K3's stateless path)
//   keys_get   thread per (key, component): gather through the peer mapping
//   keys_collect  whole-table Get: every touched key of every shard with its values, compacted
#include "mvb_common.cuh"

namespace {

struct KeysDev {
  int64_t size, per;
  int S, width;
  float* shard[MVB_MAX_RANKS];
  unsigned int* touched[MVB_MAX_RANKS];
};
MVB_DEVINL void locate(const KeysDev& m, int64_t key, int& o, int64_t& local) {
  const int64_t s = row_server(key, m.per, m.S);
  o = (int)s;
  local = key - s * m.per;
}

__global__ void __launch_bounds__(256)
keys_add_kernel(const __grid_constant__ KeysDev m, const long long* __restrict__ keys, const float* __restrict__ vals,
                int64_t n, float sign) {
  const int64_t total = n * m.width;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    const int64_t i = t / m.width;
    const int c = (int)(t - i * m.width);
    const int64_t key = keys[i];
    if (key < 0 || key >= m.size) continue;
    int o;
    int64_t local;
    locate(m, key, o, local);
    red_add_f32(m.shard[o] + local * m.width + c, sign * vals[t]);
    if (c == 0) {
      unsigned int* w = m.touched[o] + (local >> 5);
      const unsigned int bit = 1u << (local & 31);
      if (!(*reinterpret_cast<volatile unsigned int*>(w) & bit)) atomicOr_system(w, bit);
    }
  }
}

__global__ void __launch_bounds__(256)
keys_get_kernel(const __grid_constant__ KeysDev m, const long long* __restrict__ keys, float* __restrict__ out, int64_t n) {
  const int64_t total = n * m.width;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    const int64_t i = t / m.width;
    const int c = (int)(t - i * m.width);
    const int64_t key = keys[i];
    float v = 0.f;
    if (key >= 0 && key < m.size) {
      int o;
      int64_t local;
      locate(m, key, o, local);
      v = *reinterpret_cast<const volatile float*>(m.shard[o] + local * m.width + c);
    }
    out[t] = v;
  }
}

__global__ void __launch_bounds__(256)
keys_collect_kernel(const __grid_constant__ KeysDev m, long long* __restrict__ out_keys, float* __restrict__ out_vals,
                    unsigned long long* __restrict__ count, int64_t cap) {
  const int64_t words = (m.size + 31) / 32 + m.S;            // upper bound; words are per shard
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < words; t += stride) {
    // word t of the concatenated per-shard bitmaps: shard o has ceil(len_o / 32) words, and when size < S the
    // shards from `size` on hold no keys and have no bitmap words
    int64_t w = t;
    int o = 0;
    int64_t len = 0;
    for (; o < m.S; ++o) {
      const int64_t lo = min((int64_t)o * m.per, m.size);
      len = (o == m.S - 1 ? m.size : min((int64_t)(o + 1) * m.per, m.size)) - lo;
      const int64_t nw = (len + 31) / 32;
      if (w < nw) break;
      w -= nw;
    }
    if (o >= m.S) continue;
    unsigned int bits = *reinterpret_cast<const volatile unsigned int*>(m.touched[o] + w);
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      const int64_t local = w * 32 + b;
      if (local >= len) break;
      const unsigned long long pos = atomicAdd(count, 1ull);
      if ((int64_t)pos < cap) {
        out_keys[pos] = (long long)((int64_t)o * m.per + local);
        for (int c = 0; c < m.width; ++c)
          out_vals[pos * m.width + c] = *reinterpret_cast<const volatile float*>(m.shard[o] + local * m.width + c);
      }
    }
  }
}

KeysDev to_dev(const MvbKeyMap* h) {
  KeysDev m{};
  m.size = h->size;
  m.S = h->nservers;
  m.per = h->per_server;
  m.width = h->width;
  for (int s = 0; s < MVB_MAX_RANKS; ++s) {
    m.shard[s] = s < h->nservers ? (float*)h->shard_ptrs[s] : nullptr;
    m.touched[s] = s < h->nservers ? (unsigned int*)h->touched_ptrs[s] : nullptr;
  }
  return m;
}

}  // namespace

extern "C" int mvb_keys_add(const MvbKeyMap* m, const int64_t* keys, const float* vals, int64_t n, float sign,
                            void* stream) {
  if (!row_split_ok(m->nservers, m->per_server)) return MVB_BAD_ROW_MAP;
  if (m->width < 1 || m->width > 16) return -8;
  if (n <= 0) return 0;
  keys_add_kernel<<<blocks_for(n * m->width, 256, 8), 256, 0, (cudaStream_t)stream>>>(to_dev(m), (const long long*)keys, vals, n, sign);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_keys_get(const MvbKeyMap* m, const int64_t* keys, float* out, int64_t n, void* stream) {
  if (!row_split_ok(m->nservers, m->per_server)) return MVB_BAD_ROW_MAP;
  if (m->width < 1 || m->width > 16) return -8;
  if (n <= 0) return 0;
  keys_get_kernel<<<blocks_for(n * m->width, 256, 8), 256, 0, (cudaStream_t)stream>>>(to_dev(m), (const long long*)keys, out, n);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
// Every touched key (ascending inside a shard is NOT guaranteed) with its values; *count may exceed cap.
extern "C" int mvb_keys_collect(const MvbKeyMap* m, int64_t* out_keys, float* out_vals, int64_t* count, int64_t cap,
                                void* stream) {
  if (!row_split_ok(m->nservers, m->per_server)) return MVB_BAD_ROW_MAP;
  if (m->width < 1 || m->width > 16) return -8;
  cudaStream_t st = (cudaStream_t)stream;
  MVB_CUDA_CHECK(cudaMemsetAsync(count, 0, 8, st));
  keys_collect_kernel<<<blocks_for((m->size + 31) / 32 + m->nservers, 256, 8), 256, 0, st>>>(to_dev(m), (long long*)out_keys, out_vals,
                                                                                     (unsigned long long*)count, cap);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
