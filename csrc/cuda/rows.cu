// multiverso-b200 :: row-sparse table kernels.
//
//  K4 get_rows        -- MatrixWorkerTable::Get(row ids): Partition by row/num_row_each,
//                        server packs rows, client scatters (src/table/matrix_table.cpp:
//                        266-313, 442-450, 332-338) -> one gather kernel, warp per row,
//                        128-bit peer loads straight from the owner's shard.
//  K3 add_rows_red    -- row Add for stateless updaters: one-sided vector red.add into
//                        the owner shard (commutative => race-free async-PS semantics).
//     add_rows_delta  -- AddDeltaParameter: red.add of (trained - pulled) * scale per row, behind
//                        mvb_add_rows_delta and the WordEmbedding block push mvb_rows_push_delta.
//     add_rows_owner  -- row Add for stateful updaters, applied by the OWNER exactly once
//                        per (worker,row), reading ids/values from (peer) staging.
//  K10 row_nonzero_mask, stale bitmap -- zero-row skip and delta-pull bookkeeping of the
//                        sparse Matrix tables (src/table/matrix.cpp:151-164, 516-572).
#include <algorithm>
#include <type_traits>
#include "mvb_common.cuh"

namespace {

template <typename T, bool VECOK>
__global__ void __launch_bounds__(256)
get_rows_kernel(const __grid_constant__ MvbRowMap m, const int64_t* __restrict__ ids, int64_t k,
                T* __restrict__ out, int64_t out_ld) {
  constexpr int VEC = VecOf<T>::N;
  const int lane = threadIdx.x & 31;
  for (int64_t i = warp_id(); i < k; i += num_warps()) {
    const int64_t r = ids[i];
    if (r < 0 || r >= m.num_row) continue;
    const T* src = row_ptr<const T>(m, r);
    T* dst = out + i * out_ld;
    if constexpr (VECOK) {
      const int nvec = (int)(m.num_col / VEC);
      int v = lane;
      for (; v + 96 < nvec; v += 128) {
        uint4 a = ld_nc_v4(src + (int64_t)v * VEC);
        uint4 b = ld_nc_v4(src + (int64_t)(v + 32) * VEC);
        uint4 c = ld_nc_v4(src + (int64_t)(v + 64) * VEC);
        uint4 d = ld_nc_v4(src + (int64_t)(v + 96) * VEC);
        st_v4(dst + (int64_t)v * VEC, a);
        st_v4(dst + (int64_t)(v + 32) * VEC, b);
        st_v4(dst + (int64_t)(v + 64) * VEC, c);
        st_v4(dst + (int64_t)(v + 96) * VEC, d);
      }
      uint4 t[3];
      int cnt = 0;
#pragma unroll
      for (int j = 0; j < 3; ++j)
        if (v + 32 * j < nvec) { t[j] = ld_nc_v4(src + (int64_t)(v + 32 * j) * VEC); cnt = j + 1; }
#pragma unroll
      for (int j = 0; j < 3; ++j)
        if (j < cnt) st_v4(dst + (int64_t)(v + 32 * j) * VEC, t[j]);
    } else {
      for (int64_t c = lane; c < m.num_col; c += 32) dst[c] = __ldg(src + c);
    }
  }
}

template <typename T, bool VECOK>
__global__ void __launch_bounds__(256)
add_rows_red_kernel(const __grid_constant__ MvbRowMap m, const int64_t* __restrict__ ids,
                    int64_t k, const T* __restrict__ vals, int64_t vals_ld, float sign) {
  const int lane = threadIdx.x & 31;
  for (int64_t i = warp_id(); i < k; i += num_warps()) {
    const int64_t r = ids[i];
    if (r < 0 || r >= m.num_row) continue;
    T* dst = row_ptr<T>(m, r);
    const T* src = vals + i * vals_ld;
    if constexpr (VECOK && std::is_same<T, float>::value) {
      const int nvec = (int)(m.num_col / 4);
      for (int v = lane; v < nvec; v += 32) {
        float4 x = *reinterpret_cast<const float4*>(src + (int64_t)v * 4);
        x.x *= sign; x.y *= sign; x.z *= sign; x.w *= sign;
        red_add_v4_f32(reinterpret_cast<float*>(dst) + (int64_t)v * 4, x);
      }
    } else {
      for (int64_t c = lane; c < m.num_col; c += 32) red_add(dst + c, (T)(src[c] * (T)sign));
    }
  }
}

// AddDeltaParameter fused (Applications/WordEmbedding/src/communicator.cpp:157-203, 206-249): push
// (trained - pulled) * scale for every cached row straight into its owner with one-sided red.add.v4.f32 (the
// async-PS Add of a stateless updater), no delta tensor; all-zero 16-byte deltas are skipped. The row count is
// n_max, or read on the device from n_ptr (clamped to n_max).
template <typename Id>
struct DeltaArgs {
  MvbRowMap m;
  const Id* ids;           // row ids
  const int* n_ptr;        // device count (nullptr: n_max rows)
  int64_t n_max;
  const unsigned char* cur;   // trained rows [n x ld_bytes]
  const unsigned char* old;   // pulled rows  [n x ld_bytes]
  int64_t ld_bytes;
  int row_bytes;              // == the shards' row pitch
  float scale;
};

// 128-thread CTAs, no shared memory, <= 56 registers: the WordEmbedding block push runs these co-resident with
// the persistent K7 CTAs (which own the SMs' shared memory but leave threads and registers; we_block.cu).
// Warp per row, 3 vectors per lane in flight.
constexpr int kDeltaThreads = 128;

template <typename Id>
__global__ void __launch_bounds__(kDeltaThreads, 9)
add_rows_delta_kernel(const __grid_constant__ DeltaArgs<Id> a) {
  const int lane = threadIdx.x & 31;
  int64_t n = a.n_ptr ? (int64_t)*a.n_ptr : a.n_max;
  if (n > a.n_max) n = a.n_max;
  const int nvec = a.row_bytes >> 4;
  for (int64_t s = warp_id(); s < n; s += num_warps()) {
    const int64_t r = (int64_t)__ldg(a.ids + s);
    if (r < 0 || r >= a.m.num_row) continue;
    float* dst = reinterpret_cast<float*>(row_ptr<unsigned char>(a.m, r, a.row_bytes));
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

// Repeated rows must be applied one after the other, in list order (MatrixServerTable::ProcessAdd), so
// the caller passes the ids with equal ids adjacent (a stable sort) and the warp that meets the START of
// a run of equal ids applies the whole run in order, keeping the element and its state in registers.
template <int UPD, typename T>
__global__ void __launch_bounds__(256)
add_rows_owner_kernel(T* __restrict__ shard, T* __restrict__ st0, T* __restrict__ st1,
                      int64_t row_lo, int64_t row_hi, int64_t num_col, int64_t state_stride,
                      const int64_t* __restrict__ ids, int64_t k, const T* __restrict__ vals,
                      int64_t vals_ld, MvbAddOpt opt) {
  using U = Updater<UPD, T>;
  const int lane = threadIdx.x & 31;
  for (int64_t i = warp_id(); i < k; i += num_warps()) {
    const int64_t r = ids[i];
    if (i > 0 && ids[i - 1] == r) continue;  // inside a run: applied by the run's first warp
    if (r < row_lo || r >= row_hi) continue;
    int64_t end = i + 1;
    while (end < k && ids[end] == r) ++end;
    const int64_t base = (r - row_lo) * num_col;
    if constexpr (U::kRowState) {
      // the row's state (rowwise_adagrad's accumulator, adam's step count; see row_state_at) stays in registers
      // over the run; the run goes in chunks of up to 32 occurrences: first their factors in list order (occurrence
      // j sees the row state after the occurrences before it; lane j keeps the chunk's j-th factor), then one pass
      // over the row applies the chunk, with the element state (adam's m, v) in registers over the chunk
      T* hp = row_state_at<U>(st0, st1, opt.worker_id, state_stride, r - row_lo);
      T h = *hp;
      for (int64_t j0 = i; j0 < end; j0 += 32) {
        const int n = (int)(end - j0 < 32 ? end - j0 : 32);
        typename U::RowF mine{};
        for (int j = 0; j < n; ++j) {
          T part = (T)0;
          if constexpr (U::kRowSum)
            for (int64_t c = lane; c < num_col; c += 32) part += U::Square(vals[(j0 + j) * vals_ld + c], opt);
          const typename U::RowF f = row_factor<U>(part, h, hp, num_col, opt);
          if (lane == j) mine = f;
        }
        for (int64_t c0 = 0; c0 < num_col; c0 += 32) {
          const int64_t c = c0 + lane;
          T d = c < num_col ? shard[base + c] : (T)0, s0 = (T)0, s1 = (T)0;
          if (c < num_col) row_elem_load<U>(s0, s1, st0, st1, opt.worker_id, state_stride, base + c);
          for (int j = 0; j < n; ++j) {
            const typename U::RowF f = U::Shfl(mine, j);
            if (c < num_col) U::Step(d, vals[(j0 + j) * vals_ld + c], f, s0, s1, opt);
          }
          if (c < num_col) {
            row_elem_store<U>(s0, s1, st0, st1, opt.worker_id, state_stride, base + c);
            shard[base + c] = d;
          }
        }
      }
    } else {
      for (int64_t c = lane; c < num_col; c += 32) {
        T d = shard[base + c], s0 = (T)0, s1 = (T)0;
        state_load<U>(s0, s1, st0, st1, opt.worker_id, state_stride, base + c);
        for (int64_t j = i; j < end; ++j) U::Apply(d, vals[j * vals_ld + c], s0, s1, opt);
        state_store<U>(s0, s1, st0, st1, opt.worker_id, state_stride, base + c);
        shard[base + c] = d;
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
row_nonzero_kernel(const T* __restrict__ data, int64_t rows, int64_t cols, int64_t ld,
                   uint8_t* __restrict__ mask) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = warp_id(); r < rows; r += num_warps()) {
    const T* row = data + r * ld;
    int nz = 0;
    for (int64_t c = lane; c < cols; c += 32) nz |= (row[c] != (T)0);
    nz = __any_sync(0xffffffffu, nz);
    if (lane == 0) mask[r] = (uint8_t)(nz ? 1 : 0);
  }
}

__global__ void stale_mark_kernel(uint8_t* stale, int64_t rows, int nworkers, const int64_t* ids,
                                  int64_t k) {
  const int64_t n = (k < 0 ? rows : k) * nworkers;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
    const int64_t per = (k < 0 ? rows : k);
    const int w = (int)(t / per);
    const int64_t j = t - (int64_t)w * per;
    const int64_t r = k < 0 ? j : ids[j];
    if (r >= 0 && r < rows) stale[(int64_t)w * rows + r] = 1;
  }
}
__global__ void stale_take_kernel(uint8_t* stale_w, int64_t rows, const int64_t* ids, int64_t k,
                                  uint8_t* out) {
  const int64_t n = k < 0 ? rows : k;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
    const int64_t r = k < 0 ? t : ids[t];
    if (r >= 0 && r < rows) {
      out[t] = stale_w[r];
      stale_w[r] = 0;
    } else {
      out[t] = 0;
    }
  }
}

// ordered compaction of a byte mask into the list of set positions (one CTA: chunk per thread, block scan)
__global__ void __launch_bounds__(1024)
mask_compact_kernel(const uint8_t* __restrict__ mask, int64_t n, int64_t* __restrict__ out, int64_t* __restrict__ count) {
  __shared__ int64_t part[1024];
  const int64_t per = (n + 1023) / 1024;
  const int64_t lo = (int64_t)threadIdx.x * per, hi = lo + per < n ? lo + per : n;
  int64_t c = 0;
  for (int64_t i = lo; i < hi; ++i) c += mask[i] != 0;
  part[threadIdx.x] = c;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int64_t t = threadIdx.x >= o ? part[threadIdx.x - o] : 0;
    __syncthreads();
    part[threadIdx.x] += t;
    __syncthreads();
  }
  int64_t pos = part[threadIdx.x] - c;
  for (int64_t i = lo; i < hi; ++i)
    if (mask[i]) out[pos++] = i;
  if (threadIdx.x == 1023) *count = part[1023];
}

template <typename T>
int get_rows_t(const MvbRowMap* m, const int64_t* ids, int64_t k, void* out, int64_t out_ld,
               cudaStream_t st) {
  bool vec = (m->num_col % VecOf<T>::N == 0) && (out_ld % VecOf<T>::N == 0) &&
             ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
  int grid = grid_for(k);
  if (vec)
    get_rows_kernel<T, true><<<grid, 256, 0, st>>>(*m, ids, k, (T*)out, out_ld);
  else
    get_rows_kernel<T, false><<<grid, 256, 0, st>>>(*m, ids, k, (T*)out, out_ld);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

template <typename T>
int add_rows_red_t(const MvbRowMap* m, const int64_t* ids, int64_t k, const void* vals,
                   int64_t vals_ld, float sign, cudaStream_t st) {
  bool vec = (m->num_col % 4 == 0) && (vals_ld % 4 == 0) &&
             ((reinterpret_cast<uintptr_t>(vals) & 15) == 0) && sizeof(T) == 4;
  int grid = grid_for(k);
  if (vec)
    add_rows_red_kernel<T, true><<<grid, 256, 0, st>>>(*m, ids, k, (const T*)vals, vals_ld, sign);
  else
    add_rows_red_kernel<T, false><<<grid, 256, 0, st>>>(*m, ids, k, (const T*)vals, vals_ld, sign);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

template <typename Id>
int add_rows_delta_t(const MvbRowMap* m, const Id* ids, const int* n_ptr, int64_t n_max, const float* cur,
                     const float* old, int64_t ld, float scale, int64_t ctas, cudaStream_t st) {
  // whole float4 vectors: a 16-byte row pitch and 16-byte aligned rows
  if (m->num_col % 4 || ld % 4) return -9;
  if ((reinterpret_cast<uintptr_t>(cur) & 15) || (reinterpret_cast<uintptr_t>(old) & 15)) return -9;
  const DeltaArgs<Id> a{*m, ids, n_ptr, n_max, reinterpret_cast<const unsigned char*>(cur),
                        reinterpret_cast<const unsigned char*>(old), ld * 4, (int)(m->num_col * 4), scale};
  add_rows_delta_kernel<Id><<<(unsigned)ctas, kDeltaThreads, 0, st>>>(a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" int mvb_get_rows(int dtype, const MvbRowMap* m, const int64_t* row_ids, int64_t k,
                            void* out, int64_t out_ld, void* stream) {
  if (!row_split_ok(m->nservers, m->rows_per_server)) return MVB_BAD_ROW_MAP;
  if (k <= 0) return 0;
  return with_dtype<float, double, int>(dtype, [&](auto t) {
    return get_rows_t<typename decltype(t)::type>(m, row_ids, k, out, out_ld, (cudaStream_t)stream);
  });
}
extern "C" int mvb_add_rows_red(int dtype, const MvbRowMap* m, const int64_t* row_ids, int64_t k,
                                const void* vals, int64_t vals_ld, float sign, void* stream) {
  if (!row_split_ok(m->nservers, m->rows_per_server)) return MVB_BAD_ROW_MAP;
  if (k <= 0) return 0;
  return with_dtype<float, double, int>(dtype, [&](auto t) {
    return add_rows_red_t<typename decltype(t)::type>(m, row_ids, k, vals, vals_ld, sign, (cudaStream_t)stream);
  });
}
extern "C" int mvb_add_rows_delta(const MvbRowMap* m, const int64_t* row_ids, int64_t k, const float* cur,
                                  const float* old, int64_t ld, float scale, void* stream) {
  if (!row_split_ok(m->nservers, m->rows_per_server)) return MVB_BAD_ROW_MAP;
  if (k <= 0) return 0;
  // a warp per row, at most 8 x 256 threads per SM
  const int ctas = blocks_for(k * 32, kDeltaThreads, 16);
  return add_rows_delta_t<int64_t>(m, row_ids, nullptr, k, cur, old, ld, scale, ctas, (cudaStream_t)stream);
}
// rows[ids[s]] += (cur[s] - old[s]) * scale for s in [0, n), n read on the device from n_ptr when given (clamped to
// n_max); the grid is ctas_per_sm (>= 1) CTAs per SM.
extern "C" int mvb_rows_push_delta(const MvbRowMap* m, const int* ids, const int* n_ptr, int64_t n_max,
                                   const float* cur, const float* old, int64_t ld, float scale, int ctas_per_sm,
                                   void* stream) {
  if (!row_split_ok(m->nservers, m->rows_per_server)) return MVB_BAD_ROW_MAP;
  if (ctas_per_sm < 1) return -22;
  if (n_max <= 0) return 0;
  return add_rows_delta_t<int>(m, ids, n_ptr, n_max, cur, old, ld, scale, (int64_t)mvb_num_sms() * ctas_per_sm,
                               (cudaStream_t)stream);
}
extern "C" int mvb_add_rows_owner(int dtype, int updater, void* shard, void* state0, void* state1,
                                  int64_t row_lo, int64_t row_hi, int64_t num_col,
                                  int64_t state_stride, const int64_t* row_ids, int64_t k,
                                  const void* vals, int64_t vals_ld, const MvbAddOpt* opt,
                                  void* stream) {
  if (k <= 0) return 0;
  return with_dtype<float, double, int>(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    return with_updater<T>(updater, [&](auto u) {
      if constexpr (Updater<decltype(u)::value, T>::kElemState) {
        // adam: m and v are element slabs, the step counts follow v's slab
        if (num_col < 1 || state_stride < (row_hi - row_lo) * num_col) return (int)MVB_BAD_ROW_MAP;
      }
      add_rows_owner_kernel<decltype(u)::value, T><<<grid_for(k), 256, 0, (cudaStream_t)stream>>>(
          (T*)shard, (T*)state0, (T*)state1, row_lo, row_hi, num_col, state_stride, row_ids, k, (const T*)vals,
          vals_ld, *opt);
      MVB_CUDA_CHECK(cudaGetLastError());
      return 0;
    });
  });
}
extern "C" int mvb_row_nonzero_mask(int dtype, const void* data, int64_t rows, int64_t cols,
                                    int64_t ld, uint8_t* mask, void* stream) {
  if (rows <= 0) return 0;
  return with_dtype<float, double, int>(dtype, [&](auto t) {
    using T = typename decltype(t)::type;
    row_nonzero_kernel<T><<<grid_for(rows), 256, 0, (cudaStream_t)stream>>>((const T*)data, rows, cols, ld, mask);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  });
}
extern "C" int mvb_stale_mark(uint8_t* stale, int64_t rows, int nworkers, const int64_t* row_ids,
                              int64_t k, void* stream) {
  int64_t n = (k < 0 ? rows : k) * nworkers;
  if (n <= 0) return 0;
  int blocks = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  stale_mark_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(stale, rows, nworkers, row_ids, k);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
extern "C" int mvb_stale_take(uint8_t* stale_w, int64_t rows, const int64_t* row_ids, int64_t k,
                              uint8_t* out_mask, void* stream) {
  int64_t n = k < 0 ? rows : k;
  if (n <= 0) return 0;
  int blocks = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
  stale_take_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(stale_w, rows, row_ids, k, out_mask);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// Positions of the non-zero bytes of mask[0..n), ascending; *count = how many (device).
extern "C" int mvb_mask_compact(const uint8_t* mask, int64_t n, int64_t* out_ids, int64_t* count, void* stream) {
  if (n <= 0) return 0;
  mask_compact_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(mask, n, out_ids, count);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
