// multiverso-b200 :: field-aware factorization machine over a row-sharded fp32 MatrixTable
// (multiverso_b200/ops/field_aware_factorization_machine.py).
//
// F fields of k factors (k % 4 == 0), D = F k. Row r holds V_r[f] = W[r, f k : (f + 1) k] and w_r = W[r, D]. Bag b
// holds the lookups j with ids i_j, fields f_j and values x_j:
//
//   y_b = sum_j x_j w_{i_j} + sum_{j < l} x_j x_l <V_{i_j}[f_l], V_{i_l}[f_j]>
//
// The kernel computes, for every lookup j of the bag, the row H_j = dy_b / d(row values at j) (D + 1 columns):
//
//   H_j[f k + c] = x_j * sum_{l != j, f_l = f} x_l V_{i_l}[f_j][c]      H_j[D] = x_j
//
// and y_b = sum_j x_j w_{i_j} + (1/2) sum_j <H_j[0:D], W[i_j, 0:D]> (every pair is met once from each side).
//
//  fwd   one 256-thread CTA per bag over a grid-stride loop. Work items are (lookup j, 4 columns c) of the bag, item
//        j * nq + c / 4 with nq = round4(D + 1) / 4; thread t owns the items t, t + 256, t + 512, ... and takes them
//        FFM_ITEMS at a time with their sums in registers. The bag's rows are staged in shared memory with 16-byte
//        cp.async copies straight from the owners' shards, T rows per tile, and each tile's positions are grouped
//        by field with a stable counting sort. An item sums the positions of field f in position order, tile after
//        tile; a bag of at most T lookups is staged once, a longer one once per item group. Thread t then sums its
//        items' x_j w and <H_j, W> terms in item order and the CTA combines the 256 shares with a fixed tree.
//        Neither y nor H depends on T, on the sharding or on whether H is written: both are bitwise reproducible,
//        and the forward without H is bitwise the forward with it. Nothing of size n^2 is written; H ([L, ldh],
//        columns >= D + 1 written 0) is written only when asked for, as the dout rows of the embedding-bag
//        backward, which pushes G_r = sum_{j: i_j = r} dy_b(j) H_j once per unique row.
#include <atomic>

#include "emb_bag.cuh"

namespace {

constexpr int FFM_THREADS = 256;
constexpr int FFM_ITEMS = 2;                    // items per thread held in registers at a time (64 registers)
constexpr int FFM_SMEM = 100 * 1024;            // dynamic shared memory per CTA at most: 2 CTAs per SM
constexpr int FFM_MAX_TILE = 512;               // rows per tile at most

// The shared-memory tile of a launch: T rows at a pitch of ldr floats (round4(D + 1) padded to 4 mod 32 floats, so
// that the 16-byte loads of 8 rows hit 8 different bank quads), then per row its pointer, x and field, the sorted
// positions, and the count and start of every field.
struct FfmTile {
  int T, ldr;
  size_t bytes;
};

size_t tile_bytes(int T, int ldr, int F) {
  return (size_t)T * ldr * 4 + (size_t)T * (8 + 4 + 4 + 4) + (size_t)F * 8;
}

FfmTile tile_of(int64_t F, int64_t k, int64_t max_len) {
  const int r4 = (int)((F * k + 1 + 3) / 4 * 4);
  const int ldr = r4 + (4 - r4 % 32 + 32) % 32;
  int T = (int)((FFM_SMEM - F * 8) / ((int64_t)ldr * 4 + 20));
  if (T > FFM_MAX_TILE) T = FFM_MAX_TILE;
  if (max_len > 0 && max_len < T) T = (int)max_len;
  if (T < 1) T = 1;
  return FfmTile{T, ldr, tile_bytes(T, ldr, (int)F)};
}

MVB_DEVINL void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}

struct FfmSmem {
  float* rows;                                   // [T][ldr]
  const float** rp;                              // [T] row pointers
  float* xs;                                     // [T] x
  int* fl;                                       // [T] field
  int* list;                                     // [T] tile positions sorted by (field, position)
  int* cnt;                                      // [F]
  int* start;                                    // [F]
};

// Stages positions [p0, p0 + m) of the bag starting at lookup lo: rows, x, fields, and the counting sort by field.
// Called by the whole CTA; ends with a barrier.
MVB_DEVINL void stage_tile(const MvbFfm& a, const FfmSmem& s, int ldr, int nq, int64_t lo, int p0, int m) {
  const int tid = threadIdx.x, F = (int)a.F;
  for (int l = tid; l < m; l += FFM_THREADS) {
    const int64_t p = lo + p0 + l;
    s.rp[l] = row_ptr<const float>(a.wmap, __ldg(a.ids + p));
    s.xs[l] = a.values ? __ldg(a.values + p) : 1.f;
    s.fl[l] = __ldg(a.fields + p);
  }
  for (int f = tid; f < F; f += FFM_THREADS) s.cnt[f] = 0;
  __syncthreads();
  for (int e = tid; e < m * nq; e += FFM_THREADS) {
    const int l = e / nq, v = e - l * nq;
    cp_async16(s.rows + l * ldr + 4 * v, s.rp[l] + 4 * v);
  }
  for (int l = tid; l < m; l += FFM_THREADS) atomicAdd(s.cnt + s.fl[l], 1);
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();
  if (tid < 32) {                                // exclusive scan of the counts: lane i takes fields [i c, i c + c)
    const int per = (F + 31) / 32, f0 = tid * per;
    int sum = 0;
    for (int f = f0; f < f0 + per && f < F; ++f) sum += s.cnt[f];
    int inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(FULL, inc, o);
      if (tid >= o) inc += t;
    }
    int run = inc - sum;
    for (int f = f0; f < f0 + per && f < F; ++f) {
      s.start[f] = run;
      run += s.cnt[f];
    }
  }
  __syncthreads();
  for (int l = tid; l < m; l += FFM_THREADS) {   // stable: the rank of l among the earlier positions of its field
    const int f = s.fl[l];
    int r = 0;
    for (int q = 0; q < l; ++q) r += s.fl[q] == f;
    s.list[s.start[f] + r] = l;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(FFM_THREADS, 4)
ffm_fwd_kernel(const __grid_constant__ MvbFfm a, int T, int ldr) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float red[2][FFM_THREADS / 32];
  FfmSmem s;
  s.rows = reinterpret_cast<float*>(smem_raw);
  s.rp = reinterpret_cast<const float**>(s.rows + (size_t)T * ldr);
  s.xs = reinterpret_cast<float*>(s.rp + T);
  s.fl = reinterpret_cast<int*>(s.xs + T);
  s.list = s.fl + T;
  s.cnt = s.list + T;
  s.start = s.cnt + a.F;
  const int tid = threadIdx.x, k = (int)a.k, D = (int)(a.F * a.k);
  const int nq = (D + 1 + 3) / 4;
  for (int64_t b = blockIdx.x; b < a.B; b += gridDim.x) {
    const int64_t lo = a.offsets[b], hi = b + 1 < a.B ? a.offsets[b + 1] : a.L;
    const int n = (int)(hi - lo), nt = (n + T - 1) / T;
    const int64_t items = (int64_t)n * nq;
    float lin = 0.f, pair = 0.f;
    if (nt == 1) stage_tile(a, s, ldr, nq, lo, 0, n);
    for (int64_t base = 0; base < items; base += FFM_THREADS * FFM_ITEMS) {
      int jr[FFM_ITEMS], cr[FFM_ITEMS], fr[FFM_ITEMS], colr[FFM_ITEMS];
      float xr[FFM_ITEMS];
      float4 acc[FFM_ITEMS];
#pragma unroll
      for (int r = 0; r < FFM_ITEMS; ++r) {
        const int64_t it = base + tid + FFM_THREADS * r;
        acc[r] = zero4();
        jr[r] = -1;
        cr[r] = fr[r] = colr[r] = 0;
        xr[r] = 0.f;
        if (it < items) {
          const int j = (int)(it / nq), c = 4 * (int)(it - (int64_t)j * nq);
          const int fj = __ldg(a.fields + lo + j);
          jr[r] = j;
          cr[r] = c;
          fr[r] = c < D ? c / k : -1;            // the segment's field; -1: column D and the padding
          colr[r] = c < D ? fj * k + (c - fr[r] * k) : 0;
          xr[r] = a.values ? __ldg(a.values + lo + j) : 1.f;
        }
      }
      for (int t = 0; t < nt; ++t) {
        const int p0 = t * T, m = n - p0 < T ? n - p0 : T;
        if (nt > 1) {
          __syncthreads();                       // every item is done with the previous tile
          stage_tile(a, s, ldr, nq, lo, p0, m);
        }
#pragma unroll
        for (int r = 0; r < FFM_ITEMS; ++r) {
          if (jr[r] < 0 || fr[r] < 0) continue;
          const int e0 = s.start[fr[r]], e1 = e0 + s.cnt[fr[r]];
          for (int e = e0; e < e1; ++e) {
            const int l = s.list[e];
            if (p0 + l == jr[r]) continue;       // a position never meets itself
            fma4(acc[r], s.xs[l], *reinterpret_cast<const float4*>(s.rows + l * ldr + colr[r]));
          }
        }
      }
#pragma unroll
      for (int r = 0; r < FFM_ITEMS; ++r) {
        if (jr[r] < 0) continue;
        const int j = jr[r], c = cr[r];
        const float x = xr[r];
        float4 h = zero4();
        const float* row = nt == 1 ? s.rows + j * ldr : nullptr;
        if (c < D) {
          h = make_float4(x * acc[r].x, x * acc[r].y, x * acc[r].z, x * acc[r].w);
          const float4 v = row ? *reinterpret_cast<const float4*>(row + c)
                               : ld_nc_l1_v4(row_ptr<const float>(a.wmap, __ldg(a.ids + lo + j)) + c);
          pair = fmaf(h.x, v.x, pair); pair = fmaf(h.y, v.y, pair);
          pair = fmaf(h.z, v.z, pair); pair = fmaf(h.w, v.w, pair);
        } else if (c == D) {
          h.x = x;
          const float w = row ? row[D] : __ldg(row_ptr<const float>(a.wmap, __ldg(a.ids + lo + j)) + D);
          lin = fmaf(x, w, lin);
        }
        if (a.h) *reinterpret_cast<float4*>(a.h + (lo + j) * a.ldh + c) = h;
      }
    }
    if (a.h && a.ldh > 4 * nq) {                 // the pitch padding past round4(D + 1)
      const int pad = (int)(a.ldh / 4) - nq;
      for (int64_t e = tid; e < (int64_t)n * pad; e += FFM_THREADS) {
        const int64_t j = e / pad;
        *reinterpret_cast<float4*>(a.h + (lo + j) * a.ldh + 4 * (nq + (e - j * pad))) = zero4();
      }
    }
    lin = warp_sum(lin);
    pair = warp_sum(pair);
    if ((tid & 31) == 0) {
      red[0][tid >> 5] = lin;
      red[1][tid >> 5] = pair;
    }
    __syncthreads();
    if (tid == 0) {
      float l = red[0][0], p = red[1][0];
#pragma unroll
      for (int w = 1; w < FFM_THREADS / 32; ++w) {
        l += red[0][w];
        p += red[1][w];
      }
      a.y[b] = l + 0.5f * p;
    }
    __syncthreads();                             // red and the tile are free for the next bag
  }
}

// Lets the kernel take FFM_SMEM bytes of dynamic shared memory on the current device: once per device and process,
// so that a launch is one driver call
cudaError_t allow_tile_smem() {
  constexpr int kMaxDevices = 64;
  static std::atomic<bool> done[kMaxDevices];
  int dev = 0;
  if (cudaError_t e = cudaGetDevice(&dev)) return e;
  if (dev >= 0 && dev < kMaxDevices && done[dev].load(std::memory_order_acquire)) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(ffm_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FFM_SMEM);
  if (e == cudaSuccess && dev >= 0 && dev < kMaxDevices) done[dev].store(true, std::memory_order_release);
  return e;
}

}  // namespace

extern "C" int mvb_ffm_fwd(const MvbFfm* a, void* stream) {
  const MvbRowMap& m = a->wmap;
  if (!row_split_ok(m.nservers, m.rows_per_server)) return MVB_BAD_ROW_MAP;
  if (a->k < 4 || a->k % 4 != 0 || a->F < 1 || a->F * a->k + 1 > MVB_FFM_MAX_DIM) return -95;
  const int64_t D = a->F * a->k;
  if (m.num_col < D + 1 || m.num_col % 4 != 0) return -96;
  for (int s = 0; s < m.nservers; ++s)
    if ((uintptr_t)m.shard_ptrs[s] & 15) return -96;
  if (a->B < 0 || a->L < 0) return -97;
  if ((a->B > 0 && (!a->offsets || !a->y)) || (a->L > 0 && (!a->ids || !a->fields))) return -98;
  if (a->h && (a->ldh % 4 != 0 || a->ldh < (D + 1 + 3) / 4 * 4 || ((uintptr_t)a->h & 15))) return -99;
  if (a->B == 0) return 0;
  const FfmTile t = tile_of(a->F, a->k, a->max_len);
  if (t.bytes > 48 * 1024) MVB_CUDA_CHECK(allow_tile_smem());
  int per_sm = (int)((227 * 1024) / (t.bytes + 1024));
  if (per_sm > 2048 / FFM_THREADS) per_sm = 2048 / FFM_THREADS;
  if (per_sm < 1) per_sm = 1;
  const int grid = blocks_for(a->B * FFM_THREADS, FFM_THREADS, per_sm);
  ffm_fwd_kernel<<<grid, FFM_THREADS, t.bytes, (cudaStream_t)stream>>>(*a, t.T, t.ldr);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
