// multiverso-b200 :: the embedding-bag algorithms, written once for the single-table kernels (emb_bag.cu) and the
// collection (emb_bag_coll.cu). Each body below is the work of one warp on one bag, chunk, run or lookup; the
// kernels of the two files are grid-stride loops that work out their bag or chunk and call it. What differs between
// the two callers comes in as plain values (row map, dim, bag range, output rows, sorted-key segment, chunk range,
// first unique index, compact destination) or, for the dout row of a lookup and the epilogue of a run, as a small
// callable. The single table is a segment [0, L) with output column 0. Because both files run the same code, a
// collection's feature is bitwise equal to embedding_bag over its table.
//
//  gather-pool   emb_pool_bag: out = sum (or mean) over the lookups j of a bag of psw_j * W[ids_j, :dim]. For dim <
//                128 the warp splits into lane groups that each take a lookup; 4 lookups per group are in flight.
//                Group g sums the lookups g, g + NG, g + 2 NG, ... of its bag in order and the groups are combined
//                by a fixed butterfly, so the summation order depends only on positions within the bag and on dim.
//  backward      the lookups arrive sorted by (key, position), cut into chunks of EMB_CHUNK within each segment:
//    count       emb_count_runs: the run starts (unique keys) of one chunk, leaving out rows that are not pushed
//    scan        emb_block_scan: exclusive scan of the per-chunk counts, one 1024-thread CTA
//    run-sum     emb_run_sum: sums psw_j * s_bag * dout[bag(j)] over each run of equal keys of one chunk in
//                ascending position. A run inside the chunk goes straight to the epilogue; the pieces of a run
//                that crosses chunk boundaries go to scratch
//    merge       emb_merge_run: sums those pieces in chunk order, by the warp of the chunk the run starts in
//    epilogue    emb_epilogue: every unique key below the table's push bound gets exactly one
//                  push     red.add.v4.f32 of scale * g into the owner's row (default / sgd updaters)
//                  compact  grads[u] = scale * g, uniq[u] = id, u = rank of the id among the unique ids
//  psw grad      emb_psw_dot: s_bag * <dout[bag(j)], W[ids_j, :dim]> of one lookup.
#pragma once
#include <type_traits>

#include "mvb_common.cuh"

namespace {

constexpr int EMB_CHUNK = 256;   // sorted lookups per backward warp
constexpr int EMB_INFLIGHT = 4;  // lookups in flight per lane group / warp
constexpr unsigned FULL = 0xffffffffu;

// float4 vectors per lane for a dim, before the cap of 4 (the kernels' template argument): lane groups of up to 32
// lanes share a row in the forward, a whole warp in the backward
__host__ __device__ __forceinline__ int emb_vpl(int64_t dim) {
  const int64_t nv = (dim + 3) / 4;
  return nv <= 32 ? 1 : (int)((nv + 31) / 32);
}

// log2 of the forward's lane-group size: the smallest power of two >= the float4 vectors of a row, at most 32
__host__ __device__ __forceinline__ int emb_lane_group_log(int nv) {
  int lg = 0;
  while ((1 << lg) < nv && lg < 5) ++lg;
  return lg;
}

// f(std::integral_constant<int, V>) for V = min(vpl, 4): the launches of the kernel templates of a register class
template <class F>
auto with_vpl(int vpl, F&& f) {
  if (vpl <= 1) return f(std::integral_constant<int, 1>{});
  if (vpl == 2) return f(std::integral_constant<int, 2>{});
  if (vpl == 3) return f(std::integral_constant<int, 3>{});
  return f(std::integral_constant<int, 4>{});
}

MVB_DEVINL float4 f4(uint4 u) {
  return make_float4(__uint_as_float(u.x), __uint_as_float(u.y), __uint_as_float(u.z), __uint_as_float(u.w));
}
MVB_DEVINL float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }
MVB_DEVINL void fma4(float4& acc, float w, float4 x) {
  acc.x = fmaf(w, x.x, acc.x); acc.y = fmaf(w, x.y, acc.y);
  acc.z = fmaf(w, x.z, acc.z); acc.w = fmaf(w, x.w, acc.w);
}
MVB_DEVINL void add4(float4& acc, float4 x) { acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w; }

// read-only 128-bit load that allocates in L1: the hot rows of a Zipf batch are read by many warps of an SM
MVB_DEVINL float4 ld_nc_l1_v4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

// columns [c, c + 4) of a table row of which the first dim are used; columns >= dim read as 0 and are never
// loaded (pitch padding)
MVB_DEVINL float4 load_row4(const float* row, int c, int dim) {
  if (c + 4 <= dim) return ld_nc_l1_v4(row + c);
  float4 r = zero4();
  if (c < dim) r.x = __ldg(row + c);
  if (c + 1 < dim) r.y = __ldg(row + c + 1);
  if (c + 2 < dim) r.z = __ldg(row + c + 2);
  return r;
}

// the bag of lookup position p: the last b with offsets[b] <= p (offsets[0] == 0)
MVB_DEVINL int64_t bag_of(const int64_t* __restrict__ off, int64_t B, int64_t p) {
  int64_t lo = 0, hi = B;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(off + mid) <= p) lo = mid + 1; else hi = mid;
  }
  return lo - 1;
}

MVB_DEVINL int64_t bag_len(const int64_t* __restrict__ off, int64_t B, int64_t L, int64_t b) {
  return (b + 1 < B ? __ldg(off + b + 1) : L) - __ldg(off + b);
}

MVB_DEVINL bool run_start(const int64_t* __restrict__ sid, int64_t i) { return i == 0 || sid[i] != sid[i - 1]; }

// ------------------------------------------------------------------------------------------------ forward
// the lookups [lo, hi) of one bag pooled into out[0 .. dim), lane groups of 1 << lg lanes
template <int VPL>
MVB_DEVINL void emb_pool_bag(const MvbRowMap& m, int dim, int lg, const int64_t* __restrict__ ids,
                             const float* __restrict__ psw, int64_t lo, int64_t hi, bool mean, float* out) {
  const int G = 1 << lg, NG = 32 >> lg;                // lane groups of G lanes, NG groups per warp
  const int lane = threadIdx.x & 31, grp = lane >> lg, gl = lane & (G - 1);
  const int nv = (dim + 3) >> 2;
  for (int v0 = 0; v0 < nv; v0 += G * VPL) {        // column slabs (one slab up to dim = 512)
    float4 acc[VPL];
#pragma unroll
    for (int k = 0; k < VPL; ++k) acc[k] = zero4();
    for (int64_t w0 = lo; w0 < hi; w0 += 32) {       // windows of 32 lookups: ids and weights by one load per lane
      const int n = hi - w0 < 32 ? (int)(hi - w0) : 32;
      const int64_t id_l = lane < n ? __ldg(ids + w0 + lane) : 0;
      const float w_l = lane < n ? (psw ? __ldg(psw + w0 + lane) : 1.f) : 0.f;
      for (int t0 = 0; t0 < n; t0 += EMB_INFLIGHT * NG) {
        float4 x[EMB_INFLIGHT][VPL];
        float w[EMB_INFLIGHT];
#pragma unroll
        for (int u = 0; u < EMB_INFLIGHT; ++u) {
          const int t = t0 + u * NG + grp;             // group grp takes the lookups grp, grp + NG, ...
          const int64_t id = __shfl_sync(FULL, id_l, t & 31);
          w[u] = __shfl_sync(FULL, w_l, t & 31);
#pragma unroll
          for (int k = 0; k < VPL; ++k) x[u][k] = zero4();
          if (t < n) {
            const float* row = row_ptr<const float>(m, id);
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
              const int v = v0 + gl + k * G;
              if (v < nv) x[u][k] = load_row4(row, 4 * v, dim);
            }
          }
        }
#pragma unroll
        for (int u = 0; u < EMB_INFLIGHT; ++u)
          if (t0 + u * NG + grp < n) {
#pragma unroll
            for (int k = 0; k < VPL; ++k) fma4(acc[k], w[u], x[u][k]);
          }
      }
    }
    for (int o = G; o < 32; o <<= 1) {
#pragma unroll
      for (int k = 0; k < VPL; ++k) {
        acc[k].x += __shfl_xor_sync(FULL, acc[k].x, o);
        acc[k].y += __shfl_xor_sync(FULL, acc[k].y, o);
        acc[k].z += __shfl_xor_sync(FULL, acc[k].z, o);
        acc[k].w += __shfl_xor_sync(FULL, acc[k].w, o);
      }
    }
    if (mean && hi > lo) {
      const float n = (float)(hi - lo);
#pragma unroll
      for (int k = 0; k < VPL; ++k) { acc[k].x /= n; acc[k].y /= n; acc[k].z /= n; acc[k].w /= n; }
    }
    if (grp == 0) {
#pragma unroll
      for (int k = 0; k < VPL; ++k) {
        const int v = v0 + gl + k * G;
        if (v < nv) *reinterpret_cast<float4*>(out + 4 * v) = acc[k];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward
// chunk c of the sorted keys: the positions [c0, c1) of the segment [s0, s1) that holds one table's keys, whose
// chunks are numbered from cb
struct EmbChunk {
  int64_t s0, s1, cb, c, c0, c1;
};

// the starts of runs of keys below `bound` among the sorted positions [c0, c1), on every lane. Keys >= bound (rows
// that are not pushed) sort after all others, so leaving them out changes no other run's rank
MVB_DEVINL int64_t emb_count_runs(const int64_t* __restrict__ sid, int64_t c0, int64_t c1, int64_t bound) {
  const int lane = threadIdx.x & 31;
  int64_t n = 0;
  for (int64_t i0 = c0; i0 < c1; i0 += 32) {
    const int64_t i = i0 + lane;
    n += __popc(__ballot_sync(FULL, i < c1 && run_start(sid, i) && sid[i] < bound));
  }
  return n;
}

// the first key not pushed of a table whose pushed rows are [0, push_rows) (push_rows <= 0: every row is)
__host__ __device__ __forceinline__ int64_t emb_push_bound(int64_t key_base, int64_t push_rows) {
  return push_rows > 0 ? key_base + push_rows : INT64_MAX;
}

// in place: cnt[0..n) -> exclusive scan, cnt[n] = total; returns the total. One CTA of 1024 threads.
MVB_DEVINL int64_t emb_block_scan(int64_t* __restrict__ cnt, int64_t n) {
  __shared__ int64_t part[1024];
  const int64_t per = (n + 1023) / 1024;
  const int64_t lo = (int64_t)threadIdx.x * per, hi = lo + per < n ? lo + per : n;
  int64_t c = 0;
  for (int64_t i = lo; i < hi; ++i) c += cnt[i];
  part[threadIdx.x] = c;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const int64_t t = threadIdx.x >= o ? part[threadIdx.x - o] : 0;
    __syncthreads();
    part[threadIdx.x] += t;
    __syncthreads();
  }
  int64_t pos = part[threadIdx.x] - c;
  for (int64_t i = lo; i < hi; ++i) {
    const int64_t x = cnt[i];
    cnt[i] = pos;
    pos += x;
  }
  if (threadIdx.x == 1023) cnt[n] = part[1023];
  return part[1023];
}

// the epilogue of unique row id for the vectors v0 + lane + 32 k of this lane: push into the row of id, or compact:
// scale * g to grads[goff ..) and id to uniq[uoff]
template <int VPL>
MVB_DEVINL void emb_epilogue(bool push, const MvbRowMap& m, int64_t id, float* grads, int64_t goff, int64_t* uniq,
                             int64_t uoff, int dim, float scale, int v0, const float4* g) {
  const int nv = (dim + 3) >> 2, lane = threadIdx.x & 31;
  if (push) {
    float* row = row_ptr<float>(m, id);
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      const int v = v0 + lane + 32 * k;
      if (v >= nv) continue;
      float4 x = g[k];
      x.x *= scale; x.y *= scale; x.z *= scale; x.w *= scale;
      const int c = 4 * v;
      if (c + 4 <= dim) {
        red_add_v4_f32(row + c, x);
      } else {                                     // never touch the pitch padding
        red_add_f32(row + c, x.x);
        if (c + 1 < dim) red_add_f32(row + c + 1, x.y);
        if (c + 2 < dim) red_add_f32(row + c + 2, x.z);
      }
    }
  } else {
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      const int v = v0 + lane + 32 * k;
      if (v >= nv) continue;
      float4 x = g[k];
      x.x *= scale; x.y *= scale; x.z *= scale; x.w *= scale;
      *reinterpret_cast<float4*>(grads + goff + 4 * v) = x;
    }
    if (v0 == 0 && lane == 0) uniq[uoff] = id;
  }
}

// the runs of chunk k.c. Lookup i of the chunk is position perm[i] of bag g = bag_of(offsets, NB, perm[i]), its dout
// row starts at dout + drow(g). base[c] is the rank of chunk c's first run start among the unique keys; epi(key, u,
// v0, acc) is the epilogue of a whole run, part + 2 ldp c receives the pieces of the runs that cross chunk c's first
// and last boundaries.
template <int VPL, class Drow, class Epi>
MVB_DEVINL void emb_run_sum(const int64_t* __restrict__ sid, const int64_t* __restrict__ perm,
                            const int64_t* __restrict__ offsets, int64_t NB, int64_t L,
                            const float* __restrict__ psw, bool mean, const float* dout, Drow drow, int dim,
                            const EmbChunk& k, const int64_t* __restrict__ base, float* part, int ldp, Epi epi) {
  const int lane = threadIdx.x & 31, nv = (dim + 3) >> 2;
  const int64_t s0 = k.s0, s1 = k.s1, c = k.c, c0 = k.c0, c1 = k.c1;
  const bool head_continues = c0 > s0 && sid[c0 - 1] == sid[c0];
  const bool tail_continues = c1 < s1 && sid[c1] == sid[c1 - 1];
  for (int v0 = 0; v0 < nv; v0 += 32 * VPL) {       // column slabs (one slab up to dim = 512)
    float4 acc[VPL];
#pragma unroll
    for (int k = 0; k < VPL; ++k) acc[k] = zero4();
    int64_t cur = -1, seg = c0, u = base[c] - 1;
    auto flush = [&](int64_t end) {                  // segment [seg, end) of key cur
      const bool whole = (seg > c0 || !head_continues) && (end < c1 || !tail_continues);
      if (whole) {
        epi(cur, u, v0, acc);
      } else {
        float* p = part + (c * 2 + (seg == c0 ? 0 : 1)) * ldp;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
          const int v = v0 + lane + 32 * k;
          if (v < nv) *reinterpret_cast<float4*>(p + 4 * v) = acc[k];
        }
      }
    };
    for (int64_t i0 = c0; i0 < c1; i0 += 32) {
      const int64_t i = i0 + lane;
      const int n = c1 - i0 < 32 ? (int)(c1 - i0) : 32;
      int64_t id_l = -1, drow_l = 0;
      float sc_l = 0.f;
      if (i < c1) {
        id_l = sid[i];
        const int64_t p = perm[i];
        const int64_t g = bag_of(offsets, NB, p);
        drow_l = drow(g);
        sc_l = psw ? __ldg(psw + p) : 1.f;
        if (mean) sc_l /= (float)bag_len(offsets, NB, L, g);
      }
      for (int t = 0; t < n; t += EMB_INFLIGHT) {
        float4 x[EMB_INFLIGHT][VPL];
#pragma unroll
        for (int q = 0; q < EMB_INFLIGHT; ++q) {
          const int64_t dr = __shfl_sync(FULL, drow_l, (t + q) & 31);
#pragma unroll
          for (int k = 0; k < VPL; ++k) {
            const int v = v0 + lane + 32 * k;
            x[q][k] = (t + q < n && v < nv) ? f4(ld_nc_v4(dout + dr + 4 * v)) : zero4();
          }
        }
#pragma unroll
        for (int q = 0; q < EMB_INFLIGHT; ++q) {
          const int64_t id = __shfl_sync(FULL, id_l, (t + q) & 31);
          const float sc = __shfl_sync(FULL, sc_l, (t + q) & 31);
          if (t + q >= n) continue;                  // warp-uniform
          if (id != cur) {
            if (cur >= 0) flush(i0 + t + q);
            cur = id;
            seg = i0 + t + q;
            if (seg > c0 || !head_continues) ++u;
#pragma unroll
            for (int k = 0; k < VPL; ++k) acc[k] = zero4();
          }
#pragma unroll
          for (int k = 0; k < VPL; ++k) fma4(acc[k], sc, x[q][k]);
        }
      }
    }
    if (cur >= 0) flush(c1);
  }
}

// the run that crosses the last boundary of chunk k.c, if it starts in the chunk: its pieces summed in chunk order,
// then epi(key, u, v0, acc) with u = base[c + 1] - 1, the rank of the run among the unique keys. part + 2 ldp cc
// holds chunk cc's pieces.
template <int VPL, class Epi>
MVB_DEVINL void emb_merge_run(const int64_t* __restrict__ sid, const EmbChunk& k, const int64_t* __restrict__ base,
                              const float* part, int ldp, int nv, Epi epi) {
  const int lane = threadIdx.x & 31;
  const int64_t s0 = k.s0, s1 = k.s1, c = k.c, c0 = k.c0, c1 = k.c1;
  const int64_t id = sid[c1 - 1];
  if (c1 >= s1 || sid[c1] != id) return;                     // the chunk's last run ends in it
  if (c0 > s0 && sid[c0 - 1] == id) return;                  // ... or started in an earlier chunk
  int64_t lo = c1, hi = s1;                                   // end of the run: first sorted index past it
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (sid[mid] == id) lo = mid + 1; else hi = mid;
  }
  const int64_t c_last = k.cb + (lo - 1 - s0) / EMB_CHUNK;
  const int64_t u = base[c + 1] - 1;
  const float* first = part + (c * 2 + (sid[c0] == id ? 0 : 1)) * ldp;
  for (int v0 = 0; v0 < nv; v0 += 32 * VPL) {
    float4 acc[VPL];
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      const int v = v0 + lane + 32 * k;
      acc[k] = v < nv ? *reinterpret_cast<const float4*>(first + 4 * v) : zero4();
    }
    for (int64_t cc = c + 1; cc <= c_last; cc += EMB_INFLIGHT) {
      float4 x[EMB_INFLIGHT][VPL];
#pragma unroll
      for (int q = 0; q < EMB_INFLIGHT; ++q) {
        const float* p = part + (cc + q) * 2 * ldp;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
          const int v = v0 + lane + 32 * k;
          x[q][k] = (cc + q <= c_last && v < nv) ? *reinterpret_cast<const float4*>(p + 4 * v) : zero4();
        }
      }
#pragma unroll
      for (int q = 0; q < EMB_INFLIGHT; ++q)
        if (cc + q <= c_last) {
#pragma unroll
          for (int k = 0; k < VPL; ++k) add4(acc[k], x[q][k]);
        }
    }
    epi(id, u, v0, acc);
  }
}

// ------------------------------------------------------------------------------------------------ psw grad
// <d[0 .. dim), row[0 .. dim)> on every lane
MVB_DEVINL float emb_psw_dot(const float* row, const float* d, int dim) {
  const int lane = threadIdx.x & 31, nv = (dim + 3) >> 2;
  float dot = 0.f;
  for (int v = lane; v < nv; v += 32) {
    const float4 w = load_row4(row, 4 * v, dim);
    const float4 g = f4(ld_nc_v4(d + 4 * v));
    dot = fmaf(w.x, g.x, dot); dot = fmaf(w.y, g.y, dot);
    dot = fmaf(w.z, g.z, dot); dot = fmaf(w.w, g.w, dot);
  }
  return warp_sum(dot);
}

}  // namespace
