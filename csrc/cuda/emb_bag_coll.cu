// multiverso-b200 :: embedding-bag collection: F sparse features over T row-sharded fp32 MatrixTables in one call.
//
//  layout    ids holds feature 0's lookups for bags 0..B-1, then feature 1's, ...; offsets is the exclusive scan
//            of the [F x B] lengths, so bag b of feature f is the flat bag g = f B + b. The table / feature
//            descriptors are a device array built once: no call passes them by value, so T and F are not capped.
//  fwd       one warp per flat bag, exactly the lane groups, in-flight lookups and summation order that
//            emb_fwd_kernel uses for the table's dim, so each feature's columns equal mvb_embedding_bag_fwd over
//            its table bit for bit. One launch per register class (1..4 float4 per lane) present.
//  bwd       keys key_base[table] + id, sorted with their positions: each table becomes one contiguous segment
//            ordered by (id, position). Every segment is cut into its own chunks of EMB_CHUNK starting at its
//            first lookup, and the runs are summed and merged as emb_bwd_main / emb_bwd_merge do; a lookup's
//            dout columns are those of its feature. A table's gradient therefore depends only on its own lookups
//            and equals one mvb_embedding_bag_bwd over its features' bags stacked in feature order.
//              push     red.add.v4.f32 of scale * g into the owner's row (default / sgd tables)
//              compact  table t's grads[u] = scale * g, uniq[u] = id, u = rank among t's unique ids
//  psw_grad  dpsw_j = s_bag * <dout[bag(j), feature columns], W_table[ids_j, :dim]>, one warp per lookup.
#include "emb_bag.cuh"

namespace {

// float4 vectors per lane of a dim: emb_fwd_kernel's and emb_bwd_*'s template argument
MVB_DEVINL int vpl_of(int nv) { return nv <= 32 ? 1 : (nv + 31) >> 5; }
int vpl_of_host(int64_t dim) {
  const int64_t nv = (dim + 3) / 4;
  return nv <= 32 ? 1 : (int)((nv + 31) / 32);
}

// row r of a table: the address row_of gives for the same row map
MVB_DEVINL float* trow(const MvbEmbTable* t, int64_t r) {
  const int64_t rps = t->wmap.rows_per_server;
  int64_t o = r / rps;
  if (o > t->wmap.nservers - 1) o = t->wmap.nservers - 1;
  return (float*)t->wmap.shard_ptrs[o] + (r - o * rps) * t->wmap.num_col;
}

// ------------------------------------------------------------------------------------------------ forward
// flat bags of the nf features class_feats[k0 .. k0 + nf), all of register class VPL
template <int VPL>
__global__ void __launch_bounds__(256)
emb_coll_fwd_kernel(const __grid_constant__ MvbEmbColl a, int k0, int nf) {
  const int lane = threadIdx.x & 31;
  const int64_t FB = (int64_t)a.F * a.B;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = warp; w < (int64_t)nf * a.B; w += nwarps) {
    const int f = __ldg(a.class_feats + k0 + w / a.B);
    const int64_t b = w % a.B, gb = (int64_t)f * a.B + b;
    const MvbEmbFeature* ft = a.features + f;
    const MvbEmbTable* tb = a.tables + ft->table;
    const int dim = (int)tb->dim, nv = (dim + 3) >> 2;
    int lg = 0;                                      // the lane groups mvb_embedding_bag_fwd picks for dim
    while ((1 << lg) < nv && lg < 5) ++lg;
    const int G = 1 << lg, NG = 32 >> lg;
    const int grp = lane >> lg, gl = lane & (G - 1);
    const int64_t lo = a.offsets[gb], hi = gb + 1 < FB ? a.offsets[gb + 1] : a.L;
    float* out = a.out + b * a.ldo + ft->col;
    for (int v0 = 0; v0 < nv; v0 += G * VPL) {
      float4 acc[VPL];
#pragma unroll
      for (int k = 0; k < VPL; ++k) acc[k] = zero4();
      for (int64_t w0 = lo; w0 < hi; w0 += 32) {
        const int n = hi - w0 < 32 ? (int)(hi - w0) : 32;
        const int64_t id_l = lane < n ? __ldg(a.ids + w0 + lane) : 0;
        const float w_l = lane < n ? (a.psw ? __ldg(a.psw + w0 + lane) : 1.f) : 0.f;
        for (int t0 = 0; t0 < n; t0 += EMB_INFLIGHT * NG) {
          float4 x[EMB_INFLIGHT][VPL];
          float wt[EMB_INFLIGHT];
#pragma unroll
          for (int u = 0; u < EMB_INFLIGHT; ++u) {
            const int t = t0 + u * NG + grp;
            const int64_t id = __shfl_sync(FULL, id_l, t & 31);
            wt[u] = __shfl_sync(FULL, w_l, t & 31);
#pragma unroll
            for (int k = 0; k < VPL; ++k) x[u][k] = zero4();
            if (t < n) {
              const float* row = trow(tb, id);
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
              for (int k = 0; k < VPL; ++k) fma4(acc[k], wt[u], x[u][k]);
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
      if (tb->mean && hi > lo) {
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
}

// ------------------------------------------------------------------------------------------------ backward
// scratch: seg[T + 1] (first sorted position of each table's segment), cb[T + 1] (first chunk of each table),
// base[ncmax + 1] (unique keys before chunk c), part[ncmax][2][ldp] (pieces of runs that cross chunks)
struct CollScratch {
  int64_t* seg;
  int64_t* cb;
  int64_t* base;
  float* part;
  int ldp;
};

int64_t r256(int64_t b) { return (b + 255) / 256 * 256; }
int64_t nc_max(int64_t L, int T) { return (L + EMB_CHUNK - 1) / EMB_CHUNK + T; }
int64_t plan_bytes(int T) { return r256((int64_t)(2 * T + 2) * 8); }
int64_t cbase_bytes(int64_t L, int T) { return r256((nc_max(L, T) + 1) * 8); }
int64_t cpart_bytes(int64_t L, int T, int vpl) { return nc_max(L, T) * 2 * 128 * vpl * 4; }

CollScratch coll_scratch(const MvbEmbColl& a, int vpl) {
  CollScratch s;
  s.seg = (int64_t*)a.scratch;
  s.cb = s.seg + a.T + 1;
  s.base = (int64_t*)((char*)a.scratch + plan_bytes(a.T));
  s.part = (float*)((char*)s.base + cbase_bytes(a.L, a.T));
  s.ldp = 128 * vpl;
  return s;
}

// keys of every lookup; block 0 also lays out the table segments of the sorted keys and their chunks
__global__ void __launch_bounds__(256)
emb_coll_keys_kernel(const __grid_constant__ MvbEmbColl a, CollScratch s) {
  const int64_t FB = (int64_t)a.F * a.B;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    for (int t = 0; t <= a.T; ++t) s.seg[t] = 0;
    for (int f = 0; f < a.F; ++f) {
      const int64_t lo = a.offsets[(int64_t)f * a.B];
      const int64_t hi = f + 1 < a.F ? a.offsets[(int64_t)(f + 1) * a.B] : a.L;
      s.seg[a.features[f].table + 1] += hi - lo;
    }
    s.cb[0] = 0;
    for (int t = 0; t < a.T; ++t) {
      s.cb[t + 1] = s.cb[t] + (s.seg[t + 1] + EMB_CHUNK - 1) / EMB_CHUNK;
      s.seg[t + 1] += s.seg[t];
    }
  }
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < a.L; j += (int64_t)gridDim.x * blockDim.x) {
    const int64_t f = bag_of(a.offsets, FB, j) / a.B;
    a.keys[j] = a.tables[a.features[f].table].key_base + __ldg(a.ids + j);
  }
}

// the sorted positions [c0, c1) of chunk c < cb[T] and its table
struct Chunk {
  int t;
  int64_t s1, c0, c1;
};
MVB_DEVINL Chunk chunk_of(const MvbEmbColl& a, const CollScratch& s, int64_t c) {
  Chunk k;
  k.t = (int)bag_of(s.cb, a.T, c);
  k.s1 = s.seg[k.t + 1];
  k.c0 = s.seg[k.t] + (c - s.cb[k.t]) * EMB_CHUNK;
  k.c1 = k.c0 + EMB_CHUNK < k.s1 ? k.c0 + EMB_CHUNK : k.s1;
  return k;
}

__global__ void __launch_bounds__(256)
emb_coll_count_kernel(const __grid_constant__ MvbEmbColl a, CollScratch s, int64_t ncmax) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t nc = s.cb[a.T];
  for (int64_t c = warp; c < ncmax; c += nwarps) {
    int64_t n = 0;
    if (c < nc) {
      const Chunk k = chunk_of(a, s, c);
      for (int64_t i0 = k.c0; i0 < k.c1; i0 += 32) {
        const int64_t i = i0 + lane;
        n += __popc(__ballot_sync(FULL, i < k.c1 && run_start(a.skeys, i)));
      }
    }
    if (lane == 0) s.base[c] = n;
  }
}

// in place: base[0..n) -> exclusive scan, base[n] = total (one CTA); then the per-table info
__global__ void __launch_bounds__(1024)
emb_coll_scan_kernel(const __grid_constant__ MvbEmbColl a, CollScratch s, int64_t n) {
  __shared__ int64_t part[1024];
  int64_t* cnt = s.base;
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
  __syncthreads();
  if (threadIdx.x == 0) {                            // {U, first unique, grads offset, uniq offset} per table
    int64_t g = 0, q = 0;
    for (int t = 0; t < a.T; ++t) {
      const int64_t u0 = cnt[s.cb[t]], U = cnt[s.cb[t + 1]] - u0;
      int64_t* in = a.info + 4 * t;
      in[0] = U; in[1] = u0; in[2] = g; in[3] = q;
      if (a.tables[t].epilogue == MVB_EMB_COMPACT) { g += U * a.tables[t].ldg; q += U; }
    }
    a.info[4 * a.T] = g;
    a.info[4 * a.T + 1] = q;
  }
}

// the epilogue of one unique key of table tb for the vectors v0 + lane + 32 k of this lane
template <int VPL>
MVB_DEVINL void coll_epilogue(const MvbEmbColl& a, const MvbEmbTable* tb, int t, int64_t key, int64_t u, int v0,
                              const float4* g) {
  const int dim = (int)tb->dim, nv = (dim + 3) >> 2, lane = threadIdx.x & 31;
  const int64_t id = key - tb->key_base;
  const float scale = tb->scale;
  if (tb->epilogue == MVB_EMB_PUSH) {
    float* row = trow(tb, id);
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
  } else if (a.grads && a.uniq) {
    const int64_t* in = a.info + 4 * t;
    const int64_t r = u - in[1];
    float* gr = a.grads + in[2] + r * tb->ldg;
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      const int v = v0 + lane + 32 * k;
      if (v >= nv) continue;
      float4 x = g[k];
      x.x *= scale; x.y *= scale; x.z *= scale; x.w *= scale;
      *reinterpret_cast<float4*>(gr + 4 * v) = x;
    }
    if (v0 == 0 && lane == 0) a.uniq[in[3] + r] = id;
  }
}

template <int VPL>
__global__ void __launch_bounds__(256)
emb_coll_bwd_main_kernel(const __grid_constant__ MvbEmbColl a, CollScratch s) {
  const int lane = threadIdx.x & 31;
  const int ldp = s.ldp;
  const int64_t* __restrict__ sid = a.skeys;
  const int64_t FB = (int64_t)a.F * a.B;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t nc = s.cb[a.T];
  for (int64_t c = warp; c < nc; c += nwarps) {
    const Chunk ch = chunk_of(a, s, c);
    const MvbEmbTable* tb = a.tables + ch.t;
    const int dim = (int)tb->dim, nv = (dim + 3) >> 2;
    if (vpl_of(nv) != VPL || tb->epilogue == MVB_EMB_NO_PUSH) continue;
    const bool mean = tb->mean;
    const int64_t c0 = ch.c0, c1 = ch.c1;
    const bool head_continues = c0 > s.seg[ch.t] && sid[c0 - 1] == sid[c0];
    const bool tail_continues = c1 < ch.s1 && sid[c1] == sid[c1 - 1];
    for (int v0 = 0; v0 < nv; v0 += 32 * VPL) {
      float4 acc[VPL];
#pragma unroll
      for (int k = 0; k < VPL; ++k) acc[k] = zero4();
      int64_t cur = -1, sg = c0, u = s.base[c] - 1;
      auto flush = [&](int64_t end) {                // segment [sg, end) of key cur
        const bool whole = (sg > c0 || !head_continues) && (end < c1 || !tail_continues);
        if (whole) {
          coll_epilogue<VPL>(a, tb, ch.t, cur, u, v0, acc);
        } else {
          float* p = s.part + (c * 2 + (sg == c0 ? 0 : 1)) * ldp;
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
          const int64_t p = a.perm[i];
          const int64_t g = bag_of(a.offsets, FB, p), f = g / a.B;
          drow_l = (g - f * a.B) * a.ldd + a.features[f].col;
          sc_l = a.psw ? __ldg(a.psw + p) : 1.f;
          if (mean) sc_l /= (float)bag_len(a.offsets, FB, a.L, g);
        }
        for (int t = 0; t < n; t += EMB_INFLIGHT) {
          float4 x[EMB_INFLIGHT][VPL];
#pragma unroll
          for (int q = 0; q < EMB_INFLIGHT; ++q) {
            const int64_t drow = __shfl_sync(FULL, drow_l, (t + q) & 31);
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
              const int v = v0 + lane + 32 * k;
              x[q][k] = (t + q < n && v < nv) ? f4(ld_nc_v4(a.dout + drow + 4 * v)) : zero4();
            }
          }
#pragma unroll
          for (int q = 0; q < EMB_INFLIGHT; ++q) {
            const int64_t id = __shfl_sync(FULL, id_l, (t + q) & 31);
            const float sc = __shfl_sync(FULL, sc_l, (t + q) & 31);
            if (t + q >= n) continue;                // warp-uniform
            if (id != cur) {
              if (cur >= 0) flush(i0 + t + q);
              cur = id;
              sg = i0 + t + q;
              if (sg > c0 || !head_continues) ++u;
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
}

// the runs that cross chunk boundaries of their table's segment, summed in chunk order
template <int VPL>
__global__ void __launch_bounds__(256)
emb_coll_bwd_merge_kernel(const __grid_constant__ MvbEmbColl a, CollScratch s) {
  const int lane = threadIdx.x & 31;
  const int ldp = s.ldp;
  const int64_t* __restrict__ sid = a.skeys;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t nc = s.cb[a.T];
  for (int64_t c = warp; c < nc; c += nwarps) {
    const Chunk ch = chunk_of(a, s, c);
    const MvbEmbTable* tb = a.tables + ch.t;
    const int nv = ((int)tb->dim + 3) >> 2;
    if (vpl_of(nv) != VPL || tb->epilogue == MVB_EMB_NO_PUSH) continue;
    const int64_t s0 = s.seg[ch.t], c0 = ch.c0, c1 = ch.c1;
    const int64_t id = sid[c1 - 1];
    if (c1 >= ch.s1 || sid[c1] != id) continue;             // the chunk's last run ends in it
    if (c0 > s0 && sid[c0 - 1] == id) continue;             // ... or started in an earlier chunk
    int64_t lo = c1, hi = ch.s1;                             // end of the run: first sorted index past it
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (sid[mid] == id) lo = mid + 1; else hi = mid;
    }
    const int64_t c_last = s.cb[ch.t] + (lo - 1 - s0) / EMB_CHUNK;
    const int64_t u = s.base[c + 1] - 1;
    const float* first = s.part + (c * 2 + (sid[c0] == id ? 0 : 1)) * ldp;
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
          const float* p = s.part + (cc + q) * 2 * ldp;
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
      coll_epilogue<VPL>(a, tb, ch.t, id, u, v0, acc);
    }
  }
}

// ------------------------------------------------------------------------------------------------ psw grad
__global__ void __launch_bounds__(256)
emb_coll_psw_grad_kernel(const __grid_constant__ MvbEmbColl a) {
  const int lane = threadIdx.x & 31;
  const int64_t FB = (int64_t)a.F * a.B;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t j = warp; j < a.L; j += nwarps) {
    const int64_t g = bag_of(a.offsets, FB, j), f = g / a.B;
    const MvbEmbFeature* ft = a.features + f;
    const MvbEmbTable* tb = a.tables + ft->table;
    const int dim = (int)tb->dim, nv = (dim + 3) >> 2;
    const float* row = trow(tb, __ldg(a.ids + j));
    const float* d = a.dout + (g - f * a.B) * a.ldd + ft->col;
    float dot = 0.f;
    for (int v = lane; v < nv; v += 32) {
      const float4 w = load_row4(row, 4 * v, dim);
      const float4 x = f4(ld_nc_v4(d + 4 * v));
      dot = fmaf(w.x, x.x, dot); dot = fmaf(w.y, x.y, dot);
      dot = fmaf(w.z, x.z, dot); dot = fmaf(w.w, x.w, dot);
    }
    dot = warp_sum(dot);
    if (lane == 0) a.dpsw[j] = tb->mean ? dot / (float)bag_len(a.offsets, FB, a.L, g) : dot;
  }
}

int check_coll(const MvbEmbColl* a) {
  if (a->T < 1 || a->F < 1 || !a->tables || !a->features || !a->class_feats) return -60;
  if (a->class_off[0] != 0 || a->class_off[4] != a->F) return -61;
  for (int k = 1; k < 5; ++k)
    if (a->class_off[k] < a->class_off[k - 1]) return -61;
  if (a->L < 0 || a->B < 0 || (a->B > 0 && !a->offsets) || (a->L > 0 && (a->B == 0 || !a->ids))) return -62;
  return 0;
}

int check_dout_coll(const MvbEmbColl* a) {
  if (!a->dout || a->ldd % 4 != 0 || ((uintptr_t)a->dout & 15)) return -63;
  return 0;
}

int max_vpl(const MvbEmbColl* a) {
  int v = 1;
  for (int k = 1; k < 5; ++k)
    if (a->class_off[k] > a->class_off[k - 1]) v = k;
  return v;
}

}  // namespace

extern "C" int mvb_emb_coll_fwd(const MvbEmbColl* a, void* stream) {
  if (int rc = check_coll(a)) return rc;
  if (a->B == 0) return 0;
  if (!a->out || a->ldo % 4 != 0 || ((uintptr_t)a->out & 15)) return -64;
  cudaStream_t st = (cudaStream_t)stream;
  for (int k = 1; k < 5; ++k) {
    const int k0 = a->class_off[k - 1], nf = a->class_off[k] - k0;
    if (nf == 0) continue;
    const int grid = grid_for((int64_t)nf * a->B);
    if (k == 1) emb_coll_fwd_kernel<1><<<grid, 256, 0, st>>>(*a, k0, nf);
    else if (k == 2) emb_coll_fwd_kernel<2><<<grid, 256, 0, st>>>(*a, k0, nf);
    else if (k == 3) emb_coll_fwd_kernel<3><<<grid, 256, 0, st>>>(*a, k0, nf);
    else emb_coll_fwd_kernel<4><<<grid, 256, 0, st>>>(*a, k0, nf);
    MVB_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}

extern "C" int64_t mvb_emb_coll_scratch_bytes(int64_t L, int T, int64_t max_dim) {
  return plan_bytes(T) + cbase_bytes(L, T) + cpart_bytes(L, T, vpl_of_host(max_dim));
}

static int check_scratch(const MvbEmbColl* a) {
  if (!a->scratch || a->scratch_bytes < plan_bytes(a->T) + cbase_bytes(a->L, a->T) + cpart_bytes(a->L, a->T, max_vpl(a)))
    return -65;
  return 0;
}

extern "C" int mvb_emb_coll_keys(const MvbEmbColl* a, void* stream) {
  if (int rc = check_coll(a)) return rc;
  if (a->L == 0) return 0;
  if (int rc = check_scratch(a)) return rc;
  if (!a->keys) return -66;
  emb_coll_keys_kernel<<<grid_for((a->L + 31) / 32), 256, 0, (cudaStream_t)stream>>>(*a, coll_scratch(*a, max_vpl(a)));
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_emb_coll_count(const MvbEmbColl* a, void* stream) {
  if (int rc = check_coll(a)) return rc;
  if (a->L == 0) return 0;
  if (int rc = check_scratch(a)) return rc;
  if (!a->skeys || !a->info) return -67;
  cudaStream_t st = (cudaStream_t)stream;
  const CollScratch s = coll_scratch(*a, max_vpl(a));
  const int64_t ncmax = nc_max(a->L, a->T);
  emb_coll_count_kernel<<<grid_for(ncmax), 256, 0, st>>>(*a, s, ncmax);
  MVB_CUDA_CHECK(cudaGetLastError());
  emb_coll_scan_kernel<<<1, 1024, 0, st>>>(*a, s, ncmax);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_emb_coll_bwd(const MvbEmbColl* a, void* stream) {
  if (int rc = check_coll(a)) return rc;
  if (a->L == 0) return 0;
  if (int rc = check_scratch(a)) return rc;
  if (int rc = check_dout_coll(a)) return rc;
  if (!a->skeys || !a->perm || !a->info) return -67;
  cudaStream_t st = (cudaStream_t)stream;
  const CollScratch s = coll_scratch(*a, max_vpl(a));
  const int grid = grid_for(nc_max(a->L, a->T));
  for (int k = 1; k < 5; ++k) {
    if (a->class_off[k] == a->class_off[k - 1]) continue;
#define MVB_COLL_BWD(V)                                                  \
  do {                                                                   \
    emb_coll_bwd_main_kernel<V><<<grid, 256, 0, st>>>(*a, s);            \
    MVB_CUDA_CHECK(cudaGetLastError());                                  \
    emb_coll_bwd_merge_kernel<V><<<grid, 256, 0, st>>>(*a, s);           \
  } while (0)
    if (k == 1) MVB_COLL_BWD(1);
    else if (k == 2) MVB_COLL_BWD(2);
    else if (k == 3) MVB_COLL_BWD(3);
    else MVB_COLL_BWD(4);
#undef MVB_COLL_BWD
    MVB_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}

extern "C" int mvb_emb_coll_psw_grad(const MvbEmbColl* a, void* stream) {
  if (int rc = check_coll(a)) return rc;
  if (a->L == 0) return 0;
  if (int rc = check_dout_coll(a)) return rc;
  if (!a->dpsw) return -68;
  emb_coll_psw_grad_kernel<<<grid_for(a->L), 256, 0, (cudaStream_t)stream>>>(*a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
