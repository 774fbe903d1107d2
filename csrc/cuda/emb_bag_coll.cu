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
//            first lookup, and the runs are summed and merged by emb_run_sum / emb_merge_run, as in emb_bag.cu;
//            a lookup's dout columns are those of its feature. A table's gradient therefore depends only on its own
//            lookups and equals one mvb_embedding_bag_bwd over its features' bags stacked in feature order.
//              push     red.add.v4.f32 of scale * g into the owner's row (default / sgd tables)
//              compact  table t's grads[u] = scale * g, uniq[u] = id, u = rank among t's unique ids
//            a table's rows >= its push_rows get no epilogue and are not counted (see emb_bag.cu)
//  psw_grad  dpsw_j = s_bag * <dout[bag(j), feature columns], W_table[ids_j, :dim]>, one warp per lookup.
// The algorithms live in emb_bag.cuh and are the ones emb_bag.cu runs; the kernels here find each bag's table and
// output columns and each chunk's table segment, and pass them on.
#include "emb_bag.cuh"

namespace {

// ------------------------------------------------------------------------------------------------ forward
// flat bags of the nf features class_feats[k0 .. k0 + nf), all of register class VPL
template <int VPL>
__global__ void __launch_bounds__(256)
emb_coll_fwd_kernel(const __grid_constant__ MvbEmbColl a, int k0, int nf) {
  const int64_t FB = (int64_t)a.F * a.B;
  for (int64_t w = warp_id(); w < (int64_t)nf * a.B; w += num_warps()) {
    const int f = __ldg(a.class_feats + k0 + w / a.B);
    const int64_t b = w % a.B, gb = (int64_t)f * a.B + b;
    const MvbEmbFeature* ft = a.features + f;
    const MvbEmbTable* tb = a.tables + ft->table;
    const int dim = (int)tb->dim;
    const int64_t lo = a.offsets[gb], hi = gb + 1 < FB ? a.offsets[gb + 1] : a.L;
    emb_pool_bag<VPL>(tb->wmap, dim, emb_lane_group_log((dim + 3) >> 2), a.ids, a.psw, lo, hi, tb->mean,
                      a.out + b * a.ldo + ft->col);
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

// chunk c < cb[T]: its table t and its place in the table's segment of the sorted keys
MVB_DEVINL EmbChunk chunk_of(const MvbEmbColl& a, const CollScratch& s, int64_t c, int& t) {
  t = (int)bag_of(s.cb, a.T, c);
  const int64_t s0 = s.seg[t], s1 = s.seg[t + 1], c0 = s0 + (c - s.cb[t]) * EMB_CHUNK;
  return EmbChunk{s0, s1, s.cb[t], c, c0, c0 + EMB_CHUNK < s1 ? c0 + EMB_CHUNK : s1};
}

__global__ void __launch_bounds__(256)
emb_coll_count_kernel(const __grid_constant__ MvbEmbColl a, CollScratch s, int64_t ncmax) {
  const int64_t nc = s.cb[a.T];
  for (int64_t c = warp_id(); c < ncmax; c += num_warps()) {
    int64_t n = 0;
    if (c < nc) {
      int t;
      const EmbChunk k = chunk_of(a, s, c, t);
      const MvbEmbTable* tb = a.tables + t;
      n = emb_count_runs(a.skeys, k.c0, k.c1, emb_push_bound(tb->key_base, tb->push_rows));
    }
    if ((threadIdx.x & 31) == 0) s.base[c] = n;
  }
}

// in place: base[0..n) -> exclusive scan, base[n] = total (one CTA); then the per-table info
__global__ void __launch_bounds__(1024)
emb_coll_scan_kernel(const __grid_constant__ MvbEmbColl a, CollScratch s, int64_t n) {
  int64_t* cnt = s.base;
  emb_block_scan(cnt, n);
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

// the epilogue of unique key u of table t; its compact rows start at info[4 t + 2] of grads, info[4 t + 3] of uniq.
// Rows >= the table's push_rows get none
template <int VPL>
struct CollEpilogue {
  const MvbEmbColl& a;
  const MvbEmbTable* tb;
  int t;
  MVB_DEVINL void operator()(int64_t key, int64_t u, int v0, const float4* g) const {
    if (key >= emb_push_bound(tb->key_base, tb->push_rows)) return;
    const bool push = tb->epilogue == MVB_EMB_PUSH;
    if (!push && (!a.grads || !a.uniq)) return;      // no compact destination: nothing to write
    const int64_t* in = a.info + 4 * t;
    const int64_t r = u - in[1];
    emb_epilogue<VPL>(push, tb->wmap, key - tb->key_base, a.grads, in[2] + r * tb->ldg, a.uniq, in[3] + r,
                      (int)tb->dim, tb->scale, v0, g);
  }
};

template <int VPL>
__global__ void __launch_bounds__(256)
emb_coll_bwd_main_kernel(const __grid_constant__ MvbEmbColl a, CollScratch s) {
  const int64_t FB = (int64_t)a.F * a.B;
  const int64_t nc = s.cb[a.T];
  for (int64_t c = warp_id(); c < nc; c += num_warps()) {
    int t;
    const EmbChunk k = chunk_of(a, s, c, t);
    const MvbEmbTable* tb = a.tables + t;
    if (emb_vpl(tb->dim) != VPL || tb->epilogue == MVB_EMB_NO_PUSH) continue;
    auto drow = [&](int64_t g) {                     // bag b of feature f: row b of dout, the feature's columns
      const int64_t f = g / a.B;
      return (g - f * a.B) * a.ldd + a.features[f].col;
    };
    emb_run_sum<VPL>(a.skeys, a.perm, a.offsets, FB, a.L, a.psw, tb->mean, a.dout, drow, (int)tb->dim, k, s.base,
                     s.part, s.ldp, CollEpilogue<VPL>{a, tb, t});
  }
}

// the runs that cross chunk boundaries of their table's segment, summed in chunk order
template <int VPL>
__global__ void __launch_bounds__(256)
emb_coll_bwd_merge_kernel(const __grid_constant__ MvbEmbColl a, CollScratch s) {
  const int64_t nc = s.cb[a.T];
  for (int64_t c = warp_id(); c < nc; c += num_warps()) {
    int t;
    const EmbChunk k = chunk_of(a, s, c, t);
    const MvbEmbTable* tb = a.tables + t;
    if (emb_vpl(tb->dim) != VPL || tb->epilogue == MVB_EMB_NO_PUSH) continue;
    emb_merge_run<VPL>(a.skeys, k, s.base, s.part, s.ldp, ((int)tb->dim + 3) >> 2, CollEpilogue<VPL>{a, tb, t});
  }
}

// ------------------------------------------------------------------------------------------------ psw grad
__global__ void __launch_bounds__(256)
emb_coll_psw_grad_kernel(const __grid_constant__ MvbEmbColl a) {
  const int64_t FB = (int64_t)a.F * a.B;
  for (int64_t j = warp_id(); j < a.L; j += num_warps()) {
    const int64_t g = bag_of(a.offsets, FB, j), f = g / a.B;
    const MvbEmbFeature* ft = a.features + f;
    const MvbEmbTable* tb = a.tables + ft->table;
    const float dot = emb_psw_dot(row_ptr<const float>(tb->wmap, __ldg(a.ids + j)), a.dout + (g - f * a.B) * a.ldd + ft->col,
                                  (int)tb->dim);
    if ((threadIdx.x & 31) == 0) a.dpsw[j] = tb->mean ? dot / (float)bag_len(a.offsets, FB, a.L, g) : dot;
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
    with_vpl(k, [&](auto V) { emb_coll_fwd_kernel<decltype(V)::value><<<grid, 256, 0, st>>>(*a, k0, nf); });
    MVB_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}

extern "C" int64_t mvb_emb_coll_scratch_bytes(int64_t L, int T, int64_t max_dim) {
  return plan_bytes(T) + cbase_bytes(L, T) + cpart_bytes(L, T, emb_vpl(max_dim));
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
    if (int rc = with_vpl(k, [&](auto V) {
          emb_coll_bwd_main_kernel<decltype(V)::value><<<grid, 256, 0, st>>>(*a, s);
          MVB_CUDA_CHECK(cudaGetLastError());
          emb_coll_bwd_merge_kernel<decltype(V)::value><<<grid, 256, 0, st>>>(*a, s);
          MVB_CUDA_CHECK(cudaGetLastError());
          return 0;
        }))
      return rc;
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
