// multiverso-b200 :: embedding-bag lookup over a row-sharded fp32 MatrixTable.
//
//  fwd       out[b] = sum (or mean) over the lookups j of bag b of psw_j * W[ids_j, :dim]. One warp per bag,
//            rows read with ld.global.nc 128-bit loads straight from their owners' shards, summed in fp32
//            registers and written once; the summation order depends only on positions within the bag and on
//            dim, never on the grid or the shard layout. Dims above 512 are pooled in column slabs.
//  bwd       the lookups arrive sorted by (id, position): one segment [0, L) cut into chunks of EMB_CHUNK, one
//            warp per chunk. count + scan rank the unique ids, main sums each run of equal ids, merge sums the
//            runs that cross chunk boundaries in chunk order. Every unique id gets exactly one epilogue:
//              push     red.add.v4.f32 of scale * g into the owner's row (default / sgd updaters)
//              compact  grads[u] = scale * g, uniq[u] = id, u = rank of the id among the unique ids
//            with push_rows > 0, ids >= push_rows (the zero row of a hash table with admission) get none and are
//            not counted; they sort last, so every other id's rank, chunk and summation order stay as they were.
//  psw_grad  dpsw_j = s_bag * <dout[bag(j)], W[ids_j, :dim]>, one warp per lookup.
// The algorithms live in emb_bag.cuh, shared with the collection (emb_bag_coll.cu); the kernels here are the
// grid-stride loops over bags, chunks and lookups of one table.
#include "emb_bag.cuh"

namespace {

// ------------------------------------------------------------------------------------------------ forward
template <int VPL>
__global__ void __launch_bounds__(256)
emb_fwd_kernel(const __grid_constant__ MvbEmbBag a, int lg) {
  for (int64_t b = warp_id(); b < a.B; b += num_warps()) {
    const int64_t lo = a.offsets[b], hi = b + 1 < a.B ? a.offsets[b + 1] : a.L;
    emb_pool_bag<VPL>(a.wmap, (int)a.dim, lg, a.ids, a.psw, lo, hi, a.mean, a.out + b * a.ldo);
  }
}

// ------------------------------------------------------------------------------------------------ backward
struct BwdScratch {
  int64_t* base;   // [nch + 1]: unique ids before chunk c (exclusive scan of the run starts)
  float* part;     // [nch][2][4 nv]: slot 0 = piece of the run holding the chunk's first lookup, slot 1 = last
};

int64_t n_chunks(int64_t L) { return (L + EMB_CHUNK - 1) / EMB_CHUNK; }
int64_t base_bytes(int64_t L) { return ((n_chunks(L) + 1) * 8 + 255) / 256 * 256; }
int64_t part_bytes(int64_t L, int64_t dim) { return n_chunks(L) * 2 * ((dim + 3) / 4 * 4) * 4; }

BwdScratch scratch_of(const MvbEmbBag& a) {
  BwdScratch s;
  s.base = (int64_t*)a.scratch;
  s.part = (float*)((char*)a.scratch + base_bytes(a.L));
  return s;
}

// chunk c of the one segment [0, L)
MVB_DEVINL EmbChunk chunk_of(int64_t c, int64_t L) {
  return EmbChunk{0, L, 0, c, c * EMB_CHUNK, (c + 1) * EMB_CHUNK < L ? (c + 1) * EMB_CHUNK : L};
}

__global__ void __launch_bounds__(256)
emb_bwd_count_kernel(const int64_t* __restrict__ sid, int64_t L, int64_t bound, int64_t* __restrict__ cnt) {
  for (int64_t c = warp_id(); c * EMB_CHUNK < L; c += num_warps()) {
    const EmbChunk k = chunk_of(c, L);
    const int64_t n = emb_count_runs(sid, k.c0, k.c1, bound);
    if ((threadIdx.x & 31) == 0) cnt[c] = n;
  }
}

// in place: cnt[0..n) -> exclusive scan, cnt[n] = total, *total_out = total (one CTA)
__global__ void __launch_bounds__(1024)
emb_bwd_scan_kernel(int64_t* __restrict__ cnt, int64_t n, int64_t* __restrict__ total_out) {
  const int64_t total = emb_block_scan(cnt, n);
  if (threadIdx.x == 1023 && total_out) *total_out = total;
}

// the epilogue of unique id u of the table; rows >= push_rows get none
template <int VPL>
struct BwdEpilogue {
  const MvbEmbBag& a;
  MVB_DEVINL void operator()(int64_t id, int64_t u, int v0, const float4* g) const {
    if (id >= emb_push_bound(0, a.push_rows)) return;
    emb_epilogue<VPL>(a.epilogue == MVB_EMB_PUSH, a.wmap, id, a.grads, u * a.ldg, a.uniq, u, (int)a.dim, a.scale, v0,
                      g);
  }
};

template <int VPL>
__global__ void __launch_bounds__(256)
emb_bwd_main_kernel(const __grid_constant__ MvbEmbBag a, BwdScratch s) {
  const int ldp = 4 * (((int)a.dim + 3) >> 2);
  const int64_t ldd = a.ldd;
  for (int64_t c = warp_id(); c * EMB_CHUNK < a.L; c += num_warps())
    emb_run_sum<VPL>(a.ids, a.perm, a.offsets, a.B, a.L, a.psw, a.mean, a.dout, [ldd](int64_t b) { return b * ldd; },
                     (int)a.dim, chunk_of(c, a.L), s.base, s.part, ldp, BwdEpilogue<VPL>{a});
}

// the runs that cross chunk boundaries: summed in chunk order by the warp of the chunk they start in
template <int VPL>
__global__ void __launch_bounds__(256)
emb_bwd_merge_kernel(const __grid_constant__ MvbEmbBag a, BwdScratch s) {
  const int nv = ((int)a.dim + 3) >> 2;
  for (int64_t c = warp_id(); c * EMB_CHUNK < a.L; c += num_warps())
    emb_merge_run<VPL>(a.ids, chunk_of(c, a.L), s.base, s.part, 4 * nv, nv, BwdEpilogue<VPL>{a});
}

// ------------------------------------------------------------------------------------------------ psw grad
__global__ void __launch_bounds__(256)
emb_psw_grad_kernel(const __grid_constant__ MvbEmbBag a) {
  for (int64_t j = warp_id(); j < a.L; j += num_warps()) {
    const int64_t b = bag_of(a.offsets, a.B, j);
    const float dot = emb_psw_dot(row_ptr<const float>(a.wmap, __ldg(a.ids + j)), a.dout + b * a.ldd, (int)a.dim);
    if ((threadIdx.x & 31) == 0) a.dpsw[j] = a.mean ? dot / (float)bag_len(a.offsets, a.B, a.L, b) : dot;
  }
}

int check_common(const MvbEmbBag* a, bool need_out) {
  const MvbRowMap& wm = a->wmap;
  if (!row_split_ok(wm.nservers, wm.rows_per_server)) return -50;
  if (wm.num_col % 4 != 0) return -51;
  if (a->dim < 1 || a->dim > wm.num_col) return -52;
  if (a->L < 0 || a->B < 0 || (a->B > 0 && !a->offsets)) return -53;
  if (need_out && (a->ldo % 4 != 0 || a->ldo < (a->dim + 3) / 4 * 4 || ((uintptr_t)a->out & 15))) return -54;
  return 0;
}

int check_dout(const MvbEmbBag* a) {
  if (a->ldd % 4 != 0 || a->ldd < (a->dim + 3) / 4 * 4 || ((uintptr_t)a->dout & 15)) return -55;
  return 0;
}

}  // namespace

extern "C" int mvb_embedding_bag_fwd(const MvbEmbBag* a, void* stream) {
  if (int rc = check_common(a, true)) return rc;
  if (a->B == 0) return 0;
  const int lg = emb_lane_group_log((int)((a->dim + 3) / 4));
  const int grid = grid_for(a->B);
  cudaStream_t st = (cudaStream_t)stream;
  with_vpl(emb_vpl(a->dim), [&](auto V) { emb_fwd_kernel<decltype(V)::value><<<grid, 256, 0, st>>>(*a, lg); });
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int64_t mvb_embedding_bag_scratch_bytes(int64_t L, int64_t dim) {
  return base_bytes(L) + part_bytes(L, dim);
}

extern "C" int mvb_embedding_bag_bwd(const MvbEmbBag* a, void* stream) {
  if (int rc = check_common(a, false)) return rc;
  if (a->L == 0) {
    return a->n_unique ? (int)cudaMemsetAsync(a->n_unique, 0, 8, (cudaStream_t)stream) : 0;
  }
  if (int rc = check_dout(a)) return rc;
  if (!a->ids || !a->perm || a->scratch_bytes < mvb_embedding_bag_scratch_bytes(a->L, a->dim)) return -56;
  const bool compact = a->epilogue == MVB_EMB_COMPACT;
  if (!compact && a->epilogue != MVB_EMB_PUSH) return -57;
  const bool count_only = compact && !a->grads;
  if (compact && !count_only && (!a->uniq || a->ldg % 4 != 0 || a->ldg < (a->dim + 3) / 4 * 4 ||
                                 ((uintptr_t)a->grads & 15)))
    return -58;
  cudaStream_t st = (cudaStream_t)stream;
  const BwdScratch s = scratch_of(*a);
  const int64_t nch = n_chunks(a->L);
  const int grid = grid_for(nch);
  emb_bwd_count_kernel<<<grid, 256, 0, st>>>(a->ids, a->L, emb_push_bound(0, a->push_rows), s.base);
  MVB_CUDA_CHECK(cudaGetLastError());
  emb_bwd_scan_kernel<<<1, 1024, 0, st>>>(s.base, nch, a->n_unique);
  MVB_CUDA_CHECK(cudaGetLastError());
  if (count_only) return 0;
  return with_vpl(emb_vpl(a->dim), [&](auto V) {
    emb_bwd_main_kernel<decltype(V)::value><<<grid, 256, 0, st>>>(*a, s);
    MVB_CUDA_CHECK(cudaGetLastError());
    emb_bwd_merge_kernel<decltype(V)::value><<<grid, 256, 0, st>>>(*a, s);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  });
}

extern "C" int mvb_embedding_bag_psw_grad(const MvbEmbBag* a, void* stream) {
  if (int rc = check_common(a, false)) return rc;
  if (a->L == 0) return 0;
  if (int rc = check_dout(a)) return rc;
  if (!a->dpsw) return -59;
  emb_psw_grad_kernel<<<grid_for(a->L), 256, 0, (cudaStream_t)stream>>>(*a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
