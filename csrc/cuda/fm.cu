// multiverso-b200 :: factorization machine over a row-sharded fp32 MatrixTable
// (multiverso_b200/ops/factorization_machine.py).
//
// Row r holds the k = C - 1 factors v_r = W[r, 0:k] and the linear weight w_r = W[r, k]. Bag b holds the lookups j
// with ids i_j and values x_j:
//
//   S_b = sum_j x_j W[i_j, :]     q_b = sum_j x_j^2 |v_{i_j}|^2     y_b = S_b[k] + (|S_b[:k]|^2 - q_b) / 2
//
//  fwd   one warp per bag over a grid-stride loop: the gather-pool of emb_pool_bag (lane groups, 4 lookups in flight
//        per group, 16-byte ld.global.nc loads from the owners' shards, groups combined by a fixed butterfly), so
//        S_b is bitwise embedding_bag(W, ids, offsets, per_sample_weights=x). Each lane also sums x^2 |v|^2 over
//        its factor columns; y_b is one warp sum of the lanes' shares. With sp set the kernel writes S'_b, S_b
//        with column k set to 1 (the dout row of the backward). Nothing lookups x C is written; every sum has a
//        fixed order, so y and S' are bitwise reproducible and the same for every sharding.
//  bwd   dL/dW[r] = sum over the lookups j of row r of g_b x_j (S'_b - x_j v'_r) (v'_r: v_r with 0 in column k).
//        The pipeline of mvb_embedding_bag_bwd: lookups sorted by (id, position), count + scan rank the unique
//        ids, the run-sum below sums (g_b x_j) S'_b over each run piece of a chunk together with the scalar
//        c = sum (g_b x_j) x_j, and corrects the piece by -c v'_r (row r read once per piece) before it goes to
//        the epilogue or to scratch. The correction is linear, so emb_merge_run sums the corrected pieces of a
//        run that crosses chunks unchanged. Epilogue: red.add (default / sgd) or the compact rows.
#include "emb_bag.cuh"

namespace {

// the sum of squares of the columns [c, c + 4) of x that are below k (the factor columns)
MVB_DEVINL float sq_factors(float4 x, int c, int k) {
  if (c + 4 <= k) {
    float p = x.x * x.x;
    p = fmaf(x.y, x.y, p); p = fmaf(x.z, x.z, p); p = fmaf(x.w, x.w, p);
    return p;
  }
  float p = 0.f;
  if (c < k) p = x.x * x.x;
  if (c + 1 < k) p = fmaf(x.y, x.y, p);
  if (c + 2 < k) p = fmaf(x.z, x.z, p);
  return p;
}

// column k of the vector holding columns [c, c + 4), if it does
MVB_DEVINL float col_of(float4 x, int c, int k) {
  return c == k ? x.x : c + 1 == k ? x.y : c + 2 == k ? x.z : c + 3 == k ? x.w : 0.f;
}

// ------------------------------------------------------------------------------------------------ forward
// bag b: S in the lane groups of 1 << lg lanes exactly as emb_pool_bag sums it, plus the lane's share of q
template <int VPL>
__global__ void __launch_bounds__(256)
fm_fwd_kernel(const __grid_constant__ MvbFm a, int lg) {
  const int G = 1 << lg, NG = 32 >> lg;
  const int lane = threadIdx.x & 31, grp = lane >> lg, gl = lane & (G - 1);
  const int dim = (int)a.dim, kc = dim - 1, nv = (dim + 3) >> 2;
  for (int64_t b = warp_id(); b < a.B; b += num_warps()) {
    const int64_t lo = a.offsets[b], hi = b + 1 < a.B ? a.offsets[b + 1] : a.L;
    float q = 0.f, ss = 0.f, lin = 0.f;                // lane shares of q, |s|^2 and S[k]
    for (int v0 = 0; v0 < nv; v0 += G * VPL) {       // column slabs (one slab up to C = 512)
      float4 acc[VPL];
#pragma unroll
      for (int k = 0; k < VPL; ++k) acc[k] = zero4();
      for (int64_t w0 = lo; w0 < hi; w0 += 32) {
        const int n = hi - w0 < 32 ? (int)(hi - w0) : 32;
        const int64_t id_l = lane < n ? __ldg(a.ids + w0 + lane) : 0;
        const float w_l = lane < n ? (a.values ? __ldg(a.values + w0 + lane) : 1.f) : 0.f;
        for (int t0 = 0; t0 < n; t0 += EMB_INFLIGHT * NG) {
          float4 x[EMB_INFLIGHT][VPL];
          float w[EMB_INFLIGHT];
#pragma unroll
          for (int u = 0; u < EMB_INFLIGHT; ++u) {
            const int t = t0 + u * NG + grp;
            const int64_t id = __shfl_sync(FULL, id_l, t & 31);
            w[u] = __shfl_sync(FULL, w_l, t & 31);
#pragma unroll
            for (int k = 0; k < VPL; ++k) x[u][k] = zero4();
            if (t < n) {
              const float* row = row_ptr<const float>(a.wmap, id);
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
              float p = 0.f;
#pragma unroll
              for (int k = 0; k < VPL; ++k) {
                fma4(acc[k], w[u], x[u][k]);
                p += sq_factors(x[u][k], 4 * (v0 + gl + k * G), kc);
              }
              q = fmaf(w[u] * w[u], p, q);
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
      if (grp == 0) {                                // every group holds S now; group 0 takes its columns
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
          const int v = v0 + gl + k * G;
          if (v >= nv) continue;
          ss += sq_factors(acc[k], 4 * v, kc);
          lin += col_of(acc[k], 4 * v, kc);
          if (a.sp) {
            float4 s = acc[k];
            if (4 * v + 4 > kc) {                      // column k of S' is 1
              if (4 * v == kc) s.x = 1.f; else if (4 * v + 1 == kc) s.y = 1.f;
              else if (4 * v + 2 == kc) s.z = 1.f; else s.w = 1.f;
            }
            *reinterpret_cast<float4*>(a.sp + b * a.lds + 4 * v) = s;
          }
        }
      }
    }
    q = warp_sum(q);
    ss = warp_sum(ss);
    lin = warp_sum(lin);                               // one lane holds S[k], the others 0: exact
    if (lane == 0) a.y[b] = lin + 0.5f * (ss - q);
  }
}

// ------------------------------------------------------------------------------------------------ backward
// scratch: the layout of mvb_embedding_bag_scratch_bytes(L, C): base [nch + 1] int64 padded to 256 bytes, then
// part [nch][2][round4(C)] floats
int64_t n_chunks(int64_t L) { return (L + EMB_CHUNK - 1) / EMB_CHUNK; }
int64_t base_bytes(int64_t L) { return ((n_chunks(L) + 1) * 8 + 255) / 256 * 256; }

MVB_DEVINL EmbChunk chunk_of(int64_t c, int64_t L) {
  return EmbChunk{0, L, 0, c, c * EMB_CHUNK, (c + 1) * EMB_CHUNK < L ? (c + 1) * EMB_CHUNK : L};
}

__global__ void __launch_bounds__(256)
fm_bwd_count_kernel(const int64_t* __restrict__ sid, int64_t L, int64_t bound, int64_t* __restrict__ cnt) {
  for (int64_t c = warp_id(); c * EMB_CHUNK < L; c += num_warps()) {
    const EmbChunk k = chunk_of(c, L);
    const int64_t n = emb_count_runs(sid, k.c0, k.c1, bound);
    if ((threadIdx.x & 31) == 0) cnt[c] = n;
  }
}

__global__ void __launch_bounds__(1024)
fm_bwd_scan_kernel(int64_t* __restrict__ cnt, int64_t n, int64_t* __restrict__ total_out) {
  const int64_t total = emb_block_scan(cnt, n);
  if (threadIdx.x == 1023 && total_out) *total_out = total;
}

template <int VPL>
struct FmEpilogue {
  const MvbFm& a;
  MVB_DEVINL void operator()(int64_t id, int64_t u, int v0, const float4* g) const {
    if (id >= emb_push_bound(0, a.push_rows)) return;
    emb_epilogue<VPL>(a.epilogue == MVB_EMB_PUSH, a.wmap, id, a.grads, u * a.ldg, a.uniq, u, (int)a.dim, a.scale, v0,
                      g);
  }
};

// the runs of chunk k of the sorted ids, as emb_run_sum sums them with the weight g_b x_j over the dout row S'_b,
// each piece corrected by -c v'_r before the epilogue (a whole run) or scratch (a piece of a run that crosses a
// chunk boundary)
template <int VPL>
MVB_DEVINL void fm_run_sum(const MvbFm& a, const EmbChunk& k, const int64_t* __restrict__ base, float* part,
                           int ldp) {
  const int lane = threadIdx.x & 31, dim = (int)a.dim, kc = dim - 1, nv = (dim + 3) >> 2;
  const int64_t* __restrict__ sid = a.ids;
  const int64_t s0 = k.s0, s1 = k.s1, c = k.c, c0 = k.c0, c1 = k.c1;
  const bool head_continues = c0 > s0 && sid[c0 - 1] == sid[c0];
  const bool tail_continues = c1 < s1 && sid[c1] == sid[c1 - 1];
  const FmEpilogue<VPL> epi{a};
  for (int v0 = 0; v0 < nv; v0 += 32 * VPL) {
    float4 acc[VPL];
#pragma unroll
    for (int k = 0; k < VPL; ++k) acc[k] = zero4();
    float cs = 0.f;                                    // c of the current piece, the same in every lane
    int64_t cur = -1, seg = c0, u = base[c] - 1;
    auto flush = [&](int64_t end) {                    // piece [seg, end) of row cur
      const float* row = row_ptr<const float>(a.wmap, cur);
#pragma unroll
      for (int k = 0; k < VPL; ++k) {
        const int v = v0 + lane + 32 * k;
        if (v < nv) fma4(acc[k], -cs, load_row4(row, 4 * v, kc));
      }
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
      float sc_l = 0.f, cx_l = 0.f;
      if (i < c1) {
        id_l = sid[i];
        const int64_t p = a.perm[i];
        const int64_t g = bag_of(a.offsets, a.B, p);
        drow_l = g * a.lds;
        const float x = a.values ? __ldg(a.values + p) : 1.f;
        sc_l = __ldg(a.dy + g) * x;
        cx_l = sc_l * x;
      }
      for (int t = 0; t < n; t += EMB_INFLIGHT) {
        float4 x[EMB_INFLIGHT][VPL];
#pragma unroll
        for (int q = 0; q < EMB_INFLIGHT; ++q) {
          const int64_t dr = __shfl_sync(FULL, drow_l, (t + q) & 31);
#pragma unroll
          for (int k = 0; k < VPL; ++k) {
            const int v = v0 + lane + 32 * k;
            x[q][k] = (t + q < n && v < nv) ? f4(ld_nc_v4(a.sp + dr + 4 * v)) : zero4();
          }
        }
#pragma unroll
        for (int q = 0; q < EMB_INFLIGHT; ++q) {
          const int64_t id = __shfl_sync(FULL, id_l, (t + q) & 31);
          const float sc = __shfl_sync(FULL, sc_l, (t + q) & 31);
          const float cx = __shfl_sync(FULL, cx_l, (t + q) & 31);
          if (t + q >= n) continue;                    // warp-uniform
          if (id != cur) {
            if (cur >= 0) flush(i0 + t + q);
            cur = id;
            seg = i0 + t + q;
            if (seg > c0 || !head_continues) ++u;
#pragma unroll
            for (int k = 0; k < VPL; ++k) acc[k] = zero4();
            cs = 0.f;
          }
#pragma unroll
          for (int k = 0; k < VPL; ++k) fma4(acc[k], sc, x[q][k]);
          cs += cx;
        }
      }
    }
    if (cur >= 0) flush(c1);
  }
}

template <int VPL>
__global__ void __launch_bounds__(256)
fm_bwd_main_kernel(const __grid_constant__ MvbFm a, int64_t* base, float* part) {
  const int ldp = 4 * (((int)a.dim + 3) >> 2);
  for (int64_t c = warp_id(); c * EMB_CHUNK < a.L; c += num_warps())
    fm_run_sum<VPL>(a, chunk_of(c, a.L), base, part, ldp);
}

template <int VPL>
__global__ void __launch_bounds__(256)
fm_bwd_merge_kernel(const __grid_constant__ MvbFm a, const int64_t* base, const float* part) {
  const int nv = ((int)a.dim + 3) >> 2;
  for (int64_t c = warp_id(); c * EMB_CHUNK < a.L; c += num_warps())
    emb_merge_run<VPL>(a.ids, chunk_of(c, a.L), base, part, 4 * nv, nv, FmEpilogue<VPL>{a});
}

// errors shared by both entry points
int check_common(const MvbFm* a) {
  const MvbRowMap& m = a->wmap;
  if (!row_split_ok(m.nservers, m.rows_per_server)) return MVB_BAD_ROW_MAP;
  if (a->dim < 2 || a->dim > MVB_FM_MAX_DIM || a->dim > m.num_col || m.num_col % 4 != 0) return -90;
  for (int s = 0; s < m.nservers; ++s)
    if ((uintptr_t)m.shard_ptrs[s] & 15) return -90;
  if (a->B < 0 || a->L < 0 || (a->B > 0 && !a->offsets) || (a->L > 0 && !a->ids)) return -91;
  return 0;
}

bool bad_sp(const MvbFm* a) { return !a->sp || a->lds % 4 != 0 || a->lds < (a->dim + 3) / 4 * 4 || ((uintptr_t)a->sp & 15); }

}  // namespace

extern "C" int mvb_fm_fwd(const MvbFm* a, void* stream) {
  if (int rc = check_common(a)) return rc;
  if ((a->B > 0 && !a->y) || (a->sp && bad_sp(a))) return -92;
  if (a->B == 0) return 0;
  const int lg = emb_lane_group_log((int)((a->dim + 3) / 4));
  const int grid = grid_for(a->B);
  cudaStream_t st = (cudaStream_t)stream;
  with_vpl(emb_vpl(a->dim), [&](auto V) { fm_fwd_kernel<decltype(V)::value><<<grid, 256, 0, st>>>(*a, lg); });
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_fm_bwd(const MvbFm* a, void* stream) {
  if (int rc = check_common(a)) return rc;
  if (a->L > 0 && (!a->dy || !a->perm || bad_sp(a) || !a->scratch ||
                   a->scratch_bytes < mvb_embedding_bag_scratch_bytes(a->L, a->dim)))
    return -93;
  const bool compact = a->epilogue == MVB_EMB_COMPACT;
  if (!compact && a->epilogue != MVB_EMB_PUSH) return -94;
  const bool count_only = compact && !a->grads;
  if (compact && !count_only && (!a->uniq || a->ldg % 4 != 0 || a->ldg < (a->dim + 3) / 4 * 4 ||
                                 ((uintptr_t)a->grads & 15)))
    return -94;
  if (a->L == 0) {
    return a->n_unique ? (int)cudaMemsetAsync(a->n_unique, 0, 8, (cudaStream_t)stream) : 0;
  }
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* base = (int64_t*)a->scratch;
  float* part = (float*)((char*)a->scratch + base_bytes(a->L));
  const int64_t nch = n_chunks(a->L);
  const int grid = grid_for(nch);
  fm_bwd_count_kernel<<<grid, 256, 0, st>>>(a->ids, a->L, emb_push_bound(0, a->push_rows), base);
  MVB_CUDA_CHECK(cudaGetLastError());
  fm_bwd_scan_kernel<<<1, 1024, 0, st>>>(base, nch, a->n_unique);
  MVB_CUDA_CHECK(cudaGetLastError());
  if (count_only) return 0;
  return with_vpl(emb_vpl(a->dim), [&](auto V) {
    fm_bwd_main_kernel<decltype(V)::value><<<grid, 256, 0, st>>>(*a, base, part);
    MVB_CUDA_CHECK(cudaGetLastError());
    fm_bwd_merge_kernel<decltype(V)::value><<<grid, 256, 0, st>>>(*a, base, part);
    MVB_CUDA_CHECK(cudaGetLastError());
    return 0;
  });
}
