// multiverso-b200 :: embedding-bag lookup over a row-sharded fp32 MatrixTable.
//
//  fwd       out[b] = sum (or mean) over the lookups j of bag b of psw_j * W[ids_j, :dim]. One warp per bag,
//            rows read with ld.global.nc 128-bit loads straight from their owners' shards, summed in fp32
//            registers and written once. For dim < 128 the warp splits into lane groups that each take a
//            lookup; 4 lookups per group are in flight. Group g sums the lookups g, g + NG, g + 2 NG, ... of
//            its bag in order and the groups are combined by a fixed butterfly, so the summation order
//            depends only on positions within the bag and on dim: never on the grid or the shard layout.
//  bwd       the lookups arrive sorted by (id, position). The sorted list is cut into chunks of
//            EMB_CHUNK; one warp per chunk sums psw_j * s_bag * dout[bag(j)] over each run of equal ids in
//            ascending position (bag(j) by binary search over offsets). A run that lies inside its chunk
//            goes straight to the epilogue; the pieces of a run that crosses chunk boundaries go to
//            scratch and a second pass sums them in chunk order. Every unique id gets exactly one epilogue:
//              push     red.add.v4.f32 of scale * g into the owner's row (default / sgd updaters)
//              compact  grads[u] = scale * g, uniq[u] = id, u = rank of the id among the unique ids
//  psw_grad  dpsw_j = s_bag * <dout[bag(j)], W[ids_j, :dim]>, one warp per lookup.
#include "emb_bag.cuh"

namespace {

// ------------------------------------------------------------------------------------------------ forward
template <int VPL>
__global__ void __launch_bounds__(256)
emb_fwd_kernel(const __grid_constant__ EbMap m, const __grid_constant__ MvbEmbBag a, int lg) {
  const int G = 1 << lg, NG = 32 >> lg;                // lane groups of G lanes, NG groups per warp
  const int lane = threadIdx.x & 31, grp = lane >> lg, gl = lane & (G - 1);
  const int dim = (int)a.dim, nv = (dim + 3) >> 2;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t b = warp; b < a.B; b += nwarps) {
    const int64_t lo = a.offsets[b], hi = b + 1 < a.B ? a.offsets[b + 1] : a.L;
    for (int v0 = 0; v0 < nv; v0 += G * VPL) {      // column slabs (one slab up to dim = 512)
      float4 acc[VPL];
#pragma unroll
      for (int k = 0; k < VPL; ++k) acc[k] = zero4();
      for (int64_t w0 = lo; w0 < hi; w0 += 32) {     // windows of 32 lookups: ids and weights by one load per lane
        const int n = hi - w0 < 32 ? (int)(hi - w0) : 32;
        const int64_t id_l = lane < n ? __ldg(a.ids + w0 + lane) : 0;
        const float w_l = lane < n ? (a.psw ? __ldg(a.psw + w0 + lane) : 1.f) : 0.f;
        for (int t0 = 0; t0 < n; t0 += EMB_INFLIGHT * NG) {
          float4 x[EMB_INFLIGHT][VPL];
          float w[EMB_INFLIGHT];
#pragma unroll
          for (int u = 0; u < EMB_INFLIGHT; ++u) {
            const int t = t0 + u * NG + grp;           // group grp takes the lookups grp, grp + NG, ...
            const int64_t id = __shfl_sync(FULL, id_l, t & 31);
            w[u] = __shfl_sync(FULL, w_l, t & 31);
#pragma unroll
            for (int k = 0; k < VPL; ++k) x[u][k] = zero4();
            if (t < n) {
              const float* row = row_of(m, id);
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
      if (a.mean && hi > lo) {
        const float n = (float)(hi - lo);
#pragma unroll
        for (int k = 0; k < VPL; ++k) { acc[k].x /= n; acc[k].y /= n; acc[k].z /= n; acc[k].w /= n; }
      }
      if (grp == 0) {
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
          const int v = v0 + gl + k * G;
          if (v < nv) *reinterpret_cast<float4*>(a.out + b * a.ldo + 4 * v) = acc[k];
        }
      }
    }
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

__global__ void __launch_bounds__(256)
emb_bwd_count_kernel(const int64_t* __restrict__ sid, int64_t L, int64_t* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = warp; c * EMB_CHUNK < L; c += nwarps) {
    const int64_t c0 = c * EMB_CHUNK, c1 = c0 + EMB_CHUNK < L ? c0 + EMB_CHUNK : L;
    int64_t n = 0;
    for (int64_t i0 = c0; i0 < c1; i0 += 32) {
      const int64_t i = i0 + lane;
      n += __popc(__ballot_sync(FULL, i < c1 && run_start(sid, i)));
    }
    if (lane == 0) cnt[c] = n;
  }
}

// in place: cnt[0..n) -> exclusive scan, cnt[n] = total, *total_out = total (one CTA)
__global__ void __launch_bounds__(1024)
emb_bwd_scan_kernel(int64_t* __restrict__ cnt, int64_t n, int64_t* __restrict__ total_out) {
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
  if (threadIdx.x == 1023) {
    cnt[n] = part[1023];
    if (total_out) *total_out = part[1023];
  }
}

// the epilogue of one unique id for the vectors v0 + lane + 32 k of this lane
template <int VPL>
MVB_DEVINL void bwd_epilogue(const EbMap& m, const MvbEmbBag& a, int64_t id, int64_t u, int v0, const float4* g) {
  const int dim = (int)a.dim, nv = (dim + 3) >> 2, lane = threadIdx.x & 31;
  if (a.epilogue == MVB_EMB_PUSH) {
    float* row = row_of(m, id);
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      const int v = v0 + lane + 32 * k;
      if (v >= nv) continue;
      float4 x = g[k];
      x.x *= a.scale; x.y *= a.scale; x.z *= a.scale; x.w *= a.scale;
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
      x.x *= a.scale; x.y *= a.scale; x.z *= a.scale; x.w *= a.scale;
      *reinterpret_cast<float4*>(a.grads + u * a.ldg + 4 * v) = x;
    }
    if (v0 == 0 && lane == 0) a.uniq[u] = id;
  }
}

template <int VPL>
__global__ void __launch_bounds__(256)
emb_bwd_main_kernel(const __grid_constant__ EbMap m, const __grid_constant__ MvbEmbBag a, BwdScratch s) {
  const int lane = threadIdx.x & 31;
  const int dim = (int)a.dim, nv = (dim + 3) >> 2, ldp = 4 * nv;
  const int64_t* __restrict__ sid = a.ids;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = warp; c * EMB_CHUNK < a.L; c += nwarps) {
    const int64_t c0 = c * EMB_CHUNK, c1 = c0 + EMB_CHUNK < a.L ? c0 + EMB_CHUNK : a.L;
    const bool head_continues = c0 > 0 && sid[c0 - 1] == sid[c0];
    const bool tail_continues = c1 < a.L && sid[c1] == sid[c1 - 1];
    for (int v0 = 0; v0 < nv; v0 += 32 * VPL) {     // column slabs (one slab up to dim = 512)
      float4 acc[VPL];
#pragma unroll
      for (int k = 0; k < VPL; ++k) acc[k] = zero4();
      int64_t cur = -1, seg = c0, u = s.base[c] - 1;
      auto flush = [&](int64_t end) {                // segment [seg, end) of id cur
        const bool whole = (seg > c0 || !head_continues) && (end < c1 || !tail_continues);
        if (whole) {
          bwd_epilogue<VPL>(m, a, cur, u, v0, acc);
        } else {
          float* p = s.part + (c * 2 + (seg == c0 ? 0 : 1)) * ldp;
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
        int64_t id_l = -1, bag_l = 0;
        float sc_l = 0.f;
        if (i < c1) {
          id_l = sid[i];
          const int64_t p = a.perm[i];
          bag_l = bag_of(a.offsets, a.B, p);
          sc_l = a.psw ? __ldg(a.psw + p) : 1.f;
          if (a.mean) sc_l /= (float)bag_len(a.offsets, a.B, a.L, bag_l);
        }
        for (int t = 0; t < n; t += EMB_INFLIGHT) {
          float4 x[EMB_INFLIGHT][VPL];
#pragma unroll
          for (int q = 0; q < EMB_INFLIGHT; ++q) {
            const int64_t bag = __shfl_sync(FULL, bag_l, (t + q) & 31);
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
              const int v = v0 + lane + 32 * k;
              x[q][k] = (t + q < n && v < nv) ? f4(ld_nc_v4(a.dout + bag * a.ldd + 4 * v)) : zero4();
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
}

// the runs that cross chunk boundaries: summed in chunk order by the warp of the chunk they start in
template <int VPL>
__global__ void __launch_bounds__(256)
emb_bwd_merge_kernel(const __grid_constant__ EbMap m, const __grid_constant__ MvbEmbBag a, BwdScratch s) {
  const int lane = threadIdx.x & 31;
  const int dim = (int)a.dim, nv = (dim + 3) >> 2, ldp = 4 * nv;
  const int64_t* __restrict__ sid = a.ids;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c = warp; c * EMB_CHUNK < a.L; c += nwarps) {
    const int64_t c0 = c * EMB_CHUNK, c1 = c0 + EMB_CHUNK < a.L ? c0 + EMB_CHUNK : a.L;
    const int64_t id = sid[c1 - 1];
    if (c1 >= a.L || sid[c1] != id) continue;               // the chunk's last run ends in it
    if (c0 > 0 && sid[c0 - 1] == id) continue;              // ... or started in an earlier chunk
    int64_t lo = c1, hi = a.L;                               // end of the run: first sorted index past it
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (sid[mid] == id) lo = mid + 1; else hi = mid;
    }
    const int64_t c_last = (lo - 1) / EMB_CHUNK;
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
      bwd_epilogue<VPL>(m, a, id, u, v0, acc);
    }
  }
}

// ------------------------------------------------------------------------------------------------ psw grad
__global__ void __launch_bounds__(256)
emb_psw_grad_kernel(const __grid_constant__ EbMap m, const __grid_constant__ MvbEmbBag a) {
  const int lane = threadIdx.x & 31;
  const int dim = (int)a.dim, nv = (dim + 3) >> 2;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t j = warp; j < a.L; j += nwarps) {
    const int64_t b = bag_of(a.offsets, a.B, j);
    const float* row = row_of(m, __ldg(a.ids + j));
    const float* d = a.dout + b * a.ldd;
    float dot = 0.f;
    for (int v = lane; v < nv; v += 32) {
      const float4 w = load_row4(row, 4 * v, dim);
      const float4 g = f4(ld_nc_v4(d + 4 * v));
      dot = fmaf(w.x, g.x, dot); dot = fmaf(w.y, g.y, dot);
      dot = fmaf(w.z, g.z, dot); dot = fmaf(w.w, g.w, dot);
    }
    dot = warp_sum(dot);
    if (lane == 0) a.dpsw[j] = a.mean ? dot / (float)bag_len(a.offsets, a.B, a.L, b) : dot;
  }
}

int check_common(const MvbEmbBag* a, bool need_out) {
  const MvbRowMap& wm = a->wmap;
  if (wm.nservers < 1 || wm.nservers > MVB_MAX_RANKS || wm.rows_per_server < 1) return -50;
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
  const EbMap m = to_map(a->wmap);
  const int nv = (int)((a->dim + 3) / 4);
  int lg = 0;
  while ((1 << lg) < nv && lg < 5) ++lg;
  const int vpl = (nv + (1 << lg) - 1) >> lg;
  const int grid = grid_for(a->B);
  cudaStream_t st = (cudaStream_t)stream;
  if (vpl <= 1) emb_fwd_kernel<1><<<grid, 256, 0, st>>>(m, *a, lg);
  else if (vpl == 2) emb_fwd_kernel<2><<<grid, 256, 0, st>>>(m, *a, lg);
  else if (vpl == 3) emb_fwd_kernel<3><<<grid, 256, 0, st>>>(m, *a, lg);
  else emb_fwd_kernel<4><<<grid, 256, 0, st>>>(m, *a, lg);
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
  const EbMap m = to_map(a->wmap);
  const BwdScratch s = scratch_of(*a);
  const int64_t nch = n_chunks(a->L);
  const int grid = grid_for(nch);
  emb_bwd_count_kernel<<<grid, 256, 0, st>>>(a->ids, a->L, s.base);
  MVB_CUDA_CHECK(cudaGetLastError());
  emb_bwd_scan_kernel<<<1, 1024, 0, st>>>(s.base, nch, a->n_unique);
  MVB_CUDA_CHECK(cudaGetLastError());
  if (count_only) return 0;
  const int nv = (int)((a->dim + 3) / 4);
  const int vpl = nv <= 32 ? 1 : nv <= 64 ? 2 : nv <= 96 ? 3 : 4;
#define MVB_EMB_BWD(V)                                                   \
  do {                                                                   \
    emb_bwd_main_kernel<V><<<grid, 256, 0, st>>>(m, *a, s);              \
    MVB_CUDA_CHECK(cudaGetLastError());                                  \
    emb_bwd_merge_kernel<V><<<grid, 256, 0, st>>>(m, *a, s);             \
  } while (0)
  if (vpl == 1) MVB_EMB_BWD(1);
  else if (vpl == 2) MVB_EMB_BWD(2);
  else if (vpl == 3) MVB_EMB_BWD(3);
  else MVB_EMB_BWD(4);
#undef MVB_EMB_BWD
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int mvb_embedding_bag_psw_grad(const MvbEmbBag* a, void* stream) {
  if (int rc = check_common(a, false)) return rc;
  if (a->L == 0) return 0;
  if (int rc = check_dout(a)) return rc;
  if (!a->dpsw) return -59;
  emb_psw_grad_kernel<<<grid_for(a->L), 256, 0, (cudaStream_t)stream>>>(to_map(a->wmap), *a);
  MVB_CUDA_CHECK(cudaGetLastError());
  return 0;
}
